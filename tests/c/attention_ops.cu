// Op-level harness of tests/test_gpu_long_clips.py: launch_attention on raw device pointers, fp16 or fp32 storage, at
// any token count.  Linked, like kernel_ops.cu, against the objects sgmse_b200.build compiles for the engine library, so
// the kernels under test are the product's object code.  A launcher error returns a non-zero code; aops_last_error() has
// the message.
#include <string>

#include "kernels.h"

using namespace sgmse;

namespace {
thread_local std::string g_err;

TensorDesc desc(const void* p, int N, int S, int C, int fp32) {
  TensorDesc t;
  t.p = const_cast<void*>(p);
  t.N = N; t.H = 1; t.W = S; t.C = C;
  t.dt = fp32 ? DT_F32 : DT_F16;
  return t;
}
}  // namespace

extern "C" {

const char* aops_last_error() { return g_err.c_str(); }

// out[N][S][C] = softmax(q k^T / sqrt(C)) v over the S tokens of qkv[N][S][3C] (q | k | v), the product's kernel choice
int aops_attention(void* stream, int N, int S, int C, int fp32, const void* qkv, void* out) {
  try {
    g_attn_variant = 0;
    const TensorDesc q = desc(qkv, N, S, 3 * C, fp32);
    TensorDesc o = desc(out, N, S, C, fp32);
    launch_attention(static_cast<cudaStream_t>(stream), q, o);
    return 0;
  } catch (const sgmse::Error& e) { g_err = e.msg; return 1; }
  catch (const std::exception& e) { g_err = e.what(); return 2; }
}

}  // extern "C"
