// Common device/host helpers for the sgmse_b200 engine (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

namespace sgmse {

// ----------------------------------------------------------------------------------------------
// error plumbing: C-ABI never throws; everything funnels into a thread-local message + int code
// ----------------------------------------------------------------------------------------------
void set_last_error(const std::string& msg);
const char* get_last_error();

struct Error {
  std::string msg;
};

#define SG_CHECK(cond, ...)                                                        \
  do {                                                                             \
    if (!(cond)) {                                                                 \
      char _b[512];                                                                \
      snprintf(_b, sizeof(_b), __VA_ARGS__);                                       \
      throw ::sgmse::Error{std::string(__FILE__) + ":" + std::to_string(__LINE__) + ": " + _b}; \
    }                                                                              \
  } while (0)

// Pinned, device-mapped word that a kernel's bounded barrier wait writes its code into before it traps; host memory
// survives the trap, so the error message can say which wait timed out.
extern volatile int* g_wait_code_host;
#define CUDA_OK(expr)                                                              \
  do {                                                                             \
    cudaError_t _e = (expr);                                                       \
    if (_e != cudaSuccess)                                                         \
      throw ::sgmse::Error{std::string(__FILE__) + ":" + std::to_string(__LINE__) + ": " + #expr + \
                           " -> " + cudaGetErrorString(_e) +                      \
                           ((::sgmse::g_wait_code_host && *::sgmse::g_wait_code_host)                   \
                                ? " [kernel barrier wait code " + std::to_string(*::sgmse::g_wait_code_host) + "]" \
                                : std::string())};                                 \
  } while (0)

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// cudaFuncSetAttribute is per device: a launcher remembers (bit per device ordinal) where its kernel already has the
// attribute, so that engines on several devices of one process all get it.  Not a stream operation: legal during capture.
static inline bool first_use_on_device(unsigned long long& mask) {
  int dev = 0;
  CUDA_OK(cudaGetDevice(&dev));
  const unsigned long long bit = 1ull << (dev & 63);
  if (mask & bit) return false;
  mask |= bit;
  return true;
}

// ----------------------------------------------------------------------------------------------
// Programmatic dependent launch (PDL).  Compiled in only with -DSGMSE_B200_PDL (sgmse_b200/build.py --pdl builds a
// second library, libsgmse_b200_pdl.so): the default library's SASS carries none of these instructions.  Contract of
// a PDL-aware kernel: pdl_trigger() first (the next kernel of the stream may start its prologue as soon as every CTA
// of this grid is resident), then pdl_wait() in EVERY thread before the first access to global memory that an
// earlier kernel of the stream writes or reads (only weights -- constant after load_weights -- may be touched
// before it), and never an exit without it (a grid whose CTAs all left early would "complete" before its
// predecessor and break the chain for the kernel after it).
// ----------------------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_trigger() {
#ifdef SGMSE_B200_PDL
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#endif
}
__device__ __forceinline__ void pdl_wait() {
#ifdef SGMSE_B200_PDL
  asm volatile("griddepcontrol.wait;" ::: "memory");
#endif
}
#endif
extern thread_local int g_pdl;              // runtime switch (option "pdl"); refused unless the library was built with SGMSE_B200_PDL
bool pdl_compiled();

#ifdef __CUDACC__
// Launch of a PDL-aware kernel: plain <<<>>> unless g_pdl, else cudaLaunchKernelEx with the programmatic stream
// serialization attribute (captured into a CUDA graph as a programmatic dependency edge).
template <typename... P, typename... A>
inline void launch_k(void (*kern)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, A&&... args) {
  if (!g_pdl) {
    kern<<<grid, block, smem, st>>>(static_cast<P>(args)...);
    return;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  CUDA_OK(cudaLaunchKernelEx(&cfg, kern, static_cast<P>(args)...));
}
#endif

// ----------------------------------------------------------------------------------------------
// activation element types: float (exact mode) or __half (fast modes)
// ----------------------------------------------------------------------------------------------
template <typename T> struct Act;
template <> struct Act<float> {
  static __device__ __forceinline__ float ld(const float* p) { return *p; }
  static __device__ __forceinline__ void st(float* p, float v) { *p = v; }
  static __device__ __forceinline__ float rnd(float v) { return v; }       // value as it will be read back
};
template <> struct Act<__half> {
  static __device__ __forceinline__ float ld(const __half* p) { return __half2float(*p); }
  static __device__ __forceinline__ void st(__half* p, float v) { *p = __float2half_rn(v); }
  static __device__ __forceinline__ float rnd(float v) { return __half2float(__float2half_rn(v)); }
};

// 8-element vectors (16 B of half / 32 B of float)
template <typename T> struct Vec8;
template <> struct Vec8<__half> {
  uint4 raw;
  __device__ __forceinline__ void load(const __half* p) { raw = *reinterpret_cast<const uint4*>(p); }
  __device__ __forceinline__ void store(__half* p) const { *reinterpret_cast<uint4*>(p) = raw; }
  __device__ __forceinline__ void get(float (&f)[8]) const {
    const __half2* h = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 v = __half22float2(h[i]); f[2 * i] = v.x; f[2 * i + 1] = v.y; }
  }
  __device__ __forceinline__ void set(const float (&f)[8]) {
    __half2* h = reinterpret_cast<__half2*>(&raw);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  }
};
template <> struct Vec8<float> {
  float4 a, b;
  __device__ __forceinline__ void load(const float* p) {
    a = *reinterpret_cast<const float4*>(p); b = *reinterpret_cast<const float4*>(p + 4);
  }
  __device__ __forceinline__ void store(float* p) const {
    *reinterpret_cast<float4*>(p) = a; *reinterpret_cast<float4*>(p + 4) = b;
  }
  __device__ __forceinline__ void get(float (&f)[8]) const {
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  }
  __device__ __forceinline__ void set(const float (&f)[8]) {
    a = make_float4(f[0], f[1], f[2], f[3]); b = make_float4(f[4], f[5], f[6], f[7]);
  }
};

__device__ __forceinline__ float silu_f(float x) { return __fdividef(x, 1.0f + __expf(-x)); }

// FIR taps of the StyleGAN2 resampler: outer([1,3,3,1])/64 (x4 for up-sampling)
__device__ __forceinline__ float fir_tap(int i) { return (i == 0 || i == 3) ? 0.125f : 0.375f; }

#ifdef __CUDACC__
// ----------------------------------------------------------------------------------------------
// PTX wrappers (mbarrier / TMA).  Waits are bounded: a protocol bug traps instead of
// hanging the GPU.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// non-blocking probe (try_wait may suspend the thread for a while; a poller of several barriers must not)
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// try_wait with an explicit suspend-time hint: the thread sleeps (no issue slots) until the phase completes or ~ns pass
__device__ __forceinline__ bool mbar_try_wait_ns(uint64_t* bar, uint32_t parity, uint32_t ns) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"(ns)
      : "memory");
  return ok != 0;
}
// Bounded wait (~ a few seconds at most), then trap with a diagnostic code in *dbg.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int* dbg = nullptr, int code = 0) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) {
      if (dbg) atomicExch(dbg, code ? code : -1);
      __threadfence_system();
      asm volatile("trap;");
    }
  }
}

__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem, const void* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem, const void* tmap, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_4d(const void* tmap, const void* smem, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
#endif  // __CUDACC__

}  // namespace sgmse
