// CUDA's own Philox4x32-10 (curand_philox4x32_x.h) compiled for the host: the known-answer oracle of the numpy Philox
// in tests/test_gpu_sampler_ops.py, which in turn checks the engine's in-kernel generator (misc.cu: philox4x32_10).
// ctr [n][4], key [n][2] -> out [n][4].
#define QUALIFIERS static inline __host__ __device__
#include <curand_philox4x32_x.h>

extern "C" void curand_philox_batch(const unsigned* ctr, const unsigned* key, unsigned* out, long long n) {
  for (long long i = 0; i < n; ++i) {
    const uint4 c = make_uint4(ctr[4 * i], ctr[4 * i + 1], ctr[4 * i + 2], ctr[4 * i + 3]);
    const uint2 k = make_uint2(key[2 * i], key[2 * i + 1]);
    const uint4 r = curand_Philox4x32_10(c, k);
    out[4 * i] = r.x; out[4 * i + 1] = r.y; out[4 * i + 2] = r.z; out[4 * i + 3] = r.w;
  }
}
