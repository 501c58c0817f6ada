// JAX-compatible random bits on the device (SURVEY §8(f) #2, the part that can be pinned without a jax install):
// threefry2x32 (the counter-based generator behind jax.random at the pinned jax 0.3.10) and
// jax.random.uniform(key, shape, float32) — what iqn/agent.py:45-50,182-190,222 uses for its tau samples.
//
//   bits = threefry_2x32(key, iota(n))   : the n counters are split into a first and a second half (zero-padded to an
//                                          even length); pair i = (ctr[i], ctr[i + half]) -> output words (i, i + half)
//   u    = bitcast<float>((bits >> 9) | 0x3F800000) - 1.0f                       in [0, 1)
//
// Known answers this file is tested against (tests/test_jax_prng.py; Random123 / jax's own test vectors and the
// values printed in the jax documentation): threefry2x32(key 0,0; ctr 0,0) = 6b200159 99ba4efe;
// (ffffffff.. ; ffffffff..) = 1cb996fc bb002be7; (13198a2e 03707344; 243f6a88 85a308d3) = c4923a9c 483df7a0;
// split(PRNGKey(0)) = [[4146024105, 967050713], [2718843009, 1272950319]]; uniform(PRNGKey(0)) = 0.41845703.
#include "dz_common.cuh"
#include "dz_threefry.cuh"

namespace dz {

namespace {

constexpr int kMaxBlocks = 4;
struct UniformJob {
  const uint32_t* keys;            // device: [nblocks][2]
  long long count[kMaxBlocks];     // floats in block b
  long long offset[kMaxBlocks];    // start of block b in `out`
  float* out;
  int nblocks;
};

__global__ void __launch_bounds__(256) jax_uniform_kernel(const UniformJob job) {
  dz::pdl_enter();
  const int b = blockIdx.y;
  const long long n = job.count[b];
  const long long half = (n + 1) >> 1;                      // counters are zero-padded to an even length
  const uint32_t k0 = job.keys[2 * b], k1 = job.keys[2 * b + 1];
  float* out = job.out + job.offset[b];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < half; i += (long long)gridDim.x * blockDim.x) {
    const long long j = i + half;
    const uint32_t c1 = j < n ? (uint32_t)j : 0u;           // the padding counter is 0
    uint32_t o0, o1;
    threefry2x32(k0, k1, (uint32_t)i, c1, &o0, &o1);
    out[i] = __uint_as_float((o0 >> 9) | 0x3F800000u) - 1.0f;
    if (j < n) out[j] = __uint_as_float((o1 >> 9) | 0x3F800000u) - 1.0f;
  }
}

}  // namespace
}  // namespace dz

using namespace dz;

extern "C" int dz_jax_uniform(const uint32_t* d_keys, const int64_t* counts, int32_t nblocks, float* d_out, void* stream) {
  if (nblocks < 1 || nblocks > kMaxBlocks) return fail(DZ_EINVAL, "dz_jax_uniform: 1..4 blocks");
  if (!d_keys || !counts || !d_out) return fail(DZ_EINVAL, "dz_jax_uniform: null argument");
  UniformJob job;
  memset(&job, 0, sizeof(job));
  job.keys = d_keys; job.out = d_out; job.nblocks = nblocks;
  long long off = 0, mx = 0;
  for (int b = 0; b < nblocks; ++b) {
    if (counts[b] < 0 || counts[b] >= (1LL << 32)) return fail(DZ_EINVAL, "dz_jax_uniform: block size must be below 2^32");
    job.count[b] = counts[b]; job.offset[b] = off;
    off += counts[b];
    mx = counts[b] > mx ? counts[b] : mx;
  }
  if (mx == 0) return DZ_OK;
  dim3 grid((unsigned)std::min<long long>(ceil_div((mx + 1) / 2, 256), kNumSMs * 8), (unsigned)nblocks);
  DZ_LAUNCH(jax_uniform_kernel, grid, 256, 0, stream, job);
  return DZ_OK;
}

// The same threefry2x32 function compiled for the host: lets the CPU test-suite check the arithmetic the kernel runs.
extern "C" int dz_test_threefry2x32(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t* out2) {
  threefry2x32(k0, k1, c0, c1, &out2[0], &out2[1]);
  return DZ_OK;
}
