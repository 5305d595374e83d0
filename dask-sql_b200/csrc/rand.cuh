// rand.cuh — counter-based random numbers keyed on a base-table row's number.
// RAND / RANDOM / RAND_INTEGER (the reference's physical/rex/core/call.py:809-881) and TABLESAMPLE BERNOULLI
// (physical/rel/logical/sample.py) draw from Philox4x32-10 (Salmon et al., SC'11) with the 64-bit seed as key
// and the row's number in its table as counter, so a value depends on the row alone and never on how the
// table is partitioned, pruned or sharded (DESIGN.md section 3).
#pragma once
#include "common.cuh"

__device__ __forceinline__ uint4 b2_philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    if (i) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

// w0 | w1 << 32 of Philox(counter (row mod 2^32, row >> 32, site, 0), key).  Out of line, like the math
// functions of expr.cuh, so the interpreter loop does not carry the ten rounds' registers.
__device__ __noinline__ uint64_t b2_rand_u64(int64_t row, int64_t key, int site) {
  const uint64_t r = (uint64_t)row, k = (uint64_t)key;
  const uint4 w = b2_philox4x32_10(make_uint4((uint32_t)r, (uint32_t)(r >> 32), (uint32_t)site, 0u),
                                   (uint32_t)k, (uint32_t)(k >> 32));
  return (uint64_t)w.x | ((uint64_t)w.y << 32);
}

// One thread per group of four rows g = (row_base + i) >> 2: one Philox call (counter word 3 = 1) decides all
// four, row r kept iff w[r & 3] < threshold.  A group may straddle the start or end of the partition; its
// rows outside [0, n) are not written.
__global__ void __launch_bounds__(B2_BLOCK)
b2_sample_mask_kernel(int64_t n, int64_t row_base, int64_t key, int site, int64_t threshold,
                      uint8_t* __restrict__ out) {
  const int64_t g0 = row_base >> 2, ngroups = ((row_base + n - 1) >> 2) - g0 + 1;
  const uint64_t k = (uint64_t)key;
  const bool aligned = (row_base & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 3) == 0;
  for (int64_t t = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; t < ngroups; t += (int64_t)gridDim.x * B2_BLOCK) {
    const uint64_t g = (uint64_t)(g0 + t);
    uint32_t keep[4];
    if (threshold <= 0 || threshold > 0xFFFFFFFFll) {
      const uint32_t all = threshold > 0;
      keep[0] = keep[1] = keep[2] = keep[3] = all;
    } else {
      const uint4 w = b2_philox4x32_10(make_uint4((uint32_t)g, (uint32_t)(g >> 32), (uint32_t)site, 1u),
                                       (uint32_t)k, (uint32_t)(k >> 32));
      const uint32_t th = (uint32_t)threshold;
      keep[0] = w.x < th; keep[1] = w.y < th; keep[2] = w.z < th; keep[3] = w.w < th;
    }
    const int64_t lo = (int64_t)(g << 2) - row_base;          // partition index of the group's first row
    if (aligned && lo + 3 < n) {
      reinterpret_cast<uint32_t*>(out)[lo >> 2] = keep[0] | keep[1] << 8 | keep[2] << 16 | keep[3] << 24;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (lo + j >= 0 && lo + j < n) out[lo + j] = (uint8_t)keep[j];
    }
  }
}

extern "C" {

int32_t b2_sample_mask(int64_t n, int64_t row_base, int64_t key, int32_t site, int64_t threshold, uint8_t* out,
                       void* stream) {
  B2_REQUIRE(n >= 0 && row_base >= 0, "n and row_base must be >= 0");
  B2_REQUIRE(n == 0 || out, "null argument");
  B2_REQUIRE(n <= INT64_MAX - row_base, "row_base + n overflows");
  if (n == 0) return B2_OK;
  const int64_t ngroups = ((row_base + n - 1) >> 2) - (row_base >> 2) + 1;
  int grid = b2_wave_grid(b2_sample_mask_kernel, B2_BLOCK, (ngroups + B2_BLOCK - 1) / B2_BLOCK);
  b2_sample_mask_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(n, row_base, key, site, threshold, out);
  B2_CHECK_LAUNCH("b2_sample_mask_kernel");
  return B2_OK;
}

}  // extern "C"
