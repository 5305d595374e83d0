// sort.cuh — ORDER BY: stable LSD radix sort of (64-bit key image, row id) pairs.
// The reference sorts with dask's sort_values / nsmallest per partition + merge
// (dask_sql/physical/utils/sort.py:9-140); here a sort key becomes a 64-bit order-preserving image
// (sign-flipped int64, ordered float64 image, inverted for DESC) and eight 8-bit counting-sort
// passes permute (image, row id).  Multi-key ORDER BY sorts by the last key first (stability).
#pragma once
#include "common.cuh"

#define B2_SORT_BLOCK 256
#define B2_SORT_WARPS (B2_SORT_BLOCK / 32)
#define B2_SORT_ITEMS_PER_WARP 2048   // rows of one warp's contiguous sub-chunk
#define B2_SORT_CHUNK (B2_SORT_WARPS * B2_SORT_ITEMS_PER_WARP)

// image of col[src row] for the sort order; out_null[i] = 1 for NULL rows (NaN for floats)
__global__ void __launch_bounds__(B2_BLOCK)
b2_sort_image_kernel(const __grid_constant__ b2_col_t c, const int32_t* __restrict__ idx, int64_t n, int descending,
                     int nulls_first, uint64_t* __restrict__ out_img, uint8_t* __restrict__ out_null) {
  for (int64_t i = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; i < n; i += (int64_t)gridDim.x * B2_BLOCK) {
    const int64_t r = idx ? idx[i] : i;
    int64_t raw = c.dtype == B2_U8 ? (int64_t) reinterpret_cast<const uint8_t*>(c.data)[r]
                                   : __ldg(reinterpret_cast<const long long*>(c.data) + r);
    const bool isnull = b2_is_null(c, r, raw);
    if (c.dtype == B2_F64) {
      if (raw == (int64_t)0x8000000000000000LL) raw = 0;  // -0.0 sorts with 0.0
      raw = b2_ordered_from_bits(raw);
    }
    uint64_t img = (uint64_t)raw ^ 0x8000000000000000ULL;  // signed -> unsigned order
    if (descending) img = ~img;
    out_img[i] = isnull ? 0 : img;
    // most significant digit: 0 sorts first.  NULLS FIRST -> NULL rows get 0, others 1 (and vice versa)
    out_null[i] = (uint8_t)((isnull ? 1 : 0) ^ (nulls_first ? 1 : 0));
  }
}

__device__ __forceinline__ uint32_t b2_sort_digit(const uint64_t* __restrict__ keys, const uint8_t* __restrict__ nulls,
                                                  int64_t i, int shift) {
  // shift < 0: the one-bit NULL key
  return shift < 0 ? (uint32_t)nulls[i] : (uint32_t)((keys[i] >> shift) & 0xff);
}

// per-warp histogram of its sub-chunk into shared counters cnt[warp][256]
__device__ __forceinline__ void b2_sort_warp_hist(const uint64_t* __restrict__ keys, const uint8_t* __restrict__ nulls,
                                                  int64_t lo, int64_t hi, int shift, uint32_t* cnt) {
  const int lane = threadIdx.x & 31;
  for (int64_t base = lo; base < hi; base += 32) {
    const int64_t i = base + lane;
    const bool act = i < hi;
    const uint32_t mask = __ballot_sync(FULL_MASK, act);
    if (act) {
      const uint32_t d = b2_sort_digit(keys, nulls, i, shift);
      const uint32_t peers = __match_any_sync(mask, d);
      if ((peers & ((1u << lane) - 1)) == 0) cnt[d] += __popc(peers);  // leader of the peer group
    }
    __syncwarp();
  }
}

__global__ void __launch_bounds__(B2_SORT_BLOCK)
b2_sort_hist_kernel(const uint64_t* __restrict__ keys, const uint8_t* __restrict__ nulls, int64_t n, int shift,
                    uint32_t* __restrict__ hist /* [nblocks][256] */) {
  __shared__ uint32_t cnt[B2_SORT_WARPS][256];
  const int warp = threadIdx.x >> 5;
  for (int d = threadIdx.x; d < B2_SORT_WARPS * 256; d += B2_SORT_BLOCK) (&cnt[0][0])[d] = 0;
  __syncthreads();
  const int64_t lo = (int64_t)blockIdx.x * B2_SORT_CHUNK + (int64_t)warp * B2_SORT_ITEMS_PER_WARP;
  const int64_t hi = lo + B2_SORT_ITEMS_PER_WARP < n ? lo + B2_SORT_ITEMS_PER_WARP : n;
  if (lo < n) b2_sort_warp_hist(keys, nulls, lo, hi, shift, cnt[warp]);
  __syncthreads();
  for (int d = threadIdx.x; d < 256; d += B2_SORT_BLOCK) {
    uint32_t t = 0;
    for (int w = 0; w < B2_SORT_WARPS; ++w) t += cnt[w][d];
    hist[(int64_t)blockIdx.x * 256 + d] = t;
  }
}

// offsets[b][d] = rows with a smaller digit, plus rows with digit d in earlier blocks (one block)
__global__ void __launch_bounds__(256)
b2_sort_scan_kernel(const uint32_t* __restrict__ hist, int64_t nblocks, int64_t* __restrict__ offsets) {
  __shared__ int64_t total[256];
  const int d = threadIdx.x;
  int64_t run = 0;
  for (int64_t b = 0; b < nblocks; ++b) {
    const uint32_t h = hist[b * 256 + d];
    offsets[b * 256 + d] = run;
    run += h;
  }
  total[d] = run;
  __syncthreads();
  int64_t before = 0;
  for (int k = 0; k < d; ++k) before += total[k];
  for (int64_t b = 0; b < nblocks; ++b) offsets[b * 256 + d] += before;
}

__global__ void __launch_bounds__(B2_SORT_BLOCK)
b2_sort_scatter_kernel(const uint64_t* __restrict__ keys, const uint8_t* __restrict__ nulls,
                       const int32_t* __restrict__ idx, int64_t n, int shift, const int64_t* __restrict__ offsets,
                       uint64_t* __restrict__ keys_out, uint8_t* __restrict__ nulls_out, int32_t* __restrict__ idx_out) {
  __shared__ uint32_t cnt[B2_SORT_WARPS][256];
  __shared__ int64_t base_sh[B2_SORT_WARPS][256];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int d = threadIdx.x; d < B2_SORT_WARPS * 256; d += B2_SORT_BLOCK) (&cnt[0][0])[d] = 0;
  __syncthreads();
  const int64_t lo = (int64_t)blockIdx.x * B2_SORT_CHUNK + (int64_t)warp * B2_SORT_ITEMS_PER_WARP;
  const int64_t hi = lo + B2_SORT_ITEMS_PER_WARP < n ? lo + B2_SORT_ITEMS_PER_WARP : n;
  if (lo < n) b2_sort_warp_hist(keys, nulls, lo, hi, shift, cnt[warp]);
  __syncthreads();
  for (int d = threadIdx.x; d < 256; d += B2_SORT_BLOCK) {
    int64_t run = offsets[(int64_t)blockIdx.x * 256 + d];
    for (int w = 0; w < B2_SORT_WARPS; ++w) {
      base_sh[w][d] = run;
      run += cnt[w][d];
    }
  }
  __syncthreads();
  // stable placement: rows of a warp's sub-chunk are visited in order, 32 at a time
  if (lo < n) {
    int64_t* base = base_sh[warp];
    for (int64_t b0 = lo; b0 < hi; b0 += 32) {
      const int64_t i = b0 + lane;
      const bool act = i < hi;
      const uint32_t mask = __ballot_sync(FULL_MASK, act);
      if (act) {
        const uint32_t d = b2_sort_digit(keys, nulls, i, shift);
        const uint32_t peers = __match_any_sync(mask, d);
        const int rank = __popc(peers & ((1u << lane) - 1));
        const int64_t pos = base[d] + rank;
        keys_out[pos] = keys[i];
        nulls_out[pos] = nulls[i];
        idx_out[pos] = idx[i];
        __syncwarp(mask);
        if (rank == 0) base[d] += __popc(peers);
      }
      __syncwarp();
    }
  }
}

__global__ void __launch_bounds__(B2_BLOCK)
b2_iota_kernel(int32_t* __restrict__ out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; i < n; i += (int64_t)gridDim.x * B2_BLOCK) out[i] = (int32_t)i;
}

__global__ void __launch_bounds__(B2_BLOCK)
b2_bitwise_combine_kernel(uint32_t* __restrict__ dst, const uint32_t* __restrict__ src, int64_t nwords, int op) {
  for (int64_t i = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; i < nwords; i += (int64_t)gridDim.x * B2_BLOCK) {
    const uint32_t a = dst[i], b = src[i];
    dst[i] = op == B2_AGG_AND ? a & b : op == B2_AGG_OR ? a | b : a ^ b;
  }
}

extern "C" {

// dst = dst <op> src over nwords 32-bit words: the fold of bitwise accumulators exchanged between GPUs
// (NCCL offers no bitwise reduction).
int32_t b2_bitwise_combine(uint32_t* dst, const uint32_t* src, int64_t nwords, int32_t op, void* stream) {
  B2_REQUIRE((dst && src) || nwords == 0, "null argument");
  B2_REQUIRE(op == B2_AGG_AND || op == B2_AGG_OR || op == B2_AGG_XOR, "bad bitwise op");
  if (nwords <= 0) return B2_OK;
  int grid = b2_wave_grid(b2_bitwise_combine_kernel, B2_BLOCK, (nwords + B2_BLOCK - 1) / B2_BLOCK);
  b2_bitwise_combine_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(dst, src, nwords, op);
  B2_CHECK_LAUNCH("b2_bitwise_combine_kernel");
  return B2_OK;
}

int64_t b2_sort_ws_bytes(int64_t n) {
  const int64_t nblocks = (n + B2_SORT_CHUNK - 1) / B2_SORT_CHUNK;
  // two (image, null, idx) buffers + histogram + offsets
  return 2 * (n * 8 + n + n * 4) + nblocks * 256 * (4 + 8) + 4096;
}

// Reorders `idx` (int32[n], a permutation; use b2_iota first) so that rows are stably sorted by
// `col` (ascending / descending, NULLs first / last).  For a multi-key ORDER BY call it once per
// key from the LAST key to the FIRST.  ws: b2_sort_ws_bytes(n) bytes of device scratch.
int32_t b2_sort_by(const b2_col_t* col, int64_t n, int32_t descending, int32_t nulls_first, int32_t* idx,
                   void* ws, void* stream) {
  B2_REQUIRE(col && idx && ws, "null argument");
  B2_REQUIRE(n < ((int64_t)1 << 31), "sort handles < 2^31 rows");
  if (n <= 1) return B2_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t nblocks = (n + B2_SORT_CHUNK - 1) / B2_SORT_CHUNK;
  uint8_t* p = reinterpret_cast<uint8_t*>(ws);
  auto take = [&](int64_t bytes) { uint8_t* r = p; p += (bytes + 63) & ~(int64_t)63; return r; };
  uint64_t* img[2] = {reinterpret_cast<uint64_t*>(take(n * 8)), reinterpret_cast<uint64_t*>(take(n * 8))};
  uint8_t* nul[2] = {take(n), take(n)};
  int32_t* ix[2] = {reinterpret_cast<int32_t*>(take(n * 4)), reinterpret_cast<int32_t*>(take(n * 4))};
  uint32_t* hist = reinterpret_cast<uint32_t*>(take(nblocks * 256 * 4));
  int64_t* offsets = reinterpret_cast<int64_t*>(take(nblocks * 256 * 8));
  int grid = b2_wave_grid(b2_sort_image_kernel, B2_BLOCK, (n + B2_BLOCK - 1) / B2_BLOCK);
  b2_sort_image_kernel<<<grid, B2_BLOCK, 0, st>>>(*col, idx, n, descending, nulls_first, img[0], nul[0]);
  B2_CUDA_TRY(cudaMemcpyAsync(ix[0], idx, n * 4, cudaMemcpyDeviceToDevice, st));
  int cur = 0;
  // eight value digits, then the one-bit NULL key as the most significant digit
  for (int pass = 0; pass < 9; ++pass) {
    const int shift = pass < 8 ? pass * 8 : -1;
    b2_sort_hist_kernel<<<(int)nblocks, B2_SORT_BLOCK, 0, st>>>(img[cur], nul[cur], n, shift, hist);
    b2_sort_scan_kernel<<<1, 256, 0, st>>>(hist, nblocks, offsets);
    b2_sort_scatter_kernel<<<(int)nblocks, B2_SORT_BLOCK, 0, st>>>(img[cur], nul[cur], ix[cur], n, shift, offsets,
                                                                   img[cur ^ 1], nul[cur ^ 1], ix[cur ^ 1]);
    cur ^= 1;
  }
  B2_CHECK_LAUNCH("b2_sort kernels");
  B2_CUDA_TRY(cudaMemcpyAsync(idx, ix[cur], n * 4, cudaMemcpyDeviceToDevice, st));
  return B2_OK;
}

int32_t b2_iota(int32_t* out, int64_t n, void* stream) {
  B2_REQUIRE(out || n == 0, "null argument");
  if (n <= 0) return B2_OK;
  int grid = b2_wave_grid(b2_iota_kernel, B2_BLOCK, (n + B2_BLOCK - 1) / B2_BLOCK);
  b2_iota_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(out, n);
  B2_CHECK_LAUNCH("b2_iota_kernel");
  return B2_OK;
}

}  // extern "C"
