// select.cuh — exact order statistics of one column: one pass of a multi-target MSD radix select.
// ANALYZE TABLE ... COMPUTE STATISTICS needs the 25 / 50 / 75 % quantiles of every numeric column; the
// reference takes them from dask's describe() (approximate per-partition percentiles merged).  Here the
// host walks the column's 64-bit order-preserving image from its highest differing bit down, up to 11
// bits per pass: each pass histograms, for every target rank, the next digit of the rows that still
// share the target's prefix, and the host picks the digit that holds the rank.  A pass reads 8 bytes
// (plus a bitmap bit) per row and writes only the histogram; once the rows that can still matter are
// few, one pass also copies them to a dense buffer that the later passes read instead of the column.
#pragma once
#include "common.cuh"

#define B2_SELECT_BLOCK 256
#define B2_SELECT_ROWS 4      // rows per thread per iteration: four independent 8-byte loads in flight

// unsigned order-preserving image of a non-NULL value: the sign-flipped int64, or the ordered float64
// image (the one MIN / MAX and b2_sort_by use) sign-flipped
template <bool F64>
__device__ __forceinline__ uint64_t b2_select_image(int64_t raw) {
  return (uint64_t)(F64 ? b2_ordered_from_bits(raw) : raw) ^ 0x8000000000000000ULL;
}

// Block-private histograms (nsel << bits uint32 counters in dynamic shared memory), flushed with one
// global atomic per non-zero bin.  COMPACT: also append the raw value of every row that matches some
// target's prefix to out[]: the block's rows of one iteration reserve their places with one atomic on
// *out_count (a warp-level reservation serialises millions of atomics on that one word).
template <bool F64, bool COMPACT>
__global__ void __launch_bounds__(B2_SELECT_BLOCK)
b2_select_hist_kernel(const __grid_constant__ b2_col_t c, int64_t n, const __grid_constant__ b2_select_t sel,
                      unsigned long long* __restrict__ hist, int64_t* __restrict__ out,
                      unsigned long long* __restrict__ out_count) {
  extern __shared__ uint32_t sh[];
  __shared__ uint32_t warp_off[B2_SELECT_BLOCK / 32];
  __shared__ unsigned long long block_base;
  const int nbins = sel.nsel << sel.bits;
  for (int b = threadIdx.x; b < nbins; b += B2_SELECT_BLOCK) sh[b] = 0;
  __syncthreads();
  const int hs = sel.shift + sel.bits;
  const uint32_t dmask = (1u << sel.bits) - 1u;
  const int64_t* data = reinterpret_cast<const int64_t*>(c.data);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t step = (int64_t)B2_SELECT_BLOCK * B2_SELECT_ROWS;
  // the loop bound is uniform across the block, so every thread reaches the barriers and ballots below
  for (int64_t base = (int64_t)blockIdx.x * step; base < n; base += (int64_t)gridDim.x * step) {
    int64_t raw[B2_SELECT_ROWS];
#pragma unroll
    for (int j = 0; j < B2_SELECT_ROWS; ++j) {
      const int64_t i = base + j * B2_SELECT_BLOCK + threadIdx.x;
      raw[j] = i < n ? b2_ld_stream(data + i) : 0;
    }
    uint32_t hits = 0;   // bit j: row j matches some target
#pragma unroll
    for (int j = 0; j < B2_SELECT_ROWS; ++j) {
      const int64_t i = base + j * B2_SELECT_BLOCK + threadIdx.x;
      bool ok = i < n;
      if (ok && c.valid) ok = b2_bit(c.valid, i);
      if (F64 && ok) {
        const double d = __longlong_as_double(raw[j]);
        ok = d == d;
      }
      if (ok) {
        const uint64_t u = b2_select_image<F64>(raw[j]);
        const uint64_t p = hs >= 64 ? 0 : u >> hs;
        const uint32_t d = (uint32_t)(u >> sel.shift) & dmask;
#pragma unroll
        for (int k = 0; k < B2_SELECT_MAX_TARGETS; ++k) {
          if (k < sel.nsel && p == sel.prefix[k]) {
            atomicAdd(&sh[(k << sel.bits) + d], 1u);
            hits |= 1u << j;
          }
        }
      }
    }
    if (COMPACT) {
      uint32_t m[B2_SELECT_ROWS];
      uint32_t total = 0;
#pragma unroll
      for (int j = 0; j < B2_SELECT_ROWS; ++j) {
        m[j] = __ballot_sync(FULL_MASK, (hits >> j) & 1u);
        total += __popc(m[j]);
      }
      if (lane == 0) warp_off[warp] = total;
      __syncthreads();
      if (threadIdx.x == 0) {
        uint32_t run = 0;
        for (int w = 0; w < B2_SELECT_BLOCK / 32; ++w) {
          const uint32_t t = warp_off[w];
          warp_off[w] = run;
          run += t;
        }
        block_base = run ? atomicAdd(out_count, (unsigned long long)run) : 0ull;
      }
      __syncthreads();
      unsigned long long pos = block_base + warp_off[warp];
      const uint32_t below = (1u << lane) - 1u;
#pragma unroll
      for (int j = 0; j < B2_SELECT_ROWS; ++j) {
        if ((hits >> j) & 1u) out[pos + __popc(m[j] & below)] = raw[j];
        pos += __popc(m[j]);
      }
      // warp_off[warp] is rewritten by lane 0 in the next iteration; block_base only after the next barrier
      __syncwarp();
    }
  }
  __syncthreads();
  for (int b = threadIdx.x; b < nbins; b += B2_SELECT_BLOCK)
    if (sh[b]) atomicAdd(hist + b, (unsigned long long)sh[b]);
}

template <bool F64, bool COMPACT>
static int32_t b2_select_launch(const b2_col_t& c, int64_t n, const b2_select_t& sel, uint64_t* hist, int64_t* out,
                                uint64_t* out_count, cudaStream_t st) {
  auto kernel = b2_select_hist_kernel<F64, COMPACT>;
  const int smem = (sel.nsel << sel.bits) * (int)sizeof(uint32_t);
  if (smem > 48 * 1024)
    B2_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int occ = 1;
  B2_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, B2_SELECT_BLOCK, smem));
  if (occ < 1) occ = 1;
  const int64_t step = (int64_t)B2_SELECT_BLOCK * B2_SELECT_ROWS;
  int64_t grid = (int64_t)b2_sm_count() * occ;
  if (grid > (n + step - 1) / step) grid = (n + step - 1) / step;
  kernel<<<(int)grid, B2_SELECT_BLOCK, smem, st>>>(c, n, sel, reinterpret_cast<unsigned long long*>(hist), out,
                                                   reinterpret_cast<unsigned long long*>(out_count));
  B2_CHECK_LAUNCH("b2_select_hist_kernel");
  return B2_OK;
}

extern "C" {

int32_t b2_select_hist(const b2_col_t* col, int64_t n, const b2_select_t* sel, uint64_t* hist, int64_t* out,
                       uint64_t* out_count, void* stream) {
  B2_REQUIRE(col && sel && hist, "null argument");
  B2_REQUIRE(col->dtype == B2_I64 || col->dtype == B2_F64, "column must be B2_I64 or B2_F64");
  B2_REQUIRE(sel->nsel >= 1 && sel->nsel <= B2_SELECT_MAX_TARGETS, "nsel must be 1..B2_SELECT_MAX_TARGETS");
  B2_REQUIRE(sel->bits >= 1 && sel->bits <= B2_SELECT_MAX_BITS, "bits must be 1..B2_SELECT_MAX_BITS");
  B2_REQUIRE(sel->shift >= 0 && sel->shift + sel->bits <= 64, "shift + bits must lie in [bits, 64]");
  B2_REQUIRE(!out || out_count, "a compacting pass needs out_count");
  const int hs = sel->shift + sel->bits;
  for (int k = 0; k < sel->nsel; ++k)
    B2_REQUIRE(hs == 64 ? sel->prefix[k] == 0 : (sel->prefix[k] >> (64 - hs)) == 0,
               "prefix wider than 64 - shift - bits");
  if (n <= 0) return B2_OK;
  B2_REQUIRE(col->data, "null column data");
  cudaStream_t st = (cudaStream_t)stream;
  const bool f = col->dtype == B2_F64;
  if (out) return f ? b2_select_launch<true, true>(*col, n, *sel, hist, out, out_count, st)
                    : b2_select_launch<false, true>(*col, n, *sel, hist, out, out_count, st);
  return f ? b2_select_launch<true, false>(*col, n, *sel, hist, nullptr, nullptr, st)
           : b2_select_launch<false, false>(*col, n, *sel, hist, nullptr, nullptr, st);
}

}  // extern "C"
