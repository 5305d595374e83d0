// partition.cuh — range partitioning of (group key, aggregate inputs) for group tables far beyond L2.
//
// A direct-address group table of 100M slots (C5) is 0.8 GB per accumulator array: every atomic of
// b2_groupby_dense is then a random DRAM read-modify-write.  Rows are
// therefore first reordered by key range so that all rows of one bucket -- whose slice of the table
// is a few tens of MB -- are contiguous; b2_groupby_dense over the reordered arrays then walks the
// buckets in order and its atomics stay L2-resident.  Three launches, no host round trip:
//   b2_part_hist_kernel    rows per bucket (key + predicate columns only)
//   b2_part_scan_kernel    bucket starts, write cursors
//   b2_part_scatter_kernel per 2048-row tile: shared-memory ranks, one global reservation per
//                          (tile, bucket), then key' = kmin + slot and the carried columns are
//                          written to their bucket's region
// Rows that fail the scan's terms are dropped; a NULL key goes to slot nslots-1 (encoded as the key
// value kmin + nslots - 1, so the consumer runs with one slot more and no bitmap).
#pragma once
#include "common.cuh"

#define B2_PART_R 8
#define B2_PART_TILE (B2_BLOCK * B2_PART_R)
#define B2_PART_MAX_BUCKETS 1024
// Output positions are reserved with returning atomics on per-bucket cursors.  Atomics on ONE address are
// served one at a time by the L2 (scripts/microbench/redg.cu "red_hot": 1.76 ns each without a return
// value on H100, far more with one), and with ~100 buckets every reservation of the whole GPU lands on
// ~100 addresses -- that alone would be most of the scatter's time.  So every bucket is fed through
// B2_PART_GROUPS independent cursors: CTA c only ever touches group c % B2_PART_GROUPS, the histogram
// pass counts per (group, bucket) with the same tile -> CTA assignment, and the scan lays a bucket's
// groups out back to back.  Contention per address drops by the number of groups.
#define B2_PART_GROUPS 64
static inline int b2_part_grid(int64_t ntiles) {   // hist and scatter MUST use the same grid (tile -> CTA -> group)
  int64_t g = (int64_t)b2_sm_count() * 4;
  if (g > ntiles) g = ntiles;
  return (int)(g < 1 ? 1 : g);
}

struct b2_partcarry_arg {
  int32_t n;
  int32_t cols[B2_MAX_GATHER];
  void* out[B2_MAX_GATHER];
};

// slots of the batch (-1 = row does not take part)
template <int R>
__device__ __forceinline__ void b2_part_slots(const b2_scan_t& s, int key_col, int64_t kmin, int64_t nslots,
                                              int64_t row0, int64_t (&slot)[R]) {
  const b2_col_t& kc = s.cols[key_col];
  bool full;
  const uint32_t bits = b2_eval_terms<R>(s, row0, full);
  int64_t key[R];
  b2_load_batch<R>(kc, row0, bits, full, key);
  uint32_t kvalid = bits;
  if (kc.valid) kvalid = b2_valid_bits<R>(kc.valid, row0, bits);
#pragma unroll
  for (int j = 0; j < R; ++j) {
    slot[j] = -1;
    if ((bits >> j) & 1) {
      if (!((kvalid >> j) & 1)) slot[j] = nslots - 1;
      else {
        const uint64_t d = (uint64_t)key[j] - (uint64_t)kmin;
        slot[j] = d < (uint64_t)(nslots - 1) ? (int64_t)d : -1;
      }
    }
  }
}

__global__ void __launch_bounds__(B2_BLOCK)
b2_part_hist_kernel(const __grid_constant__ b2_scan_t s, int key_col, int64_t kmin, int64_t nslots, int shift,
                    int nbuckets, int64_t ntiles, unsigned long long* __restrict__ counts) {
  __shared__ int hist[B2_PART_MAX_BUCKETS];
  for (int b = threadIdx.x; b < nbuckets; b += B2_BLOCK) hist[b] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * B2_PART_TILE + (int64_t)warp * (32 * B2_PART_R) + lane;
    int64_t slot[B2_PART_R];
    b2_part_slots<B2_PART_R>(s, key_col, kmin, nslots, row0, slot);
#pragma unroll
    for (int j = 0; j < B2_PART_R; ++j)
      if (slot[j] >= 0) atomicAdd(&hist[(int)(slot[j] >> shift)], 1);
  }
  __syncthreads();
  unsigned long long* mine = counts + (size_t)(blockIdx.x % B2_PART_GROUPS) * nbuckets;
  for (int b = threadIdx.x; b < nbuckets; b += B2_BLOCK)
    if (hist[b]) atomicAdd(mine + b, (unsigned long long)hist[b]);
}

// ws: [0, nb] bucket starts (out), then cursors[group][bucket] (in: row counts from the histogram pass,
// out: first output row of that group's share of the bucket)
__global__ void __launch_bounds__(1024) b2_part_scan_kernel(int64_t* __restrict__ ws, int nbuckets) {
  __shared__ int64_t warp_tot[32];
  int64_t* cur = ws + nbuckets + 1;
  const int b = threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t total = 0;
  if (b < nbuckets)
    for (int g = 0; g < B2_PART_GROUPS; ++g) total += cur[(size_t)g * nbuckets + b];
  int64_t incl = total;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t t = __shfl_up_sync(FULL_MASK, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  int64_t off = 0;
  for (int w = 0; w < warp; ++w) off += warp_tot[w];
  int64_t run = off + incl - total;          // first output row of bucket b
  if (b < nbuckets) {
    ws[b] = run;
    for (int g = 0; g < B2_PART_GROUPS; ++g) {
      const int64_t c = cur[(size_t)g * nbuckets + b];
      cur[(size_t)g * nbuckets + b] = run;
      run += c;
    }
    if (b == nbuckets - 1) ws[nbuckets] = run;
  }
}

// Scatter one 2048-row tile: ranks by shared-memory atomics, then the tile's rows are ordered by
// bucket in shared memory (key' + source row + bucket id: 24 KB) so that consecutive threads write
// consecutive output rows -- coalesced stores instead of 32 different sectors per store instruction.
// The carried columns are gathered from the tile (16 KB per column, just read: L1/L2 hits).
__global__ void __launch_bounds__(B2_BLOCK)
b2_part_scatter_kernel(const __grid_constant__ b2_scan_t s, int key_col, int64_t kmin, int64_t nslots, int shift,
                       int nbuckets, int64_t ntiles, unsigned long long* __restrict__ cursor,
                       int64_t* __restrict__ out_key, const __grid_constant__ b2_partcarry_arg carry) {
  __shared__ int hist[B2_PART_MAX_BUCKETS];          // rows of this tile per bucket
  __shared__ int prefix[B2_PART_MAX_BUCKETS];        // exclusive scan of hist
  __shared__ long long base[B2_PART_MAX_BUCKETS];    // first output row of this tile in each bucket
  __shared__ int64_t st_key[B2_PART_TILE];
  __shared__ uint16_t st_src[B2_PART_TILE];
  __shared__ uint16_t st_bkt[B2_PART_TILE];
  __shared__ int warp_tot[B2_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int PER = B2_PART_MAX_BUCKETS / B2_BLOCK;  // buckets per thread in the scan (4)
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    for (int b = threadIdx.x; b < nbuckets; b += B2_BLOCK) hist[b] = 0;
    __syncthreads();
    const int local0 = warp * (32 * B2_PART_R) + lane;                 // row within the tile of batch row 0
    const int64_t row0 = tile * B2_PART_TILE + local0;
    int64_t slot[B2_PART_R];
    int rank[B2_PART_R];
    b2_part_slots<B2_PART_R>(s, key_col, kmin, nslots, row0, slot);
#pragma unroll
    for (int j = 0; j < B2_PART_R; ++j) {
      rank[j] = 0;
      if (slot[j] >= 0) rank[j] = atomicAdd(&hist[(int)(slot[j] >> shift)], 1);
    }
    __syncthreads();
    // exclusive scan of hist[0..nbuckets) + one global reservation per non-empty bucket
    {
      int v[PER], tsum = 0;
#pragma unroll
      for (int k = 0; k < PER; ++k) {
        const int b = threadIdx.x * PER + k;
        v[k] = b < nbuckets ? hist[b] : 0;
        tsum += v[k];
      }
      int incl = tsum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(FULL_MASK, incl, o);
        if (lane >= o) incl += t;
      }
      if (lane == 31) warp_tot[warp] = incl;
      __syncthreads();
      int woff = 0;
      for (int w = 0; w < warp; ++w) woff += warp_tot[w];
      int run = woff + incl - tsum;
#pragma unroll
      for (int k = 0; k < PER; ++k) {
        const int b = threadIdx.x * PER + k;
        if (b < nbuckets) {
          prefix[b] = run;
          base[b] = v[k] ? (long long)atomicAdd(cursor + (size_t)(blockIdx.x % B2_PART_GROUPS) * nbuckets + b,
                                                (unsigned long long)v[k]) : 0;
          run += v[k];
        }
      }
    }
    __syncthreads();
    int total = 0;
    for (int w = 0; w < B2_WARPS; ++w) total += warp_tot[w];
    // stage the tile in bucket order
#pragma unroll
    for (int j = 0; j < B2_PART_R; ++j) {
      if (slot[j] >= 0) {
        const int b = (int)(slot[j] >> shift);
        const int p = prefix[b] + rank[j];
        st_key[p] = (int64_t)((uint64_t)kmin + (uint64_t)slot[j]);   // wraps: the NULL slot may lie past INT64_MAX
        st_src[p] = (uint16_t)(local0 + j * 32);
        st_bkt[p] = (uint16_t)b;
      }
    }
    __syncthreads();
    const int64_t tile_row0 = tile * B2_PART_TILE;
    for (int p = threadIdx.x; p < total; p += B2_BLOCK) {
      const int b = st_bkt[p];
      const int64_t dst = base[b] + (p - prefix[b]);
      b2_st_stream(out_key + dst, st_key[p]);
      const int64_t src = tile_row0 + st_src[p];
      for (int c = 0; c < carry.n; ++c) {
        const int64_t v = __ldg(reinterpret_cast<const long long*>(s.cols[carry.cols[c]].data) + src);
        b2_st_stream(reinterpret_cast<int64_t*>(carry.out[c]) + dst, v);
      }
    }
    __syncthreads();   // shared arrays are reused by the next tile
  }
}

extern "C" {

int64_t b2_range_partition_ws_bytes(int32_t nbuckets) {
  return 8 * ((int64_t)nbuckets + 2 + (int64_t)B2_PART_GROUPS * nbuckets);
}

static int32_t b2_part_check(const b2_scan_t* scan, int32_t key_col, int64_t nslots, int32_t shift, int32_t nbuckets,
                             const void* d_ws) {
  int32_t rc = b2_check_scan(scan);
  if (rc) return rc;
  B2_REQUIRE(key_col >= 0 && key_col < scan->ncols && scan->cols[key_col].dtype == B2_I64, "range partition needs an int64 key");
  B2_REQUIRE(nslots >= 2 && shift >= 0 && shift < 62, "bad slot range");
  B2_REQUIRE(nbuckets >= 1 && nbuckets <= B2_PART_MAX_BUCKETS && ((nslots - 1) >> shift) < nbuckets, "bad bucket count");
  B2_REQUIRE(d_ws, "null workspace");
  return B2_OK;
}

int32_t b2_range_partition_hist(const b2_scan_t* scan, int32_t key_col, int64_t kmin, int64_t nslots, int32_t shift,
                                int32_t nbuckets, void* d_ws, void* stream) {
  int32_t rc = b2_part_check(scan, key_col, nslots, shift, nbuckets, d_ws);
  if (rc) return rc;
  const int64_t ntiles = (scan->n + B2_PART_TILE - 1) / B2_PART_TILE;
  if (ntiles <= 0) return B2_OK;
  const int grid = b2_part_grid(ntiles);
  b2_part_hist_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(
      *scan, key_col, kmin, nslots, shift, nbuckets, ntiles,
      reinterpret_cast<unsigned long long*>(reinterpret_cast<int64_t*>(d_ws) + nbuckets + 1));
  B2_CHECK_LAUNCH("b2_part_hist_kernel");
  return B2_OK;
}

int32_t b2_range_partition_scan(int32_t nbuckets, void* d_ws, void* stream) {
  B2_REQUIRE(nbuckets >= 1 && nbuckets <= B2_PART_MAX_BUCKETS && d_ws, "bad arguments");
  b2_part_scan_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(reinterpret_cast<int64_t*>(d_ws), nbuckets);
  B2_CHECK_LAUNCH("b2_part_scan_kernel");
  return B2_OK;
}

int32_t b2_range_partition_scatter(const b2_scan_t* scan, int32_t key_col, int64_t kmin, int64_t nslots, int32_t shift,
                                   int32_t nbuckets, int32_t ncarry, const int32_t* carry_cols, int64_t* out_key,
                                   void* const* out_cols, void* d_ws, void* stream) {
  int32_t rc = b2_part_check(scan, key_col, nslots, shift, nbuckets, d_ws);
  if (rc) return rc;
  B2_REQUIRE(ncarry >= 0 && ncarry <= B2_MAX_GATHER && out_key, "bad arguments");
  b2_partcarry_arg carry;
  memset(&carry, 0, sizeof(carry));
  carry.n = ncarry;
  for (int c = 0; c < ncarry; ++c) {
    B2_REQUIRE(carry_cols[c] >= 0 && carry_cols[c] < scan->ncols && out_cols[c], "bad carried column");
    const b2_col_t& col = scan->cols[carry_cols[c]];
    B2_REQUIRE(col.dtype != B2_U8 && !col.valid, "carried columns must be 8-byte columns without a validity bitmap");
    carry.cols[c] = carry_cols[c];
    carry.out[c] = out_cols[c];
  }
  const int64_t ntiles = (scan->n + B2_PART_TILE - 1) / B2_PART_TILE;
  if (ntiles <= 0) return B2_OK;
  int64_t* ws = reinterpret_cast<int64_t*>(d_ws);
  // The scatter is CTA-wide so that its stores fill whole sectors: a 2048-row tile puts ~20 rows into each
  // of ~100 buckets, so the staged stores of one bucket are a run of ~170 bytes.
  const int grid = b2_part_grid(ntiles);
  b2_part_scatter_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(
      *scan, key_col, kmin, nslots, shift, nbuckets, ntiles, reinterpret_cast<unsigned long long*>(ws + nbuckets + 1),
      out_key, carry);
  B2_CHECK_LAUNCH("b2_part_scatter_kernel");
  return B2_OK;
}

int32_t b2_range_partition(const b2_scan_t* scan, int32_t key_col, int64_t kmin, int64_t nslots, int32_t shift,
                           int32_t nbuckets, int32_t ncarry, const int32_t* carry_cols, int64_t* out_key,
                           void* const* out_cols, void* d_ws, void* stream) {
  int32_t rc = b2_range_partition_hist(scan, key_col, kmin, nslots, shift, nbuckets, d_ws, stream);
  if (rc) return rc;
  rc = b2_range_partition_scan(nbuckets, d_ws, stream);
  if (rc) return rc;
  return b2_range_partition_scatter(scan, key_col, kmin, nslots, shift, nbuckets, ncarry, carry_cols, out_key,
                                    out_cols, d_ws, stream);
}

}  // extern "C"
