// filter.cuh — predicate scan kernels: fused filter+global-aggregate, order-preserving
// selection (count / scan / write+gather), gather.
#pragma once
#include "common.cuh"
#include "pipeline.cuh"

// =======================================================================================
// fused filter + global aggregate   (SELECT SUM(x) FROM t WHERE x > 0)
// each warp owns 32*R consecutive rows per step; lanes read 8-byte words 256 B apart per row
// group so every warp-load is one fully coalesced 256-byte request.
// =======================================================================================
#define B2_AGG_R 16   // rows per lane per batch on the direct path (the staged path uses B2_PIPE_R)
#define B2_AGG_ROWS_PER_BLOCK (B2_BLOCK * B2_AGG_R)

struct b2_partial {
  int64_t acc[B2_MAX_AGGS];
  int64_t cnt[B2_MAX_AGGS];
};

template <bool BITS = true>   // false: the caller has no bitwise aggregate
__device__ __forceinline__ int64_t b2_combine(int op, int dtype, int64_t a, int64_t b) {
  if (BITS && op >= B2_AGG_AND) return op == B2_AGG_AND ? a & b : op == B2_AGG_OR ? a | b : a ^ b;
  switch (op) {
    case B2_AGG_SUM:
      if (dtype == B2_F64) return __double_as_longlong(__longlong_as_double(a) + __longlong_as_double(b));
      return (int64_t)((uint64_t)a + (uint64_t)b);
    case B2_AGG_SUMF:
      return __double_as_longlong(__longlong_as_double(a) + __longlong_as_double(b));
    case B2_AGG_MIN: return a < b ? a : b;
    case B2_AGG_MAX: return a > b ? a : b;
    default: return 0;
  }
}
template <bool BITS = true>
__device__ __forceinline__ int64_t b2_identity(int op) {
  if (op == B2_AGG_MIN) return LLONG_MAX;
  if (op == B2_AGG_MAX) return LLONG_MIN;
  if (BITS && op == B2_AGG_AND) return -1;
  return 0;  // +0.0 has the same bit pattern
}

// per-lane combine of one batch into a running accumulator, compile-time kind
template <int R, int KIND>
__device__ __forceinline__ int64_t b2_fold_batch(int64_t acc, const int64_t (&raw)[R], uint32_t ok) {
#pragma unroll
  for (int j = 0; j < R; ++j) {
    if (!((ok >> j) & 1)) continue;
    if (KIND == B2_K_SUM_I) acc = (int64_t)((uint64_t)acc + (uint64_t)raw[j]);
    else if (KIND == B2_K_SUM_F) acc = __double_as_longlong(__longlong_as_double(acc) + __longlong_as_double(raw[j]));
    else if (KIND == B2_K_SUMF_I) acc = __double_as_longlong(__longlong_as_double(acc) + (double)raw[j]);
    else if (KIND == B2_K_MIN_I) acc = raw[j] < acc ? raw[j] : acc;
    else if (KIND == B2_K_MAX_I) acc = raw[j] > acc ? raw[j] : acc;
    else if (KIND == B2_K_MIN_F) { const int64_t v = b2_ordered_from_bits(raw[j]); acc = v < acc ? v : acc; }
    else if (KIND == B2_K_MAX_F) { const int64_t v = b2_ordered_from_bits(raw[j]); acc = v > acc ? v : acc; }
    else if (KIND == B2_K_AND) acc &= raw[j];
    else if (KIND == B2_K_OR) acc |= raw[j];
    else if (KIND == B2_K_XOR) acc ^= raw[j];
  }
  return acc;
}

// Accumulators live in shared memory, one slot per (aggregate, thread): the aggregate loop is a
// run-time loop (no 8-way unrolled register file), the kind switch sits outside the row loop.
// BITS: the instance that also folds AND / OR / XOR.  Those cases live in a kernel instance of their own:
// inlined into the one every other query runs, they made C1 (a SUM) 4 % slower on H100.
template <int R, bool BITS, class LD>
__device__ __forceinline__ void b2_scan_agg_body(const b2_scan_t& s, const LD& ld, const b2_aggs_arg& aggs,
                                                 int64_t (*sh_acc)[B2_BLOCK], int32_t (*sh_cnt)[B2_BLOCK], int tid) {
  bool full;
  int cached_col;
  int64_t cached[R];
  const uint32_t bits = b2_eval_terms<R>(s, ld, full, cached_col, cached);
  for (int a = 0; a < aggs.n; ++a) {
    const b2_agg_t ag = aggs.a[a];
    if (ag.col < 0) {  // COUNT(*)
      sh_cnt[a][tid] += __popc(bits);
      continue;
    }
    const b2_col_t& c = s.cols[ag.col];
    int64_t raw[R];
    if (ag.col == cached_col) {  // the predicate already loaded this column: reuse the registers
#pragma unroll
      for (int j = 0; j < R; ++j) raw[j] = cached[j];
    } else {
      ld.template load<R>(ag.col, bits, full, raw);
    }
    uint32_t ok = bits;
    if (c.valid || c.dtype == B2_F64) ok &= ~b2_null_bits<R>(c, ld.row0, bits, raw);
    sh_cnt[a][tid] += __popc(ok);
    int64_t acc = sh_acc[a][tid];
    const int kind = b2_agg_kind<BITS>(ag.op, c.dtype);
    if (BITS && kind >= B2_K_AND) {
      if (kind == B2_K_AND) acc = b2_fold_batch<R, B2_K_AND>(acc, raw, ok);
      else if (kind == B2_K_OR) acc = b2_fold_batch<R, B2_K_OR>(acc, raw, ok);
      else acc = b2_fold_batch<R, B2_K_XOR>(acc, raw, ok);
      sh_acc[a][tid] = acc;
      continue;
    }
    switch (kind) {
      case B2_K_SUM_I: acc = b2_fold_batch<R, B2_K_SUM_I>(acc, raw, ok); break;
      case B2_K_SUM_F: acc = b2_fold_batch<R, B2_K_SUM_F>(acc, raw, ok); break;
      case B2_K_SUMF_I: acc = b2_fold_batch<R, B2_K_SUMF_I>(acc, raw, ok); break;
      case B2_K_MIN_I: acc = b2_fold_batch<R, B2_K_MIN_I>(acc, raw, ok); break;
      case B2_K_MAX_I: acc = b2_fold_batch<R, B2_K_MAX_I>(acc, raw, ok); break;
      case B2_K_MIN_F: acc = b2_fold_batch<R, B2_K_MIN_F>(acc, raw, ok); break;
      case B2_K_MAX_F: acc = b2_fold_batch<R, B2_K_MAX_F>(acc, raw, ok); break;
      default: break;
    }
    sh_acc[a][tid] = acc;
  }
}

template <bool PIPE, bool BITS>
__global__ void __launch_bounds__(PIPE ? B2_PIPE_THREADS : B2_BLOCK)
b2_scan_agg_kernel(const __grid_constant__ b2_scan_t s, const __grid_constant__ b2_pipe_t pp,
                   const __grid_constant__ b2_aggs_arg aggs, b2_partial* __restrict__ partials) {
  __shared__ int64_t sh_acc[B2_MAX_AGGS][B2_BLOCK];
  __shared__ int32_t sh_cnt[B2_MAX_AGGS][B2_BLOCK];
  const int tid = threadIdx.x;
  if (tid < B2_BLOCK) {
    for (int a = 0; a < aggs.n; ++a) {
      sh_acc[a][tid] = b2_identity<BITS>(aggs.a[a].op);
      sh_cnt[a][tid] = 0;
    }
  }
  if (PIPE) b2_tile_pipeline(s, pp, [&](const auto& ld) { b2_scan_agg_body<B2_PIPE_R, BITS>(s, ld, aggs, sh_acc, sh_cnt, tid); });
  else b2_tile_direct<B2_AGG_R>(s, [&](const auto& ld) { b2_scan_agg_body<B2_AGG_R, BITS>(s, ld, aggs, sh_acc, sh_cnt, tid); });
  __syncthreads();
  // block reduction in a fixed order: thread a folds the 256 per-thread slots of aggregate a.
  // (int32 per-thread counts cannot overflow: a thread sees < 2^31 rows of a < 2^31-row partition)
  if (tid < aggs.n) {
    const int a = tid;
    const int op = aggs.a[a].op;
    const int dt = aggs.a[a].col >= 0 ? s.cols[aggs.a[a].col].dtype : B2_I64;
    int64_t r = b2_identity<BITS>(op), c = 0;
    for (int t = 0; t < B2_BLOCK; ++t) {
      r = b2_combine<BITS>(op, dt, r, sh_acc[a][t]);
      c += sh_cnt[a][t];
    }
    partials[blockIdx.x].acc[a] = r;
    partials[blockIdx.x].cnt[a] = c;
  }
}

// deterministic final reduce over the per-block partials (fixed order)
struct b2_final_arg {   // what the final reduce needs to know about each aggregate
  int32_t op[B2_MAX_AGGS];
  int32_t dtype[B2_MAX_AGGS];   // type the accumulator is combined in (B2_I64 / B2_F64)
  int32_t n;
};
__global__ void b2_scan_agg_final_kernel(const __grid_constant__ b2_final_arg fa,
                                         const b2_partial* __restrict__ partials, int nblocks,
                                         int64_t* __restrict__ out_acc, int64_t* __restrict__ out_cnt,
                                         int accumulate) {
  // one block per aggregate; thread t folds partials t, t+256, ... then a fixed-order tree in
  // shared memory: the result does not depend on scheduling (bit-reproducible float sums).
  __shared__ int64_t sh_r[B2_BLOCK];
  __shared__ int64_t sh_c[B2_BLOCK];
  const int a = blockIdx.x, t = threadIdx.x;
  const int op = fa.op[a];
  const int dt = fa.dtype[a];
  int64_t r = b2_identity(op), c = 0;
  for (int b = t; b < nblocks; b += B2_BLOCK) {
    r = b2_combine(op, dt, r, partials[b].acc[a]);
    c += partials[b].cnt[a];
  }
  sh_r[t] = r;
  sh_c[t] = c;
  __syncthreads();
  for (int w = B2_BLOCK / 2; w > 0; w >>= 1) {
    if (t < w) {
      sh_r[t] = b2_combine(op, dt, sh_r[t], sh_r[t + w]);
      sh_c[t] += sh_c[t + w];
    }
    __syncthreads();
  }
  if (t == 0) {
    out_acc[a] = accumulate ? b2_combine(op, dt, out_acc[a], sh_r[0]) : sh_r[0];
    out_cnt[a] = accumulate ? out_cnt[a] + sh_c[0] : sh_c[0];
  }
}

// =======================================================================================
// order-preserving selection.  One block owns one B2_TILE (4096 rows): 8 warps x 512 rows,
// warp rows are consecutive so ballots give in-order ranks.
// =======================================================================================
#define B2_SEL_R 16
static_assert(B2_BLOCK * B2_SEL_R == B2_TILE, "tile geometry");

__global__ void __launch_bounds__(B2_BLOCK)
b2_select_count_kernel(const __grid_constant__ b2_scan_t s, int64_t ntiles, int64_t* __restrict__ tile_cnt) {
  __shared__ int sh[B2_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * B2_TILE + (int64_t)warp * (32 * B2_SEL_R) + lane;
    const uint32_t bits = b2_eval_terms<B2_SEL_R>(s, row0);
    int c = __popc(bits);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(FULL_MASK, c, o);
    if (lane == 0) sh[warp] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
      int t = 0;
      for (int w = 0; w < B2_WARPS; ++w) t += sh[w];
      tile_cnt[tile] = t;
    }
    __syncthreads();
  }
}

// single-block exclusive scan in place: element i is read as io.get(i) and replaced by its exclusive
// prefix through io.put(i, prefix); returns the total (in every thread).  Run by one block of
// B2_SCAN_THREADS threads.
#define B2_SCAN_THREADS 1024
#define B2_SCAN_PER_THREAD 8
template <class IO>
__device__ __forceinline__ int64_t b2_block_exclusive_scan(const IO& io, int64_t n) {
  __shared__ int64_t warp_sums[32];
  __shared__ int64_t carry_sh;
  if (threadIdx.x == 0) carry_sh = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t chunk = (int64_t)B2_SCAN_THREADS * B2_SCAN_PER_THREAD;
  for (int64_t base = 0; base < n; base += chunk) {
    const int64_t i0 = base + (int64_t)threadIdx.x * B2_SCAN_PER_THREAD;
    int64_t v[B2_SCAN_PER_THREAD];
    int64_t tsum = 0;
#pragma unroll
    for (int k = 0; k < B2_SCAN_PER_THREAD; ++k) {
      v[k] = (i0 + k < n) ? io.get(i0 + k) : 0;
      tsum += v[k];
    }
    int64_t incl = tsum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int64_t t = __shfl_up_sync(FULL_MASK, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int64_t w = warp_sums[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int64_t t = __shfl_up_sync(FULL_MASK, w, o);
        if (lane >= o) w += t;
      }
      warp_sums[lane] = w;  // inclusive over warps
    }
    __syncthreads();
    const int64_t carry = carry_sh;
    int64_t excl = carry + (warp ? warp_sums[warp - 1] : 0) + (incl - tsum);
#pragma unroll
    for (int k = 0; k < B2_SCAN_PER_THREAD; ++k) {
      if (i0 + k < n) io.put(i0 + k, excl);
      excl += v[k];
    }
    __syncthreads();
    if (threadIdx.x == B2_SCAN_THREADS - 1) carry_sh = carry + warp_sums[31];
    __syncthreads();
  }
  return carry_sh;
}

struct b2_scan_io_i64 {
  int64_t* a;
  __device__ int64_t get(int64_t i) const { return a[i]; }
  __device__ void put(int64_t i, int64_t v) const { a[i] = v; }
};

// exclusive scan of int64 counts in place; a[n] receives the total.
__global__ void __launch_bounds__(B2_SCAN_THREADS)
b2_exclusive_scan_kernel(int64_t* __restrict__ a, int64_t n) {
  const int64_t total = b2_block_exclusive_scan(b2_scan_io_i64{a}, n);
  if (threadIdx.x == 0) a[n] = total;
}

struct b2_gather_arg {
  int32_t n;
  int32_t cols[B2_MAX_GATHER];
  void* out_data[B2_MAX_GATHER];
  uint32_t* out_valid[B2_MAX_GATHER];
};

__global__ void __launch_bounds__(B2_BLOCK)
b2_select_write_kernel(const __grid_constant__ b2_scan_t s, int64_t ntiles,
                       const int64_t* __restrict__ tile_off, int32_t* __restrict__ out_idx,
                       const __grid_constant__ b2_gather_arg g) {
  __shared__ int sh[B2_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lt_mask = (1u << lane) - 1;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * B2_TILE + (int64_t)warp * (32 * B2_SEL_R) + lane;
    const uint32_t bits = b2_eval_terms<B2_SEL_R>(s, row0);
    uint32_t ballots[B2_SEL_R];
    int wtotal = 0;
#pragma unroll
    for (int j = 0; j < B2_SEL_R; ++j) {
      ballots[j] = __ballot_sync(FULL_MASK, (bits >> j) & 1);
      wtotal += __popc(ballots[j]);
    }
    if (lane == 0) sh[warp] = wtotal;
    __syncthreads();
    int64_t off = tile_off[tile];
    for (int w = 0; w < warp; ++w) off += sh[w];
    __syncthreads();
    // ranks of this lane's rows
    int64_t pos[B2_SEL_R];
#pragma unroll
    for (int j = 0; j < B2_SEL_R; ++j) {
      pos[j] = ((bits >> j) & 1) ? off + __popc(ballots[j] & lt_mask) : -1;
      off += __popc(ballots[j]);
    }
    if (out_idx) {
#pragma unroll
      for (int j = 0; j < B2_SEL_R; ++j)
        if (pos[j] >= 0) out_idx[pos[j]] = (int32_t)(row0 - tile * B2_TILE + (int64_t)j * 32 + tile * B2_TILE);
    }
    for (int k = 0; k < g.n; ++k) {
      const b2_col_t& c = s.cols[g.cols[k]];
      if (c.dtype == B2_U8) {
        uint8_t* o = reinterpret_cast<uint8_t*>(g.out_data[k]);
        const uint8_t* p = reinterpret_cast<const uint8_t*>(c.data);
#pragma unroll
        for (int j = 0; j < B2_SEL_R; ++j)
          if (pos[j] >= 0) o[pos[j]] = p[row0 + (int64_t)j * 32];
      } else {
        int64_t* o = reinterpret_cast<int64_t*>(g.out_data[k]);
        int64_t raw[B2_SEL_R];
#pragma unroll
        for (int j = 0; j < B2_SEL_R; ++j)
          raw[j] = pos[j] >= 0 ? b2_ld_stream(reinterpret_cast<const int64_t*>(c.data) + row0 + (int64_t)j * 32) : 0;
#pragma unroll
        for (int j = 0; j < B2_SEL_R; ++j)
          if (pos[j] >= 0) o[pos[j]] = raw[j];
      }
      if (g.out_valid[k]) {
        uint32_t* ov = g.out_valid[k];
#pragma unroll
        for (int j = 0; j < B2_SEL_R; ++j)
          if (pos[j] >= 0 && (!c.valid || b2_bit(c.valid, row0 + (int64_t)j * 32)))
            atomicOr(ov + (pos[j] >> 5), 1u << (pos[j] & 31));
      }
    }
  }
}

// out[i] = col[idx[i]]; idx -1 -> NULL
__global__ void __launch_bounds__(B2_BLOCK)
b2_gather_kernel(const __grid_constant__ b2_col_t c, const int32_t* __restrict__ idx, int64_t n,
                 void* __restrict__ out, uint32_t* __restrict__ out_valid) {
  const int64_t n32 = (n + 31) & ~(int64_t)31;
  for (int64_t i = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; i < n32;
       i += (int64_t)gridDim.x * B2_BLOCK) {
    bool ok = false;
    if (i < n) {
      const int32_t r = idx[i];
      ok = r >= 0 && (!c.valid || b2_bit(c.valid, r));
      if (c.dtype == B2_U8) {
        reinterpret_cast<uint8_t*>(out)[i] = r >= 0 ? reinterpret_cast<const uint8_t*>(c.data)[r] : 0;
      } else {
        int64_t v = r >= 0 ? __ldg(reinterpret_cast<const long long*>(c.data) + r) : 0;
        if (r < 0 && c.dtype == B2_F64) v = 0x7ff8000000000000LL;  // NaN fill, like pandas take(-1)
        reinterpret_cast<int64_t*>(out)[i] = v;
      }
    }
    if (out_valid) {
      const uint32_t w = __ballot_sync(FULL_MASK, ok);
      if ((threadIdx.x & 31) == 0) out_valid[i >> 5] = w;
    }
  }
}

extern "C" {

int64_t b2_scan_agg_ws_bytes(void) { return (int64_t)sizeof(b2_partial) * B2_MAX_PARTIALS; }

static int32_t b2_check_scan(const b2_scan_t* s) {
  B2_REQUIRE(s, "null scan");
  B2_REQUIRE(s->ncols >= 0 && s->ncols <= B2_MAX_COLS, "bad ncols");
  B2_REQUIRE(s->nterms >= 0 && s->nterms <= B2_MAX_TERMS, "bad nterms");
  B2_REQUIRE(s->n >= 0 && s->n < ((int64_t)1 << 31), "partition must hold < 2^31 rows");
  for (int t = 0; t < s->nterms; ++t) {
    B2_REQUIRE(s->terms[t].col >= 0 && s->terms[t].col < s->ncols, "term column out of range");
    B2_REQUIRE(s->terms[t].op >= B2_EQ && s->terms[t].op <= B2_IS_TRUE, "bad term op");
  }
  return B2_OK;
}
static int32_t b2_check_aggs(const b2_scan_t* s, const b2_agg_t* aggs, int32_t naggs, b2_aggs_arg* out) {
  B2_REQUIRE(naggs >= 0 && naggs <= B2_MAX_AGGS, "bad naggs");
  B2_REQUIRE(naggs == 0 || aggs, "null aggs");
  memset(out, 0, sizeof(*out));
  out->n = naggs;
  for (int a = 0; a < naggs; ++a) {
    B2_REQUIRE(aggs[a].col >= -1 && aggs[a].col < s->ncols, "agg column out of range");
    B2_REQUIRE(aggs[a].op >= B2_AGG_SUM && aggs[a].op <= B2_AGG_XOR, "bad agg op");
    B2_REQUIRE(aggs[a].op < B2_AGG_AND || aggs[a].col < 0 || s->cols[aggs[a].col].dtype != B2_F64,
               "bitwise aggregates take int64 or boolean inputs");
    out->a[a] = aggs[a];
  }
  return B2_OK;
}

int32_t b2_scan_agg(const b2_scan_t* scan, const b2_agg_t* aggs, int32_t naggs, int64_t* d_out_acc,
                    int64_t* d_out_cnt, int32_t accumulate, void* ws, void* stream) {
  int32_t rc = b2_check_scan(scan);
  if (rc) return rc;
  b2_aggs_arg aa;
  rc = b2_check_aggs(scan, aggs, naggs, &aa);
  if (rc) return rc;
  B2_REQUIRE(d_out_acc && d_out_cnt && ws, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  b2_pipe_t pp;
  b2_make_pipe(*scan, &pp);
  b2_partial* partials = reinterpret_cast<b2_partial*>(ws);
  bool bits = false;
  for (int a = 0; a < naggs; ++a) bits |= aa.a[a].op >= B2_AGG_AND;
  int grid;
  if (pp.enabled) {
    auto k = bits ? b2_scan_agg_kernel<true, true> : b2_scan_agg_kernel<true, false>;
    grid = b2_pipe_grid(k, pp, scan->n);
    if (grid > B2_MAX_PARTIALS) grid = B2_MAX_PARTIALS;
    k<<<grid, B2_PIPE_THREADS, pp.smem_bytes, st>>>(*scan, pp, aa, partials);
  } else {
    auto k = bits ? b2_scan_agg_kernel<false, true> : b2_scan_agg_kernel<false, false>;
    int64_t nblk = (scan->n + B2_AGG_ROWS_PER_BLOCK - 1) / B2_AGG_ROWS_PER_BLOCK;
    grid = b2_wave_grid(k, B2_BLOCK, nblk);
    if (grid > B2_MAX_PARTIALS) grid = B2_MAX_PARTIALS;
    k<<<grid, B2_BLOCK, 0, st>>>(*scan, pp, aa, partials);
  }
  B2_CHECK_LAUNCH("b2_scan_agg_kernel");
  if (naggs > 0) {
    b2_final_arg fa;
    memset(&fa, 0, sizeof(fa));
    fa.n = naggs;
    for (int a = 0; a < naggs; ++a) {
      fa.op[a] = aa.a[a].op;
      fa.dtype[a] = aa.a[a].col >= 0 ? scan->cols[aa.a[a].col].dtype : B2_I64;
    }
    b2_scan_agg_final_kernel<<<naggs, B2_BLOCK, 0, st>>>(fa, partials, grid, d_out_acc, d_out_cnt, accumulate);
  }
  B2_CHECK_LAUNCH("b2_scan_agg_final_kernel");
  return B2_OK;
}

int32_t b2_select_count(const b2_scan_t* scan, int64_t* d_tile_off, void* stream) {
  int32_t rc = b2_check_scan(scan);
  if (rc) return rc;
  B2_REQUIRE(d_tile_off, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t ntiles = b2_num_tiles(scan->n);
  if (ntiles > 0) {
    int grid = b2_wave_grid(b2_select_count_kernel, B2_BLOCK, ntiles);
    b2_select_count_kernel<<<grid, B2_BLOCK, 0, st>>>(*scan, ntiles, d_tile_off);
    B2_CHECK_LAUNCH("b2_select_count_kernel");
  }
  b2_exclusive_scan_kernel<<<1, B2_SCAN_THREADS, 0, st>>>(d_tile_off, ntiles);
  B2_CHECK_LAUNCH("b2_exclusive_scan_kernel");
  return B2_OK;
}

int32_t b2_select_write(const b2_scan_t* scan, const int64_t* d_tile_off, int32_t* out_idx,
                        int32_t ngather, const int32_t* gather_cols, void* const* out_data,
                        uint32_t* const* out_valid, void* stream) {
  int32_t rc = b2_check_scan(scan);
  if (rc) return rc;
  B2_REQUIRE(d_tile_off, "null argument");
  B2_REQUIRE(ngather >= 0 && ngather <= B2_MAX_GATHER, "bad ngather");
  b2_gather_arg g;
  memset(&g, 0, sizeof(g));
  g.n = ngather;
  for (int k = 0; k < ngather; ++k) {
    B2_REQUIRE(gather_cols[k] >= 0 && gather_cols[k] < scan->ncols, "gather column out of range");
    B2_REQUIRE(out_data[k], "null gather output");
    g.cols[k] = gather_cols[k];
    g.out_data[k] = out_data[k];
    g.out_valid[k] = out_valid ? out_valid[k] : nullptr;
  }
  const int64_t ntiles = b2_num_tiles(scan->n);
  if (ntiles == 0) return B2_OK;
  int grid = b2_wave_grid(b2_select_write_kernel, B2_BLOCK, ntiles);
  b2_select_write_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(*scan, ntiles, d_tile_off, out_idx, g);
  B2_CHECK_LAUNCH("b2_select_write_kernel");
  return B2_OK;
}

int32_t b2_gather(const b2_col_t* col, const int32_t* idx, int64_t n_idx, void* out_data,
                  uint32_t* out_valid, void* stream) {
  B2_REQUIRE(col && out_data, "null argument");
  if (n_idx <= 0) return B2_OK;
  B2_REQUIRE(idx, "null idx");
  int grid = b2_wave_grid(b2_gather_kernel, B2_BLOCK, (n_idx + B2_BLOCK - 1) / B2_BLOCK);
  b2_gather_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(*col, idx, n_idx, out_data, out_valid);
  B2_CHECK_LAUNCH("b2_gather_kernel");
  return B2_OK;
}

}  // extern "C"
