// window.cuh — window functions over the order b2_sort_by leaves in idx (partition keys, then order keys).
// The reference computes them with pandas groupby().rolling / expanding per partition
// (dask_sql/physical/rel/logical/window.py); here the sorted positions get partition / peer-group head flags
// (b2_window_heads), segmented scans turn them into start / end positions, ranks and prefix sums
// (b2_window_positions, b2_window_scan), and one kernel per function evaluates every row's frame
// (b2_window_frame): SUM / COUNT / AVG as prefix differences, MIN / MAX from a running scan or a sparse
// table, FIRST_VALUE / LAST_VALUE as reads at the frame's ends.
#pragma once
#include "common.cuh"
#include "sort.cuh"

#define B2_WIN_ITEMS 8                              // consecutive positions per thread in a scan tile
#define B2_WIN_TILE (B2_BLOCK * B2_WIN_ITEMS)

// ---------------------------------------------------------------------------------------------
// heads
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(B2_BLOCK)
b2_window_heads_kernel(const __grid_constant__ b2_col_t c, const int32_t* __restrict__ idx, int64_t n, uint8_t bits,
                       uint8_t* __restrict__ flags) {
  for (int64_t i = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; i < n; i += (int64_t)gridDim.x * B2_BLOCK) {
    bool differs = i == 0;
    if (!differs) {
      bool na, nb;
      const uint64_t a = b2_sort_key_image(c, idx[i - 1], na);
      const uint64_t b = b2_sort_key_image(c, idx[i], nb);
      differs = na != nb || (!na && a != b);
    }
    if (differs) flags[i] |= i == 0 ? 3 : bits;   // position 0 starts everything
  }
}

// ---------------------------------------------------------------------------------------------
// segmented scans: reduce each tile, scan the tile totals in one block, rescan each tile with its carry
// ---------------------------------------------------------------------------------------------
// An Op supplies S (the state), identity(), combine(a, b) (a before b), and over scan positions j:
// head(j) (a segment starts at j), load(j) and store(j, inclusive state).
template <class S>
struct b2_seg_t {
  S s;
  int h;
};

template <class Op, class S>
__device__ __forceinline__ void b2_seg_add(S& run, int& h, const S& x, int xh) {   // run = run (+) x
  if (xh) { run = x; h = 1; } else { run = Op::combine(run, x); }
}

// inclusive segmented scan of (s, h) over the threads of the block, in thread order
template <class Op, class S>
__device__ __forceinline__ void b2_block_seg_scan(S& s, int& h, b2_seg_t<S>* sh) {
  const int t = threadIdx.x;
  for (int off = 1; off < B2_BLOCK; off <<= 1) {
    sh[t].s = s;
    sh[t].h = h;
    __syncthreads();
    if (t >= off && !h) {
      s = Op::combine(sh[t - off].s, s);
      h = sh[t - off].h;
    }
    __syncthreads();
  }
}

// this thread's total over its B2_WIN_ITEMS positions of the tile
template <class Op, class S>
__device__ __forceinline__ void b2_thread_total(const Op& op, int64_t j0, int64_t n, S& s, int& h) {
  s = Op::identity();
  h = 0;
#pragma unroll
  for (int k = 0; k < B2_WIN_ITEMS; ++k) {
    const int64_t j = j0 + k;
    if (j < n) b2_seg_add<Op>(s, h, op.load(j), op.head(j));
  }
}

template <class Op, class S>
__global__ void __launch_bounds__(B2_BLOCK)
b2_window_reduce_kernel(const Op op, int64_t n, b2_seg_t<S>* __restrict__ tiles) {
  __shared__ b2_seg_t<S> sh[B2_BLOCK];
  S s;
  int h;
  b2_thread_total(op, (int64_t)blockIdx.x * B2_WIN_TILE + (int64_t)threadIdx.x * B2_WIN_ITEMS, n, s, h);
  b2_block_seg_scan<Op>(s, h, sh);
  if (threadIdx.x == B2_BLOCK - 1) tiles[blockIdx.x] = b2_seg_t<S>{s, h};
}

// carry[t] = segmented total of tiles [0, t) (one block; each thread takes a contiguous run of tiles)
template <class Op, class S>
__global__ void __launch_bounds__(B2_BLOCK)
b2_window_carry_kernel(const b2_seg_t<S>* __restrict__ tiles, int64_t ntiles, b2_seg_t<S>* __restrict__ carry) {
  __shared__ b2_seg_t<S> sh[B2_BLOCK];
  const int64_t per = (ntiles + B2_BLOCK - 1) / B2_BLOCK;
  const int64_t t0 = (int64_t)threadIdx.x * per;
  const int64_t t1 = t0 + per < ntiles ? t0 + per : ntiles;
  S s = Op::identity();
  int h = 0;
  for (int64_t t = t0; t < t1; ++t) b2_seg_add<Op>(s, h, tiles[t].s, tiles[t].h);
  b2_block_seg_scan<Op>(s, h, sh);
  sh[threadIdx.x].s = s;
  sh[threadIdx.x].h = h;
  __syncthreads();
  S run = threadIdx.x ? sh[threadIdx.x - 1].s : Op::identity();
  int rh = threadIdx.x ? sh[threadIdx.x - 1].h : 0;
  for (int64_t t = t0; t < t1; ++t) {
    carry[t] = b2_seg_t<S>{run, rh};
    b2_seg_add<Op>(run, rh, tiles[t].s, tiles[t].h);
  }
}

template <class Op, class S>
__global__ void __launch_bounds__(B2_BLOCK)
b2_window_rescan_kernel(const Op op, int64_t n, const b2_seg_t<S>* __restrict__ carry) {
  __shared__ b2_seg_t<S> sh[B2_BLOCK];
  const int64_t j0 = (int64_t)blockIdx.x * B2_WIN_TILE + (int64_t)threadIdx.x * B2_WIN_ITEMS;
  S s;
  int h;
  b2_thread_total(op, j0, n, s, h);
  b2_block_seg_scan<Op>(s, h, sh);
  sh[threadIdx.x].s = s;
  sh[threadIdx.x].h = h;
  __syncthreads();
  S run = carry[blockIdx.x].s;
  int rh = carry[blockIdx.x].h;
  if (threadIdx.x) b2_seg_add<Op>(run, rh, sh[threadIdx.x - 1].s, sh[threadIdx.x - 1].h);
#pragma unroll
  for (int k = 0; k < B2_WIN_ITEMS; ++k) {
    const int64_t j = j0 + k;
    if (j < n) {
      b2_seg_add<Op>(run, rh, op.load(j), op.head(j));
      op.store(j, run);
    }
  }
}

template <class Op>
static int32_t b2_window_run_scan(const Op& op, int64_t n, void* ws, cudaStream_t st) {
  typedef typename Op::S S;
  const int64_t ntiles = (n + B2_WIN_TILE - 1) / B2_WIN_TILE;
  b2_seg_t<S>* tiles = reinterpret_cast<b2_seg_t<S>*>(ws);
  b2_seg_t<S>* carry = tiles + ntiles;
  b2_window_reduce_kernel<Op, S><<<(int)ntiles, B2_BLOCK, 0, st>>>(op, n, tiles);
  b2_window_carry_kernel<Op, S><<<1, B2_BLOCK, 0, st>>>(tiles, ntiles, carry);
  b2_window_rescan_kernel<Op, S><<<(int)ntiles, B2_BLOCK, 0, st>>>(op, n, carry);
  B2_CHECK_LAUNCH("b2_window scan kernels");
  return B2_OK;
}

// partition / peer starts, DENSE_RANK, and the ends written at the start positions
struct b2_win_pos_state {
  int32_t ps, qs, dn;
};
struct b2_win_pos_op {
  typedef b2_win_pos_state S;
  const uint8_t* flags;
  int64_t n;
  int32_t *ps, *qs, *dn, *pend, *qend;
  __device__ static S identity() { return S{-1, -1, 0}; }
  __device__ static S combine(const S& a, const S& b) {
    return S{a.ps > b.ps ? a.ps : b.ps, a.qs > b.qs ? a.qs : b.qs, a.dn + b.dn};
  }
  __device__ int head(int64_t j) const { return flags[j] & 1; }
  __device__ S load(int64_t j) const {
    const uint8_t f = flags[j];
    return S{(f & 1) ? (int32_t)j : -1, (f & 2) ? (int32_t)j : -1, (f & 2) ? 1 : 0};
  }
  __device__ void store(int64_t j, const S& s) const {
    ps[j] = s.ps;
    qs[j] = s.qs;
    dn[j] = s.dn;
    const uint8_t next = j + 1 < n ? flags[j + 1] : 3;
    if (next & 1) pend[s.ps] = (int32_t)j;
    if (next & 2) qend[s.qs] = (int32_t)j;
  }
};

// scans of a sorted argument column; scan position j is sorted position j, or n-1-j when reversed
struct b2_win_val_base {
  const uint8_t* flags;
  b2_col_t val;
  int64_t n;
  int32_t seg_mask, reverse;
  b2_win_prefix_t out;
  __device__ int64_t pos(int64_t j) const { return reverse ? n - 1 - j : j; }
  __device__ int head(int64_t j) const {
    if (!reverse) return flags[j] & seg_mask;
    const int64_t p = n - 1 - j;              // a reversed segment starts at a forward segment's last position
    return p + 1 >= n || (flags[p + 1] & seg_mask);
  }
  __device__ int64_t raw(int64_t p, bool& isnull) const {
    const int64_t r = b2_load_raw(val, p);
    isnull = b2_is_null(val, p, r);
    return r;
  }
};

struct b2_win_sumi_state {
  int64_t s;
  int32_t c;
};
struct b2_win_sumi_op : b2_win_val_base {
  typedef b2_win_sumi_state S;
  __device__ static S identity() { return S{0, 0}; }
  __device__ static S combine(const S& a, const S& b) {
    return S{(int64_t)((uint64_t)a.s + (uint64_t)b.s), a.c + b.c};   // wraps as the GROUP BY SUM does
  }
  __device__ S load(int64_t j) const {
    bool isnull;
    const int64_t r = raw(pos(j), isnull);
    return isnull ? S{0, 0} : S{r, 1};
  }
  __device__ void store(int64_t j, const S& s) const {
    const int64_t p = pos(j);
    reinterpret_cast<int64_t*>(out.val)[p] = s.s;
    if (out.cnt) out.cnt[p] = s.c;
  }
};

// double-double sum of the finite values, infinities counted apart so that prefix differences stay exact
struct b2_win_sumf_state {
  double hi, lo;
  int32_t c, pinf, ninf;
};
__device__ __forceinline__ void b2_two_sum(double a, double b, double& s, double& e) {
  s = a + b;
  const double bb = s - a;
  e = (a - (s - bb)) + (b - bb);
}
__device__ __forceinline__ void b2_fast_two_sum(double a, double b, double& s, double& e) {   // |a| >= |b|
  s = a + b;
  e = b - (s - a);
}
__device__ __forceinline__ void b2_dd_add(double ahi, double alo, double bhi, double blo, double& hi, double& lo) {
  double s, e;
  b2_two_sum(ahi, bhi, s, e);
  e += alo + blo;
  b2_fast_two_sum(s, e, hi, lo);
  if (!isfinite(hi)) lo = 0.0;                 // a finite sum that overflowed: keep the infinity
}
struct b2_win_sumf_op : b2_win_val_base {
  typedef b2_win_sumf_state S;
  __device__ static S identity() { return S{0.0, 0.0, 0, 0, 0}; }
  __device__ static S combine(const S& a, const S& b) {
    S r;
    b2_dd_add(a.hi, a.lo, b.hi, b.lo, r.hi, r.lo);
    r.c = a.c + b.c;
    r.pinf = a.pinf + b.pinf;
    r.ninf = a.ninf + b.ninf;
    return r;
  }
  __device__ S load(int64_t j) const {
    bool isnull;
    const int64_t r = raw(pos(j), isnull);
    if (isnull) return identity();
    const double x = val.dtype == B2_F64 ? __longlong_as_double(r) : (double)r;
    if (isinf(x)) return S{0.0, 0.0, 1, x > 0, x < 0};
    return S{x, 0.0, 1, 0, 0};
  }
  __device__ void store(int64_t j, const S& s) const {
    const int64_t p = pos(j);
    reinterpret_cast<double*>(out.val)[p] = s.hi;
    out.lo[p] = s.lo;
    out.pinf[p] = s.pinf;
    out.ninf[p] = s.ninf;
    if (out.cnt) out.cnt[p] = s.c;
  }
};

// MIN / MAX order image: the int64 value, or b2_ordered_from_bits of a double (-0.0 below +0.0, as the
// GROUP BY MIN / MAX order them)
__device__ __forceinline__ int64_t b2_win_image(const b2_col_t& c, int64_t raw) {
  return c.dtype == B2_F64 ? b2_ordered_from_bits(raw) : raw;
}

struct b2_win_ext_state {
  int64_t m;
  int32_t c;
};
template <bool MAX>
struct b2_win_ext_op : b2_win_val_base {
  typedef b2_win_ext_state S;
  __device__ static S identity() { return S{MAX ? INT64_MIN : INT64_MAX, 0}; }
  __device__ static S combine(const S& a, const S& b) {
    return S{MAX ? (a.m > b.m ? a.m : b.m) : (a.m < b.m ? a.m : b.m), a.c + b.c};
  }
  __device__ S load(int64_t j) const {
    bool isnull;
    const int64_t r = raw(pos(j), isnull);
    return isnull ? identity() : S{b2_win_image(val, r), 1};
  }
  __device__ void store(int64_t j, const S& s) const {
    const int64_t p = pos(j);
    reinterpret_cast<int64_t*>(out.val)[p] = s.m;
    if (out.cnt) out.cnt[p] = s.c;
  }
};

// ---------------------------------------------------------------------------------------------
// sparse table of MIN / MAX images
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(B2_BLOCK)
b2_window_rmq_base_kernel(const __grid_constant__ b2_col_t c, int64_t n, int is_max, int64_t* __restrict__ t0) {
  for (int64_t i = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; i < n; i += (int64_t)gridDim.x * B2_BLOCK) {
    const int64_t r = b2_load_raw(c, i);
    t0[i] = b2_is_null(c, i, r) ? (is_max ? INT64_MIN : INT64_MAX) : b2_win_image(c, r);
  }
}

__global__ void __launch_bounds__(B2_BLOCK)
b2_window_rmq_level_kernel(const int64_t* __restrict__ prev, int64_t n, int64_t half, int is_max,
                           int64_t* __restrict__ next) {
  for (int64_t i = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; i < n; i += (int64_t)gridDim.x * B2_BLOCK) {
    const int64_t a = prev[i];
    const int64_t b = prev[i + half < n ? i + half : n - 1];   // past the end: never read by a query
    next[i] = is_max ? (a > b ? a : b) : (a < b ? a : b);
  }
}

// ---------------------------------------------------------------------------------------------
// frame evaluation
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int32_t b2_win_frame_cnt(const int32_t* cnt, int64_t lo, int64_t hi, int64_t ps) {
  return cnt[hi] - (lo > ps ? cnt[lo - 1] : 0);
}

__global__ void __launch_bounds__(B2_BLOCK)
b2_window_frame_kernel(const __grid_constant__ b2_win_frame_t f) {
  const int64_t n = f.n;
  const int64_t stride = (int64_t)gridDim.x * B2_BLOCK;
  // whole warps iterate together, so that each warp's validity word is one ballot
  for (int64_t base = (int64_t)blockIdx.x * B2_BLOCK; base < n; base += stride) {
    const int64_t i = base + threadIdx.x;
    const bool live = i < n;
    bool valid = false;
    if (live) {
      const int64_t ps = f.ps[i];
      const int64_t pe = f.pend[ps];
      int64_t lo, hi;
      if (f.range) {
        const int64_t qs = f.qs[i];
        lo = f.lo <= -B2_WIN_UNBOUNDED ? ps : f.lo >= B2_WIN_UNBOUNDED ? pe + 1 : qs;
        hi = f.hi >= B2_WIN_UNBOUNDED ? pe : f.hi <= -B2_WIN_UNBOUNDED ? ps - 1 : f.qend[qs];
      } else {
        lo = f.lo <= -B2_WIN_UNBOUNDED ? ps : f.lo >= B2_WIN_UNBOUNDED ? pe + 1 : i + f.lo;
        hi = f.hi >= B2_WIN_UNBOUNDED ? pe : f.hi <= -B2_WIN_UNBOUNDED ? ps - 1 : i + f.hi;
      }
      if (lo < ps) lo = ps;
      if (hi > pe) hi = pe;
      const bool empty = lo > hi;
      int64_t iv = 0;
      double dv = 0.0;
      bool is_f = false;
      switch (f.fn) {
        case B2_WF_ROW_NUMBER: iv = i - ps + 1; valid = true; break;
        case B2_WF_RANK: iv = f.qs[i] - ps + 1; valid = true; break;
        case B2_WF_DENSE_RANK: iv = f.dn[i]; valid = true; break;
        case B2_WF_COUNT_STAR: iv = empty ? 0 : hi - lo + 1; valid = true; break;
        case B2_WF_COUNT: iv = empty ? 0 : b2_win_frame_cnt(f.pre.cnt, lo, hi, ps); valid = true; break;
        case B2_WF_SUM_I: {
          if (!empty && b2_win_frame_cnt(f.pre.cnt, lo, hi, ps) > 0) {
            const int64_t* p = reinterpret_cast<const int64_t*>(f.pre.val);
            iv = (int64_t)((uint64_t)p[hi] - (lo > ps ? (uint64_t)p[lo - 1] : 0ull));
            valid = true;
          }
          break;
        }
        case B2_WF_SUM_F:
        case B2_WF_AVG: {
          is_f = true;
          const int32_t c = empty ? 0 : b2_win_frame_cnt(f.pre.cnt, lo, hi, ps);
          if (c > 0) {
            const double* ph = reinterpret_cast<const double*>(f.pre.val);
            const bool cut = lo > ps;
            const int32_t pinf = f.pre.pinf[hi] - (cut ? f.pre.pinf[lo - 1] : 0);
            const int32_t ninf = f.pre.ninf[hi] - (cut ? f.pre.ninf[lo - 1] : 0);
            if (pinf && ninf) {
              dv = __longlong_as_double(0x7ff8000000000000LL);
            } else if (pinf || ninf) {
              dv = pinf ? INFINITY : -INFINITY;
            } else {
              double hi_, lo_;
              b2_dd_add(ph[hi], f.pre.lo[hi], cut ? -ph[lo - 1] : 0.0, cut ? -f.pre.lo[lo - 1] : 0.0, hi_, lo_);
              dv = hi_ + lo_;
            }
            if (f.fn == B2_WF_AVG) dv = dv / (double)c;
            valid = true;
          }
          break;
        }
        case B2_WF_MIN:
        case B2_WF_MAX: {
          if (empty) break;
          const b2_win_prefix_t* src = nullptr;
          int64_t at = hi;
          if (lo == ps) {
            src = &f.pre;
          } else if (hi == pe && f.suf.val) {
            src = &f.suf;
            at = lo;
          } else if (f.peer.val && lo == f.qs[hi] && hi == f.qend[lo]) {
            src = &f.peer;
          }
          int64_t img;
          if (src) {
            if (src->cnt[at] == 0) break;
            img = reinterpret_cast<const int64_t*>(src->val)[at];
          } else {
            if (b2_win_frame_cnt(f.pre.cnt, lo, hi, ps) == 0) break;
            const uint64_t w = (uint64_t)(hi - lo + 1);
            const int k = 63 - __clzll((long long)w);
            const int64_t a = f.rmq[(int64_t)k * n + lo], b = f.rmq[(int64_t)k * n + hi - ((int64_t)1 << k) + 1];
            img = f.fn == B2_WF_MAX ? (a > b ? a : b) : (a < b ? a : b);
          }
          if (f.val.dtype == B2_F64) {
            is_f = true;
            dv = __longlong_as_double(b2_ordered_from_bits(img));
          } else {
            iv = img;
          }
          valid = true;
          break;
        }
        default: {   // FIRST_VALUE / LAST_VALUE
          if (empty) break;
          const int64_t at = f.fn == B2_WF_FIRST_VALUE ? lo : hi;
          const int64_t r = b2_load_raw(f.val, at);
          valid = !b2_is_null(f.val, at, r);
          if (f.val.dtype == B2_U8) {
            reinterpret_cast<uint8_t*>(f.out)[i] = valid ? (uint8_t)r : 0;
            goto done;
          }
          is_f = f.val.dtype == B2_F64;
          iv = r;
          dv = __longlong_as_double(r);
          break;
        }
      }
      if (is_f) reinterpret_cast<double*>(f.out)[i] = valid ? dv : __longlong_as_double(0x7ff8000000000000LL);
      else reinterpret_cast<int64_t*>(f.out)[i] = valid ? iv : 0;
    }
  done:
    const uint32_t word = __ballot_sync(FULL_MASK, live && valid);
    if (f.out_valid && (threadIdx.x & 31) == 0 && live) f.out_valid[i >> 5] = word;
  }
}

__global__ void __launch_bounds__(B2_BLOCK)
b2_window_invert_kernel(const int32_t* __restrict__ idx, int64_t n, int32_t* __restrict__ inv) {
  for (int64_t i = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; i < n; i += (int64_t)gridDim.x * B2_BLOCK)
    inv[idx[i]] = (int32_t)i;
}

extern "C" {

int32_t b2_window_heads(const b2_col_t* key, const int32_t* idx, int64_t n, int32_t partition, uint8_t* flags,
                        void* stream) {
  B2_REQUIRE(key && idx && flags, "null argument");
  B2_REQUIRE(n >= 0 && n < ((int64_t)1 << 31), "window functions take < 2^31 rows");
  B2_REQUIRE(key->dtype == B2_I64 || key->dtype == B2_F64 || key->dtype == B2_U8, "bad key dtype");
  if (n == 0) return B2_OK;
  int grid = b2_wave_grid(b2_window_heads_kernel, B2_BLOCK, (n + B2_BLOCK - 1) / B2_BLOCK);
  b2_window_heads_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(*key, idx, n, partition ? 3 : 2, flags);
  B2_CHECK_LAUNCH("b2_window_heads_kernel");
  return B2_OK;
}

int64_t b2_window_ws_bytes(int64_t n) {
  const int64_t ntiles = (n + B2_WIN_TILE - 1) / B2_WIN_TILE;
  return 2 * ntiles * (int64_t)sizeof(b2_seg_t<b2_win_sumf_state>) + 256;
}

int32_t b2_window_positions(const uint8_t* flags, int64_t n, int32_t* ps, int32_t* qs, int32_t* dn, int32_t* pend,
                            int32_t* qend, void* ws, void* stream) {
  B2_REQUIRE(flags && ps && qs && dn && pend && qend && ws, "null argument");
  B2_REQUIRE(n >= 0 && n < ((int64_t)1 << 31), "window functions take < 2^31 rows");
  if (n == 0) return B2_OK;
  b2_win_pos_op op{flags, n, ps, qs, dn, pend, qend};
  return b2_window_run_scan(op, n, ws, (cudaStream_t)stream);
}

int32_t b2_window_scan(const uint8_t* flags, const b2_col_t* val, int64_t n, int32_t kind, int32_t seg_mask,
                       int32_t reverse, const b2_win_prefix_t* out, void* ws, void* stream) {
  B2_REQUIRE(flags && val && out && out->val && ws, "null argument");
  B2_REQUIRE(n >= 0 && n < ((int64_t)1 << 31), "window functions take < 2^31 rows");
  B2_REQUIRE(val->dtype == B2_I64 || val->dtype == B2_F64 || val->dtype == B2_U8, "bad value dtype");
  B2_REQUIRE(seg_mask == 1 || seg_mask == 2, "seg_mask is 1 (partitions) or 2 (peer groups)");
  B2_REQUIRE(kind >= B2_WIN_SUM_I && kind <= B2_WIN_MAX, "bad scan kind");
  B2_REQUIRE(kind != B2_WIN_SUM_F || (out->lo && out->pinf && out->ninf), "B2_WIN_SUM_F needs lo, pinf and ninf");
  if (n == 0) return B2_OK;
  const b2_win_val_base base{flags, *val, n, seg_mask, reverse ? 1 : 0, *out};
  cudaStream_t st = (cudaStream_t)stream;
  if (kind == B2_WIN_SUM_I) return b2_window_run_scan(b2_win_sumi_op{base}, n, ws, st);
  if (kind == B2_WIN_SUM_F) return b2_window_run_scan(b2_win_sumf_op{base}, n, ws, st);
  if (kind == B2_WIN_MIN) return b2_window_run_scan(b2_win_ext_op<false>{base}, n, ws, st);
  return b2_window_run_scan(b2_win_ext_op<true>{base}, n, ws, st);
}

int32_t b2_window_rmq(const b2_col_t* val, int64_t n, int32_t is_max, int32_t levels, int64_t* table,
                      void* stream) {
  B2_REQUIRE(val && table, "null argument");
  B2_REQUIRE(n >= 0 && n < ((int64_t)1 << 31), "window functions take < 2^31 rows");
  B2_REQUIRE(val->dtype == B2_I64 || val->dtype == B2_F64 || val->dtype == B2_U8, "bad value dtype");
  B2_REQUIRE(levels >= 1 && levels <= 32, "levels is 1 .. 32");
  if (n == 0) return B2_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int grid = b2_wave_grid(b2_window_rmq_base_kernel, B2_BLOCK, (n + B2_BLOCK - 1) / B2_BLOCK);
  b2_window_rmq_base_kernel<<<grid, B2_BLOCK, 0, st>>>(*val, n, is_max, table);
  grid = b2_wave_grid(b2_window_rmq_level_kernel, B2_BLOCK, (n + B2_BLOCK - 1) / B2_BLOCK);
  for (int k = 1; k < levels; ++k)
    b2_window_rmq_level_kernel<<<grid, B2_BLOCK, 0, st>>>(table + (int64_t)(k - 1) * n, n, (int64_t)1 << (k - 1),
                                                          is_max, table + (int64_t)k * n);
  B2_CHECK_LAUNCH("b2_window_rmq kernels");
  return B2_OK;
}

int32_t b2_window_frame(const b2_win_frame_t* f, void* stream) {
  B2_REQUIRE(f && f->ps && f->qs && f->dn && f->pend && f->qend && f->out, "null argument");
  B2_REQUIRE(f->n >= 0 && f->n < ((int64_t)1 << 31), "window functions take < 2^31 rows");
  B2_REQUIRE(f->fn >= B2_WF_ROW_NUMBER && f->fn <= B2_WF_LAST_VALUE, "bad window function");
  B2_REQUIRE(f->fn <= B2_WF_COUNT_STAR || f->out_valid || f->fn == B2_WF_COUNT, "out_valid is required");
  const auto unb_or_current = [](int64_t b) { return b == 0 || b == -B2_WIN_UNBOUNDED || b == B2_WIN_UNBOUNDED; };
  B2_REQUIRE(!f->range || (unb_or_current(f->lo) && unb_or_current(f->hi)), "RANGE bounds are UNBOUNDED or CURRENT ROW");
  B2_REQUIRE(f->lo >= -B2_WIN_UNBOUNDED && f->lo <= B2_WIN_UNBOUNDED && f->hi >= -B2_WIN_UNBOUNDED &&
             f->hi <= B2_WIN_UNBOUNDED, "bound outside +-B2_WIN_UNBOUNDED");
  const int fn = f->fn;
  B2_REQUIRE(fn < B2_WF_COUNT || fn > B2_WF_MAX || ((f->pre.val || fn == B2_WF_COUNT) && f->pre.cnt),
             "the function needs the forward partition scan (pre)");
  B2_REQUIRE((fn != B2_WF_SUM_F && fn != B2_WF_AVG) || (f->pre.lo && f->pre.pinf && f->pre.ninf),
             "SUM_F / AVG need a B2_WIN_SUM_F scan");
  B2_REQUIRE(fn < B2_WF_MIN || fn > B2_WF_MAX ||
             ((f->suf.val == nullptr || f->suf.cnt) && (f->peer.val == nullptr || f->peer.cnt)), "suf / peer need cnt");
  B2_REQUIRE(fn < B2_WF_MIN || f->val.data || fn == B2_WF_MIN || fn == B2_WF_MAX, "FIRST / LAST_VALUE need val");
  B2_REQUIRE(f->val.data == nullptr || f->val.dtype == B2_I64 || f->val.dtype == B2_F64 || f->val.dtype == B2_U8,
             "bad value dtype");
  if (fn == B2_WF_MIN || fn == B2_WF_MAX) {
    // frames of bounded width that start after the partition start and end before its end read the table
    // (hi < lo: every row's frame is empty, and the kernel returns NULL before it reads any table)
    const bool needs_rmq = !f->range && f->lo > -B2_WIN_UNBOUNDED && f->hi < B2_WIN_UNBOUNDED && f->hi >= f->lo;
    if (needs_rmq) {
      const int64_t w = f->hi - f->lo + 1 < f->n ? f->hi - f->lo + 1 : f->n;   // no frame is wider than n
      int need = 1;
      while (w > 0 && ((int64_t)1 << need) <= w) ++need;
      B2_REQUIRE(f->rmq && f->rmq_levels >= need, "the frame needs a sparse table of more levels");
    }
    B2_REQUIRE(!(f->hi >= B2_WIN_UNBOUNDED && f->lo > -B2_WIN_UNBOUNDED) || f->suf.val,
               "frames ending UNBOUNDED FOLLOWING need the reverse scan (suf)");
    B2_REQUIRE(!(f->range && f->lo == 0 && f->hi == 0) || f->peer.val,
               "RANGE CURRENT ROW .. CURRENT ROW needs the peer scan");
  }
  if (f->n == 0) return B2_OK;
  int grid = b2_wave_grid(b2_window_frame_kernel, B2_BLOCK, (f->n + B2_BLOCK - 1) / B2_BLOCK);
  b2_window_frame_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(*f);
  B2_CHECK_LAUNCH("b2_window_frame_kernel");
  return B2_OK;
}

int32_t b2_window_invert(const int32_t* idx, int64_t n, int32_t* inv, void* stream) {
  B2_REQUIRE((idx && inv) || n == 0, "null argument");
  B2_REQUIRE(n >= 0 && n < ((int64_t)1 << 31), "window functions take < 2^31 rows");
  if (n == 0) return B2_OK;
  int grid = b2_wave_grid(b2_window_invert_kernel, B2_BLOCK, (n + B2_BLOCK - 1) / B2_BLOCK);
  b2_window_invert_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(idx, n, inv);
  B2_CHECK_LAUNCH("b2_window_invert_kernel");
  return B2_OK;
}

}  // extern "C"
