// joinagg.cuh — inner join on a unique dense key fused with GLOBAL aggregates over expressions
// that mix both sides (C3's non-materialising variant: SELECT SUM(f.v * d.w) FROM fact f JOIN dim d
// ON f.fk = d.pk).  The reference materialises the whole join (join.py:241-246: merge = factorize +
// two indexers + take on every column) and then reduces it (aggregate.py:305-306,576: constant-key
// groupby); here one pass over the probe partition does predicate -> presence/payload lookup at the
// key offset -> combine -> per-thread accumulators, nothing is written but 2 x naggs words.
//
// The build side is the key-ordered layout of b2_join_key_layout (jt->dense == 2): `lookup` is the
// presence bitmap and payload column b holds build value at [key - kmin] (int64 / float64, or uint32
// offsets from bbase[b]).
#pragma once
#include "common.cuh"
#include "filter.cuh"

#define B2_JA_R 8
#define B2_JA_ROWS_PER_BLOCK (B2_BLOCK * B2_JA_R)

struct b2_joinagg_arg {
  b2_joinagg_t a[B2_MAX_AGGS];
  int32_t n;
  int32_t nb;
  b2_col_t bcols[B2_JA_MAX_BUILD];
  int64_t bbase[B2_JA_MAX_BUILD];
};

// build value of one matched row as a raw 64-bit word of the payload's LOGICAL type
__device__ __forceinline__ int64_t b2_ja_payload(const b2_col_t& c, int64_t base, uint32_t d) {
  if (c.dtype == B2_U32) return base + (int64_t)(uint32_t)b2_ld_keep_i32(reinterpret_cast<const int32_t*>(c.data) + d);
  return b2_ld_keep_i64(reinterpret_cast<const int64_t*>(c.data) + d);
}

template <int R>
__device__ __forceinline__ void b2_join_agg_body(const b2_scan_t& s, const b2_gld& ld, int key_col,
                                                 const b2_jointable_t& jt, const b2_joinagg_arg& ja,
                                                 int64_t (*sh_acc)[B2_BLOCK], int32_t (*sh_cnt)[B2_BLOCK], int tid) {
  const b2_col_t& kc = s.cols[key_col];
  // trip 1: the join key is requested together with the predicate columns.  Only the key OFFSETS are
  // kept (32 bits: a key-ordered table spans < 2^31 keys), the keys themselves die here.
  uint32_t d[R];
  uint32_t inr = 0;
  {
    bool full0;
    const uint32_t inb = b2_bounds_bits<R>(ld.row0, s.n, full0);
    int64_t key[R];
    ld.template load<R>(key_col, inb, full0, key);
    bool full;
    const uint32_t bits = b2_eval_terms<R>(s, ld, full);
    uint32_t live = bits;
    if (kc.valid) live &= b2_valid_bits<R>(kc.valid, ld.row0, bits);
    const uint64_t range = (uint64_t)jt.range;
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const uint64_t dd = (uint64_t)key[j] - (uint64_t)jt.kmin;
      inr |= (uint32_t)(((live >> j) & 1) && dd < range) << j;
      d[j] = (uint32_t)dd;
    }
  }
  // trip 2: presence words, and -- speculatively, for every in-range row -- both inputs of the first
  // aggregate (the payload at an offset without a build row is garbage that nobody reads)
  const b2_joinagg_t a0 = ja.a[0];
  const bool pre_b = ja.n > 0 && a0.bcol >= 0 && ja.bcols[a0.bcol].dtype != B2_U8;
  const bool pre_p = ja.n > 0 && a0.pcol >= 0 && s.cols[a0.pcol].dtype != B2_U8;
  int64_t pb[R], pp[R];
  uint32_t matched = 0;
  if (pre_b && (ja.bcols[a0.bcol].flags & B2_COL_SENTINEL)) {
    // the payload marks absent keys itself (0xFFFFFFFF): no presence-bitmap request at all
    const int32_t* pay32 = reinterpret_cast<const int32_t*>(ja.bcols[a0.bcol].data);
    const int64_t base = ja.bbase[a0.bcol];
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const uint32_t raw = (inr >> j) & 1 ? (uint32_t)b2_ld_keep_i32(pay32 + d[j]) : 0xffffffffu;
      matched |= (uint32_t)(raw != 0xffffffffu) << j;
      pb[j] = base + (int64_t)raw;
    }
    if (pre_p) ld.template load<R>(a0.pcol, inr, false, pp);
  } else {
    uint32_t word[R];
#pragma unroll
    for (int j = 0; j < R; ++j) word[j] = (inr >> j) & 1 ? (uint32_t)b2_ld_keep_i32(jt.lookup + (d[j] >> 5)) : 0u;
    if (pre_b) {
#pragma unroll
      for (int j = 0; j < R; ++j) pb[j] = (inr >> j) & 1 ? b2_ja_payload(ja.bcols[a0.bcol], ja.bbase[a0.bcol], d[j]) : 0;
    }
    if (pre_p) ld.template load<R>(a0.pcol, inr, false, pp);
#pragma unroll
    for (int j = 0; j < R; ++j) matched |= ((word[j] >> (d[j] & 31)) & 1u) << j;
  }

  for (int a = 0; a < ja.n; ++a) {
    const b2_joinagg_t ag = ja.a[a];
    if (ag.combine == B2_JA_ROWS) {  // COUNT(*) of the join
      sh_cnt[a][tid] += __popc(matched);
      continue;
    }
    uint32_t ok = matched;
    int64_t x[R];          // probe input, then the combined value
    bool pf = false, bf = false;
    if (ag.pcol >= 0) {
      const b2_col_t& c = s.cols[ag.pcol];
      pf = c.dtype == B2_F64;
      if (a == 0 && pre_p) {
#pragma unroll
        for (int j = 0; j < R; ++j) x[j] = pp[j];
      } else {
        ld.template load<R>(ag.pcol, matched, false, x);
      }
      if (c.valid || pf) ok &= ~b2_null_bits<R>(c, ld.row0, matched, x);
    }
    if (ag.bcol >= 0) {
      const b2_col_t& c = ja.bcols[ag.bcol];
      bf = c.dtype == B2_F64;
      const bool isf = pf || bf;
      uint32_t bnull = 0;
#pragma unroll
      for (int j = 0; j < R; ++j) {
        int64_t y = 0;
        if (a == 0 && pre_b) y = pb[j];
        else if ((matched >> j) & 1) y = b2_ja_payload(c, ja.bbase[ag.bcol], d[j]);
        if (bf) { const double t = __longlong_as_double(y); bnull |= (uint32_t)(t != t) << j; }
        if (ag.combine == B2_JA_B) { x[j] = y; continue; }
        if (isf) {
          const double u = pf ? __longlong_as_double(x[j]) : (double)x[j];
          const double w = bf ? __longlong_as_double(y) : (double)y;
          double r;
          switch (ag.combine) {
            case B2_JA_MUL: r = u * w; break;
            case B2_JA_ADD: r = u + w; break;
            case B2_JA_SUB: r = u - w; break;
            default: r = w - u; break;  // B2_JA_RSUB
          }
          x[j] = __double_as_longlong(r);
        } else {
          const uint64_t u = (uint64_t)x[j], w = (uint64_t)y;
          uint64_t r;
          switch (ag.combine) {
            case B2_JA_MUL: r = u * w; break;
            case B2_JA_ADD: r = u + w; break;
            case B2_JA_SUB: r = u - w; break;
            default: r = w - u; break;
          }
          x[j] = (int64_t)r;
        }
      }
      ok &= ~bnull;
      if (c.valid) {
#pragma unroll
        for (int j = 0; j < R; ++j)
          if (((ok >> j) & 1) && !b2_bit(c.valid, (int64_t)d[j])) ok &= ~(1u << j);
      }
    }
    const bool isf = pf || bf;
    sh_cnt[a][tid] += __popc(ok);
    int64_t acc = sh_acc[a][tid];
    switch (b2_agg_kind(ag.op, isf ? B2_F64 : B2_I64)) {
      case B2_K_SUM_I: acc = b2_fold_batch<R, B2_K_SUM_I>(acc, x, ok); break;
      case B2_K_SUM_F: acc = b2_fold_batch<R, B2_K_SUM_F>(acc, x, ok); break;
      case B2_K_SUMF_I: acc = b2_fold_batch<R, B2_K_SUMF_I>(acc, x, ok); break;
      case B2_K_MIN_I: acc = b2_fold_batch<R, B2_K_MIN_I>(acc, x, ok); break;
      case B2_K_MAX_I: acc = b2_fold_batch<R, B2_K_MAX_I>(acc, x, ok); break;
      case B2_K_MIN_F: acc = b2_fold_batch<R, B2_K_MIN_F>(acc, x, ok); break;
      case B2_K_MAX_F: acc = b2_fold_batch<R, B2_K_MAX_F>(acc, x, ok); break;
      case B2_K_AND: acc = b2_fold_batch<R, B2_K_AND>(acc, x, ok); break;
      case B2_K_OR: acc = b2_fold_batch<R, B2_K_OR>(acc, x, ok); break;
      case B2_K_XOR: acc = b2_fold_batch<R, B2_K_XOR>(acc, x, ok); break;
      default: break;
    }
    sh_acc[a][tid] = acc;
  }
}

template <int MINB>   // CTAs per SM the register allocation aims for: 2 = no spills (116 regs), 3 = 80 regs + ~270 B spills
__global__ void __launch_bounds__(B2_BLOCK, MINB)
b2_join_agg_kernel(const __grid_constant__ b2_scan_t s, int key_col, const __grid_constant__ b2_jointable_t jt,
                   const __grid_constant__ b2_joinagg_arg ja, b2_partial* __restrict__ partials) {
  __shared__ int64_t sh_acc[B2_MAX_AGGS][B2_BLOCK];
  __shared__ int32_t sh_cnt[B2_MAX_AGGS][B2_BLOCK];
  const int tid = threadIdx.x;
  for (int a = 0; a < ja.n; ++a) {
    sh_acc[a][tid] = b2_identity(ja.a[a].op);
    sh_cnt[a][tid] = 0;
  }
  b2_tile_direct<B2_JA_R>(s, [&](const b2_gld& ld) { b2_join_agg_body<B2_JA_R>(s, ld, key_col, jt, ja, sh_acc, sh_cnt, tid); });
  __syncthreads();
  if (tid < ja.n) {   // fixed-order block reduce, like b2_scan_agg_kernel
    const int a = tid;
    const b2_joinagg_t ag = ja.a[a];
    const bool isf = (ag.pcol >= 0 && s.cols[ag.pcol].dtype == B2_F64) || (ag.bcol >= 0 && ja.bcols[ag.bcol].dtype == B2_F64);
    const int dt = isf ? B2_F64 : B2_I64;
    int64_t r = b2_identity(ag.op), c = 0;
    for (int t = 0; t < B2_BLOCK; ++t) {
      r = b2_combine(ag.op, dt, r, sh_acc[a][t]);
      c += sh_cnt[a][t];
    }
    partials[blockIdx.x].acc[a] = r;
    partials[blockIdx.x].cnt[a] = c;
  }
}

// ---- the common shape, specialised: ONE aggregate SUM(P o B) (o = * + -) plus the join's row count,
// nothing nullable by bitmap.  The generic kernel above spends most of its instructions per row on run-time
// dispatch over aggregates, combines and types; with the types fixed at
// compile time and the accumulators in registers the same work is a few dozen.
// PF: probe column is float64 (else int64).  BK: build payload 0 = uint32 offsets with the 0xFFFFFFFF
// "no row" sentinel (no bitmap access), 1 = uint32 + bitmap, 2 = int64 + bitmap, 3 = float64 + bitmap.
template <bool PF, int BK>
__global__ void __launch_bounds__(B2_BLOCK, 3)
b2_join_agg_fast_kernel(const __grid_constant__ b2_scan_t s, int key_col, int p_col, const __grid_constant__ b2_jointable_t jt,
                        const void* __restrict__ payload, int64_t pay_base, int combine, int sumf,
                        b2_partial* __restrict__ partials) {
  constexpr int R = B2_JA_R;
  constexpr bool ISF = PF || BK == 3;
  __shared__ int64_t sh_acc[B2_BLOCK];
  __shared__ int32_t sh_cnt[2][B2_BLOCK];
  double facc = 0.0;
  uint64_t iacc = 0;
  int cnt = 0, rows = 0;
  const uint64_t range = (uint64_t)jt.range;
  const int tile_off = (threadIdx.x >> 5) * (32 * R) + (threadIdx.x & 31);
  for (int64_t base = (int64_t)blockIdx.x * B2_JA_ROWS_PER_BLOCK; base < s.n; base += (int64_t)gridDim.x * B2_JA_ROWS_PER_BLOCK) {
    const int64_t row0 = base + tile_off;
    bool full0;
    const uint32_t inb = b2_bounds_bits<R>(row0, s.n, full0);
    int64_t key[R], pv[R];
    b2_load_batch64<R>(s.cols[key_col].data, row0, inb, full0, key);
    b2_load_batch64<R>(s.cols[p_col].data, row0, inb, full0, pv);
    bool full;
    const uint32_t bits = s.nterms ? b2_eval_terms<R>(s, row0, full) : inb;
    int64_t pay[R];
    uint32_t m = 0;
    if (BK == 0) {
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const uint64_t d = (uint64_t)key[j] - (uint64_t)jt.kmin;
        const bool ok = ((bits >> j) & 1) && d < range;
        const uint32_t raw = ok ? (uint32_t)b2_ld_keep_i32(reinterpret_cast<const int32_t*>(payload) + d) : 0xffffffffu;
        m |= (uint32_t)(raw != 0xffffffffu) << j;
        pay[j] = pay_base + (int64_t)raw;
      }
    } else {
      uint32_t word[R];
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const uint64_t d = (uint64_t)key[j] - (uint64_t)jt.kmin;
        const bool ok = ((bits >> j) & 1) && d < range;
        word[j] = ok ? (uint32_t)b2_ld_keep_i32(jt.lookup + (d >> 5)) : 0u;
        pay[j] = 0;
        if (ok) pay[j] = BK == 1 ? pay_base + (int64_t)(uint32_t)b2_ld_keep_i32(reinterpret_cast<const int32_t*>(payload) + d)
                                 : b2_ld_keep_i64(reinterpret_cast<const int64_t*>(payload) + d);
      }
#pragma unroll
      for (int j = 0; j < R; ++j) m |= ((word[j] >> (((uint64_t)key[j] - (uint64_t)jt.kmin) & 31)) & 1u) << j;
    }
    rows += __popc(m);
#pragma unroll
    for (int j = 0; j < R; ++j) {
      if (!((m >> j) & 1)) continue;
      if (ISF) {
        const double x = PF ? __longlong_as_double(pv[j]) : (double)pv[j];
        const double y = BK == 3 ? __longlong_as_double(pay[j]) : (double)pay[j];
        if ((PF && x != x) || (BK == 3 && y != y)) continue;      // NaN = NULL: the row does not contribute
        double r;
        switch (combine) {
          case B2_JA_MUL: r = x * y; break;
          case B2_JA_ADD: r = x + y; break;
          case B2_JA_SUB: r = x - y; break;
          default: r = y - x; break;
        }
        facc += r;
      } else {
        const uint64_t x = (uint64_t)pv[j], y = (uint64_t)pay[j];
        uint64_t r;
        switch (combine) {
          case B2_JA_MUL: r = x * y; break;
          case B2_JA_ADD: r = x + y; break;
          case B2_JA_SUB: r = x - y; break;
          default: r = y - x; break;
        }
        if (sumf) facc += (double)(int64_t)r;
        else iacc += r;
      }
      ++cnt;
    }
  }
  const bool fres = ISF || sumf;
  sh_acc[threadIdx.x] = fres ? __double_as_longlong(facc) : (int64_t)iacc;
  sh_cnt[0][threadIdx.x] = cnt;
  sh_cnt[1][threadIdx.x] = rows;
  __syncthreads();
  if (threadIdx.x == 0) {   // fixed order, like b2_scan_agg_kernel: bit-reproducible for a given grid
    double f = 0.0;
    uint64_t u = 0;
    int64_t c = 0, rws = 0;
    for (int t = 0; t < B2_BLOCK; ++t) {
      if (fres) f += __longlong_as_double(sh_acc[t]);
      else u += (uint64_t)sh_acc[t];
      c += sh_cnt[0][t];
      rws += sh_cnt[1][t];
    }
    partials[blockIdx.x].acc[0] = fres ? __double_as_longlong(f) : (int64_t)u;
    partials[blockIdx.x].cnt[0] = c;
    partials[blockIdx.x].acc[1] = 0;
    partials[blockIdx.x].cnt[1] = rws;
  }
}

template <bool PF, int BK>
static int b2_launch_join_agg_fast(const b2_scan_t* scan, int key_col, int p_col, const b2_jointable_t* jt,
                                   const void* payload, int64_t base, int combine, int sumf, b2_partial* partials,
                                   cudaStream_t st) {
  int64_t nblk = (scan->n + B2_JA_ROWS_PER_BLOCK - 1) / B2_JA_ROWS_PER_BLOCK;
  int grid = b2_wave_grid(b2_join_agg_fast_kernel<PF, BK>, B2_BLOCK, nblk);
  if (grid > B2_MAX_PARTIALS) grid = B2_MAX_PARTIALS;
  b2_join_agg_fast_kernel<PF, BK><<<grid, B2_BLOCK, 0, st>>>(*scan, key_col, p_col, *jt, payload, base, combine, sumf, partials);
  return grid;
}

extern "C" {

int32_t b2_join_agg(const b2_scan_t* scan, int32_t probe_key, const b2_jointable_t* jt, int32_t nbuild,
                    const b2_col_t* build_cols, const int64_t* build_base, const b2_joinagg_t* aggs, int32_t naggs,
                    int64_t* d_out_acc, int64_t* d_out_cnt, int32_t accumulate, void* ws, void* stream) {
  int32_t rc = b2_check_scan(scan);
  if (rc) return rc;
  B2_REQUIRE(jt && d_out_acc && d_out_cnt && ws, "null argument");
  B2_REQUIRE(jt->dense == 2 && jt->nkeys == 1 && jt->lookup && jt->range > 0, "b2_join_agg needs a key-ordered table");
  B2_REQUIRE(probe_key >= 0 && probe_key < scan->ncols && scan->cols[probe_key].dtype == B2_I64, "probe key must be int64");
  B2_REQUIRE(naggs >= 1 && naggs <= B2_MAX_AGGS && aggs, "bad aggregate list");
  B2_REQUIRE(nbuild >= 0 && nbuild <= B2_JA_MAX_BUILD && (nbuild == 0 || build_cols), "bad build column list");
  b2_joinagg_arg ja;
  memset(&ja, 0, sizeof(ja));
  ja.n = naggs;
  ja.nb = nbuild;
  for (int b = 0; b < nbuild; ++b) {
    B2_REQUIRE(build_cols[b].data, "null build column");
    B2_REQUIRE(build_cols[b].dtype != B2_U32 || build_base, "uint32 payloads need their base");
    ja.bcols[b] = build_cols[b];
    ja.bbase[b] = build_base ? build_base[b] : 0;
  }
  b2_final_arg fa;
  memset(&fa, 0, sizeof(fa));
  fa.n = naggs;
  for (int a = 0; a < naggs; ++a) {
    const b2_joinagg_t& ag = aggs[a];
    B2_REQUIRE(ag.combine >= B2_JA_P && ag.combine <= B2_JA_ROWS, "bad combine");
    B2_REQUIRE(ag.op >= B2_AGG_SUM && ag.op <= B2_AGG_XOR, "bad agg op");
    const bool needp = ag.combine != B2_JA_B && ag.combine != B2_JA_ROWS;
    const bool needb = ag.combine != B2_JA_P && ag.combine != B2_JA_ROWS;
    B2_REQUIRE(!needp || (ag.pcol >= 0 && ag.pcol < scan->ncols), "probe column out of range");
    B2_REQUIRE(!needb || (ag.bcol >= 0 && ag.bcol < nbuild), "build column out of range");
    B2_REQUIRE(!needp || scan->cols[ag.pcol].dtype != B2_U8, "aggregate inputs must be 8-byte columns");
    B2_REQUIRE(!needb || build_cols[ag.bcol].dtype != B2_U8, "aggregate inputs must be 8-byte columns");
    ja.a[a] = ag;
    if (!needp) ja.a[a].pcol = -1;
    if (!needb) ja.a[a].bcol = -1;
    const bool isf = (needp && scan->cols[ag.pcol].dtype == B2_F64) || (needb && build_cols[ag.bcol].dtype == B2_F64);
    B2_REQUIRE(ag.combine == B2_JA_ROWS || ag.op < B2_AGG_AND || !isf, "bitwise aggregates take int64 inputs");
    fa.op[a] = ag.combine == B2_JA_ROWS ? B2_AGG_COUNT : ag.op;
    fa.dtype[a] = isf ? B2_F64 : B2_I64;
    if (ag.combine == B2_JA_ROWS) ja.a[a].op = B2_AGG_COUNT;
  }
  cudaStream_t st = (cudaStream_t)stream;
  b2_partial* partials = reinterpret_cast<b2_partial*>(ws);
  {
    // the specialised kernel when the call is  SUM(P o B) [+ COUNT(*)]  over bitmap-free 8-byte columns
    const b2_joinagg_t& a0 = ja.a[0];
    const char* off = getenv("B200SQL_JA_GENERIC");
    bool fast = !(off && off[0] == '1') && naggs == 2 && ja.a[1].combine == B2_JA_ROWS &&
                (a0.combine == B2_JA_MUL || a0.combine == B2_JA_ADD || a0.combine == B2_JA_SUB || a0.combine == B2_JA_RSUB) &&
                (a0.op == B2_AGG_SUM || a0.op == B2_AGG_SUMF) && !scan->cols[probe_key].valid;
    if (fast) {
      const b2_col_t& pc = scan->cols[a0.pcol];
      const b2_col_t& bc = ja.bcols[a0.bcol];
      fast = !pc.valid && !bc.valid && pc.dtype != B2_U8;
      if (fast) {
        const bool pf = pc.dtype == B2_F64;
        int bk;
        if (bc.dtype == B2_U32) bk = (bc.flags & B2_COL_SENTINEL) ? 0 : 1;
        else bk = bc.dtype == B2_F64 ? 3 : 2;
        const int sumf = a0.op == B2_AGG_SUMF;
        int grid = 0;
#define B2_JAF(PF, BK) grid = b2_launch_join_agg_fast<PF, BK>(scan, probe_key, a0.pcol, jt, bc.data, ja.bbase[a0.bcol], a0.combine, sumf, partials, st)
        if (pf) { if (bk == 0) B2_JAF(true, 0); else if (bk == 1) B2_JAF(true, 1); else if (bk == 2) B2_JAF(true, 2); else B2_JAF(true, 3); }
        else { if (bk == 0) B2_JAF(false, 0); else if (bk == 1) B2_JAF(false, 1); else if (bk == 2) B2_JAF(false, 2); else B2_JAF(false, 3); }
#undef B2_JAF
        B2_CHECK_LAUNCH("b2_join_agg_fast_kernel");
        b2_scan_agg_final_kernel<<<naggs, B2_BLOCK, 0, st>>>(fa, partials, grid, d_out_acc, d_out_cnt, accumulate);
        B2_CHECK_LAUNCH("b2_scan_agg_final_kernel");
        return B2_OK;
      }
    }
  }
  int64_t nblk = (scan->n + B2_JA_ROWS_PER_BLOCK - 1) / B2_JA_ROWS_PER_BLOCK;
  int minb = 3;
  if (const char* e = getenv("B200SQL_JA_MINB")) minb = atoi(e) == 2 ? 2 : 3;
  int grid;
  if (minb == 2) {
    grid = b2_wave_grid(b2_join_agg_kernel<2>, B2_BLOCK, nblk);
    if (grid > B2_MAX_PARTIALS) grid = B2_MAX_PARTIALS;
    b2_join_agg_kernel<2><<<grid, B2_BLOCK, 0, st>>>(*scan, probe_key, *jt, ja, partials);
  } else {
    grid = b2_wave_grid(b2_join_agg_kernel<3>, B2_BLOCK, nblk);
    if (grid > B2_MAX_PARTIALS) grid = B2_MAX_PARTIALS;
    b2_join_agg_kernel<3><<<grid, B2_BLOCK, 0, st>>>(*scan, probe_key, *jt, ja, partials);
  }
  B2_CHECK_LAUNCH("b2_join_agg_kernel");
  b2_scan_agg_final_kernel<<<naggs, B2_BLOCK, 0, st>>>(fa, partials, grid, d_out_acc, d_out_cnt, accumulate);
  B2_CHECK_LAUNCH("b2_scan_agg_final_kernel");
  return B2_OK;
}

}  // extern "C"
