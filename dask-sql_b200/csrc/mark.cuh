// mark.cuh — the mark of an IN / EXISTS subquery: one three-valued BOOLEAN per probe row, from the
// candidates the existing join tables list (b2_join_build / _build_dense / b2_join_key_layout) and up to
// B2_MARK_MAX_TERMS pair terms  probe_col <cmp> build  on each (probe row, candidate) pair.
#pragma once
#include "common.cuh"
#include "join.cuh"

struct b2_markterms_arg {
  b2_mark_term_t t[B2_MARK_MAX_TERMS];
  int32_t n;
};

// 1 TRUE, 0 FALSE, -1 NULL: SQL's AND of the pair terms on (probe row, build row).  A NULL on either side
// makes a term NULL, and a NULL B2_MARK_WHERE term FALSE.
__device__ __forceinline__ int b2_mark_pair(const b2_scan_t& s, const b2_markterms_arg& mt, int64_t prow,
                                            int32_t brow) {
  int v = 1;
  for (int t = 0; t < mt.n; ++t) {
    const b2_mark_term_t& tm = mt.t[t];
    const b2_col_t& pc = s.cols[tm.probe_col];
    const int64_t a = b2_load_raw(pc, prow);
    const int64_t b = __ldg(reinterpret_cast<const long long*>(tm.build.data) + brow);
    const bool where = tm.cmp & B2_MARK_WHERE;
    // a float NULL is a NaN without a bitmap: the IN's own x = y treats it as NULL, as the IN's key does
    // (b2_is_null); WHERE terms compare NaN as IEEE, as scan terms do
    const bool null = where ? (pc.valid && !b2_bit(pc.valid, prow)) || (tm.build.valid && !b2_bit(tm.build.valid, brow))
                            : b2_is_null(pc, prow, a) || b2_is_null(tm.build, brow, b);
    if (null) {
      if (where) return 0;
      v = -1;
      continue;
    }
    const int cmp = tm.cmp & ~B2_MARK_WHERE;
    bool ok;
    if (pc.dtype == B2_F64) {
      const double x = __longlong_as_double(a), y = __longlong_as_double(b);
      switch (cmp) {
        case B2_EQ: ok = x == y; break;
        case B2_NE: ok = x != y; break;
        case B2_LT: ok = x < y; break;
        case B2_LE: ok = x <= y; break;
        case B2_GT: ok = x > y; break;
        default: ok = x >= y;
      }
    } else {
      switch (cmp) {
        case B2_EQ: ok = a == b; break;
        case B2_NE: ok = a != b; break;
        case B2_LT: ok = a < b; break;
        case B2_LE: ok = a <= b; break;
        case B2_GT: ok = a > b; break;
        default: ok = a >= b;
      }
    }
    if (!ok) return 0;
  }
  return v;
}

// One thread per probe row, rows row0 + 32*j of a lane as in the join probes, so that the 32 rows of one
// j are one validity word, built by one ballot.  The walk stops at the first TRUE candidate.
__global__ void __launch_bounds__(B2_BLOCK)
b2_join_mark_kernel(const __grid_constant__ b2_scan_t s, const __grid_constant__ b2_probekeys_arg pk,
                    const __grid_constant__ b2_jointable_t jt, const __grid_constant__ b2_markterms_arg mt,
                    int32_t flags, int64_t ntiles, uint8_t* __restrict__ out, uint32_t* __restrict__ out_valid) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * B2_TILE + (int64_t)warp * (32 * B2_JOIN_R) + lane;
    const uint32_t bits = b2_eval_terms<B2_JOIN_R>(s, row0);
#pragma unroll 1
    for (int j = 0; j < B2_JOIN_R; ++j) {
      const int64_t row = row0 + (int64_t)j * 32;
      int m = 0;                                    // a row that fails the scan's terms is FALSE
      if ((bits >> j) & 1) {
        int64_t key[B2_MAX_KEYS];
        if (!b2_probe_key(s, pk, jt.nkeys, row, key)) {
          // NULL IN (non-empty set) is NULL; a NULL correlation key has no candidates
          m = ((flags & B2_MARK_NULL_AWARE) && (flags & B2_MARK_BUILD_NONEMPTY)) ? -1 : 0;
        } else if (jt.dense) {
          const uint64_t d = (uint64_t)key[0] - (uint64_t)jt.kmin;
          if (d < (uint64_t)jt.range) {
            if (jt.dense == 2) {
              m = (__ldg(jt.lookup + (d >> 5)) >> (d & 31)) & 1;
            } else {
              const int32_t r = __ldg(jt.lookup + d);
              if (r >= 0) m = b2_mark_pair(s, mt, row, r);
            }
          }
        } else {
          const uint64_t h = b2_hash_keys(key, jt.nkeys) & (uint64_t)(jt.cap - 1);
          for (int32_t r = __ldg(jt.head + h); r >= 0 && m != 1; r = __ldg(jt.next + r)) {
            bool same = true;
            for (int k = 0; same && k < jt.nkeys; ++k)
              same = b2_key_image(jt.keys[k], __ldg(reinterpret_cast<const long long*>(jt.keys[k].data) + r)) == key[k];
            if (!same) continue;
            const int v = b2_mark_pair(s, mt, row, r);
            if (v != 0) m = v;                      // TRUE ends the walk; NULL holds unless a TRUE follows
          }
        }
        // x NOT found among a set that holds a NULL: x IN (...) is NULL
        if (m == 0 && (flags & B2_MARK_NULL_AWARE) && (flags & B2_MARK_BUILD_HAS_NULL)) m = -1;
      }
      const bool live = row < s.n;
      const uint32_t word = __ballot_sync(FULL_MASK, live && m >= 0);
      if (live) out[row] = m == 1;
      if (lane == 0 && row < s.n) out_valid[row >> 5] = word;
    }
  }
}

extern "C" {

int32_t b2_join_mark(const b2_scan_t* scan, const int32_t* probe_keys, const b2_jointable_t* jt,
                     const b2_mark_term_t* terms, int32_t nterms, int32_t flags, uint8_t* out, uint32_t* out_valid,
                     void* stream) {
  b2_probekeys_arg pk;
  int32_t rc = b2_check_join(scan, probe_keys, jt, B2_JOIN_SEMI, &pk);
  if (rc) return rc;
  B2_REQUIRE(nterms >= 0 && nterms <= B2_MARK_MAX_TERMS, "bad number of pair terms");
  B2_REQUIRE(nterms == 0 || terms, "null argument");
  B2_REQUIRE((flags & ~(B2_MARK_NULL_AWARE | B2_MARK_BUILD_NONEMPTY | B2_MARK_BUILD_HAS_NULL)) == 0, "bad flags");
  B2_REQUIRE(!(flags & B2_MARK_NULL_AWARE) || jt->nkeys == 1, "a NULL-aware mark has one key");
  // pair terms need every candidate: a key-ordered table lists a key once and keeps no build row
  B2_REQUIRE(nterms == 0 || jt->dense != 2, "pair terms need a chained or direct-address table");
  B2_REQUIRE(scan->n == 0 || (out && out_valid), "null argument");
  b2_markterms_arg mt;
  memset(&mt, 0, sizeof(mt));
  mt.n = nterms;
  for (int t = 0; t < nterms; ++t) {
    const b2_mark_term_t& tm = terms[t];
    B2_REQUIRE(tm.probe_col >= 0 && tm.probe_col < scan->ncols, "pair term column out of range");
    const int32_t cmp = tm.cmp & ~B2_MARK_WHERE;
    B2_REQUIRE(cmp >= B2_EQ && cmp <= B2_GE, "bad pair term comparison");
    B2_REQUIRE(tm.build.dtype == B2_I64 || tm.build.dtype == B2_F64, "pair terms compare int64 or float64");
    B2_REQUIRE(scan->cols[tm.probe_col].dtype == tm.build.dtype, "pair term sides differ in type");
    mt.t[t] = tm;
  }
  const int64_t ntiles = b2_num_tiles(scan->n);
  if (ntiles == 0) return B2_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = b2_wave_grid(b2_join_mark_kernel, B2_BLOCK, ntiles);
  b2_join_mark_kernel<<<grid, B2_BLOCK, 0, st>>>(*scan, pk, *jt, mt, flags, ntiles, out, out_valid);
  B2_CHECK_LAUNCH("b2_join_mark_kernel");
  return B2_OK;
}

}  // extern "C"
