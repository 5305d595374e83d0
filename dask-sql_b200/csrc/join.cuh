// join.cuh — hash join: chained build (duplicates allowed), direct-address build (unique dense
// keys), two-pass probe that emits matches in probe-row order and, in the same pass, gathers the
// requested probe / build columns straight into the output (no index round trip).
#pragma once
#include "common.cuh"

#define B2_JOIN_R 16
static_assert(B2_BLOCK * B2_JOIN_R == B2_TILE, "tile geometry");

struct b2_keycols_arg {
  b2_col_t c[B2_MAX_KEYS];
  int32_t n;
};
struct b2_probekeys_arg {
  int32_t cols[B2_MAX_KEYS];
};
struct b2_joingather_arg {
  int32_t nprobe, nbuild;
  int32_t probe_cols[B2_MAX_GATHER];
  void* probe_out[B2_MAX_GATHER];
  uint32_t* probe_valid[B2_MAX_GATHER];
  b2_col_t build_cols[B2_MAX_GATHER];
  void* build_out[B2_MAX_GATHER];
  uint32_t* build_valid[B2_MAX_GATHER];
  int64_t build_base[B2_MAX_GATHER];  // B2_U32 storage: value = base + (uint32)stored
};

// normalised key image: -0.0 -> +0.0 so float keys compare like pandas; ints unchanged
__device__ __forceinline__ int64_t b2_key_image(const b2_col_t& c, int64_t raw) {
  if (c.dtype == B2_F64 && raw == (int64_t)0x8000000000000000LL) return 0;
  return raw;
}
__device__ __forceinline__ uint64_t b2_hash_keys(const int64_t* key, int nkeys) {
  uint64_t hv = 0x9e3779b97f4a7c15ULL;
  for (int k = 0; k < nkeys; ++k) hv = b2_mix64(hv ^ (uint64_t)key[k]);
  return hv;
}

__global__ void __launch_bounds__(B2_BLOCK)
b2_join_build_kernel(const __grid_constant__ b2_keycols_arg keys, int64_t n, int32_t* __restrict__ head,
                     int32_t* __restrict__ next, int64_t cap) {
  for (int64_t i = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; i < n; i += (int64_t)gridDim.x * B2_BLOCK) {
    int64_t key[B2_MAX_KEYS];
    bool isnull = false;
#pragma unroll
    for (int k = 0; k < B2_MAX_KEYS; ++k) {
      key[k] = 0;
      if (k < keys.n) {
        const int64_t raw = b2_load_raw(keys.c[k], i);
        isnull |= b2_is_null(keys.c[k], i, raw);
        key[k] = b2_key_image(keys.c[k], raw);
      }
    }
    if (isnull) { next[i] = -1; continue; }  // NULL keys never join (join.py:202-213)
    const uint64_t h = b2_hash_keys(key, keys.n) & (uint64_t)(cap - 1);
    next[i] = atomicExch(head + h, (int32_t)i);
  }
}

__global__ void __launch_bounds__(B2_BLOCK)
b2_join_build_dense_kernel(const __grid_constant__ b2_col_t key, int64_t n, int64_t kmin, int64_t range,
                           int32_t* __restrict__ lookup, int32_t* __restrict__ flags) {
  for (int64_t i = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; i < n; i += (int64_t)gridDim.x * B2_BLOCK) {
    const int64_t raw = b2_load_raw(key, i);
    if (b2_is_null(key, i, raw)) continue;
    const uint64_t d = (uint64_t)raw - (uint64_t)kmin;
    if (d >= (uint64_t)range) continue;
    if (atomicExch(lookup + d, (int32_t)i) != -1) flags[0] = 1;
  }
}

// Key-ordered layout of one build column of a unique dense-key table: out[key - kmin] = col[row]
// (optionally narrowed to uint32 offsets from `base`), so that a probe reaches the payload with ONE
// random access at the key offset instead of lookup[key] -> row -> col[row]; `present` marks the
// offsets that hold a build row (it replaces the int32 lookup: range/8 bytes instead of range*4).
__global__ void __launch_bounds__(B2_BLOCK)
b2_join_key_layout_kernel(const __grid_constant__ b2_col_t key, int64_t n, int64_t kmin, int64_t range,
                          const __grid_constant__ b2_col_t col, int has_col, int out_dtype, int64_t base,
                          void* __restrict__ out_data, uint32_t* __restrict__ out_valid,
                          uint32_t* __restrict__ present) {
  for (int64_t i = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; i < n; i += (int64_t)gridDim.x * B2_BLOCK) {
    const int64_t kraw = b2_load_raw(key, i);
    if (b2_is_null(key, i, kraw)) continue;
    const uint64_t d = (uint64_t)kraw - (uint64_t)kmin;
    if (d >= (uint64_t)range) continue;
    if (present) atomicOr(present + (d >> 5), 1u << (d & 31));
    if (!has_col) continue;
    if (col.dtype == B2_U8) {
      reinterpret_cast<uint8_t*>(out_data)[d] = reinterpret_cast<const uint8_t*>(col.data)[i];
    } else {
      const int64_t v = b2_load_raw(col, i);
      if (out_dtype == B2_U32) reinterpret_cast<uint32_t*>(out_data)[d] = (uint32_t)((uint64_t)v - (uint64_t)base);
      else reinterpret_cast<int64_t*>(out_data)[d] = v;
    }
    if (out_valid && (!col.valid || b2_bit(col.valid, i))) atomicOr(out_valid + (d >> 5), 1u << (d & 31));
  }
}

// Walk the chain of one probe row.  F(build_row) is called for every match.
template <class F>
__device__ __forceinline__ int b2_for_matches(const b2_jointable_t& jt, const int64_t* pkey, F f) {
  int cnt = 0;
  const uint64_t h = b2_hash_keys(pkey, jt.nkeys) & (uint64_t)(jt.cap - 1);
  for (int32_t r = __ldg(jt.head + h); r >= 0; r = __ldg(jt.next + r)) {
    bool same = true;
    for (int k = 0; same && k < jt.nkeys; ++k) {
      const int64_t braw = __ldg(reinterpret_cast<const long long*>(jt.keys[k].data) + r);
      same = b2_key_image(jt.keys[k], braw) == pkey[k];
    }
    if (same) { f(r); ++cnt; }
  }
  return cnt;
}

// load + normalise the probe keys of one row; returns false if any key is NULL
__device__ __forceinline__ bool b2_probe_key(const b2_scan_t& s, const b2_probekeys_arg& pk, int nkeys,
                                             int64_t row, int64_t* key) {
  bool ok = true;
#pragma unroll
  for (int k = 0; k < B2_MAX_KEYS; ++k) {
    key[k] = 0;
    if (k < nkeys) {
      const b2_col_t& c = s.cols[pk.cols[k]];
      const int64_t raw = b2_load_raw(c, row);
      ok &= !b2_is_null(c, row, raw);
      key[k] = b2_key_image(c, raw);
    }
  }
  return ok;
}

__device__ __forceinline__ int b2_emit_count(int mode, int matches) {
  switch (mode) {
    case B2_JOIN_INNER: return matches;
    case B2_JOIN_LEFT: return matches ? matches : 1;
    case B2_JOIN_SEMI: return matches ? 1 : 0;
    default: return matches ? 0 : 1;  // ANTI
  }
}

// ---- direct-address table: at most one match per probe row, everything is batched --------------
// returns the bits of rows that emit; brow[j] = matching build row or -1
template <int R>
__device__ __forceinline__ uint32_t b2_dense_probe(const b2_scan_t& s, int key_col, const b2_jointable_t& jt,
                                                   int mode, int64_t row0, int32_t (&brow)[R]) {
  bool full;
  const uint32_t bits = b2_eval_terms<R>(s, row0, full);
  const b2_col_t& kc = s.cols[key_col];
  int64_t key[R];
  b2_load_batch<R>(kc, row0, bits, full, key);
  uint32_t live = bits;
  if (kc.valid) live &= b2_valid_bits<R>(kc.valid, row0, bits);
  uint32_t matched = 0;
  const uint64_t range = (uint64_t)jt.range;
  if (jt.dense == 2) {
    // key-ordered layout: `lookup` is the presence bitmap and the build row IS the key offset
    uint32_t word[R];
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const uint64_t d = (uint64_t)key[j] - (uint64_t)jt.kmin;
      word[j] = (((live >> j) & 1) && d < range) ? (uint32_t)b2_ld_keep_i32(jt.lookup + (d >> 5)) : 0u;
    }
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const uint64_t d = (uint64_t)key[j] - (uint64_t)jt.kmin;
      brow[j] = ((word[j] >> (d & 31)) & 1) ? (int32_t)d : -1;
    }
  } else {
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const uint64_t d = (uint64_t)key[j] - (uint64_t)jt.kmin;
      brow[j] = (((live >> j) & 1) && d < range) ? b2_ld_keep_i32(jt.lookup + d) : -1;
    }
  }
#pragma unroll
  for (int j = 0; j < R; ++j) matched |= (uint32_t)(brow[j] >= 0) << j;
  switch (mode) {
    case B2_JOIN_INNER:
    case B2_JOIN_SEMI: return matched;
    case B2_JOIN_LEFT: return bits;
    default: return bits & ~matched;  // ANTI
  }
}

template <bool DENSE>
__global__ void __launch_bounds__(B2_BLOCK)
b2_join_count_kernel(const __grid_constant__ b2_scan_t s, const __grid_constant__ b2_probekeys_arg pk,
                     const __grid_constant__ b2_jointable_t jt, int mode, int64_t ntiles,
                     int64_t* __restrict__ tile_cnt) {
  __shared__ int64_t sh[B2_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * B2_TILE + (int64_t)warp * (32 * B2_JOIN_R) + lane;
    int64_t c = 0;
    if (DENSE) {
      int32_t brow[B2_JOIN_R];
      c = __popc(b2_dense_probe<B2_JOIN_R>(s, pk.cols[0], jt, mode, row0, brow));
    } else {
      const uint32_t bits = b2_eval_terms<B2_JOIN_R>(s, row0);
#pragma unroll 1
      for (int j = 0; j < B2_JOIN_R; ++j) {
        if (!((bits >> j) & 1)) continue;
        int64_t key[B2_MAX_KEYS];
        int m = 0;
        if (b2_probe_key(s, pk, jt.nkeys, row0 + (int64_t)j * 32, key))
          m = b2_for_matches(jt, key, [](int32_t) {});
        c += b2_emit_count(mode, m);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(FULL_MASK, c, o);
    if (lane == 0) sh[warp] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
      int64_t t = 0;
      for (int w = 0; w < B2_WARPS; ++w) t += sh[w];
      tile_cnt[tile] = t;
    }
    __syncthreads();
  }
}

// one output row: indices and gathered columns
__device__ __forceinline__ void b2_join_emit(const b2_scan_t& s, const b2_joingather_arg& g, int64_t pos,
                                             int64_t prow, int32_t brow, int32_t* __restrict__ out_probe,
                                             int32_t* __restrict__ out_build) {
  if (out_probe) out_probe[pos] = (int32_t)prow;
  if (out_build) out_build[pos] = brow;
  for (int k = 0; k < g.nprobe; ++k) {
    const b2_col_t& c = s.cols[g.probe_cols[k]];
    if (c.dtype == B2_U8) reinterpret_cast<uint8_t*>(g.probe_out[k])[pos] = reinterpret_cast<const uint8_t*>(c.data)[prow];
    else reinterpret_cast<int64_t*>(g.probe_out[k])[pos] = b2_ld_stream(reinterpret_cast<const int64_t*>(c.data) + prow);
    if (g.probe_valid[k] && (!c.valid || b2_bit(c.valid, prow)))
      atomicOr(g.probe_valid[k] + (pos >> 5), 1u << (pos & 31));
  }
  for (int k = 0; k < g.nbuild; ++k) {
    const b2_col_t& c = g.build_cols[k];
    const bool has = brow >= 0;
    if (c.dtype == B2_U8) {
      reinterpret_cast<uint8_t*>(g.build_out[k])[pos] = has ? reinterpret_cast<const uint8_t*>(c.data)[brow] : 0;
    } else {
      int64_t v = has ? __ldg(reinterpret_cast<const long long*>(c.data) + brow) : 0;
      if (!has && c.dtype == B2_F64) v = 0x7ff8000000000000LL;  // NaN fill, like pandas take(-1)
      reinterpret_cast<int64_t*>(g.build_out[k])[pos] = v;
    }
    if (g.build_valid[k] && has && (!c.valid || b2_bit(c.valid, brow)))
      atomicOr(g.build_valid[k] + (pos >> 5), 1u << (pos & 31));
  }
}

template <bool DENSE>
__global__ void __launch_bounds__(B2_BLOCK, 3)
b2_join_write_kernel(const __grid_constant__ b2_scan_t s, const __grid_constant__ b2_probekeys_arg pk,
                     const __grid_constant__ b2_jointable_t jt, int mode, int64_t ntiles,
                     const int64_t* __restrict__ tile_off, int32_t* __restrict__ out_probe,
                     int32_t* __restrict__ out_build, uint8_t* __restrict__ build_matched,
                     const __grid_constant__ b2_joingather_arg g) {
  __shared__ int64_t sh[B2_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lt_mask = (1u << lane) - 1;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * B2_TILE + (int64_t)warp * (32 * B2_JOIN_R) + lane;
    if (DENSE) {
      // ---- at most one output per probe row: ballot ranks, batched gathers
      int32_t brow[B2_JOIN_R];
      const uint32_t emit = b2_dense_probe<B2_JOIN_R>(s, pk.cols[0], jt, mode, row0, brow);
      uint32_t ballots[B2_JOIN_R];
      int wtotal = 0;
#pragma unroll
      for (int j = 0; j < B2_JOIN_R; ++j) {
        ballots[j] = __ballot_sync(FULL_MASK, (emit >> j) & 1);
        wtotal += __popc(ballots[j]);
      }
      if (lane == 0) sh[warp] = wtotal;
      __syncthreads();
      int64_t off = tile_off[tile];
      for (int w = 0; w < warp; ++w) off += sh[w];
      __syncthreads();
      // output position = off + rel[j]; rel is 32-bit (a tile emits <= 4096 rows) to save registers
      int32_t rel[B2_JOIN_R];
      {
        int run = 0;
#pragma unroll
        for (int j = 0; j < B2_JOIN_R; ++j) {
          rel[j] = ((emit >> j) & 1) ? run + __popc(ballots[j] & lt_mask) : -1;
          run += __popc(ballots[j]);
        }
      }
      const bool semi = mode == B2_JOIN_SEMI || mode == B2_JOIN_ANTI;
#pragma unroll
      for (int j = 0; j < B2_JOIN_R; ++j) {
        if (rel[j] < 0) continue;
        if (out_probe) out_probe[off + rel[j]] = (int32_t)(row0 + (int64_t)j * 32);
        if (out_build) out_build[off + rel[j]] = semi ? -1 : brow[j];
        if (build_matched && brow[j] >= 0) build_matched[brow[j]] = 1;
      }
      for (int k = 0; k < g.nprobe; ++k) {
        const b2_col_t& c = s.cols[g.probe_cols[k]];
        const uint32_t v = (g.probe_valid[k] && c.valid) ? b2_valid_bits<B2_JOIN_R>(c.valid, row0, emit) : emit;
#pragma unroll
        for (int h = 0; h < B2_JOIN_R; h += 8) {   // two half-batches: 8 gathers in flight, 16 registers
          int64_t raw[8];
          if (c.dtype == B2_U8) {
            const uint8_t* p = reinterpret_cast<const uint8_t*>(c.data) + row0;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) raw[jj] = rel[h + jj] >= 0 ? (int64_t)p[(h + jj) * 32] : 0;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
              if (rel[h + jj] >= 0) reinterpret_cast<uint8_t*>(g.probe_out[k])[off + rel[h + jj]] = (uint8_t)raw[jj];
          } else {
            const int64_t* p = reinterpret_cast<const int64_t*>(c.data) + row0;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) raw[jj] = rel[h + jj] >= 0 ? b2_ld_stream(p + (h + jj) * 32) : 0;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
              if (rel[h + jj] >= 0) reinterpret_cast<int64_t*>(g.probe_out[k])[off + rel[h + jj]] = raw[jj];
          }
        }
        if (g.probe_valid[k]) {
#pragma unroll
          for (int j = 0; j < B2_JOIN_R; ++j)
            if (rel[j] >= 0 && ((v >> j) & 1))
              atomicOr(g.probe_valid[k] + ((off + rel[j]) >> 5), 1u << ((off + rel[j]) & 31));
        }
      }
      for (int k = 0; k < g.nbuild; ++k) {
        const b2_col_t& c = g.build_cols[k];
#pragma unroll
        for (int h = 0; h < B2_JOIN_R; h += 8) {
          int64_t raw[8];
          if (c.dtype == B2_U8) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
              raw[jj] = (rel[h + jj] >= 0 && brow[h + jj] >= 0) ? reinterpret_cast<const uint8_t*>(c.data)[brow[h + jj]] : 0;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
              if (rel[h + jj] >= 0) reinterpret_cast<uint8_t*>(g.build_out[k])[off + rel[h + jj]] = (uint8_t)raw[jj];
          } else if (c.dtype == B2_U32) {   // narrowed key-ordered payload
            const int64_t base = g.build_base[k];
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
              raw[jj] = (rel[h + jj] >= 0 && brow[h + jj] >= 0)
                            ? base + (int64_t)(uint32_t)b2_ld_keep_i32(reinterpret_cast<const int32_t*>(c.data) + brow[h + jj]) : 0;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
              if (rel[h + jj] >= 0) reinterpret_cast<int64_t*>(g.build_out[k])[off + rel[h + jj]] = raw[jj];
          } else {
            const int64_t fill = c.dtype == B2_F64 ? 0x7ff8000000000000LL : 0;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
              raw[jj] = (rel[h + jj] >= 0 && brow[h + jj] >= 0)
                            ? b2_ld_keep_i64(reinterpret_cast<const int64_t*>(c.data) + brow[h + jj]) : fill;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
              if (rel[h + jj] >= 0) reinterpret_cast<int64_t*>(g.build_out[k])[off + rel[h + jj]] = raw[jj];
          }
        }
        if (g.build_valid[k]) {
#pragma unroll
          for (int j = 0; j < B2_JOIN_R; ++j)
            if (rel[j] >= 0 && brow[j] >= 0 && (!c.valid || b2_bit(c.valid, brow[j])))
              atomicOr(g.build_valid[k] + ((off + rel[j]) >> 5), 1u << ((off + rel[j]) & 31));
        }
      }
    } else {
      // ---- chained table: any number of matches per probe row
      const uint32_t bits = b2_eval_terms<B2_JOIN_R>(s, row0);
      int cnt[B2_JOIN_R];
      int32_t first[B2_JOIN_R];
      int64_t wtotal = 0;
#pragma unroll 1
      for (int j = 0; j < B2_JOIN_R; ++j) {
        int c = 0;
        int32_t f0 = -1;
        if ((bits >> j) & 1) {
          int64_t key[B2_MAX_KEYS];
          int m = 0;
          if (b2_probe_key(s, pk, jt.nkeys, row0 + (int64_t)j * 32, key))
            m = b2_for_matches(jt, key, [&](int32_t r) { if (f0 < 0) f0 = r; });
          c = b2_emit_count(mode, m) | (m > 1 ? 0x40000000 : 0);  // flag: chain must be re-walked
        }
#pragma unroll
        for (int jj = 0; jj < B2_JOIN_R; ++jj)
          if (jj == j) { cnt[jj] = c; first[jj] = f0; }
        wtotal += c & 0x3fffffff;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) wtotal += __shfl_xor_sync(FULL_MASK, wtotal, o);
      if (lane == 0) sh[warp] = wtotal;
      __syncthreads();
      int64_t off = tile_off[tile];
      for (int w = 0; w < warp; ++w) off += sh[w];
      __syncthreads();
#pragma unroll
      for (int j = 0; j < B2_JOIN_R; ++j) {
        const int c = cnt[j] & 0x3fffffff;
        int incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int t = __shfl_up_sync(FULL_MASK, incl, o);
          if (lane >= o) incl += t;
        }
        const int total = __shfl_sync(FULL_MASK, incl, 31);
        int64_t pos = off + incl - c;
        off += total;
        if (c == 0) continue;
        const int64_t prow = row0 + (int64_t)j * 32;
        if (mode == B2_JOIN_SEMI || mode == B2_JOIN_ANTI) {
          b2_join_emit(s, g, pos, prow, -1, out_probe, out_build);
          if (build_matched && first[j] >= 0) build_matched[first[j]] = 1;
        } else if (!(cnt[j] & 0x40000000)) {
          b2_join_emit(s, g, pos, prow, first[j], out_probe, out_build);  // first = -1 for an unmatched LEFT row
          if (build_matched && first[j] >= 0) build_matched[first[j]] = 1;
        } else {
          int64_t key[B2_MAX_KEYS];
          b2_probe_key(s, pk, jt.nkeys, prow, key);
          b2_for_matches(jt, key, [&](int32_t r) {
            b2_join_emit(s, g, pos, prow, r, out_probe, out_build);
            if (build_matched) build_matched[r] = 1;
            ++pos;
          });
        }
      }
    }
  }
}

// ---- single-pass probe of a direct-address table ------------------------------------------------
// Every probe row emits at most one output row, so one kernel can do the whole join: each warp owns
// 256 consecutive probe rows of a 2048-row tile, ranks its emitting rows by ballot and reserves its
// output range with one atomicAdd on *total.  Rows of one warp batch stay contiguous and in probe
// order; the batches land in the order the warps reserve.  The loads are front-loaded so that a
// batch costs two dependent memory round trips instead of one per gathered column:
//   trip 1: probe key, predicate columns and the first other 8-byte probe column (streaming)
//   trip 2: presence word and -- on a key-ordered table (dense == 2) -- the first build column's
//           payload at the key offset, fetched speculatively together with the presence word
// Remaining columns (rare: more than two per side) are gathered after the offsets are known.
#define B2_JOP_R 8
#define B2_JOP_TILE (B2_BLOCK * B2_JOP_R)

__global__ void __launch_bounds__(B2_BLOCK, 2)
b2_join_onepass_kernel(const __grid_constant__ b2_scan_t s, int key_col, const __grid_constant__ b2_jointable_t jt,
                       int mode, int64_t ntiles, unsigned long long* __restrict__ total,
                       const __grid_constant__ b2_joingather_arg g) {
  constexpr int R = B2_JOP_R;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lt_mask = (1u << lane) - 1;
  const b2_col_t& kc = s.cols[key_col];
  int preA = -1;   // probe gather column held in registers from trip 1
  for (int k = 0; k < g.nprobe; ++k) {
    if (g.probe_cols[k] != key_col && s.cols[g.probe_cols[k]].dtype != B2_U8) { preA = k; break; }
  }
  const bool spec = jt.dense == 2 && g.nbuild > 0 && g.build_cols[0].dtype != B2_U8;
  const bool spec32 = spec && g.build_cols[0].dtype == B2_U32;
  const uint64_t range = (uint64_t)jt.range;

  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * B2_JOP_TILE + (int64_t)warp * (32 * R) + lane;
    bool full;
    const uint32_t bits = b2_eval_terms<R>(s, row0, full);
    int64_t key[R], pre[R];
    b2_load_batch<R>(kc, row0, bits, full, key);
    if (preA >= 0) b2_load_batch64<R>(s.cols[g.probe_cols[preA]].data, row0, bits, full, pre);
    uint32_t live = bits;
    if (kc.valid) live &= b2_valid_bits<R>(kc.valid, row0, bits);

    int32_t brow[R];
    int64_t pay[R];
    if (jt.dense == 2) {
      uint32_t word[R];
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const uint64_t d = (uint64_t)key[j] - (uint64_t)jt.kmin;
        const bool ok = ((live >> j) & 1) && d < range;
        word[j] = ok ? (uint32_t)b2_ld_keep_i32(jt.lookup + (d >> 5)) : 0u;
        pay[j] = 0;
        if (spec && ok) {
          pay[j] = spec32 ? (int64_t)(uint32_t)b2_ld_keep_i32(reinterpret_cast<const int32_t*>(g.build_cols[0].data) + d)
                          : b2_ld_keep_i64(reinterpret_cast<const int64_t*>(g.build_cols[0].data) + d);
        }
      }
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const uint64_t d = (uint64_t)key[j] - (uint64_t)jt.kmin;
        brow[j] = ((word[j] >> (d & 31)) & 1) ? (int32_t)d : -1;
      }
    } else {
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const uint64_t d = (uint64_t)key[j] - (uint64_t)jt.kmin;
        brow[j] = (((live >> j) & 1) && d < range) ? b2_ld_keep_i32(jt.lookup + d) : -1;
      }
    }
    uint32_t matched = 0;
#pragma unroll
    for (int j = 0; j < R; ++j) matched |= (uint32_t)(brow[j] >= 0) << j;
    uint32_t emit;
    switch (mode) {
      case B2_JOIN_INNER:
      case B2_JOIN_SEMI: emit = matched; break;
      case B2_JOIN_LEFT: emit = bits; break;
      default: emit = bits & ~matched; break;  // ANTI
    }

    // ---- positions: ballot ranks inside the warp, one reservation per warp batch
    int32_t rel[R];
    int wtotal = 0;
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const uint32_t b = __ballot_sync(FULL_MASK, (emit >> j) & 1);
      rel[j] = ((emit >> j) & 1) ? wtotal + __popc(b & lt_mask) : -1;
      wtotal += __popc(b);
    }
    unsigned long long r = 0;
    if (lane == 0 && wtotal) r = atomicAdd(total, (unsigned long long)wtotal);
    const int64_t off = (int64_t)__shfl_sync(FULL_MASK, r, 0);

    // ---- probe-side columns
    for (int k = 0; k < g.nprobe; ++k) {
      const b2_col_t& c = s.cols[g.probe_cols[k]];
      if (c.dtype == B2_U8) {
        const uint8_t* p = reinterpret_cast<const uint8_t*>(c.data) + row0;
        uint8_t raw[R];
#pragma unroll
        for (int j = 0; j < R; ++j) raw[j] = rel[j] >= 0 ? p[j * 32] : 0;
#pragma unroll
        for (int j = 0; j < R; ++j)
          if (rel[j] >= 0) reinterpret_cast<uint8_t*>(g.probe_out[k])[off + rel[j]] = raw[j];
      } else {
        int64_t* out = reinterpret_cast<int64_t*>(g.probe_out[k]);
        if (g.probe_cols[k] == key_col) {
#pragma unroll
          for (int j = 0; j < R; ++j)
            if (rel[j] >= 0) b2_st_stream(out + off + rel[j], key[j]);
        } else if (k == preA) {
#pragma unroll
          for (int j = 0; j < R; ++j)
            if (rel[j] >= 0) b2_st_stream(out + off + rel[j], pre[j]);
        } else {
          const int64_t* p = reinterpret_cast<const int64_t*>(c.data) + row0;
          int64_t raw[R];
#pragma unroll
          for (int j = 0; j < R; ++j) raw[j] = rel[j] >= 0 ? b2_ld_stream(p + j * 32) : 0;
#pragma unroll
          for (int j = 0; j < R; ++j)
            if (rel[j] >= 0) b2_st_stream(out + off + rel[j], raw[j]);
        }
      }
      if (g.probe_valid[k]) {
        const uint32_t v = c.valid ? b2_valid_bits<R>(c.valid, row0, emit) : emit;
#pragma unroll
        for (int j = 0; j < R; ++j)
          if (rel[j] >= 0 && ((v >> j) & 1))
            atomicOr(g.probe_valid[k] + ((off + rel[j]) >> 5), 1u << ((off + rel[j]) & 31));
      }
    }
    // ---- build-side columns (by build row; on a key-ordered table the row is the key offset)
    for (int k = 0; k < g.nbuild; ++k) {
      const b2_col_t& c = g.build_cols[k];
      if (c.dtype == B2_U8) {
        uint8_t raw[R];
#pragma unroll
        for (int j = 0; j < R; ++j)
          raw[j] = (rel[j] >= 0 && brow[j] >= 0) ? reinterpret_cast<const uint8_t*>(c.data)[brow[j]] : 0;
#pragma unroll
        for (int j = 0; j < R; ++j)
          if (rel[j] >= 0) reinterpret_cast<uint8_t*>(g.build_out[k])[off + rel[j]] = raw[j];
      } else {
        const int64_t fill = c.dtype == B2_F64 ? 0x7ff8000000000000LL : 0;   // NaN like pandas take(-1)
        const int64_t base = g.build_base[k];
        int64_t raw[R];
        if (k == 0 && spec) {
#pragma unroll
          for (int j = 0; j < R; ++j) raw[j] = brow[j] >= 0 ? (spec32 ? base + pay[j] : pay[j]) : fill;
        } else if (c.dtype == B2_U32) {
#pragma unroll
          for (int j = 0; j < R; ++j)
            raw[j] = (rel[j] >= 0 && brow[j] >= 0)
                         ? base + (int64_t)(uint32_t)b2_ld_keep_i32(reinterpret_cast<const int32_t*>(c.data) + brow[j]) : fill;
        } else {
#pragma unroll
          for (int j = 0; j < R; ++j)
            raw[j] = (rel[j] >= 0 && brow[j] >= 0) ? b2_ld_keep_i64(reinterpret_cast<const int64_t*>(c.data) + brow[j]) : fill;
        }
#pragma unroll
        for (int j = 0; j < R; ++j)
          if (rel[j] >= 0) b2_st_stream(reinterpret_cast<int64_t*>(g.build_out[k]) + off + rel[j], raw[j]);
      }
      if (g.build_valid[k]) {
#pragma unroll
        for (int j = 0; j < R; ++j)
          if (rel[j] >= 0 && brow[j] >= 0 && (!c.valid || b2_bit(c.valid, brow[j])))
            atomicOr(g.build_valid[k] + ((off + rel[j]) >> 5), 1u << ((off + rel[j]) & 31));
      }
    }
  }
}


// ---- streaming probe, specialised --------------------------------------------------------------------
// The shape of C3 (and of most star-schema joins): INNER / SEMI probe of a key-ordered table, output =
// [probe key] [one more 8-byte probe column] [one build column], nothing nullable.  One launch, every
// input byte read once, no count pass:
//   trip 1  key + predicate columns + the probe column      (streaming, coalesced)
//   trip 2  presence word + payload at the key offset        (L2-resident table, evict_last)
//   ranks   ballots inside the warp, warp counts summed in shared memory; ONE atomicAdd per 2048-row
//           tile reserves the output range
//   stores  streaming (evict_first), consecutive lanes -> consecutive rows of the reserved range
// Output rows of one tile stay in probe order; tiles land in the order their CTAs reserve.  SQL leaves
// the row order of a join unspecified (the reference's tests sort before comparing,
// tests/integration/test_compatibility.py:7-9).
// BMODE: how the build column is stored -- 0 none, 1 eight bytes, 2 uint32 offsets (+ presence bitmap),
// 3 uint32 offsets in which 0xFFFFFFFF marks "no build row" (B2_COL_SENTINEL: no bitmap access at all)
// The 8 warps of a tile reserve together (two barriers, one atomic) rather than one atomic per warp
// batch: *total is ONE address, and the L2 serves same-address atomics one at a time (~1.5 ns each,
// scripts/microbench/redg.cu) -- 488k reservations per 125M-row partition were most of the kernel's time.
template <bool HAS_P, int BMODE, bool OUT_KEY>
__global__ void __launch_bounds__(B2_BLOCK, 3)
b2_join_stream_kernel(const __grid_constant__ b2_scan_t s, int key_col, int p_col, const __grid_constant__ b2_jointable_t jt,
                      const void* __restrict__ payload, int64_t pay_base, int64_t ntiles, int64_t* __restrict__ out_key,
                      int64_t* __restrict__ out_p, int64_t* __restrict__ out_b, unsigned long long* __restrict__ total) {
  constexpr int R = B2_JOP_R;
  constexpr bool HAS_B = BMODE != 0;
  __shared__ int sh_cnt[2][B2_WARPS];
  __shared__ long long sh_base[2];
  int phase = 0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lt_mask = (1u << lane) - 1;
  const uint64_t range = (uint64_t)jt.range;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * B2_JOP_TILE + (int64_t)warp * (32 * R) + lane;
    bool full0;
    const uint32_t inb = b2_bounds_bits<R>(row0, s.n, full0);
    int64_t key[R], pv[R];
    b2_load_batch64<R>(s.cols[key_col].data, row0, inb, full0, key);
    if (HAS_P) b2_load_batch64<R>(s.cols[p_col].data, row0, inb, full0, pv);
    bool full;
    const uint32_t bits = s.nterms ? b2_eval_terms<R>(s, row0, full) : inb;
    int64_t pay[R];
    uint32_t emit = 0;
    if (BMODE == 3) {
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const uint64_t d = (uint64_t)key[j] - (uint64_t)jt.kmin;
        const bool ok = ((bits >> j) & 1) && d < range;
        const uint32_t raw = ok ? (uint32_t)b2_ld_keep_i32(reinterpret_cast<const int32_t*>(payload) + d) : 0xffffffffu;
        pay[j] = (int64_t)raw;
        emit |= (uint32_t)(raw != 0xffffffffu) << j;
      }
    } else {
      uint32_t word[R];
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const uint64_t d = (uint64_t)key[j] - (uint64_t)jt.kmin;
        const bool ok = ((bits >> j) & 1) && d < range;
        word[j] = ok ? (uint32_t)b2_ld_keep_i32(jt.lookup + (d >> 5)) : 0u;
        if (HAS_B) {
          pay[j] = 0;
          if (ok) pay[j] = BMODE == 2 ? (int64_t)(uint32_t)b2_ld_keep_i32(reinterpret_cast<const int32_t*>(payload) + d)
                                      : b2_ld_keep_i64(reinterpret_cast<const int64_t*>(payload) + d);
        }
      }
#pragma unroll
      for (int j = 0; j < R; ++j) emit |= ((word[j] >> (((uint64_t)key[j] - (uint64_t)jt.kmin) & 31)) & 1u) << j;
    }
    int rel[R];
    int wtotal = 0;
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const uint32_t b = __ballot_sync(FULL_MASK, (emit >> j) & 1);
      rel[j] = ((emit >> j) & 1) ? wtotal + __popc(b & lt_mask) : -1;
      wtotal += __popc(b);
    }
    // double-buffered by tile parity: a warp that runs ahead writes the OTHER buffer
    if (lane == 0) sh_cnt[phase][warp] = wtotal;
    __syncthreads();
    if (threadIdx.x == 0) {
      int t = 0;
#pragma unroll
      for (int w = 0; w < B2_WARPS; ++w) t += sh_cnt[phase][w];
      sh_base[phase] = t ? (long long)atomicAdd(total, (unsigned long long)t) : 0;
    }
    __syncthreads();
    int64_t off = sh_base[phase];
    for (int w = 0; w < warp; ++w) off += sh_cnt[phase][w];
    phase ^= 1;
#pragma unroll
    for (int j = 0; j < R; ++j) {
      if (rel[j] < 0) continue;
      if (OUT_KEY) b2_st_stream(out_key + off + rel[j], key[j]);
      if (HAS_P) b2_st_stream(out_p + off + rel[j], pv[j]);
      if (HAS_B) b2_st_stream(out_b + off + rel[j], BMODE >= 2 ? pay_base + pay[j] : pay[j]);
    }
  }
}

extern "C" {

int32_t b2_join_build(const b2_col_t* keys, int32_t nkeys, int64_t n, int32_t* head, int32_t* next,
                      int64_t cap, void* stream) {
  B2_REQUIRE(keys && head && (next || n == 0), "null argument");
  B2_REQUIRE(nkeys >= 1 && nkeys <= B2_MAX_KEYS, "bad nkeys");
  B2_REQUIRE(b2_pow2(cap), "cap must be a power of two");
  B2_REQUIRE(n < ((int64_t)1 << 31), "build side must hold < 2^31 rows");
  if (n <= 0) return B2_OK;
  b2_keycols_arg ka;
  memset(&ka, 0, sizeof(ka));
  ka.n = nkeys;
  for (int k = 0; k < nkeys; ++k) {
    B2_REQUIRE(keys[k].dtype != B2_U8, "join keys must be 64-bit columns");
    ka.c[k] = keys[k];
  }
  int grid = b2_wave_grid(b2_join_build_kernel, B2_BLOCK, (n + B2_BLOCK - 1) / B2_BLOCK);
  b2_join_build_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(ka, n, head, next, cap);
  B2_CHECK_LAUNCH("b2_join_build_kernel");
  return B2_OK;
}

int32_t b2_join_build_dense(const b2_col_t* key, int64_t n, int64_t kmin, int64_t range, int32_t* lookup,
                            int32_t* d_flags, void* stream) {
  B2_REQUIRE(key && lookup && d_flags, "null argument");
  B2_REQUIRE(key->dtype == B2_I64, "dense join needs an int64 key");
  B2_REQUIRE(range > 0, "bad range");
  if (n <= 0) return B2_OK;
  int grid = b2_wave_grid(b2_join_build_dense_kernel, B2_BLOCK, (n + B2_BLOCK - 1) / B2_BLOCK);
  b2_join_build_dense_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(*key, n, kmin, range, lookup, d_flags);
  B2_CHECK_LAUNCH("b2_join_build_dense_kernel");
  return B2_OK;
}

int32_t b2_join_key_layout(const b2_col_t* key, int64_t n, int64_t kmin, int64_t range, const b2_col_t* col,
                           int32_t out_dtype, int64_t base, void* out_data, uint32_t* out_valid,
                           uint32_t* present, void* stream) {
  B2_REQUIRE(key, "null argument");
  B2_REQUIRE(key->dtype == B2_I64, "dense join needs an int64 key");
  B2_REQUIRE(range > 0 && range < (1LL << 31), "bad range");
  B2_REQUIRE(col || present, "nothing to lay out");
  b2_col_t c;
  memset(&c, 0, sizeof(c));
  if (col) {
    B2_REQUIRE(out_data, "null output");
    B2_REQUIRE(out_dtype == col->dtype || (out_dtype == B2_U32 && col->dtype == B2_I64), "bad output type");
    c = *col;
  }
  if (n <= 0) return B2_OK;
  int grid = b2_wave_grid(b2_join_key_layout_kernel, B2_BLOCK, (n + B2_BLOCK - 1) / B2_BLOCK);
  b2_join_key_layout_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(*key, n, kmin, range, c, col ? 1 : 0,
                                                                         out_dtype, base, out_data, out_valid, present);
  B2_CHECK_LAUNCH("b2_join_key_layout_kernel");
  return B2_OK;
}

static int32_t b2_check_join(const b2_scan_t* scan, const int32_t* probe_keys, const b2_jointable_t* jt,
                             int32_t mode, b2_probekeys_arg* pk) {
  int32_t rc = b2_check_scan(scan);
  if (rc) return rc;
  B2_REQUIRE(probe_keys && jt, "null argument");
  B2_REQUIRE(jt->nkeys >= 1 && jt->nkeys <= B2_MAX_KEYS, "bad nkeys");
  B2_REQUIRE(mode >= B2_JOIN_INNER && mode <= B2_JOIN_ANTI, "bad join mode");
  B2_REQUIRE(jt->dense >= 0 && jt->dense <= 2, "bad table kind");
  memset(pk, 0, sizeof(*pk));
  for (int k = 0; k < jt->nkeys; ++k) {
    // b2_for_matches loads build keys as 8-byte words: a one-byte key column would be read past its end
    B2_REQUIRE(jt->keys[k].dtype == B2_I64 || jt->keys[k].dtype == B2_F64, "join keys must be int64 or float64");
    B2_REQUIRE(probe_keys[k] >= 0 && probe_keys[k] < scan->ncols, "probe key out of range");
    B2_REQUIRE(scan->cols[probe_keys[k]].dtype == jt->keys[k].dtype, "probe/build key types differ");
    pk->cols[k] = probe_keys[k];
  }
  if (jt->dense) {
    B2_REQUIRE(jt->nkeys == 1 && jt->lookup && jt->range > 0, "bad dense table");
    B2_REQUIRE(jt->keys[0].dtype == B2_I64, "a direct-address table needs an int64 key");
    // a key-ordered table's build row is the key offset, held in an int32
    B2_REQUIRE(jt->dense == 1 || jt->range < (1LL << 31), "key-ordered table needs range < 2^31");
  } else {
    B2_REQUIRE(jt->head && b2_pow2(jt->cap), "bad chained table");
  }
  return B2_OK;
}

int32_t b2_join_count(const b2_scan_t* scan, const int32_t* probe_keys, const b2_jointable_t* jt, int32_t mode,
                      int64_t* d_tile_off, void* stream) {
  b2_probekeys_arg pk;
  int32_t rc = b2_check_join(scan, probe_keys, jt, mode, &pk);
  if (rc) return rc;
  B2_REQUIRE(d_tile_off, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t ntiles = b2_num_tiles(scan->n);
  if (ntiles > 0) {
    if (jt->dense) {
      int grid = b2_wave_grid(b2_join_count_kernel<true>, B2_BLOCK, ntiles);
      b2_join_count_kernel<true><<<grid, B2_BLOCK, 0, st>>>(*scan, pk, *jt, mode, ntiles, d_tile_off);
    } else {
      int grid = b2_wave_grid(b2_join_count_kernel<false>, B2_BLOCK, ntiles);
      b2_join_count_kernel<false><<<grid, B2_BLOCK, 0, st>>>(*scan, pk, *jt, mode, ntiles, d_tile_off);
    }
    B2_CHECK_LAUNCH("b2_join_count_kernel");
  }
  b2_exclusive_scan_kernel<<<1, B2_SCAN_THREADS, 0, st>>>(d_tile_off, ntiles);
  B2_CHECK_LAUNCH("b2_exclusive_scan_kernel");
  return B2_OK;
}

static int32_t b2_fill_joingather(const b2_scan_t* scan, const b2_jointable_t* jt, int32_t mode, int32_t nprobe,
                                  const int32_t* probe_cols, void* const* probe_out, uint32_t* const* probe_valid,
                                  int32_t nbuild, const b2_col_t* build_cols, const int64_t* build_base,
                                  void* const* build_out, uint32_t* const* build_valid, b2_joingather_arg* g) {
  B2_REQUIRE(nprobe >= 0 && nprobe <= B2_MAX_GATHER && nbuild >= 0 && nbuild <= B2_MAX_GATHER, "too many gather columns");
  // a SEMI / ANTI row has no build row: the chained and direct-address kernels would fill such columns differently
  B2_REQUIRE(nbuild == 0 || mode == B2_JOIN_INNER || mode == B2_JOIN_LEFT, "build columns need an INNER or LEFT join");
  memset(g, 0, sizeof(*g));
  g->nprobe = nprobe;
  g->nbuild = nbuild;
  for (int k = 0; k < nprobe; ++k) {
    B2_REQUIRE(probe_cols[k] >= 0 && probe_cols[k] < scan->ncols && probe_out[k], "bad probe gather");
    g->probe_cols[k] = probe_cols[k];
    g->probe_out[k] = probe_out[k];
    g->probe_valid[k] = probe_valid ? probe_valid[k] : nullptr;
  }
  for (int k = 0; k < nbuild; ++k) {
    B2_REQUIRE(build_out[k], "bad build gather");
    B2_REQUIRE(build_cols[k].dtype != B2_U32 || (jt->dense == 2 && build_base), "uint32 payloads need a key-ordered table");
    g->build_cols[k] = build_cols[k];
    g->build_base[k] = build_base ? build_base[k] : 0;
    g->build_out[k] = build_out[k];
    g->build_valid[k] = build_valid ? build_valid[k] : nullptr;
  }
  return B2_OK;
}

int32_t b2_join_write_gather_keyed(const b2_scan_t* scan, const int32_t* probe_keys, const b2_jointable_t* jt,
                                   int32_t mode, const int64_t* d_tile_off, int32_t* out_probe_idx,
                                   int32_t* out_build_idx, uint8_t* build_matched, int32_t nprobe,
                                   const int32_t* probe_cols, void* const* probe_out,
                                   uint32_t* const* probe_valid, int32_t nbuild, const b2_col_t* build_cols,
                                   const int64_t* build_base, void* const* build_out,
                                   uint32_t* const* build_valid, void* stream) {
  b2_probekeys_arg pk;
  int32_t rc = b2_check_join(scan, probe_keys, jt, mode, &pk);
  if (rc) return rc;
  B2_REQUIRE(d_tile_off, "null argument");
  // the chained SEMI probe stops at the first partner; ANTI rows have none
  B2_REQUIRE(!build_matched || mode == B2_JOIN_INNER || mode == B2_JOIN_LEFT, "build_matched needs an INNER or LEFT join");
  b2_joingather_arg g;
  rc = b2_fill_joingather(scan, jt, mode, nprobe, probe_cols, probe_out, probe_valid, nbuild, build_cols, build_base,
                          build_out, build_valid, &g);
  if (rc) return rc;
  const int64_t ntiles = b2_num_tiles(scan->n);
  if (ntiles == 0) return B2_OK;
  if (jt->dense) {
    int grid = b2_wave_grid(b2_join_write_kernel<true>, B2_BLOCK, ntiles);
    b2_join_write_kernel<true><<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(
        *scan, pk, *jt, mode, ntiles, d_tile_off, out_probe_idx, out_build_idx, build_matched, g);
  } else {
    int grid = b2_wave_grid(b2_join_write_kernel<false>, B2_BLOCK, ntiles);
    b2_join_write_kernel<false><<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(
        *scan, pk, *jt, mode, ntiles, d_tile_off, out_probe_idx, out_build_idx, build_matched, g);
  }
  B2_CHECK_LAUNCH("b2_join_write_kernel");
  return B2_OK;
}

int32_t b2_join_onepass(const b2_scan_t* scan, const int32_t* probe_keys, const b2_jointable_t* jt, int32_t mode,
                        int64_t* d_total, int32_t nprobe, const int32_t* probe_cols,
                        void* const* probe_out, uint32_t* const* probe_valid, int32_t nbuild,
                        const b2_col_t* build_cols, const int64_t* build_base, void* const* build_out,
                        uint32_t* const* build_valid, void* stream) {
  b2_probekeys_arg pk;
  int32_t rc = b2_check_join(scan, probe_keys, jt, mode, &pk);
  if (rc) return rc;
  B2_REQUIRE(d_total, "null argument");
  B2_REQUIRE(jt->dense, "single-pass probe needs a direct-address table");
  b2_joingather_arg g;
  rc = b2_fill_joingather(scan, jt, mode, nprobe, probe_cols, probe_out, probe_valid, nbuild, build_cols, build_base,
                          build_out, build_valid, &g);
  if (rc) return rc;
  const int64_t ntiles = (scan->n + B2_JOP_TILE - 1) / B2_JOP_TILE;
  if (ntiles <= 0) return B2_OK;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* total = reinterpret_cast<unsigned long long*>(d_total);
  // specialised kernel when the shape is [key] [<=1 more probe column] [<=1 build column] on a
  // key-ordered table with nothing nullable; the generic kernel otherwise
  const b2_col_t& kc = scan->cols[pk.cols[0]];
  bool fits = jt->dense == 2 && (mode == B2_JOIN_INNER || mode == B2_JOIN_SEMI) && kc.dtype == B2_I64 && !kc.valid &&
              nbuild <= 1 && nprobe <= 2;
  int p_col = -1, key_out = -1, p_out = -1;
  for (int k = 0; fits && k < nprobe; ++k) {
    const b2_col_t& c = scan->cols[g.probe_cols[k]];
    if (g.probe_valid[k] || c.valid || c.dtype == B2_U8) fits = false;
    else if (g.probe_cols[k] == pk.cols[0] && key_out < 0) key_out = k;
    else if (p_col < 0) { p_col = g.probe_cols[k]; p_out = k; }
    else fits = false;
  }
  if (fits && nbuild == 1)
    fits = !g.build_valid[0] && !g.build_cols[0].valid && g.build_cols[0].dtype != B2_U8;
  if (fits) {
    const bool hp = p_col >= 0, hb = nbuild == 1, ok = key_out >= 0;
    int bmode = 0;
    if (hb) bmode = g.build_cols[0].dtype != B2_U32 ? 1 : ((g.build_cols[0].flags & B2_COL_SENTINEL) ? 3 : 2);
    const void* payload = hb ? g.build_cols[0].data : nullptr;
    const int64_t base = hb ? g.build_base[0] : 0;
    int64_t* o_key = ok ? reinterpret_cast<int64_t*>(g.probe_out[key_out]) : nullptr;
    int64_t* o_p = hp ? reinterpret_cast<int64_t*>(g.probe_out[p_out]) : nullptr;
    int64_t* o_b = hb ? reinterpret_cast<int64_t*>(g.build_out[0]) : nullptr;
#define B2_JS_LAUNCH(HP, BM, OK)                                                                                 \
    do {                                                                                                         \
      int sg = b2_wave_grid(b2_join_stream_kernel<HP, BM, OK>, B2_BLOCK, ntiles);                                \
      b2_join_stream_kernel<HP, BM, OK><<<sg, B2_BLOCK, 0, st>>>(*scan, pk.cols[0], hp ? p_col : 0, *jt,         \
                                                                 payload, base, ntiles, o_key, o_p, o_b, total); \
    } while (0)
#define B2_JS_BM(HP, OK)                                                                                         \
    do {                                                                                                         \
      if (bmode == 0) B2_JS_LAUNCH(HP, 0, OK);                                                                   \
      else if (bmode == 1) B2_JS_LAUNCH(HP, 1, OK);                                                              \
      else if (bmode == 2) B2_JS_LAUNCH(HP, 2, OK);                                                              \
      else B2_JS_LAUNCH(HP, 3, OK);                                                                              \
    } while (0)
    if (!hp && !hb && !ok) fits = false;
    else if (hp && ok) B2_JS_BM(true, true);
    else if (hp) B2_JS_BM(true, false);
    else if (ok) B2_JS_BM(false, true);
    else B2_JS_BM(false, false);
#undef B2_JS_BM
#undef B2_JS_LAUNCH
    if (fits) {
      B2_CHECK_LAUNCH("b2_join_stream_kernel");
      return B2_OK;
    }
  }
  int grid = b2_wave_grid(b2_join_onepass_kernel, B2_BLOCK, ntiles);
  b2_join_onepass_kernel<<<grid, B2_BLOCK, 0, st>>>(*scan, pk.cols[0], *jt, mode, ntiles, total, g);
  B2_CHECK_LAUNCH("b2_join_onepass_kernel");
  return B2_OK;
}

int32_t b2_join_write_gather(const b2_scan_t* scan, const int32_t* probe_keys, const b2_jointable_t* jt,
                             int32_t mode, const int64_t* d_tile_off, int32_t* out_probe_idx,
                             int32_t* out_build_idx, uint8_t* build_matched, int32_t nprobe,
                             const int32_t* probe_cols, void* const* probe_out, uint32_t* const* probe_valid,
                             int32_t nbuild, const b2_col_t* build_cols, void* const* build_out,
                             uint32_t* const* build_valid, void* stream) {
  return b2_join_write_gather_keyed(scan, probe_keys, jt, mode, d_tile_off, out_probe_idx, out_build_idx,
                                    build_matched, nprobe, probe_cols, probe_out, probe_valid, nbuild, build_cols,
                                    nullptr, build_out, build_valid, stream);
}

int32_t b2_join_write(const b2_scan_t* scan, const int32_t* probe_keys, const b2_jointable_t* jt, int32_t mode,
                      const int64_t* d_tile_off, int32_t* out_probe_idx, int32_t* out_build_idx,
                      uint8_t* build_matched, void* stream) {
  B2_REQUIRE(out_probe_idx, "null argument");
  B2_REQUIRE(out_build_idx || mode == B2_JOIN_SEMI || mode == B2_JOIN_ANTI, "out_build_idx required");
  return b2_join_write_gather(scan, probe_keys, jt, mode, d_tile_off, out_probe_idx, out_build_idx, build_matched,
                              0, nullptr, nullptr, nullptr, 0, nullptr, nullptr, nullptr, stream);
}

}  // extern "C"
