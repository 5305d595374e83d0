// groupby.cuh — group tables fused with the predicate scan:
//   dense  (direct-address, key range known from ingest statistics)
//   hash1  (open addressing, one 64-bit key stored in the table, CAS insert)
//   hashk  (open addressing, 1..4 key columns of any type, per-slot state word)
// plus the fused star pipeline (filter -> key lookup -> aggregate).
#pragma once
#include "common.cuh"
#include "warpagg.cuh"

#define B2_GB_R 8
#define B2_GB_ROWS_PER_BLOCK (B2_BLOCK * B2_GB_R)
#define B2_MAX_PROBE 1024

// ---- dense ------------------------------------------------------------------------------
template <int R>
__device__ __forceinline__ void b2_dense_slots_of(const b2_scan_t& s, const b2_gld& ld, int key_col, int64_t kmin,
                                                  int64_t nslots, int64_t (&slot)[R]) {
  const b2_col_t& kc = s.cols[key_col];
  bool full;
  const uint32_t bits = b2_eval_terms<R>(s, ld, full);
  int64_t key[R];
  ld.load<R>(key_col, bits, full, key);
  uint32_t kvalid = bits;
  if (kc.valid) kvalid = b2_valid_bits<R>(kc.valid, ld.row0, bits);
#pragma unroll
  for (int j = 0; j < R; ++j) {
    slot[j] = -1;
    if ((bits >> j) & 1) {
      if (!((kvalid >> j) & 1)) slot[j] = nslots - 1;
      else {
        const uint64_t d = (uint64_t)key[j] - (uint64_t)kmin;
        slot[j] = d < (uint64_t)(nslots - 1) ? (int64_t)d : -1;  // out of range cannot happen if stats are right
      }
    }
  }
}

__device__ __forceinline__ void b2_dense_body(const b2_scan_t& s, const b2_gld& ld, int key_col, int64_t kmin,
                                              int64_t nslots, const b2_aggs_arg& aggs, const b2_aggstate_t& st) {
  int64_t slot[B2_GB_R];
  b2_dense_slots_of<B2_GB_R>(s, ld, key_col, kmin, nslots, slot);
  b2_apply_aggs<B2_GB_R>(s, ld, aggs.a, aggs.n, st, slot);
}

__global__ void __launch_bounds__(B2_BLOCK)
b2_groupby_dense_kernel(const __grid_constant__ b2_scan_t s, int key_col, int64_t kmin, int64_t nslots,
                        const __grid_constant__ b2_aggs_arg aggs, const __grid_constant__ b2_aggstate_t st,
                        unsigned long long* ticket) {
  auto body = [&](const b2_gld& ld) { b2_dense_body(s, ld, key_col, kmin, nslots, aggs, st); };
  if (ticket) b2_tile_ticket<B2_GB_R>(s, ticket, body);
  else b2_tile_direct<B2_GB_R>(s, body);
}

// Keys that repeat inside a warp (skewed distributions; chosen by the host from the column's repeat
// statistic): batches whose first step shows duplicate slots pre-aggregate per warp and per CTA
// (warpagg.cuh) instead of issuing one atomic per row.  A separate kernel so that the per-row-atomic
// kernel above keeps its 48 registers / 5 CTAs per SM.
__global__ void __launch_bounds__(B2_BLOCK)
b2_groupby_dense_grouped_kernel(const __grid_constant__ b2_scan_t s, int key_col, int64_t kmin, int64_t nslots,
                                const __grid_constant__ b2_aggs_arg aggs, const __grid_constant__ b2_aggstate_t st,
                                const __grid_constant__ b2_hot_t hot) {
  extern __shared__ __align__(128) uint8_t b2_smem[];
  const b2_hot_smem hs = b2_hot_init(hot, b2_smem);
  b2_tile_direct<B2_GB_R>(s, [&](const b2_gld& ld) {
    int64_t slot[B2_GB_R];
    b2_dense_slots_of<B2_GB_R>(s, ld, key_col, kmin, nslots, slot);
    if (b2_batch_repeats<B2_GB_R>(slot, threadIdx.x & 31))
      b2_apply_aggs_grouped<B2_GB_R>(s, ld, aggs.a, aggs.n, st, slot, hot, hs);
    else
      b2_apply_aggs<B2_GB_R>(s, ld, aggs.a, aggs.n, st, slot);
  });
  b2_hot_flush(hot, hs, aggs, st);
}

// The same for a handful of HEAVY HITTERS named by b2_hot_slots: their rows accumulate in thread-private
// shared-memory partials (no atomics, no match), everything else takes the per-row atomic.
__global__ void __launch_bounds__(B2_BLOCK)
b2_groupby_dense_hh_kernel(const __grid_constant__ b2_scan_t s, int key_col, int64_t kmin, int64_t nslots,
                           const __grid_constant__ b2_aggs_arg aggs, const __grid_constant__ b2_aggstate_t st,
                           const __grid_constant__ b2_hot_t hot, const int32_t* __restrict__ d_hot, int cap) {
  extern __shared__ __align__(128) uint8_t b2_smem[];
  const b2_hh_smem hs = b2_hh_init(hot, d_hot, cap, b2_smem);
  b2_tile_direct<B2_GB_R>(s, [&](const b2_gld& ld) {
    int64_t slot[B2_GB_R];
    b2_dense_slots_of<B2_GB_R>(s, ld, key_col, kmin, nslots, slot);
    b2_apply_aggs_hh<B2_GB_R>(s, ld, aggs.a, aggs.n, st, slot, hot, hs);
  });
  b2_hh_flush(hot, hs, d_hot, aggs, st);
}

// ---- hash, single 64-bit key ----------------------------------------------------------------
__device__ __forceinline__ int64_t b2_hash1_slot(int64_t* __restrict__ tk, int64_t cap, int64_t key,
                                                 int32_t* __restrict__ flags) {
  uint64_t h = b2_mix64((uint64_t)key) & (uint64_t)(cap - 1);
  for (int probe = 0; probe < B2_MAX_PROBE; ++probe) {
    const int64_t cur = b2_ld_cg_i64(tk + h);
    if (cur == key) return (int64_t)h;
    if (cur == B2_EMPTY_KEY) {
      const unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(tk + h),
                                               (unsigned long long)B2_EMPTY_KEY, (unsigned long long)key);
      if (old == (unsigned long long)B2_EMPTY_KEY || old == (unsigned long long)key) return (int64_t)h;
    }
    h = (h + 1) & (uint64_t)(cap - 1);
  }
  flags[0] = 1;  // overflow: caller retries with a larger table
  return -1;
}

__device__ __forceinline__ void b2_hash1_body(const b2_scan_t& s, const b2_gld& ld, int key_col, int64_t* __restrict__ tk,
                                              int64_t cap, const b2_aggs_arg& aggs, const b2_aggstate_t& st,
                                              int32_t* __restrict__ flags) {
  const b2_col_t& kc = s.cols[key_col];
  bool full;
  const uint32_t bits = b2_eval_terms<B2_GB_R>(s, ld, full);
  int64_t key[B2_GB_R];
  ld.load<B2_GB_R>(key_col, bits, full, key);
  const uint32_t knull = b2_null_bits<B2_GB_R>(kc, ld.row0, bits, key);
  int64_t slot[B2_GB_R];
#pragma unroll
  for (int j = 0; j < B2_GB_R; ++j) {
    slot[j] = -1;
    if (!((bits >> j) & 1)) continue;
    int64_t k = key[j];
    if ((knull >> j) & 1) { slot[j] = cap; flags[1] = 1; continue; }
    if (kc.dtype == B2_F64 && k == (int64_t)0x8000000000000000LL) k = 0;  // -0.0 groups with 0.0
    else if (k == B2_EMPTY_KEY) { slot[j] = cap + 1; flags[2] = 1; continue; }
    slot[j] = b2_hash1_slot(tk, cap, k, flags);
  }
  b2_apply_aggs<B2_GB_R>(s, ld, aggs.a, aggs.n, st, slot);
}

__global__ void __launch_bounds__(B2_BLOCK)
b2_groupby_hash1_kernel(const __grid_constant__ b2_scan_t s, int key_col, int64_t* __restrict__ tk, int64_t cap,
                        const __grid_constant__ b2_aggs_arg aggs, const __grid_constant__ b2_aggstate_t st,
                        int32_t* __restrict__ flags) {
  b2_tile_direct<B2_GB_R>(s, [&](const b2_gld& ld) { b2_hash1_body(s, ld, key_col, tk, cap, aggs, st, flags); });
}

// ---- hash, composite keys -------------------------------------------------------------------
struct b2_keys_arg {
  int32_t cols[B2_MAX_KEYS];
  int32_t n;
};

__device__ __forceinline__ int64_t b2_hashk_slot(int64_t* __restrict__ tk, uint8_t* __restrict__ tnull,
                                                 int32_t* __restrict__ tstate, int64_t cap, int nkeys,
                                                 const int64_t* key, uint32_t nullmask,
                                                 int32_t* __restrict__ flags) {
  uint64_t hv = 0x9e3779b97f4a7c15ULL ^ nullmask;
  for (int k = 0; k < nkeys; ++k) hv = b2_mix64(hv ^ (uint64_t)key[k]);
  uint64_t h = hv & (uint64_t)(cap - 1);
  int probe = 0;
  int spins = 0;
  while (probe < B2_MAX_PROBE) {
    int32_t stt = __ldcg(tstate + h);
    if (stt == 0) {
      const int32_t old = atomicCAS(tstate + h, 0, 1);
      if (old == 0) {  // we own the slot: publish the key, then mark ready
        for (int k = 0; k < nkeys; ++k) tk[(int64_t)k * cap + h] = key[k];
        tnull[h] = (uint8_t)nullmask;
        __threadfence();
        atomicExch(tstate + h, 2);
        return (int64_t)h;
      }
      stt = old;
    }
    if (stt == 1) {
      // another thread is publishing this slot: re-read (independent thread scheduling lets the
      // publisher progress).  The spin is bounded so that no input can ever hang the kernel: on
      // exhaustion the caller sees the overflow flag and retries with a fresh, larger table.
      if (++spins > (1 << 20)) break;
      continue;
    }
    // ready: compare
    bool same = __ldcg(reinterpret_cast<const unsigned char*>(tnull) + h) == (uint8_t)nullmask;
    for (int k = 0; same && k < nkeys; ++k) same = b2_ld_cg_i64(tk + (int64_t)k * cap + h) == key[k];
    if (same) return (int64_t)h;
    h = (h + 1) & (uint64_t)(cap - 1);
    ++probe;
  }
  flags[0] = 1;
  return -1;
}

__device__ __forceinline__ void b2_hashk_body(const b2_scan_t& s, const b2_gld& ld, const b2_keys_arg& keys,
                                              int64_t* __restrict__ tk, uint8_t* __restrict__ tnull,
                                              int32_t* __restrict__ tstate, int64_t cap, const b2_aggs_arg& aggs,
                                              const b2_aggstate_t& st, int32_t* __restrict__ flags) {
  bool full;
  const uint32_t bits = b2_eval_terms<B2_GB_R>(s, ld, full);
  int64_t kv[B2_MAX_KEYS][B2_GB_R];
  uint32_t knull[B2_MAX_KEYS];
#pragma unroll
  for (int k = 0; k < B2_MAX_KEYS; ++k) {
    knull[k] = 0;
    if (k < keys.n) {
      ld.load<B2_GB_R>(keys.cols[k], bits, full, kv[k]);
      knull[k] = b2_null_bits<B2_GB_R>(s.cols[keys.cols[k]], ld.row0, bits, kv[k]);
    }
  }
  int64_t slot[B2_GB_R];
#pragma unroll
  for (int j = 0; j < B2_GB_R; ++j) {
    slot[j] = -1;
    if (!((bits >> j) & 1)) continue;
    int64_t key[B2_MAX_KEYS];
    uint32_t nullmask = 0;
#pragma unroll
    for (int k = 0; k < B2_MAX_KEYS; ++k) {
      key[k] = 0;
      if (k < keys.n) {
        int64_t v = kv[k][j];
        if ((knull[k] >> j) & 1) { nullmask |= 1u << k; v = 0; }
        else if (s.cols[keys.cols[k]].dtype == B2_F64 && v == (int64_t)0x8000000000000000LL) v = 0;
        key[k] = v;
      }
    }
    slot[j] = b2_hashk_slot(tk, tnull, tstate, cap, keys.n, key, nullmask, flags);
  }
  b2_apply_aggs<B2_GB_R>(s, ld, aggs.a, aggs.n, st, slot);
}

__global__ void __launch_bounds__(B2_BLOCK)
b2_groupby_hashk_kernel(const __grid_constant__ b2_scan_t s, const __grid_constant__ b2_keys_arg keys,
                        int64_t* __restrict__ tk, uint8_t* __restrict__ tnull, int32_t* __restrict__ tstate,
                        int64_t cap, const __grid_constant__ b2_aggs_arg aggs,
                        const __grid_constant__ b2_aggstate_t st, int32_t* __restrict__ flags) {
  b2_tile_direct<B2_GB_R>(s, [&](const b2_gld& ld) {
    b2_hashk_body(s, ld, keys, tk, tnull, tstate, cap, aggs, st, flags);
  });
}

// ---- fused star pipeline ----------------------------------------------------------------------
__global__ void __launch_bounds__(B2_BLOCK)
b2_dense_slots_kernel(const __grid_constant__ b2_col_t key, int64_t n, int64_t kmin, int32_t null_slot,
                      int32_t* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; i < n; i += (int64_t)gridDim.x * B2_BLOCK) {
    const int64_t raw = b2_load_raw(key, i);
    out[i] = b2_is_null(key, i, raw) ? null_slot : (int32_t)(raw - kmin);
  }
}

// the 32-bit image that the star scans stream in place of an int64 column (include/b200sql.h, b2_narrow_image)
__global__ void __launch_bounds__(B2_BLOCK)
b2_narrow_image_kernel(const int64_t* __restrict__ data, const uint8_t* __restrict__ valid, int64_t n, int64_t base,
                       uint32_t* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; i < n; i += (int64_t)gridDim.x * B2_BLOCK)
    out[i] = (valid && !b2_bit(valid, i)) ? 0u : (uint32_t)((uint64_t)data[i] - (uint64_t)base);
}

__global__ void __launch_bounds__(B2_BLOCK)
b2_star_build_dense_kernel(const __grid_constant__ b2_col_t pk, const int32_t* __restrict__ sel, int64_t n_sel,
                           const int32_t* __restrict__ slot_of_row, int64_t kmin, int64_t range,
                           int32_t* __restrict__ lookup, int32_t* __restrict__ flags) {
  for (int64_t i = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; i < n_sel; i += (int64_t)gridDim.x * B2_BLOCK) {
    const int64_t r = sel ? sel[i] : i;
    const int64_t raw = b2_load_raw(pk, r);
    if (b2_is_null(pk, r, raw)) continue;  // NULL keys never join (join.py:202-213)
    const uint64_t d = (uint64_t)raw - (uint64_t)kmin;
    if (d >= (uint64_t)range) continue;
    const int32_t old = atomicExch(lookup + d, slot_of_row[i]);
    if (old != -1) flags[0] = 1;  // duplicate build key
  }
}

// Build side of the star pipeline straight from the UNFILTERED dimension partitions when both the join
// key and the group key are dense: a ranked bitmap (include/b200sql.h, b2_starlookup_t.dir) instead of
// an int32 per key, so that keys whose dimension row fails the predicate cost one bit of L2, not four
// bytes.  Three steps over all partitions, in stream order, no host sync and nothing materialised:
//   MARK  (every partition): predicate -> set the key's bit; a bit already set is a duplicate build key;
//   rank  (once): exclusive scan of the words' popcounts into their rank fields;
//   FILL  (every partition): predicate again -> slots[rank + set bits below the key's] = group slot.
// The rank is global, so every partition's MARK must precede the scan.
//
// The slots are packed `slot_bits` (16, 21 or 32) wide, k = 64 / slot_bits to a 64-bit word, none
// crossing a word: entry i is bits [(i mod k) * slot_bits, + slot_bits) of word i / k.  32 bits is
// a plain int32 array.  b2_slot_word is the only place that divides by k.
__device__ __forceinline__ uint32_t b2_slot_word(uint32_t pos, int slot_bits) {
  return slot_bits == 16 ? pos >> 2 : __umulhi(pos, 0x55555556u);   // pos / 3, exact for pos < 2^31
}

template <bool FILL>
__global__ void __launch_bounds__(B2_BLOCK)
b2_star_build_scan_kernel(const __grid_constant__ b2_scan_narrow_t sn, int pk_col, int grp_col, int64_t pk_min,
                          int64_t pk_range, int64_t grp_min, int32_t null_slot, uint64_t* __restrict__ dir,
                          void* __restrict__ slots, int slot_bits, int32_t* __restrict__ flags) {
  const b2_scan_t& s = sn.s;
  const int tile_off = (threadIdx.x >> 5) * (32 * B2_GB_R) + (threadIdx.x & 31);
  const b2_col_t& pc = s.cols[pk_col];
  const b2_col_t& gc = s.cols[grp_col];
  for (int64_t base = (int64_t)blockIdx.x * B2_GB_ROWS_PER_BLOCK; base < s.n;
       base += (int64_t)gridDim.x * B2_GB_ROWS_PER_BLOCK) {
    const b2_gld_t<true> ld{&s, base + tile_off};
    bool full;
    const uint32_t bits = b2_eval_terms<B2_GB_R>(s, ld, full);
    int64_t pk[B2_GB_R];
    ld.template load<B2_GB_R>(pk_col, bits, full, pk);
    uint32_t live = bits;
    if (pc.valid) live &= b2_valid_bits<B2_GB_R>(pc.valid, ld.row0, bits);   // NULL keys never join
#pragma unroll
    for (int j = 0; j < B2_GB_R; ++j) {
      const uint64_t d = (uint64_t)pk[j] - (uint64_t)pk_min;
      if (!(((live >> j) & 1) && d < (uint64_t)pk_range)) live &= ~(1u << j);
    }
    if (!FILL) {
#pragma unroll
      for (int j = 0; j < B2_GB_R; ++j) {
        if (!((live >> j) & 1)) continue;
        const uint64_t d = (uint64_t)pk[j] - (uint64_t)pk_min;
        const uint32_t b = 1u << (d & 31);
        if (atomicOr(reinterpret_cast<uint32_t*>(dir + (d >> 5)), b) & b) flags[0] = 1;  // duplicate build key
      }
    } else {
      int64_t grp[B2_GB_R];
      ld.template load<B2_GB_R>(grp_col, live, false, grp);
      uint32_t gnull = 0;
      if (gc.valid) gnull = live & ~b2_valid_bits<B2_GB_R>(gc.valid, ld.row0, live);
      uint32_t pos[B2_GB_R];
      int32_t v[B2_GB_R];
#pragma unroll
      for (int j = 0; j < B2_GB_R; ++j) {
        pos[j] = 0;
        v[j] = 0;
        if (!((live >> j) & 1)) continue;
        const uint64_t d = (uint64_t)pk[j] - (uint64_t)pk_min;
        const uint64_t w = dir[d >> 5];
        pos[j] = (uint32_t)(w >> 32) + __popc((uint32_t)w & ((1u << (d & 31)) - 1));
        v[j] = (gnull >> j) & 1 ? null_slot : (int32_t)(grp[j] - grp_min);
      }
      if (slot_bits == 32 || slot_bits == 16) {
        // whole aligned int32 / halfword entries: a plain store, the last writer wins (16 bits: the little-
        // endian halfword `pos` is bits [(pos mod 4) * 16, + 16) of word pos / 4)
#pragma unroll
        for (int j = 0; j < B2_GB_R; ++j) {
          if (!((live >> j) & 1)) continue;
          if (slot_bits == 32) static_cast<int32_t*>(slots)[pos[j]] = v[j];
          else static_cast<uint16_t*>(slots)[pos[j]] = (uint16_t)v[j];
        }
      } else {
        // 21 bits: the 3 entries of a word come from different dim rows, so the word is updated by CAS, and
        // the entry is REPLACED, not ORed in: two passing rows with the same pk share one directory bit and
        // so one entry, and an OR of their slots could exceed null_slot and send the probe's atomics past
        // the group table before the host reads the duplicate flag.  As with the plain stores, one of the
        // two valid slots wins.  The first guess is the zeroed word.  A round issues the CAS of every
        // pending entry before looking at any result, and the next round retries only the entries that
        // lost, each from the word its CAS returned: a lane waits for a few round trips to L2, not for
        // one per entry and attempt.
        unsigned long long e[B2_GB_R], old[B2_GB_R];
        uint32_t q[B2_GB_R], sh[B2_GB_R];
#pragma unroll
        for (int j = 0; j < B2_GB_R; ++j) {
          q[j] = b2_slot_word(pos[j], 21);
          sh[j] = (pos[j] - q[j] * 3) * 21;
          e[j] = ((unsigned long long)(uint32_t)v[j] & 0x1FFFFFull) << sh[j];
          old[j] = 0;
        }
        unsigned long long* w = reinterpret_cast<unsigned long long*>(slots);
        for (uint32_t pend = live; pend;) {
          unsigned long long seen[B2_GB_R];
#pragma unroll
          for (int j = 0; j < B2_GB_R; ++j)
            if ((pend >> j) & 1) seen[j] = atomicCAS(w + q[j], old[j], (old[j] & ~(0x1FFFFFull << sh[j])) | e[j]);
#pragma unroll
          for (int j = 0; j < B2_GB_R; ++j) {
            if (!((pend >> j) & 1)) continue;
            if (seen[j] == old[j]) pend &= ~(1u << j);
            else old[j] = seen[j];
          }
        }
      }
    }
  }
}

// RANK over tiles of B2_RANK_TILE directory words, in three launches and without scratch memory:
//   (a) b2_star_rank_tile_kernel: every tile's popcount total into the rank half of its first word;
//   (b) b2_star_rank_carry_kernel: one block scans those totals in place into the tiles' offsets;
//   (c) b2_star_rank_tile_kernel<true>: every tile scans its own popcounts from its offset and writes
//       every rank.
// MARK writes only the bit halves, and (a) stores the whole rank half of the words it uses, so nothing
// has to be zeroed for the rank.  2048-word tiles put the C4 directory (10M keys, 312.5k words) on 153
// blocks, all resident at once on an H100.
#define B2_RANK_PER_THREAD 8
#define B2_RANK_TILE (B2_BLOCK * B2_RANK_PER_THREAD)

__device__ __forceinline__ uint32_t* b2_rank_half(uint64_t* dir, int64_t i) {
  return reinterpret_cast<uint32_t*>(dir + i) + 1;   // little-endian: the high half of word i
}

template <bool WRITE>
__global__ void __launch_bounds__(B2_BLOCK) b2_star_rank_tile_kernel(uint64_t* __restrict__ dir, int64_t nwords) {
  __shared__ int warp_sums[B2_WARPS];
  __shared__ uint32_t tile_off;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t t0 = (int64_t)blockIdx.x * B2_RANK_TILE;
  const int64_t i0 = t0 + (int64_t)threadIdx.x * B2_RANK_PER_THREAD;   // a thread's words are consecutive
  if (WRITE && threadIdx.x == 0) tile_off = *b2_rank_half(dir, t0);
  uint32_t bits[B2_RANK_PER_THREAD];
  int tsum = 0;
#pragma unroll
  for (int k = 0; k < B2_RANK_PER_THREAD; ++k) {
    bits[k] = i0 + k < nwords ? (uint32_t)dir[i0 + k] : 0u;
    tsum += __popc(bits[k]);
  }
  int incl = tsum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(FULL_MASK, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();   // also orders thread 0's read of the tile offset before any write of the tile's ranks
  if (!WRITE) {
    if (threadIdx.x == 0) {
      int total = 0;
      for (int w = 0; w < B2_WARPS; ++w) total += warp_sums[w];
      *b2_rank_half(dir, t0) = (uint32_t)total;
    }
    return;
  }
  uint32_t r = tile_off + (uint32_t)(incl - tsum);
  for (int w = 0; w < warp; ++w) r += (uint32_t)warp_sums[w];
#pragma unroll
  for (int k = 0; k < B2_RANK_PER_THREAD; ++k) {
    if (i0 + k < nwords) dir[i0 + k] = (uint64_t)bits[k] | ((uint64_t)r << 32);
    r += __popc(bits[k]);
  }
}

struct b2_scan_io_tile_off {
  uint64_t* dir;
  __device__ int64_t get(int64_t t) const { return *b2_rank_half(dir, t * B2_RANK_TILE); }
  __device__ void put(int64_t t, int64_t v) const { *b2_rank_half(dir, t * B2_RANK_TILE) = (uint32_t)v; }
};

__global__ void __launch_bounds__(B2_SCAN_THREADS) b2_star_rank_carry_kernel(uint64_t* __restrict__ dir, int64_t ntiles) {
  b2_block_exclusive_scan(b2_scan_io_tile_off{dir}, ntiles);
}

__global__ void __launch_bounds__(B2_BLOCK)
b2_star_build_hash_kernel(const __grid_constant__ b2_col_t pk, const int32_t* __restrict__ sel, int64_t n_sel,
                          const int32_t* __restrict__ slot_of_row, int64_t* __restrict__ tk,
                          int32_t* __restrict__ ts, int64_t cap, int32_t* __restrict__ flags) {
  for (int64_t i = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; i < n_sel; i += (int64_t)gridDim.x * B2_BLOCK) {
    const int64_t r = sel ? sel[i] : i;
    const int64_t key = b2_load_raw(pk, r);
    if (b2_is_null(pk, r, key)) continue;
    if (key == B2_EMPTY_KEY) { flags[1] = 1; continue; }  // caller falls back to the general join
    uint64_t h = b2_mix64((uint64_t)key) & (uint64_t)(cap - 1);
    bool done = false;
    for (int probe = 0; probe < B2_MAX_PROBE && !done; ++probe) {
      const unsigned long long old = atomicCAS(reinterpret_cast<unsigned long long*>(tk + h),
                                               (unsigned long long)B2_EMPTY_KEY, (unsigned long long)key);
      if (old == (unsigned long long)B2_EMPTY_KEY) { ts[h] = slot_of_row[i]; done = true; }
      else if (old == (unsigned long long)key) { flags[0] = 1; done = true; }
      else h = (h + 1) & (uint64_t)(cap - 1);
    }
    if (!done) flags[1] = 1;
  }
}

__device__ __forceinline__ int32_t b2_star_lookup(const b2_starlookup_t& lk, int64_t key) {
  if (lk.dense) {
    const uint64_t d = (uint64_t)key - (uint64_t)lk.kmin;
    return d < (uint64_t)lk.range ? b2_ld_keep_i32(lk.lookup + d) : -1;
  }
  uint64_t h = b2_mix64((uint64_t)key) & (uint64_t)(lk.cap - 1);
  for (int probe = 0; probe < B2_MAX_PROBE; ++probe) {
    const int64_t cur = __ldg(reinterpret_cast<const long long*>(lk.table_keys) + h);
    if (cur == key) return b2_ld_keep_i32(lk.table_slots + h);
    if (cur == B2_EMPTY_KEY) return -1;
    h = (h + 1) & (uint64_t)(lk.cap - 1);
  }
  return -1;
}

// rows per lane per batch of the star kernel: 16 rather than 8 or 4 although it halves occupancy, for
// more independent loads in flight per thread.
#define B2_STAR_R 16
template <int R>
__device__ __forceinline__ void b2_star_body(const b2_scan_t& s, const b2_gld_t<true>& ld, int fk_col, const b2_starlookup_t& lk,
                                             const b2_aggs_arg& aggs, const b2_aggstate_t& st) {
  // Two memory round trips per batch instead of four:
  //   1. the join-key column is requested together with the predicate columns (its sectors are
  //      touched anyway unless the predicate is very selective);
  //   2. the first aggregate's input is requested for the rows that passed the predicate WHILE the
  //      pk -> slot lookups are in flight;
  //   3. atomics are fire-and-forget.
  const b2_col_t& kc = s.cols[fk_col];
  bool full0;
  const uint32_t inb = b2_bounds_bits<R>(ld.row0, s.n, full0);
  int64_t key[R];
  ld.load<R>(fk_col, inb, full0, key);
  bool full;
  const uint32_t bits = b2_eval_terms<R>(s, ld, full);
  uint32_t live = bits;
  if (kc.valid) live &= b2_valid_bits<R>(kc.valid, ld.row0, bits);
  // all lookups of the batch are issued before the first one is consumed
  const bool prefetch = aggs.n > 0 && aggs.a[0].col >= 0;
  int64_t pre[R];   // only read when `prefetch`: otherwise aggregate 0 has no input column, or is absent
  int32_t found[R];
  int64_t slot[R];
  if (lk.dense == 2) {
    // ranked bitmap: every directory word first, then the slot reads for the keys whose bit is set.
    // The prefetch is issued between the two so that it stays in flight across both round trips.
    const uint64_t range = (uint64_t)lk.range;
    uint64_t w[R];
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const uint64_t d = (uint64_t)key[j] - (uint64_t)lk.kmin;
      w[j] = (((live >> j) & 1) && d < range) ? (uint64_t)b2_ld_keep_i64(reinterpret_cast<const int64_t*>(lk.dir) + (d >> 5)) : 0;
    }
    if (prefetch) ld.load<R>(aggs.a[0].col, live, false, pre);
    const int sb = lk.slot_bits;   // 16, 21 or 32 (b2_star_agg normalises 0); uniform across the grid
    if (sb == 32) {
      // never a 64-bit read here: with an odd entry count it would run 4 bytes past the array
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const uint32_t b = (uint32_t)((uint64_t)key[j] - (uint64_t)lk.kmin) & 31;
        const uint32_t bits = (uint32_t)w[j];
        found[j] = (bits >> b) & 1 ? b2_ld_keep_i32(lk.lookup + (uint32_t)(w[j] >> 32) + __popc(bits & ((1u << b) - 1))) : -1;
      }
    } else {
      // packed: slot[j] holds the loaded word until it is decoded, found[j] the entry's shift (-1: no
      // partner).  The decoded slot goes to found[j]: kept 32 bits wide it costs the aggregation that
      // follows 16 fewer registers than a 64-bit one.
      const int k = 64 / sb;
      const uint64_t* words = reinterpret_cast<const uint64_t*>(lk.lookup);
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const uint32_t b = (uint32_t)((uint64_t)key[j] - (uint64_t)lk.kmin) & 31;
        const uint32_t bits = (uint32_t)w[j];
        found[j] = -1;
        slot[j] = 0;
        if ((bits >> b) & 1) {
          const uint32_t pos = (uint32_t)(w[j] >> 32) + __popc(bits & ((1u << b) - 1));
          const uint32_t q = b2_slot_word(pos, sb);
          found[j] = (int32_t)((pos - q * k) * sb);
          slot[j] = b2_ld_keep_i64(reinterpret_cast<const int64_t*>(words + q));
        }
      }
      const uint64_t mask = (1ull << sb) - 1;
#pragma unroll
      for (int j = 0; j < R; ++j)
        found[j] = found[j] < 0 ? -1 : (int32_t)(((uint64_t)slot[j] >> found[j]) & mask);
    }
  } else if (lk.dense) {
    const uint64_t range = (uint64_t)lk.range;
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const uint64_t d = (uint64_t)key[j] - (uint64_t)lk.kmin;
      found[j] = (((live >> j) & 1) && d < range) ? b2_ld_keep_i32(lk.lookup + d) : -1;
    }
  } else {
#pragma unroll
    for (int j = 0; j < R; ++j) {
      found[j] = -1;
      if (((live >> j) & 1) && key[j] != B2_EMPTY_KEY) found[j] = b2_star_lookup(lk, key[j]);
    }
  }
  if (lk.dense != 2 && prefetch) ld.load<R>(aggs.a[0].col, live, false, pre);
#pragma unroll
  for (int j = 0; j < R; ++j) slot[j] = found[j];
  // `pre` is passed as it is, never as a pointer chosen at run time: that would put it in local memory
  b2_apply_aggs<R>(s, ld, aggs.a, aggs.n, st, slot, pre);
}

__global__ void __launch_bounds__(B2_BLOCK)
b2_star_agg_kernel(const __grid_constant__ b2_scan_narrow_t sn, int fk_col, const __grid_constant__ b2_starlookup_t lk,
                   const __grid_constant__ b2_aggs_arg aggs, const __grid_constant__ b2_aggstate_t st) {
  const b2_scan_t& s = sn.s;
  b2_tile_direct<B2_STAR_R, true>(s, [&](const b2_gld_t<true>& ld) { b2_star_body<B2_STAR_R>(s, ld, fk_col, lk, aggs, st); });
}

// The partitions of one b2_star_agg_multi launch, all in parameter space: the body reads a partition's scan
// from the constant bank exactly as b2_star_agg_kernel reads its one scan.  Tiles of B2_BLOCK x B2_STAR_R
// rows never cross a partition; partition p owns tiles [tile0[p], tile0[p + 1]).  Tiles [0, nstatic) are
// strided over the CTAs as in b2_tile_direct (no ticket round trip), the rest are handed out by a ticket, so
// that a CTA that runs ahead takes more of the tail and the grid ends together.
struct b2_star_parts_arg {
  b2_scan_narrow_t p[B2_STAR_MAX_PARTS];
  int64_t tile0[B2_STAR_MAX_PARTS + 1];
  int64_t nstatic;
  int32_t nparts;
};

__global__ void __launch_bounds__(B2_BLOCK, 2)
b2_star_agg_multi_kernel(const __grid_constant__ b2_star_parts_arg pa, int fk_col,
                         const __grid_constant__ b2_starlookup_t lk, const __grid_constant__ b2_aggs_arg aggs,
                         const __grid_constant__ b2_aggstate_t st, unsigned long long* __restrict__ ticket) {
  __shared__ long long sh_tile[2];
  const int tile_off = (threadIdx.x >> 5) * (32 * B2_STAR_R) + (threadIdx.x & 31);
  const int64_t tile = (int64_t)B2_BLOCK * B2_STAR_R;
  const int64_t ntiles = pa.tile0[pa.nparts];
  // One call site of the body (a second inlined copy spills).  The ticket of the next tile is taken while
  // the current one runs, into the other half of sh_tile; every CTA takes one ticket past the end.
  auto take = [&](int k) {
    if (threadIdx.x == 0) sh_tile[k] = pa.nstatic + (long long)atomicAdd(ticket, 1ULL);
  };
  int64_t t = blockIdx.x;
  int k = 0;
  if (t >= pa.nstatic) {
    take(0);
    __syncthreads();
    t = sh_tile[0];
  }
  while (t < ntiles) {
    const bool by_ticket = t + gridDim.x >= pa.nstatic;   // the next tile is not a static one: uniform in the CTA
    if (by_ticket) take(k ^ 1);
    int p = 0;
    while (p + 1 < pa.nparts && pa.tile0[p + 1] <= t) ++p;   // skips empty partitions: tile0[p + 1] == tile0[p]
    const b2_scan_t& s = pa.p[p].s;
    const b2_gld_t<true> ld{&s, (t - pa.tile0[p]) * tile + tile_off};
    b2_star_body<B2_STAR_R>(s, ld, fk_col, lk, aggs, st);
    if (by_ticket) {
      __syncthreads();
      k ^= 1;
      t = sh_tile[k];
    } else {
      t += gridDim.x;
    }
  }
}

// 21-bit slots packed from their int32 staging array (b2_star_build_pack): word q = entries 3q .. 3q + 2; the
// entries past the last set bit of the directory were never stored, and are 0
__global__ void __launch_bounds__(B2_BLOCK)
b2_star_pack21_kernel(const uint64_t* __restrict__ dir, int64_t nwords, const int32_t* __restrict__ staged,
                      int64_t nout, uint64_t* __restrict__ slots) {
  const uint64_t last = dir[nwords - 1];
  const int64_t nset = (int64_t)(last >> 32) + __popc((uint32_t)last);
  for (int64_t q = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; q < nout; q += (int64_t)gridDim.x * B2_BLOCK) {
    uint64_t w = 0;
#pragma unroll
    for (int e = 0; e < 3; ++e)
      if (3 * q + e < nset) w |= ((uint64_t)(uint32_t)staged[3 * q + e] & 0x1FFFFFull) << (21 * e);
    slots[q] = w;
  }
}

extern "C" {

static int32_t b2_check_state(const b2_aggs_arg& aa, const b2_aggstate_t* st) {
  B2_REQUIRE(st, "null aggstate");
  for (int a = 0; a < aa.n; ++a) {
    if (aa.a[a].col < 0) { B2_REQUIRE(st->rows, "COUNT(*) needs aggstate.rows"); continue; }
    if (aa.a[a].op == B2_AGG_COUNT) B2_REQUIRE(st->cnt[a], "COUNT needs a cnt array");
    else B2_REQUIRE(st->acc[a], "aggregate needs an acc array");
  }
  return B2_OK;
}
static inline bool b2_pow2(int64_t x) { return x > 0 && (x & (x - 1)) == 0; }
// an int64 column, or its B2_U32 image, which the star scans widen back to int64 as they load it
static inline bool b2_is_int64_scan_col(const b2_col_t& c) { return c.dtype == B2_I64 || c.dtype == B2_U32; }
// the scan check of the star entry points (B2_U32 image columns only with their bases; NULL: none) and their
// kernel parameter
static int32_t b2_check_narrow_scan(const b2_scan_t* scan, const int64_t* bases, b2_scan_narrow_t* out) {
  int32_t rc = b2_check_scan(scan, bases != nullptr);
  if (rc) return rc;
  memset(out, 0, sizeof(*out));
  out->s = *scan;
  if (bases)
    for (int c = 0; c < scan->ncols; ++c) out->base[c] = bases[c];
  return B2_OK;
}

static int32_t b2_groupby_dense_impl(const b2_scan_t* scan, int32_t key_col, int64_t kmin, int64_t nslots,
                                     const b2_agg_t* aggs, int32_t naggs, const b2_aggstate_t* st,
                                     unsigned long long* ticket, void* stream) {
  int32_t rc = b2_check_scan(scan);
  if (rc) return rc;
  b2_aggs_arg aa;
  if ((rc = b2_check_aggs(scan, aggs, naggs, &aa))) return rc;
  if ((rc = b2_check_state(aa, st))) return rc;
  B2_REQUIRE(key_col >= 0 && key_col < scan->ncols, "key column out of range");
  B2_REQUIRE(scan->cols[key_col].dtype == B2_I64 || scan->cols[key_col].dtype == B2_U8, "dense keys must be integers");
  B2_REQUIRE(nslots >= 2, "nslots must cover the key range plus the NULL slot");
  if (scan->n == 0) return B2_OK;
  int64_t nblk = (scan->n + B2_GB_ROWS_PER_BLOCK - 1) / B2_GB_ROWS_PER_BLOCK;
  int grid = b2_wave_grid(b2_groupby_dense_kernel, B2_BLOCK, nblk);
  b2_groupby_dense_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(*scan, key_col, kmin, nslots, aa, *st, ticket);
  B2_CHECK_LAUNCH("b2_groupby_dense_kernel");
  return B2_OK;
}

int32_t b2_groupby_dense(const b2_scan_t* scan, int32_t key_col, int64_t kmin, int64_t nslots,
                         const b2_agg_t* aggs, int32_t naggs, const b2_aggstate_t* st, void* stream) {
  return b2_groupby_dense_impl(scan, key_col, kmin, nslots, aggs, naggs, st, nullptr, stream);
}

int32_t b2_groupby_dense_grouped(const b2_scan_t* scan, int32_t key_col, int64_t kmin, int64_t nslots,
                                 const b2_agg_t* aggs, int32_t naggs, const b2_aggstate_t* st, void* stream) {
  int32_t rc = b2_check_scan(scan);
  if (rc) return rc;
  b2_aggs_arg aa;
  if ((rc = b2_check_aggs(scan, aggs, naggs, &aa))) return rc;
  if ((rc = b2_check_state(aa, st))) return rc;
  B2_REQUIRE(key_col >= 0 && key_col < scan->ncols, "key column out of range");
  B2_REQUIRE(scan->cols[key_col].dtype == B2_I64 || scan->cols[key_col].dtype == B2_U8, "dense keys must be integers");
  B2_REQUIRE(nslots >= 2 && nslots < ((int64_t)1 << 31), "nslots must cover the key range plus the NULL slot, below 2^31");
  if (scan->n == 0) return B2_OK;
  b2_hot_t hot;
  b2_make_hot(*scan, aa, *st, &hot);
  const size_t smem = b2_hot_smem_bytes(hot);
  if (smem > 48 * 1024)
    B2_CUDA_TRY(cudaFuncSetAttribute(b2_groupby_dense_grouped_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int64_t nblk = (scan->n + B2_GB_ROWS_PER_BLOCK - 1) / B2_GB_ROWS_PER_BLOCK;
  int occ = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, b2_groupby_dense_grouped_kernel, B2_BLOCK, smem);
  int64_t grid = (int64_t)b2_sm_count() * (occ < 1 ? 1 : occ);
  if (grid > nblk) grid = nblk;
  if (grid < 1) grid = 1;
  b2_groupby_dense_grouped_kernel<<<(int)grid, B2_BLOCK, smem, (cudaStream_t)stream>>>(*scan, key_col, kmin, nslots, aa, *st, hot);
  B2_CHECK_LAUNCH("b2_groupby_dense_grouped_kernel");
  return B2_OK;
}

int32_t b2_hot_slots(const b2_col_t* key, int64_t n, int64_t kmin, int64_t nslots, int32_t* d_hot, void* stream) {
  B2_REQUIRE(key && d_hot, "null argument");
  B2_REQUIRE(key->dtype == B2_I64, "heavy hitters are sampled from an int64 key column");
  B2_REQUIRE(nslots >= 2 && nslots < ((int64_t)1 << 31), "bad slot range");
  b2_hot_slots_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(*key, n > 0 ? n : 0, kmin, nslots, d_hot);
  B2_CHECK_LAUNCH("b2_hot_slots_kernel");
  return B2_OK;
}

int32_t b2_groupby_dense_hot(const b2_scan_t* scan, int32_t key_col, int64_t kmin, int64_t nslots,
                             const b2_agg_t* aggs, int32_t naggs, const b2_aggstate_t* st, const int32_t* d_hot,
                             void* stream) {
  int32_t rc = b2_check_scan(scan);
  if (rc) return rc;
  b2_aggs_arg aa;
  if ((rc = b2_check_aggs(scan, aggs, naggs, &aa))) return rc;
  if ((rc = b2_check_state(aa, st))) return rc;
  B2_REQUIRE(d_hot, "null heavy-hitter list");
  B2_REQUIRE(key_col >= 0 && key_col < scan->ncols, "key column out of range");
  B2_REQUIRE(scan->cols[key_col].dtype == B2_I64 || scan->cols[key_col].dtype == B2_U8, "dense keys must be integers");
  B2_REQUIRE(nslots >= 2 && nslots < ((int64_t)1 << 31), "nslots must cover the key range plus the NULL slot, below 2^31");
  if (scan->n == 0) return B2_OK;
  b2_hot_t hot;
  b2_make_hot(*scan, aa, *st, &hot, true);
  const int cap = b2_hh_capacity(hot.narrays);
  if (cap == 0)   // nothing SUM-like or bitwise to privatise (MIN / MAX only): the plain kernel
    return b2_groupby_dense(scan, key_col, kmin, nslots, aggs, naggs, st, stream);
  const size_t smem = b2_hh_smem_bytes(hot.narrays);
  if (smem > 48 * 1024)
    B2_CUDA_TRY(cudaFuncSetAttribute(b2_groupby_dense_hh_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int64_t nblk = (scan->n + B2_GB_ROWS_PER_BLOCK - 1) / B2_GB_ROWS_PER_BLOCK;
  int occ = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, b2_groupby_dense_hh_kernel, B2_BLOCK, smem);
  int64_t grid = (int64_t)b2_sm_count() * (occ < 1 ? 1 : occ);
  if (grid > nblk) grid = nblk;
  if (grid < 1) grid = 1;
  b2_groupby_dense_hh_kernel<<<(int)grid, B2_BLOCK, smem, (cudaStream_t)stream>>>(*scan, key_col, kmin, nslots, aa, *st, hot,
                                                                                 d_hot, cap);
  B2_CHECK_LAUNCH("b2_groupby_dense_hh_kernel");
  return B2_OK;
}

int32_t b2_groupby_dense_ordered(const b2_scan_t* scan, int32_t key_col, int64_t kmin, int64_t nslots,
                                 const b2_agg_t* aggs, int32_t naggs, const b2_aggstate_t* st, uint64_t* d_ticket,
                                 void* stream) {
  B2_REQUIRE(d_ticket, "null ticket");
  return b2_groupby_dense_impl(scan, key_col, kmin, nslots, aggs, naggs, st,
                               reinterpret_cast<unsigned long long*>(d_ticket), stream);
}

int32_t b2_groupby_hash1(const b2_scan_t* scan, int32_t key_col, int64_t* table_keys, int64_t cap,
                         const b2_agg_t* aggs, int32_t naggs, const b2_aggstate_t* st, int32_t* d_flags,
                         void* stream) {
  int32_t rc = b2_check_scan(scan);
  if (rc) return rc;
  b2_aggs_arg aa;
  if ((rc = b2_check_aggs(scan, aggs, naggs, &aa))) return rc;
  if ((rc = b2_check_state(aa, st))) return rc;
  B2_REQUIRE(key_col >= 0 && key_col < scan->ncols, "key column out of range");
  B2_REQUIRE(scan->cols[key_col].dtype != B2_U8, "hash1 keys must be 64-bit");
  B2_REQUIRE(table_keys && d_flags, "null argument");
  B2_REQUIRE(b2_pow2(cap), "cap must be a power of two");
  if (scan->n == 0) return B2_OK;
  int64_t nblk = (scan->n + B2_GB_ROWS_PER_BLOCK - 1) / B2_GB_ROWS_PER_BLOCK;
  int grid = b2_wave_grid(b2_groupby_hash1_kernel, B2_BLOCK, nblk);
  b2_groupby_hash1_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(*scan, key_col, table_keys, cap, aa, *st, d_flags);
  B2_CHECK_LAUNCH("b2_groupby_hash1_kernel");
  return B2_OK;
}

int32_t b2_groupby_hashk(const b2_scan_t* scan, const int32_t* key_cols, int32_t nkeys, int64_t* table_keys,
                         uint8_t* table_nulls, int32_t* table_state, int64_t cap, const b2_agg_t* aggs,
                         int32_t naggs, const b2_aggstate_t* st, int32_t* d_flags, void* stream) {
  int32_t rc = b2_check_scan(scan);
  if (rc) return rc;
  b2_aggs_arg aa;
  if ((rc = b2_check_aggs(scan, aggs, naggs, &aa))) return rc;
  if ((rc = b2_check_state(aa, st))) return rc;
  B2_REQUIRE(nkeys >= 1 && nkeys <= B2_MAX_KEYS && key_cols, "bad key list");
  B2_REQUIRE(table_keys && table_nulls && table_state && d_flags, "null argument");
  B2_REQUIRE(b2_pow2(cap), "cap must be a power of two");
  b2_keys_arg ka;
  memset(&ka, 0, sizeof(ka));
  ka.n = nkeys;
  for (int k = 0; k < nkeys; ++k) {
    B2_REQUIRE(key_cols[k] >= 0 && key_cols[k] < scan->ncols, "key column out of range");
    ka.cols[k] = key_cols[k];
  }
  if (scan->n == 0) return B2_OK;
  int64_t nblk = (scan->n + B2_GB_ROWS_PER_BLOCK - 1) / B2_GB_ROWS_PER_BLOCK;
  int grid = b2_wave_grid(b2_groupby_hashk_kernel, B2_BLOCK, nblk);
  b2_groupby_hashk_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(*scan, ka, table_keys, table_nulls, table_state, cap,
                                                                       aa, *st, d_flags);
  B2_CHECK_LAUNCH("b2_groupby_hashk_kernel");
  return B2_OK;
}

int32_t b2_dense_slots(const b2_col_t* key, int64_t n, int64_t kmin, int32_t null_slot, int32_t* out_slot,
                       void* stream) {
  B2_REQUIRE(key && out_slot, "null argument");
  if (n <= 0) return B2_OK;
  int grid = b2_wave_grid(b2_dense_slots_kernel, B2_BLOCK, (n + B2_BLOCK - 1) / B2_BLOCK);
  b2_dense_slots_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(*key, n, kmin, null_slot, out_slot);
  B2_CHECK_LAUNCH("b2_dense_slots_kernel");
  return B2_OK;
}

int32_t b2_narrow_image(const b2_col_t* col, int64_t n, int64_t base, uint32_t* out, void* stream) {
  B2_REQUIRE(col && out, "null argument");
  B2_REQUIRE(col->dtype == B2_I64, "an image is made of an int64 column");
  if (n <= 0) return B2_OK;
  int grid = b2_wave_grid(b2_narrow_image_kernel, B2_BLOCK, (n + B2_BLOCK - 1) / B2_BLOCK);
  b2_narrow_image_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(static_cast<const int64_t*>(col->data), col->valid,
                                                                       n, base, out);
  B2_CHECK_LAUNCH("b2_narrow_image_kernel");
  return B2_OK;
}

int32_t b2_star_build_dense(const b2_col_t* pk, const int32_t* sel, int64_t n_sel, const int32_t* slot_of_row,
                            int64_t kmin, int64_t range, int32_t* lookup, int32_t* d_flags, void* stream) {
  B2_REQUIRE(pk && slot_of_row && lookup && d_flags, "null argument");
  B2_REQUIRE(pk->dtype == B2_I64, "dense lookup needs an int64 key");
  if (n_sel <= 0) return B2_OK;
  int grid = b2_wave_grid(b2_star_build_dense_kernel, B2_BLOCK, (n_sel + B2_BLOCK - 1) / B2_BLOCK);
  b2_star_build_dense_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(*pk, sel, n_sel, slot_of_row, kmin,
                                                                           range, lookup, d_flags);
  B2_CHECK_LAUNCH("b2_star_build_dense_kernel");
  return B2_OK;
}

static int32_t b2_star_build_pass(bool fill, const b2_scan_t* scan, const int64_t* bases, int32_t pk_col,
                                  int32_t grp_col, int64_t pk_min, int64_t pk_range, int64_t grp_min,
                                  int32_t null_slot, uint64_t* dir, void* slots, int32_t slot_bits, int32_t* d_flags,
                                  void* stream) {
  b2_scan_narrow_t sn;
  int32_t rc = b2_check_narrow_scan(scan, bases, &sn);
  if (rc) return rc;
  B2_REQUIRE(pk_col >= 0 && pk_col < scan->ncols && grp_col >= 0 && grp_col < scan->ncols, "column out of range");
  B2_REQUIRE(b2_is_int64_scan_col(scan->cols[pk_col]) && b2_is_int64_scan_col(scan->cols[grp_col]),
             "dense keys must be int64");
  B2_REQUIRE(pk_range > 0 && pk_range < ((int64_t)1 << 31), "bad range");
  if (scan->n == 0) return B2_OK;
  int64_t nblk = (scan->n + B2_GB_ROWS_PER_BLOCK - 1) / B2_GB_ROWS_PER_BLOCK;
  if (fill) {
    int grid = b2_wave_grid(b2_star_build_scan_kernel<true>, B2_BLOCK, nblk);
    b2_star_build_scan_kernel<true><<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(sn, pk_col, grp_col, pk_min, pk_range,
                                                                                  grp_min, null_slot, dir, slots, slot_bits, d_flags);
  } else {
    int grid = b2_wave_grid(b2_star_build_scan_kernel<false>, B2_BLOCK, nblk);
    b2_star_build_scan_kernel<false><<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(sn, pk_col, grp_col, pk_min, pk_range,
                                                                                   grp_min, null_slot, dir, slots, slot_bits, d_flags);
  }
  B2_CHECK_LAUNCH("b2_star_build_scan_kernel");
  return B2_OK;
}

int32_t b2_star_build_mark_narrow(const b2_scan_t* scan, const int64_t* bases, int32_t pk_col, int64_t pk_min,
                                  int64_t pk_range, uint64_t* dir, int32_t* d_flags, void* stream) {
  B2_REQUIRE(dir && d_flags, "null argument");
  return b2_star_build_pass(false, scan, bases, pk_col, pk_col, pk_min, pk_range, 0, 0, dir, nullptr, 32, d_flags,
                            stream);
}

int32_t b2_star_build_mark(const b2_scan_t* scan, int32_t pk_col, int64_t pk_min, int64_t pk_range, uint64_t* dir,
                           int32_t* d_flags, void* stream) {
  return b2_star_build_mark_narrow(scan, nullptr, pk_col, pk_min, pk_range, dir, d_flags, stream);
}

int32_t b2_star_build_rank(uint64_t* dir, int64_t pk_range, void* stream) {
  B2_REQUIRE(dir, "null argument");
  B2_REQUIRE(pk_range > 0 && pk_range < ((int64_t)1 << 31), "bad range");
  const int64_t nwords = (pk_range + 31) / 32;
  const int64_t ntiles = (nwords + B2_RANK_TILE - 1) / B2_RANK_TILE;
  b2_star_rank_tile_kernel<false><<<(unsigned)ntiles, B2_BLOCK, 0, (cudaStream_t)stream>>>(dir, nwords);
  B2_CHECK_LAUNCH("b2_star_rank_tile_kernel<false>");
  b2_star_rank_carry_kernel<<<1, B2_SCAN_THREADS, 0, (cudaStream_t)stream>>>(dir, ntiles);
  B2_CHECK_LAUNCH("b2_star_rank_carry_kernel");
  b2_star_rank_tile_kernel<true><<<(unsigned)ntiles, B2_BLOCK, 0, (cudaStream_t)stream>>>(dir, nwords);
  B2_CHECK_LAUNCH("b2_star_rank_tile_kernel<true>");
  return B2_OK;
}

int32_t b2_star_build_fill(const b2_scan_t* scan, int32_t pk_col, int32_t grp_col, int64_t pk_min,
                           int64_t pk_range, int64_t grp_min, int32_t null_slot, const uint64_t* dir,
                           int32_t* slots, void* stream) {
  return b2_star_build_fill_packed(scan, pk_col, grp_col, pk_min, pk_range, grp_min, null_slot, dir,
                                   reinterpret_cast<uint64_t*>(slots), 32, stream);
}

int32_t b2_star_build_fill_packed(const b2_scan_t* scan, int32_t pk_col, int32_t grp_col, int64_t pk_min,
                                  int64_t pk_range, int64_t grp_min, int32_t null_slot, const uint64_t* dir,
                                  uint64_t* slots, int32_t slot_bits, void* stream) {
  return b2_star_build_fill_narrow(scan, nullptr, pk_col, grp_col, pk_min, pk_range, grp_min, null_slot, dir, slots,
                                   slot_bits, stream);
}

int32_t b2_star_build_fill_narrow(const b2_scan_t* scan, const int64_t* bases, int32_t pk_col, int32_t grp_col,
                                  int64_t pk_min, int64_t pk_range, int64_t grp_min, int32_t null_slot,
                                  const uint64_t* dir, uint64_t* slots, int32_t slot_bits, void* stream) {
  B2_REQUIRE(dir && slots, "null argument");
  B2_REQUIRE(slot_bits == 16 || slot_bits == 21 || slot_bits == 32, "slot_bits must be 16, 21 or 32");
  B2_REQUIRE(slot_bits == 32 || (null_slot >= 0 && null_slot < (1 << slot_bits)), "null_slot does not fit slot_bits");
  B2_REQUIRE(slot_bits == 32 || ((uintptr_t)slots & 7) == 0, "packed slots must be 8-byte aligned");
  return b2_star_build_pass(true, scan, bases, pk_col, grp_col, pk_min, pk_range, grp_min, null_slot,
                            const_cast<uint64_t*>(dir), slots, slot_bits, nullptr, stream);
}

int32_t b2_star_build_hash(const b2_col_t* pk, const int32_t* sel, int64_t n_sel, const int32_t* slot_of_row,
                           int64_t* table_keys, int32_t* table_slots, int64_t cap, int32_t* d_flags,
                           void* stream) {
  B2_REQUIRE(pk && slot_of_row && table_keys && table_slots && d_flags, "null argument");
  B2_REQUIRE(pk->dtype == B2_I64, "star lookup needs an int64 key");
  B2_REQUIRE(b2_pow2(cap), "cap must be a power of two");
  if (n_sel <= 0) return B2_OK;
  int grid = b2_wave_grid(b2_star_build_hash_kernel, B2_BLOCK, (n_sel + B2_BLOCK - 1) / B2_BLOCK);
  b2_star_build_hash_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(*pk, sel, n_sel, slot_of_row, table_keys,
                                                                          table_slots, cap, d_flags);
  B2_CHECK_LAUNCH("b2_star_build_hash_kernel");
  return B2_OK;
}

// the lookup check of the star probes; *out is the kernel parameter (slot_bits 0 normalised to 32)
static int32_t b2_check_starlookup(const b2_starlookup_t* lk, b2_starlookup_t* out) {
  B2_REQUIRE(lk, "null lookup");
  B2_REQUIRE(lk->dense >= 0 && lk->dense <= 2, "bad lookup kind");
  b2_starlookup_t l = *lk;
  if (l.dense == 2) {
    B2_REQUIRE(l.dir && l.lookup && l.range > 0 && l.range < ((int64_t)1 << 31), "bad bitmap lookup");
    if (l.slot_bits == 0) l.slot_bits = 32;
    B2_REQUIRE(l.slot_bits == 16 || l.slot_bits == 21 || l.slot_bits == 32, "slot_bits must be 0, 16, 21 or 32");
    B2_REQUIRE(l.slot_bits == 32 || ((uintptr_t)l.lookup & 7) == 0, "packed slots must be 8-byte aligned");
  }
  else if (l.dense) B2_REQUIRE(l.lookup && l.range > 0, "bad dense lookup");
  else B2_REQUIRE(l.table_keys && l.table_slots && b2_pow2(l.cap), "bad hash lookup");
  *out = l;
  return B2_OK;
}

int32_t b2_star_build_pack(const uint64_t* dir, int64_t pk_range, const int32_t* staged, int64_t capacity,
                           uint64_t* slots, int32_t slot_bits, void* stream) {
  B2_REQUIRE(dir && staged && slots, "null argument");
  B2_REQUIRE(slot_bits == 21, "only 21-bit slots are packed from a staging array");
  B2_REQUIRE(pk_range > 0 && pk_range < ((int64_t)1 << 31), "bad range");
  B2_REQUIRE(capacity >= 0 && capacity <= pk_range, "bad capacity");
  const int64_t nout = (capacity + 2) / 3;
  if (nout == 0) return B2_OK;
  int grid = b2_wave_grid(b2_star_pack21_kernel, B2_BLOCK, (nout + B2_BLOCK - 1) / B2_BLOCK);
  b2_star_pack21_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(dir, (pk_range + 31) / 32, staged, nout, slots);
  B2_CHECK_LAUNCH("b2_star_pack21_kernel");
  return B2_OK;
}

int32_t b2_star_agg_multi(const b2_scan_t* scans, const int64_t* const* bases, int32_t nparts, int32_t fk_col,
                          const b2_starlookup_t* lk, const b2_agg_t* aggs, int32_t naggs, const b2_aggstate_t* st,
                          uint64_t* d_tickets, void* stream) {
  B2_REQUIRE(scans && d_tickets && nparts >= 0, "null argument");
  // out_slot is indexed by the row within a partition: with several partitions they would overwrite each other
  B2_REQUIRE(!st || !st->out_slot || nparts <= 1, "out_slot needs a single partition");
  b2_starlookup_t l;
  int32_t rc = b2_check_starlookup(lk, &l);
  if (rc) return rc;
  b2_aggs_arg aa;
  const int64_t tile = (int64_t)B2_BLOCK * B2_STAR_R;
  for (int32_t first = 0, launch = 0; first < nparts; first += B2_STAR_MAX_PARTS, ++launch) {
    static thread_local b2_star_parts_arg pa;   // 13 KB: not on the caller's stack; the launch copies it
    memset(&pa, 0, sizeof(pa));
    pa.nparts = nparts - first < B2_STAR_MAX_PARTS ? nparts - first : B2_STAR_MAX_PARTS;
    for (int p = 0; p < pa.nparts; ++p) {
      const b2_scan_t* scan = scans + first + p;
      if ((rc = b2_check_narrow_scan(scan, bases ? bases[first + p] : nullptr, &pa.p[p]))) return rc;
      if ((rc = b2_check_aggs(scan, aggs, naggs, &aa))) return rc;
      B2_REQUIRE(fk_col >= 0 && fk_col < scan->ncols, "fk column out of range");
      B2_REQUIRE(b2_is_int64_scan_col(scan->cols[fk_col]), "fk must be int64");
      pa.tile0[p + 1] = pa.tile0[p] + (scan->n + tile - 1) / tile;
    }
    if ((rc = b2_check_state(aa, st))) return rc;
    const int64_t ntiles = pa.tile0[pa.nparts];
    if (ntiles == 0) continue;
    const int grid = b2_wave_grid(b2_star_agg_multi_kernel, B2_BLOCK, ntiles);
    // 90 % static: on C4 (8 x 125M rows, H100) tickets for every tile or for the last 25 % measured the same
    pa.nstatic = ntiles * 9 / 10 / grid * grid;
    if (pa.nstatic > ntiles) pa.nstatic = ntiles;
    b2_star_agg_multi_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(
        pa, fk_col, l, aa, *st, reinterpret_cast<unsigned long long*>(d_tickets) + launch);
    B2_CHECK_LAUNCH("b2_star_agg_multi_kernel");
  }
  return B2_OK;
}

int32_t b2_star_agg(const b2_scan_t* scan, int32_t fk_col, const b2_starlookup_t* lk, const b2_agg_t* aggs,
                    int32_t naggs, const b2_aggstate_t* st, void* stream) {
  return b2_star_agg_narrow(scan, nullptr, fk_col, lk, aggs, naggs, st, stream);
}

int32_t b2_star_agg_narrow(const b2_scan_t* scan, const int64_t* bases, int32_t fk_col, const b2_starlookup_t* lk,
                           const b2_agg_t* aggs, int32_t naggs, const b2_aggstate_t* st, void* stream) {
  b2_scan_narrow_t sn;
  int32_t rc = b2_check_narrow_scan(scan, bases, &sn);
  if (rc) return rc;
  b2_aggs_arg aa;
  if ((rc = b2_check_aggs(scan, aggs, naggs, &aa))) return rc;
  if ((rc = b2_check_state(aa, st))) return rc;
  B2_REQUIRE(fk_col >= 0 && fk_col < scan->ncols, "fk column out of range");
  B2_REQUIRE(b2_is_int64_scan_col(scan->cols[fk_col]), "fk must be int64");
  b2_starlookup_t l;
  if ((rc = b2_check_starlookup(lk, &l))) return rc;
  if (scan->n == 0) return B2_OK;
  int64_t nblk = (scan->n + (int64_t)B2_BLOCK * B2_STAR_R - 1) / ((int64_t)B2_BLOCK * B2_STAR_R);
  int grid = b2_wave_grid(b2_star_agg_kernel, B2_BLOCK, nblk);
  b2_star_agg_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(sn, fk_col, l, aa, *st);
  B2_CHECK_LAUNCH("b2_star_agg_kernel");
  return B2_OK;
}

}  // extern "C"
