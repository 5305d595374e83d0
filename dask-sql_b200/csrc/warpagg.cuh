// warpagg.cuh — warp-aggregated atomics for group keys that repeat (skewed key distributions).
//
// b2_apply_aggs issues one fire-and-forget atomic per row.  That is the right thing for keys that rarely
// collide inside a warp, but the L2 serialises atomics PER ADDRESS (scripts/microbench/redg.cu, "red_hot"):
// under Zipf(1.1) the hottest of 1M keys receives 12 % of all rows and alone costs several times the
// whole uniform-key query.  Two levels of pre-aggregation, entered only for batches that show duplicate
// slots (one MATCH per 32*R rows decides, so uniform keys pay nothing):
//   1. per 32-row step: __match_any_sync groups the lanes by slot; each group's values are combined by
//      shuffles (trip count = the largest group of the step) and its lowest lane issues ONE atomic;
//   2. per CTA: slots seen twice in one step claim an entry of a small shared-memory table (tag by 32-bit
//      CAS).  Every warp then adds its group totals for a claimed slot into ITS OWN row of the entry --
//      plain read-modify-write, race-free because one lane leads a slot per step and steps are sequential
//      within a warp (64-bit shared atomics would be CAS spin loops: ATOMS.CAST.SPIN) -- and the CTA flushes
//      each entry with one global atomic per accumulator when it is done.
#pragma once
#include "common.cuh"

#define B2_HOT_SLOTS 256            // entries of the per-CTA table
#define B2_HOT_MAX_ARRAYS 4         // accumulator arrays it can carry (acc / cnt / rows); more -> level 1 only

struct b2_hot_t {                   // lives in kernel-parameter space; smem pointers are derived per CTA
  int32_t enabled;                  // 0: level 1 only
  int32_t narrays;
  int8_t acc_arr[B2_MAX_AGGS];      // array index of aggregate a's accumulator, -1 = not carried
  int8_t cnt_arr[B2_MAX_AGGS];
  int8_t rows_arr;
  int8_t is_f64[B2_HOT_MAX_ARRAYS]; // array holds doubles (else int64)
  int8_t bit_op[B2_HOT_MAX_ARRAYS]; // B2_AGG_AND / OR / XOR: a bitwise accumulator (heavy-hitter path only); 0 = a sum
};

static inline size_t b2_hot_smem_bytes(const b2_hot_t& h) {
  return h.enabled ? (size_t)B2_HOT_SLOTS * 4 + (size_t)h.narrays * B2_WARPS * B2_HOT_SLOTS * 8 : 0;
}

// host: which accumulator arrays the table carries (SUM-like ones and counts; with `bitwise`, which only the
// heavy-hitter kernel sets, also AND / OR / XOR accumulators)
static inline void b2_make_hot(const b2_scan_t& s, const b2_aggs_arg& aa, const b2_aggstate_t& st, b2_hot_t* h,
                               bool bitwise = false) {
  memset(h, 0, sizeof(*h));
  h->rows_arr = -1;
  int n = 0;
  bool fits = true;
  for (int a = 0; a < B2_MAX_AGGS; ++a) h->acc_arr[a] = h->cnt_arr[a] = -1;
  for (int a = 0; a < aa.n && fits; ++a) {
    if (aa.a[a].col < 0) continue;
    const int dt = s.cols[aa.a[a].col].dtype;
    const int op = aa.a[a].op;
    if (st.acc[a] && (op == B2_AGG_SUM || op == B2_AGG_SUMF)) {
      if (n >= B2_HOT_MAX_ARRAYS) { fits = false; break; }
      h->is_f64[n] = (op == B2_AGG_SUMF || dt == B2_F64) ? 1 : 0;
      h->acc_arr[a] = (int8_t)n++;
    } else if (st.acc[a] && bitwise && op >= B2_AGG_AND && op <= B2_AGG_XOR) {
      if (n >= B2_HOT_MAX_ARRAYS) { fits = false; break; }
      h->bit_op[n] = (int8_t)op;
      h->acc_arr[a] = (int8_t)n++;
    }
    if (st.cnt[a]) {
      if (n >= B2_HOT_MAX_ARRAYS) { fits = false; break; }
      h->is_f64[n] = 0;
      h->cnt_arr[a] = (int8_t)n++;
    }
  }
  if (fits && st.rows) {
    if (n >= B2_HOT_MAX_ARRAYS) fits = false;
    else { h->is_f64[n] = 0; h->rows_arr = (int8_t)n++; }
  }
  const char* e1 = getenv("B200SQL_NO_HOT_TABLE");     // A/B: level 1 (warp) only
  h->narrays = n;
  h->enabled = (fits && n > 0 && !(e1 && e1[0] == '1')) ? 1 : 0;
}

struct b2_hot_smem {                // per-CTA view of the dynamic shared memory
  int32_t* tag;                     // [B2_HOT_SLOTS]  slot id or -1
  int64_t* arr;                     // [narrays][B2_WARPS][B2_HOT_SLOTS]
};

__device__ __forceinline__ b2_hot_smem b2_hot_init(const b2_hot_t& h, uint8_t* smem) {
  b2_hot_smem hs;
  hs.tag = reinterpret_cast<int32_t*>(smem + (size_t)h.narrays * B2_WARPS * B2_HOT_SLOTS * 8);
  hs.arr = reinterpret_cast<int64_t*>(smem);
  if (h.enabled) {
    for (int i = threadIdx.x; i < B2_HOT_SLOTS; i += blockDim.x) hs.tag[i] = -1;
    for (int i = threadIdx.x; i < h.narrays * B2_WARPS * B2_HOT_SLOTS; i += blockDim.x) hs.arr[i] = 0;
    __syncthreads();
  }
  return hs;
}

// combine the values of all lanes whose bit is set in m (the lanes holding the same slot this step);
// every lane of the group ends up with the group's total.  maxc = largest group of the step (warp-uniform).
template <bool F64>
__device__ __forceinline__ int64_t b2_group_sum(uint32_t m, int64_t v, int maxc, int lane) {
  uint32_t others = m & ~(1u << lane);
  int64_t acc = v;
  for (int it = 1; it < maxc; ++it) {
    const int src = others ? __ffs(others) - 1 : lane;
    others &= others - 1;
    const int64_t o = __shfl_sync(FULL_MASK, v, src);
    if (src != lane) {
      if (F64) acc = __double_as_longlong(__longlong_as_double(acc) + __longlong_as_double(o));
      else acc = (int64_t)((uint64_t)acc + (uint64_t)o);
    }
  }
  return acc;
}
// the same for an order-free op: KIND = B2_K_MIN_I / MAX_I (ints or ordered images) / AND / OR / XOR
template <int KIND>
__device__ __forceinline__ int64_t b2_group_reduce(uint32_t m, int64_t v, int maxc, int lane) {
  uint32_t others = m & ~(1u << lane);
  int64_t acc = v;
  for (int it = 1; it < maxc; ++it) {
    const int src = others ? __ffs(others) - 1 : lane;
    others &= others - 1;
    const int64_t o = __shfl_sync(FULL_MASK, v, src);
    if (src != lane) {
      if (KIND == B2_K_MIN_I) acc = o < acc ? o : acc;
      else if (KIND == B2_K_MAX_I) acc = o > acc ? o : acc;
      else if (KIND == B2_K_AND) acc &= o;
      else if (KIND == B2_K_OR) acc |= o;
      else acc ^= o;
    }
  }
  return acc;
}
template <int KIND>
__device__ __forceinline__ void b2_group_reduce_flush(void* acc, int64_t slot, uint32_t m, int64_t v, int maxc, int lane,
                                                      bool issue) {
  const int64_t t = b2_group_reduce<KIND>(m, v, maxc, lane);
  if (issue) b2_atomic_k<KIND>(acc, slot, t);   // one REDG per group
}

// Does this batch repeat slots?  One MATCH on the first step's rows: warp-uniform answer.
template <int R>
__device__ __forceinline__ bool b2_batch_repeats(const int64_t (&slot)[R], int lane) {
  const int64_t k = slot[0] >= 0 ? slot[0] : ~(int64_t)lane;    // dead rows never match anybody
  const uint32_t m = __match_any_sync(FULL_MASK, k);
  return __any_sync(FULL_MASK, __popc(m) > 1);
}

// The aggregated counterpart of b2_apply_aggs (same arguments, same results up to float summation order).
template <int R, class LD>
__device__ __forceinline__ void b2_apply_aggs_grouped(const b2_scan_t& s, const LD& ld, const b2_agg_t* __restrict__ aggs,
                                                      int naggs, const b2_aggstate_t& st, const int64_t (&slot)[R],
                                                      const b2_hot_t& hot, const b2_hot_smem& hs) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t row0 = ld.row0;
  uint32_t live = 0;
#pragma unroll
  for (int j = 0; j < R; ++j) live |= (uint32_t)(slot[j] >= 0) << j;
  if (st.out_slot) {
#pragma unroll
    for (int j = 0; j < R; ++j)
      if (row0 + (int64_t)j * 32 < s.n) st.out_slot[row0 + (int64_t)j * 32] = (int32_t)slot[j];
  }
  // ---- groups of every step, their leaders, and where each group's totals go
  uint32_t grp[R];          // lanes sharing this lane's slot in step j
  uint32_t lead = 0;        // bit j: this lane leads its group in step j (and the row is live)
  int16_t where[R];         // >= 0: entry of the CTA's hot table; -1: global memory
  uint8_t maxc[R];
#pragma unroll
  for (int j = 0; j < R; ++j) {
    const int64_t k = slot[j] >= 0 ? slot[j] : ~(int64_t)lane;
    grp[j] = __match_any_sync(FULL_MASK, k);
    const int c = __popc(grp[j]);
    maxc[j] = (uint8_t)__reduce_max_sync(FULL_MASK, (unsigned)c);
    const bool leader = ((live >> j) & 1) && (__ffs(grp[j]) - 1 == lane);
    lead |= (uint32_t)leader << j;
    where[j] = -1;
    if (hot.enabled && leader) {
      const uint32_t h0 = (uint32_t)(((uint64_t)slot[j] * 0x9e3779b97f4a7c15ULL) >> 40) & (B2_HOT_SLOTS - 1);
#pragma unroll
      for (int probe = 0; probe < 2; ++probe) {
        const uint32_t h = (h0 + probe) & (B2_HOT_SLOTS - 1);
        int32_t t = hs.tag[h];
        if (t == -1 && c > 1) {       // seen twice in one step: worth an entry
          const int32_t old = atomicCAS(hs.tag + h, -1, (int32_t)slot[j]);
          t = old == -1 ? (int32_t)slot[j] : old;
        }
        if (t == (int32_t)slot[j]) { where[j] = (int16_t)h; break; }
        if (t == -1) break;           // empty and not claimed: the slot is not in the table
      }
    }
    __syncwarp();                     // claims of this step are visible to the next step's lookups of this warp
  }
  // ---- COUNT(*) and existence
  if (st.rows) {
#pragma unroll
    for (int j = 0; j < R; ++j) {
      if ((lead >> j) & 1) {
        const unsigned long long c = (unsigned long long)__popc(grp[j]);
        if (where[j] >= 0) hs.arr[((size_t)hot.rows_arr * B2_WARPS + warp) * B2_HOT_SLOTS + where[j]] += (int64_t)c;
        else atomicAdd(reinterpret_cast<unsigned long long*>(st.rows) + slot[j], c);
      }
      if (hot.enabled) __syncwarp();   // another lane may lead the same slot in the next step
    }
  }
  if (st.present) {
#pragma unroll
    for (int j = 0; j < R; ++j) {
      if (!((lead >> j) & 1)) continue;
      const uint32_t b = 1u << (slot[j] & 31);
      if (!(__ldca(st.present + (slot[j] >> 5)) & b)) atomicOr(st.present + (slot[j] >> 5), b);
    }
  }
  // ---- the aggregates
  for (int a = 0; a < naggs; ++a) {
    const b2_agg_t ag = aggs[a];
    if (ag.col < 0) continue;
    const b2_col_t& c = s.cols[ag.col];
    int64_t raw[R];
    ld.template load<R>(ag.col, live, false, raw);
    uint32_t ok = live;
    if (c.valid || c.dtype == B2_F64) ok &= ~b2_null_bits<R>(c, row0, live, raw);
    void* acc = st.acc[a];
    int64_t* cnt = st.cnt[a];
    const int kind = acc ? b2_agg_kind(ag.op, c.dtype) : B2_K_NONE;
    const int acc_arr = hot.enabled ? hot.acc_arr[a] : -1;
    const int cnt_arr = hot.enabled ? hot.cnt_arr[a] : -1;
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const bool mine = (ok >> j) & 1;
      const bool leader = (lead >> j) & 1;
      const int mc = maxc[j];
      if (cnt) {
        const int64_t n = b2_group_sum<false>(grp[j], mine ? 1 : 0, mc, lane);
        if (leader && n) {
          if (where[j] >= 0 && cnt_arr >= 0) hs.arr[((size_t)cnt_arr * B2_WARPS + warp) * B2_HOT_SLOTS + where[j]] += n;
          else atomicAdd(reinterpret_cast<unsigned long long*>(cnt) + slot[j], (unsigned long long)n);
        }
      }
      if (kind == B2_K_NONE) {
        if (hot.enabled) __syncwarp();
        continue;
      }
      // does ANY row of the group carry a value?  (a group of NULLs must not touch the accumulator)
      const uint32_t okb = __ballot_sync(FULL_MASK, mine);
      const bool any = (okb & grp[j]) != 0;
      if (kind == B2_K_SUM_I || kind == B2_K_SUM_F || kind == B2_K_SUMF_I) {
        const bool f = kind != B2_K_SUM_I;
        int64_t v = 0;
        if (mine) {
          if (kind == B2_K_SUM_I) v = raw[j];
          else if (kind == B2_K_SUM_F) v = __double_as_longlong(__dadd_rn(__longlong_as_double(raw[j]), 0.0));
          else v = __double_as_longlong((double)raw[j]);
        }
        const int64_t t = f ? b2_group_sum<true>(grp[j], v, mc, lane) : b2_group_sum<false>(grp[j], v, mc, lane);
        if (leader && any) {
          if (where[j] >= 0 && acc_arr >= 0) {
            int64_t* p = hs.arr + ((size_t)acc_arr * B2_WARPS + warp) * B2_HOT_SLOTS + where[j];
            *p = f ? __double_as_longlong(__longlong_as_double(*p) + __longlong_as_double(t)) : (int64_t)((uint64_t)*p + (uint64_t)t);
          } else if (f) {
            atomicAdd(reinterpret_cast<double*>(acc) + slot[j], __longlong_as_double(t));
          } else {
            atomicAdd(reinterpret_cast<unsigned long long*>(acc) + slot[j], (unsigned long long)t);
          }
        }
      } else {
        // MIN / MAX (float values as their ordered images) and the bitwise ops: lanes without a value
        // contribute the op's identity
        const bool flt = kind == B2_K_MIN_F || kind == B2_K_MAX_F;
        int64_t ident = 0;
        if (kind == B2_K_MIN_I || kind == B2_K_MIN_F) ident = LLONG_MAX;
        else if (kind == B2_K_MAX_I || kind == B2_K_MAX_F) ident = LLONG_MIN;
        else if (kind == B2_K_AND) ident = -1;
        const int64_t v = mine ? (flt ? b2_ordered_from_bits(raw[j]) : raw[j]) : ident;
        const bool issue = leader && any;
        switch (kind) {
          case B2_K_MIN_I: case B2_K_MIN_F: b2_group_reduce_flush<B2_K_MIN_I>(acc, slot[j], grp[j], v, mc, lane, issue); break;
          case B2_K_MAX_I: case B2_K_MAX_F: b2_group_reduce_flush<B2_K_MAX_I>(acc, slot[j], grp[j], v, mc, lane, issue); break;
          case B2_K_AND: b2_group_reduce_flush<B2_K_AND>(acc, slot[j], grp[j], v, mc, lane, issue); break;
          case B2_K_OR: b2_group_reduce_flush<B2_K_OR>(acc, slot[j], grp[j], v, mc, lane, issue); break;
          default: b2_group_reduce_flush<B2_K_XOR>(acc, slot[j], grp[j], v, mc, lane, issue); break;
        }
      }
      if (hot.enabled) __syncwarp();   // shared-table updates of this step before the next step's
    }
  }
}

// CTA epilogue: one global atomic per (claimed entry, carried array)
__device__ __forceinline__ void b2_hot_flush(const b2_hot_t& hot, const b2_hot_smem& hs, const b2_aggs_arg& aggs,
                                             const b2_aggstate_t& st) {
  if (!hot.enabled) return;
  __syncthreads();
  for (int h = threadIdx.x; h < B2_HOT_SLOTS; h += blockDim.x) {
    const int32_t slot = hs.tag[h];
    if (slot < 0) continue;
    for (int a = 0; a < aggs.n; ++a) {
      if (hot.acc_arr[a] >= 0) {
        const int k = hot.acc_arr[a];
        if (hot.is_f64[k]) {
          double t = 0.0;
          for (int w = 0; w < B2_WARPS; ++w) t += __longlong_as_double(hs.arr[((size_t)k * B2_WARPS + w) * B2_HOT_SLOTS + h]);
          // a claimed entry received at least one row; for a never-NULL input (the -0.0 existence
          // indicator's case) it therefore received a value, and t is +0.0 or a real sum, never -0.0
          atomicAdd(reinterpret_cast<double*>(st.acc[a]) + slot, t);
        } else {
          uint64_t t = 0;
          for (int w = 0; w < B2_WARPS; ++w) t += (uint64_t)hs.arr[((size_t)k * B2_WARPS + w) * B2_HOT_SLOTS + h];
          if (t) atomicAdd(reinterpret_cast<unsigned long long*>(st.acc[a]) + slot, (unsigned long long)t);
        }
      }
      if (hot.cnt_arr[a] >= 0) {
        uint64_t t = 0;
        for (int w = 0; w < B2_WARPS; ++w) t += (uint64_t)hs.arr[((size_t)hot.cnt_arr[a] * B2_WARPS + w) * B2_HOT_SLOTS + h];
        if (t) atomicAdd(reinterpret_cast<unsigned long long*>(st.cnt[a]) + slot, (unsigned long long)t);
      }
    }
    if (hot.rows_arr >= 0) {
      uint64_t t = 0;
      for (int w = 0; w < B2_WARPS; ++w) t += (uint64_t)hs.arr[((size_t)hot.rows_arr * B2_WARPS + w) * B2_HOT_SLOTS + h];
      if (t) atomicAdd(reinterpret_cast<unsigned long long*>(st.rows) + slot, (unsigned long long)t);
    }
  }
}

// =====================================================================================================
// Level 0 for heavy hitters: thread-private accumulators.
//
// Measured on H100 (scripts/microbench/redg.cu): MATCH.ANY costs ~4 cycles per DISTINCT value per warp
// instruction and the unit is shared by the SM, so grouping every 32-row step by match (above) is capped
// by it.  The rows that hurt, though, belong to a handful of keys.  A sampling pre-pass
// (b2_hot_slots) names up to B2_HH_MAX heavy hitters; the aggregation kernel keeps, for each of them and
// each carried accumulator, one partial PER THREAD in shared memory ([array][hitter][thread]: consecutive
// lanes -> consecutive words, conflict-free) and updates it with a plain load-add-store -- no atomics, no
// cross-lane traffic.  Every other row takes the usual fire-and-forget global atomic.  At the end the CTA
// folds its 256 partials per (hitter, array) and issues ONE global atomic each.
// =====================================================================================================
#define B2_HH_MAX 32          // heavy hitters tracked (top of the sample)
#define B2_HH_MAP 512         // single-probe slot -> hitter index map in shared memory (power of two)
#define B2_HH_SAMPLE 32768    // rows sampled by the pre-pass
#define B2_HH_COUNTERS 4096   // counters of the pre-pass (power of two)
#define B2_HH_MIN_COUNT 6     // sample occurrences that make a slot a heavy hitter (share >~ 0.02 %)

__device__ __forceinline__ uint32_t b2_hh_hash(int32_t slot) { return (uint32_t)slot * 0x9e3779b1u; }

// One CTA of 1024 threads: strided sample of the key column -> exact counts of the sampled slots in a
// shared hash table -> the B2_HH_MAX most frequent ones (count >= B2_HH_MIN_COUNT) to d_hot, -1 padded.
// A performance hint only: results never depend on which slots are listed.
__global__ void __launch_bounds__(1024)
b2_hot_slots_kernel(const __grid_constant__ b2_col_t key, int64_t n, int64_t kmin, int64_t nslots,
                    int32_t* __restrict__ d_hot) {
  __shared__ int32_t tag[B2_HH_COUNTERS];
  __shared__ uint32_t cnt[B2_HH_COUNTERS];
  __shared__ unsigned long long best;
  for (int i = threadIdx.x; i < B2_HH_COUNTERS; i += 1024) { tag[i] = -1; cnt[i] = 0; }
  __syncthreads();
  const int64_t m = n < B2_HH_SAMPLE ? n : B2_HH_SAMPLE;
  for (int64_t i = threadIdx.x; i < m; i += 1024) {
    // 32 consecutive rows per sample group, groups spread over the partition
    const int64_t grp = i >> 5, ngrp = (m + 31) >> 5;
    int64_t row = (n / ngrp) * grp + (i & 31);
    if (row >= n) row = n - 1;
    if (key.valid && !b2_bit(key.valid, row)) continue;
    const uint64_t d = (uint64_t)(reinterpret_cast<const int64_t*>(key.data)[row]) - (uint64_t)kmin;
    if (d >= (uint64_t)(nslots - 1)) continue;
    const int32_t slot = (int32_t)d;
    uint32_t h = b2_hh_hash(slot) >> 20;
    for (int probe = 0; probe < 8; ++probe, h = (h + 1) & (B2_HH_COUNTERS - 1)) {
      h &= B2_HH_COUNTERS - 1;
      int32_t t = tag[h];
      if (t == -1) t = atomicCAS(&tag[h], -1, slot), t = (t == -1 ? slot : t);
      if (t == slot) { atomicAdd(&cnt[h], 1u); break; }
    }
  }
  __syncthreads();
  for (int round = 0; round < B2_HH_MAX; ++round) {
    if (threadIdx.x == 0) best = 0;
    __syncthreads();
    unsigned long long mine = 0;
    for (int i = threadIdx.x; i < B2_HH_COUNTERS; i += 1024)
      if (cnt[i] >= B2_HH_MIN_COUNT) {
        const unsigned long long v = ((unsigned long long)cnt[i] << 32) | (unsigned)i;
        mine = v > mine ? v : mine;
      }
    if (mine) atomicMax(&best, mine);
    __syncthreads();
    const unsigned long long b = best;
    if (threadIdx.x == 0) {
      d_hot[round] = b ? tag[(int)(b & 0xffffffffu)] : -1;
      if (b) cnt[(int)(b & 0xffffffffu)] = 0;
    }
    __syncthreads();
  }
}

struct b2_hh_smem {
  int2* map;             // [B2_HH_MAP]  {slot or -1, hitter index}: ONE probe decides
  int64_t* part;         // [narrays][nh][B2_BLOCK] thread-private partials
  int nh;                // hitters the shared memory budget tracks
};

// hitters the shared memory budget allows: 64 KB / (arrays x 256 threads x 8 B)
static inline int b2_hh_capacity(int narrays) {
  if (narrays <= 0) return 0;
  int cap = (64 * 1024) / (narrays * B2_BLOCK * 8);
  return cap > B2_HH_MAX ? B2_HH_MAX : cap;
}
static inline size_t b2_hh_smem_bytes(int narrays) {
  return (size_t)B2_HH_MAP * 8 + (size_t)narrays * b2_hh_capacity(narrays) * B2_BLOCK * 8;
}

__device__ __forceinline__ uint32_t b2_hh_bucket(int32_t slot) { return (b2_hh_hash(slot) >> 16) & (B2_HH_MAP - 1); }

__device__ __forceinline__ b2_hh_smem b2_hh_init(const b2_hot_t& hot, const int32_t* __restrict__ d_hot, int cap,
                                                 uint8_t* smem) {
  b2_hh_smem hs;
  hs.part = reinterpret_cast<int64_t*>(smem);
  hs.map = reinterpret_cast<int2*>(smem + (size_t)hot.narrays * cap * B2_BLOCK * 8);
  for (int i = threadIdx.x; i < B2_HH_MAP; i += blockDim.x) hs.map[i] = make_int2(-1, -1);
  // float partials start at -0.0 (the INT64_MIN bit pattern) and only ever receive x + 0.0: a partial that
  // still reads -0.0 saw no row, -0.0 + -0.0 = -0.0 survives the fold, and anything else (+0.0 included)
  // means "this CTA met the hitter" -- the same convention as the global accumulators' existence mark
  // bitwise partials start at the op's identity (all ones for AND)
  for (int i = threadIdx.x; i < hot.narrays * cap * B2_BLOCK; i += blockDim.x) {
    const int k = i / (cap * B2_BLOCK);
    hs.part[i] = hot.is_f64[k] ? (int64_t)0x8000000000000000LL : hot.bit_op[k] == B2_AGG_AND ? -1 : 0;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // most frequent first; a hitter whose bucket is taken is simply not tracked (its rows take atomics)
    for (int k = 0; k < cap; ++k) {
      const int32_t slot = d_hot[k];
      if (slot < 0) break;
      const uint32_t h = b2_hh_bucket(slot);
      if (hs.map[h].x == -1) hs.map[h] = make_int2(slot, k);
    }
  }
  __syncthreads();
  hs.nh = cap;
  return hs;
}

__device__ __forceinline__ int b2_hh_find(const b2_hh_smem& hs, int64_t slot) {
  const int2 e = hs.map[b2_hh_bucket((int32_t)slot)];
  return (slot >= 0 && e.x == (int32_t)slot) ? e.y : -1;
}

// one aggregate's batch: rows of tracked hitters go to the thread's partial, the rest to global atomics
template <int R, int KIND>
__device__ __forceinline__ void b2_hh_batch(void* acc, int64_t* cnt, const int64_t (&slot)[R], const int64_t (&raw)[R],
                                            uint32_t ok, const int8_t (&hit)[R], int64_t* part_acc, int64_t* part_cnt,
                                            int stride) {
  // part_acc / part_cnt: this thread's partial of hitter 0 for the array (NULL = array not carried);
  // hitter h's partial is `stride` words further per index
#pragma unroll
  for (int j = 0; j < R; ++j) {
    if (!((ok >> j) & 1)) continue;
    const int h = hit[j];
    if (cnt) {
      if (h >= 0 && part_cnt) part_cnt[h * stride] += 1;
      else atomicAdd(reinterpret_cast<unsigned long long*>(cnt) + slot[j], 1ULL);
    }
    if (KIND == B2_K_NONE) continue;
    if (h >= 0 && part_acc && (KIND == B2_K_SUM_I || KIND == B2_K_SUM_F || KIND == B2_K_SUMF_I)) {
      int64_t* p = part_acc + h * stride;
      if (KIND == B2_K_SUM_I) *p = (int64_t)((uint64_t)*p + (uint64_t)raw[j]);
      else if (KIND == B2_K_SUM_F)
        *p = __double_as_longlong(__longlong_as_double(*p) + __dadd_rn(__longlong_as_double(raw[j]), 0.0));
      else *p = __double_as_longlong(__longlong_as_double(*p) + __dadd_rn((double)raw[j], 0.0));
    } else if (h >= 0 && part_acc && (KIND == B2_K_AND || KIND == B2_K_OR || KIND == B2_K_XOR)) {
      int64_t* p = part_acc + h * stride;
      if (KIND == B2_K_AND) *p &= raw[j];
      else if (KIND == B2_K_OR) *p |= raw[j];
      else *p ^= raw[j];
    } else {
      b2_atomic_k<KIND>(acc, slot[j], raw[j]);
    }
  }
}

// b2_apply_aggs with the heavy hitters' rows diverted to the thread-private partials
template <int R, class LD>
__device__ __forceinline__ void b2_apply_aggs_hh(const b2_scan_t& s, const LD& ld, const b2_agg_t* __restrict__ aggs,
                                                 int naggs, const b2_aggstate_t& st, const int64_t (&slot)[R],
                                                 const b2_hot_t& hot, const b2_hh_smem& hs) {
  const int64_t row0 = ld.row0;
  const int tid = threadIdx.x;
  const int stride = B2_BLOCK;           // words between the partials of consecutive hitters
  uint32_t live = 0;
  int8_t hit[R];                         // index of the tracked heavy hitter this row belongs to, -1 = none
#pragma unroll
  for (int j = 0; j < R; ++j) {
    live |= (uint32_t)(slot[j] >= 0) << j;
    hit[j] = (int8_t)b2_hh_find(hs, slot[j]);
  }
  if (st.out_slot) {
#pragma unroll
    for (int j = 0; j < R; ++j)
      if (row0 + (int64_t)j * 32 < s.n) st.out_slot[row0 + (int64_t)j * 32] = (int32_t)slot[j];
  }
  if (st.rows) {
    int64_t* pr = hot.rows_arr >= 0 ? hs.part + (size_t)hot.rows_arr * hs.nh * stride + tid : nullptr;
#pragma unroll
    for (int j = 0; j < R; ++j) {
      if (!((live >> j) & 1)) continue;
      if (hit[j] >= 0 && pr) pr[hit[j] * stride] += 1;
      else atomicAdd(reinterpret_cast<unsigned long long*>(st.rows) + slot[j], 1ULL);
    }
  }
  if (st.present) {
#pragma unroll
    for (int j = 0; j < R; ++j) {
      if (!((live >> j) & 1)) continue;
      const uint32_t b = 1u << (slot[j] & 31);
      if (!(__ldca(st.present + (slot[j] >> 5)) & b)) atomicOr(st.present + (slot[j] >> 5), b);
    }
  }
  for (int a = 0; a < naggs; ++a) {
    const b2_agg_t ag = aggs[a];
    if (ag.col < 0) continue;
    const b2_col_t& c = s.cols[ag.col];
    int64_t raw[R];
    ld.template load<R>(ag.col, live, false, raw);
    uint32_t ok = live;
    if (c.valid || c.dtype == B2_F64) ok &= ~b2_null_bits<R>(c, row0, live, raw);
    void* acc = st.acc[a];
    int64_t* cnt = st.cnt[a];
    int64_t* pa = hot.acc_arr[a] >= 0 ? hs.part + (size_t)hot.acc_arr[a] * hs.nh * stride + tid : nullptr;
    int64_t* pc = hot.cnt_arr[a] >= 0 ? hs.part + (size_t)hot.cnt_arr[a] * hs.nh * stride + tid : nullptr;
    switch (acc ? b2_agg_kind(ag.op, c.dtype) : B2_K_NONE) {
      case B2_K_SUM_I: b2_hh_batch<R, B2_K_SUM_I>(acc, cnt, slot, raw, ok, hit, pa, pc, stride); break;
      case B2_K_SUM_F: b2_hh_batch<R, B2_K_SUM_F>(acc, cnt, slot, raw, ok, hit, pa, pc, stride); break;
      case B2_K_SUMF_I: b2_hh_batch<R, B2_K_SUMF_I>(acc, cnt, slot, raw, ok, hit, pa, pc, stride); break;
      case B2_K_MIN_I: b2_hh_batch<R, B2_K_MIN_I>(acc, cnt, slot, raw, ok, hit, pa, pc, stride); break;
      case B2_K_MAX_I: b2_hh_batch<R, B2_K_MAX_I>(acc, cnt, slot, raw, ok, hit, pa, pc, stride); break;
      case B2_K_MIN_F: b2_hh_batch<R, B2_K_MIN_F>(acc, cnt, slot, raw, ok, hit, pa, pc, stride); break;
      case B2_K_MAX_F: b2_hh_batch<R, B2_K_MAX_F>(acc, cnt, slot, raw, ok, hit, pa, pc, stride); break;
      case B2_K_AND: b2_hh_batch<R, B2_K_AND>(acc, cnt, slot, raw, ok, hit, pa, pc, stride); break;
      case B2_K_OR: b2_hh_batch<R, B2_K_OR>(acc, cnt, slot, raw, ok, hit, pa, pc, stride); break;
      case B2_K_XOR: b2_hh_batch<R, B2_K_XOR>(acc, cnt, slot, raw, ok, hit, pa, pc, stride); break;
      default: b2_hh_batch<R, B2_K_NONE>(acc, cnt, slot, raw, ok, hit, pa, pc, stride); break;
    }
  }
}

// CTA epilogue: fold the 256 thread partials of every (array, hitter) and issue one global atomic each.
// A hitter that this CTA never met contributes exact zeros (or, for AND, all ones), which are skipped (an
// untouched float SUM accumulator must keep its -0.0 "no group" mark).
__device__ __forceinline__ void b2_hh_flush(const b2_hot_t& hot, const b2_hh_smem& hs, const int32_t* __restrict__ d_hot,
                                            const b2_aggs_arg& aggs, const b2_aggstate_t& st) {
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k = warp; k < hot.narrays * hs.nh; k += B2_WARPS) {      // one warp per (array, hitter)
    const int arr = k / hs.nh, idx = k % hs.nh;
    const int32_t slot = d_hot[idx];
    if (slot < 0) continue;
    const int64_t* p = hs.part + (size_t)k * B2_BLOCK;
    const bool f = hot.is_f64[arr];
    const int bop = hot.bit_op[arr];
    if (bop) {
      uint64_t b = bop == B2_AGG_AND ? ~0ULL : 0ULL;
      for (int t = lane; t < B2_BLOCK; t += 32) {
        const uint64_t v = (uint64_t)p[t];
        b = bop == B2_AGG_AND ? b & v : bop == B2_AGG_OR ? b | v : b ^ v;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const uint64_t v = __shfl_xor_sync(FULL_MASK, b, o);
        b = bop == B2_AGG_AND ? b & v : bop == B2_AGG_OR ? b | v : b ^ v;
      }
      if (lane != 0 || b == (bop == B2_AGG_AND ? ~0ULL : 0ULL)) continue;   // the identity changes nothing
      for (int a = 0; a < aggs.n; ++a) {
        if (hot.acc_arr[a] != arr) continue;
        unsigned long long* d = reinterpret_cast<unsigned long long*>(st.acc[a]) + slot;
        if (bop == B2_AGG_AND) atomicAnd(d, b);
        else if (bop == B2_AGG_OR) atomicOr(d, b);
        else atomicXor(d, b);
      }
      continue;
    }
    double fs = -0.0;
    uint64_t is = 0;
    for (int t = lane; t < B2_BLOCK; t += 32) {
      const int64_t v = p[t];
      if (f) fs += __longlong_as_double(v);
      else is += (uint64_t)v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      fs += __shfl_xor_sync(FULL_MASK, fs, o);
      is += __shfl_xor_sync(FULL_MASK, is, o);
    }
    const bool touched = f ? __double_as_longlong(fs) != (int64_t)0x8000000000000000LL : is != 0;
    if (lane != 0 || !touched) continue;
    // which destination does array `arr` belong to?
    for (int a = 0; a < aggs.n; ++a) {
      if (hot.acc_arr[a] == arr) {
        if (f) atomicAdd(reinterpret_cast<double*>(st.acc[a]) + slot, fs);
        else atomicAdd(reinterpret_cast<unsigned long long*>(st.acc[a]) + slot, (unsigned long long)is);
      }
      if (hot.cnt_arr[a] == arr) atomicAdd(reinterpret_cast<unsigned long long*>(st.cnt[a]) + slot, (unsigned long long)is);
    }
    if (hot.rows_arr == arr) atomicAdd(reinterpret_cast<unsigned long long*>(st.rows) + slot, (unsigned long long)is);
  }
}
