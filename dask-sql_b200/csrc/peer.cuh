// peer.cuh — the multi-GPU merge of dense partial group tables as ONE kernel over NVLink peer memory.
//
// What it replaces.  After the fact scan every GPU holds a partial direct-address group table (the
// reference's per-partition `groupby().agg()` chunk, aggregate.py:575-581); the reference combines them
// with dask's tree of concat + re-aggregate.  The NCCL restatement is: presence pass (b2_expr_eval) ->
// ncclReduceScatter per accumulator array -> ncclReduceScatter of the presence bytes -- three to five
// launches, each with NCCL's fixed cost, on a step that lasts well under a millisecond at 8 GPUs.
//
// Here the partial tables live in symmetric memory (the same allocation mapped into every process over
// NVLink / NVSwitch).  Rank r owns the slots [r*count, (r+1)*count).  One launch per rank:
//   1. cross-GPU barrier inside the kernel: CTA 0 stores this step's epoch into every peer's signal row
//      (st.release.sys over NVLink), spins on its own row (ld.acquire.sys), then releases the other CTAs
//      of its grid through a device-scope flag.  After it, every peer's scan of this step has finished.
//   2. every thread owns two consecutive slots of the rank's slice and, per accumulator array, issues the
//      16-byte loads of ALL peers back to back (world requests in flight per thread; remote ones cross
//      NVLink and are served by the owner's L2), then combines them in RANK ORDER -- the result is the
//      same bit pattern on every run and for every rank count's tree shape, which ncclReduceScatter does
//      not promise -- and writes the merged slice to local HBM.
//   3. existence is merged in the same pass, from what the scan kernels maintained: a row counter (> 0
//      after the sum), the -0.0 "never touched" mark of a float SUM accumulator (tested on every peer's
//      RAW bits before anything is added, so no collective ever sees a signed zero), or a presence
//      bitmap (OR of the peers' words).  Output: one byte per slot, what the compaction reads.
// No second barrier: tables are double-buffered by the caller, and a rank can only pass barrier k+1 after
// every rank has finished step k's merge (it precedes their step k+1 scan in stream order), so the table
// of step k is free to be refilled when step k+2 starts.
#pragma once
#include "common.cuh"

__device__ __forceinline__ void b2_st_release_sys(uint64_t* p, uint64_t v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t b2_ld_acquire_sys(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void b2_st_release_gpu(uint64_t* p, uint64_t v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t b2_ld_acquire_gpu(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
// peer data: never through the non-coherent L1 (the same addresses are rewritten every other step)
__device__ __forceinline__ longlong2 b2_ld_peer2(const void* p) {
  longlong2 v;
  asm volatile("ld.relaxed.sys.global.v2.s64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t b2_ld_peer_u32(const void* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ int64_t b2_peer_combine(int op, int64_t a, int64_t b) {
  switch (op) {
    case B2_PEER_SUM_F64: return __double_as_longlong(__longlong_as_double(a) + __longlong_as_double(b));
    case B2_PEER_SUM_I64: return (int64_t)((uint64_t)a + (uint64_t)b);      // wraps like numpy
    case B2_PEER_MIN_I64: return a < b ? a : b;
    case B2_PEER_AND_I64: return a & b;
    case B2_PEER_OR_I64: return a | b;
    case B2_PEER_XOR_I64: return a ^ b;
    default: return a > b ? a : b;                                            // B2_PEER_MAX_I64
  }
}

template <int W>   // W = world size when it is a compile-time 2 / 4 / 8 (fully unrolled peer loop), 0 = generic
__global__ void __launch_bounds__(B2_BLOCK)
b2_peer_merge_kernel(const __grid_constant__ b2_peer_merge_t m) {
  const int world = W ? W : m.world;
  // ---- 1. barrier across the GPUs
  if (blockIdx.x == 0) {
    if ((int)threadIdx.x < world) {
      uint64_t* theirs = reinterpret_cast<uint64_t*>(reinterpret_cast<char*>(m.peer_base[threadIdx.x]) + m.signal_off) + m.rank;
      b2_st_release_sys(theirs, m.epoch);
      const uint64_t* mine = reinterpret_cast<const uint64_t*>(reinterpret_cast<const char*>(m.peer_base[m.rank]) + m.signal_off) + threadIdx.x;
      while (b2_ld_acquire_sys(mine) < m.epoch) __nanosleep(20);
    }
    __syncthreads();
    if (threadIdx.x == 0) b2_st_release_gpu(m.local_ready, m.epoch);
  } else {
    if (threadIdx.x == 0)
      while (b2_ld_acquire_gpu(m.local_ready) < m.epoch) __nanosleep(20);
    __syncthreads();
  }
  // ---- 2 + 3. merge this rank's slice, two slots per thread
  const int64_t npairs = m.count >> 1;          // count is a multiple of 32
  for (int64_t pair = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; pair < npairs; pair += (int64_t)gridDim.x * B2_BLOCK) {
    const int64_t slot = m.lo + 2 * pair;       // global slot of the pair's first element
    bool p0 = false, p1 = false;
    for (int a = 0; a < m.narrays; ++a) {
      const int64_t off = m.array_off[a] + slot * 8;
      longlong2 v[W ? W : B2_MAX_PEERS];
#pragma unroll
      for (int p = 0; p < (W ? W : B2_MAX_PEERS); ++p)
        if (p < world) v[p] = b2_ld_peer2(reinterpret_cast<const char*>(m.peer_base[p]) + off);
      const int op = m.ops[a];
      longlong2 r = v[0];
      if (m.presence_kind == B2_PEER_PRESENT_INDICATOR && a == m.presence_array) {
        p0 = r.x != B2_EMPTY_KEY;
        p1 = r.y != B2_EMPTY_KEY;
      }
#pragma unroll
      for (int p = 1; p < (W ? W : B2_MAX_PEERS); ++p) {
        if (p < world) {
          if (m.presence_kind == B2_PEER_PRESENT_INDICATOR && a == m.presence_array) {
            p0 |= v[p].x != B2_EMPTY_KEY;
            p1 |= v[p].y != B2_EMPTY_KEY;
          }
          r.x = b2_peer_combine(op, r.x, v[p].x);
          r.y = b2_peer_combine(op, r.y, v[p].y);
        }
      }
      if (m.presence_kind == B2_PEER_PRESENT_ROWS && a == m.presence_array) {
        p0 = r.x > 0;
        p1 = r.y > 0;
      }
      *reinterpret_cast<longlong2*>(reinterpret_cast<char*>(m.out[a]) + 16 * pair) = r;
    }
    if (m.presence_kind == B2_PEER_PRESENT_BITMAP) {
      uint32_t w = 0;
      const int64_t woff = m.bitmap_off + (slot >> 5) * 4;
#pragma unroll
      for (int p = 0; p < (W ? W : B2_MAX_PEERS); ++p)
        if (p < world) w |= b2_ld_peer_u32(reinterpret_cast<const char*>(m.peer_base[p]) + woff);
      p0 = (w >> (slot & 31)) & 1;
      p1 = (w >> ((slot & 31) + 1)) & 1;
    }
    *reinterpret_cast<uchar2*>(m.out_present + 2 * pair) = make_uchar2(p0 ? 1 : 0, p1 ? 1 : 0);
  }
}

extern "C" {

int32_t b2_peer_merge(const b2_peer_merge_t* m, void* stream) {
  B2_REQUIRE(m, "null argument");
  B2_REQUIRE(m->world >= 2 && m->world <= B2_MAX_PEERS && m->rank >= 0 && m->rank < m->world, "bad world / rank");
  B2_REQUIRE(m->narrays >= 0 && m->narrays <= B2_PEER_MAX_ARRAYS, "too many arrays");
  B2_REQUIRE(m->count >= 0 && m->count % 32 == 0 && m->lo % 32 == 0, "slices are multiples of 32 slots");
  B2_REQUIRE(m->out_present && m->local_ready && m->epoch > 0, "null output / flag, or epoch 0");
  B2_REQUIRE(m->presence_kind >= B2_PEER_PRESENT_ROWS && m->presence_kind <= B2_PEER_PRESENT_BITMAP, "bad presence kind");
  if (m->presence_kind != B2_PEER_PRESENT_BITMAP)
    B2_REQUIRE(m->presence_array >= 0 && m->presence_array < m->narrays, "presence array out of range");
  for (int p = 0; p < m->world; ++p) B2_REQUIRE(m->peer_base[p], "null peer base");
  for (int a = 0; a < m->narrays; ++a) {
    B2_REQUIRE(m->out[a] && m->array_off[a] % 16 == 0, "null or misaligned array");
    B2_REQUIRE(m->ops[a] >= B2_PEER_SUM_F64 && m->ops[a] <= B2_PEER_XOR_I64, "bad op");
  }
  // enough CTAs to keep world x narrays 16-byte requests per thread in flight on every SM, few enough that
  // a concurrent NCCL kernel (the next step's lookup broadcast) always finds room beside the spinning grid
  int64_t want = (m->count / 2 + B2_BLOCK - 1) / B2_BLOCK;
  const int64_t cap = (int64_t)b2_sm_count() * 4;
  if (want > cap) want = cap;
  if (want < 1) want = 1;
  cudaStream_t st = (cudaStream_t)stream;
  switch (m->world) {
    case 2: b2_peer_merge_kernel<2><<<(int)want, B2_BLOCK, 0, st>>>(*m); break;
    case 4: b2_peer_merge_kernel<4><<<(int)want, B2_BLOCK, 0, st>>>(*m); break;
    case 8: b2_peer_merge_kernel<8><<<(int)want, B2_BLOCK, 0, st>>>(*m); break;
    default: b2_peer_merge_kernel<0><<<(int)want, B2_BLOCK, 0, st>>>(*m); break;
  }
  B2_CHECK_LAUNCH("b2_peer_merge_kernel");
  return B2_OK;
}

}  // extern "C"
