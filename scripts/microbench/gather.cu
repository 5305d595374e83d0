// gather.cu — H100 micro-benchmark behind the star-join lookup layout (DESIGN.md §4): the rate of random
// 4-byte table reads (ld.global.nc.L2::cache_hint with an evict_last policy, the instruction of
// b2_ld_keep_i32) against the table's size, to find where random reads start to miss L2.
//   alone:  random reads only;
//   mix:    next to C4's traffic: an evict_first stream of 24 B per row (fk, x, val), a lookup for every
//           other row, one f64 REDG per two lookups into an 8 MB group table;
//   pair:   the ranked-bitmap probe: an 8-byte directory read {bits, rank}, then, when the key's bit is
//           set (half the keys), the 4-byte slot read it points at.  "table_mb" is the slot array; the
//           directory covers twice as many keys at 8 B per 32 keys (table_mb / 8);
//   star_mix (`gather star`): one C4 partition of b2_star_agg as it is: 125M rows streamed at 24 B per
//           row (evict_first), the directory word (2.5 MB, 10M keys, half of them set) for every row with
//           x > 0 (half), the val prefetch, the slot read for the rows whose bit is set, one f64 REDG
//           into an 8 MB group table per slot read.  The 5M slots are int32 (20 MB), packed 21 bits
//           (13.3 MB) or packed 16 bits (10 MB), in the layout of b2_star_build_fill_packed.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o gather gather.cu ; run on one H100.
// Prints one JSON object per line.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("{\"error\": \"%s at %s:%d\"}\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

__device__ __forceinline__ uint64_t mix64(uint64_t k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33; return k;
}
__device__ __forceinline__ uint64_t policy_keep() {
  uint64_t p;
  asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t policy_stream() {
  uint64_t p;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ int32_t ld_keep_i32(const int32_t* p) {
  int32_t v;
  asm volatile("ld.global.nc.L2::cache_hint.b32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(policy_keep()));
  return v;
}
__device__ __forceinline__ uint64_t ld_keep_u64(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.global.nc.L2::cache_hint.b64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(policy_keep()));
  return v;
}
__device__ __forceinline__ int64_t ld_stream(const int64_t* p) {
  int64_t v;
  asm volatile("ld.global.nc.L2::cache_hint.b64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(policy_stream()));
  return v;
}

#define R 16   // independent rows per thread per batch, as in b2_star_agg_kernel

__global__ void __launch_bounds__(256) alone_kernel(const int32_t* __restrict__ t, uint64_t n, uint64_t nreads, int* out) {
  const uint64_t nthreads = (uint64_t)gridDim.x * blockDim.x;
  int32_t acc = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nreads; i += R * nthreads) {
    int32_t v[R];
#pragma unroll
    for (int j = 0; j < R; ++j) v[j] = ld_keep_i32(t + mix64(i + j * nthreads) % n);
#pragma unroll
    for (int j = 0; j < R; ++j) acc += v[j];
  }
  if (acc == 0x7fffffff) out[0] = acc;
}

// row i: fk[i], x[i], val[i] streamed; rows with x > 0 (half) look fk up; rows whose slot is even (half of
// those) add val into grp[slot % ngrp]
__global__ void __launch_bounds__(256) mix_kernel(const int64_t* __restrict__ fk, const int64_t* __restrict__ x,
                                                  const int64_t* __restrict__ val, const int32_t* __restrict__ t,
                                                  double* grp, uint64_t ngrp, uint64_t nrows) {
  const uint64_t nthreads = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += R * nthreads) {
    int64_t k[R], xv[R], vv[R];
    int32_t s[R];
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const uint64_t r = i + j * nthreads;
      k[j] = r < nrows ? ld_stream(fk + r) : 0;
      xv[j] = r < nrows ? ld_stream(x + r) : 0;
    }
#pragma unroll
    for (int j = 0; j < R; ++j) s[j] = xv[j] > 0 ? ld_keep_i32(t + k[j]) : -1;
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const uint64_t r = i + j * nthreads;
      vv[j] = (s[j] >= 0 && r < nrows) ? ld_stream(val + r) : 0;
    }
#pragma unroll
    for (int j = 0; j < R; ++j)
      if (s[j] >= 0 && !(s[j] & 1)) atomicAdd(grp + (uint64_t)s[j] % ngrp, __longlong_as_double(vv[j]));
  }
}

__global__ void __launch_bounds__(256) pair_kernel(const uint64_t* __restrict__ dir, const int32_t* __restrict__ slots,
                                                   uint64_t nkeys, uint64_t nreads, int* out) {
  const uint64_t nthreads = (uint64_t)gridDim.x * blockDim.x;
  int32_t acc = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nreads; i += R * nthreads) {
    uint64_t key[R], w[R];
#pragma unroll
    for (int j = 0; j < R; ++j) {
      key[j] = mix64(i + j * nthreads) % nkeys;
      w[j] = ld_keep_u64(dir + (key[j] >> 5));
    }
    int32_t v[R];
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const uint32_t bits = (uint32_t)w[j], b = (uint32_t)(key[j] & 31);
      v[j] = (bits >> b) & 1 ? ld_keep_i32(slots + (w[j] >> 32) + __popc(bits & ((1u << b) - 1))) : 0;
    }
#pragma unroll
    for (int j = 0; j < R; ++j) acc += v[j];
  }
  if (acc == 0x7fffffff) out[0] = acc;
}

// star_mix: SB = slot width in bits (32: int32 array; 21 / 16: 3 / 4 entries per 64-bit word)
template <int SB>
__global__ void __launch_bounds__(256, 2) star_mix_kernel(const int64_t* __restrict__ fk, const int64_t* __restrict__ x,
                                                          const int64_t* __restrict__ val, const uint64_t* __restrict__ dir,
                                                          const void* __restrict__ slots, double* grp, uint64_t nrows) {
  const uint64_t nthreads = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += R * nthreads) {
    int64_t k[R], vv[R];
    uint64_t w[R];
    uint32_t live = 0;
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const uint64_t r = i + j * nthreads;
      k[j] = r < nrows ? ld_stream(fk + r) : 0;
      if (r < nrows && ld_stream(x + r) > 0) live |= 1u << j;
    }
#pragma unroll
    for (int j = 0; j < R; ++j) w[j] = (live >> j) & 1 ? ld_keep_u64(dir + (k[j] >> 5)) : 0;
#pragma unroll
    for (int j = 0; j < R; ++j) vv[j] = (live >> j) & 1 ? ld_stream(val + i + j * nthreads) : 0;
    int32_t s[R];
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const uint32_t bits = (uint32_t)w[j], b = (uint32_t)(k[j] & 31);
      s[j] = -1;
      if ((bits >> b) & 1) {
        const uint32_t pos = (uint32_t)(w[j] >> 32) + __popc(bits & ((1u << b) - 1));
        if (SB == 32) {
          s[j] = ld_keep_i32(static_cast<const int32_t*>(slots) + pos);
        } else {
          const uint32_t q = SB == 16 ? pos >> 2 : __umulhi(pos, 0x55555556u);
          const uint64_t word = ld_keep_u64(static_cast<const uint64_t*>(slots) + q);
          s[j] = (int32_t)((word >> ((pos - q * (64 / SB)) * SB)) & ((1ull << SB) - 1));
        }
      }
    }
#pragma unroll
    for (int j = 0; j < R; ++j)
      if (s[j] >= 0) atomicAdd(grp + s[j], __longlong_as_double(vv[j]));
  }
}

// slot values in [0, ngrp), in the packed layout of width SB
template <int SB>
__global__ void fill_slots(void* slots, uint64_t nentries, uint64_t ngrp) {
  const int k = 64 / SB;
  const uint64_t nwords = (nentries + k - 1) / k;
  for (uint64_t q = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; q < nwords; q += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t word = 0;
    for (int e = 0; e < k && q * k + e < nentries; ++e) word |= (mix64(q * k + e + 99) % ngrp) << (e * SB);
    static_cast<uint64_t*>(slots)[q] = word;
  }
}

__global__ void fill_i32(int32_t* t, uint64_t n) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    t[i] = (int32_t)(mix64(i + 99) & 0x3ffffff);
}
// 16 of every 32 bits set (alternating pattern, flipped on odd words): rank = 16 per earlier word
__global__ void fill_dir(uint64_t* dir, uint64_t nwords) {
  for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < nwords; w += (uint64_t)gridDim.x * blockDim.x)
    dir[w] = ((uint64_t)(16 * w) << 32) | (w & 1 ? 0xaaaaaaaaULL : 0x55555555ULL);
}
__global__ void fill_rows(int64_t* fk, int64_t* x, int64_t* val, uint64_t nrows, uint64_t nkeys) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t h = mix64(i + 7);
    fk[i] = (int64_t)(h % nkeys);
    x[i] = (h >> 40) & 1 ? 1 : -1;
    val[i] = __double_as_longlong((double)(h & 4095) / 4096.0);
  }
}

template <class F>
static float time_it(F launch, int reps = 3) {
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  launch();   // warm-up: loads the module and brings the table into L2 as far as it fits
  CK(cudaDeviceSynchronize());
  float best = 1e30f;
  for (int r = 0; r < reps; ++r) {
    CK(cudaEventRecord(a));
    launch();
    CK(cudaEventRecord(b));
    CK(cudaEventSynchronize(b));
    float ms; CK(cudaEventElapsedTime(&ms, a, b));
    if (ms < best) best = ms;
  }
  CK(cudaGetLastError());
  return best;
}

static void star_mix(int sms) {
  const uint64_t nrows = 125000000ULL, nkeys = 10000000ULL, nentries = nkeys / 2, ngrp = (1ULL << 20) - 1;
  const uint64_t nwords = nkeys / 32;
  int64_t *fk, *x, *val; uint64_t *dir, *slots; double* grp;
  CK(cudaMalloc(&fk, nrows * 8)); CK(cudaMalloc(&x, nrows * 8)); CK(cudaMalloc(&val, nrows * 8));
  CK(cudaMalloc(&dir, nwords * 8)); CK(cudaMalloc(&slots, nentries * 4)); CK(cudaMalloc(&grp, (ngrp + 1) * 8));
  CK(cudaMemset(grp, 0, (ngrp + 1) * 8));
  fill_rows<<<sms * 8, 256>>>(fk, x, val, nrows, nkeys);
  fill_dir<<<sms * 8, 256>>>(dir, nwords);
  CK(cudaDeviceSynchronize());
  const int grid = sms * 2;   // 2 CTAs of 256 threads per SM, as b2_star_agg_kernel<false> at 128 registers
  for (int rep = 0; rep < 3; ++rep) {   // the three widths alternate, so that drift hits all of them alike
    for (int sb : {32, 21, 16}) {
      float ms;
      if (sb == 32) {
        fill_slots<32><<<sms * 8, 256>>>(slots, nentries, ngrp);
        ms = time_it([&] { star_mix_kernel<32><<<grid, 256>>>(fk, x, val, dir, slots, grp, nrows); }, 5);
      } else if (sb == 21) {
        fill_slots<21><<<sms * 8, 256>>>(slots, nentries, ngrp);
        ms = time_it([&] { star_mix_kernel<21><<<grid, 256>>>(fk, x, val, dir, slots, grp, nrows); }, 5);
      } else {
        fill_slots<16><<<sms * 8, 256>>>(slots, nentries, ngrp);
        ms = time_it([&] { star_mix_kernel<16><<<grid, 256>>>(fk, x, val, dir, slots, grp, nrows); }, 5);
      }
      const int k = 64 / sb;
      const double slot_mb = (double)((nentries + k - 1) / k) * 8 / 1e6;
      printf("{\"test\": \"star_mix\", \"slot_bits\": %d, \"slot_mb\": %.1f, \"dir_mb\": %.1f, \"group_mb\": %.1f, "
             "\"rows\": %llu, \"rep\": %d, \"ms\": %.4f, \"stream_gbs_24B_per_row\": %.1f}\n",
             sb, slot_mb, nwords * 8 / 1e6, (ngrp + 1) * 8 / 1e6, (unsigned long long)nrows, rep, ms,
             nrows * 24.0 / ms / 1e6);
      fflush(stdout);
    }
  }
  CK(cudaFree(fk)); CK(cudaFree(x)); CK(cudaFree(val)); CK(cudaFree(dir)); CK(cudaFree(slots)); CK(cudaFree(grp));
}

int main(int argc, char** argv) {
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  const int sms = prop.multiProcessorCount;
  printf("{\"device\": \"%s\", \"sms\": %d, \"l2_bytes\": %d}\n", prop.name, sms, prop.l2CacheSize);
  if (argc > 1 && !strcmp(argv[1], "star")) {
    star_mix(sms);
    return 0;
  }
  const int grid = sms * 8;   // 8 CTAs of 256 threads per SM: full occupancy, the most reads in flight
  const uint64_t sizes_mb[] = {8, 16, 24, 32, 40, 48, 64};
  const uint64_t max_entries = 64ULL << 18;                // 64 MB of int32
  const uint64_t nreads = 256ULL << 20;
  const uint64_t nrows = 125000000ULL;                     // one C4 fact partition
  const uint64_t ngrp = 1ULL << 20;                        // 8 MB of f64
  int32_t* t; uint64_t* dir; int* out; double* grp; int64_t *fk, *x, *val;
  CK(cudaMalloc(&t, max_entries * 4));
  CK(cudaMalloc(&dir, max_entries / 16 * 8));
  CK(cudaMalloc(&out, 64));
  CK(cudaMalloc(&grp, ngrp * 8));
  CK(cudaMalloc(&fk, nrows * 8)); CK(cudaMalloc(&x, nrows * 8)); CK(cudaMalloc(&val, nrows * 8));
  CK(cudaMemset(grp, 0, ngrp * 8));
  fill_i32<<<sms * 8, 256>>>(t, max_entries);
  fill_dir<<<sms * 8, 256>>>(dir, max_entries / 16);
  CK(cudaDeviceSynchronize());
  for (uint64_t mb : sizes_mb) {
    const uint64_t n = mb << 18;
    const float a_ms = time_it([&] { alone_kernel<<<grid, 256>>>(t, n, nreads, out); });
    printf("{\"test\": \"gather_alone\", \"table_mb\": %llu, \"reads\": %llu, \"ms\": %.4f, \"g_reads_per_s\": %.2f}\n",
           (unsigned long long)mb, (unsigned long long)nreads, a_ms, nreads / a_ms / 1e6);
    fflush(stdout);
    fill_rows<<<sms * 8, 256>>>(fk, x, val, nrows, n);
    CK(cudaDeviceSynchronize());
    const float m_ms = time_it([&] { mix_kernel<<<grid, 256>>>(fk, x, val, t, grp, ngrp, nrows); });
    const double lookups = nrows / 2.0;
    printf("{\"test\": \"gather_mix_c4\", \"table_mb\": %llu, \"rows\": %llu, \"ms\": %.4f, \"g_reads_per_s\": %.2f, "
           "\"stream_gbs_24B_per_row\": %.1f}\n",
           (unsigned long long)mb, (unsigned long long)nrows, m_ms, lookups / m_ms / 1e6, nrows * 24.0 / m_ms / 1e6);
    fflush(stdout);
    const float p_ms = time_it([&] { pair_kernel<<<grid, 256>>>(dir, t, 2 * n, nreads, out); });
    printf("{\"test\": \"gather_pair\", \"table_mb\": %llu, \"dir_mb\": %.1f, \"keys\": %llu, \"ms\": %.4f, "
           "\"g_keys_per_s\": %.2f}\n",
           (unsigned long long)mb, mb / 8.0, (unsigned long long)nreads, p_ms, nreads / p_ms / 1e6);
    fflush(stdout);
  }
  // the same C4 mix with no table read at all: the streaming + atomic floor
  {
    fill_rows<<<sms * 8, 256>>>(fk, x, val, nrows, 1ULL << 20);
    CK(cudaDeviceSynchronize());
    const float m_ms = time_it([&] { mix_kernel<<<grid, 256>>>(fk, x, val, t, grp, ngrp, nrows); });
    printf("{\"test\": \"gather_mix_c4\", \"table_mb\": 4, \"note\": \"1M-entry table: reads hit L2\", \"rows\": %llu, "
           "\"ms\": %.4f, \"stream_gbs_24B_per_row\": %.1f}\n",
           (unsigned long long)nrows, m_ms, nrows * 24.0 / m_ms / 1e6);
  }
  return 0;
}
