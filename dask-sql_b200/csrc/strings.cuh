// strings.cuh — per-dictionary-entry work of VARCHAR columns (b2_str_like, b2_str_lower_bound).
// A VARCHAR column is int64 codes into a sorted dictionary (offsets + UTF-8 chars); row-level work
// runs on the codes with the ordinary kernels.  These two kernels run once per DICTIONARY ENTRY and
// produce a table that b2_expr_eval's B2_OP_MAP then looks up per row.
#pragma once
#include "common.cuh"

// bytes of the UTF-8 sequence introduced by lead byte b (a stray continuation byte counts as one)
__device__ __forceinline__ int b2_utf8_len(uint8_t b) {
  return b < 0xC0 ? 1 : b < 0xE0 ? 2 : b < 0xF0 ? 3 : 4;
}

__device__ __forceinline__ uint8_t b2_fold_ascii(uint8_t c, bool fold) {
  return (fold && c >= 'A' && c <= 'Z') ? (uint8_t)(c + 32) : c;
}

// code point of the sequence at p[0..len) (no validation: the value is only compared with `escape`)
__device__ __forceinline__ uint32_t b2_utf8_decode(const uint8_t* p, int len) {
  if (len == 1) return p[0];
  uint32_t cp = p[0] & (0x7F >> len);
  for (int i = 1; i < len; ++i) cp = (cp << 6) | (p[i] & 0x3F);
  return cp;
}

enum { B2_LIKE_LIT = 0, B2_LIKE_ANY = 1, B2_LIKE_ONE = 2 };

// the pattern token at pat[p]: kind, literal bytes [*lo, *lo + *len), and the position after it
__device__ __forceinline__ int b2_like_token(const uint8_t* pat, int64_t plen, int64_t p, uint32_t escape,
                                             int64_t* lo, int* len, int64_t* next) {
  int l = b2_utf8_len(pat[p]);
  if (p + l > plen) l = (int)(plen - p);
  if (escape != 0xFFFFFFFFu && b2_utf8_decode(pat + p, l) == escape && p + l < plen) {
    const int64_t q = p + l;                 // the escaped code point is a literal, whatever it is
    int m = b2_utf8_len(pat[q]);
    if (q + m > plen) m = (int)(plen - q);
    *lo = q; *len = m; *next = q + m;
    return B2_LIKE_LIT;
  }
  *lo = p; *len = l; *next = p + l;
  if (l == 1 && pat[p] == '%') return B2_LIKE_ANY;
  if (l == 1 && pat[p] == '_') return B2_LIKE_ONE;
  return B2_LIKE_LIT;
}

// One thread per dictionary entry.  Greedy matcher that backtracks only to the last '%': linear in
// the entry length for patterns without '%', O(len x pattern) in the worst case.
__global__ void __launch_bounds__(B2_BLOCK)
b2_str_like_kernel(const int64_t* __restrict__ offsets, const uint8_t* __restrict__ chars, int64_t ndict,
                   const uint8_t* __restrict__ pat, int64_t plen, uint32_t escape, int32_t fold,
                   uint8_t* __restrict__ out) {
  for (int64_t e = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; e < ndict; e += (int64_t)gridDim.x * B2_BLOCK) {
    const int64_t s0 = offsets[e];
    const uint8_t* str = chars + s0;
    const int64_t slen = offsets[e + 1] - s0;
    int64_t s = 0, p = 0, star_p = -1, star_s = 0;
    bool ok = true;
    while (s < slen) {
      if (p < plen) {
        int64_t lo, next;
        int len;
        const int kind = b2_like_token(pat, plen, p, escape, &lo, &len, &next);
        if (kind == B2_LIKE_ANY) {
          star_p = next; star_s = s; p = next;
          continue;
        }
        if (kind == B2_LIKE_ONE) {
          s += b2_utf8_len(str[s]);
          if (s > slen) s = slen;
          p = next;
          continue;
        }
        if (s + len <= slen) {
          bool eq = true;
          for (int i = 0; i < len; ++i)
            eq = eq && b2_fold_ascii(str[s + i], fold) == b2_fold_ascii(pat[lo + i], fold);
          if (eq) { s += len; p = next; continue; }
        }
      }
      if (star_p < 0) { ok = false; break; }
      star_s += b2_utf8_len(str[star_s]);   // let the last '%' swallow one more code point
      if (star_s > slen) star_s = slen;
      s = star_s; p = star_p;
    }
    while (ok && p < plen) {              // the entry is used up: only '%' may remain
      int64_t lo, next;
      int len;
      if (b2_like_token(pat, plen, p, escape, &lo, &len, &next) != B2_LIKE_ANY) ok = false;
      p = next;
    }
    out[e] = ok;
  }
}

// bytes a[0..la) <=> b[0..lb): <0, 0, >0 (unsigned byte order = code-point order for UTF-8)
__device__ __forceinline__ int b2_bytes_cmp(const uint8_t* a, int64_t la, const uint8_t* b, int64_t lb) {
  const int64_t m = la < lb ? la : lb;
  for (int64_t i = 0; i < m; ++i)
    if (a[i] != b[i]) return (int)a[i] - (int)b[i];
  return la < lb ? -1 : (la > lb ? 1 : 0);
}

__global__ void __launch_bounds__(B2_BLOCK)
b2_str_lower_bound_kernel(const int64_t* __restrict__ a_off, const uint8_t* __restrict__ a_chars, int64_t na,
                          const int64_t* __restrict__ b_off, const uint8_t* __restrict__ b_chars, int64_t nb,
                          int32_t mode, int64_t* __restrict__ out, uint32_t* __restrict__ out_valid) {
  const int64_t n32 = (nb + 31) & ~(int64_t)31;
  for (int64_t i = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; i < n32; i += (int64_t)gridDim.x * B2_BLOCK) {
    bool valid = false;
    if (i < nb) {
      const uint8_t* key = b_chars + b_off[i];
      const int64_t klen = b_off[i + 1] - b_off[i];
      int64_t lo = 0, hi = na;              // first A entry >= key
      while (lo < hi) {
        const int64_t mid = lo + ((hi - lo) >> 1);
        const int64_t m0 = a_off[mid];
        if (b2_bytes_cmp(a_chars + m0, a_off[mid + 1] - m0, key, klen) < 0) lo = mid + 1;
        else hi = mid;
      }
      const bool found = lo < na && b2_bytes_cmp(a_chars + a_off[lo], a_off[lo + 1] - a_off[lo], key, klen) == 0;
      if (mode == B2_STR_LB_MATCH) {
        out[i] = found ? lo : 0;
        valid = found;
      } else {
        out[i] = 2 * lo - (found ? 0 : 1);
        valid = true;
      }
    }
    if (out_valid) {
      const uint32_t w = __ballot_sync(FULL_MASK, valid);
      if ((threadIdx.x & 31) == 0) out_valid[i >> 5] = w;
    }
  }
}

extern "C" {

int32_t b2_str_like(const int64_t* offsets, const uint8_t* chars, int64_t ndict, const uint8_t* pattern,
                    int64_t plen, uint32_t escape, int32_t flags, uint8_t* out, void* stream) {
  B2_REQUIRE(ndict >= 0 && plen >= 0, "negative size");
  B2_REQUIRE((flags & ~B2_STR_ILIKE) == 0, "unknown flag");
  if (ndict == 0) return B2_OK;
  B2_REQUIRE(offsets && out, "null argument");
  B2_REQUIRE(plen == 0 || pattern, "null pattern");
  const int grid = b2_wave_grid(b2_str_like_kernel, B2_BLOCK, (ndict + B2_BLOCK - 1) / B2_BLOCK);
  b2_str_like_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(offsets, chars, ndict, pattern, plen, escape,
                                                                  (flags & B2_STR_ILIKE) != 0, out);
  B2_CHECK_LAUNCH("b2_str_like_kernel");
  return B2_OK;
}

int32_t b2_str_lower_bound(const int64_t* a_offsets, const uint8_t* a_chars, int64_t na, const int64_t* b_offsets,
                           const uint8_t* b_chars, int64_t nb, int32_t mode, int64_t* out, uint32_t* out_valid,
                           void* stream) {
  B2_REQUIRE(na >= 0 && nb >= 0, "negative size");
  B2_REQUIRE(mode == B2_STR_LB_MATCH || mode == B2_STR_LB_ORDER, "unknown mode");
  B2_REQUIRE(mode == B2_STR_LB_ORDER || out_valid || nb == 0, "B2_STR_LB_MATCH needs out_valid");
  if (nb == 0) return B2_OK;
  B2_REQUIRE(a_offsets && b_offsets && out, "null argument");
  const int grid = b2_wave_grid(b2_str_lower_bound_kernel, B2_BLOCK, (nb + B2_BLOCK - 1) / B2_BLOCK);
  b2_str_lower_bound_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(a_offsets, a_chars, na, b_offsets,
                                                                         b_chars, nb, mode, out, out_valid);
  B2_CHECK_LAUNCH("b2_str_lower_bound_kernel");
  return B2_OK;
}

}  // extern "C"
