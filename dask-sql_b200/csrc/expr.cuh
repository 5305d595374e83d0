// expr.cuh — per-row postfix expression interpreter (b2_expr_eval) and column statistics.
// One pass per expression TREE (the reference does one pandas pass per operator NODE,
// physical/rex/core/call.py:1158-1216).  The program is warp-uniform (kernel parameter
// space), so the interpreter loop never diverges; the value stack lives in local memory.
#pragma once
#include "common.cuh"
#include "rand.cuh"

#define B2_STACK 16

struct b2_cols_arg {
  b2_col_t c[B2_MAX_COLS];
};

// ---- calendar arithmetic (proleptic Gregorian, days since 1970-01-01) ---------------------
// Howard Hinnant's civil_from_days / days_from_civil: int64 arithmetic with constant divisors only,
// exact for every day an int64 tick count of any unit can reach (and the whole date32 range).
__device__ __forceinline__ int64_t b2_floordiv(int64_t a, int64_t b) {  // b > 0
  const int64_t q = a / b;
  return q - (q * b > a);
}

__device__ __forceinline__ void b2_civil_from_days(int64_t z, int64_t& y, int& m, int& d) {
  z += 719468;
  const int64_t era = b2_floordiv(z, 146097);
  const int64_t doe = z - era * 146097;                                       // [0, 146096]
  const int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;  // [0, 399]
  const int64_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);                // [0, 365], from March 1
  const int64_t mp = (5 * doy + 2) / 153;                                     // [0, 11]
  d = (int)(doy - (153 * mp + 2) / 5 + 1);
  m = (int)(mp < 10 ? mp + 3 : mp - 9);
  y = yoe + era * 400 + (m <= 2);
}

__device__ __forceinline__ int64_t b2_days_from_civil(int64_t y, int m, int d) {
  y -= m <= 2;
  const int64_t era = b2_floordiv(y, 400);
  const int64_t yoe = y - era * 400;
  const int64_t doy = (153 * (m > 2 ? m - 3 : m + 9) + 2) / 5 + d - 1;
  const int64_t doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
  return era * 146097 + doe - 719468;
}

// Kept out of line: the interpreter loop is walked by every instruction of every program, and the
// calendar code would otherwise add its registers to all of them.
__device__ __noinline__ int64_t b2_datepart(int64_t x, int field, int64_t tps) {
  const int64_t tpd = tps ? tps * 86400 : 1;
  const int64_t day = b2_floordiv(x, tpd);
  const int64_t tod = x - day * tpd;
  if (field == B2_DP_DAYS) return day;
  if (field == B2_DP_DOW) return b2_floordiv(day + 4, 7) * -7 + day + 4;   // 1970-01-01 was a Thursday
  if (field >= B2_DP_HOUR) {
    if (!tps) return 0;
    if (field == B2_DP_HOUR) return tod / (tps * 3600);
    if (field == B2_DP_MINUTE) return tod / (tps * 60) % 60;
    if (field == B2_DP_SECOND) return tod / tps % 60;
    const int64_t sub = tod % tps;
    return field == B2_DP_MILLISECOND ? sub * 1000 / tps : sub * 1000000 / tps;
  }
  int64_t y; int m, d;
  if (field == B2_DP_ISOWEEK) {
    // the ISO week belongs to the year of its Thursday
    const int64_t th = day - (b2_floordiv(day + 3, 7) * -7 + day + 3) + 3;   // Mon = 0 .. Sun = 6
    b2_civil_from_days(th, y, m, d);
    return (th - b2_days_from_civil(y, 1, 1)) / 7 + 1;
  }
  b2_civil_from_days(day, y, m, d);
  if (field == B2_DP_YEAR) return y;
  if (field == B2_DP_QUARTER) return (m - 1) / 3 + 1;
  if (field == B2_DP_MONTH) return m;
  if (field == B2_DP_DAY) return d;
  return day - b2_days_from_civil(y, 1, 1) + 1;                              // B2_DP_DOY
}

__device__ __noinline__ int64_t b2_addmonths(int64_t x, int64_t n, int64_t tps, int to_last) {
  const int64_t tpd = tps ? tps * 86400 : 1;
  const int64_t day = b2_floordiv(x, tpd);
  const int64_t tod = x - day * tpd;
  int64_t y; int m, d;
  b2_civil_from_days(day, y, m, d);
  const int64_t total = (int64_t)((uint64_t)(y * 12 + (m - 1)) + (uint64_t)n);
  const int64_t y2 = b2_floordiv(total, 12);
  const int m2 = (int)(total - y2 * 12) + 1;
  const int64_t first = b2_days_from_civil(y2, m2, 1);
  const int last = (int)(b2_days_from_civil(y2 + (m2 == 12), m2 == 12 ? 1 : m2 + 1, 1) - first);
  const int d2 = to_last ? last : (d < last ? d : last);
  return (int64_t)((uint64_t)(first + d2 - 1) * (uint64_t)tpd + (uint64_t)tod);
}

// ---- numeric SQL functions (B2_OP_MATH_F / MATH2_F / POW_I) ---------------------------------
// Out of line for the same reason as the calendar code.  The slow path of sin / cos / tan (argument
// reduction of huge x) uses a 40 B local array; ptxas counts it in the kernel's frame, but only that path
// touches it (DESIGN.md section 4).
__device__ __noinline__ int64_t b2_math_f(int64_t bits, int fn, double f, int64_t div_first) {
  const double x = __longlong_as_double(bits);
  double r;
  switch (fn) {
    case B2_FN_CEIL:    r = ceil(x); break;
    case B2_FN_FLOOR:   r = floor(x); break;
    case B2_FN_TRUNC:   r = trunc(x); break;
    case B2_FN_ROUND:   r = div_first ? rint(x / f) * f : rint(x * f) / f; break;
    case B2_FN_SIGN:    r = x > 0.0 ? 1.0 : x < 0.0 ? -1.0 : x == 0.0 ? 0.0 : x; break;
    case B2_FN_DEGREES: r = x * (180.0 / 3.141592653589793238462643383279502884); break;
    case B2_FN_RADIANS: r = x * (3.141592653589793238462643383279502884 / 180.0); break;
    case B2_FN_EXP:     r = exp(x); break;
    case B2_FN_LN:      r = log(x); break;
    case B2_FN_LOG10:   r = log10(x); break;
    case B2_FN_CBRT:    r = cbrt(x); break;
    case B2_FN_SIN:     r = sin(x); break;
    case B2_FN_COS:     r = cos(x); break;
    case B2_FN_TAN:     r = tan(x); break;
    case B2_FN_COT:     r = 1.0 / tan(x); break;
    case B2_FN_ASIN:    r = asin(x); break;
    case B2_FN_ACOS:    r = acos(x); break;
    default:            r = atan(x); break;   // B2_FN_ATAN (b2_expr_eval rejects other ids)
  }
  return __double_as_longlong(r);
}

__device__ __noinline__ int64_t b2_math2_f(int64_t xbits, int64_t ybits, int fn) {
  const double x = __longlong_as_double(xbits), y = __longlong_as_double(ybits);
  double r;
  if (fn == B2_FN_ATAN2) r = atan2(x, y);
  else if (fn == B2_FN_POW) r = pow(x, y);
  else {                                       // B2_FN_MOD: NumPy's npy_divmod remainder
    r = fmod(x, y);
    if (y != 0.0) {
      if (r != 0.0) { if ((y < 0.0) != (r < 0.0)) r += y; }
      else r = copysign(0.0, y);
    }
  }
  return __double_as_longlong(r);
}

__device__ __noinline__ int64_t b2_pow_i(int64_t x, int64_t y) {   // y >= 0; wraps like np.power
  uint64_t base = (uint64_t)x, r = 1;
  for (uint64_t e = (uint64_t)y; e; e >>= 1) {
    if (e & 1) r *= base;
    base *= base;
  }
  return (int64_t)r;
}

__global__ void __launch_bounds__(B2_BLOCK)
b2_expr_kernel(const __grid_constant__ b2_prog_t prog, const __grid_constant__ b2_cols_arg cols,
               int64_t n, int64_t row_base, void* __restrict__ out_data, uint32_t* __restrict__ out_valid) {
  const int64_t n32 = (n + 31) & ~(int64_t)31;
  for (int64_t row = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; row < n32;
       row += (int64_t)gridDim.x * B2_BLOCK) {
    const bool active = row < n;
    int64_t sv[B2_STACK];
    bool sn[B2_STACK];
    int sp = 0;
    if (active) {
      for (int pc = 0; pc < prog.n; ++pc) {
        const b2_instr_t ins = prog.code[pc];
        const int op = ins.op;
        if (op == B2_OP_LOAD) {
          const b2_col_t& c = cols.c[ins.a];
          int64_t raw = c.dtype == B2_U8 ? (int64_t) reinterpret_cast<const uint8_t*>(c.data)[row]
                                         : reinterpret_cast<const int64_t*>(c.data)[row];
          sv[sp] = raw;
          sn[sp] = c.valid ? !b2_bit(c.valid, row) : false;
          ++sp;
        } else if (op == B2_OP_CONST_I) {
          sv[sp] = ins.imm_i; sn[sp] = false; ++sp;
        } else if (op == B2_OP_CONST_F) {
          sv[sp] = __double_as_longlong(ins.imm_f); sn[sp] = false; ++sp;
        } else if (op == B2_OP_CONST_NULL) {
          sv[sp] = 0; sn[sp] = true; ++sp;
        } else if (op == B2_OP_I2F) {
          sv[sp - 1] = __double_as_longlong((double)sv[sp - 1]);
        } else if (op == B2_OP_F2I) {
          double d = __longlong_as_double(sv[sp - 1]);
          if (d != d) { sn[sp - 1] = true; sv[sp - 1] = 0; }
          else sv[sp - 1] = (int64_t)d;
        } else if (op == B2_OP_NEG_I) {
          sv[sp - 1] = (int64_t)(0ULL - (uint64_t)sv[sp - 1]);
        } else if (op == B2_OP_ABS_I) {
          int64_t v = sv[sp - 1]; sv[sp - 1] = v < 0 ? (int64_t)(0ULL - (uint64_t)v) : v;
        } else if (op == B2_OP_NEG_F) {
          sv[sp - 1] = __double_as_longlong(-__longlong_as_double(sv[sp - 1]));
        } else if (op == B2_OP_SQRT_F) {
          sv[sp - 1] = __double_as_longlong(sqrt(__longlong_as_double(sv[sp - 1])));
        } else if (op == B2_OP_ABS_F) {
          sv[sp - 1] = __double_as_longlong(fabs(__longlong_as_double(sv[sp - 1])));
        } else if (op == B2_OP_ORD2F) {
          sv[sp - 1] = b2_ordered_from_bits(sv[sp - 1]);
        } else if (op == B2_OP_NOT) {
          sv[sp - 1] = sv[sp - 1] == 0;
        } else if (op == B2_OP_ISNULL_I) {
          sv[sp - 1] = sn[sp - 1]; sn[sp - 1] = false;
        } else if (op == B2_OP_ISNULL_F) {
          double d = __longlong_as_double(sv[sp - 1]);
          sv[sp - 1] = sn[sp - 1] || d != d; sn[sp - 1] = false;
        } else if (op == B2_OP_CASE) {
          // stack: cond, then, else
          const int64_t ev = sv[sp - 1]; const bool en = sn[sp - 1];
          const int64_t tv = sv[sp - 2]; const bool tn = sn[sp - 2];
          const bool take = !sn[sp - 3] && sv[sp - 3] != 0;
          sp -= 2;
          sv[sp - 1] = take ? tv : ev;
          sn[sp - 1] = take ? tn : en;
        } else if (op == B2_OP_FILLNA) {
          // stack: x, fill
          if (sn[sp - 2]) { sv[sp - 2] = sv[sp - 1]; sn[sp - 2] = sn[sp - 1]; }
          --sp;
        } else if (op == B2_OP_DATEPART) {
          sv[sp - 1] = b2_datepart(sv[sp - 1], ins.a, ins.imm_i);
        } else if (op == B2_OP_MAP) {
          const b2_col_t& c = cols.c[ins.a];
          const int64_t x = sv[sp - 1];
          const bool hit = !sn[sp - 1] && x >= 0 && x < ins.imm_i && (!c.valid || b2_bit(c.valid, x));
          sv[sp - 1] = !hit ? 0 : c.dtype == B2_U8 ? (int64_t) reinterpret_cast<const uint8_t*>(c.data)[x]
                                                   : reinterpret_cast<const int64_t*>(c.data)[x];
          sn[sp - 1] = !hit;
        } else if (op == B2_OP_MATH_F) {
          sv[sp - 1] = b2_math_f(sv[sp - 1], ins.a, ins.imm_f, ins.imm_i);
        } else if (op == B2_OP_RAND_F) {
          const uint64_t u = b2_rand_u64(row_base + row, ins.imm_i, ins.a);
          sv[sp] = __double_as_longlong((double)(u >> 11) * 0x1.0p-53); sn[sp] = false; ++sp;
        } else if (op == B2_OP_RAND_I) {
          // h > 0 (the planner's rule); a NULL or non-positive h gives NULL
          const int64_t h = sv[sp - 1];
          const bool ok = !sn[sp - 1] && h > 0;
          sv[sp - 1] = ok ? (int64_t)__umul64hi(b2_rand_u64(row_base + row, ins.imm_i, ins.a), (uint64_t)h) : 0;
          sn[sp - 1] = !ok;
        } else if (op == B2_OP_ADDMONTHS) {
          // stack: x, n
          sv[sp - 2] = b2_addmonths(sv[sp - 2], sv[sp - 1], ins.imm_i, ins.a);
          sn[sp - 2] = sn[sp - 2] || sn[sp - 1];
          --sp;
        } else {
          // binary operators: pops b then a
          const int64_t b = sv[sp - 1]; const bool bn = sn[sp - 1];
          const int64_t a = sv[sp - 2]; const bool an = sn[sp - 2];
          --sp;
          int64_t r = 0; bool rn = an || bn;
          if (op == B2_OP_AND) {  // Kleene: False wins over NULL
            const bool af = !an && a == 0, bf = !bn && b == 0;
            rn = (an || bn) && !(af || bf);
            r = (!an && a != 0) && (!bn && b != 0);
          } else if (op == B2_OP_OR) {  // Kleene: True wins over NULL
            const bool at = !an && a != 0, bt = !bn && b != 0;
            rn = (an || bn) && !(at || bt);
            r = at || bt;
          } else if (op >= B2_OP_EQ_F && op <= B2_OP_EQ_F + 5) {
            r = b2_cmp_f(op - B2_OP_EQ_F, __longlong_as_double(a), __longlong_as_double(b));
          } else if (op >= B2_OP_EQ_I && op <= B2_OP_EQ_I + 5) {
            r = b2_cmp_i(op - B2_OP_EQ_I, a, b);
          } else if (op == B2_OP_ADD_I) r = (int64_t)((uint64_t)a + (uint64_t)b);
          else if (op == B2_OP_SUB_I) r = (int64_t)((uint64_t)a - (uint64_t)b);
          else if (op == B2_OP_MUL_I) r = (int64_t)((uint64_t)a * (uint64_t)b);
          else if (op == B2_OP_DIV_I) {
            if (b == 0) rn = true;
            else if (b == -1) r = (int64_t)(0ULL - (uint64_t)a);
            else r = a / b;  // C++ '/' truncates toward zero = SQL semantics
          } else if (op == B2_OP_MOD_I) {  // floored, like NumPy / Python: the result takes b's sign
            if (b == 0) rn = true;
            else if (b == -1) r = 0;
            else {
              r = a % b;
              if (r != 0 && (r ^ b) < 0) r += b;
            }
          } else if (op == B2_OP_ADD_F) r = __double_as_longlong(__longlong_as_double(a) + __longlong_as_double(b));
          else if (op == B2_OP_SUB_F) r = __double_as_longlong(__longlong_as_double(a) - __longlong_as_double(b));
          else if (op == B2_OP_MUL_F) r = __double_as_longlong(__longlong_as_double(a) * __longlong_as_double(b));
          else if (op == B2_OP_DIV_F) r = __double_as_longlong(__longlong_as_double(a) / __longlong_as_double(b));
          else if (op == B2_OP_MATH2_F) r = b2_math2_f(a, b, ins.a);
          else if (op == B2_OP_POW_I) {  // np.power raises on a negative exponent: NULL here
            if (b < 0) rn = true;
            else r = b2_pow_i(a, b);
          }
          sv[sp - 1] = r;
          sn[sp - 1] = rn;
        }
      }
    }
    const bool isnull = active ? sn[0] : true;
    const int64_t v = (active && !isnull) ? sv[0] : 0;
    if (active) {
      if (prog.out_dtype == B2_U8) reinterpret_cast<uint8_t*>(out_data)[row] = (uint8_t)(v != 0);
      else reinterpret_cast<int64_t*>(out_data)[row] = v;
    }
    if (out_valid) {
      const uint32_t w = __ballot_sync(FULL_MASK, active && !isnull);
      if ((threadIdx.x & 31) == 0) out_valid[row >> 5] = w;
    }
  }
}

// ---- column statistics ------------------------------------------------------------------
// out: {min(ordered image), max(ordered image), nulls, nans, repeating rows of the sample, rows sampled}
__global__ void b2_stats_init_kernel(int64_t* out) {
  out[0] = LLONG_MAX; out[1] = LLONG_MIN; out[2] = 0; out[3] = 0; out[4] = 0; out[5] = 0;
}
__global__ void __launch_bounds__(B2_BLOCK)
b2_stats_kernel(const __grid_constant__ b2_col_t col, int64_t n, int64_t* __restrict__ out) {
  long long mn = LLONG_MAX, mx = LLONG_MIN;
  unsigned long long nulls = 0, nans = 0;
  {
    // repeat sample: of the 32 consecutive rows each warp meets first (spread over the whole column by
    // the grid stride), how many share their value with another one?  Decides whether a GROUP BY on
    // this column pre-aggregates per warp (out[4] = such rows, out[5] = rows sampled).
    const int64_t row = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x;
    bool ok = row < n && !(col.valid && !b2_bit(col.valid, row));
    int64_t raw = ok ? b2_load_raw(col, row) : 0;
    if (ok && col.dtype == B2_F64) { const double d = __longlong_as_double(raw); ok = d == d; }
    const uint32_t act = __ballot_sync(FULL_MASK, ok);
    uint32_t m = 0;
    if (ok) m = __match_any_sync(act, raw);
    const uint32_t rep = __ballot_sync(FULL_MASK, ok && __popc(m) > 1);
    if ((threadIdx.x & 31) == 0 && act) {
      atomicAdd(reinterpret_cast<unsigned long long*>(out + 4), (unsigned long long)__popc(rep));
      atomicAdd(reinterpret_cast<unsigned long long*>(out + 5), (unsigned long long)__popc(act));
    }
  }
  for (int64_t row = (int64_t)blockIdx.x * B2_BLOCK + threadIdx.x; row < n;
       row += (int64_t)gridDim.x * B2_BLOCK) {
    if (col.valid && !b2_bit(col.valid, row)) { ++nulls; continue; }
    int64_t raw = b2_load_raw(col, row);
    if (col.dtype == B2_F64) {
      double d = __longlong_as_double(raw);
      if (d != d) { ++nans; continue; }
      raw = b2_ordered_from_bits(raw);
    }
    mn = raw < mn ? raw : mn;
    mx = raw > mx ? raw : mx;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    long long omn = __shfl_xor_sync(FULL_MASK, mn, o), omx = __shfl_xor_sync(FULL_MASK, mx, o);
    mn = omn < mn ? omn : mn;
    mx = omx > mx ? omx : mx;
    nulls += __shfl_xor_sync(FULL_MASK, nulls, o);
    nans += __shfl_xor_sync(FULL_MASK, nans, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (mn != LLONG_MAX) atomicMin(reinterpret_cast<long long*>(out), mn);
    if (mx != LLONG_MIN) atomicMax(reinterpret_cast<long long*>(out + 1), mx);
    if (nulls) atomicAdd(reinterpret_cast<unsigned long long*>(out + 2), nulls);
    if (nans) atomicAdd(reinterpret_cast<unsigned long long*>(out + 3), nans);
  }
}
__global__ void b2_stats_fini_kernel(int64_t* out, int is_f64) {
  if (is_f64) {
    if (out[0] != LLONG_MAX || out[1] != LLONG_MIN) {
      out[0] = b2_ordered_from_bits(out[0]);
      out[1] = b2_ordered_from_bits(out[1]);
    }
  }
}

extern "C" {

int64_t b2_stats_ws_bytes(void) { return 256; }

int32_t b2_col_stats(const b2_col_t* col, int64_t n, int64_t* d_out, void* ws, void* stream) {
  (void)ws;
  B2_REQUIRE(col && d_out, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  b2_stats_init_kernel<<<1, 1, 0, st>>>(d_out);
  if (n > 0) {
    int grid = b2_wave_grid(b2_stats_kernel, B2_BLOCK, (n + B2_BLOCK - 1) / B2_BLOCK);
    b2_stats_kernel<<<grid, B2_BLOCK, 0, st>>>(*col, n, d_out);
  }
  b2_stats_fini_kernel<<<1, 1, 0, st>>>(d_out, col->dtype == B2_F64);
  B2_CHECK_LAUNCH("b2_stats_kernel");
  return B2_OK;
}

int32_t b2_expr_eval_rows(const b2_prog_t* prog, const b2_col_t* cols, int32_t ncols, int64_t n, int64_t row_base,
                          void* out_data, uint32_t* out_valid, void* stream) {
  B2_REQUIRE(prog && out_data, "null argument");
  B2_REQUIRE(row_base >= 0 && (n <= 0 || n <= INT64_MAX - row_base), "row_base must be >= 0 and row_base + n fit");
  B2_REQUIRE(ncols >= 0 && ncols <= B2_MAX_COLS, "too many columns");
  B2_REQUIRE(prog->n > 0 && prog->n <= B2_MAX_PROG, "bad program length");
  // static stack-depth check so the kernel cannot run off its local stack
  int sp = 0;
  for (int i = 0; i < prog->n; ++i) {
    int op = prog->code[i].op;
    if (op == B2_OP_LOAD) {
      B2_REQUIRE(prog->code[i].a >= 0 && prog->code[i].a < ncols, "LOAD of unknown column");
      ++sp;
    } else if (op == B2_OP_CONST_I || op == B2_OP_CONST_F || op == B2_OP_CONST_NULL) ++sp;
    else if (op == B2_OP_RAND_F || op == B2_OP_RAND_I) {
      B2_REQUIRE(prog->code[i].a >= 0, "RAND: the call site a must be >= 0");
      if (op == B2_OP_RAND_F) ++sp;
      else B2_REQUIRE(sp >= 1, "stack underflow");
    }
    else if (op == B2_OP_I2F || op == B2_OP_F2I || op == B2_OP_NEG_I || op == B2_OP_ABS_I ||
             op == B2_OP_NEG_F || op == B2_OP_ABS_F || op == B2_OP_SQRT_F || op == B2_OP_NOT || op == B2_OP_ISNULL_I ||
             op == B2_OP_ISNULL_F || op == B2_OP_ORD2F) { B2_REQUIRE(sp >= 1, "stack underflow"); }
    else if (op == B2_OP_DATEPART || op == B2_OP_ADDMONTHS) {
      const int64_t tps = prog->code[i].imm_i;
      B2_REQUIRE(tps == 0 || tps == 1 || tps == 1000 || tps == 1000000 || tps == 1000000000,
                 "calendar opcode: ticks per second must be 0, 1, 10^3, 10^6 or 10^9");
      if (op == B2_OP_DATEPART) {
        B2_REQUIRE(prog->code[i].a >= 0 && prog->code[i].a < B2_DP_NFIELDS, "DATEPART: unknown field");
        B2_REQUIRE(sp >= 1, "stack underflow");
      } else {
        B2_REQUIRE(prog->code[i].a == 0 || prog->code[i].a == 1, "ADDMONTHS: a must be 0 or 1");
        B2_REQUIRE(sp >= 2, "stack underflow");
        sp -= 1;
      }
    }
    else if (op == B2_OP_MAP) {
      const int a = prog->code[i].a;
      B2_REQUIRE(a >= 0 && a < ncols, "MAP of unknown column");
      B2_REQUIRE(cols[a].dtype == B2_I64 || cols[a].dtype == B2_U8, "MAP table must be B2_I64 or B2_U8");
      B2_REQUIRE(prog->code[i].imm_i >= 0, "MAP table length must be >= 0");
      B2_REQUIRE(sp >= 1, "stack underflow");
    }
    else if (op == B2_OP_MATH_F) {
      const int a = prog->code[i].a;
      B2_REQUIRE(a >= 0 && a < B2_FN_ATAN2, "MATH_F: unknown function");
      B2_REQUIRE(a != B2_FN_ROUND || prog->code[i].imm_i == 0 || prog->code[i].imm_i == 1,
                 "MATH_F: ROUND's imm_i must be 0 or 1");
      B2_REQUIRE(sp >= 1, "stack underflow");
    }
    else if (op == B2_OP_CASE) { B2_REQUIRE(sp >= 3, "stack underflow"); sp -= 2; }
    else {
      if (op == B2_OP_MATH2_F)
        B2_REQUIRE(prog->code[i].a >= B2_FN_ATAN2 && prog->code[i].a < B2_FN_NFUNCS, "MATH2_F: unknown function");
      B2_REQUIRE(sp >= 2, "stack underflow");
      sp -= 1;
    }
    B2_REQUIRE(sp <= B2_STACK, "expression too deep");
  }
  B2_REQUIRE(sp == 1, "program must leave exactly one value");
  if (n <= 0) return B2_OK;
  b2_cols_arg ca;
  memset(&ca, 0, sizeof(ca));
  for (int i = 0; i < ncols; ++i) ca.c[i] = cols[i];
  int grid = b2_wave_grid(b2_expr_kernel, B2_BLOCK, (n + B2_BLOCK - 1) / B2_BLOCK);
  b2_expr_kernel<<<grid, B2_BLOCK, 0, (cudaStream_t)stream>>>(*prog, ca, n, row_base, out_data, out_valid);
  B2_CHECK_LAUNCH("b2_expr_kernel");
  return B2_OK;
}

int32_t b2_expr_eval(const b2_prog_t* prog, const b2_col_t* cols, int32_t ncols, int64_t n,
                     void* out_data, uint32_t* out_valid, void* stream) {
  return b2_expr_eval_rows(prog, cols, ncols, n, 0, out_data, out_valid, stream);
}

}  // extern "C"
