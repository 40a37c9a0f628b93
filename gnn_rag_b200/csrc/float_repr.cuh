// Python's repr of a float64, as json.dumps writes it, on the device and on the host.
//
// repr(x) is the shortest decimal string that reads back to x and, among the strings of that length, the one closest
// to x.  With x = 0.d1 d2 .. dn * 10^decpt it is written in exponent notation (d1[.d2 .. dn]e+XX, a sign and at least
// two exponent digits) when decpt <= -4 or decpt > 16, else in fixed notation with ".0" appended when there is no
// fractional part.  -0.0 keeps its sign; json.dumps writes NaN, Infinity and -Infinity.
//
// The digits come from the Ryu algorithm (Adams, "Ryu: fast float-to-string conversion", PLDI 2018): the bounds of the
// rounding interval of x, scaled to 4 * m * 2^e2, are multiplied by a 125-bit power of five (or its inverse) that
// brings them to a few more decimal digits than any shortest result needs; digits are then removed while the interval
// still holds a number with fewer digits, and the last one is rounded to nearest, ties to even.  The power-of-five
// tables are generated at build time (gnn_rag_b200/_build.py, float_repr_table.h).  Integer arithmetic only.
//
// Everything here is __host__ __device__: the kernels of csrc/info_rows.cu call it, and a host build of the same code
// is held against Python's repr.
#pragma once
#include <stdint.h>
#include <string.h>

#include "float_repr_table.h"

#ifdef __CUDACC__
#define GR_FR_HD __host__ __device__ __forceinline__
#else
#define GR_FR_HD inline
#endif

namespace gr {
namespace fr {

// the longest repr: "-" 17 digits "." "e-308" (24 bytes); "-Infinity" is 9
constexpr int kMaxReprLen = 24;

GR_FR_HD uint64_t pow5_inv(int q, int w) {
#ifdef __CUDA_ARCH__
  return __ldg(&d_pow5_inv[q][w]);
#else
  return h_pow5_inv[q][w];
#endif
}

GR_FR_HD uint64_t pow5(int i, int w) {
#ifdef __CUDA_ARCH__
  return __ldg(&d_pow5[i][w]);
#else
  return h_pow5[i][w];
#endif
}

GR_FR_HD uint64_t umulhi(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
  return __umul64hi(a, b);
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

// floor(m * mul / 2^j) for m < 2^55, mul = mul_hi * 2^64 + mul_lo (125 bits) and 64 < j < 128 (the table's scaling
// keeps the shift there)
GR_FR_HD uint64_t mul_shift(uint64_t m, uint64_t mul_lo, uint64_t mul_hi, int j) {
  const uint64_t lo_hi = umulhi(m, mul_lo);              // (m * mul_lo) >> 64
  const uint64_t hi_lo = m * mul_hi, hi_hi = umulhi(m, mul_hi);
  const uint64_t sum_lo = hi_lo + lo_hi;                  // the 128-bit sum m * mul_hi + (m * mul_lo >> 64)
  const uint64_t sum_hi = hi_hi + (sum_lo < hi_lo ? 1 : 0);
  const int s = j - 64;                                   // in (0, 64)
  return (sum_hi << (64 - s)) | (sum_lo >> s);
}

// floor(log10(2^e)), floor(log10(5^e)) and ceil(log2(5^e)) (1 for e = 0), exact for the ranges used here
GR_FR_HD int log10_pow2(int e) { return (int)(((uint32_t)e * 78913u) >> 18); }
GR_FR_HD int log10_pow5(int e) { return (int)(((uint32_t)e * 732923u) >> 20); }
GR_FR_HD int pow5_bits(int e) { return (int)(((uint32_t)e * 1217359u) >> 19) + 1; }

GR_FR_HD bool multiple_of_pow5(uint64_t v, int p) {
  int n = 0;
  while (v % 5 == 0 && v != 0) {
    v /= 5;
    ++n;
  }
  return n >= p;
}

GR_FR_HD bool multiple_of_pow2(uint64_t v, int p) { return (v & ((1ull << p) - 1)) == 0; }

GR_FR_HD int decimal_length(uint64_t v) {
  int n = 1;
  while (n < 20 && v >= 10) {
    v /= 10;
    ++n;
  }
  return n;
}

// A float64 split for printing.  kind: 0 finite nonzero (digits * 10^exp10, `ndigits` decimal digits), 1 zero,
// 2 NaN, 3 infinity.
struct Decimal {
  uint64_t digits;
  int exp10;
  int ndigits;
  int kind;
  bool neg;
};

// the shortest, closest decimal of x
GR_FR_HD Decimal shortest(double x) {
  uint64_t bits;
  memcpy(&bits, &x, sizeof(bits));
  Decimal d;
  d.neg = (bits >> 63) != 0;
  d.digits = 0;
  d.exp10 = 0;
  d.ndigits = 1;
  const uint64_t mant = bits & ((1ull << 52) - 1);
  const int bexp = (int)((bits >> 52) & 0x7ff);
  if (bexp == 0x7ff) {
    d.kind = mant ? 2 : 3;
    return d;
  }
  if (bexp == 0 && mant == 0) {
    d.kind = 1;
    return d;
  }
  d.kind = 0;
  // x = m2 * 2^e2 / 4 with the bounds of its rounding interval at 4 m2 - 1 - mm_shift and 4 m2 + 2
  const int e2 = (bexp == 0 ? 1 : bexp) - 1023 - 52 - 2;
  const uint64_t m2 = bexp == 0 ? mant : (1ull << 52) | mant;
  const bool accept_bounds = (m2 & 1) == 0;              // round-half-even reading includes the bounds
  const uint64_t mv = 4 * m2;
  const uint64_t mm_shift = (mant != 0 || bexp <= 1) ? 1 : 0;   // the lower gap is half as wide at a power of two
  uint64_t vr, vp, vm;
  int e10;
  bool vm_zeros = false, vr_zeros = false;                // the removed digits of vm / vr are all zero
  if (e2 >= 0) {
    const int q = log10_pow2(e2) - (e2 > 3 ? 1 : 0);
    e10 = q;
    const int j = -e2 + q + 125 + pow5_bits(q) - 1;
    const uint64_t lo = pow5_inv(q, 0), hi = pow5_inv(q, 1);
    vr = mul_shift(mv, lo, hi, j);
    vp = mul_shift(mv + 2, lo, hi, j);
    vm = mul_shift(mv - 1 - mm_shift, lo, hi, j);
    if (q <= 21) {                                         // exact products: the division by 10^q may be exact
      if (mv % 5 == 0) vr_zeros = multiple_of_pow5(mv, q);
      else if (accept_bounds) vm_zeros = multiple_of_pow5(mv - 1 - mm_shift, q);
      else vp -= multiple_of_pow5(mv + 2, q) ? 1 : 0;
    }
  } else {
    const int q = log10_pow5(-e2) - (-e2 > 1 ? 1 : 0);
    e10 = q + e2;
    const int i = -e2 - q;
    const int j = q - (pow5_bits(i) - 125);
    const uint64_t lo = pow5(i, 0), hi = pow5(i, 1);
    vr = mul_shift(mv, lo, hi, j);
    vp = mul_shift(mv + 2, lo, hi, j);
    vm = mul_shift(mv - 1 - mm_shift, lo, hi, j);
    if (q <= 1) {
      vr_zeros = true;                                     // mv has at least q trailing zero bits
      if (accept_bounds) vm_zeros = mm_shift == 1;
      else --vp;
    } else if (q < 63) {
      vr_zeros = multiple_of_pow2(mv, q);
    }
  }
  int removed = 0;
  uint64_t out;
  if (vm_zeros || vr_zeros) {                              // exact ties possible: track the removed digits
    int last = 0;
    while (vp / 10 > vm / 10) {
      vm_zeros &= vm % 10 == 0;
      vr_zeros &= last == 0;
      last = (int)(vr % 10);
      vr /= 10; vp /= 10; vm /= 10;
      ++removed;
    }
    if (vm_zeros) {
      while (vm % 10 == 0) {
        vr_zeros &= last == 0;
        last = (int)(vr % 10);
        vr /= 10; vp /= 10; vm /= 10;
        ++removed;
      }
    }
    if (vr_zeros && last == 5 && vr % 2 == 0) last = 4;   // an exact half: round to even
    out = vr + (((vr == vm && (!accept_bounds || !vm_zeros)) || last >= 5) ? 1 : 0);
  } else {
    bool round_up = false;
    if (vp / 100 > vm / 100) {
      round_up = vr % 100 >= 50;
      vr /= 100; vp /= 100; vm /= 100;
      removed += 2;
    }
    while (vp / 10 > vm / 10) {
      round_up = vr % 10 >= 5;
      vr /= 10; vp /= 10; vm /= 10;
      ++removed;
    }
    out = vr + ((vr == vm || round_up) ? 1 : 0);
  }
  d.digits = out;
  d.exp10 = e10 + removed;
  d.ndigits = decimal_length(out);
  return d;
}

// decpt of x = 0.d1 .. dn * 10^decpt
GR_FR_HD int decpt(const Decimal& d) { return d.exp10 + d.ndigits; }

GR_FR_HD bool exponent_notation(const Decimal& d) { return decpt(d) <= -4 || decpt(d) > 16; }

// bytes of the repr of d
GR_FR_HD int repr_len(const Decimal& d) {
  if (d.kind == 2) return 3;                              // NaN
  if (d.kind == 3) return d.neg ? 9 : 8;                  // -Infinity, Infinity
  const int sign = d.neg ? 1 : 0;
  if (d.kind == 1) return sign + 3;                       // 0.0
  const int n = d.ndigits, dp = decpt(d);
  if (exponent_notation(d)) {
    const int e = dp - 1 < 0 ? 1 - dp : dp - 1;
    return sign + n + (n > 1 ? 1 : 0) + 2 + (e >= 100 ? 3 : 2);
  }
  if (dp <= 0) return sign + 2 - dp + n;                  // 0.000ddd
  if (dp < n) return sign + n + 1;                        // ddd.ddd
  return sign + dp + 2;                                   // ddd000.0
}

// writes the repr_len(d) bytes of the repr of d at out
template <typename Byte>
GR_FR_HD void write_repr(const Decimal& d, Byte* out) {
  int o = 0;
  auto put = [&](char c) { out[o++] = (Byte)c; };
  if (d.kind == 2) {
    put('N'); put('a'); put('N');
    return;
  }
  if (d.neg) put('-');
  if (d.kind == 3) {
    const char* s = "Infinity";
    for (int i = 0; i < 8; ++i) put(s[i]);
    return;
  }
  if (d.kind == 1) {
    put('0'); put('.'); put('0');
    return;
  }
  const int n = d.ndigits, dp = decpt(d);
  // the digits most significant first, from a running divisor
  uint64_t p10 = 1;
  for (int i = 1; i < n; ++i) p10 *= 10;
  uint64_t rest = d.digits;
  auto next_digit = [&]() {
    const uint64_t q = rest / p10;
    rest -= q * p10;
    p10 /= 10;
    return (char)('0' + q);
  };
  if (exponent_notation(d)) {
    put(next_digit());
    if (n > 1) {
      put('.');
      for (int i = 1; i < n; ++i) put(next_digit());
    }
    int e = dp - 1;
    put('e');
    put(e < 0 ? '-' : '+');
    if (e < 0) e = -e;
    if (e >= 100) put((char)('0' + e / 100));
    put((char)('0' + e / 10 % 10));
    put((char)('0' + e % 10));
    return;
  }
  if (dp <= 0) {
    put('0'); put('.');
    for (int i = 0; i < -dp; ++i) put('0');
    for (int i = 0; i < n; ++i) put(next_digit());
    return;
  }
  for (int i = 0; i < n; ++i) {
    if (i == dp) put('.');
    put(next_digit());
  }
  if (dp >= n) {
    for (int i = n; i < dp; ++i) put('0');
    put('.'); put('0');
  }
}

}  // namespace fr
}  // namespace gr
