// Decimal text to binary32 — the value glibc strtof returns for a token — one token at a time, on the host and on the
// device.  Round to nearest, ties to even, with subnormals; past the largest float +-inf, below half the smallest
// subnormal +-0.  The grammar is [+-]?(d+[.d*]|.d+)([eE][+-]?d+)? and, with an optional sign and in any case, nan, inf
// and infinity ("%lf" writes -nan for a NaN whose sign bit is set); anything else (hex floats, an empty token, trailing
// characters) is refused.
//
// Exactness (DESIGN section 4.4, "Text vector files"):
//  * fast path: at most 19 significant digits w, trailing zeros moved into the exponent, w < 2^53 and |E| <= 22.  Then
//    w and 10^|E| are exact doubles, q = w * 10^E (or w / 10^-E) is w x 10^E correctly rounded to double, and the
//    fma residual r = w x 10^E - q is exact.  r = 0: q is the value and (float)q rounds it once.  r != 0: rounding q
//    to float gives the float of w x 10^E unless q is exactly a midpoint between two floats (every midpoint of
//    binary32 is a double, and rounding to double is monotone, so q and the exact value lie on the same side of every
//    other midpoint).  That one case goes to the slow path.
//  * slow path: a float f within a few units of the answer (from the first 19 digits and pow), then moved one unit at
//    a time until the exact value lies between its two midpoints, each comparison done on integers: the token's first
//    120 significant digits N (and whether any later digit is non-zero) against a midpoint (2m + 1) x 2^(k-1), scaled
//    by powers of 5 and 2 until both sides are integers.  A binary32 midpoint has at most 113 significant decimal
//    digits, so digits past the 120th only matter when N equals the midpoint, and then they make the value larger.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define W2B_TEXT_HD __host__ __device__ __forceinline__
#define W2B_TEXT_SLOW __host__ __device__ __noinline__
#else
#define W2B_TEXT_HD inline
#define W2B_TEXT_SLOW inline
#endif

namespace w2b {
namespace text {

// the characters fscanf's %s stops at
W2B_TEXT_HD bool is_space(char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\v' || c == '\f' || c == '\r'; }

W2B_TEXT_HD uint32_t f2u(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
}
W2B_TEXT_HD float u2f(uint32_t u) {
  float f;
  memcpy(&f, &u, 4);
  return f;
}

constexpr int kKeep = 120;  // significant digits the exact comparison reads
constexpr int kLimbs = 40;  // 1280 bits; the largest operand of a comparison has fewer than 700

// A non-negative decimal: the integer N of its significant digits times 10^e.
struct Decimal {
  uint64_t w = 0;      // the first nw significant digits of N
  int nw = 0, nsig = 0;  // digits in w; significant digits in the token (first non-zero digit to the last digit)
  long long e = 0;
  const char *m0 = nullptr, *m1 = nullptr;  // the digits and '.' of the token
};

struct Big {  // unsigned integer, 32-bit limbs, least significant first
  uint32_t d[kLimbs];
  int n;
};

W2B_TEXT_HD void big_set(Big &a, uint64_t v) {
  a.n = 0;
  while (v) {
    a.d[a.n++] = (uint32_t)v;
    v >>= 32;
  }
}
W2B_TEXT_HD void big_mul_add(Big &a, uint32_t m, uint32_t add) {
  uint64_t carry = add;
  for (int i = 0; i < a.n; ++i) {
    const uint64_t t = (uint64_t)a.d[i] * m + carry;
    a.d[i] = (uint32_t)t;
    carry = t >> 32;
  }
  if (carry && a.n < kLimbs) a.d[a.n++] = (uint32_t)carry;
}
W2B_TEXT_HD void big_mul_pow5(Big &a, long long k) {
  for (; k >= 13; k -= 13) big_mul_add(a, 1220703125u, 0);  // 5^13
  uint32_t m = 1;
  for (; k > 0; --k) m *= 5;
  big_mul_add(a, m, 0);
}
W2B_TEXT_HD void big_shl(Big &a, long long s) {
  if (a.n == 0) return;
  const int limbs = (int)(s >> 5), bits = (int)(s & 31);
  int n = a.n + limbs + 1;
  if (n > kLimbs) n = kLimbs;
  for (int i = n - 1; i >= 0; --i) {
    const int j = i - limbs;
    const uint32_t hi = (j >= 0 && j < a.n) ? a.d[j] : 0u, lo = (j - 1 >= 0 && j - 1 < a.n) ? a.d[j - 1] : 0u;
    a.d[i] = bits ? (hi << bits) | (lo >> (32 - bits)) : hi;
  }
  a.n = n;
  while (a.n && !a.d[a.n - 1]) --a.n;
}
W2B_TEXT_HD int big_cmp(const Big &a, const Big &b) {
  if (a.n != b.n) return a.n < b.n ? -1 : 1;
  for (int i = a.n - 1; i >= 0; --i)
    if (a.d[i] != b.d[i]) return a.d[i] < b.d[i] ? -1 : 1;
  return 0;
}

// 10^k, 0 <= k <= 22: a product of exact powers whose partial products stay exact
W2B_TEXT_HD double pow10_exact(int k) {
  double r = 1.0, p = 10.0;
  for (; k; k >>= 1, p *= p)
    if (k & 1) r *= p;
  return r;
}

// sign of (N x 10^E + sticky) - (the midpoint between the floats with bits b and b + 1)
W2B_TEXT_HD int cmp_midpoint(const Big &N, long long E, bool sticky, uint32_t b) {
  const uint32_t be = b >> 23, frac = b & 0x7fffffu;
  const uint32_t m = be ? (frac | 0x800000u) : frac;
  const long long K = (be ? (long long)be - 150 : -149) - 1;  // midpoint = (2m + 1) x 2^K
  Big A = N, B;
  big_set(B, 2ull * m + 1);
  if (E >= 0)
    big_mul_pow5(A, E);
  else
    big_mul_pow5(B, -E);
  if (E - K >= 0)
    big_shl(A, E - K);
  else
    big_shl(B, K - E);
  const int c = big_cmp(A, B);
  return c ? c : (sticky ? 1 : 0);
}

// the float of a decimal that the fast path could not settle; 1e-46 <= value < 1e40
W2B_TEXT_SLOW uint32_t slow_bits(const Decimal &d) {
  Big N;
  N.n = 0;
  int kept = 0;
  bool sticky = false;
  uint32_t group = 0, gmul = 1;
  for (const char *p = d.m0; p < d.m1; ++p) {
    if (*p == '.' || (kept == 0 && *p == '0')) continue;
    if (kept == kKeep) {
      sticky |= *p != '0';
      continue;
    }
    group = group * 10 + (uint32_t)(*p - '0');
    gmul *= 10;
    ++kept;
    if (gmul == 1000000000u) {
      if (N.n == 0) big_set(N, group); else big_mul_add(N, gmul, group);
      group = 0;
      gmul = 1;
    }
  }
  if (gmul > 1) {
    if (N.n == 0) big_set(N, group); else big_mul_add(N, gmul, group);
  }
  const long long E = d.e + (d.nsig - kept);
  float f = (float)((double)d.w * pow(10.0, (double)(d.e + d.nsig - d.nw)));
  uint32_t b = f2u(f);
  if (b > 0x7f7fffffu) b = 0x7f7fffffu;
  for (int it = 0; it < 64; ++it) {
    if (b < 0x7f800000u) {
      const int c = cmp_midpoint(N, E, sticky, b);
      if (c > 0 || (c == 0 && (b & 1))) { ++b; continue; }
    }
    if (b > 0) {
      const int c = cmp_midpoint(N, E, sticky, b - 1);
      if (c < 0 || (c == 0 && (b & 1))) { --b; continue; }
    }
    break;
  }
  return b;
}

// bits of the float of a decimal (non-negative)
W2B_TEXT_HD uint32_t decimal_bits(const Decimal &d) {
  if (d.nsig == 0) return 0;
  const long long mag = d.e + d.nsig;  // 10^(mag-1) <= value < 10^mag
  if (mag <= -46) return 0;            // below 1e-46 < 2^-150, half the smallest subnormal
  if (mag >= 40) return 0x7f800000u;   // at least 1e39 > FLT_MAX
  if (d.nsig == d.nw) {
    uint64_t w = d.w;
    long long E = d.e;
    while (w % 10 == 0) {
      w /= 10;
      ++E;
    }
    if (w < (1ull << 53) && E >= -22 && E <= 22) {
      const double x = (double)w, p = pow10_exact((int)(E < 0 ? -E : E));
      double q, r;
      if (E >= 0) {
        q = x * p;
        r = fma(x, p, -q);
      } else {
        q = x / p;
        r = fma(-q, p, x);
      }
      const float f = (float)q;  // normal: 1e-22 <= q < 2^53 x 1e22 < FLT_MAX
      if (r == 0.0 || (double)f == q) return f2u(f);
      const uint32_t fb = f2u(f), gb = q > (double)f ? fb + 1 : fb - 1;
      if (((double)f + (double)u2f(gb)) * 0.5 != q) return fb;  // q is not a midpoint
    }
  }
  return slow_bits(d);
}

W2B_TEXT_HD char lower(char c) { return (c >= 'A' && c <= 'Z') ? (char)(c + 32) : c; }

// s[0..n) equals word (lower case) in any case
W2B_TEXT_HD bool word_is(const char *s, long long n, const char *word) {
  long long i = 0;
  for (; word[i]; ++i)
    if (i >= n || lower(s[i]) != word[i]) return false;
  return i == n;
}

// The token [s, end): *out = its float.  false: not in the grammar.
W2B_TEXT_HD bool parse_token(const char *s, const char *end, float *out) {
  const char *p = s;
  uint32_t sign = 0;
  if (p < end && (*p == '+' || *p == '-')) sign = (*p++ == '-') ? 0x80000000u : 0u;
  if (p < end && (lower(*p) == 'n' || lower(*p) == 'i')) {
    const long long n = end - p;
    if (word_is(p, n, "nan")) { *out = u2f(sign | 0x7fc00000u); return true; }
    if (word_is(p, n, "inf") || word_is(p, n, "infinity")) { *out = u2f(sign | 0x7f800000u); return true; }
    return false;
  }
  Decimal d;
  d.m0 = p;
  int ndig = 0, nfrac = 0;
  bool point = false;
  for (; p < end; ++p) {
    const char c = *p;
    if (c == '.' && !point) {
      point = true;
      continue;
    }
    if (c < '0' || c > '9') break;
    ++ndig;
    if (point) ++nfrac;
    if (d.nsig == 0 && c == '0') continue;
    if (d.nw < 19) {
      d.w = d.w * 10 + (uint64_t)(c - '0');
      ++d.nw;
    }
    ++d.nsig;
  }
  d.m1 = p;
  if (ndig == 0) return false;
  long long ex = 0;
  if (p < end && (*p == 'e' || *p == 'E')) {
    ++p;
    bool eneg = false;
    if (p < end && (*p == '+' || *p == '-')) eneg = *p++ == '-';
    if (p == end || *p < '0' || *p > '9') return false;
    for (; p < end && *p >= '0' && *p <= '9'; ++p)
      if (ex < 1000000000LL) ex = ex * 10 + (*p - '0');  // beyond 1e9 the result is 0 or inf either way
    if (eneg) ex = -ex;
  }
  if (p != end) return false;
  d.e = ex - nfrac;  // value = N x 10^(ex - nfrac), N = the integer of every digit
  *out = u2f(sign | decimal_bits(d));
  return true;
}

// end of the token starting at s (the first space at or after s, or end)
W2B_TEXT_HD const char *token_end(const char *s, const char *end) {
  while (s < end && !is_space(*s)) ++s;
  return s;
}

}  // namespace text
}  // namespace w2b
