// One float as PCL's ASCII PCD writer prints it (pcl::PCDWriter::writeASCII: `ostream << float` at precision 8 in the
// classic locale, `nan` for every NaN). libstdc++ widens the float to double and prints it with "%.8g", so the text is
// glibc's correctly rounded %.8g of the exact binary value (ties to even). Computed here in exact integer arithmetic:
// double arithmetic cannot decide the near-ties of small floats, which need more than 100 bits.
//
// __host__ __device__ so that the encode kernels (pcd_codec.cu) and the host tests (tests/hostmath/pcd_host.cpp, checked
// against snprintf) run the same code.
#pragma once
#include <stdint.h>
#include <string.h>

#if !defined(B200_HD)
#if defined(__CUDACC__)
#define B200_HD __host__ __device__ __forceinline__
#else
#define B200_HD inline
#endif
#endif

namespace b200 {

constexpr int PCD_FLOAT_MAX_CHARS = 14;                        // "-1.2345678e-38", "-0.00012345678"
constexpr int PCD_LINE_MAX_CHARS = 4 * PCD_FLOAT_MAX_CHARS + 4;  // four fields, three spaces and '\n'

namespace pcdfmt {

B200_HD uint64_t mulhi64(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
  return __umul64hi(a, b);
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}

B200_HD uint64_t pow5_u64(int q) {  // q <= 27 (5^27 < 2^64)
  uint64_t r = 1, b = 5;
  while (q) {
    if (q & 1) r *= b;
    b *= b;
    q >>= 1;
  }
  return r;
}

// (x[0..2], little-endian 64-bit limbs) *= y
B200_HD void mul3(uint64_t (&x)[3], uint64_t y) {
  const uint64_t l0 = x[0] * y, h0 = mulhi64(x[0], y);
  const uint64_t l1 = x[1] * y, h1 = mulhi64(x[1], y);
  const uint64_t l2 = x[2] * y;
  const uint64_t m1 = l1 + h0;
  x[0] = l0;
  x[1] = m1;
  x[2] = l2 + h1 + (m1 < l1 ? 1u : 0u);
}

B200_HD bool bit3(const uint64_t (&x)[3], int i) { return (x[i >> 6] >> (i & 63)) & 1u; }

// any of bits [0, i) set
B200_HD bool any_below3(const uint64_t (&x)[3], int i) {
  for (int w = 0; w < 3; w++) {
    const int lo = w * 64;
    if (i <= lo) break;
    const uint64_t mask = (i - lo >= 64) ? ~(uint64_t)0 : (((uint64_t)1 << (i - lo)) - 1u);
    if (x[w] & mask) return true;
  }
  return false;
}

// bits [i, i + 64) of x
B200_HD uint64_t extract3(const uint64_t (&x)[3], int i) {
  const int w = i >> 6, b = i & 63;
  uint64_t r = x[w] >> b;
  if (b && w + 1 < 3) r |= x[w + 1] << (64 - b);
  return r;
}

// 128-bit numerator held as four 32-bit words, most significant first: n /= d, returns the remainder
B200_HD uint32_t div4x32(uint32_t (&n)[4], uint32_t d) {
  uint64_t rem = 0;
  for (int k = 0; k < 4; k++) {
    const uint64_t cur = (rem << 32) | n[k];
    n[k] = (uint32_t)(cur / d);
    rem = cur % d;
  }
  return (uint32_t)rem;
}

}  // namespace pcdfmt

// Writes the text of one float as PCL's writeASCII does (no terminator); returns its length (<= PCD_FLOAT_MAX_CHARS).
B200_HD int pcd_format_float(float f, char* out) {
  using namespace pcdfmt;
  uint32_t bits;
  memcpy(&bits, &f, sizeof bits);
  const bool neg = bits >> 31;
  const uint32_t ef = (bits >> 23) & 0xffu, frac = bits & 0x7fffffu;
  int len = 0;
  if (ef == 0xffu && frac) {  // writeASCII prints every NaN as "nan", whatever its sign and payload
    out[0] = 'n'; out[1] = 'a'; out[2] = 'n';
    return 3;
  }
  if (neg) out[len++] = '-';
  if (ef == 0xffu) {
    out[len] = 'i'; out[len + 1] = 'n'; out[len + 2] = 'f';
    return len + 3;
  }
  if (ef == 0 && frac == 0) {
    out[len] = '0';
    return len + 1;
  }
  // value = m * 2^e, 0 < m < 2^24
  const uint32_t m = ef ? (frac | 0x800000u) : frac;
  const int e = ef ? (int)ef - 150 : -149;
  int bl = 0;
  for (uint32_t t = m; t; t >>= 1) bl++;
  const int e2 = e + bl - 1;                     // floor(log2 value)
  int k = (e2 * 78913) >> 18;                    // floor(e2 log10 2): the decimal exponent, or one less (floor division)
  // S = value * 10^(7 - k) in [10^7, 10^9): integer part I, then the fraction as (half bit, sticky rest)
  uint64_t I;
  bool half, sticky;
  const int q = 7 - k;
  if (q >= 0) {  // S = m 5^q 2^(e + q); q <= 52, m 5^q < 2^146
    uint64_t P[3] = {m, 0, 0};
    const int qa = q < 27 ? q : 27;
    mul3(P, pow5_u64(qa));
    if (q > qa) mul3(P, pow5_u64(q - qa));
    const int s = e + q;
    if (s >= 0) {
      I = P[0] << s;  // only when S is small enough to be exact in 64 bits
      half = sticky = false;
    } else {
      I = extract3(P, -s);
      half = bit3(P, -s - 1);
      sticky = any_below3(P, -s - 1);
    }
  } else {  // S = m 2^e / 10^p, p = k - 7 <= 31; e - p >= 2 here. Divide 2 m 2^(e - p) (one guard bit) by 5^p.
    const int p = -q;
    const int sh = e - p + 1;  // <= 74: the numerator has at most 98 bits
    uint32_t n4[4];
    {
      const uint64_t lo = sh >= 64 ? 0 : (uint64_t)m << sh;
      const uint64_t hi = sh >= 64 ? (uint64_t)m << (sh - 64) : (sh ? (uint64_t)m >> (64 - sh) : 0);
      n4[0] = (uint32_t)(hi >> 32); n4[1] = (uint32_t)hi; n4[2] = (uint32_t)(lo >> 32); n4[3] = (uint32_t)lo;
    }
    bool rem = false;
    for (int left = p; left > 0; left -= 13) {  // 5^13 < 2^32: at most three 32-bit-divisor long divisions
      rem |= div4x32(n4, (uint32_t)pow5_u64(left < 13 ? left : 13)) != 0;
    }
    const uint64_t T = ((uint64_t)n4[2] << 32) | n4[3];  // 2 S < 2^31: the upper words are zero
    I = T >> 1;
    half = T & 1u;
    sticky = rem;
  }
  if (I >= 100000000u) {  // k was one short: S / 10, the dropped digit joins the fraction
    const unsigned r = (unsigned)(I % 10u);
    I /= 10u;
    k += 1;
    // new fraction (r + f) / 10: at least 1/2 iff r >= 5, and then above 1/2 iff r > 5 or f > 0 (sticky only matters
    // when half is set)
    sticky = r > 5 || half || sticky;
    half = r >= 5;
  }
  uint32_t N = (uint32_t)I;
  if (half && (sticky || (N & 1u))) N += 1;  // round half to even
  if (N == 100000000u) {
    N = 10000000u;
    k += 1;
  }
  char d[8];
  for (int i = 7; i >= 0; i--) {
    d[i] = (char)('0' + N % 10u);
    N /= 10u;
  }
  int nd = 8;  // significant digits left after stripping trailing zeros (%g without '#')
  while (nd > 1 && d[nd - 1] == '0') nd--;
  if (k >= -4 && k < 8) {  // style f, precision 7 - k
    if (k >= 0) {
      for (int i = 0; i <= k; i++) out[len++] = i < nd ? d[i] : '0';
      if (nd > k + 1) {
        out[len++] = '.';
        for (int i = k + 1; i < nd; i++) out[len++] = d[i];
      }
    } else {
      out[len++] = '0';
      out[len++] = '.';
      for (int i = 0; i < -k - 1; i++) out[len++] = '0';
      for (int i = 0; i < nd; i++) out[len++] = d[i];
    }
  } else {  // style e, at least two exponent digits
    out[len++] = d[0];
    if (nd > 1) {
      out[len++] = '.';
      for (int i = 1; i < nd; i++) out[len++] = d[i];
    }
    out[len++] = 'e';
    out[len++] = k < 0 ? '-' : '+';
    const int ax = k < 0 ? -k : k;
    out[len++] = (char)('0' + ax / 10);
    out[len++] = (char)('0' + ax % 10);
  }
  return len;
}

// One point's line: x y z intensity, single spaces, '\n'. Returns its length (<= PCD_LINE_MAX_CHARS).
B200_HD int pcd_format_line(float x, float y, float z, float intensity, char* out) {
  int len = pcd_format_float(x, out);
  out[len++] = ' ';
  len += pcd_format_float(y, out + len);
  out[len++] = ' ';
  len += pcd_format_float(z, out + len);
  out[len++] = ' ';
  len += pcd_format_float(intensity, out + len);
  out[len++] = '\n';
  return len;
}

}  // namespace b200
