// The reading side of pcd_format.cuh: one data line of an ASCII PCD file as PCL 1.12's PCDReader::readBodyASCII reads it
// (tokens split on ' ', '\t' and '\r', runs of separators compressed) and one token as copyStringValue<float> converts
// it: iequals("nan") gives quiet_NaN, everything else goes through `istringstream >> float` in the classic locale, which
// is glibc's strtof, correctly rounded (subnormals included, ties to even, overflow to +-inf), and the signed nan / inf /
// infinity spellings that stream rejects take the value of PCL's atof fallback. Tokens outside that grammar are refused
// here (PCL would take atof's prefix value): see b200reg_load_pcd in include/b200reg.h.
//
// The conversion: the first 19 significant digits go to a u64, scaled by a power of ten in double (relative error below
// 2^-50), rounded to float; when that double lies within 2^-48 of a halfway point between two floats, the token's digits
// (all of them) are compared exactly with the decimal expansion of the halfway point, computed in 32-bit limbs. The
// halfway point is a dyadic number of at most 26 significant bits whose expansion has at most 113 digits.
//
// __host__ __device__ so that the parse kernel (pcd_load.cu) and the host tests (tests/hostmath/pcd_parse_host.cpp,
// checked against strtof and the restated PCL reader) run the same code. The header parser at the end is host-only.
#pragma once
#include <stdint.h>
#include <string.h>

#include <string>
#include <vector>

#if !defined(B200_HD)
#if defined(__CUDACC__)
#define B200_HD __host__ __device__ __forceinline__
#else
#define B200_HD inline
#endif
#endif
#if defined(__CUDACC__)
#define B200_HD_COLD inline __host__ __device__ __noinline__
#else
#define B200_HD_COLD inline
#endif

namespace b200 {

namespace pcdparse {

B200_HD bool is_sep(char c) { return c == ' ' || c == '\t' || c == '\r'; }
B200_HD bool is_digit(char c) { return (unsigned)(c - '0') < 10u; }

// s[0..n) equals the lower-case literal `lit`, ignoring case
B200_HD bool ieq(const char* s, int n, const char* lit) {
  for (int i = 0; i < n; i++) {
    char c = s[i];
    if (c >= 'A' && c <= 'Z') c = (char)(c + 32);
    if (c != lit[i]) return false;
  }
  return true;
}

// v * 10^x, |x| <= 64: at most three correctly rounded products or quotients by exact powers of ten (<= 10^22)
B200_HD double mul_pow10(double v, int x) {
  const bool down = x < 0;
  if (down) x = -x;
  while (x > 0) {
    const int k = x < 22 ? x : 22;
    double p = 1.0;
    for (int i = 0; i < k; i++) p *= 10.0;
    v = down ? v / p : v * p;
    x -= k;
  }
  return v;
}

B200_HD uint32_t pow5_u32(int q) {  // q <= 13 (5^13 < 2^32)
  uint32_t r = 1;
  for (int i = 0; i < q; i++) r *= 5u;
  return r;
}

constexpr int BIG_LIMBS = 12;  // 384 bits: the largest expansion is (2^25 - 1) * 5^150 < 2^374

// Compares the decimal value 0.d1d2... * 10^e10 (digits: the text [first, end), '.' skipped, first is a nonzero digit) with
// the positive double H. Returns -1, 0 or 1.
B200_HD_COLD int compare_exact(const char* first, const char* end, long long e10, double H) {
  uint64_t bits;
  memcpy(&bits, &H, sizeof bits);
  uint64_t hm = (bits & 0xFFFFFFFFFFFFFull) | (1ull << 52);
  int hk = (int)((bits >> 52) & 0x7ff) - 1075;
  while (!(hm & 1u)) {
    hm >>= 1;
    hk++;
  }
  // H = hm * 2^hk = N * 10^min(hk, 0), with N = hm * 2^hk or hm * 5^-hk
  uint32_t N[BIG_LIMBS] = {0};
  N[0] = (uint32_t)hm;
  N[1] = (uint32_t)(hm >> 32);
  int n = N[1] ? 2 : 1;
  for (int left = hk >= 0 ? hk : -hk; left > 0;) {
    const int k = hk >= 0 ? (left < 31 ? left : 31) : (left < 13 ? left : 13);
    const uint32_t m = hk >= 0 ? (1u << k) : pow5_u32(k);
    uint64_t carry = 0;
    for (int j = 0; j < n; j++) {
      const uint64_t t = (uint64_t)N[j] * m + carry;
      N[j] = (uint32_t)t;
      carry = t >> 32;
    }
    if (carry) N[n++] = (uint32_t)carry;
    left -= k;
  }
  uint32_t groups[BIG_LIMBS * 10 / 9 + 2];  // base-10^9 digits, least significant first
  int ng = 0;
  while (n > 0) {
    uint64_t rem = 0;
    for (int j = n - 1; j >= 0; j--) {
      const uint64_t cur = (rem << 32) | N[j];
      N[j] = (uint32_t)(cur / 1000000000u);
      rem = cur % 1000000000u;
    }
    groups[ng++] = (uint32_t)rem;
    while (n > 0 && N[n - 1] == 0) n--;
  }
  char dig[(BIG_LIMBS * 10 / 9 + 2) * 9];
  int nd = 0;
  for (int g = ng - 1; g >= 0; g--) {
    char t[9];
    uint32_t v = groups[g];
    for (int j = 8; j >= 0; j--) {
      t[j] = (char)('0' + v % 10u);
      v /= 10u;
    }
    int j = 0;
    if (g == ng - 1)
      while (j < 8 && t[j] == '0') j++;
    for (; j < 9; j++) dig[nd++] = t[j];
  }
  const long long eh = nd + (hk < 0 ? hk : 0);  // H = 0.dig * 10^eh
  if (e10 != eh) return e10 < eh ? -1 : 1;
  const char* p = first;
  for (int i = 0;; i++, p++) {
    while (p < end && *p == '.') p++;
    if (p >= end) {
      for (; i < nd; i++)
        if (dig[i] != '0') return -1;
      return 0;
    }
    if (i >= nd) {
      for (; p < end; p++)
        if (*p != '.' && *p != '0') return 1;
      return 0;
    }
    if (*p != dig[i]) return *p < dig[i] ? -1 : 1;
  }
}

// |value| = 0.(digits) * 10^e10 with -45 <= e10 <= 39; w = its first nw (<= 19) significant digits. Returns float bits.
B200_HD uint32_t round_decimal(uint64_t w, int nw, long long e10, const char* first, const char* end) {
  const double d = mul_pow10((double)w, (int)(e10 - nw));
  const double tol = d * 0x1p-48;
  const double T = 0x1.ffffffp127;  // FLT_MAX + half an ulp: from here on strtof overflows
  const float c = (float)d;
  uint32_t cb;
  memcpy(&cb, &c, sizeof cb);
  if (cb == 0x7f800000u) {
    if (d - T > tol) return cb;
    return compare_exact(first, end, e10, T) >= 0 ? 0x7f800000u : 0x7f7fffffu;
  }
  float up, down;
  const uint32_t ub = cb + 1u, db = cb - 1u;
  memcpy(&up, &ub, sizeof up);
  memcpy(&down, &db, sizeof down);
  const double hp = cb == 0x7f7fffffu ? T : ((double)c + (double)up) * 0.5;
  if ((d > hp ? d - hp : hp - d) <= tol) {
    const int r = compare_exact(first, end, e10, hp);
    return (r > 0 || (r == 0 && (cb & 1u))) ? ub : cb;
  }
  if (cb != 0) {
    const double hm = ((double)c + (double)down) * 0.5;
    if ((d > hm ? d - hm : hm - d) <= tol) {
      const int r = compare_exact(first, end, e10, hm);
      return (r < 0 || (r == 0 && (cb & 1u))) ? db : cb;
    }
  }
  return cb;
}

}  // namespace pcdparse

// One token s[0..len) as copyStringValue<float> reads it. Grammar: [+-] (digits [. [digits]] | . digits)
// [(e|E) [+-] digits], or [+-] nan | inf | infinity in any case. Returns false for anything else.
B200_HD bool pcd_parse_float(const char* s, int len, float* out) {
  using namespace pcdparse;
  int i = 0;
  bool neg = false;
  if (len > 0 && (s[0] == '+' || s[0] == '-')) {
    neg = s[0] == '-';
    i = 1;
  }
  const int rl = len - i;
  uint32_t bits;
  if (rl == 3 && ieq(s + i, 3, "nan")) {
    bits = neg ? 0xffc00000u : 0x7fc00000u;  // quiet_NaN, or atof's signed NaN
    memcpy(out, &bits, sizeof bits);
    return true;
  }
  if ((rl == 3 && ieq(s + i, 3, "inf")) || (rl == 8 && ieq(s + i, 8, "infinity"))) {
    bits = neg ? 0xff800000u : 0x7f800000u;
    memcpy(out, &bits, sizeof bits);
    return true;
  }
  bool dot = false;
  int ndig = 0, nw = 0;
  const char* first = nullptr;  // first nonzero digit
  long long e10 = 0;            // |value| = 0.(significant digits) * 10^e10
  uint64_t w = 0;
  for (; i < len; i++) {
    const char ch = s[i];
    if (ch == '.') {
      if (dot) return false;
      dot = true;
      continue;
    }
    if (!is_digit(ch)) break;
    ndig++;
    if (!first) {
      if (ch == '0') {
        if (dot) e10--;
        continue;
      }
      first = s + i;
    }
    if (!dot) e10++;
    if (nw < 19) {
      w = w * 10u + (uint64_t)(ch - '0');
      nw++;
    }
  }
  if (ndig == 0) return false;
  const char* mend = s + i;
  if (i < len && (s[i] == 'e' || s[i] == 'E')) {
    i++;
    bool eneg = false;
    if (i < len && (s[i] == '+' || s[i] == '-')) {
      eneg = s[i] == '-';
      i++;
    }
    long long ex = 0;
    int nexp = 0;
    for (; i < len && is_digit(s[i]); i++, nexp++)
      if (ex < 1000000000000000ll) ex = ex * 10 + (s[i] - '0');  // saturates far beyond any digit count of a token
    if (nexp == 0) return false;
    e10 += eneg ? -ex : ex;
  }
  if (i != len) return false;
  if (!first) bits = 0;
  else if (e10 > 39) bits = 0x7f800000u;  // >= 10^39
  else if (e10 < -45) bits = 0;           // < 10^-46, below half the smallest subnormal
  else bits = round_decimal(w, nw, e10, first, mend);
  if (neg) bits |= 0x80000000u;
  memcpy(out, &bits, sizeof bits);
  return true;
}

// Where the four values of a point sit in a data line: n_tokens = sum of COUNT, tok[k] = token index of x, y, z,
// intensity (tok[3] = -1: no intensity field, .w = 0)
struct PcdLineLayout {
  int n_tokens;
  int tok[4];
};
enum PcdLineStatus { PCD_LINE_OK = 0, PCD_LINE_COUNT = 1, PCD_LINE_TOKEN = 2 };

// One data line from s up to its '\n' or `end` (*stop = where it stopped). xyzi[0..3] = x, y, z, intensity. A token
// count other than n_tokens is PCD_LINE_COUNT (checked first, as PCL does), a refused x / y / z / intensity token
// PCD_LINE_TOKEN; the other tokens are only counted.
B200_HD int pcd_parse_line(const char* s, const char* end, const PcdLineLayout& L, float* xyzi, const char** stop) {
  using namespace pcdparse;
  xyzi[0] = xyzi[1] = xyzi[2] = xyzi[3] = 0.0f;
  int t = 0;
  bool bad = false;
  const char* p = s;
  while (p < end && *p != '\n') {
    if (is_sep(*p)) {
      p++;
      continue;
    }
    const char* a = p;
    while (p < end && *p != '\n' && !is_sep(*p)) p++;
    if (t < L.n_tokens)
      for (int k = 0; k < 4; k++)
        if (L.tok[k] == t && !pcd_parse_float(a, (int)(p - a), &xyzi[k])) bad = true;
    t++;
  }
  *stop = p;
  if (t != L.n_tokens) return PCD_LINE_COUNT;
  return bad ? PCD_LINE_TOKEN : PCD_LINE_OK;
}

// ---- the header (host only) -------------------------------------------------------------------------------------
enum PcdData { PCD_DATA_ASCII = 0, PCD_DATA_BINARY = 1, PCD_DATA_BINARY_COMPRESSED = 2 };
struct PcdHeader {
  size_t points = 0;
  int data = -1;
  PcdLineLayout layout{0, {-1, -1, -1, -1}};
  size_t record_bytes = 0;            // sum of SIZE * COUNT
  long offset[4] = {-1, -1, -1, -1};  // byte offsets of x, y, z, intensity in a binary record
};

// text: the header lines, the DATA line included. PCD v0.7 as PCL reads it: '#' comments and empty lines skipped,
// unknown keys ignored, COUNT optional (1 each), HEIGHT optional (1), WIDTH * HEIGHT must equal POINTS when both are
// given. x, y, z required and intensity optional, each TYPE F, SIZE 4, COUNT 1. Returns false with `err` set otherwise.
inline bool pcd_parse_header(const std::string& text, PcdHeader& h, std::string& err) {
  h = PcdHeader{};
  std::vector<std::string> fields, type;
  std::vector<long long> size, count;
  long long width = -1, height = -1, points = -1;
  auto num = [](const std::string& s, long long& v) {
    if (s.empty() || s.size() > 18) return false;
    v = 0;
    for (char c : s) {
      if (!pcdparse::is_digit(c)) return false;
      v = v * 10 + (c - '0');
    }
    return true;
  };
  size_t pos = 0;
  while (pos < text.size() && h.data < 0) {
    size_t e = text.find('\n', pos);
    if (e == std::string::npos) e = text.size();
    std::vector<std::string> tk;
    for (size_t i = pos; i < e;) {
      while (i < e && (pcdparse::is_sep(text[i]) || text[i] == '\v' || text[i] == '\f')) i++;
      size_t j = i;
      while (j < e && !(pcdparse::is_sep(text[j]) || text[j] == '\v' || text[j] == '\f')) j++;
      if (j > i) tk.push_back(text.substr(i, j - i));
      i = j;
    }
    pos = e + 1;
    if (tk.empty() || tk[0][0] == '#') continue;
    const std::string& key = tk[0];
    std::vector<std::string> v(tk.begin() + 1, tk.end());
    auto nums = [&](std::vector<long long>& out) {
      out.clear();
      for (const std::string& s : v) {
        long long x;
        if (!num(s, x)) return false;
        out.push_back(x);
      }
      return true;
    };
    if (key == "FIELDS" || key == "COLUMNS") fields = v;
    else if (key == "TYPE") type = v;
    else if (key == "SIZE") {
      if (!nums(size)) return err = "SIZE: not a list of integers", false;
    } else if (key == "COUNT") {
      if (!nums(count)) return err = "COUNT: not a list of integers", false;
    } else if (key == "WIDTH" || key == "HEIGHT" || key == "POINTS") {
      long long x;
      if (v.size() != 1 || !num(v[0], x)) return err = key + ": not an integer", false;
      (key == "WIDTH" ? width : key == "HEIGHT" ? height : points) = x;
    } else if (key == "DATA") {
      const std::string d = v.empty() ? "" : v[0];
      if (d == "ascii") h.data = PCD_DATA_ASCII;
      else if (d == "binary") h.data = PCD_DATA_BINARY;
      else if (d == "binary_compressed") h.data = PCD_DATA_BINARY_COMPRESSED;
      else return err = "DATA: unknown storage '" + d + "'", false;
    }
  }
  if (h.data < 0) return err = "no DATA line", false;
  if (fields.empty()) return err = "no FIELDS", false;
  if (count.empty()) count.assign(fields.size(), 1);
  if (size.size() != fields.size() || type.size() != fields.size() || count.size() != fields.size())
    return err = "FIELDS, SIZE, TYPE and COUNT differ in length", false;
  if (height < 0) height = 1;
  if (points < 0) {
    if (width < 0) return err = "neither POINTS nor WIDTH", false;
    if (height > 0 && width > (1ll << 62) / height) return err = "WIDTH * HEIGHT too large", false;
    points = width * height;
  } else if (width >= 0 && (height == 0 ? points != 0 : (width > points / height || width * height != points))) {
    return err = "WIDTH * HEIGHT differs from POINTS", false;
  }
  const char* names[4] = {"x", "y", "z", "intensity"};
  long long tok = 0, off = 0;
  for (size_t f = 0; f < fields.size(); f++) {
    const long long sz = size[f], ct = count[f];
    if (!(sz == 1 || sz == 2 || sz == 4 || sz == 8) || ct < 1 || ct > (1 << 20) ||
        !(type[f] == "F" || type[f] == "I" || type[f] == "U"))
      return err = "field '" + fields[f] + "': bad SIZE, TYPE or COUNT", false;
    for (int k = 0; k < 4; k++) {
      if (fields[f] != names[k] || h.layout.tok[k] >= 0) continue;
      if (type[f] != "F" || sz != 4 || ct != 1)
        return err = std::string("field '") + names[k] + "' must be TYPE F, SIZE 4, COUNT 1", false;
      h.layout.tok[k] = (int)tok;
      h.offset[k] = (long)off;
    }
    tok += ct;
    off += sz * ct;
  }
  for (int k = 0; k < 3; k++)
    if (h.layout.tok[k] < 0) return err = std::string("no field '") + names[k] + "'", false;
  h.layout.n_tokens = (int)tok;
  h.record_bytes = (size_t)off;
  h.points = (size_t)points;
  return true;
}

}  // namespace b200
