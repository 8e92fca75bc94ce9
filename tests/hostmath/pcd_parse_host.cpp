// TEST INFRASTRUCTURE: the host build of the PCD token parser (csrc/pcd_parse.cuh) checked against glibc's strtof, and
// the restated PCL ASCII reader (pcd_reader_ref.hpp) that the load tests compare clouds with. Compiled with g++ (and
// OpenMP when available) by tests/test_pcd_parse_cpu.py and tests/diag/sweep_pcd_parse.py.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "../../lidarslam_ros2_b200/csrc/pcd_parse.cuh"
#include "pcd_reader_ref.hpp"

namespace {
uint32_t bits_of(float f) {
  uint32_t b;
  memcpy(&b, &f, sizeof b);
  return b;
}

// the device parser on `s` equals strtof on it (and strtof reads all of it)
bool same_as_strtof(const char* s, int len) {
  float ours;
  if (!b200::pcd_parse_float(s, len, &ours)) return false;
  char* e = nullptr;
  const float want = strtof(s, &e);
  return e == s + len && bits_of(ours) == bits_of(want);
}

// %.<prec>g of the widened float, then parsed
bool same_bits(uint32_t b, int prec) {
  float f;
  memcpy(&f, &b, sizeof f);
  char buf[48];
  const int n = snprintf(buf, sizeof buf, "%.*g", prec, (double)f);
  return same_as_strtof(buf, n);
}

long long check_strided(uint64_t lo, uint64_t count, int prec, uint32_t* first) {
  long long bad = 0;
  uint64_t first_i = UINT64_MAX;
#pragma omp parallel for schedule(static, 1 << 16) reduction(+ : bad) reduction(min : first_i)
  for (long long i = 0; i < (long long)count; i++) {
    if (!same_bits((uint32_t)(lo + (uint64_t)i), prec)) {
      bad++;
      if ((uint64_t)i < first_i) first_i = (uint64_t)i;
    }
  }
  if (bad && first) *first = (uint32_t)(lo + first_i);
  return bad;
}
}  // namespace

extern "C" {
// 1 and *bits for a token of the grammar, 0 for a refused token
int pp_parse(const char* s, int len, uint32_t* bits) {
  float f = 0;
  const bool ok = b200::pcd_parse_float(s, len, &f);
  *bits = bits_of(f);
  return ok ? 1 : 0;
}

// the restated copyStringValue<float> (the real istringstream and atof)
void pp_ref_value(const char* s, uint32_t* bits) {
  std::istringstream is;
  is.imbue(std::locale::classic());
  *bits = bits_of(pcdref::copy_string_value(s, is));
}

// glibc strtof; returns the number of characters it consumed
int pp_strtof(const char* s, uint32_t* bits) {
  char* e = nullptr;
  *bits = bits_of(strtof(s, &e));
  return (int)(e - s);
}

// every bit pattern in [lo, hi] (inclusive, hi < 2^32) through "%.<prec>g"
long long pp_check_range(uint64_t lo, uint64_t hi, int prec, uint32_t* first) { return check_strided(lo, hi - lo + 1, prec, first); }

long long pp_check_list(const uint32_t* bits, uint64_t n, int prec, uint32_t* first) {
  long long bad = 0;
  uint64_t first_i = UINT64_MAX;
#pragma omp parallel for schedule(static, 1 << 14) reduction(+ : bad) reduction(min : first_i)
  for (long long i = 0; i < (long long)n; i++) {
    if (!same_bits(bits[i], prec)) {
      bad++;
      if ((uint64_t)i < first_i) first_i = (uint64_t)i;
    }
  }
  if (bad && first) *first = bits[first_i];
  return bad;
}

// n NUL-terminated strings back to back: mismatches against strtof (*first = index of the first)
long long pp_check_strings(const char* buf, uint64_t n, uint64_t* first) {
  std::vector<const char*> at;
  at.reserve(n);
  for (uint64_t i = 0; i < n; i++) {
    at.push_back(buf);
    buf += strlen(buf) + 1;
  }
  long long bad = 0;
  uint64_t first_i = UINT64_MAX;
#pragma omp parallel for schedule(dynamic, 256) reduction(+ : bad) reduction(min : first_i)
  for (long long i = 0; i < (long long)n; i++) {
    if (!same_as_strtof(at[i], (int)strlen(at[i]))) {
      bad++;
      if ((uint64_t)i < first_i) first_i = (uint64_t)i;
    }
  }
  if (bad && first) *first = first_i;
  return bad;
}

// one data line; layout5 = {n_tokens, tok x, y, z, intensity}
int pp_parse_line(const char* s, int len, const int* layout5, float* xyzi, int* consumed) {
  const b200::PcdLineLayout L{layout5[0], {layout5[1], layout5[2], layout5[3], layout5[4]}};
  const char* stop = nullptr;
  const int r = b200::pcd_parse_line(s, s + len, L, xyzi, &stop);
  *consumed = (int)(stop - s);
  return r;
}

// out13 = points, data, n_tokens, tok x y z i, record_bytes, offset x y z i, 0. Returns 1, or 0 with the reason in err.
int pp_parse_header(const char* text, size_t len, long long* out13, char* err, size_t err_cap) {
  b200::PcdHeader h;
  std::string e;
  if (!b200::pcd_parse_header(std::string(text, len), h, e)) {
    snprintf(err, err_cap, "%s", e.c_str());
    return 0;
  }
  const long long v[13] = {(long long)h.points, h.data, h.layout.n_tokens, h.layout.tok[0], h.layout.tok[1], h.layout.tok[2],
                           h.layout.tok[3], (long long)h.record_bytes, h.offset[0], h.offset[1], h.offset[2], h.offset[3], 0};
  memcpy(out13, v, sizeof v);
  return 1;
}

// the restated PCL reader on a file: status (pcdref::READ_*), *n = POINTS, min(POINTS, capacity) points copied
int pp_read_ascii_ref(const char* path, float* xyzi, size_t capacity, size_t* n, size_t* bad_line) {
  std::ifstream fs(path, std::ios::binary);
  if (!fs.is_open()) return -10;
  std::vector<float> v;
  const int r = pcdref::read_ascii_xyzi(fs, v, bad_line);
  *n = v.size() / 4;
  if (xyzi) memcpy(xyzi, v.data(), 4 * sizeof(float) * (*n < capacity ? *n : capacity));
  return r;
}
}
