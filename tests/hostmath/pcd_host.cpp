// TEST INFRASTRUCTURE: the host build of the PCD float formatter (csrc/pcd_format.cuh) checked against glibc's
// snprintf("%.8g"), and the restated PCL ASCII writer (pcd_writer_ref.hpp) that the encode tests compare bytes with.
// Compiled with g++ (and OpenMP when available) by tests/test_pcd_format_cpu.py and the scripts in tests/diag/.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <sstream>
#include <string>

#include "../../lidarslam_ros2_b200/csrc/pcd_format.cuh"
#include "pcd_writer_ref.hpp"

namespace {
// what writeASCII prints for one float: "nan" for a NaN, else the widened value through "%.8g"
int glibc_text(float f, char* out) {
  if (f != f) {
    memcpy(out, "nan", 3);
    return 3;
  }
  return snprintf(out, 32, "%.8g", (double)f);
}

bool same(uint32_t bits) {
  float f;
  memcpy(&f, &bits, sizeof f);
  char a[32], b[32];
  const int la = b200::pcd_format_float(f, a);
  const int lb = glibc_text(f, b);
  return la == lb && memcmp(a, b, la) == 0;
}

// mismatches among bit patterns lo + i * step (i < count); *first = the first mismatching pattern found
long long check_strided(uint64_t lo, uint64_t count, uint64_t step, uint32_t* first) {
  long long bad = 0;
  uint64_t first_i = UINT64_MAX;
#pragma omp parallel for schedule(static, 1 << 16) reduction(+ : bad) reduction(min : first_i)
  for (long long i = 0; i < (long long)count; i++) {
    if (!same((uint32_t)(lo + (uint64_t)i * step))) {
      bad++;
      if ((uint64_t)i < first_i) first_i = (uint64_t)i;
    }
  }
  if (bad && first) *first = (uint32_t)(lo + first_i * step);
  return bad;
}
}  // namespace

extern "C" {
int ph_format(float f, char* out) { return b200::pcd_format_float(f, out); }
int ph_format_line(const float* xyzi, char* out) { return b200::pcd_format_line(xyzi[0], xyzi[1], xyzi[2], xyzi[3], out); }

// every bit pattern in [lo, hi] (inclusive, hi < 2^32)
long long ph_check_range(uint64_t lo, uint64_t hi, uint32_t* first) { return check_strided(lo, hi - lo + 1, 1, first); }

long long ph_check_list(const uint32_t* bits, uint64_t n, uint32_t* first) {
  long long bad = 0;
  uint64_t first_i = UINT64_MAX;
#pragma omp parallel for schedule(static, 1 << 14) reduction(+ : bad) reduction(min : first_i)
  for (long long i = 0; i < (long long)n; i++) {
    if (!same(bits[i])) {
      bad++;
      if ((uint64_t)i < first_i) first_i = (uint64_t)i;
    }
  }
  if (bad && first) *first = bits[first_i];
  return bad;
}

// the restated writer into memory: *n_bytes = full size, min(size, capacity) bytes copied; -1 for an empty cloud
int ph_write_pcd_ascii_mem(const float* xyzi, size_t n, char* out, size_t capacity, size_t* n_bytes) {
  std::ostringstream fs;
  if (!pcdref::write_ascii_xyzi(fs, xyzi, n)) return -1;
  const std::string s = fs.str();
  *n_bytes = s.size();
  if (out) memcpy(out, s.data(), s.size() < capacity ? s.size() : capacity);
  return 0;
}

// ... and into a file, as savePCDFileASCII does (std::ofstream, binary mode); -1 empty cloud, -2 open or write failure
int ph_save_pcd_ascii(const char* path, const float* xyzi, size_t n) {
  if (n == 0) return -1;
  std::ofstream fs(path, std::ios::binary);
  if (!fs.is_open() || fs.fail()) return -2;
  pcdref::write_ascii_xyzi(fs, xyzi, n);
  fs.close();
  return fs.fail() ? -2 : 0;
}
}
