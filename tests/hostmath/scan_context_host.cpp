// CPU harness of lidarslam_ros2_b200/csrc/scan_context.hpp (the Scan Context bins, descriptors, distances, ranking and
// guess of b200sm_search_loop_place), built by tests/test_scan_context_cpu.py with g++ -ffp-contract=off as the library
// builds it.
#include <cstring>
#include <vector>

#include "../../lidarslam_ros2_b200/csrc/scan_context.hpp"

namespace {
b200::ScParams params(int num_rings, int num_sectors, double max_radius, double lidar_height) {
  b200::ScParams p;
  p.num_rings = num_rings;
  p.num_sectors = num_sectors;
  p.max_radius = max_radius;
  p.lidar_height = lidar_height;
  return p;
}
}  // namespace

extern "C" {

int sch_valid(int num_rings, int num_sectors, double max_radius, double lidar_height) {
  return b200::sc_params_valid(params(num_rings, num_sectors, max_radius, lidar_height)) ? 1 : 0;
}

// bin[i] of n points (x, y, z floats at `stride` floats per row): ring * num_sectors + sector, or -1
void sch_bins(const float* pts, long n, int stride, int num_rings, int num_sectors, double max_radius, int* bin) {
  std::vector<double> rb, su;
  b200::sc_tables(params(num_rings, num_sectors, max_radius, 0.0), rb, su);
  for (long i = 0; i < n; i++) {
    const float* p = pts + i * stride;
    bin[i] = b200::sc_bin(p[0], p[1], p[2], rb.data(), num_rings, su.data(), num_sectors);
  }
}

// the descriptor (num_rings * num_sectors floats, ring-major) and its column norms
void sch_descriptor(const float* pts, long n, int stride, int num_rings, int num_sectors, double max_radius, double lidar_height,
                    float* D, double* norms) {
  std::vector<double> rb, su;
  b200::sc_tables(params(num_rings, num_sectors, max_radius, lidar_height), rb, su);
  std::vector<uint32_t> keys((size_t)num_rings * num_sectors, 0u);
  for (long i = 0; i < n; i++) {
    const float* p = pts + i * stride;
    const int b = b200::sc_bin(p[0], p[1], p[2], rb.data(), num_rings, su.data(), num_sectors);
    if (b < 0) continue;
    const uint32_t k = b200::sc_order_key(b200::sc_value(p[2], (float)lidar_height));
    if (k > keys[b]) keys[b] = k;
  }
  for (size_t b = 0; b < keys.size(); b++) D[b] = b200::sc_from_key(keys[b]);
  for (int j = 0; j < num_sectors; j++) norms[j] = b200::sc_column_norm(D, num_rings, num_sectors, j);
}

double sch_distance_at(const float* Q, const double* nQ, const float* C, const double* nC, int num_rings, int num_sectors, int s) {
  return b200::sc_distance_at(Q, nQ, C, nC, num_rings, num_sectors, s);
}

double sch_distance(const float* Q, const double* nQ, const float* C, const double* nC, int num_rings, int num_sectors, int* shift) {
  return b200::sc_distance(Q, nQ, C, nC, num_rings, num_sectors, shift);
}

int sch_rank(const double* D, const int* ids, long n, double threshold, int* out) {
  const std::vector<int> r = b200::sc_rank(D, ids, (size_t)n, threshold);
  if (!r.empty()) std::memcpy(out, r.data(), r.size() * sizeof(int));
  return (int)r.size();
}

// P_cand, P_new row-major 4x4 doubles; G column-major floats
void sch_guess(const double* P_cand, const double* P_new, int shift, int num_sectors, float* G) {
  b200::sc_guess(P_cand, P_new, shift, num_sectors, G);
}
}
