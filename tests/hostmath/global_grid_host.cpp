// CPU harness of lidarslam_ros2_b200/csrc/global_grid.hpp (the hypothesis grid and the top-k choice of
// b200sm_localize_global), built by tests/test_global_grid_cpu.py with g++ -ffp-contract=off as the library builds it.
#include <cstring>

#include "../../lidarslam_ros2_b200/csrc/global_grid.hpp"

extern "C" {

long long gg_count(double radius, double step, int yaw_steps, int top_k) {
  return b200::global_grid_count(radius, step, yaw_steps, top_k);
}

// the poses of a valid spec (16 floats each, column-major); returns the number of hypotheses
long long gg_build(const double* position, const double* quat, double radius, double step, int yaw_steps, float* out,
                   long long capacity) {
  std::vector<float> poses;
  b200::global_grid_build(position, quat, radius, step, yaw_steps, poses);
  const long long n = (long long)(poses.size() / 16);
  const long long m = n < capacity ? n : capacity;
  if (m > 0) std::memcpy(out, poses.data(), (size_t)m * 16 * sizeof(float));
  return n;
}

int gg_select(const double* scores, long long n, int top_k, int* out) {
  const std::vector<int> top = b200::global_select_top_k(scores, n, top_k);
  if (!top.empty()) std::memcpy(out, top.data(), top.size() * sizeof(int));
  return (int)top.size();
}
}
