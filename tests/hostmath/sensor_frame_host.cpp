// TEST INFRASTRUCTURE: compiles the product's host frame arithmetic (csrc/sensor_frame.hpp) with g++ so that
// tests/test_sensor_frame_cpu.py can compare it bit for bit with tests/frontendref.py. Matrices are row-major.
#include "../../lidarslam_ros2_b200/csrc/sensor_frame.hpp"

using namespace b200;

extern "C" {
// n transforms: t (n x 3), q (n x 4) -> T (n x 12)
void sf_sensor_matrix(int n, const double* t, const double* q, float* T) {
  for (int i = 0; i < n; i++) sensor_matrix_f(t + 3 * i, q + 4 * i, T + 12 * i);
}
// n points (n x 3) through one 3x4 T -> out (n x 3)
void sf_transform_points(int n, const float* T, const float* p, float* out) {
  for (int i = 0; i < n; i++) transform_point_f(T, p + 3 * i, out + 3 * i);
}
void sf_odom_matrix(const double* t, const double* q, float* M) { odom_matrix_f(t, q, M); }
void sf_inverse(const float* M, float* out) { mat4_inverse_f(M, out); }
// one use_odom step: sim and previous are updated in place
void sf_odom_guess(float* sim, float* previous, const float* odom) { odom_guess_f(sim, previous, odom); }
}
