// The hypothesis grid of global localisation (b200sm_localize_global) and the choice of the hypotheses it refines.
// Host code, header-only and free of CUDA so that a CPU harness (tests/hostmath/global_grid_host.cpp) compiles it with g++;
// built -ffp-contract=off (every product and sum below is rounded on its own, as a float64 replay evaluates it).
#pragma once
#include <algorithm>
#include <cmath>
#include <numeric>
#include <vector>

#include "pose_graph.hpp"

namespace b200 {

constexpr double GLOBAL_MAX_HALF_WIDTH = 4096;          // K = floor(radius / step) at most
constexpr long long GLOBAL_MAX_HYPOTHESES = 1LL << 24;
constexpr int GLOBAL_MAX_YAW_STEPS = 4096;
constexpr int GLOBAL_MAX_TOP_K = 1024;

// Positions of the grid: (i, j) for j = -K-1 .. K+1 (outer), i = -K-1 .. K+1 (inner), kept when a * a + b * b <= r * r with
// a = (double)i * step, b = (double)j * step. Returns the number of kept positions (and appends them to `ij` when given), or
// -1 when a field is invalid or K > GLOBAL_MAX_HALF_WIDTH.
inline long long global_grid_positions(double radius, double step, std::vector<int>* ij = nullptr) {
  if (!std::isfinite(radius) || !std::isfinite(step) || !(radius >= 0) || !(step > 0)) return -1;
  const double kd = std::floor(radius / step);
  if (!(kd <= GLOBAL_MAX_HALF_WIDTH)) return -1;
  const int K = (int)kd;
  const double r2 = radius * radius;
  long long n = 0;
  for (int j = -K - 1; j <= K + 1; j++) {
    const double b = (double)j * step;
    const double bb = b * b;
    for (int i = -K - 1; i <= K + 1; i++) {
      const double a = (double)i * step;
      if (a * a + bb <= r2) {
        n++;
        if (ij) {
          ij->push_back(i);
          ij->push_back(j);
        }
      }
    }
  }
  return n;
}

// Number of hypotheses of a search (positions x yaw_steps), or -1 when the spec is invalid: radius finite >= 0, step finite
// > 0, 1 <= yaw_steps <= 4096, 1 <= top_k <= 1024, K <= 4096 and at most 2^24 hypotheses.
inline long long global_grid_count(double radius, double step, int yaw_steps, int top_k) {
  if (yaw_steps < 1 || yaw_steps > GLOBAL_MAX_YAW_STEPS || top_k < 1 || top_k > GLOBAL_MAX_TOP_K) return -1;
  const long long p = global_grid_positions(radius, step);
  if (p < 0 || p * yaw_steps > GLOBAL_MAX_HYPOTHESES) return -1;
  return p * yaw_steps;
}

// The rotations Rz(theta_m) * R0 for m = 0 .. yaw_steps - 1, row-major 3x3 in double: R0 the rotation of the row-major M,
// theta_m = 2 pi m / yaw_steps, products summed left to right. b200sm_localize_global and b200sm_relocalize share them.
inline void global_yaw_rotations(const double* M, int yaw_steps, std::vector<double>& rot) {
  rot.assign((size_t)yaw_steps * 9, 0.0);
  for (int m = 0; m < yaw_steps; m++) {
    const double th = 2.0 * 3.141592653589793 * (double)m / (double)yaw_steps;  // math.pi
    const double c = std::cos(th), s = std::sin(th);
    const double Rz[9] = {c, -s, 0.0, s, c, 0.0, 0.0, 0.0, 1.0};
    for (int r = 0; r < 3; r++)
      for (int col = 0; col < 3; col++)
        rot[(size_t)m * 9 + r * 3 + col] = Rz[r * 3 + 0] * M[0 * 4 + col] + Rz[r * 3 + 1] * M[1 * 4 + col] + Rz[r * 3 + 2] * M[2 * 4 + col];
  }
}

// The hypotheses of a valid spec around the pose (position, quaternion x y z w), 16 floats each, column-major. Hypothesis
// k = position_index * yaw_steps + m: translation (cx + a, cy + b, z0), rotation global_yaw_rotations' R_m with R0 the
// rotation of pose_to_matrix_d (the session's sim_trans), cast to float.
inline void global_grid_build(const double* position, const double* quat, double radius, double step, int yaw_steps,
                              std::vector<float>& poses) {
  std::vector<int> ij;
  const long long n_pos = global_grid_positions(radius, step, &ij);
  poses.assign((size_t)(n_pos < 0 ? 0 : n_pos) * (size_t)yaw_steps * 16, 0.0f);
  double M[16];
  pose_to_matrix_d(position, quat, M);
  std::vector<double> rot;
  global_yaw_rotations(M, yaw_steps, rot);
  for (long long q = 0; q < n_pos; q++) {
    const double t[3] = {M[3] + (double)ij[2 * q] * step, M[7] + (double)ij[2 * q + 1] * step, M[11]};
    for (int m = 0; m < yaw_steps; m++) {
      float* P = poses.data() + ((size_t)q * yaw_steps + m) * 16;
      const double* R = rot.data() + (size_t)m * 9;
      for (int r = 0; r < 3; r++) {
        for (int col = 0; col < 3; col++) P[col * 4 + r] = (float)R[r * 3 + col];
        P[12 + r] = (float)t[r];
      }
      P[15] = 1.0f;
    }
  }
}

// The top_k highest scores in descending order, the lower index first among equal scores: min(top_k, n) indices.
inline std::vector<int> global_select_top_k(const double* scores, long long n, int top_k) {
  std::vector<int> idx((size_t)n);
  std::iota(idx.begin(), idx.end(), 0);
  const size_t k = (size_t)std::min<long long>(top_k, n);
  std::partial_sort(idx.begin(), idx.begin() + k, idx.end(),
                    [&](int a, int b) { return scores[a] > scores[b] || (scores[a] == scores[b] && a < b); });
  idx.resize(k);
  return idx;
}

}  // namespace b200
