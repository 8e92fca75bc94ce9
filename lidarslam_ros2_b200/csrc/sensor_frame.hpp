// Frame arithmetic of the frontend's cloud callback on the host, in float: the sensor-to-robot matrix of
// tf2::doTransform(PointCloud2) (scanmatcher_component.cpp:188-199) and the use_odom initial guess of receiveCloud
// (:333-348). Header-only and free of CUDA so that a CPU harness (tests/hostmath/sensor_frame_host.cpp) compiles it with
// g++ and compares it bit for bit with the float32 restatement in tests/frontendref.py.
//
// Every expression is written in the order it is evaluated, one float rounding per operation. It must be compiled
// without floating-point contraction (build.sh passes -ffp-contract=off for scanmatcher.cu; baseline x86-64 has no FMA).
#pragma once
#include "pose_graph.hpp"

namespace b200 {

// tf2_sensor_msgs' doTransform: Eigen::Translation3f(t) * Eigen::Quaternionf(w, x, y, z), the doubles of the
// TransformStamped cast to float first, then QuaternionBase::toRotationMatrix evaluated in float. The quaternion is used
// as given (tf2 does not normalise it). T: 3x4 row-major.
inline void sensor_matrix_f(const double* t3, const double* q_xyzw, float* T) {
  const float x = (float)q_xyzw[0], y = (float)q_xyzw[1], z = (float)q_xyzw[2], w = (float)q_xyzw[3];
  const float tx = 2.0f * x, ty = 2.0f * y, tz = 2.0f * z;
  const float twx = tx * w, twy = ty * w, twz = tz * w;
  const float txx = tx * x, txy = ty * x, txz = tz * x;
  const float tyy = ty * y, tyz = tz * y, tzz = tz * z;
  T[0] = 1.0f - (tyy + tzz); T[1] = txy - twz;          T[2] = txz + twy;           T[3] = (float)t3[0];
  T[4] = txy + twz;          T[5] = 1.0f - (txx + tzz); T[6] = tyz - twx;           T[7] = (float)t3[1];
  T[8] = txz - twy;          T[9] = tyz + twx;          T[10] = 1.0f - (txx + tyy); T[11] = (float)t3[2];
}

// Affine3f * Vector3f for a fixed 3x3: ((r0 x + r1 y) + r2 z) + t per row — transform_point of common.cuh on the host,
// bitwise what the unpack pass stores for the same record.
inline void transform_point_f(const float* T, const float* p, float* out) {
  const float x = p[0], y = p[1], z = p[2];
  out[0] = ((T[0] * x + T[1] * y) + T[2] * z) + T[3];
  out[1] = ((T[4] * x + T[5] * y) + T[6] * z) + T[7];
  out[2] = ((T[8] * x + T[9] * y) + T[10] * z) + T[11];
}

// tf2::transformToEigen(odom_trans).matrix().cast<float>(): Translation3d * Quaterniond in double, then each entry cast.
// M: 4x4 row-major.
inline void odom_matrix_f(const double* t3, const double* q_xyzw, float* M) {
  double D[16];
  pose_to_matrix_d(t3, q_xyzw, D);
  for (int k = 0; k < 16; k++) M[k] = (float)D[k];
}

// C = A * B, 4x4 row-major float, each entry ((a0 b0 + a1 b1) + a2 b2) + a3 b3
inline void mat4_mul_f(const float* A, const float* B, float* C) {
  for (int r = 0; r < 4; r++)
    for (int c = 0; c < 4; c++)
      C[r * 4 + c] = ((A[r * 4] * B[c] + A[r * 4 + 1] * B[4 + c]) + A[r * 4 + 2] * B[8 + c]) + A[r * 4 + 3] * B[12 + c];
}

// General 4x4 inverse by Laplace expansion in 2x2 minors: s0..s5 are the minors of rows 0-1, c0..c5 those of rows 2-3,
//   det = ((((s0 c5 - s1 c4) + s2 c3) + s3 c2) - s4 c1) + s5 c0,  inv = adj(M) * (1 / det),
// every adjugate entry a signed sum of three products, left to right. (Eigen 3.4 inverts a 4x4 float with an SSE
// cofactor kernel whose association cannot be consulted here; the two differ by a few ulp, see DESIGN.md §3.)
inline void mat4_inverse_f(const float* m, float* o) {
  const float a00 = m[0], a01 = m[1], a02 = m[2], a03 = m[3];
  const float a10 = m[4], a11 = m[5], a12 = m[6], a13 = m[7];
  const float a20 = m[8], a21 = m[9], a22 = m[10], a23 = m[11];
  const float a30 = m[12], a31 = m[13], a32 = m[14], a33 = m[15];
  const float s0 = a00 * a11 - a10 * a01, s1 = a00 * a12 - a10 * a02, s2 = a00 * a13 - a10 * a03;
  const float s3 = a01 * a12 - a11 * a02, s4 = a01 * a13 - a11 * a03, s5 = a02 * a13 - a12 * a03;
  const float c5 = a22 * a33 - a32 * a23, c4 = a21 * a33 - a31 * a23, c3 = a21 * a32 - a31 * a22;
  const float c2 = a20 * a33 - a30 * a23, c1 = a20 * a32 - a30 * a22, c0 = a20 * a31 - a30 * a21;
  const float det = ((((s0 * c5 - s1 * c4) + s2 * c3) + s3 * c2) - s4 * c1) + s5 * c0;
  const float inv = 1.0f / det;
  o[0] = (a11 * c5 - a12 * c4 + a13 * c3) * inv;
  o[1] = (-a01 * c5 + a02 * c4 - a03 * c3) * inv;
  o[2] = (a31 * s5 - a32 * s4 + a33 * s3) * inv;
  o[3] = (-a21 * s5 + a22 * s4 - a23 * s3) * inv;
  o[4] = (-a10 * c5 + a12 * c2 - a13 * c1) * inv;
  o[5] = (a00 * c5 - a02 * c2 + a03 * c1) * inv;
  o[6] = (-a30 * s5 + a32 * s2 - a33 * s1) * inv;
  o[7] = (a20 * s5 - a22 * s2 + a23 * s1) * inv;
  o[8] = (a10 * c4 - a11 * c2 + a13 * c0) * inv;
  o[9] = (-a00 * c4 + a01 * c2 - a03 * c0) * inv;
  o[10] = (a30 * s4 - a31 * s2 + a33 * s0) * inv;
  o[11] = (-a20 * s4 + a21 * s2 - a23 * s0) * inv;
  o[12] = (-a10 * c3 + a11 * c1 - a12 * c0) * inv;
  o[13] = (a00 * c3 - a01 * c1 + a02 * c0) * inv;
  o[14] = (-a30 * s3 + a31 * s1 - a32 * s0) * inv;
  o[15] = (a20 * s3 - a21 * s1 + a22 * s0) * inv;
}

// use_odom (sm.cpp:342-347): when previous_odom != Identity (all 16 entries compared exactly),
// sim = (sim * previous_odom^-1) * odom; then previous_odom = odom. All 4x4 row-major float.
inline void odom_guess_f(float* sim, float* previous_odom, const float* odom) {
  bool identity = true;
  for (int k = 0; k < 16; k++) identity = identity && previous_odom[k] == ((k % 5) == 0 ? 1.0f : 0.0f);
  if (!identity) {
    float inv[16], tmp[16];
    mat4_inverse_f(previous_odom, inv);
    mat4_mul_f(sim, inv, tmp);
    mat4_mul_f(tmp, odom, sim);
  }
  for (int k = 0; k < 16; k++) previous_odom[k] = odom[k];
}

}  // namespace b200
