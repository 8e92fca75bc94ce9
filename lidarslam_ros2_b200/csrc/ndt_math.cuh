// Scalar control math of the NDT solver, shared by the device-side controller (ndt_solver.cu) and the host
// (initial pose/tables in engine code). __host__ __device__ so the very same functions can be unit-tested on
// the host (tests/test_hostmath.py builds them with g++); they are NOT a compute fallback — the per-point
// work exists only as CUDA kernels.
//
// Reference semantics implemented here (Thirdparty/ndt_omp_ros2/include/pclomp/ndt_omp_impl.hpp):
//   angle_tables        computeAngleDerivatives  :287-393 (incl. the +sy / -sy discrepancy :359 vs :381)
//   pose_to_matrix      Translation*AngleAxis(X)*AngleAxis(Y)*AngleAxis(Z) in float  :146-149, :811-814
//   euler_angles_012    Eigen::Matrix3f::eulerAngles(0,1,2) at :109
//   solve6              JacobiSVD<6x6>::solve(-g) at :127-129
//   mt_*                updateIntervalMT :632-670, trialValueSelectionMT :673-753, psi/dpsi ndt_omp.h:425-442
//   gauss_constants     :88-93
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define B200_HD __host__ __device__ __forceinline__
#else
#define B200_HD inline
#endif
// un-fused float multiply/add (the reference's float matrix products are not FMA-contracted; host test
// builds use -ffp-contract=off)
#if defined(__CUDA_ARCH__)
#define B200_MULF(a, b) __fmul_rn((a), (b))
#define B200_ADDF(a, b) __fadd_rn((a), (b))
#define B200_SUBF(a, b) __fsub_rn((a), (b))
#else
#define B200_MULF(a, b) ((a) * (b))
#define B200_ADDF(a, b) ((a) + (b))
#define B200_SUBF(a, b) ((a) - (b))
#endif
// the same for double: the More-Thuente arithmetic is spelled out un-fused, in the reference's evaluation order, so that
// every psi, slope and trial value the controller decides on is bitwise the reference's for the same inputs (ties
// included: once the interval has collapsed, f_t is compared with an f_l that an earlier round computed the same way)
#if defined(__CUDA_ARCH__)
#define B200_MULD(a, b) __dmul_rn((a), (b))
#define B200_ADDD(a, b) __dadd_rn((a), (b))
#define B200_SUBD(a, b) __dsub_rn((a), (b))
#else
#define B200_MULD(a, b) ((a) * (b))
#define B200_ADDD(a, b) ((a) + (b))
#define B200_SUBD(a, b) ((a) - (b))
#endif

namespace b200 {

struct GaussConsts {
  double d1, d2, d3;
};

B200_HD GaussConsts gauss_constants(double outlier_ratio, float resolution) {
  GaussConsts g;
  double c1 = 10 * (1 - outlier_ratio);
  double c2 = outlier_ratio / pow((double)resolution, 3);
  g.d3 = -log(c2);
  g.d1 = -log(c1 + c2) - g.d3;
  g.d2 = -2 * log((-log(c1 * exp(-0.5) + c2) - g.d3) / g.d1);
  return g;
}

// jang: 8 rows x 3 (f32 table), hang: 15 rows x 3 (f32 table, row 6 = d1 keeps +sy).
// jd/hd (optional, may be nullptr): the f64 vectors used by computeHessian (row 6 of hd has -sy).
B200_HD void angle_tables(const double* p, float* jang, float* hang, double* jd, double* hd) {
  double cx, cy, cz, sx, sy, sz;
  if (fabs(p[3]) < 10e-5) { cx = 1.0; sx = 0.0; } else { cx = cos(p[3]); sx = sin(p[3]); }
  if (fabs(p[4]) < 10e-5) { cy = 1.0; sy = 0.0; } else { cy = cos(p[4]); sy = sin(p[4]); }
  if (fabs(p[5]) < 10e-5) { cz = 1.0; sz = 0.0; } else { cz = cos(p[5]); sz = sin(p[5]); }
  double J[24], H[45];
  J[0] = -sx * sz + cx * sy * cz;  J[1] = -sx * cz - cx * sy * sz;  J[2] = -cx * cy;
  J[3] = cx * sz + sx * sy * cz;   J[4] = cx * cz - sx * sy * sz;   J[5] = -sx * cy;
  J[6] = -sy * cz;                 J[7] = sy * sz;                  J[8] = cy;
  J[9] = sx * cy * cz;             J[10] = -sx * cy * sz;           J[11] = sx * sy;
  J[12] = -cx * cy * cz;           J[13] = cx * cy * sz;            J[14] = -cx * sy;
  J[15] = -cy * sz;                J[16] = -cy * cz;                J[17] = 0;
  J[18] = cx * cz - sx * sy * sz;  J[19] = -cx * sz - sx * sy * cz; J[20] = 0;
  J[21] = sx * cz + cx * sy * sz;  J[22] = cx * sy * cz - sx * sz;  J[23] = 0;

  H[0] = -cx * sz - sx * sy * cz;  H[1] = -cx * cz + sx * sy * sz;  H[2] = sx * cy;     // a2
  H[3] = -sx * sz + cx * sy * cz;  H[4] = -cx * sy * sz - sx * cz;  H[5] = -cx * cy;    // a3
  H[6] = cx * cy * cz;             H[7] = -cx * cy * sz;            H[8] = cx * sy;     // b2
  H[9] = sx * cy * cz;             H[10] = -sx * cy * sz;           H[11] = sx * sy;    // b3
  H[12] = -sx * cz - cx * sy * sz; H[13] = sx * sz - cx * sy * cz;  H[14] = 0;          // c2
  H[15] = cx * cz - sx * sy * sz;  H[16] = -sx * sy * cz - cx * sz; H[17] = 0;          // c3
  H[18] = -cy * cz;                H[19] = cy * sz;                 H[20] = -sy;        // d1 (f64: -sy)
  H[21] = -sx * sy * cz;           H[22] = sx * sy * sz;            H[23] = sx * cy;    // d2
  H[24] = cx * sy * cz;            H[25] = -cx * sy * sz;           H[26] = -cx * cy;   // d3
  H[27] = sy * sz;                 H[28] = sy * cz;                 H[29] = 0;          // e1
  H[30] = -sx * cy * sz;           H[31] = -sx * cy * cz;           H[32] = 0;          // e2
  H[33] = cx * cy * sz;            H[34] = cx * cy * cz;            H[35] = 0;          // e3
  H[36] = -cy * cz;                H[37] = cy * sz;                 H[38] = 0;          // f1
  H[39] = -cx * sz - sx * sy * cz; H[40] = -cx * cz + sx * sy * sz; H[41] = 0;          // f2
  H[42] = -sx * sz + cx * sy * cz; H[43] = -cx * sy * sz - sx * cz; H[44] = 0;          // f3
  for (int k = 0; k < 24; k++) {
    jang[k] = (float)J[k];
    if (jd) jd[k] = J[k];
  }
  for (int k = 0; k < 45; k++) {
    hang[k] = (float)H[k];
    if (hd) hd[k] = H[k];
  }
  hang[20] = (float)sy;  // the live f32 table has +sy (ndt_omp_impl.hpp:381)
}

// The same 69 table entries (24 of J then 45 of H, f64 values) in coded form, so that independent lanes can evaluate
// them: each entry is sign0 * f[a0]*f[a1]*f[a2] + sign1 * f[b0]*f[b1]*f[b2] with f = {sx,cx,sy,cy,sz,cz,1}
// (angle_table_code.inc, generated by tools/gen_angle_table_code.py from the formulas above).
#if defined(__CUDACC__)
__device__ __constant__
#endif
    static const unsigned kAngleTableCode[69] = {
#include "angle_table_code.inc"
};

B200_HD double angle_table_term(unsigned code, const double* f) {
  const unsigned sign = code & 3u;
  if (sign == 0u) return 0.0;
  const double v = f[(code >> 2) & 7u] * f[(code >> 5) & 7u] * f[(code >> 8) & 7u];
  return sign == 2u ? -v : v;
}
// f64 value of entry e (0..23: J, 24..68: H with the f64 sign convention, i.e. d1.z = -sy)
B200_HD double angle_table_entry(unsigned word, const double* f) {
  return angle_table_term(word & 0x7ffu, f) + angle_table_term((word >> 11) & 0x7ffu, f);
}

// Symmetric 6x6 solve  H x = b  by LDL^T elimination on the UPPER triangle, no pivoting, entirely in registers:
// U[r][c] (c >= r) holds the upper triangle of H on entry. Returns false when a pivot collapses relative to the largest
// diagonal entry or anything is non-finite (the caller then takes the pivoted-LU / SVD path that reproduces
// JacobiSVD::solve, ndt_omp_impl.hpp:127-129). Straight-line code: the controller warp of the solver executes it once per
// Newton iteration (ndt_solver.cu, controller_fast).
B200_HD bool ldlt_solve6_upper(double (&U)[6][6], double (&rhs)[6], double (&x)[6]) {
  double dmax = 0.0;
#pragma unroll
  for (int r = 0; r < 6; r++) dmax = fmax(dmax, fabs(U[r][r]));
  bool ok = dmax > 0.0 && dmax <= 1.7e308;
  double inv[6];
#pragma unroll
  for (int k = 0; k < 6; k++) {
    ok = ok && (fabs(U[k][k]) > 1e-10 * dmax);  // false for NaN
    inv[k] = 1.0 / U[k][k];
#pragma unroll
    for (int r = k + 1; r < 6; r++) {
      const double l = U[k][r] * inv[k];
#pragma unroll
      for (int c = r; c < 6; c++) U[r][c] = fma(-l, U[k][c], U[r][c]);
      rhs[r] = fma(-l, rhs[k], rhs[r]);
    }
  }
  if (!ok) return false;
#pragma unroll
  for (int k = 5; k >= 0; k--) {
    double t = rhs[k];
#pragma unroll
    for (int c = k + 1; c < 6; c++) t = fma(-U[k][c], x[c], t);
    x[k] = t * inv[k];
  }
  return true;
}

// sin/cos of a moderate angle (|x| << 1e5; Euler angles live in [-pi, pi]) to < 1 ulp: Cody-Waite reduction by pi/2
// and the fdlibm kernel polynomials. Compact on purpose: the device-side controller is instruction-fetch bound (ndt_solver.cu).
B200_HD void sincos_compact(double x, double* s_out, double* c_out) {
  const double n = rint(x * 6.36619772367581382433e-01);
  double r = fma(-n, 1.57079632673412561417e+00, x);
  r = fma(-n, 6.07710050650619224932e-11, r);
  r = fma(-n, 2.02226624879595063154e-21, r);
  const double z = r * r;
  double ps = 1.58969099521155010221e-10;
  ps = fma(ps, z, -2.50507602534068634195e-08);
  ps = fma(ps, z, 2.75573137070700676789e-06);
  ps = fma(ps, z, -1.98412698298579493134e-04);
  ps = fma(ps, z, 8.33333333332248946124e-03);
  ps = fma(ps, z, -1.66666666666666324348e-01);
  const double sn = fma(r * z, ps, r);
  double pc = -1.13596475577881948265e-11;
  pc = fma(pc, z, 2.08757232129817482790e-09);
  pc = fma(pc, z, -2.75573143513906633035e-07);
  pc = fma(pc, z, 2.48015872894767294178e-05);
  pc = fma(pc, z, -1.38888888888741095749e-03);
  pc = fma(pc, z, 4.16666666666666019037e-02);
  const double cs = fma(z * z, pc, fma(-0.5, z, 1.0));
  const int q = ((int)n) & 3;
  const double s0 = (q & 1) ? cs : sn, c0 = (q & 1) ? sn : cs;
  *s_out = (q == 2 || q == 3) ? -s0 : s0;
  *c_out = (q == 1 || q == 2) ? -c0 : c0;
}

// T: 3x4 row-major float
B200_HD void pose_to_matrix(const double* p, float* T) {
  float a = (float)p[3], b = (float)p[4], c = (float)p[5];
  float cx = cosf(a), sx = sinf(a), cy = cosf(b), sy = sinf(b), cz = cosf(c), sz = sinf(c);
  // A = Rx * Ry, R = A * Rz, float products in the order a dense 3x3 product forms them
  float A[9];
  A[0] = cy;                  A[1] = 0.0f;  A[2] = sy;
  A[3] = sx * sy;             A[4] = cx;    A[5] = -sx * cy;
  A[6] = -cx * sy;            A[7] = sx;    A[8] = cx * cy;
  for (int r = 0; r < 3; r++) {
    float a0 = A[r * 3 + 0], a1 = A[r * 3 + 1], a2 = A[r * 3 + 2];
    T[r * 4 + 0] = B200_ADDF(B200_MULF(a0, cz), B200_MULF(a1, sz));
    T[r * 4 + 1] = B200_ADDF(B200_MULF(a0, -sz), B200_MULF(a1, cz));
    T[r * 4 + 2] = a2;
    T[r * 4 + 3] = (float)p[r];
  }
}

// m: 3x3 row-major float
B200_HD void euler_angles_012(const float* m, float* out) {
  const float kPi = 3.14159265358979323846f;
  float r0 = atan2f(m[5], m[8]);
  float c2 = sqrtf(m[0] * m[0] + m[1] * m[1]);
  float r1;
  if (r0 > 0.0f) {
    r0 -= kPi;
    r1 = atan2f(-m[2], -c2);
  } else {
    r1 = atan2f(-m[2], c2);
  }
  float s1 = sinf(r0), c1 = cosf(r0);
  float r2 = atan2f(s1 * m[6] - c1 * m[3], c1 * m[4] - s1 * m[7]);
  out[0] = -r0;
  out[1] = -r1;
  out[2] = -r2;
}

// Minimum-norm solve of the symmetric 6x6 system H x = b, equivalent to JacobiSVD(H).solve(b).
// Fast path: LU with partial pivoting (well-conditioned H — every practical case). If a pivot collapses
// (rank deficiency, where the SVD's truncation matters) fall back to a one-sided Jacobi SVD.
B200_HD void solve6_svd(const double* Hin, const double* b, double* x) {
  double W[36], V[36];
  for (int i = 0; i < 36; i++) { W[i] = Hin[i]; V[i] = 0; }
  for (int i = 0; i < 6; i++) V[i * 6 + i] = 1;
  const double eps = 2.220446049250313e-16;
  for (int sweep = 0; sweep < 60; sweep++) {
    bool rotated = false;
    for (int p = 0; p < 5; p++)
      for (int q = p + 1; q < 6; q++) {
        double al = 0, be = 0, ga = 0;
        for (int k = 0; k < 6; k++) {
          al += W[k * 6 + p] * W[k * 6 + p];
          be += W[k * 6 + q] * W[k * 6 + q];
          ga += W[k * 6 + p] * W[k * 6 + q];
        }
        if (ga == 0.0 || fabs(ga) <= eps * sqrt(al * be)) continue;
        rotated = true;
        double zeta = (be - al) / (2.0 * ga);
        double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
        for (int k = 0; k < 6; k++) {
          double wp = W[k * 6 + p], wq = W[k * 6 + q];
          W[k * 6 + p] = c * wp - s * wq;
          W[k * 6 + q] = s * wp + c * wq;
          double vp = V[k * 6 + p], vq = V[k * 6 + q];
          V[k * 6 + p] = c * vp - s * vq;
          V[k * 6 + q] = s * vp + c * vq;
        }
      }
    if (!rotated) break;
  }
  double smax = 0, sv[6];
  for (int j = 0; j < 6; j++) {
    double s = 0;
    for (int k = 0; k < 6; k++) s += W[k * 6 + j] * W[k * 6 + j];
    sv[j] = sqrt(s);
    if (sv[j] > smax) smax = sv[j];
  }
  const double thr = smax * 6.0 * eps;
  for (int i = 0; i < 6; i++) x[i] = 0;
  for (int j = 0; j < 6; j++) {
    if (!(sv[j] > thr)) continue;
    double d = 0;
    for (int k = 0; k < 6; k++) d += W[k * 6 + j] * b[k];  // U_j . b * sv[j]
    d /= sv[j] * sv[j];
    for (int k = 0; k < 6; k++) x[k] += d * V[k * 6 + j];
  }
}

B200_HD void solve6(const double* H, const double* b, double* x) {
  double A[36], y[6];
  double amax = 0;
  bool finite = true;
  for (int i = 0; i < 36; i++) {
    A[i] = H[i];
    double a = fabs(H[i]);
    if (!(a == a) || a > 1.7e308) finite = false;
    if (a > amax) amax = a;
  }
  for (int i = 0; i < 6; i++) y[i] = b[i];
  if (!finite) {  // NaN/inf propagate like the SVD would (delta_p_norm != delta_p_norm branch, :134-139)
    for (int i = 0; i < 6; i++) x[i] = NAN;
    return;
  }
  bool ok = amax > 0;
  for (int k = 0; k < 6 && ok; k++) {
    int piv = k;
    double pm = fabs(A[k * 6 + k]);
    for (int r = k + 1; r < 6; r++)
      if (fabs(A[r * 6 + k]) > pm) { pm = fabs(A[r * 6 + k]); piv = r; }
    if (pm <= 1e-13 * amax) { ok = false; break; }
    if (piv != k) {
      for (int c = 0; c < 6; c++) { double t = A[k * 6 + c]; A[k * 6 + c] = A[piv * 6 + c]; A[piv * 6 + c] = t; }
      double t = y[k]; y[k] = y[piv]; y[piv] = t;
    }
    double inv = 1.0 / A[k * 6 + k];
    for (int r = k + 1; r < 6; r++) {
      double f = A[r * 6 + k] * inv;
      for (int c = k + 1; c < 6; c++) A[r * 6 + c] -= f * A[k * 6 + c];
      y[r] -= f * y[k];
    }
  }
  if (!ok) {
    solve6_svd(H, b, x);
    return;
  }
  for (int k = 5; k >= 0; k--) {
    double s = y[k];
    for (int c = k + 1; c < 6; c++) s -= A[k * 6 + c] * x[c];
    x[k] = s / A[k * 6 + k];
  }
}

// ---- More-Thuente helpers -------------------------------------------------------------------------------
B200_HD double mt_psi(double a, double f_a, double f_0, double g_0, double mu) {
  return B200_SUBD(B200_SUBD(f_a, f_0), B200_MULD(B200_MULD(mu, g_0), a));
}
B200_HD double mt_dpsi(double g_a, double g_0, double mu) { return B200_SUBD(g_a, B200_MULD(mu, g_0)); }

B200_HD bool mt_update_interval(double& a_l, double& f_l, double& g_l, double& a_u, double& f_u, double& g_u,
                                double a_t, double f_t, double g_t) {
  if (f_t > f_l) {
    a_u = a_t; f_u = f_t; g_u = g_t;
    return false;
  }
  if (g_t * (a_l - a_t) > 0) {
    a_l = a_t; f_l = f_t; g_l = g_t;
    return false;
  }
  if (g_t * (a_l - a_t) < 0) {
    a_u = a_l; f_u = f_l; g_u = g_l;
    a_l = a_t; f_l = f_t; g_l = g_t;
    return false;
  }
  return true;
}

B200_HD double mt_cubic_min(double a_l, double f_l, double g_l, double a_t, double f_t, double g_t) {
  double z = B200_SUBD(B200_SUBD(B200_MULD(3.0, B200_SUBD(f_t, f_l)) / B200_SUBD(a_t, a_l), g_t), g_l);
  double w = sqrt(B200_SUBD(B200_MULD(z, z), B200_MULD(g_t, g_l)));
  return B200_ADDD(a_l, B200_MULD(B200_SUBD(a_t, a_l), B200_SUBD(B200_SUBD(w, g_l), z)) /
                            B200_ADDD(B200_SUBD(g_t, g_l), B200_MULD(2.0, w)));
}

// a_l - (a_l - a_t) / (g_l - g_t) * g_l
B200_HD double mt_secant(double a_l, double g_l, double a_t, double g_t) {
  return B200_SUBD(a_l, B200_MULD(B200_SUBD(a_l, a_t) / B200_SUBD(g_l, g_t), g_l));
}

B200_HD double mt_trial_value(double a_l, double f_l, double g_l, double a_u, double f_u, double g_u, double a_t,
                              double f_t, double g_t) {
  if (f_t > f_l) {  // case 1
    double a_c = mt_cubic_min(a_l, f_l, g_l, a_t, f_t, g_t);
    double a_q = B200_SUBD(a_l, B200_MULD(B200_MULD(0.5, B200_SUBD(a_l, a_t)), g_l) /
                                    B200_SUBD(g_l, B200_SUBD(f_l, f_t) / B200_SUBD(a_l, a_t)));
    return (fabs(B200_SUBD(a_c, a_l)) < fabs(B200_SUBD(a_q, a_l))) ? a_c : B200_MULD(0.5, B200_ADDD(a_q, a_c));
  }
  if (B200_MULD(g_t, g_l) < 0) {  // case 2
    double a_c = mt_cubic_min(a_l, f_l, g_l, a_t, f_t, g_t);
    double a_s = mt_secant(a_l, g_l, a_t, g_t);
    return (fabs(B200_SUBD(a_c, a_t)) >= fabs(B200_SUBD(a_s, a_t))) ? a_c : a_s;
  }
  if (fabs(g_t) <= fabs(g_l)) {  // case 3
    double a_c = mt_cubic_min(a_l, f_l, g_l, a_t, f_t, g_t);
    double a_s = mt_secant(a_l, g_l, a_t, g_t);
    double a_n = (fabs(B200_SUBD(a_c, a_t)) < fabs(B200_SUBD(a_s, a_t))) ? a_c : a_s;
    const double a_far = B200_ADDD(a_t, B200_MULD(0.66, B200_SUBD(a_u, a_t)));
    if (a_t > a_l) return fmin(a_far, a_n);
    return fmax(a_far, a_n);
  }
  return mt_cubic_min(a_u, f_u, g_u, a_t, f_t, g_t);  // case 4
}

}  // namespace b200
