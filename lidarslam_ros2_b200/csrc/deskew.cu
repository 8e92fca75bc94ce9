// IMU de-skew kernels (SURVEY.md §8f row 4) — LidarUndistortion::adjustDistortion, lidar_undistortion.hpp:110-226.
//
// The reference walks the points of a scan in firing order and carries two pieces of state from point to point: the
// `half_passed` flag of the azimuth unwrapping and the IMU ring pointer `imu_ptr_last_iter_` (with a `continue` that
// skips the carry for points outside the IMU coverage). Both have an exact data-parallel form (proven equal to the
// sequential loop on the CPU, oracle/deskew.py + tests/test_deskew_oracle.py):
//   * half_passed is set by the FIRST point whose pre-half-turn azimuth is more than pi past the start  -> atomicMin;
//   * the carried pointer is the running maximum, over the previous NON-skipped points, of an independent per-point
//     lower bound into the ring (first sample later than the point's time stamp)  -> exclusive prefix-max scan, repeated
//     until the set of skipped points is stable (one pass when the IMU covers the scan). The lower bound uses the
//     walk's own test `t < time`, so a NaN time (a NaN ray) carries the newest sample as in the reference. The form is
//     exact only while the stamps of the ring window never decrease; when the IMU clock steps back inside the window
//     (checked on the host) one thread of deskew_scan runs the walk literally instead;
//   * interpolation of roll/pitch/yaw/shift/velocity and the rigid correction are independent per point.
// Kernels: deskew_orient (azimuth, first-index reduction) -> deskew_time (relative time, ring lower bound) ->
// deskew_scan (one CTA: prefix-max fix point, carried pointers, start pose) -> deskew_apply (per-point correction).
// Float semantics follow the C++ (float members, double literals promote); trigonometry is evaluated in double and
// rounded to float, i.e. the correctly rounded value of std::atan2(float, float) / std::sin(float) to within double
// rounding — agreement with a glibc build is to float rounding, not bit-exact (DESIGN.md).
#include "deskew.hpp"

#include <cmath>
#include <cstring>

namespace b200 {

namespace {

constexpr double PI_D = 3.14159265358979323846;  // M_PI

struct DeskewParams {
  float start_ori, end_ori, ori_diff;
  double scan_period, scan_time;
  int base, span;  // ring positions 0..span map to ring indices (base + pos) % IMU_QUE, in the walk's order
  int monotone;    // the stamps at positions 0..span never decrease (the binary search and the fix point are exact)
};

struct DeskewShared {  // small device-side block shared by the kernels of one call
  int k_first;          // first index that sets half_passed (n if none)
  int ptr_front_pos;    // ring position of imu_ptr_front_ after the last point
  int ptr_iter_pos;     // ring position carried past the last non-skipped point (-1: none)
  int ok0;              // point 0 was not skipped: the start pose below is valid
  int rounds;           // passes of the fix point (0: the literal walk ran instead)
  float r_s_i[9];       // r_c.inverse() of the first point (row-major)
  float shift0[3], velo0[3];
};
constexpr int DESKEW_SHARED_INTS = 5;  // the leading int fields, initialised and read back by the host

__device__ __forceinline__ float neg_atan2_f(float y, float x) { return -(float)atan2((double)y, (double)x); }

__global__ void deskew_orient_kernel(const float4* __restrict__ cloud, int n, DeskewParams P, float* __restrict__ ori,
                                     float* __restrict__ a_out, DeskewShared* sh) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = cloud[i];
  const float o = neg_atan2_f(p.y, p.x);
  ori[i] = o;
  // formula A, before the half turn (:131-139)
  float a = o;
  const double so = (double)P.start_ori;
  if ((double)a < so - PI_D * 0.5) a = (float)((double)a + 2 * PI_D);
  else if ((double)a > so + PI_D * 1.5) a = (float)((double)a - 2 * PI_D);
  a_out[i] = a;
  if ((double)__fsub_rn(a, P.start_ori) > PI_D) atomicMin(&sh->k_first, i);
}

__global__ void deskew_time_kernel(int n, DeskewParams P, const ImuSample* __restrict__ ring, const float* __restrict__ ori,
                                   const float* __restrict__ a_in, const DeskewShared* __restrict__ sh, float* __restrict__ rel_out,
                                   double* __restrict__ t_out, int* __restrict__ lb_out) {
  __shared__ double times[IMU_QUE];
  for (int j = threadIdx.x; j <= P.span; j += blockDim.x) times[j] = ring[(P.base + j) % IMU_QUE].time;
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float oh;
  if (i <= sh->k_first) {  // the point that sets half_passed still uses formula A itself
    oh = a_in[i];
  } else {  // formula B (:140-147)
    const double eo = (double)P.end_ori;
    oh = (float)((double)ori[i] + 2 * PI_D);
    if ((double)oh < eo - 1.5 * PI_D) oh = (float)((double)oh + 2 * PI_D);
    else if ((double)oh > eo + 0.5 * PI_D) oh = (float)((double)oh - 2 * PI_D);
  }
  // float rel_time = (ori_h - start_ori) / ori_diff * scan_period_   (:149): float quotient, double product, float store
  const float rel = (float)((double)__fdiv_rn(__fsub_rn(oh, P.start_ori), P.ori_diff) * P.scan_period);
  const double t = P.scan_time + (double)rel;
  // first ring position whose stamp is later than t (the walk :153-158 stops there), clamped to the newest sample. The
  // walk's own test `t < time` decides, so a NaN t (a NaN ray) runs to the newest sample like in the reference.
  int lo = 0, hi = P.span + 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (!(t < times[mid])) lo = mid + 1;
    else hi = mid;
  }
  rel_out[i] = rel;
  t_out[i] = t;
  lb_out[i] = min(lo, P.span);
}

// rpy / shift / velocity at time t with the ring pointer at `front` (:169-197)
__device__ __forceinline__ void imu_interp(const ImuSample* __restrict__ ring, int front, double t, float* rpy, float* shift,
                                           float* velo) {
  const ImuSample f = ring[front];
  if (t > f.time) {
    rpy[0] = f.roll; rpy[1] = f.pitch; rpy[2] = f.yaw;
#pragma unroll
    for (int c = 0; c < 3; c++) {
      shift[c] = f.shift[c];
      velo[c] = f.velo[c];
    }
    return;
  }
  const ImuSample b = ring[(front - 1 + IMU_QUE) % IMU_QUE];
  const float rf = (float)((t - b.time) / (f.time - b.time));
  const float rb = (float)(1.0 - (double)rf);
  auto mix = [&](float vf, float vb) { return __fadd_rn(__fmul_rn(vf, rf), __fmul_rn(vb, rb)); };
  rpy[0] = mix(f.roll, b.roll); rpy[1] = mix(f.pitch, b.pitch); rpy[2] = mix(f.yaw, b.yaw);
#pragma unroll
  for (int c = 0; c < 3; c++) {
    shift[c] = mix(f.shift[c], b.shift[c]);
    velo[c] = mix(f.velo[c], b.velo[c]);
  }
}

// (AngleAxisf(yaw, Z) * AngleAxisf(pitch, Y) * AngleAxisf(roll, X)).toRotationMatrix() (:199-206): Eigen multiplies
// angle-axis objects as quaternions, then QuaternionBase::toRotationMatrix — all float, un-fused.
__device__ __forceinline__ void rot_zyx(float roll, float pitch, float yaw, float* R) {
  auto half = [](float ang, float& s, float& c) {
    const double h = (double)__fmul_rn(0.5f, ang);
    s = (float)sin(h);
    c = (float)cos(h);
  };
  float sz, cz, sy, cy, sx, cx;
  half(yaw, sz, cz);
  half(pitch, sy, cy);
  half(roll, sx, cx);
  auto qmul = [](const float* a, const float* b, float* o) {  // (x, y, z, w)
    const float ax = a[0], ay = a[1], az = a[2], aw = a[3], bx = b[0], by = b[1], bz = b[2], bw = b[3];
    o[0] = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(aw, bx), __fmul_rn(ax, bw)), __fmul_rn(ay, bz)), __fmul_rn(az, by));
    o[1] = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(aw, by), __fmul_rn(ay, bw)), __fmul_rn(az, bx)), __fmul_rn(ax, bz));
    o[2] = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(aw, bz), __fmul_rn(az, bw)), __fmul_rn(ax, by)), __fmul_rn(ay, bx));
    o[3] = __fsub_rn(__fsub_rn(__fsub_rn(__fmul_rn(aw, bw), __fmul_rn(ax, bx)), __fmul_rn(ay, by)), __fmul_rn(az, bz));
  };
  const float qz[4] = {0.f, 0.f, sz, cz}, qy[4] = {0.f, sy, 0.f, cy}, qx[4] = {sx, 0.f, 0.f, cx};
  float q1[4], q[4];
  qmul(qz, qy, q1);
  qmul(q1, qx, q);
  const float x = q[0], y = q[1], z = q[2], w = q[3];
  const float tx = __fmul_rn(2.f, x), ty = __fmul_rn(2.f, y), tz = __fmul_rn(2.f, z);
  const float twx = __fmul_rn(tx, w), twy = __fmul_rn(ty, w), twz = __fmul_rn(tz, w);
  const float txx = __fmul_rn(tx, x), txy = __fmul_rn(ty, x), txz = __fmul_rn(tz, x);
  const float tyy = __fmul_rn(ty, y), tyz = __fmul_rn(tz, y), tzz = __fmul_rn(tz, z);
  R[0] = __fsub_rn(1.f, __fadd_rn(tyy, tzz)); R[1] = __fsub_rn(txy, twz);                 R[2] = __fadd_rn(txz, twy);
  R[3] = __fadd_rn(txy, twz);                 R[4] = __fsub_rn(1.f, __fadd_rn(txx, tzz)); R[5] = __fsub_rn(tyz, twx);
  R[6] = __fsub_rn(txz, twy);                 R[7] = __fadd_rn(tyz, twx);                 R[8] = __fsub_rn(1.f, __fadd_rn(txx, tyy));
}

// One CTA: fix point of   skipped_i = |t_i - time[max(carried_i, lb_i)]| > scan_period,
//                         carried_i = max(0, max_{j < i, !skipped_j} lb_j)                    (exclusive prefix max)
// Thread q owns the contiguous chunk [q * per, (q + 1) * per). Converges in one pass when the IMU covers the scan.
// Stamps that step back (P.monotone == 0): thread 0 walks the points literally instead and no fix point runs.
constexpr int SCAN_THREADS = 1024;
__global__ void __launch_bounds__(SCAN_THREADS) deskew_scan_kernel(int n, DeskewParams P, const ImuSample* __restrict__ ring,
                                                                   const double* __restrict__ t, const int* __restrict__ lb,
                                                                   unsigned char* skip2, int* __restrict__ front,
                                                                   DeskewShared* sh) {
  __shared__ double times[IMU_QUE];
  __shared__ int part[SCAN_THREADS];
  __shared__ int warp_tot[32];
  __shared__ int changed;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int j = tid; j <= P.span; j += SCAN_THREADS) times[j] = ring[(P.base + j) % IMU_QUE].time;
  const int per = (n + SCAN_THREADS - 1) / SCAN_THREADS;
  const int c0 = min(n, tid * per), c1 = min(n, c0 + per);
  for (int i = c0; i < c1; i++) skip2[i] = 0;
  __syncthreads();
  int cur = 0, rounds = 0;
  if (!P.monotone) {
    // The stamps step back inside the window (a replayed bag, a restamping driver): the lower bounds of deskew_time do
    // not describe the walk, so thread 0 runs it literally (:152-158, :223) from the carried pointer, position 0.
    if (tid == 0) {
      int carried_pos = 0;
      for (int i = 0; i < n; i++) {
        const double ti = t[i];
        int fp = carried_pos;
        while (fp != P.span && !(ti < times[fp])) fp++;
        const bool s = fabs(ti - times[fp]) > P.scan_period;
        front[i] = fp;
        skip2[i] = s ? 1 : 0;
        if (!s) carried_pos = fp;
      }
    }
    __syncthreads();
  }
  for (int iter = 0; P.monotone && iter <= n; iter++) {
    rounds++;
    const unsigned char* sk = skip2 + (size_t)cur * n;
    unsigned char* sk_new = skip2 + (size_t)(cur ^ 1) * n;
    if (tid == 0) changed = 0;
    int m = -1;  // max contribution of this chunk
    for (int i = c0; i < c1; i++)
      if (!sk[i]) m = max(m, lb[i]);
    // exclusive max-scan of the chunk maxima over the CTA
    int incl = m;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl = max(incl, o);
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int w = warp_tot[lane];
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, w, d);
        if (lane >= d) w = max(w, o);
      }
      warp_tot[lane] = w;
    }
    __syncthreads();
    int carry = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) carry = -1;
    if (warp > 0) carry = max(carry, warp_tot[warp - 1]);
    int carried = max(0, carry);
    bool ch = false;
    for (int i = c0; i < c1; i++) {
      const int l = lb[i];
      const int fp = max(carried, l);
      const bool s_new = fabs(t[i] - times[fp]) > P.scan_period;
      ch = ch || (s_new != (sk[i] != 0));
      sk_new[i] = s_new ? 1 : 0;
      front[i] = fp;
      if (!sk[i]) carried = max(carried, l);
    }
    if (ch) changed = 1;
    __syncthreads();
    cur ^= 1;
    const int again = changed;
    __syncthreads();
    if (!again) break;
  }
  // `cur` now indexes the stable set. Carried pointers and the start pose.
  const unsigned char* sk = skip2 + (size_t)cur * n;
  if (cur == 1) {  // the apply kernel reads the first half
    for (int i = c0; i < c1; i++) skip2[i] = sk[i];
  }
  int last_ok = -1;
  for (int i = c0; i < c1; i++)
    if (!sk[i]) last_ok = i;
  part[tid] = last_ok;
  __syncthreads();
  if (tid == 0) {
    int best = -1;
    for (int q = 0; q < SCAN_THREADS; q++) best = max(best, part[q]);
    sh->ptr_front_pos = front[n - 1];            // assigned before the skip test, for every point (:152-158)
    sh->ptr_iter_pos = best >= 0 ? front[best] : -1;  // carried only past non-skipped points (:223)
    sh->ok0 = sk[0] ? 0 : 1;
    sh->rounds = rounds;
    if (!sk[0]) {
      float rpy[3], shift[3], velo[3], R[9];
      imu_interp(ring, (P.base + front[0]) % IMU_QUE, t[0], rpy, shift, velo);
      rot_zyx(rpy[0], rpy[1], rpy[2], R);
      // r_s_i = r_c.inverse(): the transpose of a rotation (Eigen evaluates the general 3x3 inverse; equal to rounding)
      for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) sh->r_s_i[r * 3 + c] = R[c * 3 + r];
      for (int c = 0; c < 3; c++) {
        sh->shift0[c] = shift[c];
        sh->velo0[c] = velo[c];
      }
    }
  }
}

__global__ void deskew_apply_kernel(float4* __restrict__ cloud, int n, DeskewParams P, const ImuSample* __restrict__ ring,
                                    const double* __restrict__ t, const float* __restrict__ rel, const int* __restrict__ front,
                                    const unsigned char* __restrict__ skip, const DeskewShared* __restrict__ sh) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || i == 0 || !sh->ok0 || skip[i]) return;  // point 0 defines the start pose and stays (:208-212)
  float rpy[3], shift[3], velo[3], R[9];
  imu_interp(ring, (P.base + front[i]) % IMU_QUE, t[i], rpy, shift, velo);
  rot_zyx(rpy[0], rpy[1], rpy[2], R);
  const float rt = rel[i];
  float4 p = cloud[i];
  float v[3];
#pragma unroll
  for (int r = 0; r < 3; r++) {
    // shift_from_start = shift_cur - shift_start - velo_start * rel_time;  r_c * p + shift_from_start   (:213-214)
    const float sfs = __fsub_rn(__fsub_rn(shift[r], sh->shift0[r]), __fmul_rn(sh->velo0[r], rt));
    const float rp = __fadd_rn(__fadd_rn(__fmul_rn(R[r * 3 + 0], p.x), __fmul_rn(R[r * 3 + 1], p.y)), __fmul_rn(R[r * 3 + 2], p.z));
    v[r] = __fadd_rn(rp, sfs);
  }
  const float* S = sh->r_s_i;
  p.x = __fadd_rn(__fadd_rn(__fmul_rn(S[0], v[0]), __fmul_rn(S[1], v[1])), __fmul_rn(S[2], v[2]));
  p.y = __fadd_rn(__fadd_rn(__fmul_rn(S[3], v[0]), __fmul_rn(S[4], v[1])), __fmul_rn(S[5], v[2]));
  p.z = __fadd_rn(__fadd_rn(__fmul_rn(S[6], v[0]), __fmul_rn(S[7], v[1])), __fmul_rn(S[8], v[2]));
  cloud[i] = p;
}

}  // namespace

// ---- host: getImu (:52-106), one call per IMU message ------------------------------------------------------------
void ImuDeskew::get_imu(const float* w, const float* acc_in, const float* q, double imu_time) {
  // Eigen::Quaternionf::toRotationMatrix, float
  const float x = q[0], y = q[1], z = q[2], qw = q[3];
  const float tx = 2.f * x, ty = 2.f * y, tz = 2.f * z;
  const float twx = tx * qw, twy = ty * qw, twz = tz * qw;
  const float txx = tx * x, txy = ty * x, txz = tz * x;
  const float tyy = ty * y, tyz = tz * y, tzz = tz * z;
  const float R[9] = {1.f - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1.f - (txx + tzz), tyz - twx,
                      txz - twy, tyz + twx, 1.f - (txx + tyy)};
  // pcl::getEulerAngles(Affine3f, roll, pitch, yaw)
  const float r = std::atan2(R[7], R[8]);
  const float p = std::asin(-R[6]);
  const float yw = std::atan2(R[3], R[0]);
  ptr_last = (ptr_last + 1) % IMU_QUE;
  if ((ptr_last + 1) % IMU_QUE == ptr_front) ptr_front = (ptr_front + 1) % IMU_QUE;
  const int k = ptr_last;
  time[k] = imu_time;
  roll[k] = r;
  pitch[k] = p;
  yaw[k] = yw;
  float a[3];
  for (int i = 0; i < 3; i++) a[i] = (R[i * 3 + 0] * acc_in[0] + R[i * 3 + 1] * acc_in[1]) + R[i * 3 + 2] * acc_in[2];  // acc = rot * acc
  const int back = (k - 1 + IMU_QUE) % IMU_QUE;
  const double dt = time[k] - time[back];
  if (dt < scan_period) {
    for (int i = 0; i < 3; i++) {  // float member = float + float * double + float * double * double * 0.5 (double, stored as float)
      shift[k][i] = (float)((double)shift[back][i] + (double)velo[back][i] * dt + (double)a[i] * dt * dt * 0.5);
      velo[k][i] = (float)((double)velo[back][i] + (double)a[i] * dt);
      ang_rot[k][i] = (float)((double)ang_rot[back][i] + (double)w[i] * dt);
    }
  }
}

// ---- host: adjustDistortion (:110-226) --------------------------------------------------------------------------
void ImuDeskew::adjust_distortion(float4* d_cloud, size_t n_sz, const float* first_xy, const float* last_xy, double scan_time,
                                  cudaStream_t s) {
  const int n = (int)n_sz;
  trace_n = 0;
  if (n == 0) return;
  if (ptr_last <= 0) {  // `if (imu_ptr_last_ > 0)` (:151) is false: no point is touched; the carry at :223 still runs
    ptr_last_iter = ptr_front;
    return;
  }
  DeskewParams P{};
  auto neg_atan2 = [](float y, float x) { return -(float)std::atan2((double)y, (double)x); };
  float start_ori = neg_atan2(first_xy[1], first_xy[0]);
  float end_ori = neg_atan2(last_xy[1], last_xy[0]);
  if ((double)(end_ori - start_ori) > 3 * PI_D) end_ori = (float)((double)end_ori - 2 * PI_D);
  else if ((double)(end_ori - start_ori) < PI_D) end_ori = (float)((double)end_ori + 2 * PI_D);
  P.start_ori = start_ori;
  P.end_ori = end_ori;
  P.ori_diff = end_ori - start_ori;
  P.scan_period = scan_period;
  P.scan_time = scan_time;
  P.base = ptr_last_iter;
  P.span = ((ptr_last - ptr_last_iter) % IMU_QUE + IMU_QUE) % IMU_QUE;

  d_ori.ensure(n); d_a.ensure(n); d_rel.ensure(n); d_t.ensure(n); d_lb.ensure(n); d_front.ensure(n);
  d_skip.ensure((size_t)2 * n);
  const size_t ring_bytes = sizeof(ImuSample) * IMU_QUE;
  d_small.ensure(ring_bytes + sizeof(DeskewShared));
  h_out.ensure(IMU_QUE * sizeof(ImuSample) / sizeof(int) + 16);
  ImuSample* h_ring = reinterpret_cast<ImuSample*>(h_out.ptr + 16);
  for (int k = 0; k < IMU_QUE; k++) {
    ImuSample& e = h_ring[k];
    e.time = time[k];
    e.roll = roll[k]; e.pitch = pitch[k]; e.yaw = yaw[k];
    for (int c = 0; c < 3; c++) {
      e.shift[c] = shift[k][c];
      e.velo[c] = velo[k][c];
    }
    e.pad = 0.f;
  }
  P.monotone = 1;  // the walk's order; NaN stamps also take the literal walk
  for (int j = 0; j < P.span; j++)
    if (!(time[(P.base + j + 1) % IMU_QUE] >= time[(P.base + j) % IMU_QUE])) P.monotone = 0;
  ImuSample* d_ring = reinterpret_cast<ImuSample*>(d_small.ptr);
  DeskewShared* d_sh = reinterpret_cast<DeskewShared*>(d_small.ptr + ring_bytes);
  DeskewShared init{};
  init.k_first = n;
  init.ptr_iter_pos = -1;
  std::memcpy(h_out.ptr + 8, &init, sizeof(int) * DESKEW_SHARED_INTS);
  B200_CUDA(cudaMemcpyAsync(d_ring, h_ring, ring_bytes, cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaMemcpyAsync(d_sh, h_out.ptr + 8, sizeof(int) * DESKEW_SHARED_INTS, cudaMemcpyHostToDevice, s));
  const int blocks = (n + 255) / 256;
  deskew_orient_kernel<<<blocks, 256, 0, s>>>(d_cloud, n, P, d_ori.ptr, d_a.ptr, d_sh);
  deskew_time_kernel<<<blocks, 256, 0, s>>>(n, P, d_ring, d_ori.ptr, d_a.ptr, d_sh, d_rel.ptr, d_t.ptr, d_lb.ptr);
  deskew_scan_kernel<<<1, SCAN_THREADS, 0, s>>>(n, P, d_ring, d_t.ptr, d_lb.ptr, d_skip.ptr, d_front.ptr, d_sh);
  deskew_apply_kernel<<<blocks, 256, 0, s>>>(d_cloud, n, P, d_ring, d_t.ptr, d_rel.ptr, d_front.ptr, d_skip.ptr, d_sh);
  B200_CUDA(cudaGetLastError());
  launches += 4;
  B200_CUDA(cudaMemcpyAsync(h_out.ptr, d_sh, sizeof(int) * DESKEW_SHARED_INTS, cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  // imu_ptr_front_ / imu_ptr_last_iter_ after the loop
  ptr_front = (P.base + h_out.ptr[1]) % IMU_QUE;
  if (h_out.ptr[2] >= 0) ptr_last_iter = (P.base + h_out.ptr[2]) % IMU_QUE;
  trace_n = n;
  trace_base = P.base;
  trace_k_first = h_out.ptr[0];
  trace_rounds = h_out.ptr[4];
}

// ---- read-back of the last adjust_distortion's per-point scratch (tests) -----------------------------------------
size_t ImuDeskew::get_trace(size_t capacity, float* rel_time, double* t, int* front, unsigned char* skip, int* k_first,
                            int* rounds, cudaStream_t s) {
  const size_t n = trace_n, m = capacity < n ? capacity : n;
  if (k_first) *k_first = trace_k_first;
  if (rounds) *rounds = trace_rounds;
  if (m == 0) return n;
  if (rel_time) B200_CUDA(cudaMemcpyAsync(rel_time, d_rel.ptr, m * sizeof(float), cudaMemcpyDeviceToHost, s));
  if (t) B200_CUDA(cudaMemcpyAsync(t, d_t.ptr, m * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (front) B200_CUDA(cudaMemcpyAsync(front, d_front.ptr, m * sizeof(int), cudaMemcpyDeviceToHost, s));
  if (skip) B200_CUDA(cudaMemcpyAsync(skip, d_skip.ptr, m, cudaMemcpyDeviceToHost, s));  // the stable half
  B200_CUDA(cudaStreamSynchronize(s));
  if (front)
    for (size_t i = 0; i < m; i++) front[i] = (trace_base + front[i]) % IMU_QUE;  // ring positions -> ring indices
  return n;
}

}  // namespace b200
