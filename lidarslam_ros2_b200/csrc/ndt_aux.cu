// Off-hot-path NDT kernels, all f64 over the radius neighbourhood:
//   K2  ndt_hessian_radius   computeHessian / updateHessian          ndt_omp_impl.hpp:538-629 (+ :441-479)
//       ndt_score            calculateScore                           ndt_omp_impl.hpp:919-953
//       transform_cloud      the `output` cloud of align()            pcl::transformPointCloud (external)
// The radius neighbourhood reproduces VoxelGridCovariance::radiusSearch (voxel_grid_covariance_omp.h:470-499): every
// voxel whose centroid passes |centroid - x|^2 < r^2 in un-fused f32. It is NOT confined to the 27 cells around the
// query's lookup cell: the builder's cell floor(x * inv_leaf) and the lookup's floor(x / leaf) disagree near a cell
// face, so a centroid two lookup cells away can be closer than the resolution. for_radius_voxels (ndt_solver.cuh)
// probes the build cells that can hold a hit instead.
#include "ndt_solver.cuh"

namespace b200 {

namespace {

struct AuxParams {
  const float4* src;
  const RankWord* index;
  const VoxelRecord* records;
  const double* icov_d;
  const float4* centroids;
  GridGeom geom;
  int n;
  float resolution;  // search radius
  float radius2;     // (float)(resolution * resolution) in double, the FLANN radius
  double d1, d2, d3;
  const float* T_dev;  // 12 floats on the device, or nullptr (cloud already transformed)
  const double* jd;  // 24 (device)
  const double* hd;  // 45 (device)
  double* out;       // 21 (hessian upper triangle) or 1 (score)
};

template <typename F>
__device__ __forceinline__ void for_radius_neighbours(const AuxParams& P, float3 xt, F&& f) {
  for_radius_voxels<false>(P.geom, P.index, P.centroids, P.resolution, P.radius2, xt, f);
}

__device__ __forceinline__ void matvec3(const double* C, const double* v, double* o) {
  o[0] = C[0] * v[0] + C[1] * v[1] + C[2] * v[2];
  o[1] = C[3] * v[0] + C[4] * v[1] + C[5] * v[2];
  o[2] = C[6] * v[0] + C[7] * v[1] + C[8] * v[2];
}
__device__ __forceinline__ double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

__global__ void __launch_bounds__(128) hessian_radius_kernel(AuxParams P) {
  __shared__ float Ts[12];
  if (P.T_dev && threadIdx.x < 12) Ts[threadIdx.x] = __ldcg(P.T_dev + threadIdx.x);
  __syncthreads();
  double acc[21];
#pragma unroll
  for (int k = 0; k < 21; k++) acc[k] = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P.n; i += gridDim.x * blockDim.x) {
    const float4 p = P.src[i];
    const float3 xt = P.T_dev ? transform_point(Ts, p) : make_float3(p.x, p.y, p.z);
    const double x[3] = {p.x, p.y, p.z};
    // point gradient columns (3x6) and second-derivative vectors in f64 (ndt_omp_impl.hpp:441-479)
    double J[6][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    J[3][1] = dot3(x, P.jd + 0);
    J[3][2] = dot3(x, P.jd + 3);
    J[4][0] = dot3(x, P.jd + 6);
    J[4][1] = dot3(x, P.jd + 9);
    J[4][2] = dot3(x, P.jd + 12);
    J[5][0] = dot3(x, P.jd + 15);
    J[5][1] = dot3(x, P.jd + 18);
    J[5][2] = dot3(x, P.jd + 21);
    const double va[3] = {0, dot3(x, P.hd + 0), dot3(x, P.hd + 3)};
    const double vb[3] = {0, dot3(x, P.hd + 6), dot3(x, P.hd + 9)};
    const double vc[3] = {0, dot3(x, P.hd + 12), dot3(x, P.hd + 15)};
    const double vd[3] = {dot3(x, P.hd + 18), dot3(x, P.hd + 21), dot3(x, P.hd + 24)};
    const double ve[3] = {dot3(x, P.hd + 27), dot3(x, P.hd + 30), dot3(x, P.hd + 33)};
    const double vf[3] = {dot3(x, P.hd + 36), dot3(x, P.hd + 39), dot3(x, P.hd + 42)};
    for_radius_neighbours(P, xt, [&](int r) {
      const VoxelRecord* rec = P.records + r;
      const double xd[3] = {(double)xt.x - record_mean(*rec, 0), (double)xt.y - record_mean(*rec, 1),
                            (double)xt.z - record_mean(*rec, 2)};
      const double* C = P.icov_d + (size_t)r * 9;
      double Cx[3];
      matvec3(C, xd, Cx);
      double e = P.d2 * exp(-P.d2 * dot3(xd, Cx) / 2);
      if (e > 1 || e < 0 || e != e) return;
      e *= P.d1;
      double CJ[6][3], xCJ[6];
      for (int k = 0; k < 6; k++) {
        matvec3(C, J[k], CJ[k]);
        xCJ[k] = dot3(xd, CJ[k]);
      }
      int t = 0;
      for (int a = 0; a < 6; a++)
        for (int b = a; b < 6; b++, t++) {
          double h2 = 0.0;
          if (a >= 3 && b >= 3) {
            const double* hv = (a == 3) ? (b == 3 ? va : (b == 4 ? vb : vc)) : (a == 4 ? (b == 4 ? vd : ve) : vf);
            double Ch[3];
            matvec3(C, hv, Ch);
            h2 = dot3(xd, Ch);
          }
          acc[t] += e * (-P.d2 * xCJ[a] * xCJ[b] + h2 + dot3(J[b], CJ[a]));
        }
    });
  }
#pragma unroll
  for (int k = 0; k < 21; k++) {
    double v = acc[k];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    if ((threadIdx.x & 31) == 0) atomicAdd(P.out + k, v);
  }
}

__global__ void __launch_bounds__(128) score_kernel(AuxParams P) {
  double acc = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P.n; i += gridDim.x * blockDim.x) {
    const float4 p = P.src[i];
    const float3 xt = make_float3(p.x, p.y, p.z);  // calculateScore takes an already transformed cloud
    int nb = 0;
    double s = 0.0;
    for_radius_neighbours(P, xt, [&](int r) {
      const VoxelRecord* rec = P.records + r;
      const double xd[3] = {(double)xt.x - record_mean(*rec, 0), (double)xt.y - record_mean(*rec, 1),
                            (double)xt.z - record_mean(*rec, 2)};
      double Cx[3];
      matvec3(P.icov_d + (size_t)r * 9, xd, Cx);
      const double e = exp(-P.d2 * dot3(xd, Cx) / 2);
      s += -P.d1 * e - P.d3;
      nb++;
    });
    if (nb > 0) acc += s / (double)nb;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
  if ((threadIdx.x & 31) == 0) atomicAdd(P.out, acc);
}

// after a K2 pass requested by the persistent solver: mirror the 21 sums into state.H and re-arm the control block
__global__ void hessian_to_state_kernel(const double* upper21, NdtSolverWork* W) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    for (int i = 0; i < 6; i++)
      for (int j = i; j < 6; j++) {
        double v = upper21[tri_index(i, j)];
        W->state.H[i * 6 + j] = v;
        W->state.H[j * 6 + i] = v;
      }
    W->control.mode = EVAL_DERIV;
  }
}

// pcl::transformPointCloud(in, out, Eigen::Matrix4f): xyz <- R xyz + t in float, other fields (intensity) copied
__global__ void __launch_bounds__(256) transform_cloud_kernel(const float4* __restrict__ in, size_t n, Mat34f T,
                                                              float4* __restrict__ out) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = in[i];
  const float3 r = transform_point(T.m, p);
  out[i] = make_float4(r.x, r.y, r.z, p.w);
}

}  // namespace

// ---- host wrappers (declared in ndt_aux.hpp) ----------------------------------------------------------------
void ndt_hessian_radius(const VoxelMap& map, const float4* src, size_t n, const NdtConfig& cfg, const float* d_T12,
                        const double* d_jd, const double* d_hd, double* d_out21, cudaStream_t s) {
  AuxParams P{};
  P.src = src;
  P.index = map.index.ptr;
  P.records = map.records.ptr;
  P.icov_d = map.icov_d.ptr;
  P.centroids = map.centroids.ptr;
  P.geom = map.geom;
  P.n = (int)n;
  P.resolution = cfg.resolution;
  P.radius2 = static_cast<float>((double)cfg.resolution * (double)cfg.resolution);
  GaussConsts gc = gauss_constants(cfg.outlier_ratio, cfg.resolution);
  P.d1 = gc.d1;
  P.d2 = gc.d2;
  P.d3 = gc.d3;
  P.T_dev = d_T12;
  P.jd = d_jd;
  P.hd = d_hd;
  P.out = d_out21;
  B200_CUDA(cudaMemsetAsync(d_out21, 0, 21 * sizeof(double), s));
  int blocks = (int)std::min<size_t>((n + 127) / 128, H100_SMS * 8);
  if (blocks < 1) blocks = 1;
  hessian_radius_kernel<<<blocks, 128, 0, s>>>(P);
  B200_CUDA(cudaGetLastError());
}

void ndt_hessian_into_state(const double* d_upper21, NdtSolverWork* work, cudaStream_t s) {
  hessian_to_state_kernel<<<1, 32, 0, s>>>(d_upper21, work);
  B200_CUDA(cudaGetLastError());
}

void ndt_score(const VoxelMap& map, const float4* cloud, size_t n, const NdtConfig& cfg, double* d_out1, cudaStream_t s) {
  AuxParams P{};
  P.src = cloud;
  P.index = map.index.ptr;
  P.records = map.records.ptr;
  P.icov_d = map.icov_d.ptr;
  P.centroids = map.centroids.ptr;
  P.geom = map.geom;
  P.n = (int)n;
  P.resolution = cfg.resolution;
  P.radius2 = static_cast<float>((double)cfg.resolution * (double)cfg.resolution);
  GaussConsts gc = gauss_constants(cfg.outlier_ratio, cfg.resolution);
  P.d1 = gc.d1;
  P.d2 = gc.d2;
  P.d3 = gc.d3;
  P.T_dev = nullptr;
  P.out = d_out1;
  B200_CUDA(cudaMemsetAsync(d_out1, 0, sizeof(double), s));
  int blocks = (int)std::min<size_t>((n + 127) / 128, H100_SMS * 8);
  if (blocks < 1) blocks = 1;
  score_kernel<<<blocks, 128, 0, s>>>(P);
  B200_CUDA(cudaGetLastError());
}

void transform_cloud_device(const float4* in, size_t n, float4* out, const Mat34f& T, cudaStream_t s) {
  if (n == 0) return;
  transform_cloud_kernel<<<(int)((n + 255) / 256), 256, 0, s>>>(in, n, T, out);
  B200_CUDA(cudaGetLastError());
}

}  // namespace b200
