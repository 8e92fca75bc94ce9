// Shared device/host definitions of the registration engine (H100, sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdio>
#include <stdexcept>
#include <string>

namespace b200 {

// SM count of the H100 SXM: the grid-stride launches are capped at a few waves of it.
constexpr int H100_SMS = 132;

struct CudaError : std::runtime_error {
  using std::runtime_error::runtime_error;
};

#define B200_CUDA(call)                                                                              \
  do {                                                                                               \
    cudaError_t err__ = (call);                                                                      \
    if (err__ != cudaSuccess)                                                                        \
      throw ::b200::CudaError(std::string(#call) + ": " + cudaGetErrorString(err__) + " @" + __FILE__ + \
                              ":" + std::to_string(__LINE__));                                       \
  } while (0)

// Geometry of a PCL-style voxel grid (voxel_grid_covariance_omp_impl.hpp:67-103): leaf index
//   idx = (i - min_b.x) + (j - min_b.y) * div_b.x + (k - min_b.z) * div_b.x * div_b.y   (< 2^31, guarded).
struct GridGeom {
  float leaf;      // leaf_size_
  float inv_leaf;  // inverse_leaf_size_ = 1.0f / leaf
  int min_b[3];
  int max_b[3];
  int div_b[3];
  int mul[3];        // divb_mul_
  long long n_cells;  // div_b.x * div_b.y * div_b.z
  int n_words;        // ceil(n_cells / 32)
};

// Occupancy-bitmap rank index ("perfect voxel hash"): one entry per 32 consecutive leaf indices.
//   bits   — occupancy of the 32 cells
//   prefix — number of occupied cells in all previous words
// record index of an occupied cell = prefix + popc(bits & ((1u << bit) - 1)). Because the rank is monotone in
// the leaf index, records are stored in ascending leaf index — the iteration order of the reference's
// std::map<size_t, Leaf> (voxel_grid_covariance_omp.h:195).
struct RankWord {
  unsigned bits;
  unsigned prefix;
};

// One NDT voxel as the fused kernel reads it (48 B, three 16-byte loads):
//   mean as a float-float pair (hi + lo carries the f64 mean to ~2^-48 relative) so that
//   x' = (x_trans - mean_hi) - mean_lo is within one float ulp of the reference's f64 subtraction followed by the cast
//   to float (ndt_omp_impl.hpp:259-262, 490; not always equal to it) without FP64 instructions on the hot path;
//   inverse covariance as the f32 cast the reference applies at ndt_omp_impl.hpp:490-492 (symmetric 6).
struct __align__(16) VoxelRecord {
  float mhx, mhy, mhz, mlx;
  float mly, mlz, c00, c01;
  float c02, c11, c12, c22;
};
static_assert(sizeof(VoxelRecord) == 48, "VoxelRecord must be 48 bytes");
__host__ __device__ inline double record_mean(const VoxelRecord& r, int axis) {
  return axis == 0 ? (double)r.mhx + (double)r.mlx : (axis == 1 ? (double)r.mhy + (double)r.mly : (double)r.mhz + (double)r.mlz);
}

// slots of the 32-wide reduction vector produced by one derivative pass
enum : int { SLOT_SCORE = 0, SLOT_G = 1, SLOT_H = 7, SLOT_HITS = 28, SLOT_COUNT = 32 };

__host__ __device__ inline int tri_index(int i, int j) {  // upper-triangular (i <= j) row-major index in 6x6
  return i * 6 - (i * (i - 1)) / 2 + (j - i);
}

// top 3x4 of a row-major 4x4 float transform, passed to kernels by value
struct Mat34f {
  float m[12];
};

// 4x4 column-major <-> row-major, each entry static_cast to the destination's element type
template <typename S, typename D>
inline void col_to_row(const S* c, D* r) {
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) r[i * 4 + j] = static_cast<D>(c[j * 4 + i]);
}
template <typename S, typename D>
inline void row_to_col(const S* r, D* c) {
  for (int i = 0; i < 4; i++)
    for (int j = 0; j < 4; j++) c[j * 4 + i] = static_cast<D>(r[i * 4 + j]);
}

// A caller's host records: x, y, z float32 at bytes 0, 4, 8 of every `stride_bytes`-byte record (4-byte fields, so the
// stride is a multiple of 4), and an intensity float at `intensity_offset_bytes` when that is >= 0. The intensity must lie
// inside the record: the unpack kernels read, and VoxelGrid's write-back writes, 4 bytes at that offset of every record.
inline bool valid_record_layout(size_t stride_bytes, long intensity_offset_bytes) {
  return stride_bytes >= 12 && (stride_bytes % 4) == 0 &&
         (intensity_offset_bytes < 0 ||
          ((intensity_offset_bytes % 4) == 0 && (size_t)intensity_offset_bytes + 4 <= stride_bytes));
}

// ---- small PTX helpers ------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ unsigned ld_relaxed_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned atom_add_acq_rel_gpu(unsigned* p, unsigned v) {
  unsigned old;
  asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}
__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }

// The entry of a launch's table that serves `v` (a tile, a word): the last of the n entries whose `key` is <= v (the
// table is sorted by `key`, its first entry's key is 0; an entry that owns nothing shares its key with the next one).
template <typename E, typename K, typename V>
__device__ __forceinline__ int entry_of(const E* __restrict__ table, int n, V v, K E::*key) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (table[mid].*key <= v) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// order-preserving float <-> uint mapping for atomicMin/atomicMax on floats
__device__ __forceinline__ unsigned float_to_ordered(float f) {
  unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ inline float ordered_to_float(unsigned u) {
  unsigned v = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
#ifdef __CUDA_ARCH__
  return __uint_as_float(v);
#else
  float f;
  memcpy(&f, &v, 4);
  return f;
#endif
}

// leaf index of a point at BUILD time: (int)(floorf(p * inv_leaf) - (float)min_b)
// (voxel_grid_covariance_omp_impl.hpp:218-223). __fmul_rn keeps the product un-fused like the reference.
__device__ __forceinline__ int build_leaf_index(const GridGeom& g, float x, float y, float z) {
  int i0 = static_cast<int>(floorf(__fmul_rn(x, g.inv_leaf)) - static_cast<float>(g.min_b[0]));
  int i1 = static_cast<int>(floorf(__fmul_rn(y, g.inv_leaf)) - static_cast<float>(g.min_b[1]));
  int i2 = static_cast<int>(floorf(__fmul_rn(z, g.inv_leaf)) - static_cast<float>(g.min_b[2]));
  return i0 * g.mul[0] + i1 * g.mul[1] + i2 * g.mul[2];
}

// T (3x4 row-major) applied to p.xyz: ((T0*x + T1*y) + T2*z) + T3, un-fused like pcl::transformPointCloud's float
// arithmetic. The only f32 point transform: the solver, the NN queries, GICP and the frontend all use it.
__device__ __forceinline__ float3 transform_point(const float* T, float4 p) {
  float3 r;
  r.x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[0], p.x), __fmul_rn(T[1], p.y)), __fmul_rn(T[2], p.z)), T[3]);
  r.y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4], p.x), __fmul_rn(T[5], p.y)), __fmul_rn(T[6], p.z)), T[7]);
  r.z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[8], p.x), __fmul_rn(T[9], p.y)), __fmul_rn(T[10], p.z)), T[11]);
  return r;
}
#endif

}  // namespace b200
