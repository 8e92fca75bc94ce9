// K21: the surface mesh of the session's submaps (b200sm_build_mesh). Every decision follows csrc/mesh.hpp, which a host
// compile also builds. The field is fused with integer atomics and every output position comes from a scan of per-tile
// counts, so the voxels, vertices and faces are bitwise the host's whatever the order of the work.
#include "grid_index.cuh"
#include "mesh.cuh"

namespace b200 {
namespace {

constexpr unsigned MS_NONE = 0xffffffffu;

// The band walk of point p of entry e: visit(x, y, z, s) for every voxel; false when the point is not a ray.
template <class Visit>
__device__ __forceinline__ bool ms_ray_walk(const SmEntry& e, const MsConst& c, float4 p, Visit&& visit) {
  float q[3];
  og_transform(e.T, p.x, p.y, p.z, q);
  int v[3];
  long long E[3];
  if (!sm_ray(c.sm, e.o, q[0], q[1], q[2], &v[0], &v[1], &v[2], &E[0], &E[1], &E[2])) return false;
  long long A[3], B[3];
  double L;
  if (!ms_band(c.T, e.o, E[0], E[1], E[2], A, B, &L)) return true;  // zero length: a ray that walks nothing
  const long long dx = E[0] - e.o[0], dy = E[1] - e.o[1], dz = E[2] - e.o[2];
  const long long T = c.T;
  sm_walk(A[0], A[1], A[2], B[0], B[1], B[2],
          [&](int x, int y, int z) { visit(x, y, z, ms_sdf(T, E[0], E[1], E[2], dx, dy, dz, L, x, y, z)); });
  return true;
}

// K21a. Block b serves tile b of the whole map (the static map's tiles); a thread walks SM_PER_THREAD points of it.
__global__ void __launch_bounds__(SM_THREADS) ms_mark_kernel(const SmEntry* __restrict__ table, int n_entries, MsConst c, SmBox box,
                                                             RankWord* __restrict__ index, unsigned long long* __restrict__ counters) {
  const int k = entry_of(table, n_entries, blockIdx.x, &SmEntry::first_tile);
  const SmEntry& e = table[k];
  const unsigned base = (blockIdx.x - e.first_tile) * (unsigned)SM_TILE + threadIdx.x;
  unsigned tripped = 0;
  for (int j = 0; j < SM_PER_THREAD; j++) {
    const unsigned i = base + j * SM_THREADS;
    if (i >= e.n) break;
    ms_ray_walk(e, c, e.cloud[i], [&](int x, int y, int z, long long) {
      unsigned lin;
      if (sm_lin(box, x, y, z, &lin)) mark_occupied(index, (int)lin);
      else tripped = 1u;
    });
  }
  if (tripped) atomicAdd(&counters[SM_CTR_TRIPPED], 1ull);
}

// K21b. The same walks: each voxel's s and one ray into its sum and weight.
__global__ void __launch_bounds__(SM_THREADS) ms_fuse_kernel(const SmEntry* __restrict__ table, int n_entries, MsConst c, SmBox box,
                                                             const RankWord* __restrict__ index, unsigned n_band,
                                                             unsigned long long* __restrict__ sum, uint32_t* __restrict__ weight,
                                                             unsigned long long* __restrict__ counters) {
  const int k = entry_of(table, n_entries, blockIdx.x, &SmEntry::first_tile);
  const SmEntry& e = table[k];
  const unsigned base = (blockIdx.x - e.first_tile) * (unsigned)SM_TILE + threadIdx.x;
  unsigned tripped = 0, walked = 0;
  for (int j = 0; j < SM_PER_THREAD; j++) {
    const unsigned i = base + j * SM_THREADS;
    if (i >= e.n) break;
    ms_ray_walk(e, c, e.cloud[i], [&](int x, int y, int z, long long s) {
      unsigned r;
      if (sm_rank(index, box, x, y, z, &r) && r < n_band) {
        atomicAdd(sum + r, (unsigned long long)s);
        atomicAdd(weight + r, 1u);
        walked++;
      } else {
        tripped = 1u;
      }
    });
  }
  walked = __reduce_add_sync(0xffffffffu, walked);
  if ((threadIdx.x & 31) == 0 && walked) atomicAdd(&counters[MS_CTR_WALKED], (unsigned long long)walked);
  if (tripped) atomicAdd(&counters[SM_CTR_TRIPPED], 1ull);
}

// the rank of voxel (x, y, z) when it is an observed band voxel
__device__ __forceinline__ bool ms_observed(const RankWord* __restrict__ index, const SmBox& box, const uint32_t* __restrict__ weight,
                                            unsigned n_band, unsigned min_weight, int x, int y, int z, unsigned* r) {
  return sm_rank(index, box, x, y, z, r) && *r < n_band && __ldg(weight + *r) >= min_weight;
}

// whether the cell whose lowest corner is (i, j, k) is ACTIVE; D[] and neg[] of its corners when it is
__device__ __forceinline__ bool ms_cell(const RankWord* __restrict__ index, const SmBox& box, const unsigned long long* __restrict__ sum,
                                        const uint32_t* __restrict__ weight, unsigned n_band, unsigned min_weight, int i, int j, int k,
                                        double* D, bool* neg) {
  int n_neg = 0;
#pragma unroll
  for (int m = 0; m < 8; m++) {
    unsigned r;
    if (!ms_observed(index, box, weight, n_band, min_weight, i + (m & 1), j + ((m >> 1) & 1), k + ((m >> 2) & 1), &r)) return false;
    const long long s = (long long)__ldg(sum + r);
    D[m] = ms_dist(s, __ldg(weight + r));
    neg[m] = ms_neg(s);
    n_neg += neg[m];
  }
  return n_neg > 0 && n_neg < 8;
}

// K21c. One thread per band voxel, tile = block.
__global__ void __launch_bounds__(MS_THREADS) ms_active_kernel(const int* __restrict__ ijk, const unsigned long long* __restrict__ sum,
                                                               const uint32_t* __restrict__ weight, const RankWord* __restrict__ index,
                                                               SmBox box, unsigned n_band, unsigned min_weight,
                                                               unsigned char* __restrict__ active, unsigned* __restrict__ counts,
                                                               unsigned long long* __restrict__ counters) {
  const unsigned r = blockIdx.x * MS_THREADS + threadIdx.x;
  bool act = false, obs = false;
  if (r < n_band) {
    obs = __ldg(weight + r) >= min_weight;
    double D[8];
    bool neg[8];
    act = obs && ms_cell(index, box, sum, weight, n_band, min_weight, ijk[3ull * r], ijk[3ull * r + 1], ijk[3ull * r + 2], D, neg);
    active[r] = act ? 1 : 0;
  }
  const unsigned o = __reduce_add_sync(0xffffffffu, obs ? 1u : 0u);
  if ((threadIdx.x & 31) == 0 && o) atomicAdd(&counters[MS_CTR_OBSERVED], (unsigned long long)o);
  const int n = __syncthreads_count(act);
  if (threadIdx.x == 0) counts[blockIdx.x] = (unsigned)n;
}

// the faces of band voxel v = (i, j, k)'s edge along axis a: 2 when the edge changes sign and its four cells are ACTIVE;
// ids[] = the cells' vertex ids when vid is given
__device__ __forceinline__ int ms_edge(const RankWord* __restrict__ index, const SmBox& box, const unsigned long long* __restrict__ sum,
                                       const uint32_t* __restrict__ weight, unsigned n_band, unsigned min_weight,
                                       const unsigned char* __restrict__ active, const uint32_t* __restrict__ vid, int a, int i, int j,
                                       int k, bool v_neg, unsigned* ids) {
  unsigned w;
  if (!ms_observed(index, box, weight, n_band, min_weight, i + (a == 0), j + (a == 1), k + (a == 2), &w)) return 0;
  if (ms_neg((long long)__ldg(sum + w)) == v_neg) return 0;
#pragma unroll
  for (int m = 0; m < 4; m++) {
    int cc[3];
    ms_edge_cell(a, m & 1, m >> 1, i, j, k, cc);
    unsigned r;
    if (!sm_rank(index, box, cc[0], cc[1], cc[2], &r) || r >= n_band) return 0;
    if (vid) {
      ids[m] = __ldg(vid + r);
      if (ids[m] == MS_NONE) return 0;
    } else if (!__ldg(active + r)) {
      return 0;
    }
  }
  return 2;
}

// K21d. One thread per band voxel: its cell's vertex id and vertex, and its edges' face count.
__global__ void __launch_bounds__(MS_THREADS) ms_vertex_kernel(const int* __restrict__ ijk, const unsigned long long* __restrict__ sum,
                                                               const uint32_t* __restrict__ weight, const RankWord* __restrict__ index,
                                                               SmBox box, unsigned n_band, MsConst c,
                                                               const unsigned char* __restrict__ active,
                                                               const unsigned* __restrict__ tile_offsets, unsigned n_vertices,
                                                               uint32_t* __restrict__ vid, float* __restrict__ xyz,
                                                               unsigned* __restrict__ face_counts,
                                                               unsigned long long* __restrict__ counters) {
  __shared__ unsigned block_faces;
  if (threadIdx.x == 0) block_faces = 0;
  const unsigned r = blockIdx.x * MS_THREADS + threadIdx.x;
  const bool in = r < n_band;
  const bool act = in && active[r];
  unsigned total;
  const unsigned id = tile_offsets[blockIdx.x] + block_exclusive_scan<MS_THREADS>(act ? 1u : 0u, total);  // has a barrier
  unsigned tripped = 0, faces = 0;
  if (in) {
    const int i = ijk[3ull * r], j = ijk[3ull * r + 1], k = ijk[3ull * r + 2];
    vid[r] = act ? id : MS_NONE;
    if (act) {
      double D[8];
      bool neg[8];
      ms_cell(index, box, sum, weight, n_band, c.min_weight, i, j, k, D, neg);
      float v[3];
      ms_vertex(D, neg, i, j, k, c.resolution, v);
      if (id < n_vertices) {
        xyz[3ull * id] = v[0];
        xyz[3ull * id + 1] = v[1];
        xyz[3ull * id + 2] = v[2];
      } else {
        tripped = 1u;
      }
    }
    if (__ldg(weight + r) >= c.min_weight) {
      const bool vn = ms_neg((long long)__ldg(sum + r));
#pragma unroll
      for (int a = 0; a < 3; a++) faces += ms_edge(index, box, sum, weight, n_band, c.min_weight, active, nullptr, a, i, j, k, vn, nullptr);
    }
  }
  const unsigned f = __reduce_add_sync(0xffffffffu, faces);
  if ((threadIdx.x & 31) == 0 && f) atomicAdd(&block_faces, f);
  if (tripped) atomicAdd(&counters[SM_CTR_TRIPPED], 1ull);
  __syncthreads();
  if (threadIdx.x == 0) {
    face_counts[blockIdx.x] = block_faces;
    if (block_faces) atomicAdd(&counters[MS_CTR_FACES], (unsigned long long)block_faces);
  }
}

// K21e. One thread per band voxel: its faces at the tile's offset plus the faces of the lower threads of the tile.
__global__ void __launch_bounds__(MS_THREADS) ms_face_kernel(const int* __restrict__ ijk, const unsigned long long* __restrict__ sum,
                                                             const uint32_t* __restrict__ weight, const RankWord* __restrict__ index,
                                                             SmBox box, unsigned n_band, unsigned min_weight,
                                                             const uint32_t* __restrict__ vid, const unsigned* __restrict__ face_offsets,
                                                             unsigned n_faces, uint32_t* __restrict__ out,
                                                             unsigned long long* __restrict__ counters) {
  const unsigned r = blockIdx.x * MS_THREADS + threadIdx.x;
  unsigned ids[3][4];
  int nf[3] = {0, 0, 0};
  bool vn = false;
  if (r < n_band && __ldg(weight + r) >= min_weight) {
    const int i = ijk[3ull * r], j = ijk[3ull * r + 1], k = ijk[3ull * r + 2];
    vn = ms_neg((long long)__ldg(sum + r));
#pragma unroll
    for (int a = 0; a < 3; a++) nf[a] = ms_edge(index, box, sum, weight, n_band, min_weight, nullptr, vid, a, i, j, k, vn, ids[a]);
  }
  unsigned total;
  unsigned at = face_offsets[blockIdx.x] + block_exclusive_scan<MS_THREADS>((unsigned)(nf[0] + nf[1] + nf[2]), total);
  unsigned tripped = 0;
#pragma unroll
  for (int a = 0; a < 3; a++) {
    if (!nf[a]) continue;
    unsigned tri[6];
    ms_quad(ids[a], vn, tri);
#pragma unroll
    for (int t = 0; t < 2; t++, at++) {
      if (at < n_faces) {
        out[3ull * at] = tri[3 * t];
        out[3ull * at + 1] = tri[3 * t + 1];
        out[3ull * at + 2] = tri[3 * t + 2];
      } else {
        tripped = 1u;
      }
    }
  }
  if (tripped) atomicAdd(&counters[SM_CTR_TRIPPED], 1ull);
}

unsigned ms_blocks(unsigned n) { return (n + MS_THREADS - 1) / MS_THREADS; }

}  // namespace

void ms_mark_launch(const SmEntry* table, int n_entries, unsigned tiles, const MsConst& c, const SmBox& box, RankWord* index,
                    unsigned long long* counters, cudaStream_t stream) {
  if (tiles == 0) return;
  ms_mark_kernel<<<tiles, SM_THREADS, 0, stream>>>(table, n_entries, c, box, index, counters);
  B200_CUDA(cudaGetLastError());
}

void ms_fuse_launch(const SmEntry* table, int n_entries, unsigned tiles, const MsConst& c, const SmBox& box, const RankWord* index,
                    unsigned n_band, unsigned long long* sum, uint32_t* weight, unsigned long long* counters, cudaStream_t stream) {
  if (tiles == 0 || n_band == 0) return;
  ms_fuse_kernel<<<tiles, SM_THREADS, 0, stream>>>(table, n_entries, c, box, index, n_band, sum, weight, counters);
  B200_CUDA(cudaGetLastError());
}

void ms_active_launch(const int* ijk, const unsigned long long* sum, const uint32_t* weight, const RankWord* index, const SmBox& box,
                      unsigned n_band, unsigned min_weight, unsigned char* active, unsigned* counts, unsigned long long* counters,
                      cudaStream_t stream) {
  if (n_band == 0) return;
  ms_active_kernel<<<ms_blocks(n_band), MS_THREADS, 0, stream>>>(ijk, sum, weight, index, box, n_band, min_weight, active, counts,
                                                                  counters);
  B200_CUDA(cudaGetLastError());
}

void ms_vertex_launch(const int* ijk, const unsigned long long* sum, const uint32_t* weight, const RankWord* index, const SmBox& box,
                      unsigned n_band, const MsConst& c, const unsigned char* active, const unsigned* tile_offsets, unsigned n_vertices,
                      uint32_t* vid, float* xyz, unsigned* face_counts, unsigned long long* counters, cudaStream_t stream) {
  if (n_band == 0) return;
  ms_vertex_kernel<<<ms_blocks(n_band), MS_THREADS, 0, stream>>>(ijk, sum, weight, index, box, n_band, c, active, tile_offsets,
                                                                  n_vertices, vid, xyz, face_counts, counters);
  B200_CUDA(cudaGetLastError());
}

void ms_face_launch(const int* ijk, const unsigned long long* sum, const uint32_t* weight, const RankWord* index, const SmBox& box,
                    unsigned n_band, unsigned min_weight, const uint32_t* vid, const unsigned* face_offsets, unsigned n_faces,
                    uint32_t* faces, unsigned long long* counters, cudaStream_t stream) {
  if (n_band == 0 || n_faces == 0) return;
  ms_face_kernel<<<ms_blocks(n_band), MS_THREADS, 0, stream>>>(ijk, sum, weight, index, box, n_band, min_weight, vid, face_offsets,
                                                                n_faces, faces, counters);
  B200_CUDA(cudaGetLastError());
}

}  // namespace b200
