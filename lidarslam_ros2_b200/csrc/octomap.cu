// K22: the OctoMap of the session's submaps (b200sm_build_octomap). Every decision follows csrc/octomap.hpp, which a
// host compile also builds: the voxel states are bits and the static map's integer counts, the pyramid is codes and
// counts reduced level by level, so the states and the .bt bytes are bitwise the host's whatever the order of the work.
#include "octomap.cuh"

namespace b200 {
namespace {

__device__ __forceinline__ bool om_bit(const uint32_t* __restrict__ bits, unsigned long long r) {
  return (__ldg(bits + (r >> 5)) >> (r & 31u)) & 1u;
}

// the linear index of a level-l cell (keys >> l) in the pyramid level; false outside it
__device__ __forceinline__ bool om_cell(const OmPyramid& p, int l, unsigned x, unsigned y, unsigned z, unsigned long long* at) {
  const unsigned wx = x - p.lo[l][0], wy = y - p.lo[l][1], wz = z - p.lo[l][2];  // wraps to large when below
  if (wx >= p.dims[l][0] || wy >= p.dims[l][1] || wz >= p.dims[l][2]) return false;
  *at = ((unsigned long long)wz * p.dims[l][1] + wy) * p.dims[l][0] + wx;
  return true;
}

// the level-l cell of pyramid index i (first[l] <= i < first[l + 1])
__device__ __forceinline__ void om_coords(const OmPyramid& p, int l, unsigned long long i, unsigned* x, unsigned* y, unsigned* z) {
  const unsigned long long r = i - p.first[l], plane = (unsigned long long)p.dims[l][0] * p.dims[l][1];
  const unsigned long long zz = r / plane, rem = r - zz * plane, yy = rem / p.dims[l][0];
  *x = p.lo[l][0] + (unsigned)(rem - yy * p.dims[l][0]);
  *y = p.lo[l][1] + (unsigned)yy;
  *z = p.lo[l][2] + (unsigned)zz;
}

// the 8 children's codes of level-l cell (x, y, z), l >= 2, child i at (2x + bit 0, 2y + bit 1, 2z + bit 2)
__device__ __forceinline__ void om_children(const OmPyramid& p, int l, unsigned x, unsigned y, unsigned z,
                                            const unsigned char* __restrict__ codes, unsigned char (&ch)[8],
                                            unsigned long long (&at)[8]) {
#pragma unroll
  for (int i = 0; i < 8; i++) {
    unsigned long long a;
    const bool in = om_cell(p, l - 1, 2 * x + (i & 1), 2 * y + ((i >> 1) & 1), 2 * z + ((i >> 2) & 1), &a);
    at[i] = in ? p.first[l - 1] + a : ~0ull;
    ch[i] = in ? codes[at[i]] : (unsigned char)OM_UNKNOWN;
  }
}

// the 8 voxels' states of level-1 cell (x, y, z) from the states array, and their linear indices in the box (~0 outside)
__device__ __forceinline__ void om_voxels(const OmPyramid& p, unsigned x, unsigned y, unsigned z, unsigned long long (&lin)[8]) {
#pragma unroll
  for (int i = 0; i < 8; i++) {
    unsigned long long a;
    lin[i] = om_cell(p, 0, 2 * x + (i & 1), 2 * y + ((i >> 1) & 1), 2 * z + ((i >> 2) & 1), &a) ? a : ~0ull;
  }
}

// K22a. Block b serves tile b of the whole map; thread t casts the rays of SM_PER_THREAD points: every voxel of the freed
// segment's walk into the box-wide bitmap, read first (a submap's rays cross the voxels near its origin over and over).
__global__ void __launch_bounds__(SM_THREADS) om_free_kernel(const SmEntry* __restrict__ table, int n_entries, SmConst c, SmBox box,
                                                             uint32_t* __restrict__ freed, unsigned long long* __restrict__ counters) {
  const int k = entry_of(table, n_entries, blockIdx.x, &SmEntry::first_tile);
  const SmEntry& e = table[k];
  const unsigned base = (blockIdx.x - e.first_tile) * (unsigned)SM_TILE + threadIdx.x;
  const long long* o = e.o;
  unsigned tripped = 0;
  for (int j = 0; j < SM_PER_THREAD; j++) {
    const unsigned i = base + j * SM_THREADS;
    if (i >= e.n) break;
    const float4 p = e.cloud[i];
    float q[3];
    og_transform(e.T, p.x, p.y, p.z, q);
    int v[3];
    long long f[3];
    if (!sm_ray(c, o, q[0], q[1], q[2], &v[0], &v[1], &v[2], &f[0], &f[1], &f[2])) continue;
    sm_walk(o[0], o[1], o[2], f[0], f[1], f[2], [&](int x, int y, int z) {
      unsigned lin;
      if (!sm_lin(box, x, y, z, &lin)) {
        tripped = 1u;
        return;
      }
      uint32_t* w = freed + (lin >> 5);
      const uint32_t bit = 1u << (lin & 31u);
      if (!(*w & bit)) atomicOr(w, bit);
    });
  }
  if (tripped) atomicAdd(&counters[SM_CTR_TRIPPED], 1ull);
}

// K22b. One thread per level-1 cell (grid-stride).
__global__ void __launch_bounds__(SM_THREADS) om_leaf_kernel(OmPyramid pyr, SmBox ebox, const RankWord* __restrict__ index,
                                                             const unsigned char* __restrict__ dynamic, unsigned n_voxels,
                                                             const uint32_t* __restrict__ freed, unsigned char* __restrict__ states,
                                                             unsigned char* __restrict__ codes, unsigned* __restrict__ counts,
                                                             unsigned long long* __restrict__ counters) {
  unsigned occ = 0, fre = 0;
  const unsigned long long n = pyr.first[2];
  for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
    unsigned x, y, z;
    om_coords(pyr, 1, i, &x, &y, &z);
    unsigned char ch[8];
#pragma unroll
    for (int b = 0; b < 8; b++) {
      const unsigned kx = 2 * x + (b & 1), ky = 2 * y + ((b >> 1) & 1), kz = 2 * z + ((b >> 2) & 1);
      unsigned long long lin;
      ch[b] = OM_UNKNOWN;
      if (!om_cell(pyr, 0, kx, ky, kz, &lin)) continue;
      unsigned r;
      const bool end = sm_rank(index, ebox, (int)kx - OM_KEY_OFFSET, (int)ky - OM_KEY_OFFSET, (int)kz - OM_KEY_OFFSET, &r) && r < n_voxels;
      ch[b] = om_state(end, end && dynamic[r], om_bit(freed, lin));
      states[lin] = ch[b];
      occ += ch[b] == OM_OCCUPIED;
      fre += ch[b] == OM_FREE;
    }
    const unsigned char code = om_parent(ch);
    codes[i] = code;
    counts[i] = code == OM_INNER ? 1u : 0u;
  }
  occ = __reduce_add_sync(0xffffffffu, occ);
  fre = __reduce_add_sync(0xffffffffu, fre);
  if ((threadIdx.x & 31) == 0) {
    if (occ) atomicAdd(&counters[OM_CTR_OCCUPIED_VOXELS], (unsigned long long)occ);
    if (fre) atomicAdd(&counters[OM_CTR_FREE_VOXELS], (unsigned long long)fre);
  }
}

// K22c. One thread per level-l cell (grid-stride).
__global__ void __launch_bounds__(SM_THREADS) om_reduce_kernel(OmPyramid pyr, int l, unsigned char* __restrict__ codes,
                                                               unsigned* __restrict__ counts) {
  for (unsigned long long i = pyr.first[l] + blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < pyr.first[l + 1];
       i += (unsigned long long)gridDim.x * blockDim.x) {
    unsigned x, y, z;
    om_coords(pyr, l, i, &x, &y, &z);
    unsigned char ch[8];
    unsigned long long at[8];
    om_children(pyr, l, x, y, z, codes, ch, at);
    const unsigned char code = om_parent(ch);
    unsigned n = 0;
    if (code == OM_INNER) {
      n = 1;
#pragma unroll
      for (int b = 0; b < 8; b++)
        if (ch[b] == OM_INNER) n += counts[at[b]];
    }
    codes[i] = code;
    counts[i] = n;
  }
}

// K22d. One thread per level-l cell (grid-stride); only inner cells act. Each child has one parent, so the in-place
// overwrite of its count is this thread's alone.
__global__ void __launch_bounds__(SM_THREADS) om_offset_kernel(OmPyramid pyr, int l, const unsigned char* __restrict__ codes,
                                                               unsigned* __restrict__ counts) {
  for (unsigned long long i = pyr.first[l] + blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < pyr.first[l + 1];
       i += (unsigned long long)gridDim.x * blockDim.x) {
    if (codes[i] != OM_INNER) continue;
    unsigned x, y, z;
    om_coords(pyr, l, i, &x, &y, &z);
    unsigned char ch[8];
    unsigned long long at[8];
    om_children(pyr, l, x, y, z, codes, ch, at);
    unsigned next = (l == OM_DEPTH ? 0u : counts[i]) + 2u;
#pragma unroll
    for (int b = 0; b < 8; b++)
      if (ch[b] == OM_INNER) {
        const unsigned n = counts[at[b]];
        counts[at[b]] = next;
        next += 2u * n;
      }
  }
}

// K22e. One thread per cell of levels 1..16 (grid-stride); only inner cells write.
__global__ void __launch_bounds__(SM_THREADS) om_write_kernel(OmPyramid pyr, const unsigned char* __restrict__ states,
                                                              const unsigned char* __restrict__ codes, const unsigned* __restrict__ counts,
                                                              unsigned char* __restrict__ out, unsigned long long n_bytes,
                                                              unsigned long long* __restrict__ counters) {
  unsigned inner = 0, occ = 0, fre = 0, tripped = 0;
  const unsigned long long n = pyr.first[OM_DEPTH + 1];
  for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
    if (codes[i] != OM_INNER) continue;
    int l = 1;
    while (l < OM_DEPTH && i >= pyr.first[l + 1]) l++;
    unsigned x, y, z;
    om_coords(pyr, l, i, &x, &y, &z);
    unsigned char ch[8];
    if (l == 1) {
      unsigned long long lin[8];
      om_voxels(pyr, x, y, z, lin);
#pragma unroll
      for (int b = 0; b < 8; b++) ch[b] = lin[b] == ~0ull ? (unsigned char)OM_UNKNOWN : states[lin[b]];
    } else {
      unsigned long long at[8];
      om_children(pyr, l, x, y, z, codes, ch, at);
    }
    const unsigned long long off = l == OM_DEPTH ? 0ull : counts[i];
    inner++;
#pragma unroll
    for (int b = 0; b < 8; b++) {
      occ += ch[b] == OM_OCCUPIED;
      fre += ch[b] == OM_FREE;
    }
    if (off + 1 < n_bytes) om_pack(ch, &out[off], &out[off + 1]);
    else tripped = 1u;
  }
  inner = __reduce_add_sync(0xffffffffu, inner);
  occ = __reduce_add_sync(0xffffffffu, occ);
  fre = __reduce_add_sync(0xffffffffu, fre);
  if ((threadIdx.x & 31) == 0) {
    if (inner) atomicAdd(&counters[OM_CTR_INNER], (unsigned long long)inner);
    if (occ) atomicAdd(&counters[OM_CTR_OCCUPIED_LEAVES], (unsigned long long)occ);
    if (fre) atomicAdd(&counters[OM_CTR_FREE_LEAVES], (unsigned long long)fre);
  }
  if (tripped) atomicAdd(&counters[SM_CTR_TRIPPED], 1ull);
}

unsigned grid_for(unsigned long long n) {
  const unsigned long long want = (n + SM_THREADS - 1) / SM_THREADS;
  return (unsigned)(want < 16ull * H100_SMS ? want : 16ull * H100_SMS);
}

}  // namespace

void om_free_launch(const SmEntry* table, int n_entries, unsigned tiles, const SmConst& c, const SmBox& box, uint32_t* freed,
                    unsigned long long* counters, cudaStream_t stream) {
  if (tiles == 0) return;
  om_free_kernel<<<tiles, SM_THREADS, 0, stream>>>(table, n_entries, c, box, freed, counters);
  B200_CUDA(cudaGetLastError());
}

void om_leaf_launch(const OmPyramid& pyr, const SmBox& ebox, const RankWord* index, const unsigned char* dynamic,
                    unsigned n_voxels, const uint32_t* freed, unsigned char* states, unsigned char* codes, unsigned* counts,
                    unsigned long long* counters, cudaStream_t stream) {
  om_leaf_kernel<<<grid_for(pyr.first[2]), SM_THREADS, 0, stream>>>(pyr, ebox, index, dynamic, n_voxels, freed, states, codes, counts,
                                                                    counters);
  B200_CUDA(cudaGetLastError());
}

void om_reduce_launch(const OmPyramid& pyr, int level, unsigned char* codes, unsigned* counts, cudaStream_t stream) {
  om_reduce_kernel<<<grid_for(pyr.first[level + 1] - pyr.first[level]), SM_THREADS, 0, stream>>>(pyr, level, codes, counts);
  B200_CUDA(cudaGetLastError());
}

void om_offset_launch(const OmPyramid& pyr, int level, const unsigned char* codes, unsigned* counts, cudaStream_t stream) {
  om_offset_kernel<<<grid_for(pyr.first[level + 1] - pyr.first[level]), SM_THREADS, 0, stream>>>(pyr, level, codes, counts);
  B200_CUDA(cudaGetLastError());
}

void om_write_launch(const OmPyramid& pyr, const unsigned char* states, const unsigned char* codes, const unsigned* counts,
                     unsigned char* out, unsigned long long n_bytes, unsigned long long* counters, cudaStream_t stream) {
  om_write_kernel<<<grid_for(pyr.first[OM_DEPTH + 1]), SM_THREADS, 0, stream>>>(pyr, states, codes, counts, out, n_bytes, counters);
  B200_CUDA(cudaGetLastError());
}

}  // namespace b200
