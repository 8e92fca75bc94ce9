// K13: Scan Context descriptors of the session's submaps and the place search over them (b200sm_search_loop_place).
// Every value follows csrc/scan_context.hpp, which a host compile also builds, so a descriptor, a column norm and a
// distance are bitwise the host's.
#include <math_constants.h>

#include <climits>

#include "common.cuh"
#include "place_recognition.cuh"
#include "scan_context.hpp"

namespace b200 {
namespace {

// K13a. Block b serves tile b of the launch; its submap is the last entry with first_tile <= b. The block bins its points
// into shared-memory keys (an order-preserving atomicMax, at most 8192 bins = 32 KB) and merges the bins it touched into
// the submap's global keys with atomicMax. The maximum does not depend on the order of the atomics, so the result does not
// depend on the tiling or on which submaps share the launch.
__global__ void __launch_bounds__(SC_BUILD_THREADS) scan_context_kernel(const ScBuildEntry* __restrict__ table, int n_entries,
                                                                       uint32_t* __restrict__ keys, const double* __restrict__ tables,
                                                                       int num_rings, int num_sectors, float lidar_height) {
  extern __shared__ double sc_smem[];
  const int nb = num_rings * num_sectors;
  double* ring_b = sc_smem;
  double* sector_u = ring_b + num_rings;
  uint32_t* bins = reinterpret_cast<uint32_t*>(sector_u + 2 * num_sectors);
  for (int k = threadIdx.x; k < num_rings + 2 * num_sectors; k += blockDim.x) sc_smem[k] = tables[k];
  for (int k = threadIdx.x; k < nb; k += blockDim.x) bins[k] = 0u;
  const unsigned tile = blockIdx.x;
  int lo = 0, hi = n_entries - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (table[mid].first_tile <= tile) lo = mid;
    else hi = mid - 1;
  }
  const ScBuildEntry e = table[lo];
  __syncthreads();
  const unsigned base = (tile - e.first_tile) * (unsigned)SC_BUILD_TILE + threadIdx.x;
  for (int j = 0; j < SC_BUILD_PER_THREAD; j++) {
    const unsigned i = base + j * SC_BUILD_THREADS;
    if (i >= e.n) break;
    const float4 p = e.cloud[i];
    const int b = sc_bin(p.x, p.y, p.z, ring_b, num_rings, sector_u, num_sectors);
    if (b >= 0) atomicMax(&bins[b], sc_order_key(sc_value(p.z, lidar_height)));
  }
  __syncthreads();
  uint32_t* __restrict__ dst = keys + (size_t)e.slot * nb;
  for (int k = threadIdx.x; k < nb; k += blockDim.x) {
    const uint32_t v = bins[k];
    if (v) atomicMax(&dst[k], v);
  }
}

// K13a's finishing pass: thread (slot, column j) turns the column's keys into floats in place, then sums its norm.
__global__ void scan_context_finish_kernel(uint32_t* __restrict__ keys, double* __restrict__ norms, size_t first_slot, size_t n_cols,
                                           int num_rings, int num_sectors) {
  const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (t >= n_cols) return;
  const size_t slot = first_slot + t / num_sectors;
  const int j = (int)(t % num_sectors);
  uint32_t* D = keys + slot * (size_t)num_rings * num_sectors;
  for (int i = 0; i < num_rings; i++) D[i * num_sectors + j] = __float_as_uint(sc_from_key(D[i * num_sectors + j]));
  norms[slot * num_sectors + j] = sc_column_norm(reinterpret_cast<const float*>(D), num_rings, num_sectors, j);
}

constexpr int SC_SEARCH_THREADS = 256, SC_SEARCH_WARPS = SC_SEARCH_THREADS / 32;

// K13b. The query descriptor and its norms are staged in shared memory; warp w of the grid scores candidates w, w + warps,
// ...; lane l takes the shifts l, l + 32, ... in ascending order, each summed in scan_context.hpp's fixed order, and keeps
// the first minimum. The lanes' (d, s) pairs are then reduced by a fixed xor tree that keeps the smaller d and, on equal d,
// the lower s: the minimum over all shifts with the lowest shift that attains it, whatever the lane that found it.
__global__ void __launch_bounds__(SC_SEARCH_THREADS) scan_context_search_kernel(const float* __restrict__ desc, const double* __restrict__ norms,
                                                                               size_t query_slot, const int* __restrict__ ids, int n_ids,
                                                                               double* __restrict__ distance, int* __restrict__ shift,
                                                                               int num_rings, int num_sectors) {
  extern __shared__ double sc_smem[];
  const int nb = num_rings * num_sectors;
  double* nQ = sc_smem;
  float* Q = reinterpret_cast<float*>(nQ + num_sectors);
  for (int k = threadIdx.x; k < nb; k += blockDim.x) Q[k] = desc[query_slot * nb + k];
  for (int k = threadIdx.x; k < num_sectors; k += blockDim.x) nQ[k] = norms[query_slot * num_sectors + k];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (int r = blockIdx.x * SC_SEARCH_WARPS + (threadIdx.x >> 5); r < n_ids; r += gridDim.x * SC_SEARCH_WARPS) {
    const size_t c = (size_t)ids[r];
    const float* C = desc + c * nb;
    const double* nC = norms + c * num_sectors;
    double best = CUDART_INF;  // a lane without a shift never wins the reduction
    int bs = INT_MAX;
    for (int s = lane; s < num_sectors; s += 32) {
      const double d = sc_distance_at(Q, nQ, C, nC, num_rings, num_sectors, s);
      if (bs == INT_MAX || d < best) {  // the lane's first shift, then a strictly smaller d
        best = d;
        bs = s;
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const double od = __shfl_xor_sync(0xffffffffu, best, off);
      const int os = __shfl_xor_sync(0xffffffffu, bs, off);
      if (od < best || (od == best && os < bs)) {
        best = od;
        bs = os;
      }
    }
    if (lane == 0) {
      distance[r] = best;
      shift[r] = bs;
    }
  }
}

}  // namespace

void sc_build_launch(const ScBuildEntry* table, int n_entries, unsigned tiles, uint32_t* keys, const double* tables, int num_rings,
                     int num_sectors, float lidar_height, cudaStream_t stream) {
  if (tiles == 0) return;
  const size_t smem = sizeof(double) * (num_rings + 2 * (size_t)num_sectors) + sizeof(uint32_t) * (size_t)num_rings * num_sectors;
  scan_context_kernel<<<tiles, SC_BUILD_THREADS, smem, stream>>>(table, n_entries, keys, tables, num_rings, num_sectors, lidar_height);
  B200_CUDA(cudaGetLastError());
}

void sc_finish_launch(uint32_t* keys, double* norms, size_t first_slot, size_t n_slots, int num_rings, int num_sectors,
                      cudaStream_t stream) {
  const size_t cols = n_slots * (size_t)num_sectors;
  if (cols == 0) return;
  scan_context_finish_kernel<<<(unsigned)((cols + 255) / 256), 256, 0, stream>>>(keys, norms, first_slot, cols, num_rings, num_sectors);
  B200_CUDA(cudaGetLastError());
}

void sc_search_launch(const float* desc, const double* norms, size_t query_slot, const int* ids, int n_ids, double* distance,
                      int* shift, int num_rings, int num_sectors, cudaStream_t stream) {
  if (n_ids <= 0) return;
  const size_t smem = sizeof(double) * (size_t)num_sectors + sizeof(float) * (size_t)num_rings * num_sectors;
  int dev = 0, sms = 0;
  B200_CUDA(cudaGetDevice(&dev));
  B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int want = (n_ids + SC_SEARCH_WARPS - 1) / SC_SEARCH_WARPS;
  const int blocks = want < 4 * sms ? want : 4 * sms;
  scan_context_search_kernel<<<blocks, SC_SEARCH_THREADS, smem, stream>>>(desc, norms, query_slot, ids, n_ids, distance, shift,
                                                                         num_rings, num_sectors);
  B200_CUDA(cudaGetLastError());
}

}  // namespace b200
