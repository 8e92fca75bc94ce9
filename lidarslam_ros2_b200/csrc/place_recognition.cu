// K13: Scan Context descriptors of the session's submaps and the place search over them (b200sm_search_loop_place).
// Every value follows csrc/scan_context.hpp, which a host compile also builds, so a descriptor, a column norm and a
// distance are bitwise the host's.
#include <math_constants.h>

#include <algorithm>
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
  const ScBuildEntry e = table[entry_of(table, n_entries, tile, &ScBuildEntry::first_tile)];
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

// The (minimum d, lowest s) of one query against one candidate, lanes over shifts: K13b's loop and xor tree, shared by K16.
__device__ __forceinline__ void sc_warp_best(const float* Q, const double* nQ, const float* C, const double* nC, int num_rings,
                                             int num_sectors, int lane, double* d_out, int* s_out) {
  double best = CUDART_INF;
  int bs = INT_MAX;
  for (int s = lane; s < num_sectors; s += 32) {
    const double d = sc_distance_at(Q, nQ, C, nC, num_rings, num_sectors, s);
    if (bs == INT_MAX || d < best) {
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
  *d_out = best;
  *s_out = bs;
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
    double best;
    int bs;
    sc_warp_best(Q, nQ, C, nC, num_rings, num_sectors, lane, &best, &bs);
    if (lane == 0) {
      distance[r] = best;
      shift[r] = bs;
    }
  }
}

// K16, the cross-session scores of b200sm_merge_session. Block (x, y) stages query tile x (queries x * tile ..) of the src
// descriptors and their norms in shared memory; warp w of column y of the grid streams candidates a = y * warps + w, + warps
// * gridDim.y, ... of the dst descriptors from L2 and scores each against every query of the tile with sc_warp_best.
// (D, s*) of query b and candidate a go to row b, column a of the row-major matrix.
__global__ void __launch_bounds__(SC_SEARCH_THREADS) merge_scores_kernel(const float* __restrict__ q_desc, const double* __restrict__ q_norms,
                                                                        int n_query, const float* __restrict__ c_desc,
                                                                        const double* __restrict__ c_norms, int n_cand, int tile,
                                                                        double* __restrict__ distance, int* __restrict__ shift,
                                                                        int num_rings, int num_sectors) {
  extern __shared__ double sc_smem[];
  const int nb = num_rings * num_sectors;
  const int q0 = blockIdx.x * tile, nq = min(tile, n_query - q0);
  double* nQ = sc_smem;                                   // tile * num_sectors doubles
  float* Q = reinterpret_cast<float*>(nQ + (size_t)tile * num_sectors);  // tile * nb floats
  for (int k = threadIdx.x; k < nq * nb; k += blockDim.x) Q[k] = q_desc[(size_t)q0 * nb + k];
  for (int k = threadIdx.x; k < nq * num_sectors; k += blockDim.x) nQ[k] = q_norms[(size_t)q0 * num_sectors + k];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int stride = gridDim.y * SC_SEARCH_WARPS;
  for (int a = blockIdx.y * SC_SEARCH_WARPS + (threadIdx.x >> 5); a < n_cand; a += stride) {
    const float* C = c_desc + (size_t)a * nb;
    const double* nC = c_norms + (size_t)a * num_sectors;
    for (int q = 0; q < nq; q++) {
      double d;
      int s;
      sc_warp_best(Q + (size_t)q * nb, nQ + (size_t)q * num_sectors, C, nC, num_rings, num_sectors, lane, &d, &s);
      if (lane == 0) {
        const size_t o = (size_t)(q0 + q) * n_cand + a;
        distance[o] = d;
        shift[o] = s;
      }
    }
  }
}

// K16's selection: warp b takes row b and picks, round by round, the smallest (D, a) above the previous pick with
// D < threshold; top_k rounds give the row's first top_k candidates in (D, a) order. Unused entries get a = -1.
__global__ void merge_select_kernel(const double* __restrict__ distance, const int* __restrict__ shift, int n_query, int n_cand,
                                    double threshold, int top_k, int* __restrict__ sel_a, double* __restrict__ sel_d,
                                    int* __restrict__ sel_s) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= n_query) return;
  const int lane = threadIdx.x & 31;
  const double* row = distance + (size_t)b * n_cand;
  double prev_d = -CUDART_INF;
  int prev_a = -1;
  for (int r = 0; r < top_k; r++) {
    double best = CUDART_INF;
    int ba = INT_MAX;
    for (int a = lane; a < n_cand; a += 32) {
      const double d = row[a];
      if (!(d < threshold)) continue;
      if (d < prev_d || (d == prev_d && a <= prev_a)) continue;  // already picked
      if (d < best || (d == best && a < ba)) {
        best = d;
        ba = a;
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const double od = __shfl_xor_sync(0xffffffffu, best, off);
      const int oa = __shfl_xor_sync(0xffffffffu, ba, off);
      if (od < best || (od == best && oa < ba)) {
        best = od;
        ba = oa;
      }
    }
    const size_t o = (size_t)b * top_k + r;
    if (ba == INT_MAX) {  // the row has no more candidates
      for (int k = r + lane; k < top_k; k += 32) sel_a[(size_t)b * top_k + k] = -1;
      return;
    }
    if (lane == 0) {
      sel_a[o] = ba;
      sel_d[o] = best;
      sel_s[o] = shift[(size_t)b * n_cand + ba];
    }
    prev_d = best;
    prev_a = ba;
  }
}

}  // namespace

int merge_query_tile(int num_rings, int num_sectors) {
  int dev = 0, optin = 0;
  B200_CUDA(cudaGetDevice(&dev));
  B200_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  // The scoring is latency-bound (a dependent chain of double divisions per lane), so the tile leaves room for as many
  // blocks per SM as the registers allow (48 x 256 per block: five) rather than filling one block's shared memory.
  const size_t per_query = sizeof(float) * (size_t)num_rings * num_sectors + sizeof(double) * (size_t)num_sectors;
  const size_t fit = (size_t)optin / (MERGE_BLOCKS_PER_SM * per_query);
  return (int)std::max<size_t>(1, std::min<size_t>(fit, MERGE_QUERY_TILE_MAX));
}

void merge_scores_launch(const float* q_desc, const double* q_norms, int n_query, const float* c_desc, const double* c_norms,
                         int n_cand, double* distance, int* shift, int num_rings, int num_sectors, cudaStream_t stream) {
  if (n_query <= 0 || n_cand <= 0) return;
  const int tile = merge_query_tile(num_rings, num_sectors);
  const size_t smem = ((size_t)sizeof(double) * num_sectors + sizeof(float) * (size_t)num_rings * num_sectors) * tile;
  B200_CUDA(cudaFuncSetAttribute(merge_scores_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int dev = 0, sms = 0;
  B200_CUDA(cudaGetDevice(&dev));
  B200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int tiles = (n_query + tile - 1) / tile;
  // enough columns of candidates to fill every SM, but no block without a candidate
  const int want = std::max(1, (MERGE_BLOCKS_PER_SM * sms + tiles - 1) / tiles);
  const int cols = std::min(want, (n_cand + SC_SEARCH_WARPS - 1) / SC_SEARCH_WARPS);
  merge_scores_kernel<<<dim3((unsigned)tiles, (unsigned)cols), SC_SEARCH_THREADS, smem, stream>>>(
      q_desc, q_norms, n_query, c_desc, c_norms, n_cand, tile, distance, shift, num_rings, num_sectors);
  B200_CUDA(cudaGetLastError());
}

void merge_select_launch(const double* distance, const int* shift, int n_query, int n_cand, double threshold, int top_k, int* sel_a,
                         double* sel_d, int* sel_s, cudaStream_t stream) {
  if (n_query <= 0) return;
  constexpr int warps = 8;
  merge_select_kernel<<<(n_query + warps - 1) / warps, warps * 32, 0, stream>>>(distance, shift, n_query, n_cand, threshold, top_k, sel_a,
                                                                              sel_d, sel_s);
  B200_CUDA(cudaGetLastError());
}

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
