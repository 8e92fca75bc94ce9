// Device helpers of the rank index (occupancy bitmap + popcount prefix, see RankWord in common.cuh) and of the cloud
// bounds: shared by the target-side builders (voxel_map.cu, voxelgrid.cu, nn_grid.cu, grid_index.cu), the upload
// (cloud_codec.cu) and the probes of the NDT solver and the NN search.
#pragma once
#include <cfloat>

#include "common.cuh"

namespace b200 {

// w = {bits, prefix} of the word holding the cell, bit = cell & 31: false when the cell is empty, else true with its
// record index in `rank`. Callers load the word themselves (shared-memory copy, __ldg, plain load): the probe is only
// the arithmetic. (An early-out rather than a -1 result: after inlining, the callers' branches stay branches and the
// popcount is not evaluated for empty cells.)
__device__ __forceinline__ bool rank_probe(uint2 w, unsigned bit, unsigned& rank) {
  if (!((w.x >> bit) & 1u)) return false;
  rank = w.y + __popc(w.x & ((1u << bit) - 1u));
  return true;
}

// record index of a cell the builder has marked occupied
__device__ __forceinline__ unsigned rank_of(const RankWord* __restrict__ table, int cell) {
  unsigned r = 0;
  rank_probe(*reinterpret_cast<const uint2*>(table + (cell >> 5)), cell & 31, r);
  return r;
}

// Marks a cell occupied. Most points of a cloud land in a cell that is already marked (a 1 M-point map has ~10^4
// occupied leaves): look before the atomic. A stale read can only cause a redundant atomicOr, never a missing one.
__device__ __forceinline__ void mark_occupied(RankWord* table, int cell) {
  unsigned* word = &table[cell >> 5].bits;
  if (!((__ldcg(word) >> (cell & 31)) & 1u)) atomicOr(word, 1u << (cell & 31));
}

// Min/max of the points this thread saw (mn = FLT_MAX, mx = -FLT_MAX when none) reduced over the block and merged into
// out6 = {min xyz, max xyz} in the order-preserving encoding (decode_bounds). Every thread of the block calls it
// (blockDim.x <= 256); a block without a finite point leaves out6 alone.
__device__ __forceinline__ void block_bounds_merge(float (&mn)[3], float (&mx)[3], unsigned* out6) {
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], d));
      mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], d));
    }
  __shared__ float smn[8][3], smx[8][3];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0)
    for (int a = 0; a < 3; a++) {
      smn[warp][a] = mn[a];
      smx[warp][a] = mx[a];
    }
  __syncthreads();
  if (threadIdx.x < 3) {
    const int a = threadIdx.x;
    float lo = smn[0][a], hi = smx[0][a];
    for (int w = 1; w < (int)(blockDim.x >> 5); w++) {
      lo = fminf(lo, smn[w][a]);
      hi = fmaxf(hi, smx[w][a]);
    }
    if (lo <= hi) {  // at least one finite point in this block
      atomicMin(&out6[a], float_to_ordered(lo));
      atomicMax(&out6[3 + a], float_to_ordered(hi));
    }
  }
}

// exclusive prefix of v over the block's kThreads threads; total = the block's sum (the ASCII PCD encode and parse tiles)
template <int kThreads>
__device__ __forceinline__ unsigned block_exclusive_scan(unsigned v, unsigned& total) {
  __shared__ unsigned warp_tot[kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned incl = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const unsigned t = __shfl_up_sync(0xffffffffu, incl, d);
    if (lane >= d) incl += t;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  unsigned off = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; w++) {
    if (w < warp) off += warp_tot[w];
    tot += warp_tot[w];
  }
  total = tot;
  return off + incl - v;
}

}  // namespace b200
