// K19: the map consistency of the session's submaps (b200sm_build_map_consistency). Every value follows
// csrc/map_consistency.hpp, which a host compile also builds. The moment sums are exact int64 and the aggregates integer
// sums, so neither the scatter's order nor the order of the atomics changes a bit.
#include <climits>

#include "consistency.cuh"
#include "grid_index.cuh"

namespace b200 {
namespace {

// the linear index of cell (x, y, z) in the box; false outside it
__device__ __forceinline__ bool mc_lin(const SmBox& b, long long x, long long y, long long z, unsigned* lin) {
  const long long wx = x - b.lo[0], wy = y - b.lo[1], wz = z - b.lo[2];
  if (wx < 0 || wy < 0 || wz < 0 || wx >= b.dims[0] || wy >= b.dims[1] || wz >= b.dims[2]) return false;
  *lin = (unsigned)(((unsigned long long)wz * b.dims[1] + (unsigned long long)wy) * b.dims[0] + (unsigned long long)wx);
  return true;
}

// point i of entry e moved and quantised: MC_POINT_OK / SKIPPED / RANGE
__device__ __forceinline__ int mc_load(const McEntry& e, const McConst& c, unsigned i, long long* X) {
  const float4 p = e.cloud[i];
  float q[3];
  og_transform(e.T, p.x, p.y, p.z, q);
  return mc_point(c, q, X);
}

// K19a. Block b serves tile b; a thread takes MC_PER_THREAD points of it. Each warp reduces its cells and counts, then one
// lane per warp widens the entry's bounds.
__global__ void __launch_bounds__(MC_THREADS) mc_bounds_kernel(const McEntry* __restrict__ table, int n_entries, McConst c,
                                                               int* __restrict__ bounds, unsigned long long* __restrict__ counters) {
  const int k = entry_of(table, n_entries, blockIdx.x, &McEntry::first_tile);
  const McEntry& e = table[k];
  const unsigned base = (blockIdx.x - e.first_tile) * (unsigned)MC_TILE + threadIdx.x;
  int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
  unsigned used = 0, skipped = 0, range = 0;
  for (int j = 0; j < MC_PER_THREAD; j++) {
    const unsigned i = base + j * MC_THREADS;
    if (i >= e.n) break;
    long long X[3];
    const int v = mc_load(e, c, i, X);
    skipped += v == MC_POINT_SKIPPED;
    range += v == MC_POINT_RANGE;
    if (v != MC_POINT_OK) continue;
    used++;
#pragma unroll
    for (int a = 0; a < 3; a++) {
      lo[a] = min(lo[a], og_cell(X[a]));
      hi[a] = max(hi[a], og_cell(X[a]));
    }
  }
#pragma unroll
  for (int a = 0; a < 3; a++) {
    lo[a] = __reduce_min_sync(0xffffffffu, lo[a]);
    hi[a] = __reduce_max_sync(0xffffffffu, hi[a]);
  }
  used = __reduce_add_sync(0xffffffffu, used);
  skipped = __reduce_add_sync(0xffffffffu, skipped);
  range = __reduce_add_sync(0xffffffffu, range);
  if ((threadIdx.x & 31) == 0) {
    if (used)
#pragma unroll
      for (int a = 0; a < 3; a++) {
        atomicMin(&bounds[6 * k + a], lo[a]);
        atomicMax(&bounds[6 * k + 3 + a], hi[a]);
      }
    if (skipped) atomicAdd(&counters[MC_CTR_SKIPPED], (unsigned long long)skipped);
    if (range) atomicAdd(&counters[MC_CTR_RANGE], (unsigned long long)range);
  }
}

// K19b, the three passes over the points: kPass 0 marks the cell, 1 counts, 2 scatters
template <int kPass>
__global__ void __launch_bounds__(MC_THREADS) mc_cells_kernel(const McEntry* __restrict__ table, int n_entries, McConst c, SmBox box,
                                                              RankWord* __restrict__ index, unsigned* __restrict__ count,
                                                              unsigned* __restrict__ queries, const unsigned* __restrict__ start,
                                                              unsigned* __restrict__ qcursor, unsigned* __restrict__ ocursor,
                                                              ushort4* __restrict__ offs, unsigned* __restrict__ idx,
                                                              unsigned* __restrict__ n_out, double* __restrict__ h_out,
                                                              double* __restrict__ plane_out, unsigned long long* __restrict__ counters) {
  const int k = entry_of(table, n_entries, blockIdx.x, &McEntry::first_tile);
  const McEntry& e = table[k];
  const unsigned base = (blockIdx.x - e.first_tile) * (unsigned)MC_TILE + threadIdx.x;
  unsigned tripped = 0;
  for (int j = 0; j < MC_PER_THREAD; j++) {
    const unsigned i = base + j * MC_THREADS;
    if (i >= e.n) break;
    const unsigned m = e.map_offset + i;
    if (kPass == 2) {
      n_out[m] = 0;
      h_out[m] = __longlong_as_double((long long)MC_NAN_BITS);
      plane_out[m] = __longlong_as_double((long long)MC_NAN_BITS);
    }
    long long X[3];
    if (mc_load(e, c, i, X) != MC_POINT_OK) continue;
    unsigned lin;
    if (!mc_lin(box, og_cell(X[0]), og_cell(X[1]), og_cell(X[2]), &lin)) {
      tripped = 1u;
      continue;
    }
    const bool query = (long long)m % c.stride == 0;
    if (kPass == 0) {
      mark_occupied(index, (int)lin);
    } else {
      unsigned r;
      if (!rank_probe(__ldg(reinterpret_cast<const uint2*>(index + (lin >> 5))), lin & 31u, r)) {
        tripped = 1u;
        continue;
      }
      if (kPass == 1) {
        atomicAdd(&count[r], 1u);
        if (query) atomicAdd(&queries[r], 1u);
      } else {
        const unsigned nq = queries[r], cell_n = start[r + 1] - start[r];
        const unsigned slot = query ? atomicAdd(&qcursor[r], 1u) : nq + atomicAdd(&ocursor[r], 1u);
        if ((query && slot >= nq) || slot >= cell_n) {
          tripped = 1u;
          continue;
        }
        offs[start[r] + slot] = make_ushort4((unsigned short)(X[0] & 0xffff), (unsigned short)(X[1] & 0xffff),
                                             (unsigned short)(X[2] & 0xffff), 0);
        idx[start[r] + slot] = m;
      }
    }
  }
  if (tripped) atomicAdd(&counters[MC_CTR_TRIPPED], 1ull);
}

__global__ void __launch_bounds__(MC_THREADS) mc_chunks_kernel(const unsigned* __restrict__ queries, unsigned n_cells,
                                                               unsigned* __restrict__ chunks) {
  const unsigned long long r = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  if (r < n_cells) chunks[r] = (queries[r] + MC_CHUNK - 1) / MC_CHUNK;
}

// the 64-bit sum of v over the warp (every lane calls it)
__device__ __forceinline__ long long mc_warp_sum(long long v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}

// K19c + K19d. Block b finds its cell r (the last cell whose chunk_start is at most b) and serves queries
// [j MC_CHUNK, (j + 1) MC_CHUNK) of it, one per thread. The points of the 27 cells around r form one virtual list (cell by
// cell, each in its scatter order); tiles of MC_CHUNK of them are staged in shared memory as int32 offsets from the
// lower corner of cell r - (1, 1, 1), where every coordinate of the 27 cells is below 3 * 2^16, and every query thread
// runs through the tile with its moments in registers. The moments then give the query's values in the header's order
// (K19d), stored at its map index, and the per-submap rows: a warp whose queries share one submap sums its row values
// through shuffles and adds them with one lane's atomics; a mixed warp adds per lane.
__global__ void __launch_bounds__(MC_CHUNK) mc_neighbour_kernel(const unsigned* __restrict__ chunk_start, unsigned n_cells,
                                                                const unsigned* __restrict__ start, const unsigned* __restrict__ queries,
                                                                const int* __restrict__ cell_ijk, SmBox box,
                                                                const RankWord* __restrict__ index, const ushort4* __restrict__ offs,
                                                                const unsigned* __restrict__ idx, const unsigned* __restrict__ sub_first,
                                                                int n_sub, McConst c, unsigned* __restrict__ n_out,
                                                                double* __restrict__ h_out, double* __restrict__ plane_out,
                                                                unsigned long long* __restrict__ rows,
                                                                unsigned long long* __restrict__ counters) {
  __shared__ unsigned s_start[27], s_pref[28];
  __shared__ int s_base[27][3];
  __shared__ int sx[MC_CHUNK], sy[MC_CHUNK], sz[MC_CHUNK];
  const unsigned b = blockIdx.x;
  unsigned lo = 0, hi = n_cells - 1;
  while (lo < hi) {
    const unsigned mid = (lo + hi + 1) >> 1;
    if (chunk_start[mid] <= b) lo = mid;
    else hi = mid - 1;
  }
  const unsigned r = lo;
  const unsigned q0 = start[r] + (b - chunk_start[r]) * MC_CHUNK;
  const unsigned qend = start[r] + queries[r];
  const int cx = cell_ijk[3ull * r], cy = cell_ijk[3ull * r + 1], cz = cell_ijk[3ull * r + 2];
  const int t = threadIdx.x;
  if (t < 27) {
    const int dx = t % 3 - 1, dy = (t / 3) % 3 - 1, dz = t / 9 - 1;
    unsigned lin, rr, first = 0, cnt = 0;
    if (mc_lin(box, (long long)cx + dx, (long long)cy + dy, (long long)cz + dz, &lin) &&
        rank_probe(__ldg(reinterpret_cast<const uint2*>(index + (lin >> 5))), lin & 31u, rr)) {
      first = start[rr];
      cnt = start[rr + 1] - first;
    }
    s_start[t] = first;
    s_pref[t + 1] = cnt;
    s_base[t][0] = (dx + 1) << OG_FRAC_BITS;
    s_base[t][1] = (dy + 1) << OG_FRAC_BITS;
    s_base[t][2] = (dz + 1) << OG_FRAC_BITS;
  }
  __syncthreads();
  if (t == 0) {
    s_pref[0] = 0;
    for (int k = 0; k < 27; k++) s_pref[k + 1] += s_pref[k];
  }
  __syncthreads();
  const unsigned total = s_pref[27];
  const bool active = q0 + t < qend;
  int xi = 0, yi = 0, zi = 0;
  if (active) {
    const ushort4 o = offs[q0 + t];
    xi = OG_ONE + o.x;
    yi = OG_ONE + o.y;
    zi = OG_ONE + o.z;
  }
  McMoments m;
  for (unsigned base = 0; base < total; base += MC_CHUNK) {
    const unsigned v = base + t;
    if (v < total) {
      int k = 0;
      while (s_pref[k + 1] <= v) k++;
      const ushort4 o = offs[s_start[k] + (v - s_pref[k])];
      sx[t] = s_base[k][0] + o.x;
      sy[t] = s_base[k][1] + o.y;
      sz[t] = s_base[k][2] + o.z;
    }
    __syncthreads();
    if (active) {
      const int w = (int)min((unsigned)MC_CHUNK, total - base);
      for (int j = 0; j < w; j++) {
        const int dx = sx[j] - xi, dy = sy[j] - yi, dz = sz[j] - zi;
        const long long xx = (long long)dx * dx, yy = (long long)dy * dy, zz = (long long)dz * dz;
        if (xx + yy + zz <= MC_RADIUS2) {
          m.n += 1;
          m.sx += dx;
          m.sy += dy;
          m.sz += dz;
          m.sxx += xx;
          m.sxy += (long long)dx * dy;
          m.sxz += (long long)dx * dz;
          m.syy += yy;
          m.syz += (long long)dy * dz;
          m.szz += zz;
        }
      }
    }
    __syncthreads();
  }
  // K19d
  int sub = -1;
  long long valid = 0, qh = 0, ql = 0;
  if (active) {
    const unsigned mi = idx[q0 + t];
    int a = 0, z = n_sub - 1;  // the last submap whose first map index is at most mi
    while (a < z) {
      const int mid = (a + z + 1) >> 1;
      if (sub_first[mid] <= mi) a = mid;
      else z = mid - 1;
    }
    sub = a;
    double h, pv;
    if (mc_query(c, m, &h, &pv, &qh, &ql)) {
      valid = 1;
      h_out[mi] = h;
      plane_out[mi] = pv;
    }
    n_out[mi] = (unsigned)m.n;
  }
  const unsigned lane = t & 31;
  const unsigned act = __ballot_sync(0xffffffffu, active);
  if (act) {
    const int leader = __ffs(act) - 1;
    const int s0 = __shfl_sync(0xffffffffu, sub, leader);
    const bool uniform = __all_sync(0xffffffffu, !active || sub == s0);
    const long long vals[MC_ROW_COUNT] = {active ? 1ll : 0ll, valid, m.n, qh, ql};
    if (uniform) {
#pragma unroll
      for (int f = 0; f < MC_ROW_COUNT; f++) {
        const long long sum = mc_warp_sum(vals[f]);
        if (lane == (unsigned)leader && sum) atomicAdd(&rows[(size_t)MC_ROW_COUNT * s0 + f], (unsigned long long)sum);
      }
    } else if (active) {
#pragma unroll
      for (int f = 0; f < MC_ROW_COUNT; f++)
        if (vals[f]) atomicAdd(&rows[(size_t)MC_ROW_COUNT * sub + f], (unsigned long long)vals[f]);
    }
  }
  if (t == 0) {
    const unsigned nq = min((unsigned)MC_CHUNK, qend - q0);
    atomicAdd(&counters[MC_CTR_CANDIDATES], (unsigned long long)nq * total);
  }
}

__global__ void __launch_bounds__(MC_THREADS) mc_intensity_kernel(float4* __restrict__ pts, const double* __restrict__ h, size_t n) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) pts[i].w = __double2float_rn(h[i]);
}

unsigned blocks_for(unsigned long long n) { return (unsigned)((n + MC_THREADS - 1) / MC_THREADS); }

}  // namespace

void mc_bounds_launch(const McEntry* table, int n_entries, unsigned tiles, const McConst& c, int* bounds, unsigned long long* counters,
                      cudaStream_t stream) {
  if (tiles == 0) return;
  mc_bounds_kernel<<<tiles, MC_THREADS, 0, stream>>>(table, n_entries, c, bounds, counters);
  B200_CUDA(cudaGetLastError());
}

void mc_mark_launch(const McEntry* table, int n_entries, unsigned tiles, const McConst& c, const SmBox& box, RankWord* index,
                    unsigned long long* counters, cudaStream_t stream) {
  if (tiles == 0) return;
  mc_cells_kernel<0><<<tiles, MC_THREADS, 0, stream>>>(table, n_entries, c, box, index, nullptr, nullptr, nullptr, nullptr, nullptr,
                                                      nullptr, nullptr, nullptr, nullptr, nullptr, counters);
  B200_CUDA(cudaGetLastError());
}

void mc_count_launch(const McEntry* table, int n_entries, unsigned tiles, const McConst& c, const SmBox& box, const RankWord* index,
                     unsigned* count, unsigned* queries, cudaStream_t stream) {
  if (tiles == 0) return;
  mc_cells_kernel<1><<<tiles, MC_THREADS, 0, stream>>>(table, n_entries, c, box, const_cast<RankWord*>(index), count, queries, nullptr,
                                                      nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
  B200_CUDA(cudaGetLastError());
}

void mc_chunks_launch(const unsigned* queries, unsigned n_cells, unsigned* chunks, cudaStream_t stream) {
  if (n_cells == 0) return;
  mc_chunks_kernel<<<blocks_for(n_cells), MC_THREADS, 0, stream>>>(queries, n_cells, chunks);
  B200_CUDA(cudaGetLastError());
}

void mc_scatter_launch(const McEntry* table, int n_entries, unsigned tiles, const McConst& c, const SmBox& box, const RankWord* index,
                       const unsigned* start, const unsigned* queries, unsigned* qcursor, unsigned* ocursor, ushort4* offs,
                       unsigned* idx, unsigned* n_out, double* h_out, double* plane_out, unsigned long long* counters,
                       cudaStream_t stream) {
  if (tiles == 0) return;
  mc_cells_kernel<2><<<tiles, MC_THREADS, 0, stream>>>(table, n_entries, c, box, const_cast<RankWord*>(index), nullptr,
                                                      const_cast<unsigned*>(queries), start, qcursor, ocursor, offs, idx, n_out,
                                                      h_out, plane_out, counters);
  B200_CUDA(cudaGetLastError());
}

void mc_neighbour_launch(const unsigned* chunk_start, unsigned n_chunks, unsigned n_cells, const unsigned* start, const unsigned* queries,
                         const int* cell_ijk, const SmBox& box, const RankWord* index, const ushort4* offs, const unsigned* idx,
                         const unsigned* sub_first, int n_sub, const McConst& c, unsigned* n_out, double* h_out, double* plane_out,
                         unsigned long long* rows, unsigned long long* counters, cudaStream_t stream) {
  if (n_chunks == 0 || n_cells == 0) return;
  mc_neighbour_kernel<<<n_chunks, MC_CHUNK, 0, stream>>>(chunk_start, n_cells, start, queries, cell_ijk, box, index, offs, idx, sub_first,
                                                         n_sub, c, n_out, h_out, plane_out, rows, counters);
  B200_CUDA(cudaGetLastError());
}

void mc_intensity_launch(float4* pts, const double* h, size_t n, cudaStream_t stream) {
  if (n == 0) return;
  mc_intensity_kernel<<<blocks_for(n), MC_THREADS, 0, stream>>>(pts, h, n);
  B200_CUDA(cudaGetLastError());
}

}  // namespace b200
