// K17: the branch-and-bound relocalisation search of b200sm_relocalize (csrc/relocalize.hpp holds the definitions).
//   K17a  map bounds (integer min / max of the projected cells), then the projection into g_0
//   K17b  one pyramid level per launch, one thread per stored cell
//   K17c  the discretised scan: band flags, ordered compaction, the yaw_steps x m offsets table
//   K17d  node scoring, one warp per node (lanes stride over the points, int32 sums reduced across the warp: exact and
//         order-free); implicit roots or a stored list; the tile maxima, a count pass or a write pass of the children
//   K17e  child expansion: count per block, counter_scan_async, write at block offset + rank (cut_write_kernel's pattern);
//         every store is bounded by the counted total, a destination beyond it raises a flag instead
//   dive  one block per path, all levels in one launch
// Every grid read goes through rl_read (bounds-checked), every list write is checked against its counted total.
#include <climits>
#include <cstring>

#include "relocalize.cuh"

namespace b200 {
namespace {

constexpr int RL_THREADS = 256, RL_WARPS = RL_THREADS / 32, RL_NODES_PER_BLOCK = RL_THREADS;
enum : int { RL_MODE_TILE = 0, RL_MODE_LEAF, RL_MODE_COUNT, RL_MODE_WRITE, RL_MODE_SCORES };

struct RlDev {
  const unsigned char* pyr;
  unsigned long long off[RL_MAX_LEVELS];
  RlGrid g;
  const RlOff* offs;
  long long m;
};
struct Rot9 {
  float r[9];
};

// The device time of a call's launches: an event pair around each run of launches between two host waits, summed once the
// stream is idle. The waits and the host work between runs are not counted.
class SegmentTimer {
 public:
  explicit SegmentTimer(cudaStream_t s) : s_(s) {}
  SegmentTimer(const SegmentTimer&) = delete;
  SegmentTimer& operator=(const SegmentTimer&) = delete;
  ~SegmentTimer() {
    for (cudaEvent_t e : ev_) cudaEventDestroy(e);
  }
  void begin() { record(); }
  void end() {
    if (ev_.size() % 2) record();
  }
  float total() const {  // the stream has been synchronised since the last end()
    float sum = 0;
    for (size_t k = 0; k + 1 < ev_.size(); k += 2) {
      float ms = 0;
      B200_CUDA(cudaEventElapsedTime(&ms, ev_[k], ev_[k + 1]));
      sum += ms;
    }
    return sum;
  }

 private:
  void record() {
    cudaEvent_t e;
    B200_CUDA(cudaEventCreate(&e));
    ev_.push_back(e);
    B200_CUDA(cudaEventRecord(e, s_));
  }
  cudaStream_t s_;
  std::vector<cudaEvent_t> ev_;
};

unsigned blocks_for(unsigned long long n, unsigned long long per) { return (unsigned)std::min<unsigned long long>((n + per - 1) / per, 1u << 20); }

// K17a
__global__ void __launch_bounds__(RL_THREADS) rl_bounds_kernel(const float4* __restrict__ map, size_t n, double inv, double z_min,
                                                               double z_max, int* __restrict__ box, unsigned long long* __restrict__ count) {
  int mni = INT_MAX, mnj = INT_MAX, mxi = INT_MIN, mxj = INT_MIN;
  unsigned c = 0;
  for (size_t q = blockIdx.x * (size_t)blockDim.x + threadIdx.x; q < n; q += (size_t)gridDim.x * blockDim.x) {
    const float4 p = map[q];
    int ci, cj;
    if (rl_project_row(p.x, p.y, p.z, inv, z_min, z_max, &ci, &cj)) {
      mni = min(mni, ci);
      mnj = min(mnj, cj);
      mxi = max(mxi, ci);
      mxj = max(mxj, cj);
      c++;
    }
  }
  mni = __reduce_min_sync(0xffffffffu, mni);
  mnj = __reduce_min_sync(0xffffffffu, mnj);
  mxi = __reduce_max_sync(0xffffffffu, mxi);
  mxj = __reduce_max_sync(0xffffffffu, mxj);
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) {
    atomicMin(box + 0, mni);
    atomicMin(box + 1, mnj);
    atomicMax(box + 2, mxi);
    atomicMax(box + 3, mxj);
    atomicAdd(count, (unsigned long long)c);
  }
}

__global__ void __launch_bounds__(RL_THREADS) rl_project_kernel(const float4* __restrict__ map, size_t n, double inv, double z_min,
                                                                double z_max, RlGrid g, unsigned char* __restrict__ g0,
                                                                unsigned* __restrict__ tripped) {
  for (size_t q = blockIdx.x * (size_t)blockDim.x + threadIdx.x; q < n; q += (size_t)gridDim.x * blockDim.x) {
    const float4 p = map[q];
    int ci, cj;
    if (!rl_project_row(p.x, p.y, p.z, inv, z_min, z_max, &ci, &cj)) continue;
    const long long c = (long long)ci - g.i0, r = (long long)cj - g.j0;
    if (c >= 0 && c < g.W && r >= 0 && r < g.H) g0[r * g.W + c] = 1;
    else atomicOr(tripped, 1u);
  }
}

// K17b
__global__ void __launch_bounds__(RL_THREADS) rl_level_kernel(const unsigned char* __restrict__ prev, RlGrid g, int h,
                                                              unsigned char* __restrict__ out) {
  const long long lw = rl_level_w(g, h), total = lw * rl_level_h(g, h);
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < total; q += (long long)gridDim.x * blockDim.x)
    out[q] = rl_level_cell(prev, g, h, q % lw, q / lw);
}

// K17c
__global__ void __launch_bounds__(RL_THREADS) rl_band_kernel(const float4* __restrict__ scan, size_t n, Rot9 R, double z0, double z_min,
                                                             double z_max, unsigned* __restrict__ flags) {
  const size_t q = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (q >= n) return;
  const float4 p = scan[q];
  flags[q] = rl_point_in_band(R.r, p.x, p.y, p.z, z0, z_min, z_max) ? 1u : 0u;
}

__global__ void __launch_bounds__(RL_THREADS) rl_compact_kernel(const float4* __restrict__ scan, size_t n, Rot9 R, double z0, double z_min,
                                                                double z_max, const unsigned* __restrict__ pos, unsigned m,
                                                                float4* __restrict__ out, unsigned* __restrict__ tripped) {
  const size_t q = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (q >= n) return;
  const float4 p = scan[q];
  if (!rl_point_in_band(R.r, p.x, p.y, p.z, z0, z_min, z_max)) return;
  if (pos[q] < m) out[pos[q]] = p;
  else atomicOr(tripped, 1u);
}

__global__ void __launch_bounds__(RL_THREADS) rl_offsets_kernel(const float4* __restrict__ pts, long long m, const float* __restrict__ rot,
                                                                int yaw_steps, double inv, RlOff* __restrict__ offs) {
  const long long total = m * yaw_steps;
  for (long long q = blockIdx.x * (long long)blockDim.x + threadIdx.x; q < total; q += (long long)gridDim.x * blockDim.x) {
    const long long k = q / m, t = q % m;
    const float4 p = pts[t];
    offs[q] = rl_offsets(rot + 9 * k, p.x, p.y, p.z, inv);
  }
}

// K17d: score_h of one node by a warp; every lane returns the sum
__device__ __forceinline__ int rl_warp_score(const RlDev& d, int h, RlNode n, int lane) {
  const unsigned char* __restrict__ lvl = d.pyr + d.off[h];
  const long long lw = rl_level_w(d.g, h), lh = rl_level_h(d.g, h), mg = rl_margin(h);
  const int2* __restrict__ o = reinterpret_cast<const int2*>(d.offs + (size_t)n.k * (size_t)d.m);
  int s = 0;
  for (long long t = lane; t < d.m; t += 32) {
    const int2 v = __ldg(o + t);
    s += rl_read(lvl, lw, lh, mg, (long long)n.i + v.x, (long long)n.j + v.y);
  }
  return __reduce_add_sync(0xffffffffu, s);
}

// K17d / K17e. Block b serves nodes [256 b, 256 b + 256): warp w scores nodes 256 b + 32 w + q one after the other and lane
// q keeps node q's score (with `stored`, lane q reads node q's score from an earlier pass instead); with `scores`, every
// node's score is stored. Then, by mode: TILE folds every node's key into its tile (the roots' pass), LEAF folds the leaves
// with score >= T, SCORES only stores, COUNT sums the children of the nodes with score >= T per block (counts[b], and
// *total in 64 bits), WRITE stores them at offsets[b] + their rank in the block (node order, then child order).
template <bool ROOTS>
__global__ void __launch_bounds__(RL_THREADS) rl_nodes_kernel(RlDev d, int h, int mode, const RlNode* __restrict__ list,
                                                              unsigned long long count, long long T,
                                                              unsigned long long* __restrict__ tile_keys, int* __restrict__ scores,
                                                              unsigned* __restrict__ counts, unsigned long long* __restrict__ total,
                                                              unsigned out_total, RlNode* __restrict__ out,
                                                              unsigned* __restrict__ tripped, const int* __restrict__ stored) {
  __shared__ unsigned warp_count[RL_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned long long first = (unsigned long long)blockIdx.x * RL_NODES_PER_BLOCK + (unsigned long long)warp * 32;
  int mine = -1;
  RlNode node{0, 0, 0};
  if (stored) {  // the scores an earlier pass over the same nodes stored: lane q reads node q's
    const unsigned long long idx = first + lane;
    if (idx < count) {
      mine = stored[idx];
      node = ROOTS ? rl_root(d.g, idx) : list[idx];
    }
  } else {
    for (int q = 0; q < 32; q++) {
      const unsigned long long idx = first + q;
      if (idx >= count) break;  // the same for every lane
      const RlNode n = ROOTS ? rl_root(d.g, idx) : list[idx];
      const int s = rl_warp_score(d, h, n, lane);
      if (lane == q) {
        mine = s;
        node = n;
      }
    }
  }
  const bool valid = mine >= 0;
  if (scores && valid) scores[first + lane] = mine;  // for the next pass over these nodes, or the caller
  if (mode == RL_MODE_SCORES) return;
  if (mode == RL_MODE_TILE || mode == RL_MODE_LEAF) {
    if (valid && (mode == RL_MODE_TILE || mine >= T))
      atomicMax(tile_keys + rl_tile_of(d.g, node.i, node.j), rl_key(mine, rl_leaf_index(d.g, node.k, node.i, node.j)));
    return;
  }
  const unsigned c = (valid && mine >= T) ? (unsigned)rl_child_count(d.g, node, h) : 0u;
  unsigned incl = c;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) warp_count[warp] = incl;
  __syncthreads();
  if (mode == RL_MODE_COUNT) {
    if (threadIdx.x == 0) {
      unsigned t = 0;
#pragma unroll
      for (int w = 0; w < RL_WARPS; w++) t += warp_count[w];
      counts[blockIdx.x] = t;
      atomicAdd(total, (unsigned long long)t);
    }
    return;
  }
  unsigned base = counts[blockIdx.x] + (incl - c);
  for (int w = 0; w < warp; w++) base += warp_count[w];
  for (int ch = 0; ch < 4 && c; ch++) {
    RlNode n;
    if (!rl_child(d.g, node, h, ch, &n)) continue;
    if (base < out_total) out[base] = n;
    else atomicOr(tripped, 1u);
    base++;
  }
}

// The dive: block b descends from starts[b], four warps scoring the four children of the current node per level; the
// child with the highest key goes on. leaf_scores[b] = the leaf's score.
__global__ void __launch_bounds__(128) rl_dive_kernel(RlDev d, const RlNode* __restrict__ starts, long long* __restrict__ leaf_scores) {
  __shared__ unsigned long long keys[4];
  __shared__ RlNode kids[4];
  __shared__ RlNode cur;
  __shared__ long long score;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) cur = starts[blockIdx.x];
  __syncthreads();
  if (d.g.levels == 1) {
    if (warp == 0) {
      const int s = rl_warp_score(d, 0, cur, lane);
      if (lane == 0) leaf_scores[blockIdx.x] = s;
    }
    return;
  }
  for (int h = d.g.levels - 1; h >= 1; h--) {
    RlNode ch{0, 0, 0};
    unsigned long long key = 0;
    if (rl_child(d.g, cur, h, warp, &ch)) key = rl_key(rl_warp_score(d, h - 1, ch, lane), rl_leaf_index(d.g, ch.k, ch.i, ch.j));
    if (lane == 0) {
      keys[warp] = key;
      kids[warp] = ch;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int b = 0;
      for (int c = 1; c < 4; c++)
        if (keys[c] > keys[b]) b = c;
      cur = kids[b];
      score = rl_key_score(keys[b]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) leaf_scores[blockIdx.x] = score;
}

}  // namespace

int Relocalizer::ensure_pyramid(const float4* map, size_t n, const RlParams& p, std::string& why, cudaStream_t s) {
  if (built_ && built_for_.resolution == p.resolution && built_for_.z_min == p.z_min && built_for_.z_max == p.z_max &&
      built_for_.num_levels == p.num_levels)
    return B200REG_OK;
  built_ = false;
  const double inv = 1.0 / p.resolution;
  box_.ensure(4);
  ctr_.ensure(1);
  tripped_.ensure(1);
  const int init[4] = {INT_MAX, INT_MAX, INT_MIN, INT_MIN};
  B200_CUDA(cudaMemcpyAsync(box_.ptr, init, sizeof(init), cudaMemcpyHostToDevice, s));
  B200_CUDA(cudaMemsetAsync(ctr_.ptr, 0, sizeof(unsigned long long), s));
  B200_CUDA(cudaMemsetAsync(tripped_.ptr, 0, sizeof(unsigned), s));
  rl_bounds_kernel<<<blocks_for(n, RL_THREADS * 4), RL_THREADS, 0, s>>>(map, n, inv, p.z_min, p.z_max, box_.ptr, ctr_.ptr);
  B200_CUDA(cudaGetLastError());
  int box[4];
  unsigned long long projected = 0;
  B200_CUDA(cudaMemcpyAsync(box, box_.ptr, sizeof(box), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaMemcpyAsync(&projected, ctr_.ptr, sizeof(projected), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  launches += 1;
  level_off_.assign((size_t)p.num_levels + 1, 0);
  grid = RlGrid();
  grid.levels = p.num_levels;
  if (projected) {
    why = rl_make_grid(box[0], box[1], box[2], box[3], p, &grid, level_off_.data());
    if (!why.empty()) {
      grid = RlGrid();
      return B200REG_ERR_ARG;
    }
    pyr_.ensure(level_off_[(size_t)p.num_levels]);
    B200_CUDA(cudaMemsetAsync(pyr_.ptr, 0, grid.W * grid.H, s));
    rl_project_kernel<<<blocks_for(n, RL_THREADS * 4), RL_THREADS, 0, s>>>(map, n, inv, p.z_min, p.z_max, grid, pyr_.ptr, tripped_.ptr);
    B200_CUDA(cudaGetLastError());
    launches += 1;
    for (int h = 1; h < p.num_levels; h++) {
      const unsigned long long cells = level_off_[(size_t)h + 1] - level_off_[(size_t)h];
      rl_level_kernel<<<blocks_for(cells, RL_THREADS * 4), RL_THREADS, 0, s>>>(pyr_.ptr + level_off_[(size_t)h - 1], grid, h,
                                                                              pyr_.ptr + level_off_[(size_t)h]);
      B200_CUDA(cudaGetLastError());
      launches += 1;
    }
    unsigned flag = 0;
    B200_CUDA(cudaMemcpyAsync(&flag, tripped_.ptr, sizeof(flag), cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaStreamSynchronize(s));
    if (flag) throw CudaError("relocalize: a map row projected outside the measured grid (nothing was stored there)");
  }
  built_ = true;
  built_for_ = p;
  builds += 1;
  m_ = -1;  // node scores refer to a pyramid
  return B200REG_OK;
}

int Relocalizer::search(const float4* scan, size_t n, const std::vector<float>& rot_f, double z0, const RlParams& p, RlSearchInfo& out,
                        std::string& why, cudaStream_t s) {
  out = RlSearchInfo();
  m_ = -1;
  const int Y = p.yaw_steps;
  // the limits that depend on the headings, for this call's yaw_steps (the pyramid may have been built for others),
  // before anything is launched
  grid.yaw_steps = Y;
  if (grid.W) {
    why = rl_check_headings(grid, Y);
    if (!why.empty()) return B200REG_ERR_ARG;
  }
  const double inv = 1.0 / p.resolution;
  SegmentTimer timer(s);
  // K17c: the discretised scan
  Rot9 R0;
  std::memcpy(R0.r, rot_f.data(), sizeof(R0.r));
  flags_.ensure(n + 1);
  timer.begin();
  rl_band_kernel<<<(unsigned)((n + RL_THREADS - 1) / RL_THREADS), RL_THREADS, 0, s>>>(scan, n, R0, z0, p.z_min, p.z_max, flags_.ptr);
  B200_CUDA(cudaGetLastError());
  counter_scan_async(flags_.ptr, n, scan_tmp_, s);
  timer.end();
  unsigned m = 0;
  B200_CUDA(cudaMemcpyAsync(&m, flags_.ptr + n, sizeof(unsigned), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  launches += 2;
  out.m = m;
  out.t0 = rl_t0(p.min_score, m);
  why = rl_check_points(m, Y);
  if (!why.empty()) return B200REG_ERR_ARG;
  yaw_ = Y;
  if (m == 0) {
    m_ = 0;
    out.ms = timer.total();
    return B200REG_OK;
  }
  pts_.ensure(m);
  rot_.ensure(rot_f.size());
  offs_.ensure((size_t)m * Y);
  tripped_.ensure(1);
  timer.begin();
  B200_CUDA(cudaMemsetAsync(tripped_.ptr, 0, sizeof(unsigned), s));
  B200_CUDA(cudaMemcpyAsync(rot_.ptr, rot_f.data(), rot_f.size() * sizeof(float), cudaMemcpyHostToDevice, s));
  rl_compact_kernel<<<(unsigned)((n + RL_THREADS - 1) / RL_THREADS), RL_THREADS, 0, s>>>(scan, n, R0, z0, p.z_min, p.z_max, flags_.ptr,
                                                                                         m, pts_.ptr, tripped_.ptr);
  B200_CUDA(cudaGetLastError());
  rl_offsets_kernel<<<blocks_for((unsigned long long)m * Y, RL_THREADS * 4), RL_THREADS, 0, s>>>(pts_.ptr, m, rot_.ptr, Y, inv, offs_.ptr);
  B200_CUDA(cudaGetLastError());
  launches += 2;
  m_ = m;
  if (grid.W == 0) {
    timer.end();
    B200_CUDA(cudaStreamSynchronize(s));
    out.ms = timer.total();
    return B200REG_OK;
  }

  const RlGrid& g = grid;
  const int L = g.levels;
  RlDev d;
  d.pyr = pyr_.ptr;
  for (int h = 0; h < RL_MAX_LEVELS; h++) d.off[h] = h <= L ? level_off_[(size_t)std::min(h, L)] : 0;
  d.g = g;
  d.offs = offs_.ptr;
  d.m = m;
  const size_t n_tiles = (size_t)(g.TW * g.TH);
  const unsigned long long roots = (unsigned long long)Y * n_tiles;  // <= 2^32 (rl_check_headings)
  out.nodes[L - 1] = (long long)roots;
  // (1) the roots; their scores are kept for the count and write passes when they fit the frontier's budget
  const bool keep_roots = L > 1 && roots <= RL_MAX_FRONTIER;
  if (keep_roots) root_scores_.ensure(roots);
  int* root_scores = keep_roots ? root_scores_.ptr : nullptr;
  keys_.ensure(n_tiles);
  B200_CUDA(cudaMemsetAsync(keys_.ptr, 0, n_tiles * sizeof(unsigned long long), s));
  const unsigned root_blocks = (unsigned)((roots + RL_NODES_PER_BLOCK - 1) / RL_NODES_PER_BLOCK);
  rl_nodes_kernel<true><<<root_blocks, RL_THREADS, 0, s>>>(d, L - 1, RL_MODE_TILE, nullptr, roots, 0, keys_.ptr, root_scores, nullptr,
                                                          nullptr, 0, nullptr, nullptr, nullptr);
  B200_CUDA(cudaGetLastError());
  timer.end();
  std::vector<unsigned long long> root_keys(n_tiles);
  B200_CUDA(cudaMemcpyAsync(root_keys.data(), keys_.ptr, n_tiles * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  launches += 1;
  // (2) the dive, (3) T
  std::vector<RlNode> starts;
  for (long long t : rl_top_tiles(root_keys, 0, p.top_k)) {
    const long long idx = rl_key_index(root_keys[(size_t)t]);
    starts.push_back(RlNode{(int)(idx / (g.W * g.H)), (int)(idx % g.W), (int)((idx / g.W) % g.H)});
  }
  std::vector<long long> dive_scores(starts.size());
  if (!starts.empty()) {
    starts_.ensure(starts.size());
    dive_scores_.ensure(starts.size());
    timer.begin();
    B200_CUDA(cudaMemcpyAsync(starts_.ptr, starts.data(), starts.size() * sizeof(RlNode), cudaMemcpyHostToDevice, s));
    rl_dive_kernel<<<(unsigned)starts.size(), 128, 0, s>>>(d, starts_.ptr, dive_scores_.ptr);
    B200_CUDA(cudaGetLastError());
    timer.end();
    B200_CUDA(cudaMemcpyAsync(dive_scores.data(), dive_scores_.ptr, starts.size() * sizeof(long long), cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaStreamSynchronize(s));
    launches += 1;
  }
  out.t = rl_threshold(dive_scores, out.t0, p.top_k);
  const long long T = out.t;
  // (4) the expansion, (5) the leaves. With one level the roots are the leaves: the top_k tiles >= T0 are all >= T (T > T0
  // only when top_k dives, in distinct tiles, reach it), so they are ranked from the roots' keys as they are.
  std::vector<unsigned long long> leaf_keys;
  if (L > 1) {
    timer.begin();
    B200_CUDA(cudaMemsetAsync(keys_.ptr, 0, n_tiles * sizeof(unsigned long long), s));
    unsigned long long total = 0;
    // the count pass over `cnt` nodes of level h; stored: their scores from an earlier pass, else they are scored (and
    // kept in `keep` for the write pass when it is given)
    auto count_pass = [&](bool implicit, int h, const RlNode* list, unsigned long long cnt, const int* stored, int* keep) {
      const unsigned blocks = (unsigned)((cnt + RL_NODES_PER_BLOCK - 1) / RL_NODES_PER_BLOCK);
      counts_.ensure((size_t)blocks + 1);
      B200_CUDA(cudaMemsetAsync(ctr_.ptr, 0, sizeof(unsigned long long), s));
      if (implicit)
        rl_nodes_kernel<true><<<blocks, RL_THREADS, 0, s>>>(d, h, RL_MODE_COUNT, nullptr, cnt, T, nullptr, keep, counts_.ptr, ctr_.ptr, 0,
                                                            nullptr, nullptr, stored);
      else
        rl_nodes_kernel<false><<<blocks, RL_THREADS, 0, s>>>(d, h, RL_MODE_COUNT, list, cnt, T, nullptr, keep, counts_.ptr, ctr_.ptr, 0,
                                                             nullptr, nullptr, stored);
      B200_CUDA(cudaGetLastError());
      timer.end();
      B200_CUDA(cudaMemcpyAsync(&total, ctr_.ptr, sizeof(total), cudaMemcpyDeviceToHost, s));
      B200_CUDA(cudaStreamSynchronize(s));
      launches += 1;
      return blocks;
    };
    const int* level_scores = root_scores;  // the scores of the nodes being expanded, when kept
    unsigned blocks = count_pass(true, L - 1, nullptr, roots, root_scores, nullptr);
    int cur = 0;
    unsigned long long n_front = 0;
    for (int h = L - 2; h >= 0; h--) {
      if (total > RL_MAX_FRONTIER) {
        char msg[160];
        std::snprintf(msg, sizeof(msg), "level %d would store %llu nodes, more than 2^26", h, total);
        why = msg;
        return B200REG_ERR_ARG;
      }
      // children of the level-(h + 1) nodes with score >= T, written in node order
      RlNode* dst = nullptr;
      if (total) {
        front_[cur ^ 1].ensure(total);
        node_scores_[cur ^ 1].ensure(total);  // the children's scores, kept by their count pass (front_[cur] keeps its own)
        dst = front_[cur ^ 1].ptr;
      }
      timer.begin();
      counter_scan_async(counts_.ptr, blocks, scan_tmp_, s);
      B200_CUDA(cudaMemsetAsync(tripped_.ptr, 0, sizeof(unsigned), s));
      if (h == L - 2)
        rl_nodes_kernel<true><<<blocks, RL_THREADS, 0, s>>>(d, h + 1, RL_MODE_WRITE, nullptr, roots, T, nullptr, nullptr, counts_.ptr, nullptr,
                                                            (unsigned)total, dst, tripped_.ptr, level_scores);
      else
        rl_nodes_kernel<false><<<blocks, RL_THREADS, 0, s>>>(d, h + 1, RL_MODE_WRITE, front_[cur].ptr, n_front, T, nullptr, nullptr,
                                                             counts_.ptr, nullptr, (unsigned)total, dst, tripped_.ptr, level_scores);
      B200_CUDA(cudaGetLastError());
      timer.end();
      unsigned flag = 0;
      B200_CUDA(cudaMemcpyAsync(&flag, tripped_.ptr, sizeof(flag), cudaMemcpyDeviceToHost, s));
      B200_CUDA(cudaStreamSynchronize(s));
      launches += 2;
      if (flag) throw CudaError("relocalize: the expansion's write pass met a child beyond the counted total (nothing was stored there)");
      cur ^= 1;
      n_front = total;
      out.nodes[h] = (long long)n_front;
      if (n_front == 0) break;
      timer.begin();
      if (h > 0) {
        blocks = count_pass(false, h, front_[cur].ptr, n_front, nullptr, node_scores_[cur].ptr);
        level_scores = node_scores_[cur].ptr;
      } else {
        rl_nodes_kernel<false><<<(unsigned)((n_front + RL_NODES_PER_BLOCK - 1) / RL_NODES_PER_BLOCK), RL_THREADS, 0, s>>>(
            d, 0, RL_MODE_LEAF, front_[cur].ptr, n_front, T, keys_.ptr, nullptr, nullptr, nullptr, 0, nullptr, nullptr, nullptr);
        B200_CUDA(cudaGetLastError());
        timer.end();
        launches += 1;
      }
    }
    leaf_keys.resize(n_tiles);
    B200_CUDA(cudaMemcpyAsync(leaf_keys.data(), keys_.ptr, n_tiles * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  }
  B200_CUDA(cudaStreamSynchronize(s));
  out.ms = timer.total();
  const std::vector<unsigned long long>& ranked = L > 1 ? leaf_keys : root_keys;
  out.tiles = rl_top_tiles(ranked, out.t0, p.top_k);
  for (long long t : out.tiles) out.keys.push_back(ranked[(size_t)t]);
  return B200REG_OK;
}

int Relocalizer::read_level(int h, unsigned char* out, size_t capacity, long long* w, long long* hh, std::string& why, cudaStream_t s) {
  if (!built_ || h < 0 || h >= grid.levels) {
    why = "get_relocalize_grid: no pyramid, or the level is not one of it";
    return B200REG_ERR_ARG;
  }
  const long long lw = grid.W ? rl_level_w(grid, h) : 0, lh = grid.H ? rl_level_h(grid, h) : 0;
  if (w) *w = lw;
  if (hh) *hh = lh;
  const size_t k = std::min(capacity, (size_t)(lw * lh));
  if (out && k) {
    B200_CUDA(cudaMemcpyAsync(out, pyr_.ptr + level_off_[(size_t)h], k, cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaStreamSynchronize(s));
  }
  return B200REG_OK;
}

int Relocalizer::score_nodes(int h, long long count, const int* kij, int* scores, std::string& why, cudaStream_t s) {
  if (!built_ || m_ < 0 || h < 0 || h >= grid.levels || count < 0 || (count && (!kij || !scores))) {
    why = "relocalize_score_nodes: no search since the pyramid was built, a level outside it or a NULL array";
    return B200REG_ERR_ARG;
  }
  for (long long q = 0; q < count; q++)
    if (kij[3 * q] < 0 || kij[3 * q] >= yaw_) {
      why = "relocalize_score_nodes: a heading outside the last search's";
      return B200REG_ERR_ARG;
    }
  if (count == 0) return B200REG_OK;
  if (m_ == 0 || grid.W == 0) {
    std::memset(scores, 0, (size_t)count * sizeof(int));
    return B200REG_OK;
  }
  RlDev d;
  d.pyr = pyr_.ptr;
  for (int l = 0; l < RL_MAX_LEVELS; l++) d.off[l] = l <= grid.levels ? level_off_[(size_t)std::min(l, grid.levels)] : 0;
  d.g = grid;
  d.offs = offs_.ptr;
  d.m = m_;
  front_[0].ensure((size_t)count);
  node_scores_[0].ensure((size_t)count);
  static_assert(sizeof(RlNode) == 3 * sizeof(int), "RlNode is three ints");
  B200_CUDA(cudaMemcpyAsync(front_[0].ptr, kij, (size_t)count * sizeof(RlNode), cudaMemcpyHostToDevice, s));
  rl_nodes_kernel<false><<<(unsigned)((count + RL_NODES_PER_BLOCK - 1) / RL_NODES_PER_BLOCK), RL_THREADS, 0, s>>>(
      d, h, RL_MODE_SCORES, front_[0].ptr, (unsigned long long)count, 0, nullptr, node_scores_[0].ptr, nullptr, nullptr, 0, nullptr, nullptr,
      nullptr);
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(scores, node_scores_[0].ptr, (size_t)count * sizeof(int), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  launches += 1;
  return B200REG_OK;
}

}  // namespace b200
