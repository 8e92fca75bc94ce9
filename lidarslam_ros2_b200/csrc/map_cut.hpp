// The cut a localising session takes out of its prior map (b200sm_localize_cloud, include/b200reg.h): the rows within a
// horizontal radius of the pose, in map order. This header holds what both passes of the device compaction
// (scanmatcher.cu: cut_count_kernel, cut_write_kernel) and a serial host run of the same two passes
// (tests/hostmath/map_cut_host.cpp) share: the predicate, the layout of a tile and the rank of a kept row. Free of CUDA
// types so that g++ compiles it; on the host it must be compiled without floating-point contraction.
#pragma once
#include <cstddef>

#ifdef __CUDACC__
#define B200_CUT_HD __host__ __device__
#else
#define B200_CUT_HD
#endif

namespace b200 {

// One CTA serves one tile of CUT_TILE consecutive rows: warp w owns rows [w * CUT_WARP_ROWS, (w + 1) * CUT_WARP_ROWS) of
// the tile and reads them in CUT_ROUNDS rounds of 32 consecutive rows, lane l taking row 32 * round + l of the warp's
// share. Map order within the tile is therefore (warp, round, lane) in lexicographic order.
constexpr int CUT_THREADS = 256, CUT_WARPS = CUT_THREADS / 32, CUT_ROUNDS = 8;
constexpr int CUT_WARP_ROWS = 32 * CUT_ROUNDS, CUT_TILE = CUT_WARPS * CUT_WARP_ROWS;
// Kept counts and tile offsets are 32-bit: the largest prior map a session accepts. Its ceil(n / CUT_TILE) tiles
// (at most 2^21) fit one grid dimension, and every row index is formed in size_t.
constexpr size_t CUT_MAX_POINTS = 0xffffffffull;

inline size_t cut_tiles(size_t n) { return (n + CUT_TILE - 1) / CUT_TILE; }

B200_CUT_HD inline size_t cut_row(size_t tile, int warp, int round, int lane) {
  return tile * (size_t)CUT_TILE + (size_t)(warp * CUT_WARP_ROWS + round * 32 + lane);
}

// keep = dx * dx + dy * dy <= r2 with dx = (double)x - cx, dy = (double)y - cy: five IEEE double operations, none fused,
// so that a numpy float64 replay decides every row the same way. NaN fails the comparison; z is not looked at.
B200_CUT_HD inline bool cut_keep(float x, float y, double cx, double cy, double r2) {
#ifdef __CUDA_ARCH__
  const double dx = __dsub_rn((double)x, cx), dy = __dsub_rn((double)y, cy);
  return __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)) <= r2;
#else
  const double dx = (double)x - cx, dy = (double)y - cy;
  const double xx = dx * dx, yy = dy * dy;
  return xx + yy <= r2;
#endif
}

// kept rows of a 32-row round before lane `lane`, from the round's keep mask (bit l = lane l keeps its row)
B200_CUT_HD inline unsigned cut_rank_in_round(unsigned mask, int lane) {
  const unsigned below = mask & ((1u << lane) - 1u);
#ifdef __CUDA_ARCH__
  return (unsigned)__popc(below);
#else
  return (unsigned)__builtin_popcount(below);
#endif
}

}  // namespace b200
