// TEST INFRASTRUCTURE: the two passes of the prior-map cut (csrc/map_cut.hpp: predicate, tile layout, rank of a kept row)
// run serially on the host with the index arithmetic the kernels use, so that tests/test_localize_host.py can compare the
// result with map[mask] bit for bit and AddressSanitizer sees every load and store. The output buffer has exactly `total`
// rows. Build with -ffp-contract=off (the predicate) and, for the sanitised run, -fsanitize=address,undefined.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../lidarslam_ros2_b200/csrc/map_cut.hpp"

using namespace b200;

namespace {

struct Row {
  float x, y, z, w;
};

// the 32-lane ballot of one round of one warp
unsigned round_mask(const Row* map, size_t n, size_t tile, int warp, int round, double cx, double cy, double r2) {
  unsigned mask = 0;
  for (int lane = 0; lane < 32; lane++) {
    const size_t i = cut_row(tile, warp, round, lane);
    if (i < n && cut_keep(map[i].x, map[i].y, cx, cy, r2)) mask |= 1u << lane;
  }
  return mask;
}

}  // namespace

extern "C" {

int mc_tile() { return CUT_TILE; }

// predicate alone: keep[i] for n (x, y) pairs
void mc_keep(size_t n, const float* xy, double cx, double cy, double r, unsigned char* keep) {
  const double r2 = r * r;
  for (size_t i = 0; i < n; i++) keep[i] = cut_keep(xy[2 * i], xy[2 * i + 1], cx, cy, r2) ? 1 : 0;
}

// Both passes. Returns the kept count; *out_rows is a malloc'd buffer of exactly that many rows (NULL when 0) which the
// caller releases with mc_free. *tripped counts stores the write pass refused because dst >= total.
size_t mc_cut(const float* map_xyzi, size_t n, double cx, double cy, double r, float** out_rows, int* tripped) {
  const Row* map = reinterpret_cast<const Row*>(map_xyzi);
  const double r2 = r * r;
  *out_rows = nullptr;
  *tripped = 0;
  const size_t tiles = cut_tiles(n);
  if (tiles == 0) return 0;
  // pass 1: kept rows per tile
  std::vector<unsigned> counts(tiles + 1, 0u);
  for (size_t t = 0; t < tiles; t++) {
    unsigned c = 0;
    for (int w = 0; w < CUT_WARPS; w++)
      for (int k = 0; k < CUT_ROUNDS; k++) c += (unsigned)__builtin_popcount(round_mask(map, n, t, w, k, cx, cy, r2));
    counts[t] = c;
  }
  // exclusive scan in place, total behind the last tile
  unsigned run = 0;
  for (size_t t = 0; t < tiles; t++) {
    const unsigned c = counts[t];
    counts[t] = run;
    run += c;
  }
  counts[tiles] = run;
  const size_t total = counts[tiles];
  if (total == 0) return 0;
  Row* out = static_cast<Row*>(std::malloc(total * sizeof(Row)));
  // pass 2: destination = tile offset + kept rows of the earlier warps + of this warp's earlier rounds + rank in the round
  for (size_t t = 0; t < tiles; t++) {
    unsigned warp_count[CUT_WARPS];
    unsigned masks[CUT_WARPS][CUT_ROUNDS];
    for (int w = 0; w < CUT_WARPS; w++) {
      warp_count[w] = 0;
      for (int k = 0; k < CUT_ROUNDS; k++) {
        masks[w][k] = round_mask(map, n, t, w, k, cx, cy, r2);
        warp_count[w] += (unsigned)__builtin_popcount(masks[w][k]);
      }
    }
    unsigned warp_off = 0;
    for (int w = 0; w < CUT_WARPS; w++) {
      unsigned base = counts[t] + warp_off;
      for (int k = 0; k < CUT_ROUNDS; k++) {
        for (int lane = 0; lane < 32; lane++) {
          if (!((masks[w][k] >> lane) & 1u)) continue;
          const size_t dst = (size_t)base + cut_rank_in_round(masks[w][k], lane);
          if (dst < total) out[dst] = map[cut_row(t, w, k, lane)];
          else *tripped += 1;
        }
        base += (unsigned)__builtin_popcount(masks[w][k]);
      }
      warp_off += warp_count[w];
    }
  }
  *out_rows = reinterpret_cast<float*>(out);
  return total;
}

void mc_free(float* rows) { std::free(rows); }

}

#ifdef MAP_CUT_MAIN
// The sanitised run: an executable (a sanitised shared object cannot be loaded into an unsanitised Python) that runs both
// passes over the edge sizes and keep patterns and compares with a plain serial filter. Exit code 0 when all agree.
#include <cmath>
#include <cstdio>
#include <limits>

int main() {
  const double cx = 3.0, cy = -2.0, r = 5.0;
  const size_t T = CUT_TILE;
  const size_t sizes[] = {0, 1, 31, 32, 33, T - 1, T, T + 1, 3 * T + 17};
  int failures = 0;
  for (size_t n : sizes)
    for (int pattern = 0; pattern < 5; pattern++) {  // all, none, every other, only the last, mixed with NaN / inf rows
      std::vector<float> map(4 * n);
      uint64_t state = 0x9E3779B97F4A7C15ull * (n + 1) + (uint64_t)pattern;
      for (size_t i = 0; i < n; i++) {
        state = state * 6364136223846793005ull + 1442695040888963407ull;
        const double a = (double)(state >> 40) * (6.283185307179586 / 16777216.0);
        bool in = pattern == 0 || (pattern == 2 && i % 2 == 0) || (pattern == 3 && i == n - 1) || (pattern == 4 && ((state >> 13) & 1));
        const double rad = in ? 4.5 : 9.0;
        map[4 * i + 0] = (float)(cx + rad * std::cos(a));
        map[4 * i + 1] = (float)(cy + rad * std::sin(a));
        map[4 * i + 2] = 100.0f * (float)(i % 7);
        map[4 * i + 3] = (float)i;
        if (pattern == 4 && i % 11 == 3) map[4 * i + (i % 2)] = std::numeric_limits<float>::quiet_NaN();
        if (pattern == 4 && i % 13 == 5) map[4 * i + (i % 2)] = std::numeric_limits<float>::infinity();
      }
      std::vector<float> want;
      for (size_t i = 0; i < n; i++)
        if (cut_keep(map[4 * i], map[4 * i + 1], cx, cy, r * r)) want.insert(want.end(), map.begin() + 4 * i, map.begin() + 4 * i + 4);
      float* got = nullptr;
      int tripped = 0;
      const size_t total = mc_cut(map.data(), n, cx, cy, r, &got, &tripped);
      const bool ok = tripped == 0 && total * 4 == want.size() && (total == 0 || std::memcmp(got, want.data(), want.size() * sizeof(float)) == 0);
      if (!ok) {
        std::printf("MISMATCH n=%zu pattern=%d total=%zu want=%zu tripped=%d\n", n, pattern, total, want.size() / 4, tripped);
        failures++;
      }
      mc_free(got);
    }
  std::printf("map_cut_host: %d failures\n", failures);
  return failures ? 1 : 0;
}
#endif
