// The occupancy grid of the scan-matcher session (b200sm_build_occupancy_grid): the K14 kernels of occupancy.cu. The
// arithmetic is csrc/occupancy_grid.hpp's; these are the launches, enqueued on the caller's stream.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "occupancy_grid.hpp"

namespace b200 {

// One submap of a launch: its cloud and float pose, its origin in fixed point, the first tile of the launch that serves it
// and (K14b / K14c) its window of the grid and its two bitmaps in the batch's scratch: the hit bitmap at word `words_at`,
// the free bitmap right after it, each `rows` rows of `stride` words (bit x of a row is cell x0 + x).
struct OgEntry {
  const float4* cloud;
  unsigned n, first_tile;
  float T[12];
  long long xo, yo, zo;
  int x0, y0;
  unsigned width, height;      // window, cells
  unsigned stride, rows;       // words per bitmap row, rows
  unsigned long long words_at;  // first scratch word of this submap's hit bitmap
  unsigned long long fold_first;  // first hit-bitmap word of this submap among the batch's (K14c's thread index)
};
constexpr int OG_THREADS = 256, OG_PER_THREAD = 4, OG_TILE = OG_THREADS * OG_PER_THREAD;

// counters[] slots
enum : int { OG_CTR_RAYS = 0, OG_CTR_SKIPPED, OG_CTR_OCCUPIED, OG_CTR_FREE, OG_CTR_UNKNOWN, OG_CTR_TRIPPED, OG_CTR_COUNT };

// K14a: bounds[4 k .. 4 k + 3] (min x, min y, max x, max y cell) of entry k widened by every ray's endpoint cell (the host
// initialises them with the origin's cell); counters[RAYS / SKIPPED] += the launch's rays and skipped points.
void og_bounds_launch(const OgEntry* table, int n_entries, unsigned tiles, const OgConst& c, int* bounds,
                      unsigned long long* counters, cudaStream_t stream);
// K14b: every ray of the entries marks its submap's hit and free bitmaps in `scratch` (zero beforehand). A cell outside a
// window (never, by the header's bounds) is not marked; counters[TRIPPED] is raised instead.
void og_walk_launch(const OgEntry* table, int n_entries, unsigned tiles, const OgConst& c, uint32_t* scratch,
                    unsigned long long* counters, cudaStream_t stream);
// K14c: hits[cell] += hit, frees[cell] += free && !hit for every window cell of the entries (fold_words words in all).
void og_fold_launch(const OgEntry* table, int n_entries, unsigned long long fold_words, const uint32_t* scratch, int gx0, int gy0,
                    unsigned width, uint32_t* hits, uint32_t* frees, cudaStream_t stream);
// K14d: values[cell] and the row-flipped image, and counters[OCCUPIED / FREE / UNKNOWN].
void og_classify_launch(const uint32_t* hits, const uint32_t* frees, unsigned width, unsigned height, int occ_value, int free_value,
                        signed char* values, unsigned char* image, unsigned long long* counters, cudaStream_t stream);

}  // namespace b200
