// The elevation / traversability map of the scan-matcher session (b200sm_build_elevation_map): the K18 kernels of
// elevation.cu. The arithmetic is csrc/elevation_map.hpp's; the extent is measured by occupancy's K14a (og_bounds_launch)
// over the same OgEntry table. These are the launches, enqueued on the caller's stream.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "elevation_map.hpp"
#include "occupancy.cuh"

namespace b200 {

// counters[] slots; POINTS and SKIPPED are K14a's RAYS and SKIPPED
enum : int {
  EL_CTR_POINTS = OG_CTR_RAYS,
  EL_CTR_SKIPPED = OG_CTR_SKIPPED,
  EL_CTR_OVERHANG = 2,
  EL_CTR_OBSERVED,
  EL_CTR_LETHAL,
  EL_CTR_TRAVERSABLE,
  EL_CTR_UNKNOWN,
  EL_CTR_TRIPPED,
  EL_CTR_COUNT
};
constexpr int EL_TILE_X = 32, EL_TILE_Y = 8;

// K18a: n[cell] += 1 and lo[cell] = min(lo[cell], Z) for every non-skipped point of the entries (n zero and lo EL_LO_EMPTY
// beforehand). The grid is W cells wide from cell (gx0, gy0); a cell outside it (never: the grid is K14a's extent) raises
// counters[TRIPPED] instead.
void el_lowest_launch(const OgEntry* table, int n_entries, unsigned tiles, const ElConst& c, int gx0, int gy0, unsigned W, unsigned H,
                      uint32_t* n, long long* lo, unsigned long long* counters, cudaStream_t stream);
// K18b: top[cell] = max Z over the points with Z <= lo[cell] + C (top EL_TOP_EMPTY beforehand), counters[OVERHANG] += the
// others; zrange[0] = min Z, zrange[1] = max Z over every non-skipped point (EL_LO_EMPTY / EL_TOP_EMPTY beforehand).
void el_top_launch(const OgEntry* table, int n_entries, unsigned tiles, const ElConst& c, int gx0, int gy0, unsigned W, unsigned H,
                   const long long* lo, long long* top, unsigned long long* counters, long long* zrange, cudaStream_t stream);
// K18c: the window of every cell: step, tan_slope, roughness, value, the row-flipped image byte (c.og's thresholds), and
// counters[OBSERVED / LETHAL / TRAVERSABLE / UNKNOWN].
void el_window_launch(const ElConst& c, unsigned W, unsigned H, const uint32_t* n, const long long* top,
                      float* step, float* tan_slope, float* roughness, signed char* value, unsigned char* image,
                      unsigned long long* counters, cudaStream_t stream);

}  // namespace b200
