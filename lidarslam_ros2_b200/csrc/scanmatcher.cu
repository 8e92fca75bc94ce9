// Device-resident map maintenance and per-frame scan preparation for the scan-matcher frontend (SURVEY.md §8f rows 1, 3):
// the callers either side of the registration hot path, built so that a frame costs ONE host-to-device copy.
//
// Replaces, in the reference's frontend node (scanmatcher/src/scanmatcher_component.cpp):
//   cloud_callback tf2::doTransform into robot_frame_id_   :188-199   -> the upload's unpack pass (b200sm_set_sensor_transform)
//   cloud_callback range filter                      :211-219   -> range_filter_kernel
//   receiveCloud: use_odom initial guess             :333-348   -> b200sm_receive_cloud (b200sm_odom_next_scan)
//   receiveCloud: VoxelGrid(vg_size_for_input) + setInputSource          :323-328   -> b200sm_set_scan
//   initializeMap                                    :257-297   -> b200sm_update_map (first call)
//   updateMap: VoxelGrid(vg_size_for_map), transformPointCloud(Matrix4f), concatenation of the last
//              num_targeted_cloud-1 submaps through transformPointCloud(Affine3d::matrix())      :438-463   -> b200sm_update_map
//   receiveCloud: setInputTarget(targeted) (GICP: VoxelGrid(vg_size_for_input) first)             :300-322   -> b200sm_update_map
//   receiveCloud / publishMapAndPose pose bookkeeping                     :330-353, 391-434     -> b200sm_receive_cloud
//   publishMap: transformPointCloud(Matrix4f) of every submap + concatenation                :529-552   -> b200sm_assemble_map
// and in the backend node (graph_based_slam/src/graph_based_slam_component.cpp):
//   doPoseAdjustment: g2o pose graph + LM (host, pose_graph.hpp)                            :262-319   -> b200sm_pose_adjust
//   doPoseAdjustment: modified_map / modified_map_array                                     :321-368   -> b200sm_assemble_map
//   doPoseAdjustment: savePCDFileASCII("map.pcd", modified_map)                             :369       -> b200sm_save_map_pcd_ascii
// The 2D occupancy grid of the map for a navigation stack (b200sm_build_occupancy_grid, csrc/occupancy_grid.hpp) has no
// counterpart in the reference: nav2's map_server pair is written next to map.pcd. Nor has the elevation /
// traversability map for non-flat ground (b200sm_build_elevation_map, csrc/elevation_map.hpp), saved as a second such pair.
// Removing what moved while the map was recorded (b200sm_build_static_map, csrc/static_map.hpp) has no counterpart in the
// reference either: the static map is saved as PCD in place of map.pcd. Nor has the map's consistency
// (b200sm_build_map_consistency, csrc/map_consistency.hpp), a ground-truth-free measure of how crisp the map is.
// Localising in a saved map has no counterpart in the reference: b200sm_set_prior_map* keep the map on the device and
// b200sm_localize_cloud registers each frame against a stable cut of it around the pose (csrc/map_cut.hpp).
// The submaps (sensor-frame, voxel-filtered) and the targeted cloud never leave the GPU; read-back entry points exist for
// the parity tests and for the node's publishers.
#include <cerrno>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include <sys/stat.h>

#include "../../include/b200reg.h"
#include "consistency.cuh"
#include "deskew.hpp"
#include "elevation.cuh"
#include "engine.hpp"
#include "global_grid.hpp"
#include "map_changes.cuh"
#include "mesh.cuh"
#include "map_cut.hpp"
#include "occupancy.cuh"
#include "octomap.cuh"
#include "place_recognition.cuh"
#include "pose_graph.hpp"
#include "relocalize.cuh"
#include "scan_context.hpp"
#include "sensor_frame.hpp"
#include "session_io.hpp"
#include "session_merge.hpp"
#include "static_map.cuh"

namespace b200 {
namespace {

// r = sqrt(pow(x, 2.0) + pow(y, 2.0)) in double; keep scan_min_range < r < scan_max_range (:213-216). The order of the
// kept points is not preserved (warp-aggregated atomic append): every consumer is a VoxelGrid, which is order-independent.
__global__ void range_filter_kernel(const float4* __restrict__ in, size_t n, double rmin, double rmax, float4* __restrict__ out,
                                    unsigned* __restrict__ count) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  bool keep = false;
  float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i < n) {
    p = in[i];
    const double r = sqrt((double)p.x * (double)p.x + (double)p.y * (double)p.y);
    keep = (rmin < r) && (r < rmax);
  }
  const unsigned mask = __ballot_sync(0xffffffffu, keep);
  if (mask == 0) return;
  const int lane = threadIdx.x & 31;
  unsigned base = 0;
  if (lane == __ffs(mask) - 1) base = atomicAdd(count, (unsigned)__popc(mask));
  base = __shfl_sync(0xffffffffu, base, __ffs(mask) - 1);
  if (keep) out[base + __popc(mask & ((1u << lane) - 1u))] = p;
}

// The cut of the prior map, pass 1: counts[tile] = rows of the tile that cut_keep keeps. A tile's eight 32-row rounds per
// warp are all loaded before the first ballot.
__device__ __forceinline__ void cut_round_masks(const float4* __restrict__ map, size_t n, size_t tile, int warp, int lane, double cx,
                                                double cy, double r2, float4 (&p)[CUT_ROUNDS], unsigned (&mask)[CUT_ROUNDS]) {
#pragma unroll
  for (int k = 0; k < CUT_ROUNDS; k++) {
    const size_t i = cut_row(tile, warp, k, lane);
    p[k] = i < n ? map[i] : make_float4(0.f, 0.f, 0.f, 0.f);
  }
#pragma unroll
  for (int k = 0; k < CUT_ROUNDS; k++) {
    const size_t i = cut_row(tile, warp, k, lane);
    mask[k] = __ballot_sync(0xffffffffu, i < n && cut_keep(p[k].x, p[k].y, cx, cy, r2));
  }
}

__global__ void __launch_bounds__(CUT_THREADS) cut_count_kernel(const float4* __restrict__ map, size_t n, double cx, double cy, double r2,
                                                                unsigned* __restrict__ counts) {
  __shared__ unsigned warp_count[CUT_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4 p[CUT_ROUNDS];
  unsigned mask[CUT_ROUNDS];
  cut_round_masks(map, n, blockIdx.x, warp, lane, cx, cy, r2, p, mask);
  unsigned c = 0;
#pragma unroll
  for (int k = 0; k < CUT_ROUNDS; k++) c += (unsigned)__popc(mask[k]);
  if (lane == 0) warp_count[warp] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned t = 0;
#pragma unroll
    for (int w = 0; w < CUT_WARPS; w++) t += warp_count[w];
    counts[blockIdx.x] = t;
  }
}

// Pass 2: the same predicate on the same (never modified) map; a kept row goes to tile offset + kept rows of the earlier
// warps of the tile + of the warp's earlier rounds + its rank in the round, i.e. map order. `out` has exactly `total`
// rows, the count the host read back after pass 1: a destination outside it is not stored, *tripped is raised instead.
__global__ void __launch_bounds__(CUT_THREADS) cut_write_kernel(const float4* __restrict__ map, size_t n, double cx, double cy, double r2,
                                                                const unsigned* __restrict__ tile_offsets, unsigned total,
                                                                float4* __restrict__ out, unsigned* __restrict__ tripped) {
  __shared__ unsigned warp_count[CUT_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4 p[CUT_ROUNDS];
  unsigned mask[CUT_ROUNDS];
  cut_round_masks(map, n, blockIdx.x, warp, lane, cx, cy, r2, p, mask);
  unsigned c = 0;
#pragma unroll
  for (int k = 0; k < CUT_ROUNDS; k++) c += (unsigned)__popc(mask[k]);
  if (lane == 0) warp_count[warp] = c;
  __syncthreads();
  unsigned base = tile_offsets[blockIdx.x];
  for (int w = 0; w < warp; w++) base += warp_count[w];
#pragma unroll
  for (int k = 0; k < CUT_ROUNDS; k++) {
    if ((mask[k] >> lane) & 1u) {
      const unsigned dst = base + cut_rank_in_round(mask[k], lane);
      if (dst < total) out[dst] = p[k];
      else atomicOr(tripped, 1u);
    }
    base += (unsigned)__popc(mask[k]);
  }
}

struct Mat34d {
  double m[12];
};

// pcl::transformPointCloud(in, out, Eigen::Matrix4d) — the generic Transformer<double>: every coordinate is
// static_cast<float>(m0 x + m1 y + m2 z + m3) evaluated left to right in double (:459-462, submap_affine.matrix()).
__global__ void transform_f64_kernel(const float4* __restrict__ in, size_t n, Mat34d T, float4* __restrict__ out) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = in[i];
  const double x = p.x, y = p.y, z = p.z;
  float4 q;
  q.x = (float)__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T.m[0], x), __dmul_rn(T.m[1], y)), __dmul_rn(T.m[2], z)), T.m[3]);
  q.y = (float)__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T.m[4], x), __dmul_rn(T.m[5], y)), __dmul_rn(T.m[6], z)), T.m[7]);
  q.z = (float)__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(T.m[8], x), __dmul_rn(T.m[9], y)), __dmul_rn(T.m[10], z)), T.m[11]);
  q.w = p.w;
  out[i] = q;
}

// Submap clouds live in a chunked device arena: one cudaMalloc per ~64 MB instead of one per map update (cudaMalloc costs
// tens to hundreds of microseconds and occasionally milliseconds — it would dominate a 0.5 ms frame).
struct SubmapArena {
  static constexpr size_t CHUNK_POINTS = (size_t)4 << 20;
  std::vector<std::unique_ptr<DeviceBuffer<float4>>> chunks;
  size_t used = 0, cap = 0;
  float4* alloc(size_t n) {
    if (chunks.empty() || used + n > cap) {
      chunks.emplace_back(new DeviceBuffer<float4>());
      cap = std::max(CHUNK_POINTS, n);
      chunks.back()->ensure(cap);
      cap = chunks.back()->cap;
      used = 0;
    }
    float4* p = chunks.back()->ptr + used;
    used += (n + 15) & ~(size_t)15;  // keep 256-byte alignment
    return p;
  }
};

struct Submap {
  float4* cloud = nullptr;     // VoxelGrid(vg_size_for_map) of the scan, sensor frame (arena memory)
  size_t n = 0;
  double pose[16];             // row-major 4x4: Translation * Quaternion of the pose the scan was taken at
  double distance = 0;
};

// A submap of n rows in `arena` with its row-major pose and travelled distance. The rows are copied device to device from
// `rows` on `stream`; with rows == nullptr the caller fills them.
std::unique_ptr<Submap> new_submap(SubmapArena& arena, const float4* rows, size_t n, const double* pose_rowmajor16, double distance,
                                   cudaStream_t stream) {
  std::unique_ptr<Submap> sub(new Submap());
  sub->cloud = arena.alloc(std::max<size_t>(n, 1));
  sub->n = n;
  if (rows && n) B200_CUDA(cudaMemcpyAsync(sub->cloud, rows, n * sizeof(float4), cudaMemcpyDeviceToDevice, stream));
  std::memcpy(sub->pose, pose_rowmajor16, sizeof(sub->pose));
  sub->distance = distance;
  return sub;
}

// Map assembly (publishMap sm.cpp:529-552, modified_map gbs.cpp:321-368): one table entry per submap, uploaded per call.
struct AssembleEntry {
  const float4* cloud;
  unsigned long long out_offset;  // first output point of this submap
  unsigned n, first_tile;         // points; first tile (block) of this submap in the launch
  Mat34f T;                       // pose cast to float, 3x4 row-major
};
constexpr int ASSEMBLE_THREADS = 256, ASSEMBLE_PER_THREAD = 4, ASSEMBLE_TILE = ASSEMBLE_THREADS * ASSEMBLE_PER_THREAD;

// Every submap moved by its float pose, concatenated in submap order, in ONE launch: block b serves tile b of the map; its
// submap is the last entry with first_tile <= b (empty submaps own no tile). Each point is one float4 read and one float4
// write; the arithmetic is transform_point's, so a point is bitwise what transform_cloud_device gives for its submap and
// what pcl::transformPointCloud(Matrix4f) gives on the host. The intensity in .w is copied.
__global__ void __launch_bounds__(ASSEMBLE_THREADS) assemble_map_kernel(const AssembleEntry* __restrict__ table, int n_sub,
                                                                        float4* __restrict__ out) {
  const unsigned tile = blockIdx.x;
  const AssembleEntry& e = table[entry_of(table, n_sub, tile, &AssembleEntry::first_tile)];
  float T[12];
#pragma unroll
  for (int k = 0; k < 12; k++) T[k] = e.T.m[k];
  const unsigned n = e.n;
  const unsigned base = (tile - e.first_tile) * (unsigned)ASSEMBLE_TILE + threadIdx.x;
  const float4* __restrict__ in = e.cloud;
  float4* __restrict__ dst = out + e.out_offset;
  float4 p[ASSEMBLE_PER_THREAD];
#pragma unroll
  for (int j = 0; j < ASSEMBLE_PER_THREAD; j++) {  // all loads in flight before the first store
    const unsigned i = base + j * ASSEMBLE_THREADS;
    if (i < n) p[j] = in[i];
  }
#pragma unroll
  for (int j = 0; j < ASSEMBLE_PER_THREAD; j++) {
    const unsigned i = base + j * ASSEMBLE_THREADS;
    if (i < n) {
      const float3 r = transform_point(T, p[j]);
      dst[i] = make_float4(r.x, r.y, r.z, p[j].w);
    }
  }
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200reg_adopt_source_device(b200reg_t h, const void* dev, size_t n);  // capi.cu (library-internal)
extern "C" float b200reg_last_score_ms(b200reg_t h);                                 // capi.cu (library-internal)

// The occupancy grid (b200sm_build_occupancy_grid): hits, frees, values and trinary image per cell. Its next build
// overwrites it in place.
struct OccupancyGrid {
  DeviceBuffer<uint32_t> hits, frees;
  DeviceBuffer<signed char> values;
  DeviceBuffer<unsigned char> image;
  bool built = false;
  OgParams params;
  unsigned width = 0, height = 0;
  double origin[2] = {0, 0};
};

// The static map (b200sm_build_static_map): the rank index over its box, hits, frees and flags per occupied voxel, and the
// static map with its per-submap offsets. Its next build overwrites it in place.
struct StaticMap {
  DeviceBuffer<RankWord> index;
  DeviceBuffer<uint32_t> hits, frees;
  DeviceBuffer<unsigned char> dynamic;
  DeviceBuffer<float4> points;
  bool built = false;
  SmBox box{};
  unsigned long long n_words = 0;
  b200sm_static_map_info info{};
  std::vector<size_t> offsets;  // n_submaps at the build + 1
};

// One elevation map (b200sm_build_elevation_map): its layers on the device, its parameters and its info.
struct ElevationMap {
  DeviceBuffer<uint32_t> n;
  DeviceBuffer<long long> lo, top;
  DeviceBuffer<float> step, tan_slope, roughness;
  DeviceBuffer<signed char> value;
  DeviceBuffer<unsigned char> image;
  ElParams params;
  b200sm_elevation_info info{};
};

// One map-consistency build (b200sm_build_map_consistency): the per-point layers, the cell structures K19c read, the
// per-submap rows, and what the PCD save needs to assemble the same map again.
struct MapConsistency {
  DeviceBuffer<unsigned> n;
  DeviceBuffer<double> h, plane;
  DeviceBuffer<RankWord> index;
  DeviceBuffer<unsigned> start, queries, chunks, qcursor, ocursor, sub_first;
  DeviceBuffer<int> ijk;
  DeviceBuffer<unsigned long long> rows;
  McConst c{};
  b200sm_map_consistency_info info{};
  std::vector<b200sm_submap_consistency> sub_rows;
  std::vector<double> poses;  // the build's poses, 16 column-major doubles per submap
};

// One map-change build (b200sm_build_map_changes): the rank index over its box, the per-epoch counts and labels per
// occupied voxel, the label per point, and the updated map with its per-submap offsets.
struct MapChanges {
  DeviceBuffer<RankWord> index;
  DeviceBuffer<uint32_t> hits[2], frees[2];
  DeviceBuffer<unsigned char> label, point_label;
  DeviceBuffer<float4> updated;
  SmBox box{};
  unsigned long long n_words = 0;
  b200sm_map_change_info info{};
  std::vector<size_t> offsets;  // n_submaps at the build + 1
};

// One mesh build (b200sm_build_mesh): the rank index over its band box, the band voxels (ijk, sum, weight in rank order),
// the vertices and the faces.
struct MeshBuild {
  DeviceBuffer<RankWord> index;
  DeviceBuffer<int> ijk;
  DeviceBuffer<unsigned long long> sum;
  DeviceBuffer<uint32_t> weight, faces;
  DeviceBuffer<float> xyz;
  b200sm_mesh_info info{};
};

// One OctoMap build (b200sm_build_octomap): the states of the box's voxels, the .bt file's data bytes (two per inner
// node) and its header.
struct OctoMapBuild {
  DeviceBuffer<unsigned char> states, data;
  std::string header;
  b200sm_octomap_info info{};
};

// The per-call workspace of the seven map builds and of the voxel-list read-backs, buffers named by role and shared by the
// builds that use one of the same type for the same role. Nothing in it outlives the call that filled it: no read-back
// reads what a build left here.
struct MapWorkspace {
  DeviceBuffer<OgEntry> og_table;  // the occupancy grid's and the elevation map's table
  DeviceBuffer<SmEntry> sm_table;  // the static map's, the map changes' and the mesh's
  DeviceBuffer<McEntry> mc_table;  // the map consistency's
  DeviceBuffer<int> bounds;        // the bounds pass's per-entry bounds
  DeviceBuffer<unsigned long long> counters;
  DeviceBuffer<uint32_t> bitmaps;  // a walk batch's hit and free bitmaps
  RankIndexScratch rank_scan;      // the rank pass's scan
  DeviceBuffer<unsigned> tiles;    // kept points per tile, scanned into tile offsets
  DeviceBuffer<unsigned> scan_tmp;  // counter_scan_async's tile sums
  DeviceBuffer<unsigned> map_first;  // map changes: each entry's first map index
  DeviceBuffer<long long> zrange;    // elevation map: the height extent
  DeviceBuffer<ushort4> cell_offs;   // map consistency: the points in cell order
  DeviceBuffer<unsigned> cell_idx;
  DeviceBuffer<unsigned char> active;  // mesh: ACTIVE flags, vertex ids, and vertex and face counts per tile
  DeviceBuffer<uint32_t> vertex_id;
  DeviceBuffer<unsigned> vertex_counts, face_counts;
  DeviceBuffer<RankWord> occ_index;  // octomap: the static map's front half on its own rank index, counts and flags,
  DeviceBuffer<uint32_t> occ_hits, occ_frees;  // so that the static map's result stays as it is
  DeviceBuffer<unsigned char> occ_dynamic;
  DeviceBuffer<uint32_t> freed;          // octomap: one bit per box voxel that a freed walk crosses
  DeviceBuffer<unsigned char> pyr_codes;  // octomap: the pyramid's codes and inner counts (then byte offsets) per cell
  DeviceBuffer<unsigned> pyr_counts;
  DeviceBuffer<int> ijk;  // get_map_voxels / get_change_voxels: the voxel list
};

struct b200sm_session {
  int device = 0;
  cudaStream_t stream = nullptr;
  std::string err;
  // parameters (scanmatcher_component.cpp:34-50 defaults)
  float vg_size_for_input = 0.2f, vg_size_for_map = 0.1f;
  int num_targeted_cloud = 10;
  int use_min_max_filter = 0;
  double scan_min_range = 0.1, scan_max_range = 100.0;
  double trans_for_mapupdate = 1.5;
  // state
  DeviceBuffer<float4> upload, scan;  // uploaded frame; after the optional range filter (`scan` aliases upload when off)
  const float4* d_scan = nullptr;
  size_t n_scan = 0;
  CloudUploader uploader;
  DeviceBuffer<unsigned> counter;
  VoxelGridFilter vg_input, vg_map, vg_target;
  Bounds scan_bounds{};            // min/max of d_scan when it is the uploaded cloud itself (no de-skew, no range filter)
  bool scan_bounds_valid = false;
  size_t n_filtered = 0;
  const float4* d_filtered = nullptr;  // VoxelGrid(vg_size_for_input) of the scan — the scan itself when the grid would overflow
  SubmapArena arena;
  std::vector<std::unique_ptr<Submap>> submaps;
  // first submap of every segment (one recording's contiguous run of submaps); b200sm_merge_session appends one per merge.
  // A session of more than one segment is a backend's map: the frontend's calls are refused on it.
  std::vector<int> seg_first{0};
  // b200sm_load_session: the session is a saved map (a backend's map: the frontend's calls are refused on it), and the graph
  // it was saved with (loop edges, num_adjacent_pose_cnstraints, the adjusted poses or none)
  bool loaded = false;
  std::vector<sio::LoopEdge> graph_loops;
  int graph_k = 0;
  std::vector<double> graph_poses;
  DeviceBuffer<float4> targeted;
  size_t n_targeted = 0;
  DeviceBuffer<float4> loop_src, loop_tgt;  // search_loop scratch
  DeviceBuffer<AssembleEntry> assemble_table;
  DeviceBuffer<float4> assembled;           // the last map b200sm_assemble_map / b200sm_save_map_pcd_ascii built
  PcdEncoder pcd;                           // its ASCII PCD text, chunk by chunk
  PinnedBuffer<char> pcd_staging[2];        // two chunks of text on the host: one being written while the next arrives
  int launches = 0;
  // frontend bookkeeping (ScanMatcherComponent members)
  bool initial_cloud_received = false;
  bool target_pending = false;  // is_map_updated_: a rebuilt targeted cloud waits to become the registration target
  double position[3] = {0, 0, 0}, quat[4] = {0, 0, 0, 1};  // corrent_pose_stamped_.pose (x y z, qx qy qz qw)
  double previous_position[3] = {0, 0, 0};
  double latest_distance = 0, trans = 0;
  // IMU de-skew (lidar_undistortion.hpp; use_imu, scanmatcher_component.cpp:205-209)
  ImuDeskew imu;
  bool deskew_armed = false;
  double deskew_scan_time = 0;
  // cloud_callback's tf2::doTransform into robot_frame_id_ (sm.cpp:188-199), applied by the unpack pass of every frame
  bool sensor_tf_set = false;
  Mat34f sensor_tf{};
  // use_odom (sm.cpp:333-348): the odometry armed for the next frame, and previous_odom_mat_ (row-major float)
  bool odom_armed = false;
  float odom_mat[16] = {};
  float previous_odom_mat[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  // localisation in a prior map (b200sm_set_prior_map*, b200sm_localize_cloud)
  PcdLoader pcd_loader;
  DeviceBuffer<float4> prior_map, prior_incoming;  // the map; a new one is loaded beside it and swapped in once complete
  size_t n_prior = 0;
  double crop_radius = 120.0, recrop_distance = 20.0;  // >= the default scan_max_range + recrop_distance
  DeviceBuffer<float4> cut;             // the current cut, map order; the engine holds its own copy of its target
  DeviceBuffer<unsigned> cut_counts, cut_scan_tmp;  // per-tile counts -> offsets, [tiles] total, [tiles + 1] tripwire flag
  size_t n_cut = 0, n_cut_target = 0;
  double cut_centre[2] = {0, 0}, dist_from_centre = 0;
  int n_cuts = 0;
  bool have_cut = false, cut_stale = true, cut_pending = false;
  // the grid of the last b200sm_localize_global: poses (16 floats each, column-major), scores, hits
  std::vector<float> global_poses;
  std::vector<double> global_scores;
  std::vector<long long> global_hits;
  // relocalisation (b200sm_relocalize): the pyramid of the prior map, the last search's offsets and frontier
  Relocalizer reloc;
  // place recognition (b200sm_search_loop_place): descriptors of submaps [0, sc_built) in slots of sc_keys (keys while being
  // built, then the descriptor's floats) and their column norms; room for sc_cap submaps
  ScParams sc;
  DeviceBuffer<double> sc_tables;  // ring bounds, then sector directions
  bool sc_tables_ready = false;
  DeviceBuffer<uint32_t> sc_keys;
  DeviceBuffer<double> sc_norms;
  size_t sc_built = 0, sc_cap = 0;
  DeviceBuffer<ScBuildEntry> sc_build_table;
  DeviceBuffer<int> sc_ids, sc_shift;
  DeviceBuffer<double> sc_dist;
  std::vector<double> place_distances;  // the last place search, per submap
  std::vector<int> place_shifts;
  // the last merge's K16 scores (b200sm_merge_session): n_query x n_cand, row-major, kept until the next merge; and the
  // per-row selection
  DeviceBuffer<double> merge_dist, merge_sel_d;
  DeviceBuffer<int> merge_shift, merge_sel_a, merge_sel_s;
  size_t merge_nq = 0, merge_nc = 0;
  // the map products built from the session's map. The occupancy grid and the static map are kept until their next build
  // overwrites them; the other five are built beside the last one, which stays until the new one succeeds.
  OccupancyGrid og;
  std::unique_ptr<ElevationMap> el;
  StaticMap sm;
  std::unique_ptr<MapChanges> ch;
  std::unique_ptr<MeshBuild> ms;
  std::unique_ptr<MapConsistency> mc;
  std::unique_ptr<OctoMapBuild> om;
  MapWorkspace work;
};

namespace {

template <typename F>
int sm_guarded(b200sm_t s, F&& f) {
  if (!s) return B200REG_ERR_ARG;
  try {
    cudaError_t e = cudaSetDevice(s->device);
    if (e != cudaSuccess) {
      s->err = std::string("cudaSetDevice: ") + cudaGetErrorString(e);
      return B200REG_ERR_CUDA;
    }
    return f();
  } catch (const CudaError& e) {
    s->err = e.what();
    cudaGetLastError();
    return B200REG_ERR_CUDA;
  } catch (const std::exception& e) {
    s->err = e.what();
    return B200REG_ERR_ARG;
  }
}

int sm_fail(b200sm_t s, int code, const char* msg) {
  s->err = msg;
  return code;
}

// A session of several segments or loaded from disk is a backend's map: the frontend's calls are refused on it. `what`
// prefixes the message.
int refuse_backend_map(b200sm_t s, const char* what) {
  if (s->seg_first.size() > 1)
    return sm_fail(s, B200REG_ERR_ARG, (std::string(what) + ": the session holds a merged map of several recordings").c_str());
  if (s->loaded) return sm_fail(s, B200REG_ERR_ARG, (std::string(what) + ": the session holds a map loaded by b200sm_load_session").c_str());
  return B200REG_OK;
}

// the caller's loop edges over submaps [0, n): ids in range, from != to, a finite relative pose. `what` prefixes the
// messages.
int check_loop_edges(b200sm_t s, const b200sm_loop_edge* loop_edges, int n_loop_edges, int n, const char* what) {
  for (int l = 0; l < n_loop_edges; l++) {
    const b200sm_loop_edge& e = loop_edges[l];
    if (e.from < 0 || e.from >= n || e.to < 0 || e.to >= n || e.from == e.to)
      return sm_fail(s, B200REG_ERR_ARG, (std::string(what) + ": loop edge with a submap id out of range or from == to").c_str());
    for (int k = 0; k < 16; k++)
      if (!std::isfinite(e.relative_pose[k])) return sm_fail(s, B200REG_ERR_ARG, (std::string(what) + ": non-finite relative_pose").c_str());
  }
  return B200REG_OK;
}

// the caller's loop edges appended to the pose graph's loop list: ids (from, to) and relative poses
void append_loop_edges(const b200sm_loop_edge* loop_edges, int n_loop_edges, std::vector<int>& ids, std::vector<pg::Iso>& rel) {
  for (int l = 0; l < n_loop_edges; l++) {
    ids.push_back(loop_edges[l].from);
    ids.push_back(loop_edges[l].to);
    rel.push_back(pg::iso_from_colmajor16(loop_edges[l].relative_pose));
  }
}

// a caller's poses (16 column-major per submap), when given, are finite
bool finite_poses(const double* poses_colmajor16, size_t n_sub) {
  if (poses_colmajor16)
    for (size_t k = 0; k < 16 * n_sub; k++)
      if (!std::isfinite(poses_colmajor16[k])) return false;
  return true;
}

void upload_frame(b200sm_t s, const float* points, size_t n, size_t stride, long intensity_off) {
  s->upload.ensure(n);
  // one H2D copy per frame; the unpack pass also moves the points into the robot frame when a sensor transform is set, and
  // measures the (moved) scan's min/max (both VoxelGrids of the frame are sized from it)
  s->uploader.upload_with_bounds(points, n, stride, intensity_off, 0.0f, s->upload.ptr, s->stream,
                                 s->sensor_tf_set ? &s->sensor_tf : nullptr);
  s->launches += 1;
  s->d_scan = s->upload.ptr;
  s->n_scan = n;
  s->scan_bounds_valid = false;
  bool deskewed = false;
  if (s->deskew_armed && n > 0) {  // cloud_callback: adjustDistortion before the range filter (sm.cpp:205-209)
    s->deskew_armed = false;
    deskewed = true;
    const char* b = reinterpret_cast<const char*>(points);
    const float* first = reinterpret_cast<const float*>(b);
    const float* last = reinterpret_cast<const float*>(b + (n - 1) * stride);
    float first_t[3], last_t[3];
    if (s->sensor_tf_set) {
      // the de-skew's start / end azimuths are those of the robot-frame points: the first and last records are moved on
      // the host with the kernel's un-fused float arithmetic (transform_point_f), bitwise what the unpack pass stores,
      // so neither a read-back nor a synchronisation is added before the de-skew
      transform_point_f(s->sensor_tf.m, first, first_t);
      transform_point_f(s->sensor_tf.m, last, last_t);
      first = first_t;
      last = last_t;
    }
    const int before = s->imu.launches;
    s->imu.adjust_distortion(s->upload.ptr, n, first, last, s->deskew_scan_time, s->stream);
    s->launches += s->imu.launches - before;
  }
  if (s->use_min_max_filter) {
    s->scan.ensure(n);
    s->counter.ensure(1);
    B200_CUDA(cudaMemsetAsync(s->counter.ptr, 0, sizeof(unsigned), s->stream));
    range_filter_kernel<<<(int)((n + 255) / 256), 256, 0, s->stream>>>(s->upload.ptr, n, s->scan_min_range, s->scan_max_range,
                                                                       s->scan.ptr, s->counter.ptr);
    B200_CUDA(cudaGetLastError());
    unsigned kept = 0;
    B200_CUDA(cudaMemcpyAsync(&kept, s->counter.ptr, sizeof(unsigned), cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    s->d_scan = s->scan.ptr;
    s->n_scan = kept;
    s->launches += 1;
  } else if (!deskewed) {  // the uploaded cloud IS the scan: its bounds are those measured during the upload
    B200_CUDA(cudaStreamSynchronize(s->stream));
    s->scan_bounds = s->uploader.finish_bounds();
    s->scan_bounds_valid = true;
  }
}

// VoxelGrid on the device; a grid overflow returns the input unchanged like PCL
const float4* filter_on_device(b200sm_t s, VoxelGridFilter& F, const float4* d_in, size_t n, float leaf, size_t* m,
                               const Bounds* known_bounds = nullptr) {
  const int before = F.launches;
  long long cnt = F.filter_device(d_in, n, leaf, s->stream, known_bounds);
  s->launches += F.launches - before;
  if (cnt < 0) {
    *m = n;
    return d_in;
  }
  *m = (size_t)cnt;
  return F.out.ptr;
}

int set_source_from_scan(b200sm_t s, b200reg_t reg) {
  size_t m = 0;
  const float4* f = filter_on_device(s, s->vg_input, s->d_scan, s->n_scan, s->vg_size_for_input, &m,
                                     s->scan_bounds_valid ? &s->scan_bounds : nullptr);
  s->n_filtered = m;
  s->d_filtered = f;
  if (m == 0) return sm_fail(s, B200REG_ERR_ARG, "scan is empty after filtering");
  // (the filter's read-back of the point count has synchronised this stream; the filtered scan lives in this session until
  // the next frame, so the engine reads it in place: no copy, no second synchronisation)
  const int rc = b200reg_adopt_source_device(reg, f, m);
  if (rc != B200REG_OK) s->err = std::string("setInputSource: ") + b200reg_last_error(reg);
  return rc;
}

// updateMap (:438-491) / initializeMap (:257-297) on the current scan; final_T row-major float, pose = position + quaternion
int update_map(b200sm_t s, const float* final_T, const double* position, const double* quat) {
  if (s->n_scan == 0) return sm_fail(s, B200REG_ERR_NO_SOURCE, "update_map: no scan");
  size_t m = 0;
  const float4* filtered = filter_on_device(s, s->vg_map, s->d_scan, s->n_scan, s->vg_size_for_map, &m,
                                            s->scan_bounds_valid ? &s->scan_bounds : nullptr);
  // targeted_cloud_ = T(filtered) + the last num_targeted_cloud-1 submaps, newest first, each through its pose (double)
  const int n_sub = (int)s->submaps.size();
  size_t total = m;
  for (int i = 0; i < s->num_targeted_cloud - 1; i++) {
    if (n_sub - 1 - i < 0) continue;
    total += s->submaps[n_sub - 1 - i]->n;
  }
  s->targeted.ensure(total);
  Mat34f Tf;
  for (int k = 0; k < 12; k++) Tf.m[k] = final_T[k];
  transform_cloud_device(filtered, m, s->targeted.ptr, Tf, s->stream);
  size_t off = m;
  for (int i = 0; i < s->num_targeted_cloud - 1; i++) {
    if (n_sub - 1 - i < 0) continue;
    const Submap& sub = *s->submaps[n_sub - 1 - i];
    Mat34d Td;
    for (int k = 0; k < 12; k++) Td.m[k] = sub.pose[k];
    if (sub.n) transform_f64_kernel<<<(int)((sub.n + 255) / 256), 256, 0, s->stream>>>(sub.cloud, sub.n, Td, s->targeted.ptr + off);
    off += sub.n;
    s->launches += 1;
  }
  B200_CUDA(cudaGetLastError());
  s->n_targeted = total;
  s->launches += 1;
  // the new submap keeps the FILTERED, untransformed cloud and the pose (:465-481)
  double pose[16];
  pose_to_matrix_d(position, quat, pose);
  s->submaps.push_back(new_submap(s->arena, filtered, m, pose, s->latest_distance, s->stream));
  s->target_pending = true;
  return B200REG_OK;
}

// setInputTarget(cloud) from a session buffer (GICP: VoxelGrid(vg_size_for_input) of it first, sm.cpp:311-317); *n_given =
// the points the engine received. The engine copies, so `cloud` may be rebuilt as soon as this returns.
int hand_over_target(b200sm_t s, b200reg_t reg, int is_gicp, const float4* cloud, size_t n, const char* empty_msg, size_t* n_given) {
  const float4* t = cloud;
  if (is_gicp) t = filter_on_device(s, s->vg_target, cloud, n, s->vg_size_for_input, &n);
  if (n == 0) return sm_fail(s, B200REG_ERR_NO_TARGET, empty_msg);
  B200_CUDA(cudaStreamSynchronize(s->stream));
  const int rc = b200reg_set_input_target_device(reg, t, n);
  if (rc != B200REG_OK) s->err = std::string("setInputTarget: ") + b200reg_last_error(reg);
  else if (n_given) *n_given = n;
  return rc;
}

// receiveCloud :300-322: the rebuilt targeted cloud becomes the registration target
int adopt_target(b200sm_t s, b200reg_t reg, int is_gicp) {
  if (!s->target_pending) return B200REG_OK;
  const int rc = hand_over_target(s, reg, is_gicp, s->targeted.ptr, s->n_targeted, "targeted cloud is empty", nullptr);
  if (rc == B200REG_OK) s->target_pending = false;
  return rc;
}

// sim_trans = getTransformation(corrent_pose_stamped_.pose): Affine3d matrix cast to float (:493-499), row- and column-major
void sim_trans(b200sm_t s, float* T_row, float* sim_col) {
  double M[16];
  pose_to_matrix_d(s->position, s->quat, M);
  for (int k = 0; k < 16; k++) T_row[k] = (float)M[k];
  row_to_col(M, sim_col);
}

// publishMapAndPose's pose (:391-398): position and quaternion of a column-major float final transformation
void adopt_pose(b200sm_t s, const float* final_col) {
  double R[9];
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) R[r * 3 + c] = (double)final_col[c * 4 + r];
    s->position[r] = (double)final_col[12 + r];
  }
  matrix_to_quat_d(R, s->quat);
}

// The part of a frame the mapping and the localising frontend share, once the engine has its target: VoxelGrid +
// setInputSource (:323-328), guess = current pose or the use_odom guess (:333-348), align (:350), the new pose (:391-398).
int register_frame(b200sm_t s, b200reg_t reg, bool use_odom, float* final_col) {
  int rc = set_source_from_scan(s, reg);
  if (rc != B200REG_OK) return rc;
  float sim_col[16], T_row[16];
  sim_trans(s, T_row, sim_col);
  if (use_odom) {  // sim_trans * previous_odom_mat_.inverse() * odom_mat, then previous_odom_mat_ = odom_mat
    odom_guess_f(T_row, s->previous_odom_mat, s->odom_mat);
    row_to_col(T_row, sim_col);
  }
  rc = b200reg_align(reg, sim_col, final_col);
  if (rc != B200REG_OK) {
    s->err = std::string("align: ") + b200reg_last_error(reg);
    return rc;
  }
  adopt_pose(s, final_col);
  return B200REG_OK;
}

void write_pose(b200sm_t s, double* pose7_out) {
  if (!pose7_out) return;
  for (int k = 0; k < 3; k++) pose7_out[k] = s->position[k];
  for (int k = 0; k < 4; k++) pose7_out[3 + k] = s->quat[k];
}

bool valid_frame_args(b200sm_t s, b200reg_t reg, const float* points, size_t n, size_t stride_bytes, long intensity_offset_bytes) {
  return s && reg && points && n != 0 && valid_record_layout(stride_bytes, intensity_offset_bytes);
}

int read_back(b200sm_t s, const float4* d, size_t n, float* out, size_t cap, size_t* n_out) {
  if (n_out) *n_out = n;
  const size_t k = std::min(n, cap);
  if (k && out) {
    B200_CUDA(cudaMemcpyAsync(out, d, k * sizeof(float4), cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
  }
  return B200REG_OK;
}

}  // namespace

extern "C" {

int b200sm_create(int device, b200sm_t* out) {
  if (!out) return B200REG_ERR_ARG;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count) {
    cudaGetLastError();
    return B200REG_ERR_CUDA;  // no CPU fallback
  }
  b200sm_session* s = new b200sm_session();
  s->device = device;
  if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking) != cudaSuccess) {
    cudaGetLastError();
    delete s;
    return B200REG_ERR_CUDA;
  }
  *out = s;
  return B200REG_OK;
}

void b200sm_destroy(b200sm_t s) {
  if (!s) return;
  cudaSetDevice(s->device);
  if (s->stream) {
    cudaStreamSynchronize(s->stream);
    cudaStreamDestroy(s->stream);
  }
  delete s;
}

const char* b200sm_last_error(b200sm_t s) { return s ? s->err.c_str() : "null session"; }

int b200sm_set_params(b200sm_t s, float vg_size_for_input, float vg_size_for_map, int num_targeted_cloud, double trans_for_mapupdate,
                      int use_min_max_filter, double scan_min_range, double scan_max_range) {
  if (!s || !(vg_size_for_input > 0) || !(vg_size_for_map > 0) || num_targeted_cloud < 1) return B200REG_ERR_ARG;
  s->vg_size_for_input = vg_size_for_input;
  s->vg_size_for_map = vg_size_for_map;
  s->num_targeted_cloud = num_targeted_cloud;
  s->trans_for_mapupdate = trans_for_mapupdate;
  s->use_min_max_filter = use_min_max_filter;
  s->scan_min_range = scan_min_range;
  s->scan_max_range = scan_max_range;
  return B200REG_OK;
}

int b200sm_set_initial_pose(b200sm_t s, const double* position3, const double* quat_xyzw) {
  if (!s || !position3 || !quat_xyzw) return B200REG_ERR_ARG;
  for (int k = 0; k < 3; k++) s->position[k] = s->previous_position[k] = position3[k];
  for (int k = 0; k < 4; k++) s->quat[k] = quat_xyzw[k];
  s->cut_stale = true;  // a localising session cuts its target around the new position at the next frame
  return B200REG_OK;
}

int b200sm_set_scan(b200sm_t s, b200reg_t reg, const float* points, size_t n, size_t stride_bytes, long intensity_offset_bytes,
                    size_t* n_filtered) {
  if (!valid_frame_args(s, reg, points, n, stride_bytes, intensity_offset_bytes)) return B200REG_ERR_ARG;
  if (const int rc = refuse_backend_map(s, "set_scan"); rc != B200REG_OK) return rc;
  return sm_guarded(s, [&]() {
    upload_frame(s, points, n, stride_bytes, intensity_offset_bytes);
    const int rc = set_source_from_scan(s, reg);
    if (n_filtered) *n_filtered = s->n_filtered;
    return rc;
  });
}

int b200sm_update_map(b200sm_t s, b200reg_t reg, const float* final_T_colmajor16, const double* position3, const double* quat_xyzw,
                      int adopt_now) {
  if (!s || !final_T_colmajor16 || !position3 || !quat_xyzw) return B200REG_ERR_ARG;
  if (const int rc = refuse_backend_map(s, "update_map"); rc != B200REG_OK) return rc;
  return sm_guarded(s, [&]() {
    float T[16];
    col_to_row(final_T_colmajor16, T);
    if (!s->submaps.empty()) {  // updateMap :471: latest_distance_ += trans_ (distance travelled since the last submap)
      const double dx = position3[0] - s->previous_position[0], dy = position3[1] - s->previous_position[1],
                   dz = position3[2] - s->previous_position[2];
      s->trans = std::sqrt(dx * dx + dy * dy + dz * dz);
      s->latest_distance += s->trans;
    }
    for (int k = 0; k < 3; k++) s->previous_position[k] = position3[k];
    int rc = update_map(s, T, position3, quat_xyzw);
    if (rc == B200REG_OK && adopt_now && reg) {
      int kind = B200REG_NDT;
      b200reg_get_kind(reg, &kind);
      rc = adopt_target(s, reg, kind == B200REG_GICP);
    }
    return rc;
  });
}

int b200sm_receive_cloud(b200sm_t s, b200reg_t reg, const float* points, size_t n, size_t stride_bytes, long intensity_offset_bytes,
                         double* pose7_out, float* final_T_colmajor16_out, int* map_updated) {
  if (!valid_frame_args(s, reg, points, n, stride_bytes, intensity_offset_bytes)) return B200REG_ERR_ARG;
  if (const int rc = refuse_backend_map(s, "receive_cloud"); rc != B200REG_OK) return rc;
  return sm_guarded(s, [&]() {
    if (map_updated) *map_updated = 0;
    const bool use_odom = s->odom_armed;  // armed for this frame only, like the de-skew
    s->odom_armed = false;
    int kind = B200REG_NDT;
    b200reg_get_kind(reg, &kind);
    upload_frame(s, points, n, stride_bytes, intensity_offset_bytes);
    int rc;
    if (!s->initial_cloud_received) {  // initializeMap (:257-297): the first scan, at the initial pose, is the map
      s->initial_cloud_received = true;
      float sim_col[16], T_row[16];
      sim_trans(s, T_row, sim_col);
      rc = update_map(s, T_row, s->position, s->quat);
      if (rc != B200REG_OK) return rc;
      rc = adopt_target(s, reg, /*is_gicp=*/0);  // initializeMap hands the transformed cloud over unfiltered
      if (rc != B200REG_OK) return rc;
    }
    rc = adopt_target(s, reg, kind == B200REG_GICP);  // :300-322
    if (rc != B200REG_OK) return rc;
    float final_col[16];
    rc = register_frame(s, reg, use_odom, final_col);  // :323-353, 391-398
    if (rc != B200REG_OK) return rc;
    // publishMapAndPose (:399-434)
    const double* pos = s->position;
    const double dx = pos[0] - s->previous_position[0], dy = pos[1] - s->previous_position[1], dz = pos[2] - s->previous_position[2];
    s->trans = std::sqrt(dx * dx + dy * dy + dz * dz);
    if (s->trans >= s->trans_for_mapupdate) {
      for (int k = 0; k < 3; k++) s->previous_position[k] = pos[k];
      s->latest_distance += s->trans;  // updateMap :471
      float F_row[16];
      col_to_row(final_col, F_row);
      rc = update_map(s, F_row, s->position, s->quat);
      if (rc != B200REG_OK) return rc;
      if (map_updated) *map_updated = 1;
    }
    write_pose(s, pose7_out);
    if (final_T_colmajor16_out) std::memcpy(final_T_colmajor16_out, final_col, sizeof(final_col));
    return (int)B200REG_OK;
  });
}

int b200sm_num_submaps(b200sm_t s, size_t* out) {
  if (!s || !out) return B200REG_ERR_ARG;
  *out = s->submaps.size();
  return B200REG_OK;
}

int b200sm_get_targeted(b200sm_t s, float* out_xyzi, size_t capacity, size_t* n) {
  if (!s) return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() { return read_back(s, s->targeted.ptr, s->n_targeted, out_xyzi, capacity, n); });
}

int b200sm_get_submap(b200sm_t s, size_t index, float* out_xyzi, size_t capacity, size_t* n, double* pose_colmajor16, double* distance) {
  if (!s || index >= s->submaps.size()) return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() {
    const Submap& sub = *s->submaps[index];
    if (pose_colmajor16) row_to_col(sub.pose, pose_colmajor16);
    if (distance) *distance = sub.distance;
    return read_back(s, sub.cloud, sub.n, out_xyzi, capacity, n);
  });
}

int b200sm_get_filtered_scan(b200sm_t s, float* out_xyzi, size_t capacity, size_t* n) {
  if (!s) return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() { return read_back(s, s->d_filtered, s->d_filtered ? s->n_filtered : 0, out_xyzi, capacity, n); });
}

// GraphBasedSlamComponent::searchLoop (graph_based_slam_component.cpp:144-258) over the session's own submaps — the map
// array the frontend publishes is the backend's input, here it never left the device.
}  // extern "C"

namespace {

Mat34f pose_f32(const Submap& sub) {  // affine.matrix().cast<float>()
  Mat34f T;
  for (int k = 0; k < 12; k++) T.m[k] = (float)sub.pose[k];
  return T;
}

struct LoopCandidate {
  int id;
  double dist;
};

// the gates of :187-204: travelled distance apart, position close — every submap that passes them, ascending id
std::vector<LoopCandidate> loop_candidates(b200sm_t s, double distance_loop_closure, double range_of_searching_loop_closure) {
  std::vector<LoopCandidate> out;
  const int n_sub = (int)s->submaps.size();
  if (n_sub == 0) return out;
  const Submap& latest = *s->submaps[n_sub - 1];
  for (int i = 0; i < n_sub; i++) {
    const Submap& sub = *s->submaps[i];
    const double dx = latest.pose[3] - sub.pose[3], dy = latest.pose[7] - sub.pose[7], dz = latest.pose[11] - sub.pose[11];
    const double dist = std::sqrt(dx * dx + dy * dy + dz * dz);
    if (latest.distance - sub.distance > distance_loop_closure && dist < range_of_searching_loop_closure) out.push_back({i, dist});
  }
  return out;
}

// source = a submap in its session's frame (:165-176; the searches take the latest one, a merge the other session's),
// handed to the registration object once per source
int loop_set_source(b200sm_t s, b200reg_t reg, const Submap& source) {
  s->loop_src.ensure(std::max<size_t>(source.n, 1));
  if (source.n == 0) return sm_fail(s, B200REG_ERR_NO_SOURCE, "search_loop: empty source");
  transform_cloud_device(source.cloud, source.n, s->loop_src.ptr, pose_f32(source), s->stream);
  s->launches += 1;
  B200_CUDA(cudaStreamSynchronize(s->stream));
  const int rc = b200reg_set_input_source_device(reg, s->loop_src.ptr, source.n);
  if (rc != B200REG_OK) s->err = std::string("search_loop: ") + b200reg_last_error(reg);
  return rc;
}

// one candidate: target = VoxelGrid(voxel_leaf_size) of the submaps id - search_submap_num .. id + search_submap_num
// (:206-225), align without guess (:229; the place search gives one), getFitnessScore (:230), loop edge when the score
// passes (:232-246).
// The reference does not test the upper index (undefined behaviour when the window runs past the newest submap);
// here indices outside [win_lo, win_hi) are skipped like the negative ones (the searches pass the whole session, a merge
// the candidate's segment). `source` is the submap loop_set_source handed over, the edge's `to` end. Nothing is uploaded:
// the submaps live in HBM.
int loop_evaluate(b200sm_t s, b200reg_t reg, const LoopCandidate& cand, const Submap& source, int win_lo, int win_hi,
                  float voxel_leaf_size, double threshold_loop_closure_score, int search_submap_num, b200sm_loop_result* out,
                  const float* guess = nullptr) {
  const int id_min = cand.id;
  out->is_candidate = 1;
  out->id_min = id_min;
  out->min_dist = cand.dist;
  size_t total = 0;
  for (int j = 0; j <= 2 * search_submap_num; j++) {
    const int idx = id_min + j - search_submap_num;
    if (idx < win_lo || idx >= win_hi) continue;
    total += s->submaps[idx]->n;
  }
  s->loop_tgt.ensure(std::max<size_t>(total, 1));
  size_t off = 0;
  for (int j = 0; j <= 2 * search_submap_num; j++) {
    const int idx = id_min + j - search_submap_num;
    if (idx < win_lo || idx >= win_hi) continue;
    const Submap& sub = *s->submaps[idx];
    transform_cloud_device(sub.cloud, sub.n, s->loop_tgt.ptr + off, pose_f32(sub), s->stream);
    off += sub.n;
    s->launches += 1;
  }
  B200_CUDA(cudaGetLastError());
  size_t m = 0;
  const float4* tgt = filter_on_device(s, s->vg_target, s->loop_tgt.ptr, total, voxel_leaf_size, &m);
  if (m == 0) return sm_fail(s, B200REG_ERR_NO_TARGET, "search_loop: empty target");
  B200_CUDA(cudaStreamSynchronize(s->stream));
  int rc = b200reg_set_input_target_device(reg, tgt, m);
  float fin[16];
  if (rc == B200REG_OK) rc = b200reg_align(reg, guess, fin);  // :229, no guess (a place search passes one)
  double fitness = 0;
  if (rc == B200REG_OK) rc = b200reg_get_fitness_score(reg, 1.7976931348623157e308, &fitness);  // :230
  if (rc != B200REG_OK) {
    s->err = std::string("search_loop: ") + b200reg_last_error(reg);
    return rc;
  }
  out->n_source = source.n;
  out->n_target = m;
  out->fitness = fitness;
  std::memcpy(out->final_T, fin, sizeof(fin));
  if (fitness < threshold_loop_closure_score) {  // :232-246: loop edge (id_min, newest), relative pose from^-1 * (final * init)
    out->accepted = 1;
    double F[16], to[16], rel[16];
    col_to_row(fin, F);
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++) {
        double a = 0;
        for (int k = 0; k < 4; k++) a += F[r * 4 + k] * source.pose[k * 4 + c];
        to[r * 4 + c] = a;
      }
    const double* fr = s->submaps[id_min]->pose;  // Isometry3d::inverse(): R^T, -R^T t
    double inv[16] = {fr[0], fr[4], fr[8], 0, fr[1], fr[5], fr[9], 0, fr[2], fr[6], fr[10], 0, 0, 0, 0, 1};
    for (int r = 0; r < 3; r++) inv[r * 4 + 3] = -(inv[r * 4 + 0] * fr[3] + inv[r * 4 + 1] * fr[7] + inv[r * 4 + 2] * fr[11]);
    for (int r = 0; r < 4; r++)
      for (int c = 0; c < 4; c++) {
        double a = 0;
        for (int k = 0; k < 4; k++) a += inv[r * 4 + k] * to[k * 4 + c];
        rel[r * 4 + c] = a;
      }
    row_to_col(rel, out->relative_pose);
  }
  return B200REG_OK;
}

}  // namespace

extern "C" {

int b200sm_search_loop(b200sm_t s, b200reg_t reg, float voxel_leaf_size, double threshold_loop_closure_score,
                       double distance_loop_closure, double range_of_searching_loop_closure, int search_submap_num,
                       b200sm_loop_result* out) {
  if (!s || !reg || !out || !(voxel_leaf_size > 0) || search_submap_num < 0) return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() {
    std::memset(out, 0, sizeof(*out));
    out->id_min = -1;
    // the closest of the submaps that pass the gates wins (:193-201; the first one on a tie, like the strict `<`)
    const std::vector<LoopCandidate> cands = loop_candidates(s, distance_loop_closure, range_of_searching_loop_closure);
    if (cands.empty()) return (int)B200REG_OK;
    LoopCandidate best = cands[0];
    for (const LoopCandidate& c : cands)
      if (c.dist < best.dist) best = c;
    out->is_candidate = 1;
    out->id_min = best.id;
    out->min_dist = best.dist;
    const Submap& latest = *s->submaps.back();
    int rc = loop_set_source(s, reg, latest);
    if (rc != B200REG_OK) return rc;
    return loop_evaluate(s, reg, best, latest, 0, (int)s->submaps.size(), voxel_leaf_size, threshold_loop_closure_score,
                         search_submap_num, out);
  });
}

// The generalisation SURVEY.md section 8f row 2 names: EVERY submap that passes the two gates is registered against the
// newest one (the reference keeps only the closest), all on the device-resident submaps. shard_rank / shard_world
// (0 / 1 on one GPU) deal the candidates out across processes: candidate k (ascending submap id) belongs to rank
// k mod shard_world; the caller all-gathers the rows (include/b200comm.h).
int b200sm_search_loop_all(b200sm_t s, b200reg_t reg, float voxel_leaf_size, double threshold_loop_closure_score,
                           double distance_loop_closure, double range_of_searching_loop_closure, int search_submap_num,
                           int shard_rank, int shard_world, b200sm_loop_result* out, size_t capacity, size_t* n_out,
                           size_t* n_candidates_total) {
  if (!s || !reg || !n_out || !(voxel_leaf_size > 0) || search_submap_num < 0 || shard_world < 1 || shard_rank < 0 ||
      shard_rank >= shard_world || (!out && capacity))
    return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() {
    *n_out = 0;
    const std::vector<LoopCandidate> cands = loop_candidates(s, distance_loop_closure, range_of_searching_loop_closure);
    if (n_candidates_total) *n_candidates_total = cands.size();
    if (cands.empty()) return (int)B200REG_OK;
    bool have_source = false;
    for (size_t k = 0; k < cands.size(); k++) {
      if ((int)(k % (size_t)shard_world) != shard_rank) continue;
      if (*n_out >= capacity) break;
      if (!have_source) {
        const int rc = loop_set_source(s, reg, *s->submaps.back());
        if (rc != B200REG_OK) return rc;
        have_source = true;
      }
      b200sm_loop_result* r = out + *n_out;
      std::memset(r, 0, sizeof(*r));
      const int rc = loop_evaluate(s, reg, cands[k], *s->submaps.back(), 0, (int)s->submaps.size(), voxel_leaf_size,
                                   threshold_loop_closure_score, search_submap_num, r);
      if (rc != B200REG_OK) return rc;
      *n_out += 1;
    }
    return (int)B200REG_OK;
  });
}

// A backend that runs in its own process receives the frontend's submaps as lidarslam_msgs/SubMap messages (already
// voxel-filtered cloud in the sensor frame + pose + travelled distance, graph_based_slam_component.cpp:91-101): this entry
// point appends one to the session so that b200sm_search_loop / _all work on device-resident copies there too.
int b200sm_import_submap(b200sm_t s, const float* points, size_t n, size_t stride_bytes, long intensity_offset_bytes,
                         const double* pose_colmajor16, double distance) {
  if (!s || (!points && n) || !pose_colmajor16 || !valid_record_layout(stride_bytes, intensity_offset_bytes)) return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() {
    double pose[16];
    col_to_row(pose_colmajor16, pose);
    std::unique_ptr<Submap> sub = new_submap(s->arena, nullptr, n, pose, distance, s->stream);
    if (n) {
      s->uploader.upload(points, n, stride_bytes, intensity_offset_bytes, 0.0f, sub->cloud, s->stream);
      B200_CUDA(cudaStreamSynchronize(s->stream));  // the caller may reuse its buffer
      s->launches += 1;
    }
    s->latest_distance = distance;
    s->submaps.push_back(std::move(sub));
    return (int)B200REG_OK;
  });
}

// doPoseAdjustment (gbs.cpp:262-319): the pose graph over the submaps' poses and LM on the host (csrc/pose_graph.hpp),
// the odometry edges per segment. The session's poses stay as they are.
int b200sm_pose_adjust(b200sm_t s, int num_adjacent_pose_cnstraints, const b200sm_loop_edge* loop_edges, int n_loop_edges,
                       int max_iterations, double* poses_out, b200sm_pose_adjust_result* result) {
  if (!s || !poses_out || num_adjacent_pose_cnstraints < 1 || max_iterations < 0 || n_loop_edges < 0 || (n_loop_edges && !loop_edges))
    return B200REG_ERR_ARG;
  const int n = (int)s->submaps.size();
  if (const int rc = check_loop_edges(s, loop_edges, n_loop_edges, n, "pose_adjust"); rc != B200REG_OK) return rc;
  return sm_guarded(s, [&]() {
    std::vector<pg::Iso> X(n);
    for (int i = 0; i < n; i++) X[i] = pg::iso_from_rowmajor16(s->submaps[i]->pose);
    std::vector<int> ids;
    std::vector<pg::Iso> rel;
    append_loop_edges(loop_edges, n_loop_edges, ids, rel);
    const std::vector<pg::Edge> edges = pg::build_edges(X, num_adjacent_pose_cnstraints, s->seg_first, ids.data(), rel.data(), n_loop_edges);
    const pg::LmResult r = pg::optimize(X, edges, max_iterations);
    for (int i = 0; i < n; i++) pg::iso_to_colmajor16(X[i], poses_out + 16 * (size_t)i);
    if (result) {
      result->chi2_initial = r.chi2_initial;
      result->chi2_final = r.chi2_final;
      result->iterations = r.iterations;
      result->trials = r.trials;
      result->n_vertices = n;
      result->n_edges = (int)edges.size();
    }
    return (int)B200REG_OK;
  });
}

}  // extern "C"

namespace {

size_t map_points(b200sm_t s) {
  size_t total = 0;
  for (const auto& sub : s->submaps) total += sub->n;
  return total;
}

// The table of a launch over submaps [first, size) whose blocks serve `tile` points each: entry r is submap ids[r], whose
// first tile is first_tile[r]. An empty submap owns no tile (with skip_empty, no entry either). A submap of 2^32 points or
// more, and more than 2^31 - 1 tiles in all, are refused with the caller's messages.
struct SubmapTiles {
  std::vector<size_t> ids;
  std::vector<unsigned> first_tile;
  unsigned long long tiles = 0;
};
int submap_tiles(b200sm_t s, size_t first, size_t tile, bool skip_empty, const char* too_big, const char* too_many, SubmapTiles* t) {
  for (size_t i = first; i < s->submaps.size(); i++) {
    const size_t n = s->submaps[i]->n;
    if (n == 0 && skip_empty) continue;
    if (n > 0xffffffffull) return sm_fail(s, B200REG_ERR_ARG, too_big);
    t->ids.push_back(i);
    t->first_tile.push_back((unsigned)t->tiles);
    t->tiles += (n + tile - 1) / tile;
  }
  if (t->tiles > 0x7fffffffull) return sm_fail(s, B200REG_ERR_ARG, too_many);
  return B200REG_OK;
}

// the float pose of submap k, 3x4 row-major: the caller's column-major one (poses_colmajor16 + 16 k) if given, else the
// session's, cast to float (affine.matrix().cast<float>())
void submap_pose_f(b200sm_t s, size_t k, const double* poses_colmajor16, float* T) {
  for (int r = 0; r < 3; r++)
    for (int c = 0; c < 4; c++)
      T[r * 4 + c] = poses_colmajor16 ? (float)poses_colmajor16[16 * k + c * 4 + r] : (float)s->submaps[k]->pose[r * 4 + c];
}

// publishMap (sm.cpp:529-552) / modified_map (gbs.cpp:321-368): every submap through its pose cast to float, concatenated in
// submap order, in one launch into s->assembled (total = map_points(s) > 0). Enqueue only.
int assemble_on_device(b200sm_t s, const double* poses_colmajor16, size_t total) {
  const int n_sub = (int)s->submaps.size();
  SubmapTiles t;
  const int rc = submap_tiles(s, 0, ASSEMBLE_TILE, false, "assemble_map: a submap of 2^32 points or more",
                              "assemble_map: map too large for one launch", &t);
  if (rc != B200REG_OK) return rc;
  std::vector<AssembleEntry> table(n_sub);
  for (int i = 0; i < n_sub; i++) {
    const Submap& sub = *s->submaps[i];
    AssembleEntry& e = table[i];
    e.cloud = sub.cloud;
    e.out_offset = i ? table[i - 1].out_offset + table[i - 1].n : 0;
    e.n = (unsigned)sub.n;
    e.first_tile = t.first_tile[i];
    submap_pose_f(s, i, poses_colmajor16, e.T.m);
  }
  s->assemble_table.ensure(n_sub);
  s->assembled.ensure(total);
  B200_CUDA(cudaMemcpyAsync(s->assemble_table.ptr, table.data(), n_sub * sizeof(AssembleEntry), cudaMemcpyHostToDevice, s->stream));
  assemble_map_kernel<<<(unsigned)t.tiles, ASSEMBLE_THREADS, 0, s->stream>>>(s->assemble_table.ptr, n_sub, s->assembled.ptr);
  B200_CUDA(cudaGetLastError());
  s->launches += 1;
  return (int)B200REG_OK;
}

}  // namespace

extern "C" {

// the assembled map read back (count always reported, at most capacity copied)
int b200sm_assemble_map(b200sm_t s, const double* poses_colmajor16, float* out_xyzi, size_t capacity, size_t* n, size_t* offsets) {
  if (!s || (!out_xyzi && capacity)) return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() {
    const int n_sub = (int)s->submaps.size();
    size_t total = 0;
    for (int i = 0; i < n_sub; i++) {
      if (offsets) offsets[i] = total;
      total += s->submaps[i]->n;
    }
    if (offsets) offsets[n_sub] = total;
    if (n) *n = total;
    if (capacity == 0 || total == 0) return (int)B200REG_OK;  // a size query launches nothing
    const int rc = assemble_on_device(s, poses_colmajor16, total);
    if (rc != B200REG_OK) return rc;
    return read_back(s, s->assembled.ptr, total, out_xyzi, capacity, n);
  });
}

}  // extern "C"

namespace {

// One whole file: `head`, then body_bytes bytes of `body`. nullptr once it is written and closed, else what failed
// ("cannot open " or "writing "), with errno as the failing call left it.
const char* write_file(const std::string& path, const std::string& head, const void* body = nullptr, size_t body_bytes = 0) {
  FILE* fp = std::fopen(path.c_str(), "wb");
  if (!fp) return "cannot open ";
  bool ok = std::fwrite(head.data(), 1, head.size(), fp) == head.size() && (body_bytes == 0 || std::fwrite(body, 1, body_bytes, fp) == body_bytes);
  ok = (std::fclose(fp) == 0) && ok;
  return ok ? nullptr : "writing ";
}

// Pieces [0, n) (n > 0) of device data written to files through the session's two pinned staging buffers in turn
// (`most` bytes each): piece p + 1 is copied while this thread writes piece p, and a buffer is refilled only after its
// previous piece has been written. enqueue(p, buf) puts piece p into `buf` on the session's stream; write(p, buf) writes
// it once it has arrived and returns B200REG_OK or an error code. On every return no copy into the staging buffers is
// left in flight and `fp`, the file the callbacks write, is closed.
template <typename Enqueue, typename Write>
int write_staged(b200sm_t s, size_t n, size_t most, FILE*& fp, Enqueue&& enqueue, Write&& write) {
  cudaEvent_t copied[2] = {nullptr, nullptr};
  struct Cleanup {
    cudaEvent_t* ev;
    FILE** fp;
    cudaStream_t st;
    ~Cleanup() {
      cudaStreamSynchronize(st);
      for (int b = 0; b < 2; b++)
        if (ev[b]) cudaEventDestroy(ev[b]);
      if (*fp) std::fclose(*fp);
    }
  } cleanup{copied, &fp, s->stream};
  for (auto& st : s->pcd_staging) st.ensure(most);
  for (cudaEvent_t& e : copied) B200_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  auto put = [&](size_t p) {
    enqueue(p, s->pcd_staging[p & 1].ptr);
    B200_CUDA(cudaEventRecord(copied[p & 1], s->stream));
  };
  put(0);
  for (size_t p = 0; p < n; p++) {
    if (p + 1 < n) put(p + 1);  // its buffer held piece p - 1, already written
    B200_CUDA(cudaEventSynchronize(copied[p & 1]));
    const int rc = write(p, s->pcd_staging[p & 1].ptr);
    if (rc != B200REG_OK) return rc;
  }
  return (int)B200REG_OK;
}

// pcl::io::savePCDFileASCII of the device cloud pts[0 .. total) (total > 0): formatted on the device chunk by chunk
// (one stream: encode, copy, encode, ...) and written by write_staged. `what` prefixes the error messages.
int write_pcd_ascii(b200sm_t s, const float4* pts, size_t total, const char* path, const char* what, size_t* n_points, size_t* n_bytes) {
  PcdEncoder& E = s->pcd;
  const int launches_before = E.launches;
  E.measure(pts, total, s->stream);
  s->launches += E.launches - launches_before;
  const std::string header = pcd_ascii_header(total);
  size_t file_bytes = header.size(), most = 0;
  for (size_t b : E.chunk_bytes) {
    file_bytes += b;
    most = std::max(most, b);
  }
  if (n_points) *n_points = total;
  if (n_bytes) *n_bytes = file_bytes;
  FILE* fp = std::fopen(path, "wb");
  if (!fp) {
    s->err = std::string(what) + ": cannot open " + path + ": " + std::strerror(errno);
    return (int)B200REG_ERR_IO;
  }
  const size_t chunks = E.chunk_bytes.size();
  auto enqueue = [&](size_t c, char* buf) {
    E.encode_chunk(pts, total, c, s->stream);
    s->launches += 1;
    B200_CUDA(cudaMemcpyAsync(buf, E.text.ptr, E.chunk_bytes[c], cudaMemcpyDeviceToHost, s->stream));
  };
  auto write = [&](size_t c, const char* buf) {
    bool ok = c > 0 || std::fwrite(header.data(), 1, header.size(), fp) == header.size();
    ok = ok && std::fwrite(buf, 1, E.chunk_bytes[c], fp) == E.chunk_bytes[c];
    if (ok && c + 1 == chunks) {
      ok = std::fclose(fp) == 0;
      fp = nullptr;
    }
    if (ok) return (int)B200REG_OK;
    s->err = std::string(what) + ": writing " + path + ": " + std::strerror(errno);
    return (int)B200REG_ERR_IO;
  };
  return write_staged(s, chunks, most, fp, enqueue, write);
}

}  // namespace

extern "C" {

// savePCDFileASCII("map.pcd", modified_map) (gbs.cpp:369): the map assembled and formatted on the device (write_pcd_ascii)
int b200sm_save_map_pcd_ascii(b200sm_t s, const double* poses_colmajor16, const char* path, size_t* n_points, size_t* n_bytes) {
  if (!s || !path) return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() {
    const size_t total = map_points(s);
    if (total == 0) return sm_fail(s, B200REG_ERR_ARG, "save_map_pcd_ascii: the map has no points");  // PCL throws, writes nothing
    int rc = assemble_on_device(s, poses_colmajor16, total);
    if (rc != B200REG_OK) return rc;
    return write_pcd_ascii(s, s->assembled.ptr, total, path, "save_map_pcd_ascii", n_points, n_bytes);
  });
}

int b200sm_get_stats(b200sm_t s, b200sm_stats* out) {
  if (!s || !out) return B200REG_ERR_ARG;
  out->n_scan = s->n_scan;
  out->n_filtered = s->n_filtered;
  out->n_targeted = s->n_targeted;
  out->n_submaps = s->submaps.size();
  out->kernel_launches = s->launches;
  out->trans = s->trans;
  out->latest_distance = s->latest_distance;
  return B200REG_OK;
}

}  // extern "C"

// ---- IMU de-skew (SURVEY.md section 8f row 4): LidarUndistortion of scanmatcher/include/scanmatcher/lidar_undistortion.hpp ----
extern "C" {

int b200sm_imu_set_scan_period(b200sm_t s, double scan_period) {
  if (!s || !(scan_period > 0)) return B200REG_ERR_ARG;
  s->imu.scan_period = scan_period;
  return B200REG_OK;
}

int b200sm_imu_push(b200sm_t s, const float* angular_velocity3, const float* linear_acceleration3, const float* orientation_xyzw,
                    double stamp) {
  if (!s || !angular_velocity3 || !linear_acceleration3 || !orientation_xyzw) return B200REG_ERR_ARG;
  s->imu.get_imu(angular_velocity3, linear_acceleration3, orientation_xyzw, stamp);
  return B200REG_OK;
}

int b200sm_deskew_next_scan(b200sm_t s, double scan_time) {
  if (!s) return B200REG_ERR_ARG;
  s->deskew_armed = true;
  s->deskew_scan_time = scan_time;
  return B200REG_OK;
}

}  // extern "C"

// ---- frame transforms of the cloud callback: doTransform into the robot frame (sm.cpp:188-199), use_odom (:333-348) ----
namespace {
bool valid_transform(const double* t3, const double* q_xyzw) {
  for (int k = 0; k < 3; k++)
    if (!std::isfinite(t3[k])) return false;
  for (int k = 0; k < 4; k++)
    if (!std::isfinite(q_xyzw[k])) return false;
  return q_xyzw[0] != 0.0 || q_xyzw[1] != 0.0 || q_xyzw[2] != 0.0 || q_xyzw[3] != 0.0;
}
}  // namespace

extern "C" {

int b200sm_set_sensor_transform(b200sm_t s, const double* translation3, const double* quat_xyzw) {
  if (!s) return B200REG_ERR_ARG;
  if (!translation3 && !quat_xyzw) {
    s->sensor_tf_set = false;
    return B200REG_OK;
  }
  if (!translation3 || !quat_xyzw) return sm_fail(s, B200REG_ERR_ARG, "set_sensor_transform: one of translation / quaternion is NULL");
  if (!valid_transform(translation3, quat_xyzw))
    return sm_fail(s, B200REG_ERR_ARG, "set_sensor_transform: non-finite value or zero quaternion");
  sensor_matrix_f(translation3, quat_xyzw, s->sensor_tf.m);
  s->sensor_tf_set = true;
  return B200REG_OK;
}

int b200sm_odom_next_scan(b200sm_t s, const double* translation3, const double* quat_xyzw) {
  if (!s) return B200REG_ERR_ARG;
  if (!translation3 || !quat_xyzw) return sm_fail(s, B200REG_ERR_ARG, "odom_next_scan: NULL translation or quaternion");
  if (!valid_transform(translation3, quat_xyzw)) return sm_fail(s, B200REG_ERR_ARG, "odom_next_scan: non-finite value or zero quaternion");
  odom_matrix_f(translation3, quat_xyzw, s->odom_mat);
  s->odom_armed = true;
  return B200REG_OK;
}

int b200sm_imu_adjust_distortion(b200sm_t s, float* points, size_t n, size_t stride_bytes, long intensity_offset_bytes,
                                 double scan_time) {
  if (!s || (!points && n) || !valid_record_layout(stride_bytes, intensity_offset_bytes)) return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() {
    if (n == 0) return (int)B200REG_OK;
    s->upload.ensure(n);
    s->uploader.upload(points, n, stride_bytes, intensity_offset_bytes, 0.0f, s->upload.ptr, s->stream);
    char* b = reinterpret_cast<char*>(points);
    const int before = s->imu.launches;
    s->imu.adjust_distortion(s->upload.ptr, n, reinterpret_cast<const float*>(b), reinterpret_cast<const float*>(b + (n - 1) * stride_bytes),
                             scan_time, s->stream);
    s->launches += 1 + s->imu.launches - before;
    std::vector<float4> host(n);
    B200_CUDA(cudaMemcpyAsync(host.data(), s->upload.ptr, n * sizeof(float4), cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    for (size_t i = 0; i < n; i++) {  // x, y, z back into the caller's records; every other field is untouched
      float* f = reinterpret_cast<float*>(b + i * stride_bytes);
      f[0] = host[i].x;
      f[1] = host[i].y;
      f[2] = host[i].z;
    }
    return (int)B200REG_OK;
  });
}

int b200sm_imu_get_state(b200sm_t s, int* ptr_front, int* ptr_last, int* ptr_last_iter) {
  if (!s) return B200REG_ERR_ARG;
  if (ptr_front) *ptr_front = s->imu.ptr_front;
  if (ptr_last) *ptr_last = s->imu.ptr_last;
  if (ptr_last_iter) *ptr_last_iter = s->imu.ptr_last_iter;
  return B200REG_OK;
}

int b200sm_imu_get_sample(b200sm_t s, int index, double* stamp, float* rpy3, float* shift3, float* velo3) {
  if (!s || index < 0 || index >= IMU_QUE) return B200REG_ERR_ARG;
  if (stamp) *stamp = s->imu.time[index];
  if (rpy3) {
    rpy3[0] = s->imu.roll[index];
    rpy3[1] = s->imu.pitch[index];
    rpy3[2] = s->imu.yaw[index];
  }
  for (int c = 0; c < 3; c++) {
    if (shift3) shift3[c] = s->imu.shift[index][c];
    if (velo3) velo3[c] = s->imu.velo[index][c];
  }
  return B200REG_OK;
}

int b200sm_imu_get_trace(b200sm_t s, size_t capacity, size_t* n, float* rel_time, double* t, int* front, unsigned char* skip,
                         int* k_first, int* rounds) {
  if (!s || !n) return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() {
    *n = s->imu.get_trace(capacity, rel_time, t, front, skip, k_first, rounds, s->stream);
    return (int)B200REG_OK;
  });
}

}  // extern "C"

// ---- localisation in a prior map: the map resident on the device, the registration target a stable cut around the pose ----
extern "C" int b200reg_check_target_grid_device(b200reg_t h, const void* dev, size_t n);  // capi.cu (library-internal)

namespace {

// the freshly loaded map replaces the previous one (whose memory is freed); the next frame cuts anew
int install_prior_map(b200sm_t s, size_t n) {
  std::swap(s->prior_map.ptr, s->prior_incoming.ptr);
  std::swap(s->prior_map.cap, s->prior_incoming.cap);
  s->prior_incoming.release();
  s->n_prior = n;
  s->reloc.invalidate();
  s->cut_stale = true;
  s->cut_pending = false;
  s->n_cuts = 0;
  return B200REG_OK;
}

// The rows of the prior map within crop_radius (horizontally) of (cx, cy), in map order, into s->cut: count per tile, scan,
// read the total, size the output, write. Returns with the stream synchronised. B200REG_ERR_NO_TARGET when no row is kept:
// nothing is written then and the previous cut stays as it is.
int make_cut(b200sm_t s, double cx, double cy) {
  const size_t tiles = cut_tiles(s->n_prior);
  const double r2 = s->crop_radius * s->crop_radius;
  s->cut_counts.ensure(tiles + 2);
  cut_count_kernel<<<(unsigned)tiles, CUT_THREADS, 0, s->stream>>>(s->prior_map.ptr, s->n_prior, cx, cy, r2, s->cut_counts.ptr);
  B200_CUDA(cudaGetLastError());
  counter_scan_async(s->cut_counts.ptr, tiles, s->cut_scan_tmp, s->stream);
  B200_CUDA(cudaGetLastError());
  unsigned total = 0;
  B200_CUDA(cudaMemcpyAsync(&total, s->cut_counts.ptr + tiles, sizeof(unsigned), cudaMemcpyDeviceToHost, s->stream));
  B200_CUDA(cudaStreamSynchronize(s->stream));
  s->launches += 4;
  if (total == 0) {
    char msg[200];
    std::snprintf(msg, sizeof(msg), "localize: no point of the prior map within %.3f m of (%.3f, %.3f)", s->crop_radius, cx, cy);
    return sm_fail(s, B200REG_ERR_NO_TARGET, msg);
  }
  s->have_cut = false;  // until the rows are in place
  s->cut.ensure(total);  // may free: the stream is idle and the engine keeps its own copy of its target
  unsigned* tripped = s->cut_counts.ptr + tiles + 1;
  B200_CUDA(cudaMemsetAsync(tripped, 0, sizeof(unsigned), s->stream));
  cut_write_kernel<<<(unsigned)tiles, CUT_THREADS, 0, s->stream>>>(s->prior_map.ptr, s->n_prior, cx, cy, r2, s->cut_counts.ptr, total,
                                                                   s->cut.ptr, tripped);
  B200_CUDA(cudaGetLastError());
  unsigned flag = 0;
  B200_CUDA(cudaMemcpyAsync(&flag, tripped, sizeof(unsigned), cudaMemcpyDeviceToHost, s->stream));
  B200_CUDA(cudaStreamSynchronize(s->stream));
  s->launches += 1;
  if (flag) {
    s->cut_stale = true;
    return sm_fail(s, B200REG_ERR_CUDA, "localize: the cut's write pass met a row beyond the counted total (nothing was stored there)");
  }
  s->n_cut = total;
  s->cut_centre[0] = cx;
  s->cut_centre[1] = cy;
  s->n_cuts += 1;
  s->have_cut = true;
  s->cut_stale = false;
  s->cut_pending = true;
  return B200REG_OK;
}

// step 2 of a localising frame: a cut around the current position if there is none or it is stale, then a pending cut
// becomes the engine's target. An NDT cut whose voxel grid would overflow int32 is not handed over (it stays pending).
int ensure_cut_target(b200sm_t s, b200reg_t reg, int kind) {
  if (!s->have_cut || s->cut_stale) {
    const int rc = make_cut(s, s->position[0], s->position[1]);
    if (rc != B200REG_OK) return rc;
  }
  if (!s->cut_pending) return B200REG_OK;
  if (kind == B200REG_NDT) {
    const int rc = b200reg_check_target_grid_device(reg, s->cut.ptr, s->n_cut);
    if (rc != B200REG_OK) {
      s->err = std::string("localize: ") + b200reg_last_error(reg);
      return rc;
    }
  }
  const int rc = hand_over_target(s, reg, kind == B200REG_GICP, s->cut.ptr, s->n_cut, "localize: the cut is empty after VoxelGrid",
                                  &s->n_cut_target);
  if (rc == B200REG_OK) s->cut_pending = false;
  return rc;
}

// step 3 of b200sm_localize_init / b200sm_localize_global: the filtered scan registered from `count` guesses in one batch
// launch (the scan read in place `count` times); the converged row with the highest trans_probability, the lowest index on
// a tie, becomes the pose. *best = its index, or -1 when none converged (pose unchanged).
int refine_hypotheses(b200sm_t s, b200reg_t reg, const float* guesses, int count, b200reg_batch_result* results, int* best,
                      const char* who) {
  std::vector<const void*> sources((size_t)count, s->d_filtered);
  std::vector<size_t> sizes((size_t)count, s->n_filtered);
  const int rc = b200reg_ndt_align_batch_device(reg, count, sources.data(), sizes.data(), guesses, results);
  if (rc != B200REG_OK) {
    s->err = std::string(who) + b200reg_last_error(reg);
    return rc;
  }
  int pick = -1;
  for (int k = 0; k < count; k++)
    if (results[k].status == B200REG_OK && results[k].converged &&
        (pick < 0 || results[k].trans_probability > results[pick].trans_probability))
      pick = k;
  if (pick >= 0) adopt_pose(s, results[pick].final_T);
  if (best) *best = pick;
  return (int)B200REG_OK;
}

}  // namespace

extern "C" {

int b200sm_set_prior_map_pcd(b200sm_t s, const char* path, size_t* n_points) {
  if (!s || !path) return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() {
    size_t n = 0;
    std::string why;
    const int before = s->pcd_loader.launches;
    const int rc = s->pcd_loader.load(path, s->prior_incoming, &n, why, s->stream);  // the current map is not touched
    s->launches += s->pcd_loader.launches - before;
    if (rc == B200REG_OK && n != 0 && n <= CUT_MAX_POINTS) {
      if (n_points) *n_points = n;
      return install_prior_map(s, n);
    }
    s->prior_incoming.release();
    s->err = std::string("set_prior_map_pcd: ") + path + ": ";
    if (rc != B200REG_OK) {
      s->err += why;
      return rc;
    }
    s->err += n == 0 ? "the file has no points" : "more than 2^32 - 1 points";
    return (int)B200REG_ERR_ARG;
  });
}

int b200sm_set_prior_map(b200sm_t s, const float* points, size_t n, size_t stride_bytes, long intensity_offset_bytes) {
  if (!s || !points || n == 0 || !valid_record_layout(stride_bytes, intensity_offset_bytes)) return B200REG_ERR_ARG;
  if (n > CUT_MAX_POINTS) return sm_fail(s, B200REG_ERR_ARG, "set_prior_map: more than 2^32 - 1 points");
  return sm_guarded(s, [&]() {
    s->prior_incoming.ensure(n);
    // an uploader of its own, gone on return: the session's would keep a device (and, for pageable input, a pinned host)
    // copy of the map's raw records for the rest of its life
    CloudUploader once;
    once.upload(points, n, stride_bytes, intensity_offset_bytes, 0.0f, s->prior_incoming.ptr, s->stream);
    B200_CUDA(cudaStreamSynchronize(s->stream));  // the caller may reuse its buffer
    s->launches += 1;
    return install_prior_map(s, n);
  });
}

int b200sm_set_localization_params(b200sm_t s, double crop_radius, double recrop_distance) {
  if (!s) return B200REG_ERR_ARG;
  if (!std::isfinite(crop_radius) || !std::isfinite(recrop_distance) || !(crop_radius > 0) || !(recrop_distance >= 0))
    return sm_fail(s, B200REG_ERR_ARG, "set_localization_params: crop_radius must be finite and > 0, recrop_distance finite and >= 0");
  s->crop_radius = crop_radius;
  s->recrop_distance = recrop_distance;
  s->cut_stale = true;
  return B200REG_OK;
}

int b200sm_localize_cloud(b200sm_t s, b200reg_t reg, const float* points, size_t n, size_t stride_bytes, long intensity_offset_bytes,
                          double* pose7_out, float* final_T_colmajor16_out, int* target_recut) {
  if (!valid_frame_args(s, reg, points, n, stride_bytes, intensity_offset_bytes)) return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() {
    if (target_recut) *target_recut = 0;
    if (s->n_prior == 0) return sm_fail(s, B200REG_ERR_NO_TARGET, "localize_cloud: no prior map");
    const bool use_odom = s->odom_armed;  // armed for this frame only, like the de-skew
    s->odom_armed = false;
    int kind = B200REG_NDT;
    b200reg_get_kind(reg, &kind);
    upload_frame(s, points, n, stride_bytes, intensity_offset_bytes);
    int rc = ensure_cut_target(s, reg, kind);
    if (rc != B200REG_OK) return rc;
    float final_col[16];
    rc = register_frame(s, reg, use_odom, final_col);
    if (rc != B200REG_OK) return rc;
    // the target follows the pose: once it is recrop_distance from the centre of the cut, cut again around it now; the
    // new cut becomes the target at the start of the next frame
    const double dx = s->position[0] - s->cut_centre[0], dy = s->position[1] - s->cut_centre[1];
    s->dist_from_centre = std::sqrt(dx * dx + dy * dy);
    if (s->dist_from_centre >= s->recrop_distance) {
      rc = make_cut(s, s->position[0], s->position[1]);
      if (rc == B200REG_OK) {
        if (target_recut) *target_recut = 1;
      } else if (rc != B200REG_ERR_NO_TARGET) {
        return rc;
      }  // an empty re-cut: the frame stands, the old cut and target stay, the next frame tries again
    }
    write_pose(s, pose7_out);
    if (final_T_colmajor16_out) std::memcpy(final_T_colmajor16_out, final_col, sizeof(final_col));
    return (int)B200REG_OK;
  });
}

int b200sm_localize_init(b200sm_t s, b200reg_t reg, const float* points, size_t n, size_t stride_bytes, long intensity_offset_bytes,
                         const float* guesses, int count, b200reg_batch_result* results, int* best) {
  if (!valid_frame_args(s, reg, points, n, stride_bytes, intensity_offset_bytes) || !guesses || count < 1 || !results)
    return B200REG_ERR_ARG;
  int kind = B200REG_NDT;
  b200reg_get_kind(reg, &kind);
  if (kind != B200REG_NDT) return sm_fail(s, B200REG_ERR_ARG, "localize_init: the batch solver is NDT's");
  return sm_guarded(s, [&]() {
    if (best) *best = -1;
    if (s->n_prior == 0) return sm_fail(s, B200REG_ERR_NO_TARGET, "localize_init: no prior map");
    upload_frame(s, points, n, stride_bytes, intensity_offset_bytes);
    int rc = ensure_cut_target(s, reg, kind);
    if (rc != B200REG_OK) return rc;
    rc = set_source_from_scan(s, reg);
    if (rc != B200REG_OK) return rc;
    return refine_hypotheses(s, reg, guesses, count, results, best, "localize_init: ");
  });
}

int b200sm_localize_global(b200sm_t s, b200reg_t reg, const float* points, size_t n, size_t stride_bytes,
                           long intensity_offset_bytes, const b200sm_global_search* spec, int* candidates,
                           b200reg_batch_result* results, b200sm_global_result* out) {
  if (!valid_frame_args(s, reg, points, n, stride_bytes, intensity_offset_bytes) || !spec || !candidates || !results)
    return B200REG_ERR_ARG;
  int kind = B200REG_NDT;
  b200reg_get_kind(reg, &kind);
  if (kind != B200REG_NDT) return sm_fail(s, B200REG_ERR_ARG, "localize_global: the batch solver is NDT's");
  const long long n_hyp = global_grid_count(spec->radius, spec->step, spec->yaw_steps, spec->top_k);
  if (n_hyp < 0)
    return sm_fail(s, B200REG_ERR_ARG, "localize_global: radius must be finite and >= 0, step finite and > 0, yaw_steps in "
                                       "1..4096, top_k in 1..1024, floor(radius / step) <= 4096 and at most 2^24 hypotheses");
  return sm_guarded(s, [&]() {
    if (out) {
      std::memset(out, 0, sizeof(*out));
      out->best = -1;
    }
    if (s->n_prior == 0) return sm_fail(s, B200REG_ERR_NO_TARGET, "localize_global: no prior map");
    upload_frame(s, points, n, stride_bytes, intensity_offset_bytes);
    int rc = ensure_cut_target(s, reg, B200REG_NDT);
    if (rc != B200REG_OK) return rc;
    rc = set_source_from_scan(s, reg);
    if (rc != B200REG_OK) return rc;
    std::vector<float> poses;
    global_grid_build(s->position, s->quat, spec->radius, spec->step, spec->yaw_steps, poses);
    std::vector<double> scores((size_t)n_hyp);
    std::vector<long long> hits((size_t)n_hyp);
    rc = b200reg_ndt_score_poses(reg, (int)n_hyp, poses.data(), scores.data(), hits.data());
    if (rc != B200REG_OK) {
      s->err = std::string("localize_global: ") + b200reg_last_error(reg);
      return rc;
    }
    const float score_ms = b200reg_last_score_ms(reg);
    const std::vector<int> top = global_select_top_k(scores.data(), n_hyp, spec->top_k);
    const int k = (int)top.size();
    std::vector<float> guesses((size_t)k * 16);
    for (int r = 0; r < k; r++) {
      candidates[r] = top[r];
      std::memcpy(guesses.data() + (size_t)r * 16, poses.data() + (size_t)top[r] * 16, 16 * sizeof(float));
    }
    long long hits_total = 0;
    for (long long h : hits) hits_total += h;
    s->global_poses.swap(poses);
    s->global_scores.swap(scores);
    s->global_hits.swap(hits);
    int best = -1;
    rc = refine_hypotheses(s, reg, guesses.data(), k, results, &best, "localize_global: ");
    if (out) {
      out->n_hypotheses = n_hyp;
      out->hits_total = hits_total;
      out->n_refined = k;
      out->best = best;
      out->score_ms = score_ms;
    }
    return rc;
  });
}

int b200sm_get_global_search(b200sm_t s, size_t capacity, size_t* n, float* poses_colmajor16, double* scores, long long* hits) {
  if (!s) return B200REG_ERR_ARG;
  const size_t total = s->global_scores.size(), m = std::min(capacity, total);
  if (n) *n = total;
  if (poses_colmajor16 && m) std::memcpy(poses_colmajor16, s->global_poses.data(), m * 16 * sizeof(float));
  if (scores && m) std::memcpy(scores, s->global_scores.data(), m * sizeof(double));
  if (hits && m) std::memcpy(hits, s->global_hits.data(), m * sizeof(long long));
  return B200REG_OK;
}

int b200sm_relocalize(b200sm_t s, b200reg_t reg, const float* points, size_t n, size_t stride_bytes, long intensity_offset_bytes,
                      const b200sm_relocalize_params* params, b200sm_relocalize_row* rows, size_t capacity,
                      b200sm_relocalize_result* out) {
  if (!valid_frame_args(s, reg, points, n, stride_bytes, intensity_offset_bytes) || !rows) return B200REG_ERR_ARG;
  RlParams p;
  if (params) {
    p.resolution = params->resolution;
    p.z_min = params->z_min;
    p.z_max = params->z_max;
    p.yaw_steps = params->yaw_steps;
    p.num_levels = params->num_levels;
    p.min_score = params->min_score;
    p.top_k = params->top_k;
    p.accept_fitness = params->accept_fitness;
  }
  if (!rl_params_valid(p))
    return sm_fail(s, B200REG_ERR_ARG, "relocalize: resolution must be finite and > 0, z_min < z_max finite, yaw_steps in 1..4096, "
                                       "num_levels in 1..16, min_score in [0, 1], top_k in 1..64 and accept_fitness finite and > 0");
  if (capacity < (size_t)p.top_k) return sm_fail(s, B200REG_ERR_ARG, "relocalize: fewer rows than top_k");
  int kind = B200REG_NDT;
  b200reg_get_kind(reg, &kind);
  return sm_guarded(s, [&]() {
    b200sm_relocalize_result res;
    std::memset(&res, 0, sizeof(res));
    res.best = -1;
    if (out) *out = res;
    if (s->n_prior == 0) return sm_fail(s, B200REG_ERR_NO_TARGET, "relocalize: no prior map");
    upload_frame(s, points, n, stride_bytes, intensity_offset_bytes);
    int rc = set_source_from_scan(s, reg);
    if (rc != B200REG_OK) return rc;
    std::string why;
    const int before = s->reloc.launches;
    rc = s->reloc.ensure_pyramid(s->prior_map.ptr, s->n_prior, p, why, s->stream);
    s->launches += s->reloc.launches - before;
    if (rc != B200REG_OK) return sm_fail(s, rc, ("relocalize: " + why).c_str());
    const RlGrid g = s->reloc.grid;
    std::vector<double> rot_d;
    std::vector<float> rot_f;
    rl_rotations(s->position, s->quat, p.yaw_steps, rot_d, rot_f);
    const double z0 = s->position[2];
    RlSearchInfo info;
    const int before_search = s->reloc.launches;
    rc = s->reloc.search(s->d_filtered, s->n_filtered, rot_f, z0, p, info, why, s->stream);
    s->launches += s->reloc.launches - before_search;
    res.width = g.W;
    res.height = g.H;
    res.origin_cell[0] = g.i0;
    res.origin_cell[1] = g.j0;
    res.m = info.m;
    res.t0 = info.t0;
    res.t = info.t;
    res.leaves = (unsigned long long)p.yaw_steps * (unsigned long long)g.W * (unsigned long long)g.H;
    for (int h = 0; h < RL_MAX_LEVELS; h++) res.nodes[h] = info.nodes[h];
    res.pyramid_builds = s->reloc.builds;
    res.search_ms = info.ms;
    if (out) *out = res;
    if (rc != B200REG_OK) return sm_fail(s, rc, ("relocalize: " + why).c_str());
    // the refinement: each row registered against the cut around its cell, the engine's plain calls
    const int n_rows = (int)info.tiles.size();
    for (int r = 0; r < n_rows; r++) {
      b200sm_relocalize_row& row = rows[r];
      std::memset(&row, 0, sizeof(row));
      const long long idx = rl_key_index(info.keys[(size_t)r]);
      row.yaw_index = (int)(idx / (g.W * g.H));
      row.cell_i = (int)(idx % g.W);
      row.cell_j = (int)((idx / g.W) % g.H);
      row.score = (int)rl_key_score(info.keys[(size_t)r]);
      rl_guess(rot_d.data() + 9 * (size_t)row.yaw_index, g, p.resolution, z0, row.cell_i, row.cell_j, row.guess);
      const double cx = (double)((long long)g.i0 + row.cell_i) * p.resolution, cy = (double)((long long)g.j0 + row.cell_j) * p.resolution;
      row.status = make_cut(s, cx, cy);
      if (row.status == B200REG_OK && kind == B200REG_NDT) {
        row.status = b200reg_check_target_grid_device(reg, s->cut.ptr, s->n_cut);
        if (row.status != B200REG_OK) s->err = std::string("relocalize: ") + b200reg_last_error(reg);
      }
      if (row.status == B200REG_OK) {
        row.status = hand_over_target(s, reg, kind == B200REG_GICP, s->cut.ptr, s->n_cut, "relocalize: the cut is empty after VoxelGrid",
                                      &s->n_cut_target);
        if (row.status == B200REG_OK) s->cut_pending = false;
      }
      if (row.status == B200REG_OK) row.status = b200reg_adopt_source_device(reg, s->d_filtered, s->n_filtered);
      if (row.status == B200REG_OK) row.status = b200reg_align(reg, row.guess, row.final_T);
      if (row.status == B200REG_OK) row.status = b200reg_get_fitness_score(reg, DBL_MAX, &row.fitness);
      if (row.status != B200REG_OK) {
        if (row.status == B200REG_ERR_CUDA) return sm_fail(s, row.status, ("relocalize: " + std::string(b200reg_last_error(reg))).c_str());
        continue;
      }
      b200reg_has_converged(reg, &row.converged);
      b200reg_stats st;
      if (b200reg_get_stats(reg, &st) == B200REG_OK) row.iterations = st.iterations;
      if (kind == B200REG_NDT) b200reg_ndt_get_transformation_probability(reg, &row.trans_probability);
    }
    if (n_rows > 0) s->cut_stale = true;  // the rows replaced the cut and the target: the next frame cuts around the pose
    int best = -1;
    for (int r = 0; r < n_rows; r++)
      if (rows[r].status == B200REG_OK && rows[r].converged && rows[r].fitness < p.accept_fitness &&
          (best < 0 || rows[r].fitness < rows[best].fitness))
        best = r;
    if (best >= 0) adopt_pose(s, rows[best].final_T);
    res.n_rows = n_rows;
    res.best = best;
    if (out) *out = res;
    return (int)B200REG_OK;
  });
}

int b200sm_get_relocalize_grid(b200sm_t s, int level, unsigned char* out, size_t capacity, long long* width, long long* height) {
  if (!s) return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() {
    std::string why;
    const int rc = s->reloc.read_level(level, out, capacity, width, height, why, s->stream);
    if (rc != B200REG_OK) return sm_fail(s, rc, why.c_str());
    return rc;
  });
}

int b200sm_relocalize_score_nodes(b200sm_t s, int level, long long count, const int* k_i_j, int* scores) {
  if (!s) return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() {
    std::string why;
    const int rc = s->reloc.score_nodes(level, count, k_i_j, scores, why, s->stream);
    if (rc != B200REG_OK) return sm_fail(s, rc, why.c_str());
    return rc;
  });
}

int b200sm_get_localize_stats(b200sm_t s, b200sm_localize_stats* out) {
  if (!s || !out) return B200REG_ERR_ARG;
  out->n_map = s->n_prior;
  out->n_cut = s->have_cut ? s->n_cut : 0;
  out->n_target = s->n_cut_target;
  out->cut_centre[0] = s->cut_centre[0];
  out->cut_centre[1] = s->cut_centre[1];
  out->dist_from_centre = s->dist_from_centre;
  out->n_cuts = s->n_cuts;
  out->cut_pending = s->cut_pending ? 1 : 0;
  return B200REG_OK;
}

int b200sm_get_cut(b200sm_t s, float* out_xyzi, size_t capacity, size_t* n) {
  if (!s) return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() { return read_back(s, s->cut.ptr, s->have_cut ? s->n_cut : 0, out_xyzi, capacity, n); });
}

}  // extern "C"

// ---- place recognition (b200sm_search_loop_place): Scan Context descriptors of the submaps, built lazily on the device,
// and a search over them that does not look at the poses (csrc/scan_context.hpp, csrc/place_recognition.cu)
namespace {

size_t sc_bins(const ScParams& p) { return (size_t)p.num_rings * p.num_sectors; }

void sc_drop(b200sm_t s) {
  s->sc_built = 0;
  s->sc_tables_ready = false;
}

// Descriptors for every submap that has none yet, in one K13a launch and its finishing pass. Stream-ordered: the caller
// synchronises before it reads anything back.
int sc_ensure(b200sm_t s) {
  const ScParams& p = s->sc;
  const size_t n_sub = s->submaps.size(), nb = sc_bins(p);
  if (!s->sc_tables_ready) {
    std::vector<double> ring_b, sector_u;
    sc_tables(p, ring_b, sector_u);
    ring_b.insert(ring_b.end(), sector_u.begin(), sector_u.end());
    s->sc_tables.ensure(ring_b.size());
    B200_CUDA(cudaMemcpyAsync(s->sc_tables.ptr, ring_b.data(), ring_b.size() * sizeof(double), cudaMemcpyHostToDevice, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));  // the host vector goes out of scope
    s->sc_tables_ready = true;
  }
  if (s->sc_built == n_sub) return (int)B200REG_OK;
  if (n_sub > s->sc_cap || s->sc_keys.cap < n_sub * nb || s->sc_norms.cap < n_sub * (size_t)p.num_sectors) {
    // grow, keeping the descriptors already built (DeviceBuffer::ensure does not preserve contents)
    const size_t cap = std::max(n_sub + 64, s->sc_cap + s->sc_cap / 2);
    DeviceBuffer<uint32_t> keys;
    DeviceBuffer<double> norms;
    keys.ensure(cap * nb);
    norms.ensure(cap * (size_t)p.num_sectors);
    if (s->sc_built) {
      B200_CUDA(cudaMemcpyAsync(keys.ptr, s->sc_keys.ptr, s->sc_built * nb * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s->stream));
      B200_CUDA(cudaMemcpyAsync(norms.ptr, s->sc_norms.ptr, s->sc_built * p.num_sectors * sizeof(double), cudaMemcpyDeviceToDevice,
                                s->stream));
    }
    B200_CUDA(cudaStreamSynchronize(s->stream));
    std::swap(keys.ptr, s->sc_keys.ptr);
    std::swap(keys.cap, s->sc_keys.cap);
    std::swap(norms.ptr, s->sc_norms.ptr);
    std::swap(norms.cap, s->sc_norms.cap);
    s->sc_cap = cap;
  }
  // an empty submap owns no tile: its descriptor is all zero
  SubmapTiles t;
  const int rc = submap_tiles(s, s->sc_built, SC_BUILD_TILE, true, "scan_context: a submap of 2^32 points or more",
                              "scan_context: too many points for one launch", &t);
  if (rc != B200REG_OK) return rc;
  std::vector<ScBuildEntry> table;
  for (size_t r = 0; r < t.ids.size(); r++) {
    const Submap& sub = *s->submaps[t.ids[r]];
    table.push_back({sub.cloud, (unsigned)sub.n, t.first_tile[r], (unsigned)t.ids[r], 0u});
  }
  const size_t first = s->sc_built, count = n_sub - s->sc_built;
  B200_CUDA(cudaMemsetAsync(s->sc_keys.ptr + first * nb, 0, count * nb * sizeof(uint32_t), s->stream));
  if (!table.empty()) {
    s->sc_build_table.ensure(table.size());
    B200_CUDA(cudaMemcpyAsync(s->sc_build_table.ptr, table.data(), table.size() * sizeof(ScBuildEntry), cudaMemcpyHostToDevice,
                              s->stream));
    sc_build_launch(s->sc_build_table.ptr, (int)table.size(), (unsigned)t.tiles, s->sc_keys.ptr, s->sc_tables.ptr, p.num_rings,
                    p.num_sectors, (float)p.lidar_height, s->stream);
    s->launches += 1;
  }
  sc_finish_launch(s->sc_keys.ptr, s->sc_norms.ptr, first, count, p.num_rings, p.num_sectors, s->stream);
  s->launches += 1;
  B200_CUDA(cudaStreamSynchronize(s->stream));  // the table's host copy goes out of scope
  s->sc_built = n_sub;
  return (int)B200REG_OK;
}

const float* sc_desc(b200sm_t s) { return reinterpret_cast<const float*>(s->sc_keys.ptr); }

}  // namespace

extern "C" {

int b200sm_set_scan_context_params(b200sm_t s, const b200sm_scan_context_params* p) {
  if (!s) return B200REG_ERR_ARG;
  ScParams q;
  if (p) {
    q.num_rings = p->num_rings;
    q.num_sectors = p->num_sectors;
    q.max_radius = p->max_radius;
    q.lidar_height = p->lidar_height;
  }
  if (!sc_params_valid(q)) return sm_fail(s, B200REG_ERR_ARG, "set_scan_context_params: a parameter out of range");
  s->sc = q;
  sc_drop(s);
  return B200REG_OK;
}

int b200sm_get_scan_context(b200sm_t s, size_t index, float* out, size_t capacity) {
  if (!s || !out || index >= s->submaps.size() || capacity < sc_bins(s->sc)) return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() {
    const int rc = sc_ensure(s);
    if (rc != B200REG_OK) return rc;
    const size_t nb = sc_bins(s->sc);
    B200_CUDA(cudaMemcpyAsync(out, sc_desc(s) + index * nb, nb * sizeof(float), cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    return (int)B200REG_OK;
  });
}

int b200sm_search_loop_place(b200sm_t s, b200reg_t reg, float voxel_leaf_size, double threshold_loop_closure_score,
                             double distance_loop_closure, int search_submap_num, double sc_threshold, int top_k,
                             b200sm_place_result* out, size_t capacity, size_t* n_out, size_t* n_scored) {
  if (!s || !reg || !n_out || !(voxel_leaf_size > 0) || search_submap_num < 0 || top_k < 1 || top_k > SC_MAX_TOP_K ||
      !std::isfinite(sc_threshold) || (!out && capacity))
    return B200REG_ERR_ARG;
  return sm_guarded(s, [&]() {
    *n_out = 0;
    if (n_scored) *n_scored = 0;
    const int n_sub = (int)s->submaps.size();
    s->place_distances.assign(n_sub, std::nan(""));
    s->place_shifts.assign(n_sub, -1);
    if (n_sub < 2) return (int)B200REG_OK;
    int rc = sc_ensure(s);
    if (rc != B200REG_OK) return rc;
    const ScParams& p = s->sc;
    const Submap& latest = *s->submaps[n_sub - 1];
    std::vector<int> ids;  // the reference's first gate (gbs.cpp:193), strict; no position gate
    for (int i = 0; i < n_sub - 1; i++)
      if (latest.distance - s->submaps[i]->distance > distance_loop_closure) ids.push_back(i);
    if (n_scored) *n_scored = ids.size();
    if (ids.empty()) return (int)B200REG_OK;
    const size_t m = ids.size();
    s->sc_ids.ensure(m);
    s->sc_dist.ensure(m);
    s->sc_shift.ensure(m);
    B200_CUDA(cudaMemcpyAsync(s->sc_ids.ptr, ids.data(), m * sizeof(int), cudaMemcpyHostToDevice, s->stream));
    sc_search_launch(sc_desc(s), s->sc_norms.ptr, (size_t)(n_sub - 1), s->sc_ids.ptr, (int)m, s->sc_dist.ptr, s->sc_shift.ptr,
                     p.num_rings, p.num_sectors, s->stream);
    s->launches += 1;
    std::vector<double> dist(m);
    std::vector<int> shift(m);
    B200_CUDA(cudaMemcpyAsync(dist.data(), s->sc_dist.ptr, m * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaMemcpyAsync(shift.data(), s->sc_shift.ptr, m * sizeof(int), cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    for (size_t r = 0; r < m; r++) {
      s->place_distances[ids[r]] = dist[r];
      s->place_shifts[ids[r]] = shift[r];
    }
    const std::vector<int> order = sc_rank(dist.data(), ids.data(), m, sc_threshold);
    const size_t k = std::min({order.size(), (size_t)top_k, capacity});
    bool have_source = false;
    for (size_t q = 0; q < k; q++) {
      const size_t r = (size_t)order[q];
      const int id = ids[r];
      const Submap& cand = *s->submaps[id];
      if (!have_source) {
        rc = loop_set_source(s, reg, latest);
        if (rc != B200REG_OK) return rc;
        have_source = true;
      }
      b200sm_place_result* row = out + q;
      std::memset(row, 0, sizeof(*row));
      row->sc_distance = dist[r];
      row->shift = shift[r];
      sc_guess(cand.pose, latest.pose, shift[r], p.num_sectors, row->guess);
      const double dx = latest.pose[3] - cand.pose[3], dy = latest.pose[7] - cand.pose[7], dz = latest.pose[11] - cand.pose[11];
      const LoopCandidate lc{id, std::sqrt(dx * dx + dy * dy + dz * dz)};  // loop_candidates' min_dist
      rc = loop_evaluate(s, reg, lc, latest, 0, n_sub, voxel_leaf_size, threshold_loop_closure_score, search_submap_num, &row->loop,
                         row->guess);
      if (rc != B200REG_OK) return rc;
      *n_out += 1;
    }
    return (int)B200REG_OK;
  });
}

int b200sm_get_place_scores(b200sm_t s, size_t capacity, size_t* n, double* distances, int* shifts) {
  if (!s || !n) return B200REG_ERR_ARG;
  const size_t total = s->place_distances.size(), m = std::min(capacity, total);
  *n = total;
  if (distances && m) std::memcpy(distances, s->place_distances.data(), m * sizeof(double));
  if (shifts && m) std::memcpy(shifts, s->place_shifts.data(), m * sizeof(int));
  return B200REG_OK;
}

}  // extern "C"

// ---- merging a second session (b200sm_merge_session): K16 scores and selection on the device (place_recognition.cu),
// verification by loop_evaluate, consistency, placement and joint adjustment on the host (csrc/session_merge.hpp)
namespace {

b200sm_merge_params merge_defaults() {
  b200sm_merge_params p;
  p.sc_threshold = 0.4;
  p.top_k = 3;
  p.max_verifications = 64;
  p.voxel_leaf_size = 0.3f;
  p.threshold_loop_closure_score = 1.0;
  p.search_submap_num = 1;
  p.consistency_translation = 1.5;
  p.consistency_rotation = 0.1;
  p.consistency_drift_translation = 0.02;
  p.consistency_drift_rotation = 0.003;
  p.min_inliers = 2;
  p.num_adjacent_pose_cnstraints = 5;
  p.max_iterations = 10;
  return p;
}

bool merge_params_valid(const b200sm_merge_params& p) {
  auto tol = [](double v) { return std::isfinite(v) && v >= 0; };
  return std::isfinite(p.sc_threshold) && p.top_k >= 1 && p.top_k <= MERGE_MAX_TOP_K && p.max_verifications >= 1 &&
         p.max_verifications <= MERGE_MAX_VERIFICATIONS && std::isfinite(p.voxel_leaf_size) && p.voxel_leaf_size > 0 &&
         !std::isnan(p.threshold_loop_closure_score) && p.search_submap_num >= 0 && tol(p.consistency_translation) &&
         tol(p.consistency_rotation) && tol(p.consistency_drift_translation) && tol(p.consistency_drift_rotation) &&
         p.min_inliers >= 1 && p.num_adjacent_pose_cnstraints >= 1 && p.max_iterations >= 0;
}

bool same_sc(const ScParams& a, const ScParams& b) {
  return a.num_rings == b.num_rings && a.num_sectors == b.num_sectors && a.max_radius == b.max_radius && a.lidar_height == b.lidar_height;
}

// the segment of submap a: [lo, hi)
void segment_of(b200sm_t s, int a, int* lo, int* hi) {
  size_t k = 0;
  while (k + 1 < s->seg_first.size() && s->seg_first[k + 1] <= a) k++;
  *lo = s->seg_first[k];
  *hi = k + 1 < s->seg_first.size() ? s->seg_first[k + 1] : (int)s->submaps.size();
}

}  // namespace

extern "C" {

int b200sm_merge_session(b200sm_t dst, b200sm_t src, b200reg_t reg, const b200sm_merge_params* params,
                         const b200sm_loop_edge* loop_edges, int n_loop_edges, b200sm_merge_row* rows, size_t capacity,
                         size_t* n_rows, double* poses_out, b200sm_merge_result* result) {
  if (!dst || !src || !reg || !n_rows || !result || (!rows && capacity) || n_loop_edges < 0 || (n_loop_edges && !loop_edges))
    return dst ? sm_fail(dst, B200REG_ERR_ARG, "merge_session: a NULL argument") : B200REG_ERR_ARG;
  if (dst == src) return sm_fail(dst, B200REG_ERR_ARG, "merge_session: dst and src are the same session");
  if (dst->device != src->device) return sm_fail(dst, B200REG_ERR_ARG, "merge_session: the sessions are on different devices");
  if (!same_sc(dst->sc, src->sc)) return sm_fail(dst, B200REG_ERR_ARG, "merge_session: different Scan Context parameters");
  const b200sm_merge_params p = params ? *params : merge_defaults();
  if (!merge_params_valid(p)) return sm_fail(dst, B200REG_ERR_ARG, "merge_session: a parameter out of range");
  const size_t nA = dst->submaps.size(), nB = src->submaps.size();
  if (nA == 0 || nB == 0) return sm_fail(dst, B200REG_ERR_ARG, "merge_session: an empty session");
  if ((unsigned long long)nA * nB > MERGE_MAX_PAIRS) return sm_fail(dst, B200REG_ERR_ARG, "merge_session: more than 2^28 pairs");
  const int n_all = (int)(nA + nB);
  if (const int rc = check_loop_edges(dst, loop_edges, n_loop_edges, n_all, "merge_session"); rc != B200REG_OK) return rc;
  return sm_guarded(dst, [&]() {
    *n_rows = 0;
    std::memset(result, 0, sizeof(*result));
    result->first_submap = -1;
    const ScParams& sp = dst->sc;
    // descriptors of both sessions from their lazy caches; src's stream is done with them (and its clouds) afterwards
    int rc = sc_ensure(dst);
    if (rc == B200REG_OK) {
      rc = sc_ensure(src);
      if (rc != B200REG_OK) dst->err = "merge_session: src: " + src->err;
    }
    if (rc != B200REG_OK) return rc;
    B200_CUDA(cudaStreamSynchronize(src->stream));
    // (1) K16: the whole matrix, (2) the per-row selection
    const size_t pairs = nA * nB;
    dst->merge_dist.ensure(pairs);
    dst->merge_shift.ensure(pairs);
    dst->merge_nq = nB;
    dst->merge_nc = nA;
    result->query_tile = merge_query_tile(sp.num_rings, sp.num_sectors);
    result->pairs_scored = pairs;
    merge_scores_launch(sc_desc(src), src->sc_norms.ptr, (int)nB, sc_desc(dst), dst->sc_norms.ptr, (int)nA, dst->merge_dist.ptr,
                        dst->merge_shift.ptr, sp.num_rings, sp.num_sectors, dst->stream);
    const size_t n_sel = nB * (size_t)p.top_k;
    dst->merge_sel_a.ensure(n_sel);
    dst->merge_sel_d.ensure(n_sel);
    dst->merge_sel_s.ensure(n_sel);
    merge_select_launch(dst->merge_dist.ptr, dst->merge_shift.ptr, (int)nB, (int)nA, p.sc_threshold, p.top_k, dst->merge_sel_a.ptr,
                        dst->merge_sel_d.ptr, dst->merge_sel_s.ptr, dst->stream);
    dst->launches += 2;
    std::vector<int> sel_a(n_sel), sel_s(n_sel);
    std::vector<double> sel_d(n_sel);
    B200_CUDA(cudaMemcpyAsync(sel_a.data(), dst->merge_sel_a.ptr, n_sel * sizeof(int), cudaMemcpyDeviceToHost, dst->stream));
    B200_CUDA(cudaMemcpyAsync(sel_d.data(), dst->merge_sel_d.ptr, n_sel * sizeof(double), cudaMemcpyDeviceToHost, dst->stream));
    B200_CUDA(cudaMemcpyAsync(sel_s.data(), dst->merge_sel_s.ptr, n_sel * sizeof(int), cudaMemcpyDeviceToHost, dst->stream));
    B200_CUDA(cudaStreamSynchronize(dst->stream));
    std::vector<MergeCandidate> cand;
    for (size_t b = 0; b < nB; b++)
      for (int r = 0; r < p.top_k; r++) {
        const size_t o = b * p.top_k + r;
        if (sel_a[o] < 0) break;
        cand.push_back({sel_d[o], (int)b, sel_a[o], sel_s[o]});
      }
    result->candidates = (int)cand.size();
    merge_order(cand, p.max_verifications);
    // (3) verification
    std::vector<b200sm_merge_row> all(cand.size());
    std::vector<MergeEdge> acc;
    std::vector<int> acc_row;
    int have_b = -1;
    for (size_t q = 0; q < cand.size(); q++) {
      const MergeCandidate& c = cand[q];
      const Submap& A = *dst->submaps[c.a];
      const Submap& B = *src->submaps[c.b];
      b200sm_merge_row& row = all[q];
      std::memset(&row, 0, sizeof(row));
      row.src_id = c.b;
      row.inlier = -1;
      row.place.sc_distance = c.D;
      row.place.shift = c.shift;
      sc_guess(A.pose, B.pose, c.shift, sp.num_sectors, row.place.guess);
      int lo, hi;
      segment_of(dst, c.a, &lo, &hi);
      size_t window = 0;
      for (int idx = std::max(lo, c.a - p.search_submap_num); idx < std::min(hi, c.a + p.search_submap_num + 1); idx++)
        window += dst->submaps[idx]->n;
      if (B.n == 0 || window == 0) {  // nothing to register (an empty src submap, or a window of empty submaps): not accepted
        row.place.loop.is_candidate = 1;
        row.place.loop.id_min = c.a;
        row.place.loop.n_source = B.n;
        row.place.loop.fitness = HUGE_VAL;
        result->verified += 1;
        continue;
      }
      if (c.b != have_b) {
        rc = loop_set_source(dst, reg, B);
        if (rc != B200REG_OK) return rc;
        have_b = c.b;
      }
      rc = loop_evaluate(dst, reg, LoopCandidate{c.a, 0.0}, B, lo, hi, p.voxel_leaf_size, p.threshold_loop_closure_score,
                         p.search_submap_num, &row.place.loop, row.place.guess);
      if (rc != B200REG_OK) return rc;
      double F[16], FP[16];
      merge_final_rowmajor(row.place.loop.final_T, F);
      merge_mul16(F, B.pose, FP);
      const double dx = A.pose[3] - FP[3], dy = A.pose[7] - FP[7], dz = A.pose[11] - FP[11];
      row.place.loop.min_dist = std::sqrt(dx * dx + dy * dy + dz * dz);
      result->verified += 1;
      if (row.place.loop.accepted) {
        MergeEdge e;
        e.a = c.a;
        e.b = c.b;
        e.fitness = row.place.loop.fitness;
        e.da = A.distance;
        e.db = B.distance;
        std::memcpy(e.Pa, A.pose, sizeof(e.Pa));
        std::memcpy(e.Pb, B.pose, sizeof(e.Pb));
        col_to_row(row.place.loop.relative_pose, e.Z);
        acc.push_back(e);
        acc_row.push_back((int)q);
      }
    }
    result->accepted = (int)acc.size();
    // (4) the consistent set
    const MergeTolerance tol{p.consistency_translation, p.consistency_rotation, p.consistency_drift_translation,
                             p.consistency_drift_rotation};
    const std::vector<int> in = merge_inliers(acc, tol);
    result->inliers = (int)in.size();
    for (size_t k = 0; k < in.size(); k++) all[acc_row[in[k]]].inlier = (int)k;
    *n_rows = std::min(all.size(), capacity);
    if (*n_rows) std::memcpy(rows, all.data(), *n_rows * sizeof(b200sm_merge_row));
    if ((int)in.size() < p.min_inliers) return (int)B200REG_OK;
    // (5) placement and the joint adjustment
    double T[16];
    merge_final_rowmajor(all[acc_row[in[0]]].place.loop.final_T, T);
    std::vector<double> Xb(16 * nB);
    for (size_t b = 0; b < nB; b++) merge_place(T, src->submaps[b]->pose, Xb.data() + 16 * b);
    std::vector<pg::Iso> X(n_all);
    for (size_t i = 0; i < nA; i++) X[i] = pg::iso_from_rowmajor16(dst->submaps[i]->pose);
    for (size_t b = 0; b < nB; b++) X[nA + b] = pg::iso_from_rowmajor16(Xb.data() + 16 * b);
    std::vector<int> segs = dst->seg_first;  // dst's segments, then src's (src may itself be a merged map)
    for (int f : src->seg_first) segs.push_back((int)nA + f);
    const int n_loops = n_loop_edges + (int)in.size();
    std::vector<int> ids;
    std::vector<pg::Iso> rel;
    append_loop_edges(loop_edges, n_loop_edges, ids, rel);
    for (size_t k = 0; k < in.size(); k++) {
      const MergeEdge& e = acc[in[k]];
      ids.push_back(e.a);
      ids.push_back((int)nA + e.b);
      rel.push_back(pg::iso_from_rowmajor16(e.Z));
    }
    const std::vector<pg::Edge> edges = pg::build_edges(X, p.num_adjacent_pose_cnstraints, segs, ids.data(), rel.data(), n_loops);
    const pg::LmResult r = pg::optimize(X, edges, p.max_iterations);
    // (6) append src as a new segment
    const double d_last = dst->submaps.back()->distance;
    std::vector<std::unique_ptr<Submap>> added;
    for (size_t b = 0; b < nB; b++) {
      const Submap& B = *src->submaps[b];
      added.push_back(new_submap(dst->arena, B.cloud, B.n, Xb.data() + 16 * b, d_last + B.distance, dst->stream));
    }
    B200_CUDA(cudaStreamSynchronize(dst->stream));
    for (auto& sub : added) dst->submaps.push_back(std::move(sub));
    dst->seg_first = segs;
    dst->latest_distance = dst->submaps.back()->distance;
    if (poses_out)
      for (int i = 0; i < n_all; i++) pg::iso_to_colmajor16(X[i], poses_out + 16 * (size_t)i);
    result->merged = 1;
    result->first_submap = (int)nA;
    row_to_col(T, result->T);
    result->adjust.chi2_initial = r.chi2_initial;
    result->adjust.chi2_final = r.chi2_final;
    result->adjust.iterations = r.iterations;
    result->adjust.trials = r.trials;
    result->adjust.n_vertices = n_all;
    result->adjust.n_edges = (int)edges.size();
    return (int)B200REG_OK;
  });
}

int b200sm_get_merge_scores(b200sm_t dst, size_t capacity, size_t* n_query, size_t* n_cand, double* distances, int* shifts) {
  if (!dst || !n_query || !n_cand) return B200REG_ERR_ARG;
  return sm_guarded(dst, [&]() {
    *n_query = dst->merge_nq;
    *n_cand = dst->merge_nc;
    const size_t m = std::min(capacity, dst->merge_nq * dst->merge_nc);
    if (distances && m) B200_CUDA(cudaMemcpyAsync(distances, dst->merge_dist.ptr, m * sizeof(double), cudaMemcpyDeviceToHost, dst->stream));
    if (shifts && m) B200_CUDA(cudaMemcpyAsync(shifts, dst->merge_shift.ptr, m * sizeof(int), cudaMemcpyDeviceToHost, dst->stream));
    B200_CUDA(cudaStreamSynchronize(dst->stream));
    return (int)B200REG_OK;
  });
}

int b200sm_get_segments(b200sm_t s, size_t* first, size_t capacity, size_t* n) {
  if (!s || !n || (!first && capacity)) return B200REG_ERR_ARG;
  const size_t total = s->submaps.empty() ? 0 : s->seg_first.size();
  *n = total;
  for (size_t k = 0; k < std::min(capacity, total); k++) first[k] = (size_t)s->seg_first[k];
  return B200REG_OK;
}

}  // extern "C"

// ---- saving and loading a session (csrc/session_io.hpp) ----
namespace {

constexpr size_t SIO_PIECE_BYTES = (size_t)16 << 20;  // largest device-to-host copy of a submap body: 1 Mi points

int sio_io_fail(b200sm_t s, const std::string& why) {
  s->err = why;
  return (int)B200REG_ERR_IO;
}

bool sio_make_dir(const std::string& d) {
  struct stat st;
  if (mkdir(d.c_str(), 0777) == 0) return true;
  return errno == EEXIST && stat(d.c_str(), &st) == 0 && S_ISDIR(st.st_mode);
}

// Every submap file: the binary PCD header, then the submap's float4 rows as they are on the device, in pieces of at most
// SIO_PIECE_BYTES through write_staged. An empty submap is a header alone.
int sio_write_submaps(b200sm_t s, const std::string& sub_dir, unsigned long long* bytes) {
  struct Piece {
    size_t sub, first, count;  // points
  };
  const size_t per_piece = SIO_PIECE_BYTES / sizeof(float4);
  std::vector<Piece> pieces;
  size_t most = 1;
  for (size_t i = 0; i < s->submaps.size(); i++) {
    const size_t n = s->submaps[i]->n;
    size_t first = 0;
    do {
      const size_t c = std::min(per_piece, n - first);
      pieces.push_back({i, first, c});
      most = std::max(most, c * sizeof(float4));
      first += c;
    } while (first < n);
  }
  FILE* fp = nullptr;
  std::string path;
  auto enqueue = [&](size_t p, char* buf) {
    const Piece& q = pieces[p];
    if (q.count)
      B200_CUDA(cudaMemcpyAsync(buf, s->submaps[q.sub]->cloud + q.first, q.count * sizeof(float4), cudaMemcpyDeviceToHost, s->stream));
  };
  auto write = [&](size_t p, const char* buf) {
    const Piece& q = pieces[p];
    const size_t n = s->submaps[q.sub]->n;
    if (q.first == 0) {
      path = sub_dir + "/" + sio::submap_name(q.sub);
      fp = std::fopen(path.c_str(), "wb");
      if (!fp) return sio_io_fail(s, "save_session: cannot create " + path + ": " + std::strerror(errno));
      const std::string header = sio::pcd_binary_header(n);
      if (std::fwrite(header.data(), 1, header.size(), fp) != header.size())
        return sio_io_fail(s, "save_session: writing " + path + ": " + std::strerror(errno));
      *bytes += header.size();
    }
    const size_t b = q.count * sizeof(float4);
    if (b && std::fwrite(buf, 1, b, fp) != b) return sio_io_fail(s, "save_session: writing " + path + ": " + std::strerror(errno));
    *bytes += b;
    if (q.first + q.count == n) {
      const int rc = std::fclose(fp);
      fp = nullptr;
      if (rc != 0) return sio_io_fail(s, "save_session: writing " + path + ": " + std::strerror(errno));
    }
    return (int)B200REG_OK;
  };
  return write_staged(s, pieces.size(), most, fp, enqueue, write);
}

bool sio_session_empty(b200sm_t s) { return s->submaps.empty() && !s->d_scan && !s->initial_cloud_received && !s->loaded; }

}  // namespace

extern "C" {

int b200sm_save_session(b200sm_t s, const char* dir, int num_adjacent_pose_cnstraints, const b200sm_loop_edge* loop_edges,
                        int n_loop_edges, const double* adjusted_poses_colmajor16, b200sm_session_io_info* info) {
  if (!s || !dir || !*dir || num_adjacent_pose_cnstraints < 1 || n_loop_edges < 0 || (n_loop_edges && !loop_edges))
    return s ? sm_fail(s, B200REG_ERR_ARG, "save_session: a NULL or empty argument, num_adjacent_pose_cnstraints < 1 or n_loop_edges < 0")
             : B200REG_ERR_ARG;
  const size_t n = s->submaps.size();
  if (n == 0) return sm_fail(s, B200REG_ERR_ARG, "save_session: the session has no submaps");
  if (const int rc = check_loop_edges(s, loop_edges, n_loop_edges, (int)n, "save_session"); rc != B200REG_OK) return rc;
  if (!finite_poses(adjusted_poses_colmajor16, n)) return sm_fail(s, B200REG_ERR_ARG, "save_session: non-finite adjusted pose");
  return sm_guarded(s, [&]() {
    sio::Manifest m;
    m.sc = s->sc;
    m.seg_first = s->seg_first;
    m.points.resize(n);
    m.distance.resize(n);
    m.pose.resize(16 * n);
    for (size_t i = 0; i < n; i++) {
      const Submap& sub = *s->submaps[i];
      m.points[i] = sub.n;
      m.distance[i] = sub.distance;
      row_to_col(sub.pose, m.pose.data() + 16 * i);
    }
    m.k = num_adjacent_pose_cnstraints;
    m.loops.resize(n_loop_edges);
    for (int l = 0; l < n_loop_edges; l++) {
      m.loops[l].from = loop_edges[l].from;
      m.loops[l].to = loop_edges[l].to;
      std::memcpy(m.loops[l].rel, loop_edges[l].relative_pose, sizeof(m.loops[l].rel));
    }
    m.adjusted = adjusted_poses_colmajor16 != nullptr;
    if (m.adjusted) m.adjusted_pose.assign(adjusted_poses_colmajor16, adjusted_poses_colmajor16 + 16 * n);
    const std::string d = dir, sub_dir = d + "/submaps", manifest = d + "/session.txt", tmp = manifest + ".tmp";
    if (!sio_make_dir(d) || !sio_make_dir(sub_dir))
      return sio_io_fail(s, "save_session: cannot create " + sub_dir + ": " + std::strerror(errno));
    // no manifest may name a submap file while it is being rewritten
    if (std::remove(manifest.c_str()) != 0 && errno != ENOENT)
      return sio_io_fail(s, "save_session: cannot remove " + manifest + ": " + std::strerror(errno));
    unsigned long long bytes = 0;
    int rc = sio_write_submaps(s, sub_dir, &bytes);
    if (rc != B200REG_OK) return rc;
    const std::string g2o = sio::write_g2o(m), text = sio::write_manifest(m);
    if (write_file(d + "/pose_graph.g2o", g2o))
      return sio_io_fail(s, "save_session: writing " + d + "/pose_graph.g2o: " + std::strerror(errno));
    if (write_file(tmp, text)) {
      const int e = errno;
      std::remove(tmp.c_str());
      return sio_io_fail(s, "save_session: writing " + tmp + ": " + std::strerror(e));
    }
    if (std::rename(tmp.c_str(), manifest.c_str()) != 0)
      return sio_io_fail(s, "save_session: renaming " + tmp + ": " + std::strerror(errno));
    bytes += g2o.size() + text.size();
    if (info) {
      std::size_t pts = 0;
      for (unsigned long long p : m.points) pts += (size_t)p;
      info->n_submaps = n;
      info->n_segments = m.seg_first.size();
      info->n_points = pts;
      info->n_loop_edges = n_loop_edges;
      info->num_adjacent_pose_cnstraints = m.k;
      info->adjusted = m.adjusted ? 1 : 0;
      info->n_bytes = bytes;
    }
    return (int)B200REG_OK;
  });
}

int b200sm_load_session(b200sm_t s, const char* dir, b200sm_session_io_info* info) {
  if (!s || !dir || !*dir) return s ? sm_fail(s, B200REG_ERR_ARG, "load_session: a NULL or empty directory") : B200REG_ERR_ARG;
  if (!sio_session_empty(s))
    return sm_fail(s, B200REG_ERR_ARG, "load_session: the session is not empty (it holds submaps or has received frames)");
  return sm_guarded(s, [&]() {
    const std::string d = dir, path = d + "/session.txt";
    // (1) the whole manifest, parsed before anything is allocated
    std::string text;
    {
      FILE* fp = std::fopen(path.c_str(), "rb");
      if (!fp) return sio_io_fail(s, "load_session: cannot open " + path + ": " + std::strerror(errno));
      char buf[1 << 16];
      size_t got;
      while ((got = std::fread(buf, 1, sizeof buf, fp)) > 0) text.append(buf, got);
      const bool bad = std::ferror(fp) != 0;
      std::fclose(fp);
      if (bad) return sio_io_fail(s, "load_session: reading " + path);
    }
    sio::Manifest m;
    std::string why;
    if (!sio::parse_manifest(text, m, why)) return sm_fail(s, B200REG_ERR_FORMAT, ("load_session: " + path + " " + why).c_str());
    // (2) every submap file through the PCD reader (a binary body is unpacked on the device by the upload kernel), its
    // rows copied device to device into an arena of the load's own; the session takes it over only when all are in
    const size_t n = m.n();
    SubmapArena arena;
    std::vector<std::unique_ptr<Submap>> subs;
    DeviceBuffer<float4> rows;
    unsigned long long bytes = text.size(), pts = 0;
    for (size_t i = 0; i < n; i++) {
      const std::string file = d + "/submaps/" + sio::submap_name(i);
      size_t got = 0;
      const int before = s->pcd_loader.launches;
      const int rc = s->pcd_loader.load(file.c_str(), rows, &got, why, s->stream);
      s->launches += s->pcd_loader.launches - before;
      if (rc != B200REG_OK) {
        s->err = "load_session: " + file + ": " + why;
        return rc;
      }
      if (got != m.points[i])
        return sm_fail(s, B200REG_ERR_FORMAT, ("load_session: " + file + ": POINTS " + std::to_string(got) + ", the manifest says " +
                                               std::to_string(m.points[i])).c_str());
      struct stat st;
      if (stat(file.c_str(), &st) == 0) bytes += (unsigned long long)st.st_size;
      double pose[16];
      col_to_row(m.pose.data() + 16 * i, pose);
      // stream-ordered before the next file's upload into `rows`
      subs.push_back(new_submap(arena, rows.ptr, got, pose, m.distance[i], s->stream));
      pts += got;
    }
    B200_CUDA(cudaStreamSynchronize(s->stream));
    // (3) what b200sm_import_submap of every submap in order gives, then the segments and the Scan Context parameters
    std::swap(s->arena.chunks, arena.chunks);
    s->arena.used = arena.used;
    s->arena.cap = arena.cap;
    s->submaps = std::move(subs);
    s->seg_first = m.seg_first;
    s->latest_distance = s->submaps.back()->distance;
    s->sc = m.sc;
    sc_drop(s);
    s->loaded = true;
    s->graph_loops = m.loops;
    s->graph_k = m.k;
    s->graph_poses = m.adjusted_pose;
    if (info) {
      info->n_submaps = n;
      info->n_segments = m.seg_first.size();
      info->n_points = (size_t)pts;
      info->n_loop_edges = (int)m.loops.size();
      info->num_adjacent_pose_cnstraints = m.k;
      info->adjusted = m.adjusted ? 1 : 0;
      info->n_bytes = bytes;
    }
    return (int)B200REG_OK;
  });
}

int b200sm_get_session_graph(b200sm_t s, b200sm_loop_edge* loop_edges, size_t capacity, size_t* n_loop_edges,
                             double* adjusted_poses_colmajor16, int* num_adjacent_pose_cnstraints) {
  if (!s || !n_loop_edges || (!loop_edges && capacity)) return s ? sm_fail(s, B200REG_ERR_ARG, "get_session_graph: a NULL argument") : B200REG_ERR_ARG;
  if (!s->loaded) return sm_fail(s, B200REG_ERR_ARG, "get_session_graph: the session was not loaded by b200sm_load_session");
  *n_loop_edges = s->graph_loops.size();
  for (size_t l = 0; l < std::min(capacity, s->graph_loops.size()); l++) {
    loop_edges[l].from = s->graph_loops[l].from;
    loop_edges[l].to = s->graph_loops[l].to;
    std::memcpy(loop_edges[l].relative_pose, s->graph_loops[l].rel, sizeof(loop_edges[l].relative_pose));
  }
  if (adjusted_poses_colmajor16 && !s->graph_poses.empty())
    std::memcpy(adjusted_poses_colmajor16, s->graph_poses.data(), s->graph_poses.size() * sizeof(double));
  if (num_adjacent_pose_cnstraints) *num_adjacent_pose_cnstraints = s->graph_k;
  return B200REG_OK;
}

}  // extern "C"

// ---- the map products' shared host steps: the prologue over the submaps, the bounds pass, the box, the rank pass and the
// compacted clouds' read-backs ----
namespace {

// "<what>: the sensor origin of submap k lies beyond <beyond>"
int origin_refused(b200sm_t s, const char* what, size_t k, const char* beyond) {
  s->err = std::string(what) + ": the sensor origin of submap " + std::to_string(k) + " lies beyond " + beyond;
  return (int)B200REG_ERR_ARG;
}

// A map build's prologue: refuses a session without submaps and non-finite poses, then before_tiles' message when it
// returns one, and lays out the tiles of the submaps with points (`tile` points per block) into *t. Then every submap in
// order gets a zeroed entry with its float pose, and its cloud, size and first tile when it has points; per_submap(k, e)
// adds the build's own fields or refuses (an error code, s->err set), and the entries of the submaps with points are
// appended to *table. `what` prefixes the messages.
template <class Entry, class PerSubmap>
int map_prologue(b200sm_t s, const char* what, const double* poses_colmajor16, size_t tile, const char* (*before_tiles)(b200sm_t),
                 SubmapTiles* t, std::vector<Entry>* table, PerSubmap&& per_submap) {
  const size_t n_sub = s->submaps.size();
  const std::string w = std::string(what) + ": ";
  if (n_sub == 0) return sm_fail(s, B200REG_ERR_ARG, (w + "the session has no submaps").c_str());
  if (!finite_poses(poses_colmajor16, n_sub)) return sm_fail(s, B200REG_ERR_ARG, (w + "a non-finite pose entry").c_str());
  if (const char* why = before_tiles ? before_tiles(s) : nullptr) return sm_fail(s, B200REG_ERR_ARG, (w + why).c_str());
  const int rc = submap_tiles(s, 0, tile, true, (w + "a submap of 2^32 points or more").c_str(),
                              (w + "too many points for one launch").c_str(), t);
  if (rc != B200REG_OK) return rc;
  for (size_t k = 0; k < n_sub; k++) {
    const Submap& sub = *s->submaps[k];
    Entry e;
    std::memset(&e, 0, sizeof(e));
    submap_pose_f(s, k, poses_colmajor16, e.T);
    if (sub.n) {
      e.cloud = sub.cloud;
      e.n = (unsigned)sub.n;
      e.first_tile = t->first_tile[table->size()];
    }
    const int rc = per_submap(k, e);
    if (rc != B200REG_OK) return rc;
    if (sub.n) table->push_back(e);
  }
  return (int)B200REG_OK;
}

// One bounds pass (K14a, K15a, K19a) over a build's table, D = 2 or 3 axes: zeroes n_counters counters, uploads the table
// and its bounds (2 D ints per entry: the lower corner, then the upper), runs `launch` when there are entries, reads back
// the bounds and the first k counters into ctr, synchronises once, and reduces the entries' bounds per axis into lo[D] /
// hi[D] (INT_MAX / INT_MIN without an entry). `bounds` comes in with the entries' seeds, or empty to start every entry
// empty, and leaves as the launch widened it. Must run inside sm_guarded.
template <int D, class Entry, class Const>
void bounds_pass(b200sm_t s, void (*launch)(const Entry*, int, unsigned, const Const&, int*, unsigned long long*, cudaStream_t),
                 const Const& c, const std::vector<Entry>& table, unsigned long long tiles, DeviceBuffer<Entry>& d_table,
                 std::vector<int>& bounds, int n_counters, unsigned long long* ctr, int k, int* lo, int* hi) {
  MapWorkspace& w = s->work;
  const size_t n = table.size();
  if (bounds.empty()) {
    bounds.resize(2 * D * n);
    for (size_t r = 0; r < n; r++)
      for (int a = 0; a < D; a++) {
        bounds[2 * D * r + a] = INT_MAX;
        bounds[2 * D * r + D + a] = INT_MIN;
      }
  }
  w.counters.ensure(n_counters);
  B200_CUDA(cudaMemsetAsync(w.counters.ptr, 0, n_counters * sizeof(unsigned long long), s->stream));
  if (n) {
    d_table.ensure(n);
    w.bounds.ensure(bounds.size());
    B200_CUDA(cudaMemcpyAsync(d_table.ptr, table.data(), n * sizeof(Entry), cudaMemcpyHostToDevice, s->stream));
    B200_CUDA(cudaMemcpyAsync(w.bounds.ptr, bounds.data(), bounds.size() * sizeof(int), cudaMemcpyHostToDevice, s->stream));
    launch(d_table.ptr, (int)n, (unsigned)tiles, c, w.bounds.ptr, w.counters.ptr, s->stream);
    s->launches += 1;
    B200_CUDA(cudaMemcpyAsync(bounds.data(), w.bounds.ptr, bounds.size() * sizeof(int), cudaMemcpyDeviceToHost, s->stream));
  }
  B200_CUDA(cudaMemcpyAsync(ctr, w.counters.ptr, k * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s->stream));
  B200_CUDA(cudaStreamSynchronize(s->stream));
  for (int a = 0; a < D; a++) {
    lo[a] = INT_MAX;
    hi[a] = INT_MIN;
    for (size_t r = 0; r < n; r++) {
      lo[a] = std::min(lo[a], bounds[2 * D * r + a]);
      hi[a] = std::max(hi[a], bounds[2 * D * r + D + a]);
    }
  }
}

// The W x H grid over the cells lo[2] .. hi[2]; more than 2^28 cells is refused
int grid_or_refuse(b200sm_t s, const char* what, const int* lo, const int* hi, unsigned long long* W, unsigned long long* H) {
  *W = (unsigned long long)((long long)hi[0] - lo[0] + 1);
  *H = (unsigned long long)((long long)hi[1] - lo[1] + 1);
  if (*W * *H <= OG_MAX_CELLS) return (int)B200REG_OK;
  s->err = std::string(what) + ": a grid of " + std::to_string(*W) + " x " + std::to_string(*H) + " cells exceeds 2^28 cells";
  return (int)B200REG_ERR_ARG;
}

// The box over the cells lo[3] .. hi[3] widened by r on every side (the mesh's band; 0 for the others); more than 2^31 - 1
// cells is refused as "<what>: <kind> of X x Y x Z <unit> exceeds 2^31 - 1 <unit>"
int box_or_refuse(b200sm_t s, const char* what, const char* kind, const char* unit, const int* lo, const int* hi, int r, SmBox* box,
                  unsigned long long* cells) {
  if (ms_box(lo, hi, r, box->lo, box->dims, cells)) return (int)B200REG_OK;
  auto width = [&](int a) { return std::to_string((long long)hi[a] - lo[a] + 1 + 2 * r); };
  s->err = std::string(what) + ": " + kind + " of " + width(0) + " x " + width(1) + " x " + width(2) + " " + unit + " exceeds 2^31 - 1 " +
           unit;
  return (int)B200REG_ERR_ARG;
}

// One rank pass (K15b, K19b, K21a): the rank index over n_words words cleared, mark(index) run, the index scanned, and the
// number of marked cells read back after one synchronise. Must run inside sm_guarded.
template <class Mark>
unsigned rank_pass(b200sm_t s, DeviceBuffer<RankWord>& index, unsigned long long n_words, Mark&& mark) {
  RankIndexScratch& scan = s->work.rank_scan;
  index.ensure((size_t)n_words);
  rank_index_clear(index.ptr, (int)n_words, s->stream);
  mark(index.ptr);
  scan.total.ensure(1);
  rank_index_scan_async(index.ptr, (size_t)n_words, scan, scan.total.ptr, s->stream);
  s->launches += 3;
  unsigned marked = 0;
  B200_CUDA(cudaMemcpyAsync(&marked, scan.total.ptr, sizeof(unsigned), cudaMemcpyDeviceToHost, s->stream));
  B200_CUDA(cudaStreamSynchronize(s->stream));
  return marked;
}

// Per-submap offsets into a compacted map of `kept` points, n_sub + 1 of them: a submap with points starts at its first
// tile's offset, an empty one where the next one starts
std::vector<size_t> submap_offsets(const SubmapTiles& t, size_t n_sub, const std::vector<unsigned>& tile_off, unsigned kept) {
  std::vector<size_t> offsets(n_sub + 1, (size_t)kept);
  size_t r = t.ids.size();
  for (size_t k = n_sub; k-- > 0;) {
    if (r > 0 && t.ids[r - 1] == k) offsets[k] = tile_off[t.first_tile[--r]];
    else offsets[k] = offsets[k + 1];
  }
  return offsets;
}

// A compacted cloud of `total` points read back: its size, its per-submap offsets, and at most capacity points
int get_compacted(b200sm_t s, const DeviceBuffer<float4>& pts, size_t total, const std::vector<size_t>& offs, float* out_xyzi,
                  size_t capacity, size_t* n, size_t* offsets) {
  return sm_guarded(s, [&]() {
    if (offsets) std::memcpy(offsets, offs.data(), offs.size() * sizeof(size_t));
    return read_back(s, pts.ptr, total, out_xyzi, capacity, n);
  });
}

// A compacted cloud of `total` points saved as PCL's ASCII PCD; an empty one is refused as "<what>: <empty>"
int save_compacted_pcd(b200sm_t s, const char* what, const char* empty, const DeviceBuffer<float4>& pts, size_t total, const char* path,
                       size_t* n_points, size_t* n_bytes) {
  if (total == 0) return sm_fail(s, B200REG_ERR_ARG, (std::string(what) + ": " + empty).c_str());
  return sm_guarded(s, [&]() { return write_pcd_ascii(s, pts.ptr, total, path, what, n_points, n_bytes); });
}

// Enqueues the read-back of `count` elements of src into dst when dst is given
template <class T>
void get_if(b200sm_t s, void* dst, const T* src, size_t count) {
  if (dst) B200_CUDA(cudaMemcpyAsync(dst, src, count * sizeof(T), cudaMemcpyDeviceToHost, s->stream));
}

}  // namespace

// ---- occupancy grid: free space ray-cast from every submap's sensor origin (csrc/occupancy_grid.hpp, csrc/occupancy.cu) ----
namespace {

// K14b's scratch budget: the hit and free bitmaps of a batch of submaps (2 MB each at 0.05 m and 100 m range). A submap
// whose bitmaps alone exceed it forms a batch of its own.
constexpr unsigned long long OG_SCRATCH_WORDS = 16ull << 20;  // 64 MiB

OgParams og_params_from(const b200sm_occupancy_params* p) {
  OgParams q;
  if (p) {
    q.resolution = p->resolution;
    q.z_min = p->z_min;
    q.z_max = p->z_max;
    q.max_range = p->max_range;
    for (int k = 0; k < 3; k++) q.sensor_origin[k] = p->sensor_origin[k];
    q.occupied_thresh = p->occupied_thresh;
    q.free_thresh = p->free_thresh;
  }
  return q;
}

// nav2 map_server's pair of a trinary image on the device, W x H, top row first (the occupancy grid and the
// traversability map alike); `what` prefixes the error message
int save_map_pair(b200sm_t s, const char* what, const unsigned char* image_dev, unsigned W, unsigned H, double resolution,
                  const double* origin, double occupied_thresh, double free_thresh, const char* pgm_path, const char* yaml_path) {
  return sm_guarded(s, [&]() {
    const size_t cells = (size_t)W * H;
    std::vector<unsigned char> image(cells);
    B200_CUDA(cudaMemcpyAsync(image.data(), image_dev, cells, cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    const std::string head = og_pgm_header(W, H, resolution);
    const std::string yaml = og_yaml(pgm_path, resolution, origin, occupied_thresh, free_thresh);
    auto fail = [&](const char* path, const char* why) {
      s->err = std::string(what) + why + path + ": " + std::strerror(errno);
      return (int)B200REG_ERR_IO;
    };
    if (const char* why = write_file(pgm_path, head, image.data(), cells)) return fail(pgm_path, why);
    if (const char* why = write_file(yaml_path, yaml)) return fail(yaml_path, why);
    return (int)B200REG_OK;
  });
}

}  // namespace

extern "C" {

int b200sm_build_occupancy_grid(b200sm_t s, const double* poses_colmajor16, const b200sm_occupancy_params* params,
                                b200sm_occupancy_info* info) {
  if (!s) return B200REG_ERR_ARG;
  const OgParams p = og_params_from(params);
  OgConst c;
  if (const char* why = og_prepare(p, &c)) return sm_fail(s, B200REG_ERR_ARG, (std::string("build_occupancy_grid: ") + why).c_str());
  // every submap's ray origin; the entries' bounds start at their origin's cell, and an empty submap's origin alone
  // widens the grid
  SubmapTiles t;
  std::vector<OgEntry> table;
  std::vector<int> bounds, origins;
  int rc = map_prologue(s, "build_occupancy_grid", poses_colmajor16, OG_TILE, nullptr, &t, &table, [&](size_t k, OgEntry& e) {
    long long o[3];
    if (!og_origin(c, p, e.T, o))
      return origin_refused(s, "build_occupancy_grid", k, "2^30 cells, or more than 2^16 cells from the height band");
    e.xo = o[0];
    e.yo = o[1];
    e.zo = o[2];
    const int x = og_cell(o[0]), y = og_cell(o[1]);
    origins.insert(origins.end(), {x, y});
    if (e.n) bounds.insert(bounds.end(), {x, y, x, y});
    return (int)B200REG_OK;
  });
  if (rc != B200REG_OK) return rc;
  return sm_guarded(s, [&]() {
    MapWorkspace& w = s->work;
    OccupancyGrid& G = s->og;
    // K14a over the submaps with points
    unsigned long long ctr[OG_CTR_COUNT] = {};
    int lo[2], hi[2];
    bounds_pass<2>(s, og_bounds_launch, c, table, t.tiles, w.og_table, bounds, OG_CTR_COUNT, ctr, 2, lo, hi);
    for (size_t k = 0; k < origins.size(); k += 2)
      for (int a = 0; a < 2; a++) {
        lo[a] = std::min(lo[a], origins[k + a]);
        hi[a] = std::max(hi[a], origins[k + a]);
      }
    unsigned long long W, H;
    if ((rc = grid_or_refuse(s, "build_occupancy_grid", lo, hi, &W, &H)) != B200REG_OK) return rc;
    const int gx0 = lo[0], gy0 = lo[1];
    // from here on the previous grid is replaced
    G.built = false;
    const size_t cells = (size_t)(W * H);
    G.hits.ensure(cells);
    G.frees.ensure(cells);
    G.values.ensure(cells);
    G.image.ensure(cells);
    B200_CUDA(cudaMemsetAsync(G.hits.ptr, 0, cells * sizeof(uint32_t), s->stream));
    B200_CUDA(cudaMemsetAsync(G.frees.ptr, 0, cells * sizeof(uint32_t), s->stream));
    // windows, then batches of consecutive submaps whose bitmaps fit the scratch budget (a submap whose bitmaps alone
    // exceed it forms a batch of its own); the scratch is sized to the largest batch so formed
    for (size_t r = 0; r < table.size(); r++) {
      OgEntry& e = table[r];
      const int* b = &bounds[4 * r];
      e.x0 = b[0];
      e.y0 = b[1];
      e.width = (unsigned)(b[2] - b[0] + 1);
      e.height = (unsigned)(b[3] - b[1] + 1);
      e.stride = (e.width + 31) / 32;
      e.rows = e.height;
    }
    struct Batch {
      size_t b0, b1;
      unsigned long long words, fold, tiles;
    };
    std::vector<Batch> plan;
    unsigned long long largest = 0;
    for (size_t b0 = 0; b0 < table.size();) {
      Batch bt{b0, b0, 0, 0, 0};
      while (bt.b1 < table.size()) {
        OgEntry& e = table[bt.b1];
        const unsigned long long words = 2ull * e.stride * e.rows;
        if (bt.b1 > b0 && bt.words + words > OG_SCRATCH_WORDS) break;
        e.words_at = bt.words;
        e.fold_first = bt.fold;
        e.first_tile = (unsigned)bt.tiles;
        bt.words += words;
        bt.fold += words / 2;
        bt.tiles += (e.n + OG_TILE - 1) / OG_TILE;
        bt.b1++;
      }
      largest = std::max(largest, bt.words);
      plan.push_back(bt);
      b0 = bt.b1;
    }
    w.bitmaps.ensure((size_t)largest);
    for (const Batch& bt : plan) {
      if (bt.words > w.bitmaps.cap || bt.b1 > w.og_table.cap)
        return sm_fail(s, B200REG_ERR_CUDA, "build_occupancy_grid: a walk batch larger than its scratch");
      // the previous batch's kernels read the table: this copy is stream-ordered behind them
      B200_CUDA(cudaMemcpyAsync(w.og_table.ptr + bt.b0, table.data() + bt.b0, (bt.b1 - bt.b0) * sizeof(OgEntry),
                                cudaMemcpyHostToDevice, s->stream));
      B200_CUDA(cudaMemsetAsync(w.bitmaps.ptr, 0, bt.words * sizeof(uint32_t), s->stream));
      og_walk_launch(w.og_table.ptr + bt.b0, (int)(bt.b1 - bt.b0), (unsigned)bt.tiles, c, w.bitmaps.ptr, w.counters.ptr, s->stream);
      og_fold_launch(w.og_table.ptr + bt.b0, (int)(bt.b1 - bt.b0), bt.fold, w.bitmaps.ptr, gx0, gy0, (unsigned)W, G.hits.ptr,
                     G.frees.ptr, s->stream);
      s->launches += 2;
    }
    const int batches = (int)plan.size();
    og_classify_launch(G.hits.ptr, G.frees.ptr, (unsigned)W, (unsigned)H, c.occ_value, c.free_value, G.values.ptr, G.image.ptr,
                       w.counters.ptr, s->stream);
    s->launches += 1;
    B200_CUDA(cudaMemcpyAsync(ctr, w.counters.ptr, sizeof(ctr), cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));  // the host table goes out of scope; the counts are read
    if (ctr[OG_CTR_TRIPPED]) return sm_fail(s, B200REG_ERR_CUDA, "build_occupancy_grid: a walk left its submap's window");
    G.built = true;
    G.params = p;
    G.width = (unsigned)W;
    G.height = (unsigned)H;
    G.origin[0] = (double)gx0 * p.resolution;
    G.origin[1] = (double)gy0 * p.resolution;
    if (info) {
      info->width = G.width;
      info->height = G.height;
      info->origin[0] = G.origin[0];
      info->origin[1] = G.origin[1];
      info->resolution = p.resolution;
      info->n_rays = ctr[OG_CTR_RAYS];
      info->n_skipped = ctr[OG_CTR_SKIPPED];
      info->n_batches = batches;
      info->n_occupied = ctr[OG_CTR_OCCUPIED];
      info->n_free = ctr[OG_CTR_FREE];
      info->n_unknown = ctr[OG_CTR_UNKNOWN];
    }
    return (int)B200REG_OK;
  });
}

int b200sm_get_occupancy_grid(b200sm_t s, signed char* data, unsigned* hits, unsigned* frees, size_t capacity) {
  if (!s) return B200REG_ERR_ARG;
  if (!s->og.built) return sm_fail(s, B200REG_ERR_ARG, "get_occupancy_grid: no grid has been built");
  return sm_guarded(s, [&]() {
    const OccupancyGrid& G = s->og;
    const size_t m = std::min(capacity, (size_t)G.width * G.height);
    if (m) {
      get_if(s, data, G.values.ptr, m);
      get_if(s, hits, G.hits.ptr, m);
      get_if(s, frees, G.frees.ptr, m);
      B200_CUDA(cudaStreamSynchronize(s->stream));
    }
    return (int)B200REG_OK;
  });
}

int b200sm_save_occupancy_map(b200sm_t s, const char* pgm_path, const char* yaml_path) {
  if (!s || !pgm_path || !yaml_path) return B200REG_ERR_ARG;
  if (!s->og.built) return sm_fail(s, B200REG_ERR_ARG, "save_occupancy_map: no grid has been built");
  const OccupancyGrid& G = s->og;
  return save_map_pair(s, "save_occupancy_map: ", G.image.ptr, G.width, G.height, G.params.resolution, G.origin,
                       G.params.occupied_thresh, G.params.free_thresh, pgm_path, yaml_path);
}

}  // extern "C"

// ---- elevation / traversability map: surface heights under the clearance, slope, step and roughness over a window
// (csrc/elevation_map.hpp, csrc/elevation.cu) ----
namespace {

ElParams el_params_from(const b200sm_elevation_params* p) {
  ElParams q;
  if (p) {
    q.resolution = p->resolution;
    q.max_range = p->max_range;
    for (int k = 0; k < 3; k++) q.sensor_origin[k] = p->sensor_origin[k];
    q.clearance = p->clearance;
    q.min_points = p->min_points;
    q.window_cells = p->window_cells;
    q.min_cells = p->min_cells;
    q.max_slope = p->max_slope;
    q.max_step = p->max_step;
    q.max_roughness = p->max_roughness;
    q.occupied_thresh = p->occupied_thresh;
    q.free_thresh = p->free_thresh;
  }
  return q;
}

}  // namespace

extern "C" {

int b200sm_build_elevation_map(b200sm_t s, const double* poses_colmajor16, const b200sm_elevation_params* params,
                               b200sm_elevation_info* info) {
  if (!s) return B200REG_ERR_ARG;
  const ElParams p = el_params_from(params);
  ElConst c;
  if (const char* why = el_prepare(p, &c)) return sm_fail(s, B200REG_ERR_ARG, (std::string("build_elevation_map: ") + why).c_str());
  // the submaps with points: float pose and horizontal origin (the band is the whole line, so zo plays no part)
  SubmapTiles t;
  std::vector<OgEntry> table;
  int rc = map_prologue(s, "build_elevation_map", poses_colmajor16, OG_TILE, nullptr, &t, &table, [&](size_t k, OgEntry& e) {
    if (e.n && !el_origin(c, p, e.T, &e.xo, &e.yo)) return origin_refused(s, "build_elevation_map", k, "2^30 cells");
    return (int)B200REG_OK;
  });
  if (rc != B200REG_OK) return rc;
  if (table.empty()) return sm_fail(s, B200REG_ERR_ARG, "build_elevation_map: no submap has points");
  return sm_guarded(s, [&]() {
    MapWorkspace& w = s->work;
    // K14a: the extent of the non-skipped points, bounds starting empty
    std::vector<int> bounds;
    unsigned long long ctr[EL_CTR_COUNT] = {};
    int lo[2], hi[2];
    bounds_pass<2>(s, og_bounds_launch, c.og, table, t.tiles, w.og_table, bounds, EL_CTR_COUNT, ctr, 2, lo, hi);
    if (ctr[EL_CTR_POINTS] == 0) return sm_fail(s, B200REG_ERR_ARG, "build_elevation_map: every point is skipped");
    unsigned long long W, H;
    if ((rc = grid_or_refuse(s, "build_elevation_map", lo, hi, &W, &H)) != B200REG_OK) return rc;
    const int gx0 = lo[0], gy0 = lo[1];
    // the new map is built beside the last one, which stays until this build succeeds
    const size_t cells = (size_t)(W * H);
    auto m = std::make_unique<ElevationMap>();
    m->n.ensure(cells);
    m->lo.ensure(cells);
    m->top.ensure(cells);
    m->step.ensure(cells);
    m->tan_slope.ensure(cells);
    m->roughness.ensure(cells);
    m->value.ensure(cells);
    m->image.ensure(cells);
    B200_CUDA(cudaMemsetAsync(m->n.ptr, 0, cells * sizeof(uint32_t), s->stream));
    B200_CUDA(cudaMemsetAsync(m->lo.ptr, 0x7f, cells * sizeof(long long), s->stream));   // EL_LO_EMPTY
    B200_CUDA(cudaMemsetAsync(m->top.ptr, 0x80, cells * sizeof(long long), s->stream));  // EL_TOP_EMPTY
    long long zrange[2] = {EL_LO_EMPTY, EL_TOP_EMPTY};
    w.zrange.ensure(2);
    B200_CUDA(cudaMemcpyAsync(w.zrange.ptr, zrange, sizeof(zrange), cudaMemcpyHostToDevice, s->stream));
    el_lowest_launch(w.og_table.ptr, (int)table.size(), (unsigned)t.tiles, c, gx0, gy0, (unsigned)W, (unsigned)H, m->n.ptr, m->lo.ptr,
                     w.counters.ptr, s->stream);
    el_top_launch(w.og_table.ptr, (int)table.size(), (unsigned)t.tiles, c, gx0, gy0, (unsigned)W, (unsigned)H, m->lo.ptr, m->top.ptr,
                  w.counters.ptr, w.zrange.ptr, s->stream);
    B200_CUDA(cudaMemcpyAsync(zrange, w.zrange.ptr, sizeof(zrange), cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    s->launches += 2;
    if (zrange[1] - zrange[0] >= EL_HEIGHT_EXTENT)
      return sm_fail(s, B200REG_ERR_ARG, "build_elevation_map: the map's height extent is 2^24 cells or more");
    el_window_launch(c, (unsigned)W, (unsigned)H, m->n.ptr, m->top.ptr, m->step.ptr, m->tan_slope.ptr, m->roughness.ptr, m->value.ptr,
                     m->image.ptr, w.counters.ptr, s->stream);
    s->launches += 1;
    B200_CUDA(cudaMemcpyAsync(ctr, w.counters.ptr, sizeof(ctr), cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    if (ctr[EL_CTR_TRIPPED]) return sm_fail(s, B200REG_ERR_CUDA, "build_elevation_map: a point's cell left the grid");
    m->params = p;
    b200sm_elevation_info& in = m->info;
    in.width = (unsigned)W;
    in.height = (unsigned)H;
    in.origin[0] = (double)gx0 * p.resolution;
    in.origin[1] = (double)gy0 * p.resolution;
    in.resolution = p.resolution;
    in.n_points = ctr[EL_CTR_POINTS];
    in.n_skipped = ctr[EL_CTR_SKIPPED];
    in.n_overhang = ctr[EL_CTR_OVERHANG];
    in.n_observed = ctr[EL_CTR_OBSERVED];
    in.n_lethal = ctr[EL_CTR_LETHAL];
    in.n_traversable = ctr[EL_CTR_TRAVERSABLE];
    in.n_unknown = ctr[EL_CTR_UNKNOWN];
    if (info) *info = in;
    s->el = std::move(m);
    return (int)B200REG_OK;
  });
}

int b200sm_get_elevation_map(b200sm_t s, unsigned* n, long long* h, long long* lo, float* step, float* tan_slope, float* roughness,
                             signed char* value, size_t capacity) {
  if (!s) return B200REG_ERR_ARG;
  if (!s->el) return sm_fail(s, B200REG_ERR_ARG, "get_elevation_map: no map has been built");
  return sm_guarded(s, [&]() {
    const ElevationMap& m = *s->el;
    const size_t k = std::min(capacity, (size_t)m.info.width * m.info.height);
    if (k) {
      get_if(s, n, m.n.ptr, k);
      get_if(s, h, m.top.ptr, k);
      get_if(s, lo, m.lo.ptr, k);
      get_if(s, step, m.step.ptr, k);
      get_if(s, tan_slope, m.tan_slope.ptr, k);
      get_if(s, roughness, m.roughness.ptr, k);
      get_if(s, value, m.value.ptr, k);
      B200_CUDA(cudaStreamSynchronize(s->stream));
    }
    return (int)B200REG_OK;
  });
}

int b200sm_save_traversability_map(b200sm_t s, const char* pgm_path, const char* yaml_path) {
  if (!s || !pgm_path || !yaml_path) return B200REG_ERR_ARG;
  if (!s->el) return sm_fail(s, B200REG_ERR_ARG, "save_traversability_map: no map has been built");
  const ElevationMap& m = *s->el;
  return save_map_pair(s, "save_traversability_map: ", m.image.ptr, m.info.width, m.info.height, m.params.resolution, m.info.origin,
                       m.params.occupied_thresh, m.params.free_thresh, pgm_path, yaml_path);
}

}  // extern "C"

// ---- static map: dynamic points removed by a 3D free-space ray-cast from every submap's sensor origin (csrc/static_map.hpp,
// csrc/static_map.cu) ----
namespace {

// K15c's scratch budget: the hit and free bitmaps of a batch of submaps, one bit per occupied voxel each. A submap whose
// bitmaps alone exceed it forms a batch of its own.
constexpr unsigned long long SM_SCRATCH_WORDS = 16ull << 20;  // 64 MiB

SmParams sm_params_from(const b200sm_static_map_params* p) {
  SmParams q;
  if (p) {
    q.resolution = p->resolution;
    q.max_range = p->max_range;
    for (int k = 0; k < 3; k++) q.sensor_origin[k] = p->sensor_origin[k];
    q.ray_fraction = p->ray_fraction;
    q.min_frees = p->min_frees;
    q.dynamic_thresh = p->dynamic_thresh;
  }
  return q;
}

// What the front half leaves for the rest of a build
struct SmFront {
  SmBox box{};
  unsigned long long n_words = 0;
  unsigned n_voxels = 0;
  int batches = 0;
};

// The front half the static map, the map changes and the OctoMap share, on the bounds pass and the rank pass: K15a and the
// box (refused here, before anything is sized from it), then `replacing(bounds)` with K15a's per-entry bounds (the
// caller's last build is about to be overwritten; it may refuse with an error code, s->err set, or return B200REG_OK), K15b, and the walks K15c / K15d in batches of consecutive entries. The entries [0, split_entry) fold into
// hits[0] / frees[0] and, when split_entry < table.size(), the entries [split_entry, table.size()) into hits[1] /
// frees[1]; no batch crosses split_entry. The counts are sized and zeroed here (one slot when there is no occupied voxel).
// n_counters counters are zeroed. Must run inside sm_guarded; `what` prefixes the messages.
template <class Replacing>
int sm_front_half(b200sm_t s, const char* what, std::vector<SmEntry>& table, unsigned long long tiles, const SmConst& c, int n_counters,
                  size_t split_entry, DeviceBuffer<RankWord>& index, DeviceBuffer<uint32_t>* hits, DeviceBuffer<uint32_t>* frees,
                  Replacing&& replacing, SmFront* out) {
  MapWorkspace& w = s->work;
  const int n_entries = (int)table.size();
  std::vector<int> bounds;
  unsigned long long ctr[2] = {};
  int lo[3], hi[3];
  bounds_pass<3>(s, sm_bounds_launch, c, table, tiles, w.sm_table, bounds, n_counters, ctr, 2, lo, hi);
  const bool any_ray = ctr[SM_CTR_RAYS] > 0;
  SmBox box{};
  unsigned long long cells = 0;
  if (any_ray) {
    const int rc = box_or_refuse(s, what, "a box", "voxels", lo, hi, 0, &box, &cells);
    if (rc != B200REG_OK) return rc;
  }
  if (const int rc = replacing(bounds); rc != B200REG_OK) return rc;
  const unsigned long long n_words = (cells + 31) / 32;
  unsigned n_voxels = 0;
  if (any_ray)  // K15b: the rank index over the box, then the number of occupied voxels
    n_voxels = rank_pass(s, index, n_words, [&](RankWord* idx) {
      sm_mark_launch(w.sm_table.ptr, n_entries, (unsigned)tiles, c, box, idx, w.counters.ptr, s->stream);
    });
  const int n_epochs = split_entry < table.size() ? 2 : 1;
  const size_t nv = std::max<size_t>(n_voxels, 1);
  for (int e = 0; e < n_epochs; e++) {
    hits[e].ensure(nv);
    frees[e].ensure(nv);
    B200_CUDA(cudaMemsetAsync(hits[e].ptr, 0, nv * sizeof(uint32_t), s->stream));
    B200_CUDA(cudaMemsetAsync(frees[e].ptr, 0, nv * sizeof(uint32_t), s->stream));
  }
  // K15c / K15d in batches of consecutive submaps of one epoch: every submap's two bitmaps have the same size
  const unsigned long long words_per = (n_voxels + 31ull) / 32ull;
  int batches = 0;
  if (n_voxels > 0) {
    const size_t per_batch = (size_t)std::max<unsigned long long>(1ull, SM_SCRATCH_WORDS / (2ull * words_per));
    const size_t largest = std::min(per_batch, table.size());
    w.bitmaps.ensure((size_t)(2ull * words_per * largest));
    for (int e = 0; e < n_epochs; e++) {
      const size_t r0 = e == 0 ? 0 : split_entry, r1 = e == n_epochs - 1 ? table.size() : split_entry;
      for (size_t b0 = r0; b0 < r1; b0 += per_batch) {
        const size_t b1 = std::min(r1, b0 + per_batch);
        unsigned long long bt = 0;
        for (size_t r = b0; r < b1; r++) {
          table[r].batch_tile = (unsigned)bt;
          bt += (table[r].n + SM_TILE - 1) / SM_TILE;
        }
        if (2ull * words_per * (b1 - b0) > w.bitmaps.cap || b1 > w.sm_table.cap)
          return sm_fail(s, B200REG_ERR_CUDA, (std::string(what) + ": a walk batch larger than its scratch").c_str());
        // the previous batch's kernels read the table: this copy is stream-ordered behind them
        B200_CUDA(cudaMemcpyAsync(w.sm_table.ptr + b0, table.data() + b0, (b1 - b0) * sizeof(SmEntry), cudaMemcpyHostToDevice,
                                  s->stream));
        B200_CUDA(cudaMemsetAsync(w.bitmaps.ptr, 0, 2ull * words_per * (b1 - b0) * sizeof(uint32_t), s->stream));
        sm_walk_launch(w.sm_table.ptr + b0, (int)(b1 - b0), (unsigned)bt, c, box, index.ptr, n_voxels, words_per, w.bitmaps.ptr,
                       w.counters.ptr, s->stream);
        sm_fold_launch(w.bitmaps.ptr, (int)(b1 - b0), words_per, n_voxels, hits[e].ptr, frees[e].ptr, s->stream);
        s->launches += 2;
        batches++;
      }
    }
  }
  out->box = box;
  out->n_words = n_words;
  out->n_voxels = n_voxels;
  out->batches = batches;
  return (int)B200REG_OK;
}

}  // namespace

extern "C" {

int b200sm_build_static_map(b200sm_t s, const double* poses_colmajor16, const b200sm_static_map_params* params,
                            b200sm_static_map_info* info) {
  if (!s) return B200REG_ERR_ARG;
  const SmParams p = sm_params_from(params);
  SmConst c;
  if (const char* why = sm_prepare(p, &c)) return sm_fail(s, B200REG_ERR_ARG, (std::string("build_static_map: ") + why).c_str());
  // the entries of the submaps with points (empty ones own no tile), in submap order
  SubmapTiles t;
  std::vector<SmEntry> table;
  const int rc = map_prologue(s, "build_static_map", poses_colmajor16, SM_TILE, nullptr, &t, &table, [&](size_t k, SmEntry& e) {
    return sm_origin(c, p, e.T, e.o) ? (int)B200REG_OK : origin_refused(s, "build_static_map", k, "2^30 voxels");
  });
  if (rc != B200REG_OK) return rc;
  const unsigned long long total = map_points(s);
  if (total > 0xffffffffull) return sm_fail(s, B200REG_ERR_ARG, "build_static_map: a map of 2^32 points or more");
  const size_t n_sub = s->submaps.size();
  const unsigned long long tiles = t.tiles;
  const int n_entries = (int)table.size();
  return sm_guarded(s, [&]() {
    MapWorkspace& w = s->work;
    StaticMap& M = s->sm;
    SmFront f;
    const int rc = sm_front_half(s, "build_static_map", table, tiles, c, SM_CTR_COUNT, table.size(), M.index, &M.hits, &M.frees,
                                 [&](const std::vector<int>&) {
                                   M.built = false;
                                   return (int)B200REG_OK;
                                 },
                                 &f);
    if (rc != B200REG_OK) return rc;
    const SmBox& box = f.box;
    const unsigned n_voxels = f.n_voxels;
    unsigned long long ctr[SM_CTR_COUNT] = {};
    M.dynamic.ensure(std::max<size_t>(n_voxels, 1));
    if (n_voxels > 0) {
      // K15e
      sm_classify_launch(M.hits.ptr, M.frees.ptr, n_voxels, c, M.dynamic.ptr, w.counters.ptr, s->stream);
      s->launches += 1;
    }
    // K15f: kept points per tile, scanned into tile offsets; the host reads the total and sizes the static map from it
    unsigned kept = 0;
    std::vector<unsigned> tile_off((size_t)tiles + 1, 0);
    if (tiles) {
      w.tiles.ensure((size_t)tiles + 1);
      sm_count_launch(w.sm_table.ptr, n_entries, (unsigned)tiles, c, box, M.index.ptr, M.dynamic.ptr, n_voxels, w.tiles.ptr, s->stream);
      counter_scan_async(w.tiles.ptr, (size_t)tiles, w.scan_tmp, s->stream);
      s->launches += 3;
      B200_CUDA(cudaMemcpyAsync(tile_off.data(), w.tiles.ptr, tile_off.size() * sizeof(unsigned), cudaMemcpyDeviceToHost, s->stream));
      B200_CUDA(cudaStreamSynchronize(s->stream));
      kept = tile_off[(size_t)tiles];
    }
    // K15g
    M.points.ensure(std::max<size_t>(kept, 1));
    if (kept) {
      sm_write_launch(w.sm_table.ptr, n_entries, (unsigned)tiles, c, box, M.index.ptr, M.dynamic.ptr, n_voxels, w.tiles.ptr, kept,
                      M.points.ptr, w.counters.ptr, s->stream);
      s->launches += 1;
    }
    B200_CUDA(cudaMemcpyAsync(ctr, w.counters.ptr, sizeof(ctr), cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));  // the host table goes out of scope; the counts are read
    if (ctr[SM_CTR_TRIPPED]) return sm_fail(s, B200REG_ERR_CUDA, "build_static_map: a voxel outside the box or beyond the rank index");
    M.offsets = submap_offsets(t, n_sub, tile_off, kept);
    M.box = box;
    M.n_words = f.n_words;
    b200sm_static_map_info& I = M.info;
    for (int a = 0; a < 3; a++) {
      I.box_origin[a] = box.lo[a];
      I.box_dims[a] = box.dims[a];
    }
    I.n_rays = ctr[SM_CTR_RAYS];
    I.n_skipped = ctr[SM_CTR_SKIPPED];
    I.n_voxels = n_voxels;
    I.n_dynamic_voxels = ctr[SM_CTR_DYNAMIC];
    I.n_points = total;
    I.n_static_points = kept;
    I.n_batches = f.batches;
    M.built = true;
    if (info) *info = I;
    return (int)B200REG_OK;
  });
}

int b200sm_get_static_map(b200sm_t s, float* out_xyzi, size_t capacity, size_t* n, size_t* offsets) {
  if (!s || (!out_xyzi && capacity)) return B200REG_ERR_ARG;
  if (!s->sm.built) return sm_fail(s, B200REG_ERR_ARG, "get_static_map: no static map has been built");
  const StaticMap& M = s->sm;
  return get_compacted(s, M.points, (size_t)M.info.n_static_points, M.offsets, out_xyzi, capacity, n, offsets);
}

int b200sm_get_map_voxels(b200sm_t s, int* ijk3, unsigned* hits, unsigned* frees, unsigned char* dynamic, size_t capacity, size_t* n) {
  if (!s) return B200REG_ERR_ARG;
  if (!s->sm.built) return sm_fail(s, B200REG_ERR_ARG, "get_map_voxels: no static map has been built");
  return sm_guarded(s, [&]() {
    const StaticMap& M = s->sm;
    const unsigned n_voxels = (unsigned)M.info.n_voxels;
    if (n) *n = n_voxels;
    const size_t m = std::min(capacity, (size_t)n_voxels);
    if (m == 0) return (int)B200REG_OK;
    if (ijk3) {
      DeviceBuffer<int>& ijk = s->work.ijk;
      ijk.ensure(3 * (size_t)n_voxels);
      sm_voxel_list_launch(M.index.ptr, M.n_words, M.box, n_voxels, ijk.ptr, s->stream);
      s->launches += 1;
      get_if(s, ijk3, ijk.ptr, 3 * m);
    }
    get_if(s, hits, M.hits.ptr, m);
    get_if(s, frees, M.frees.ptr, m);
    get_if(s, dynamic, M.dynamic.ptr, m);
    B200_CUDA(cudaStreamSynchronize(s->stream));
    return (int)B200REG_OK;
  });
}

int b200sm_save_static_map_pcd_ascii(b200sm_t s, const char* path, size_t* n_points, size_t* n_bytes) {
  if (!s || !path) return B200REG_ERR_ARG;
  if (!s->sm.built) return sm_fail(s, B200REG_ERR_ARG, "save_static_map_pcd_ascii: no static map has been built");
  return save_compacted_pcd(s, "save_static_map_pcd_ascii", "the static map has no points", s->sm.points,
                            (size_t)s->sm.info.n_static_points, path, n_points, n_bytes);
}

}  // extern "C"

// ---- map changes: what appeared and vanished between two recordings, and the updated map (csrc/map_changes.hpp,
// csrc/map_changes.cu, and the static map's front half) ----
extern "C" {

int b200sm_build_map_changes(b200sm_t s, const double* poses_colmajor16, const b200sm_static_map_params* params, long long split_submap,
                             b200sm_map_change_info* info) {
  if (!s) return B200REG_ERR_ARG;
  const SmParams p = sm_params_from(params);
  SmConst c;
  if (const char* why = sm_prepare(p, &c)) return sm_fail(s, B200REG_ERR_ARG, (std::string("build_map_changes: ") + why).c_str());
  const size_t n_sub = s->submaps.size();
  unsigned long long split = 0;
  const unsigned long long last_first = s->seg_first.size() > 1 ? (unsigned long long)s->seg_first.back() : 0ull;
  if (n_sub)  // a session without submaps is refused first, by the prologue
    if (const char* why = ch_split(split_submap, n_sub, last_first, &split))
      return sm_fail(s, B200REG_ERR_ARG, (std::string("build_map_changes: ") + why).c_str());
  // the entries of the submaps with points, in submap order, their first map index, and the first AFTER entry
  SubmapTiles t;
  std::vector<SmEntry> table;
  std::vector<unsigned> map_first;
  size_t split_entry = 0;
  unsigned long long at = 0;
  const int rc = map_prologue(s, "build_map_changes", poses_colmajor16, SM_TILE, nullptr, &t, &table, [&](size_t k, SmEntry& e) {
    if (!sm_origin(c, p, e.T, e.o)) return origin_refused(s, "build_map_changes", k, "2^30 voxels");
    if (k == split) split_entry = table.size();
    if (e.n) map_first.push_back((unsigned)at);
    at += e.n;
    return (int)B200REG_OK;
  });
  if (rc != B200REG_OK) return rc;
  const unsigned long long total = at;
  if (total > 0xffffffffull) return sm_fail(s, B200REG_ERR_ARG, "build_map_changes: a map of 2^32 points or more");
  const unsigned long long tiles = t.tiles;
  const int n_entries = (int)table.size();
  return sm_guarded(s, [&]() {
    MapWorkspace& w = s->work;
    // the new build is made beside the last one, which stays until this one succeeds
    auto m = std::make_unique<MapChanges>();
    SmFront f;
    const int rc = sm_front_half(s, "build_map_changes", table, tiles, c, CH_CTR_COUNT, split_entry, m->index, m->hits, m->frees,
                                 [](const std::vector<int>&) { return (int)B200REG_OK; }, &f);
    if (rc != B200REG_OK) return rc;
    const unsigned n_voxels = f.n_voxels;
    const size_t nv = std::max<size_t>(n_voxels, 1);
    for (int e = 0; e < 2; e++)
      if (!m->hits[e].ptr) {  // no AFTER submap with points: the front half folded one epoch only
        m->hits[e].ensure(nv);
        m->frees[e].ensure(nv);
        B200_CUDA(cudaMemsetAsync(m->hits[e].ptr, 0, nv * sizeof(uint32_t), s->stream));
        B200_CUDA(cudaMemsetAsync(m->frees[e].ptr, 0, nv * sizeof(uint32_t), s->stream));
      }
    // K20a
    m->label.ensure(nv);
    if (n_voxels > 0) {
      ch_classify_launch(m->hits[CH_BEFORE].ptr, m->frees[CH_BEFORE].ptr, m->hits[CH_AFTER].ptr, m->frees[CH_AFTER].ptr, n_voxels, c,
                         m->label.ptr, w.counters.ptr, s->stream);
      s->launches += 1;
    }
    // K20b: the point labels and the kept points per tile, scanned into tile offsets; the host reads the total and sizes
    // the updated map from it
    m->point_label.ensure(std::max<size_t>((size_t)total, 1));
    unsigned kept = 0;
    std::vector<unsigned> tile_off((size_t)tiles + 1, 0);
    if (tiles) {
      w.map_first.ensure(map_first.size());
      B200_CUDA(cudaMemcpyAsync(w.map_first.ptr, map_first.data(), map_first.size() * sizeof(unsigned), cudaMemcpyHostToDevice,
                                s->stream));
      w.tiles.ensure((size_t)tiles + 1);
      ch_label_launch(w.sm_table.ptr, n_entries, (unsigned)tiles, c, f.box, m->index.ptr, m->label.ptr, n_voxels, (int)split_entry,
                      w.map_first.ptr, m->point_label.ptr, w.tiles.ptr, w.counters.ptr, s->stream);
      counter_scan_async(w.tiles.ptr, (size_t)tiles, w.scan_tmp, s->stream);
      s->launches += 3;
      B200_CUDA(cudaMemcpyAsync(tile_off.data(), w.tiles.ptr, tile_off.size() * sizeof(unsigned), cudaMemcpyDeviceToHost, s->stream));
      B200_CUDA(cudaStreamSynchronize(s->stream));
      kept = tile_off[(size_t)tiles];
    }
    // K20c
    m->updated.ensure(std::max<size_t>(kept, 1));
    if (kept) {
      ch_write_launch(w.sm_table.ptr, n_entries, (unsigned)tiles, w.map_first.ptr, m->point_label.ptr, w.tiles.ptr, kept, m->updated.ptr,
                      w.counters.ptr, s->stream);
      s->launches += 1;
    }
    unsigned long long ctr[CH_CTR_COUNT] = {};
    B200_CUDA(cudaMemcpyAsync(ctr, w.counters.ptr, sizeof(ctr), cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));  // the host tables go out of scope; the counts are read
    if (ctr[SM_CTR_TRIPPED])
      return sm_fail(s, B200REG_ERR_CUDA, "build_map_changes: a voxel outside the box or beyond the rank index, or a point beyond the map");
    m->offsets = submap_offsets(t, n_sub, tile_off, kept);
    m->box = f.box;
    m->n_words = f.n_words;
    b200sm_map_change_info& I = m->info;
    for (int a = 0; a < 3; a++) {
      I.box_origin[a] = f.box.lo[a];
      I.box_dims[a] = f.box.dims[a];
    }
    I.split_submap = (long long)split;
    I.n_rays = ctr[SM_CTR_RAYS];
    I.n_skipped = ctr[SM_CTR_SKIPPED];
    I.n_voxels = n_voxels;
    I.n_appeared_voxels = ctr[CH_CTR_APPEARED_VOXELS];
    I.n_vanished_voxels = ctr[CH_CTR_VANISHED_VOXELS];
    I.n_points = total;
    I.n_appeared_points = ctr[CH_CTR_APPEARED_POINTS];
    I.n_vanished_points = ctr[CH_CTR_VANISHED_POINTS];
    I.n_updated_points = kept;
    I.n_batches = f.batches;
    if (info) *info = I;
    s->ch = std::move(m);
    return (int)B200REG_OK;
  });
}

int b200sm_get_map_changes(b200sm_t s, unsigned char* labels, size_t capacity, size_t* n) {
  if (!s || (!labels && capacity)) return B200REG_ERR_ARG;
  if (!s->ch) return sm_fail(s, B200REG_ERR_ARG, "get_map_changes: no build yet");
  return sm_guarded(s, [&]() {
    const MapChanges& m = *s->ch;
    if (n) *n = (size_t)m.info.n_points;
    const size_t k = std::min(capacity, (size_t)m.info.n_points);
    if (k) {
      get_if(s, labels, m.point_label.ptr, k);
      B200_CUDA(cudaStreamSynchronize(s->stream));
    }
    return (int)B200REG_OK;
  });
}

int b200sm_get_change_voxels(b200sm_t s, int* ijk3, unsigned* hits_before, unsigned* frees_before, unsigned* hits_after,
                             unsigned* frees_after, unsigned char* label, size_t capacity, size_t* n) {
  if (!s) return B200REG_ERR_ARG;
  if (!s->ch) return sm_fail(s, B200REG_ERR_ARG, "get_change_voxels: no build yet");
  return sm_guarded(s, [&]() {
    const MapChanges& m = *s->ch;
    const unsigned n_voxels = (unsigned)m.info.n_voxels;
    if (n) *n = n_voxels;
    const size_t k = std::min(capacity, (size_t)n_voxels);
    if (k == 0) return (int)B200REG_OK;
    if (ijk3) {
      DeviceBuffer<int>& ijk = s->work.ijk;
      ijk.ensure(3 * (size_t)n_voxels);
      sm_voxel_list_launch(m.index.ptr, m.n_words, m.box, n_voxels, ijk.ptr, s->stream);
      s->launches += 1;
      get_if(s, ijk3, ijk.ptr, 3 * k);
    }
    get_if(s, hits_before, m.hits[CH_BEFORE].ptr, k);
    get_if(s, frees_before, m.frees[CH_BEFORE].ptr, k);
    get_if(s, hits_after, m.hits[CH_AFTER].ptr, k);
    get_if(s, frees_after, m.frees[CH_AFTER].ptr, k);
    get_if(s, label, m.label.ptr, k);
    B200_CUDA(cudaStreamSynchronize(s->stream));
    return (int)B200REG_OK;
  });
}

int b200sm_get_updated_map(b200sm_t s, float* out_xyzi, size_t capacity, size_t* n, size_t* offsets) {
  if (!s || (!out_xyzi && capacity)) return B200REG_ERR_ARG;
  if (!s->ch) return sm_fail(s, B200REG_ERR_ARG, "get_updated_map: no build yet");
  const MapChanges& m = *s->ch;
  return get_compacted(s, m.updated, (size_t)m.info.n_updated_points, m.offsets, out_xyzi, capacity, n, offsets);
}

int b200sm_save_updated_map_pcd_ascii(b200sm_t s, const char* path, size_t* n_points, size_t* n_bytes) {
  if (!s || !path) return B200REG_ERR_ARG;
  if (!s->ch) return sm_fail(s, B200REG_ERR_ARG, "save_updated_map_pcd_ascii: no build yet");
  return save_compacted_pcd(s, "save_updated_map_pcd_ascii", "the updated map has no points", s->ch->updated,
                            (size_t)s->ch->info.n_updated_points, path, n_points, n_bytes);
}

}  // extern "C"

// ---- surface mesh: a TSDF fused from every submap's rays, extracted by surface nets, saved as PLY (csrc/mesh.hpp,
// csrc/mesh.cu, and the static map's rays and bounds) ----
namespace {

MsParams ms_params_from(const b200sm_mesh_params* p) {
  MsParams q;
  if (p) {
    q.resolution = p->resolution;
    q.truncation = p->truncation;
    q.max_range = p->max_range;
    for (int k = 0; k < 3; k++) q.sensor_origin[k] = p->sensor_origin[k];
    q.min_weight = p->min_weight;
  }
  return q;
}

constexpr size_t MS_PLY_PIECE = 1u << 20;  // vertices or faces per piece of the PLY write (12 MiB of staging)

}  // namespace

extern "C" {

int b200sm_build_mesh(b200sm_t s, const double* poses_colmajor16, const b200sm_mesh_params* params, b200sm_mesh_info* info) {
  if (!s) return B200REG_ERR_ARG;
  const MsParams p = ms_params_from(params);
  MsConst c;
  if (const char* why = ms_prepare(p, &c)) return sm_fail(s, B200REG_ERR_ARG, (std::string("build_mesh: ") + why).c_str());
  SubmapTiles t;
  std::vector<SmEntry> table;
  const int rc = map_prologue(s, "build_mesh", poses_colmajor16, SM_TILE, nullptr, &t, &table, [&](size_t k, SmEntry& e) {
    return ms_origin(c, p, e.T, e.o) ? (int)B200REG_OK : origin_refused(s, "build_mesh", k, "2^30 voxels");
  });
  if (rc != B200REG_OK) return rc;
  const unsigned long long total = map_points(s);
  if (total > 0xffffffffull) return sm_fail(s, B200REG_ERR_ARG, "build_mesh: a map of 2^32 points or more");
  const unsigned long long tiles = t.tiles;
  const int n_entries = (int)table.size();
  return sm_guarded(s, [&]() {
    MapWorkspace& w = s->work;
    // the new build is made beside the last one, which stays until this one succeeds
    auto m = std::make_unique<MeshBuild>();
    // K15a: the endpoint voxels' bounds and the ray counts
    std::vector<int> bounds;
    unsigned long long ctr[MS_CTR_COUNT] = {};
    int lo[3], hi[3];
    bounds_pass<3>(s, sm_bounds_launch, c.sm, table, tiles, w.sm_table, bounds, MS_CTR_COUNT, ctr, 2, lo, hi);
    const bool any_ray = ctr[SM_CTR_RAYS] > 0;
    SmBox box{};
    unsigned long long cells = 0;
    if (any_ray) {
      const int rc = box_or_refuse(s, "build_mesh", "a band box", "voxels", lo, hi, c.r, &box, &cells);
      if (rc != B200REG_OK) return rc;
    }
    const unsigned long long n_words = (cells + 31) / 32;
    unsigned n_band = 0;
    if (any_ray)  // K21a: the band walks into the rank index, then the number of band voxels
      n_band = rank_pass(s, m->index, n_words, [&](RankWord* idx) {
        ms_mark_launch(w.sm_table.ptr, n_entries, (unsigned)tiles, c, box, idx, w.counters.ptr, s->stream);
      });
    const size_t nb = std::max<size_t>(n_band, 1);
    m->sum.ensure(nb);
    m->weight.ensure(nb);
    m->ijk.ensure(3 * nb);
    B200_CUDA(cudaMemsetAsync(m->sum.ptr, 0, nb * sizeof(unsigned long long), s->stream));
    B200_CUDA(cudaMemsetAsync(m->weight.ptr, 0, nb * sizeof(uint32_t), s->stream));
    unsigned n_vert = 0;
    const unsigned vtiles = (n_band + MS_THREADS - 1) / MS_THREADS;
    if (n_band > 0) {
      // K21b, the voxel list, K21c and its scan: the vertex count
      ms_fuse_launch(w.sm_table.ptr, n_entries, (unsigned)tiles, c, box, m->index.ptr, n_band, m->sum.ptr, m->weight.ptr, w.counters.ptr,
                     s->stream);
      sm_voxel_list_launch(m->index.ptr, n_words, box, n_band, m->ijk.ptr, s->stream);
      w.active.ensure(n_band);
      w.vertex_counts.ensure((size_t)vtiles + 1);
      ms_active_launch(m->ijk.ptr, m->sum.ptr, m->weight.ptr, m->index.ptr, box, n_band, c.min_weight, w.active.ptr, w.vertex_counts.ptr,
                       w.counters.ptr, s->stream);
      counter_scan_async(w.vertex_counts.ptr, vtiles, w.scan_tmp, s->stream);
      s->launches += 5;
      B200_CUDA(cudaMemcpyAsync(&n_vert, w.vertex_counts.ptr + vtiles, sizeof(unsigned), cudaMemcpyDeviceToHost, s->stream));
      B200_CUDA(cudaStreamSynchronize(s->stream));
    }
    m->xyz.ensure(3 * std::max<size_t>(n_vert, 1));
    if (n_band > 0) {
      // K21d and its scan: the vertices, and the face count read back with the counters
      w.vertex_id.ensure(n_band);
      w.face_counts.ensure((size_t)vtiles + 1);
      ms_vertex_launch(m->ijk.ptr, m->sum.ptr, m->weight.ptr, m->index.ptr, box, n_band, c, w.active.ptr, w.vertex_counts.ptr, n_vert,
                       w.vertex_id.ptr, m->xyz.ptr, w.face_counts.ptr, w.counters.ptr, s->stream);
      counter_scan_async(w.face_counts.ptr, vtiles, w.scan_tmp, s->stream);
      s->launches += 3;
    }
    B200_CUDA(cudaMemcpyAsync(ctr, w.counters.ptr, sizeof(ctr), cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    if (ctr[MS_CTR_FACES] > 0xffffffffull) return sm_fail(s, B200REG_ERR_ARG, "build_mesh: 2^32 faces or more");
    const unsigned n_faces = (unsigned)ctr[MS_CTR_FACES];
    m->faces.ensure(3 * std::max<size_t>(n_faces, 1));
    if (n_faces > 0) {
      // K21e
      ms_face_launch(m->ijk.ptr, m->sum.ptr, m->weight.ptr, m->index.ptr, box, n_band, c.min_weight, w.vertex_id.ptr, w.face_counts.ptr,
                     n_faces, m->faces.ptr, w.counters.ptr, s->stream);
      s->launches += 1;
      B200_CUDA(cudaMemcpyAsync(ctr, w.counters.ptr, sizeof(ctr), cudaMemcpyDeviceToHost, s->stream));
    }
    B200_CUDA(cudaStreamSynchronize(s->stream));  // the host table goes out of scope; the counts are read
    if (ctr[SM_CTR_TRIPPED])
      return sm_fail(s, B200REG_ERR_CUDA, "build_mesh: a voxel outside the box or beyond the rank index, or a vertex or face beyond its count");
    b200sm_mesh_info& I = m->info;
    for (int a = 0; a < 3; a++) {
      I.box_origin[a] = any_ray ? box.lo[a] : 0;
      I.box_dims[a] = any_ray ? box.dims[a] : 0;
    }
    I.n_points = total;
    I.n_rays = ctr[SM_CTR_RAYS];
    I.n_skipped = ctr[SM_CTR_SKIPPED];
    I.n_walked = ctr[MS_CTR_WALKED];
    I.n_band_voxels = n_band;
    I.n_observed_voxels = ctr[MS_CTR_OBSERVED];
    I.n_vertices = n_vert;
    I.n_faces = n_faces;
    if (info) *info = I;
    s->ms = std::move(m);
    return (int)B200REG_OK;
  });
}

int b200sm_get_mesh(b200sm_t s, float* xyz, size_t vertex_capacity, size_t* n_vertices, unsigned* faces3, size_t face_capacity,
                    size_t* n_faces) {
  if (!s || (!xyz && vertex_capacity) || (!faces3 && face_capacity)) return B200REG_ERR_ARG;
  if (!s->ms) return sm_fail(s, B200REG_ERR_ARG, "get_mesh: no mesh has been built");
  return sm_guarded(s, [&]() {
    const MeshBuild& m = *s->ms;
    if (n_vertices) *n_vertices = (size_t)m.info.n_vertices;
    if (n_faces) *n_faces = (size_t)m.info.n_faces;
    const size_t kv = std::min(vertex_capacity, (size_t)m.info.n_vertices), kf = std::min(face_capacity, (size_t)m.info.n_faces);
    if (kv) get_if(s, xyz, m.xyz.ptr, 3 * kv);
    if (kf) get_if(s, faces3, m.faces.ptr, 3 * kf);
    if (kv || kf) B200_CUDA(cudaStreamSynchronize(s->stream));
    return (int)B200REG_OK;
  });
}

int b200sm_get_mesh_voxels(b200sm_t s, int* ijk3, long long* sdf_sum, unsigned* weight, size_t capacity, size_t* n) {
  if (!s) return B200REG_ERR_ARG;
  if (!s->ms) return sm_fail(s, B200REG_ERR_ARG, "get_mesh_voxels: no mesh has been built");
  return sm_guarded(s, [&]() {
    const MeshBuild& m = *s->ms;
    const size_t nb = (size_t)m.info.n_band_voxels;
    if (n) *n = nb;
    const size_t k = std::min(capacity, nb);
    if (k == 0) return (int)B200REG_OK;
    get_if(s, ijk3, m.ijk.ptr, 3 * k);
    get_if(s, sdf_sum, m.sum.ptr, k);
    get_if(s, weight, m.weight.ptr, k);
    B200_CUDA(cudaStreamSynchronize(s->stream));
    return (int)B200REG_OK;
  });
}

int b200sm_save_mesh_ply(b200sm_t s, const char* path, size_t* n_bytes) {
  if (!s || !path) return B200REG_ERR_ARG;
  if (!s->ms) return sm_fail(s, B200REG_ERR_ARG, "save_mesh_ply: no mesh has been built");
  const MeshBuild& m = *s->ms;
  const size_t V = (size_t)m.info.n_vertices, F = (size_t)m.info.n_faces;
  if (F == 0) return sm_fail(s, B200REG_ERR_ARG, "save_mesh_ply: the mesh has no faces");
  return sm_guarded(s, [&]() {
    const std::string header = "ply\nformat binary_little_endian 1.0\nelement vertex " + std::to_string(V) +
                               "\nproperty float x\nproperty float y\nproperty float z\nelement face " + std::to_string(F) +
                               "\nproperty list uchar uint vertex_indices\nend_header\n";
    if (n_bytes) *n_bytes = header.size() + 12 * V + 13 * F;
    FILE* fp = std::fopen(path, "wb");
    if (!fp) {
      s->err = std::string("save_mesh_ply: cannot open ") + path + ": " + std::strerror(errno);
      return (int)B200REG_ERR_IO;
    }
    // pieces: the vertices, then the faces, MS_PLY_PIECE records each (12 bytes on the device either way)
    const size_t vp = (V + MS_PLY_PIECE - 1) / MS_PLY_PIECE, fpieces = (F + MS_PLY_PIECE - 1) / MS_PLY_PIECE, n = vp + fpieces;
    auto span = [&](size_t piece, size_t* first, size_t* count) {
      const bool face = piece >= vp;
      const size_t q = face ? piece - vp : piece, all = face ? F : V;
      *first = q * MS_PLY_PIECE;
      *count = std::min(MS_PLY_PIECE, all - *first);
      return face;
    };
    auto enqueue = [&](size_t piece, char* buf) {
      size_t first, count;
      const void* src = span(piece, &first, &count) ? (const void*)(m.faces.ptr + 3 * first) : (const void*)(m.xyz.ptr + 3 * first);
      B200_CUDA(cudaMemcpyAsync(buf, src, 12 * count, cudaMemcpyDeviceToHost, s->stream));
    };
    std::vector<unsigned char> rec;
    auto write = [&](size_t piece, const char* buf) {
      size_t first, count;
      bool ok = piece > 0 || std::fwrite(header.data(), 1, header.size(), fp) == header.size();
      if (span(piece, &first, &count)) {
        rec.resize(13 * count);  // a 0x03 byte, then the three little-endian ids
        for (size_t f = 0; f < count; f++) {
          rec[13 * f] = 3;
          std::memcpy(&rec[13 * f + 1], buf + 12 * f, 12);
        }
        ok = ok && std::fwrite(rec.data(), 1, rec.size(), fp) == rec.size();
      } else {
        ok = ok && std::fwrite(buf, 1, 12 * count, fp) == 12 * count;
      }
      if (ok && piece + 1 == n) {
        ok = std::fclose(fp) == 0;
        fp = nullptr;
      }
      if (ok) return (int)B200REG_OK;
      s->err = std::string("save_mesh_ply: writing ") + path + ": " + std::strerror(errno);
      return (int)B200REG_ERR_IO;
    };
    return write_staged(s, n, 12 * MS_PLY_PIECE, fp, enqueue, write);
  });
}

}  // extern "C"

// ---- OctoMap: free and occupied voxels from every submap's rays, pruned into OctoMap's key tree and saved as a .bt file
// (csrc/octomap.hpp, csrc/octomap.cu, and the static map's front half) ----
namespace {

constexpr size_t OM_BT_PIECE = 8u << 20;  // data bytes per piece of the .bt write

}  // namespace

extern "C" {

int b200sm_build_octomap(b200sm_t s, const double* poses_colmajor16, const b200sm_static_map_params* params, b200sm_octomap_info* info) {
  if (!s) return B200REG_ERR_ARG;
  const SmParams p = sm_params_from(params);
  SmConst c;
  if (const char* why = sm_prepare(p, &c)) return sm_fail(s, B200REG_ERR_ARG, (std::string("build_octomap: ") + why).c_str());
  if (!om_resolution_exact(p.resolution))
    return sm_fail(s, B200REG_ERR_ARG, "build_octomap: the resolution does not read back from printf(\"%g\"), the .bt header's res");
  SubmapTiles t;
  std::vector<SmEntry> table;
  const int rc = map_prologue(s, "build_octomap", poses_colmajor16, SM_TILE, nullptr, &t, &table, [&](size_t k, SmEntry& e) {
    return sm_origin(c, p, e.T, e.o) ? (int)B200REG_OK : origin_refused(s, "build_octomap", k, "2^30 voxels");
  });
  if (rc != B200REG_OK) return rc;
  const unsigned long long total = map_points(s);
  if (total > 0xffffffffull) return sm_fail(s, B200REG_ERR_ARG, "build_octomap: a map of 2^32 points or more");
  const unsigned long long tiles = t.tiles;
  const int n_entries = (int)table.size();
  return sm_guarded(s, [&]() {
    MapWorkspace& w = s->work;
    // the new build is made beside the last one, which stays until this one succeeds
    auto m = std::make_unique<OctoMapBuild>();
    // K15a-K15d on the workspace's own buffers; the box is the endpoint voxels' and the origin voxels of the entries
    // with a ray (K15a left INT_MAX in an entry without one), refused before anything is sized from it
    SmBox box{};
    unsigned long long cells = 0;
    bool any_ray = false;
    SmFront f;
    const int rc = sm_front_half(s, "build_octomap", table, tiles, c, OM_CTR_COUNT, table.size(), w.occ_index, &w.occ_hits, &w.occ_frees,
                                 [&](const std::vector<int>& bounds) {
                                   int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
                                   for (size_t r = 0; r < table.size(); r++) {
                                     if (bounds[6 * r] == INT_MAX) continue;
                                     any_ray = true;
                                     for (int a = 0; a < 3; a++) {
                                       const int o = og_cell(table[r].o[a]);
                                       lo[a] = std::min({lo[a], bounds[6 * r + a], o});
                                       hi[a] = std::max({hi[a], bounds[6 * r + 3 + a], o});
                                     }
                                   }
                                   if (!any_ray) return (int)B200REG_OK;
                                   if (const char* why = om_box(lo, hi, box.dims, &cells)) {
                                     auto width = [&](int a) { return std::to_string((long long)hi[a] - lo[a] + 1); };
                                     s->err = "build_octomap: a box of " + width(0) + " x " + width(1) + " x " + width(2) + " voxels: " + why;
                                     return (int)B200REG_ERR_ARG;
                                   }
                                   for (int a = 0; a < 3; a++) box.lo[a] = lo[a];
                                   return (int)B200REG_OK;
                                 },
                                 &f);
    if (rc != B200REG_OK) return rc;
    unsigned inner = 0;
    if (any_ray) {
      const OmPyramid pyr = om_pyramid(box);
      const unsigned long long n_cells = pyr.first[OM_DEPTH + 1], words = (cells + 31) / 32;
      w.occ_dynamic.ensure(f.n_voxels);
      w.freed.ensure((size_t)words);
      w.pyr_codes.ensure((size_t)n_cells);
      w.pyr_counts.ensure((size_t)n_cells);
      m->states.ensure((size_t)cells);
      B200_CUDA(cudaMemsetAsync(w.freed.ptr, 0, words * sizeof(uint32_t), s->stream));
      // K15e, K22a, K22b, K22c per level up to the root, K22d per level down from it
      sm_classify_launch(w.occ_hits.ptr, w.occ_frees.ptr, f.n_voxels, c, w.occ_dynamic.ptr, w.counters.ptr, s->stream);
      om_free_launch(w.sm_table.ptr, n_entries, (unsigned)tiles, c, box, w.freed.ptr, w.counters.ptr, s->stream);
      om_leaf_launch(pyr, f.box, w.occ_index.ptr, w.occ_dynamic.ptr, f.n_voxels, w.freed.ptr, m->states.ptr, w.pyr_codes.ptr,
                     w.pyr_counts.ptr, w.counters.ptr, s->stream);
      for (int l = 2; l <= OM_DEPTH; l++) om_reduce_launch(pyr, l, w.pyr_codes.ptr, w.pyr_counts.ptr, s->stream);
      for (int l = OM_DEPTH; l >= 2; l--) om_offset_launch(pyr, l, w.pyr_codes.ptr, w.pyr_counts.ptr, s->stream);
      s->launches += 3 + 2 * (OM_DEPTH - 1);
      // the root's inner count sizes the data; K22e writes it
      B200_CUDA(cudaMemcpyAsync(&inner, w.pyr_counts.ptr + pyr.first[OM_DEPTH], sizeof(unsigned), cudaMemcpyDeviceToHost, s->stream));
      B200_CUDA(cudaStreamSynchronize(s->stream));
      m->data.ensure(2 * (size_t)inner);
      om_write_launch(pyr, m->states.ptr, w.pyr_codes.ptr, w.pyr_counts.ptr, m->data.ptr, 2ull * inner, w.counters.ptr, s->stream);
      s->launches += 1;
    }
    unsigned long long ctr[OM_CTR_COUNT] = {};
    B200_CUDA(cudaMemcpyAsync(ctr, w.counters.ptr, sizeof(ctr), cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));  // the host table goes out of scope; the counts are read
    if (ctr[SM_CTR_TRIPPED] || ctr[OM_CTR_INNER] != inner)
      return sm_fail(s, B200REG_ERR_CUDA, "build_octomap: a voxel outside the box or beyond the rank index, or a node beyond the data");
    b200sm_octomap_info& I = m->info;
    for (int a = 0; a < 3; a++) {
      I.box_origin[a] = box.lo[a];
      I.box_dims[a] = box.dims[a];
    }
    I.n_rays = ctr[SM_CTR_RAYS];
    I.n_skipped = ctr[SM_CTR_SKIPPED];
    I.n_occupied_voxels = ctr[OM_CTR_OCCUPIED_VOXELS];
    I.n_dynamic_voxels = ctr[SM_CTR_DYNAMIC];
    I.n_free_voxels = ctr[OM_CTR_FREE_VOXELS];
    I.n_inner_nodes = inner;
    I.n_occupied_leaves = ctr[OM_CTR_OCCUPIED_LEAVES];
    I.n_free_leaves = ctr[OM_CTR_FREE_LEAVES];
    I.tree_size = I.n_inner_nodes + I.n_occupied_leaves + I.n_free_leaves;
    m->header = om_header(I.tree_size, p.resolution);
    I.n_bytes = m->header.size() + 2ull * inner;
    I.n_batches = f.batches;
    if (info) *info = I;
    s->om = std::move(m);
    return (int)B200REG_OK;
  });
}

int b200sm_get_octomap_states(b200sm_t s, unsigned char* states, size_t capacity, size_t* n) {
  if (!s || (!states && capacity)) return B200REG_ERR_ARG;
  if (!s->om) return sm_fail(s, B200REG_ERR_ARG, "get_octomap_states: no build yet");
  return sm_guarded(s, [&]() {
    const OctoMapBuild& m = *s->om;
    const size_t cells = (size_t)m.info.box_dims[0] * m.info.box_dims[1] * m.info.box_dims[2];
    if (n) *n = cells;
    const size_t k = std::min(capacity, cells);
    if (k) {
      get_if(s, states, m.states.ptr, k);
      B200_CUDA(cudaStreamSynchronize(s->stream));
    }
    return (int)B200REG_OK;
  });
}

int b200sm_get_octomap_bt(b200sm_t s, unsigned char* bytes, size_t capacity, size_t* n_bytes) {
  if (!s || (!bytes && capacity)) return B200REG_ERR_ARG;
  if (!s->om) return sm_fail(s, B200REG_ERR_ARG, "get_octomap_bt: no build yet");
  return sm_guarded(s, [&]() {
    const OctoMapBuild& m = *s->om;
    const size_t head = m.header.size(), data = 2 * (size_t)m.info.n_inner_nodes;
    if (n_bytes) *n_bytes = head + data;
    if (capacity) std::memcpy(bytes, m.header.data(), std::min(capacity, head));
    const size_t k = capacity > head ? std::min(capacity - head, data) : 0;
    if (k) {
      get_if(s, bytes + head, m.data.ptr, k);
      B200_CUDA(cudaStreamSynchronize(s->stream));
    }
    return (int)B200REG_OK;
  });
}

int b200sm_save_octomap_bt(b200sm_t s, const char* path, size_t* n_bytes) {
  if (!s || !path) return B200REG_ERR_ARG;
  if (!s->om) return sm_fail(s, B200REG_ERR_ARG, "save_octomap_bt: no build yet");
  const OctoMapBuild& m = *s->om;
  if (m.info.tree_size == 0) return sm_fail(s, B200REG_ERR_ARG, "save_octomap_bt: the tree is empty");
  return sm_guarded(s, [&]() {
    const size_t data = 2 * (size_t)m.info.n_inner_nodes, n = (data + OM_BT_PIECE - 1) / OM_BT_PIECE;
    if (n_bytes) *n_bytes = m.header.size() + data;
    FILE* fp = std::fopen(path, "wb");
    if (!fp) {
      s->err = std::string("save_octomap_bt: cannot open ") + path + ": " + std::strerror(errno);
      return (int)B200REG_ERR_IO;
    }
    auto count = [&](size_t piece) { return std::min(OM_BT_PIECE, data - piece * OM_BT_PIECE); };
    auto enqueue = [&](size_t piece, char* buf) {
      B200_CUDA(cudaMemcpyAsync(buf, m.data.ptr + piece * OM_BT_PIECE, count(piece), cudaMemcpyDeviceToHost, s->stream));
    };
    auto write = [&](size_t piece, const char* buf) {
      bool ok = piece > 0 || std::fwrite(m.header.data(), 1, m.header.size(), fp) == m.header.size();
      ok = ok && std::fwrite(buf, 1, count(piece), fp) == count(piece);
      if (ok && piece + 1 == n) {
        ok = std::fclose(fp) == 0;
        fp = nullptr;
      }
      if (ok) return (int)B200REG_OK;
      s->err = std::string("save_octomap_bt: writing ") + path + ": " + std::strerror(errno);
      return (int)B200REG_ERR_IO;
    };
    return write_staged(s, n, OM_BT_PIECE, fp, enqueue, write);
  });
}

}  // extern "C"

// ---- map consistency: per-point neighbourhood entropy and plane variance (csrc/map_consistency.hpp, csrc/consistency.cu) ----
namespace {

McParams mc_params_from(const b200sm_map_consistency_params* p) {
  McParams q;
  if (p) {
    q.radius = p->radius;
    q.min_neighbors = p->min_neighbors;
    q.query_stride = p->query_stride;
  }
  return q;
}

// refused after the poses are checked and before the tiles are laid out
const char* mc_too_many_points(b200sm_t s) { return map_points(s) > MC_MAX_POINTS ? "a map of 2^31 points or more" : nullptr; }

}  // namespace

extern "C" {

int b200sm_build_map_consistency(b200sm_t s, const double* poses_colmajor16, const b200sm_map_consistency_params* params,
                                 b200sm_map_consistency_info* info) {
  if (!s) return B200REG_ERR_ARG;
  const McParams p = mc_params_from(params);
  McConst c;
  if (const char* why = mc_prepare(p, &c)) return sm_fail(s, B200REG_ERR_ARG, (std::string("build_map_consistency: ") + why).c_str());
  // the entries of the submaps with points, in submap order, every submap's first map index and its double pose
  const size_t n_sub = s->submaps.size();
  SubmapTiles t;
  std::vector<McEntry> table;
  std::vector<unsigned> sub_first(n_sub);
  std::vector<double> poses(16 * n_sub);
  unsigned long long at = 0;
  const int rc = map_prologue(s, "build_map_consistency", poses_colmajor16, MC_TILE, mc_too_many_points, &t, &table,
                              [&](size_t k, McEntry& e) {
                                const Submap& sub = *s->submaps[k];
                                for (int r = 0; r < 4; r++)
                                  for (int col = 0; col < 4; col++)
                                    poses[16 * k + col * 4 + r] =
                                        poses_colmajor16 ? poses_colmajor16[16 * k + col * 4 + r] : sub.pose[r * 4 + col];
                                sub_first[k] = (unsigned)at;
                                e.map_offset = (unsigned)at;
                                at += e.n;
                                return (int)B200REG_OK;
                              });
  if (rc != B200REG_OK) return rc;
  const unsigned long long total = at;
  const int n_entries = (int)table.size();
  const unsigned tiles = (unsigned)t.tiles;
  return sm_guarded(s, [&]() {
    MapWorkspace& w = s->work;
    // K19a; the refusals it decides come before anything is sized
    std::vector<int> bounds;
    unsigned long long ctr[MC_CTR_COUNT] = {};
    int lo[3], hi[3];
    bounds_pass<3>(s, mc_bounds_launch, c, table, tiles, w.mc_table, bounds, MC_CTR_COUNT, ctr, MC_CTR_COUNT, lo, hi);
    if (ctr[MC_CTR_RANGE])
      return sm_fail(s, B200REG_ERR_ARG, "build_map_consistency: a point's fixed-point coordinate is 2^46 or more in magnitude");
    const unsigned long long used = total - ctr[MC_CTR_SKIPPED];
    SmBox box{};
    unsigned long long cells = 0;
    if (used) {
      const int rc = box_or_refuse(s, "build_map_consistency", "a box", "cells", lo, hi, 0, &box, &cells);
      if (rc != B200REG_OK) return rc;
    }
    // the new build is made beside the last one, which stays until this one succeeds
    auto m = std::make_unique<MapConsistency>();
    m->c = c;
    m->poses = std::move(poses);
    const size_t np = std::max<size_t>((size_t)total, 1);
    m->n.ensure(np);
    m->h.ensure(np);
    m->plane.ensure(np);
    m->rows.ensure(MC_ROW_COUNT * n_sub);
    m->sub_first.ensure(n_sub);
    B200_CUDA(cudaMemsetAsync(m->rows.ptr, 0, MC_ROW_COUNT * n_sub * sizeof(unsigned long long), s->stream));
    B200_CUDA(cudaMemcpyAsync(m->sub_first.ptr, sub_first.data(), n_sub * sizeof(unsigned), cudaMemcpyHostToDevice, s->stream));
    const unsigned long long n_words = (cells + 31) / 32;
    unsigned n_cells = 0, n_chunks = 0;
    if (used) {
      // K19b: the occupied cells' rank index, their counts, the chunks of K19c, and the points in cell order
      n_cells = rank_pass(s, m->index, n_words, [&](RankWord* idx) {
        mc_mark_launch(w.mc_table.ptr, n_entries, tiles, c, box, idx, w.counters.ptr, s->stream);
      });
      const size_t nc = (size_t)n_cells + 1;
      m->start.ensure(nc);
      m->queries.ensure(nc);
      m->chunks.ensure(nc);
      m->qcursor.ensure(nc);
      m->ocursor.ensure(nc);
      m->ijk.ensure(3 * nc);
      B200_CUDA(cudaMemsetAsync(m->start.ptr, 0, nc * sizeof(unsigned), s->stream));
      B200_CUDA(cudaMemsetAsync(m->queries.ptr, 0, nc * sizeof(unsigned), s->stream));
      B200_CUDA(cudaMemsetAsync(m->qcursor.ptr, 0, nc * sizeof(unsigned), s->stream));
      B200_CUDA(cudaMemsetAsync(m->ocursor.ptr, 0, nc * sizeof(unsigned), s->stream));
      mc_count_launch(w.mc_table.ptr, n_entries, tiles, c, box, m->index.ptr, m->start.ptr, m->queries.ptr, s->stream);
      counter_scan_async(m->start.ptr, n_cells, w.scan_tmp, s->stream);
      mc_chunks_launch(m->queries.ptr, n_cells, m->chunks.ptr, s->stream);
      counter_scan_async(m->chunks.ptr, n_cells, w.scan_tmp, s->stream);
      sm_voxel_list_launch(m->index.ptr, n_words, box, n_cells, m->ijk.ptr, s->stream);
      s->launches += 9;
      B200_CUDA(cudaMemcpyAsync(&n_chunks, m->chunks.ptr + n_cells, sizeof(unsigned), cudaMemcpyDeviceToHost, s->stream));
      w.cell_offs.ensure((size_t)used);
      w.cell_idx.ensure((size_t)used);
    }
    // the scatter also resets every point's layers, skipped ones included
    mc_scatter_launch(w.mc_table.ptr, n_entries, tiles, c, box, m->index.ptr, m->start.ptr, m->queries.ptr, m->qcursor.ptr,
                      m->ocursor.ptr, w.cell_offs.ptr, w.cell_idx.ptr, m->n.ptr, m->h.ptr, m->plane.ptr, w.counters.ptr, s->stream);
    s->launches += tiles ? 1 : 0;
    B200_CUDA(cudaStreamSynchronize(s->stream));  // n_chunks
    // K19c + K19d
    mc_neighbour_launch(m->chunks.ptr, n_chunks, n_cells, m->start.ptr, m->queries.ptr, m->ijk.ptr, box, m->index.ptr, w.cell_offs.ptr,
                        w.cell_idx.ptr, m->sub_first.ptr, (int)n_sub, c, m->n.ptr, m->h.ptr, m->plane.ptr, m->rows.ptr, w.counters.ptr,
                        s->stream);
    s->launches += n_chunks ? 1 : 0;
    std::vector<unsigned long long> rows(MC_ROW_COUNT * n_sub);
    B200_CUDA(cudaMemcpyAsync(rows.data(), m->rows.ptr, rows.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaMemcpyAsync(ctr, w.counters.ptr, sizeof(ctr), cudaMemcpyDeviceToHost, s->stream));
    B200_CUDA(cudaStreamSynchronize(s->stream));
    if (ctr[MC_CTR_TRIPPED]) return sm_fail(s, B200REG_ERR_CUDA, "build_map_consistency: a cell outside the box or a slot beyond its cell");
    b200sm_map_consistency_info& I = m->info;
    for (int a = 0; a < 3; a++) {
      I.box_origin[a] = box.lo[a];
      I.box_dims[a] = box.dims[a];
    }
    I.n_points = total;
    I.n_skipped = ctr[MC_CTR_SKIPPED];
    I.n_cells = n_cells;
    I.n_candidates = ctr[MC_CTR_CANDIDATES];
    m->sub_rows.resize(n_sub);
    for (size_t k = 0; k < n_sub; k++) {
      const unsigned long long* row = &rows[MC_ROW_COUNT * k];
      b200sm_submap_consistency& R = m->sub_rows[k];
      R.n_points = s->submaps[k]->n;
      R.n_queries = row[MC_ROW_QUERIES];
      R.n_valid = row[MC_ROW_VALID];
      R.n_neighbors = row[MC_ROW_NEIGHBORS];
      R.sum_h_q = (long long)row[MC_ROW_SUM_H];
      R.sum_plane_q = (long long)row[MC_ROW_SUM_PLANE];
      R.mme = mc_mme(R.sum_h_q, R.n_valid);
      R.mpv = mc_mpv(c, R.sum_plane_q, R.n_valid);
      I.n_queries += R.n_queries;
      I.n_valid += R.n_valid;
      I.n_neighbors += R.n_neighbors;
      I.sum_h_q += R.sum_h_q;
      I.sum_plane_q += R.sum_plane_q;
    }
    I.mme = mc_mme(I.sum_h_q, I.n_valid);
    I.mpv = mc_mpv(c, I.sum_plane_q, I.n_valid);
    if (info) *info = I;
    s->mc = std::move(m);
    return (int)B200REG_OK;
  });
}

int b200sm_get_map_consistency(b200sm_t s, unsigned* n, double* h, double* plane_var, size_t capacity) {
  if (!s) return B200REG_ERR_ARG;
  if (!s->mc) return sm_fail(s, B200REG_ERR_ARG, "get_map_consistency: no build yet");
  return sm_guarded(s, [&]() {
    const MapConsistency& m = *s->mc;
    const size_t k = std::min(capacity, (size_t)m.info.n_points);
    if (k) {
      get_if(s, n, m.n.ptr, k);
      get_if(s, h, m.h.ptr, k);
      get_if(s, plane_var, m.plane.ptr, k);
      B200_CUDA(cudaStreamSynchronize(s->stream));
    }
    return (int)B200REG_OK;
  });
}

int b200sm_get_submap_consistency(b200sm_t s, b200sm_submap_consistency* rows, size_t capacity) {
  if (!s || (!rows && capacity)) return B200REG_ERR_ARG;
  if (!s->mc) return sm_fail(s, B200REG_ERR_ARG, "get_submap_consistency: no build yet");
  const std::vector<b200sm_submap_consistency>& r = s->mc->sub_rows;
  const size_t k = std::min(capacity, r.size());
  if (k) std::memcpy(rows, r.data(), k * sizeof(b200sm_submap_consistency));
  return B200REG_OK;
}

int b200sm_save_map_consistency_pcd_ascii(b200sm_t s, const char* path, size_t* n_points, size_t* n_bytes) {
  if (!s || !path) return B200REG_ERR_ARG;
  if (!s->mc) return sm_fail(s, B200REG_ERR_ARG, "save_map_consistency_pcd_ascii: no build yet");
  const MapConsistency& m = *s->mc;
  const size_t total = (size_t)m.info.n_points;
  if (total == 0) return sm_fail(s, B200REG_ERR_ARG, "save_map_consistency_pcd_ascii: the map has no points");
  size_t now = 0;
  for (const auto& sub : s->submaps) now += sub->n;
  if (s->submaps.size() != m.sub_rows.size() || now != total)
    return sm_fail(s, B200REG_ERR_ARG, "save_map_consistency_pcd_ascii: the session's submaps changed since the build");
  return sm_guarded(s, [&]() {
    const int rc = assemble_on_device(s, m.poses.data(), total);
    if (rc != B200REG_OK) return rc;
    mc_intensity_launch(s->assembled.ptr, m.h.ptr, total, s->stream);
    s->launches += 1;
    return write_pcd_ascii(s, s->assembled.ptr, total, path, "save_map_consistency_pcd_ascii", n_points, n_bytes);
  });
}

}  // extern "C"
