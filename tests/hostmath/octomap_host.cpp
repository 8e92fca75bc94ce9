// TEST INFRASTRUCTURE: the OctoMap of b200sm_build_octomap (csrc/octomap.hpp) built serially on the host from the same
// header and static_map.hpp: origins, rays, the static map's occupied voxels and their per-submap counts, the freed walks,
// the box and its voxel states; then the tree the way OctoMap builds it: one pointer-based node per level for every
// known voxel inserted, a recursive prune, and a recursive pre-order write. tests/test_octomap_cpu.py compares it with
// the Python replay (tests/octomapref.py) and the GPU tests compare the session with it bit for bit.
// Build with -ffp-contract=off and, for the sanitised run (-DOM_HOST_MAIN), -fsanitize=address,undefined.
#include <algorithm>
#include <array>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../lidarslam_ros2_b200/csrc/octomap.hpp"

using namespace b200;

namespace {

// One OctoMap node: its children (none for a leaf) and, for a leaf, its state
struct Node {
  std::unique_ptr<Node> child[8];
  unsigned char state = OM_UNKNOWN;
  bool leaf() const {
    for (const auto& c : child)
      if (c) return false;
    return true;
  }
};

struct Tree {
  std::unique_ptr<Node> root;
  // insert a known voxel: one node per level on the way down, created when missing
  void insert(unsigned kx, unsigned ky, unsigned kz, unsigned char state) {
    if (!root) root.reset(new Node());
    Node* n = root.get();
    for (int l = OM_DEPTH; l >= 1; l--) {
      const int i = om_child(kx, ky, kz, l);
      if (!n->child[i]) n->child[i].reset(new Node());
      n = n->child[i].get();
    }
    n->state = state;
  }
  // OctoMap's prune: bottom-up, 8 leaf children of one state collapse into their parent
  static void prune(Node* n) {
    for (auto& c : n->child)
      if (c) prune(c.get());
    for (const auto& c : n->child)
      if (!c || !c->leaf() || c->state != n->child[0]->state) return;
    n->state = n->child[0]->state;
    for (auto& c : n->child) c.reset();
  }
  static unsigned long long count(const Node* n) {
    unsigned long long k = 1;
    for (const auto& c : n->child)
      if (c) k += count(c.get());
    return k;
  }
  // OcTree::writeBinaryNode: the two bytes of an inner node, then its inner children in order
  static void write(const Node* n, std::string& out) {
    unsigned char code[8];
    for (int i = 0; i < 8; i++) code[i] = !n->child[i] ? OM_UNKNOWN : n->child[i]->leaf() ? n->child[i]->state : OM_INNER;
    unsigned char b0, b1;
    om_pack(code, &b0, &b1);
    out.push_back((char)b0);
    out.push_back((char)b1);
    for (int i = 0; i < 8; i++)
      if (code[i] == OM_INNER) write(n->child[i].get(), out);
  }
};

struct Build {
  int lo[3] = {0, 0, 0};
  unsigned dims[3] = {0, 0, 0};
  unsigned long long n_rays = 0, n_skipped = 0, n_occ = 0, n_dyn = 0, n_free = 0, n_inner = 0, n_occ_leaves = 0, n_free_leaves = 0,
                     size = 0;
  std::vector<unsigned char> states;  // box linear order
  std::string bytes;                  // the .bt file
};
Build g_build;

// the tree and file of a labelled box; fills the node counts and bytes of *B
void encode(Build* B, double resolution) {
  Tree t;
  const unsigned W = B->dims[0], H = B->dims[1], D = B->dims[2];
  for (unsigned z = 0; z < D; z++)
    for (unsigned y = 0; y < H; y++)
      for (unsigned x = 0; x < W; x++) {
        const unsigned char s = B->states[((size_t)z * H + y) * W + x];
        if (s != OM_UNKNOWN)
          t.insert((unsigned)(B->lo[0] + OM_KEY_OFFSET) + x, (unsigned)(B->lo[1] + OM_KEY_OFFSET) + y, (unsigned)(B->lo[2] + OM_KEY_OFFSET) + z,
                   s);
      }
  std::string data;
  B->n_inner = B->n_occ_leaves = B->n_free_leaves = B->size = 0;
  if (t.root) {
    Tree::prune(t.root.get());
    Tree::write(t.root.get(), data);
    B->size = Tree::count(t.root.get());
    // leaves by state, inner nodes from the data's length
    std::vector<const Node*> stack{t.root.get()};
    while (!stack.empty()) {
      const Node* n = stack.back();
      stack.pop_back();
      if (n->leaf()) (n->state == OM_OCCUPIED ? B->n_occ_leaves : B->n_free_leaves)++;
      for (const auto& c : n->child)
        if (c) stack.push_back(c.get());
    }
    B->n_inner = data.size() / 2;
  }
  B->bytes = om_header(B->size, resolution) + data;
}

}  // namespace

extern "C" {

// params: resolution, max_range, sensor_origin x y z, ray_fraction, min_frees, dynamic_thresh (the static map's).
// points: 4 floats per row, submap k = rows offsets[k] .. offsets[k + 1]; poses: 16 doubles per submap, column-major.
// Returns 0, or -1 (parameters), -2 (an origin out of range), -3 (a box of more than 2^31 - 1 voxels), -4 (no submaps),
// -5 (a box voxel outside the 16-bit key range), -6 (a resolution printf("%g") does not give back).
int omh_build(const double* params, const float* points, const long long* offsets, const double* poses, int n_sub) {
  SmParams p;
  p.resolution = params[0];
  p.max_range = params[1];
  for (int k = 0; k < 3; k++) p.sensor_origin[k] = params[2 + k];
  p.ray_fraction = params[5];
  p.min_frees = params[6] >= 0 && params[6] <= 4294967295.0 ? (unsigned)params[6] : 0u;
  p.dynamic_thresh = params[7];
  SmConst c;
  if (sm_prepare(p, &c)) return -1;
  if (!om_resolution_exact(p.resolution)) return -6;
  if (n_sub <= 0) return -4;
  std::vector<float> T(12 * (size_t)n_sub);
  std::vector<long long> O(3 * (size_t)n_sub);
  for (int k = 0; k < n_sub; k++) {
    og_pose_f(poses + 16 * (size_t)k, &T[12 * (size_t)k]);
    if (!sm_origin(c, p, &T[12 * (size_t)k], &O[3 * (size_t)k])) return -2;
  }
  // rays; the endpoint box; the OctoMap box (endpoints and the origins of submaps with a ray)
  const size_t n = (size_t)offsets[n_sub];
  std::vector<unsigned char> is_ray(n);
  std::vector<int> vox(3 * n);
  std::vector<long long> end(3 * n);
  int elo[3] = {INT_MAX, INT_MAX, INT_MAX}, ehi[3] = {INT_MIN, INT_MIN, INT_MIN};
  int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
  unsigned long long rays = 0, skipped = 0;
  for (int k = 0; k < n_sub; k++) {
    bool any = false;
    for (long long i = offsets[k]; i < offsets[k + 1]; i++) {
      float e[3];
      og_transform(&T[12 * (size_t)k], points[4 * i], points[4 * i + 1], points[4 * i + 2], e);
      int* v = &vox[3 * i];
      long long* f = &end[3 * i];
      if (!sm_ray(c, &O[3 * (size_t)k], e[0], e[1], e[2], &v[0], &v[1], &v[2], &f[0], &f[1], &f[2])) {
        skipped++;
        continue;
      }
      is_ray[i] = 1;
      rays++;
      any = true;
      for (int a = 0; a < 3; a++) {
        elo[a] = std::min(elo[a], v[a]);
        ehi[a] = std::max(ehi[a], v[a]);
      }
    }
    if (any)
      for (int a = 0; a < 3; a++) {
        const int o = og_cell(O[3 * (size_t)k + a]);
        lo[a] = std::min(lo[a], o);
        hi[a] = std::max(hi[a], o);
      }
  }
  Build& B = g_build;
  B = Build();
  B.n_rays = rays;
  B.n_skipped = skipped;
  if (!rays) {
    encode(&B, p.resolution);
    return 0;
  }
  for (int a = 0; a < 3; a++) {
    lo[a] = std::min(lo[a], elo[a]);
    hi[a] = std::max(hi[a], ehi[a]);
  }
  unsigned long long cells = 0;
  unsigned edims[3];
  unsigned long long ecells;
  if (!sm_box(elo, ehi, edims, &ecells) || !sm_box(lo, hi, B.dims, &cells)) return -3;
  if (om_box(lo, hi, B.dims, &cells)) return -5;
  for (int a = 0; a < 3; a++) B.lo[a] = lo[a];
  auto lin_of = [&](int x, int y, int z) {
    return (size_t)((((long long)z - lo[2]) * B.dims[1] + ((long long)y - lo[1])) * B.dims[0] + ((long long)x - lo[0]));
  };
  // the static map's occupied voxels (ordered by their voxel) and per-submap hit-wins counts, and the freed walks
  std::map<std::array<int, 3>, unsigned> rank;
  for (size_t i = 0; i < n; i++)
    if (is_ray[i]) rank.emplace(std::array<int, 3>{vox[3 * i + 2], vox[3 * i + 1], vox[3 * i]}, 0u);
  unsigned r0 = 0;
  for (auto& kv : rank) kv.second = r0++;
  std::vector<uint32_t> hits(rank.size()), frees(rank.size());
  std::vector<unsigned char> hit(rank.size()), fre(rank.size()), freed((size_t)cells);
  for (int k = 0; k < n_sub; k++) {
    std::fill(hit.begin(), hit.end(), 0);
    std::fill(fre.begin(), fre.end(), 0);
    const long long* o = &O[3 * (size_t)k];
    for (long long i = offsets[k]; i < offsets[k + 1]; i++) {
      if (!is_ray[i]) continue;
      hit[rank.at({vox[3 * i + 2], vox[3 * i + 1], vox[3 * i]})] = 1;
      const long long* f = &end[3 * i];
      sm_walk(o[0], o[1], o[2], f[0], f[1], f[2], [&](int x, int y, int z) {
        if (x < lo[0] || x > hi[0] || y < lo[1] || y > hi[1] || z < lo[2] || z > hi[2]) std::abort();  // the box holds every walk
        freed[lin_of(x, y, z)] = 1;
        auto it = rank.find({z, y, x});
        if (it != rank.end()) fre[it->second] = 1;
      });
    }
    for (size_t v = 0; v < rank.size(); v++) {
      if (hit[v]) hits[v]++;
      else if (fre[v]) frees[v]++;
    }
  }
  B.states.assign((size_t)cells, OM_UNKNOWN);
  for (size_t i = 0; i < (size_t)cells; i++) B.states[i] = om_state(false, false, freed[i]);
  for (const auto& kv : rank) {
    const bool dyn = sm_dynamic(hits[kv.second], frees[kv.second], c.min_frees, c.dyn_value);
    B.n_dyn += dyn;
    B.states[lin_of(kv.first[2], kv.first[1], kv.first[0])] = om_state(true, dyn, false);
  }
  for (unsigned char s : B.states) {
    B.n_occ += s == OM_OCCUPIED;
    B.n_free += s == OM_FREE;
  }
  encode(&B, p.resolution);
  return 0;
}

// lo x y z, W, H, D, n_rays, n_skipped, n_occupied, n_dynamic, n_free, n_inner, n_occupied_leaves, n_free_leaves, size,
// n_bytes
void omh_info(long long* info) {
  const Build& B = g_build;
  const long long v[16] = {B.lo[0],
                           B.lo[1],
                           B.lo[2],
                           B.dims[0],
                           B.dims[1],
                           B.dims[2],
                           (long long)B.n_rays,
                           (long long)B.n_skipped,
                           (long long)B.n_occ,
                           (long long)B.n_dyn,
                           (long long)B.n_free,
                           (long long)B.n_inner,
                           (long long)B.n_occ_leaves,
                           (long long)B.n_free_leaves,
                           (long long)B.size,
                           (long long)B.bytes.size()};
  std::memcpy(info, v, sizeof(v));
}

// any pointer may be NULL: the box's states (linear order) and the .bt bytes
void omh_result(unsigned char* states, unsigned char* bytes) {
  const Build& B = g_build;
  if (states && !B.states.empty()) std::memcpy(states, B.states.data(), B.states.size());
  if (bytes) std::memcpy(bytes, B.bytes.data(), B.bytes.size());
}

// The tree alone: the .bt bytes of a labelled box (lo, dims, states in linear order) into out (cap bytes); returns the
// file's size, the node counts in info[0..3] (inner, occupied leaves, free leaves, size)
long long omh_encode(const int* lo, const unsigned* dims, const unsigned char* states, double resolution, unsigned char* out, long long cap,
                     long long* info) {
  Build B;
  for (int a = 0; a < 3; a++) {
    B.lo[a] = lo[a];
    B.dims[a] = dims[a];
  }
  B.states.assign(states, states + (size_t)dims[0] * dims[1] * dims[2]);
  encode(&B, resolution);
  std::memcpy(out, B.bytes.data(), std::min<size_t>(B.bytes.size(), (size_t)cap));
  info[0] = (long long)B.n_inner;
  info[1] = (long long)B.n_occ_leaves;
  info[2] = (long long)B.n_free_leaves;
  info[3] = (long long)B.size;
  return (long long)B.bytes.size();
}

// the box check alone: 0 when lo .. hi is accepted, -3 more than 2^31 - 1 voxels, -5 outside the key range
int omh_box(const int* lo, const int* hi) {
  unsigned dims[3];
  unsigned long long cells;
  if (!sm_box(lo, hi, dims, &cells)) return -3;
  return om_box(lo, hi, dims, &cells) ? -5 : 0;
}

int omh_resolution_exact(double r) { return om_resolution_exact(r) ? 1 : 0; }

}  // extern "C"

#ifdef OM_HOST_MAIN
// The sanitised run: an executable (a sanitised shared object cannot be loaded into an unsanitised Python) that builds
// OctoMaps from generated submaps with non-finite rows, negative coordinates and empty submaps, and checks that the
// submaps in reverse order give the same states and bytes, that the node counts add up and that the data is two bytes
// per inner node.
#include <cmath>
#include <limits>

int main() {
  int failures = 0;
  const double params[8] = {0.25, 20.0, 0.0, 0.0, 0.3, 0.85, 2, 0.25};
  for (int trial = 0; trial < 6; trial++) {
    const int n_sub = 1 + trial * 2;
    std::vector<float> pts;
    std::vector<long long> off{0};
    std::vector<double> poses;
    uint64_t st = 0x9E3779B97F4A7C15ull * (uint64_t)(trial + 1);
    auto rnd = [&]() {
      st = st * 6364136223846793005ull + 1442695040888963407ull;
      return (double)(st >> 11) * (1.0 / 9007199254740992.0);
    };
    for (int k = 0; k < n_sub; k++) {
      const int n = (k % 3 == 2) ? 0 : 200 + 37 * k;
      for (int i = 0; i < n; i++) {
        float x = (float)(rnd() * 30 - 15), y = (float)(rnd() * 30 - 15), z = (float)(rnd() * 6 - 3);
        if (i % 41 == 7) x = std::numeric_limits<float>::quiet_NaN();
        if (i % 43 == 9) z = std::numeric_limits<float>::infinity();
        pts.insert(pts.end(), {x, y, z, (float)i});
      }
      off.push_back(off.back() + n);
      const double yaw = rnd() * 6.283185307179586, tx = rnd() * 10 - 7, ty = rnd() * 10 - 7;
      const double P[16] = {std::cos(yaw), std::sin(yaw), 0, 0, -std::sin(yaw), std::cos(yaw), 0, 0, 0, 0, 1, 0, tx, ty, 1.2, 1};
      poses.insert(poses.end(), P, P + 16);
    }
    if (omh_build(params, pts.data(), off.data(), poses.data(), n_sub) != 0) {
      failures++;
      continue;
    }
    const Build first = g_build;
    if (first.size != first.n_inner + first.n_occ_leaves + first.n_free_leaves || first.n_occ + first.n_free == 0) failures++;
    if (first.bytes.size() != om_header(first.size, params[0]).size() + 2 * first.n_inner) failures++;
    std::vector<float> rp;
    std::vector<long long> ro{0};
    std::vector<double> rpo;
    for (int k = n_sub - 1; k >= 0; k--) {
      rp.insert(rp.end(), pts.begin() + 4 * off[k], pts.begin() + 4 * off[k + 1]);
      ro.push_back(ro.back() + (off[k + 1] - off[k]));
      rpo.insert(rpo.end(), poses.begin() + 16 * k, poses.begin() + 16 * (k + 1));
    }
    if (omh_build(params, rp.data(), ro.data(), rpo.data(), n_sub) != 0 || g_build.states != first.states || g_build.bytes != first.bytes) {
      std::printf("MISMATCH trial=%d\n", trial);
      failures++;
    }
  }
  std::printf("octomap_host: %d failures\n", failures);
  return failures ? 1 : 0;
}
#endif
