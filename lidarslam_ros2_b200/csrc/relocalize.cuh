// Relocalisation anywhere in the prior map (b200sm_relocalize): the K17 kernels of relocalize.cu behind one host object the
// session keeps. The arithmetic and the search's steps are csrc/relocalize.hpp's; every launch is enqueued on the caller's
// stream.
#pragma once
#include <cuda_runtime.h>

#include <string>
#include <vector>

#include "engine.hpp"
#include "relocalize.hpp"

namespace b200 {

struct RlSearchInfo {
  long long m = 0, t0 = 0, t = 0;
  long long nodes[RL_MAX_LEVELS] = {};  // nodes scored per level by the expansion (level L - 1: the roots)
  std::vector<long long> tiles;          // the answer, ranked
  std::vector<unsigned long long> keys;  // the tiles' best leaf keys
  float ms = 0;                          // device time of the search's launches (CUDA events; host waits excluded)
};

class Relocalizer {
 public:
  int launches = 0;
  int builds = 0;  // pyramids built since creation
  RlGrid grid;     // of the current pyramid (W = H = 0: no map row is projected)

  void invalidate() { built_ = false; }
  // The pyramid of `map` for p's resolution, band and num_levels, built unless the current one is for the same values.
  // B200REG_ERR_ARG with `why` when a limit of rl_make_grid is exceeded (nothing is allocated past the bounds pass).
  int ensure_pyramid(const float4* map, size_t n, const RlParams& p, std::string& why, cudaStream_t s);
  // The search of the filtered scan (n points) for the rotations rot_f (9 floats per heading) at height z0. B200REG_ERR_ARG
  // with `why` when the points or a level's frontier exceed their caps. Synchronises the stream.
  int search(const float4* scan, size_t n, const std::vector<float>& rot_f, double z0, const RlParams& p, RlSearchInfo& out,
             std::string& why, cudaStream_t s);
  // level h of the pyramid: its stored width and height; min(capacity, w * h) bytes into out (may be NULL)
  int read_level(int h, unsigned char* out, size_t capacity, long long* w, long long* hh, std::string& why, cudaStream_t s);
  // score_h of `count` nodes (k, i, j triples) with the last search's offsets
  int score_nodes(int h, long long count, const int* kij, int* scores, std::string& why, cudaStream_t s);

 private:
  bool built_ = false;
  RlParams built_for_;
  std::vector<unsigned long long> level_off_;
  DeviceBuffer<unsigned char> pyr_;
  DeviceBuffer<int> box_;
  DeviceBuffer<unsigned long long> ctr_;  // [0] projected rows / children total
  DeviceBuffer<unsigned> flags_, scan_tmp_, counts_, tripped_;
  DeviceBuffer<float4> pts_;
  DeviceBuffer<float> rot_;
  DeviceBuffer<RlOff> offs_;
  long long m_ = -1;  // points of the last search's offsets (-1: none)
  int yaw_ = 0;
  DeviceBuffer<unsigned long long> keys_;
  DeviceBuffer<RlNode> front_[2], starts_;
  DeviceBuffer<long long> dive_scores_;
  // scores kept between a level's count and write passes (4 bytes a node): the roots' (when at most 2^26), and those of
  // front_[c] in node_scores_[c]
  DeviceBuffer<int> node_scores_[2], root_scores_;
};

}  // namespace b200
