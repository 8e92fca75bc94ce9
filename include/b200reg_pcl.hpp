// b200reg_pcl.hpp — C++ adapter over the C-ABI (b200reg.h) with the method names of pcl::Registration /
// pclomp::NormalDistributionsTransform / pclomp::GeneralizedIterativeClosestPoint, so that the two lidarslam_ros2 nodes
// change one `new` expression each (scanmatcher/src/scanmatcher_component.cpp:105-106,116-117;
// graph_based_slam/src/graph_based_slam_component.cpp:64-65,74-75). See INTEGRATION.md.
//
//  * With -DB200REG_WITH_PCL (a ROS 2 box with PCL >= 1.12) the classes derive from
//    pcl::Registration<PointSource, PointTarget>: the nodes keep holding them through
//    `boost::shared_ptr<pcl::Registration<pcl::PointXYZI, pcl::PointXYZI>> registration_`
//    (scanmatcher_component.h:93, graph_based_slam_component.h:106) and call the base-class API unchanged; the virtual
//    hook computeTransformation(output, guess) (ndt_omp.h:257-268, gicp_omp.h:332-333) forwards to b200reg_align().
//  * Without it (this repository's image has no PCL/Eigen) the same classes compile stand-alone over a minimal cloud type
//    with identical method names, which is what tests/cpp/adapter_smoke.cpp exercises.
// Header-only; link with -lb200reg. Matrices are column-major float[16] == Eigen::Matrix4f::data().
#pragma once
#include <algorithm>
#include <array>
#include <cfloat>
#include <cstdio>
#include <limits>
#include <cstddef>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "b200reg.h"

#ifdef B200REG_WITH_PCL
#include <pcl/point_cloud.h>
#include <pcl/point_types.h>
#include <pcl/registration/registration.h>
#endif

namespace b200reg {

using Matrix4f = std::array<float, 16>;  // column-major, like Eigen::Matrix4f::data()
inline Matrix4f Identity() { return {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1}; }

// pclomp::NeighborSearchMethod (ndt_omp.h:52-57)
enum NeighborSearchMethod { KDTREE = B200REG_KDTREE, DIRECT26 = B200REG_DIRECT26, DIRECT7 = B200REG_DIRECT7, DIRECT1 = B200REG_DIRECT1 };

// RAII owner of a C-ABI handle
class Handle {
 public:
  Handle(int kind, int device) {
    if (b200reg_create(kind, device, &h_) != B200REG_OK)
      throw std::runtime_error("b200reg_create failed: no CUDA device (the engine has no CPU fallback)");
  }
  ~Handle() { b200reg_destroy(h_); }
  Handle(const Handle&) = delete;
  Handle& operator=(const Handle&) = delete;
  b200reg_t get() const { return h_; }

 private:
  b200reg_t h_ = nullptr;
};

#ifndef B200REG_WITH_PCL
// Minimal stand-in for pcl::PointXYZI / pcl::PointCloud (same 32-byte layout: x y z 1 | intensity pad pad pad)
struct alignas(16) PointXYZI {
  float x = 0, y = 0, z = 0, w = 1.0f;
  float intensity = 0, pad[3] = {0, 0, 0};
};
struct PointCloud {
  std::vector<PointXYZI> points;
  std::size_t size() const { return points.size(); }
  bool empty() const { return points.empty(); }
};

// pcl::Registration-shaped base: the surface the nodes exercise (SURVEY.md §8b)
class Registration {
 public:
  virtual ~Registration() = default;
  void setInputTarget(const PointCloud& cloud) {  // Registration::setInputTarget; empty clouds are ignored like PCL
    if (cloud.empty()) return;
    check(b200reg_set_input_target(h_.get(), &cloud.points[0].x, cloud.size(), sizeof(PointXYZI)));
  }
  void setInputSource(const PointCloud& cloud) {
    if (cloud.empty()) return;
    n_source_ = cloud.size();
    check(b200reg_set_input_source(h_.get(), &cloud.points[0].x, cloud.size(), sizeof(PointXYZI)));
  }
  void setTransformationEpsilon(double eps) { check(b200reg_set_transformation_epsilon(h_.get(), eps)); }
  void setMaximumIterations(int n) { check(b200reg_set_maximum_iterations(h_.get(), n)); }
  void setMaxCorrespondenceDistance(double d) { check(b200reg_set_max_correspondence_distance(h_.get(), d)); }
  void setEuclideanFitnessEpsilon(double e) { check(b200reg_set_euclidean_fitness_epsilon(h_.get(), e)); }
  void setRANSACIterations(int n) { check(b200reg_set_ransac_iterations(h_.get(), n)); }
  // align(output [, guess]): output receives the transformed source, like pcl::Registration::align
  void align(PointCloud& output, const Matrix4f& guess = Identity()) {
    int rc = b200reg_align(h_.get(), guess.data(), final_.data());
    if (rc != B200REG_OK && rc != B200REG_ERR_NO_TARGET && rc != B200REG_ERR_NO_SOURCE) check(rc);
    output.points.resize(n_source_);
    if (rc == B200REG_OK && n_source_) check(b200reg_get_aligned(h_.get(), &output.points[0].x, sizeof(PointXYZI)));
  }
  // setInputTarget(cloud) of loadPCDFile(path, cloud), the file parsed on the device (b200reg_set_input_target_pcd);
  // throws on a file the reader refuses, keeping the previous target. Returns the number of points.
  size_t setInputTargetPCD(const std::string& path) {
    size_t n = 0;
    check(b200reg_set_input_target_pcd(h_.get(), path.c_str(), &n));
    return n;
  }
  Matrix4f getFinalTransformation() const { return final_; }
  bool hasConverged() const {
    int c = 0;
    b200reg_has_converged(h_.get(), &c);
    return c != 0;
  }
  b200reg_t handle() const { return h_.get(); }  // for ScanMatcherSession
  double getFitnessScore(double max_range = DBL_MAX) {
    double v = DBL_MAX;
    check(b200reg_get_fitness_score(h_.get(), max_range, &v));
    return v;
  }

 protected:
  Registration(int kind, int device) : h_(kind, device) {}
  void check(int rc) const {
    if (rc != B200REG_OK) throw std::runtime_error(std::string("b200reg: ") + b200reg_last_error(h_.get()));
  }
  Handle h_;
  Matrix4f final_ = Identity();
  std::size_t n_source_ = 0;
};

class NormalDistributionsTransform : public Registration {
 public:
  explicit NormalDistributionsTransform(int device = 0) : Registration(B200REG_NDT, device) {}
  void setResolution(float r) { check(b200reg_ndt_set_resolution(h_.get(), r)); }
  void setStepSize(double s) { check(b200reg_ndt_set_step_size(h_.get(), s)); }
  void setOulierRatio(double r) { check(b200reg_ndt_set_outlier_ratio(h_.get(), r)); }  // sic, ndt_omp.h:180
  void setNeighborhoodSearchMethod(NeighborSearchMethod m) { check(b200reg_ndt_set_neighborhood_search_method(h_.get(), m)); }
  void setNumThreads(int n) { check(b200reg_ndt_set_num_threads(h_.get(), n)); }
  double getTransformationProbability() const {
    double v = 0;
    b200reg_ndt_get_transformation_probability(h_.get(), &v);
    return v;
  }
  int getFinalNumIteration() const {
    int v = 0;
    b200reg_ndt_get_final_num_iteration(h_.get(), &v);
    return v;
  }
  // NDT score of the current source at poses.size() / 16 poses (column-major 4x4 each) against the current target, in one
  // launch (b200reg_ndt_score_poses); scores and hits get one entry per pose
  void scorePoses(const std::vector<float>& poses, std::vector<double>& scores, std::vector<long long>& hits) {
    scores.resize(poses.size() / 16);
    hits.resize(scores.size());
    check(b200reg_ndt_score_poses(h_.get(), (int)scores.size(), poses.data(), scores.data(), hits.data()));
  }
};

class GeneralizedIterativeClosestPoint : public Registration {
 public:
  explicit GeneralizedIterativeClosestPoint(int device = 0) : Registration(B200REG_GICP, device) {}
  void setRotationEpsilon(double e) { check(b200reg_gicp_set_rotation_epsilon(h_.get(), e)); }
  void setCorrespondenceRandomness(int k) { check(b200reg_gicp_set_correspondence_randomness(h_.get(), k)); }
  void setMaximumOptimizerIterations(int n) { check(b200reg_gicp_set_maximum_optimizer_iterations(h_.get(), n)); }
};

#else  // ---------------------------------------------------------------------------------- B200REG_WITH_PCL

// Drop-in for pclomp::NormalDistributionsTransform<PointSource, PointTarget>: derives from pcl::Registration, so
// `registration_ = ndt;` (scanmatcher_component.cpp:113, graph_based_slam_component.cpp:72) keeps compiling.
template <typename PointSource, typename PointTarget>
class RegistrationBase : public pcl::Registration<PointSource, PointTarget> {
 protected:
  using Base = pcl::Registration<PointSource, PointTarget>;
  using typename Base::PointCloudSource;
  using typename Base::PointCloudTargetConstPtr;
  using typename Base::PointCloudSourceConstPtr;
  RegistrationBase(int kind, int device) : h_(kind, device) {}

 public:
  // pcl::Registration::setInputTarget arms target_cloud_updated_, and the next align() -> initCompute() then builds a
  // FLANN kd-tree over the WHOLE target on the host (hundreds of milliseconds for a 1 M-point map) that neither engine
  // here ever queries. So the target is stored WITHOUT arming that rebuild; the cloud goes to the GPU instead.
  // setKeepHostSearchTree(true) restores PCL's behaviour for callers that need PCL's own (non-virtual, host-side)
  // getFitnessScore through a base-class pointer.
  void setInputTarget(const PointCloudTargetConstPtr& cloud) override {
    if (!cloud || cloud->points.empty()) {
      PCL_ERROR_B200("[b200reg::setInputTarget] invalid or empty point cloud given, ignored");
      return;
    }
    if (keep_host_tree_) {
      Base::setInputTarget(cloud);
    } else {
      this->target_ = cloud;
      this->target_cloud_updated_ = false;  // (PCL constructs it `true`: even the first align() would build the tree)
    }
    target_ok_ = report(b200reg_set_input_target(h_.get(), &cloud->points[0].x, cloud->size(), sizeof(PointTarget)), "setInputTarget");
  }
  void setInputSource(const PointCloudSourceConstPtr& cloud) override {
    Base::setInputSource(cloud);
    if (!cloud || cloud->points.empty()) {
      source_ok_ = false;
      return;
    }
    source_ok_ = report(b200reg_set_input_source(h_.get(), &cloud->points[0].x, cloud->size(), sizeof(PointSource)), "setInputSource");
  }
  // setInputTarget(cloud) of loadPCDFile(path, cloud) with the file parsed on the device (b200reg_set_input_target_pcd):
  // no host copy of the map exists, so PCL's own target_ is an empty cloud (align() only needs it to be set). On a file
  // the reader refuses the error is reported, the previous target stays, and 0 is returned.
  size_t setInputTargetPCD(const std::string& path) {
    size_t n = 0;
    if (!report(b200reg_set_input_target_pcd(h_.get(), path.c_str(), &n), "setInputTargetPCD")) return 0;
    this->target_.reset(new pcl::PointCloud<PointTarget>());
    this->target_cloud_updated_ = false;
    target_ok_ = true;
    return n;
  }
  void setKeepHostSearchTree(bool keep) { keep_host_tree_ = keep; }
  // align() fills `output` with the transformed source (a device-to-host copy of the whole scan per call). Both nodes
  // discard it (scanmatcher_component.cpp:350-358, graph_based_slam_component.cpp:229-231), so it is off by default:
  // `output` then keeps PCL's pre-filled copy of the input. Switch it on for callers that read the aligned cloud.
  void setComputeOutputCloud(bool on) { compute_output_ = on; }
  b200reg_t handle() const { return h_.get(); }  // for ScanMatcherSession
  // getFitnessScore on the GPU (exact 1-NN). pcl::Registration::getFitnessScore is NOT virtual: call this through the
  // concrete type, or through b200reg::getFitnessScore(registration_) below (INTEGRATION.md, gbs.cpp:231, sm.cpp:376).
  double getFitnessScore(double max_range = std::numeric_limits<double>::max()) {
    double v = std::numeric_limits<double>::max();
    report(b200reg_get_fitness_score(h_.get(), max_range, &v), "getFitnessScore");
    return v;
  }
  const char* lastError() const { return b200reg_last_error(h_.get()); }

 protected:
  // the virtual hook pcl::Registration::align() calls (ndt_omp.h:257-268, gicp_omp.h:332-333)
  void computeTransformation(PointCloudSource& output, const Eigen::Matrix4f& guess) override {
    this->converged_ = false;
    if (!target_ok_ || !source_ok_) {  // a failed upload must not be answered from the previous cloud
      PCL_ERROR_B200("[b200reg::align] the last setInputTarget / setInputSource failed; not aligning against stale data");
      return;
    }
    report(b200reg_set_transformation_epsilon(h_.get(), this->transformation_epsilon_), "setTransformationEpsilon");
    report(b200reg_set_maximum_iterations(h_.get(), this->max_iterations_), "setMaximumIterations");
    report(b200reg_set_max_correspondence_distance(h_.get(), this->corr_dist_threshold_), "setMaxCorrespondenceDistance");
    Eigen::Matrix4f final_t = Eigen::Matrix4f::Identity();
    const int rc = b200reg_align(h_.get(), guess.data(), final_t.data());
    this->final_transformation_ = final_t;
    int conv = 0;
    b200reg_has_converged(h_.get(), &conv);
    this->converged_ = report(rc, "align") && conv;
    if (rc == B200REG_OK && compute_output_ && !output.empty())
      report(b200reg_get_aligned(h_.get(), &output.points[0].x, sizeof(PointSource)), "getAligned");
  }
  bool report(int rc, const char* what) const {
    if (rc == B200REG_OK) return true;
    std::fprintf(stderr, "[b200reg::%s] error %d: %s\n", what, rc, b200reg_last_error(h_.get()));
    return false;
  }
  static void PCL_ERROR_B200(const char* msg) { std::fprintf(stderr, "%s\n", msg); }
  Handle h_;
  bool keep_host_tree_ = false, compute_output_ = false;
  bool target_ok_ = false, source_ok_ = false;
};

// getFitnessScore for code that only holds the base-class pointer (graph_based_slam_component.cpp:231,
// scanmatcher_component.cpp:376): GPU path for the engines of this header, PCL's own for anything else.
template <typename PointSource, typename PointTarget>
double getFitnessScore(pcl::Registration<PointSource, PointTarget>& reg, double max_range = std::numeric_limits<double>::max()) {
  if (auto* p = dynamic_cast<RegistrationBase<PointSource, PointTarget>*>(&reg)) return p->getFitnessScore(max_range);
  return reg.getFitnessScore(max_range);
}

template <typename PointSource, typename PointTarget>
class NormalDistributionsTransform : public RegistrationBase<PointSource, PointTarget> {
  using B = RegistrationBase<PointSource, PointTarget>;

 public:
  explicit NormalDistributionsTransform(int device = 0) : B(B200REG_NDT, device) {
    this->reg_name_ = "b200reg::NormalDistributionsTransform";
    this->transformation_epsilon_ = 0.1;  // ndt_omp_impl.hpp:71-72
    this->max_iterations_ = 35;
  }
  void setResolution(float r) { this->report(b200reg_ndt_set_resolution(this->h_.get(), r), "setResolution"); }
  void setStepSize(double s) { b200reg_ndt_set_step_size(this->h_.get(), s); }
  void setOulierRatio(double r) { b200reg_ndt_set_outlier_ratio(this->h_.get(), r); }
  void setNeighborhoodSearchMethod(NeighborSearchMethod m) { b200reg_ndt_set_neighborhood_search_method(this->h_.get(), m); }
  void setNumThreads(int n) { b200reg_ndt_set_num_threads(this->h_.get(), n); }
  double getTransformationProbability() const {
    double v = 0;
    b200reg_ndt_get_transformation_probability(this->h_.get(), &v);
    return v;
  }
  int getFinalNumIteration() const {
    int v = 0;
    b200reg_ndt_get_final_num_iteration(this->h_.get(), &v);
    return v;
  }
  // b200reg_ndt_score_poses, as in the stand-alone class; false (reported on stderr) when the call is refused
  bool scorePoses(const std::vector<float>& poses, std::vector<double>& scores, std::vector<long long>& hits) {
    scores.resize(poses.size() / 16);
    hits.resize(scores.size());
    return this->report(b200reg_ndt_score_poses(this->h_.get(), (int)scores.size(), poses.data(), scores.data(), hits.data()),
                        "scorePoses");
  }
};

template <typename PointSource, typename PointTarget>
class GeneralizedIterativeClosestPoint : public RegistrationBase<PointSource, PointTarget> {
  using B = RegistrationBase<PointSource, PointTarget>;

 public:
  explicit GeneralizedIterativeClosestPoint(int device = 0) : B(B200REG_GICP, device) {
    this->reg_name_ = "b200reg::GeneralizedIterativeClosestPoint";
    this->max_iterations_ = 200;  // gicp_omp.h:117-119
    this->transformation_epsilon_ = 5e-4;
    this->corr_dist_threshold_ = 5.;
  }
  void setRotationEpsilon(double e) { b200reg_gicp_set_rotation_epsilon(this->h_.get(), e); }
  void setCorrespondenceRandomness(int k) { b200reg_gicp_set_correspondence_randomness(this->h_.get(), k); }
  void setMaximumOptimizerIterations(int n) { b200reg_gicp_set_maximum_optimizer_iterations(this->h_.get(), n); }
};

#endif  // B200REG_WITH_PCL

// pcl::io::loadPCDFile(path, cloud) for a PointXYZI cloud, the text parsed on the device (b200reg_load_pcd): x, y, z and
// intensity of every point, WIDTH * HEIGHT points as one flat row. Returns 0, or the negative B200REG_ERR_* code (PCL: -1).
template <typename Cloud>
int loadPCDFile(const std::string& path, Cloud& cloud, int device = 0) {
  size_t n = 0;
  int rc = b200reg_load_pcd(device, path.c_str(), nullptr, 0, &n);
  if (rc != B200REG_OK) return rc;
  std::vector<float> xyzi(4 * n);
  const size_t capacity = n;
  if (n && (rc = b200reg_load_pcd(device, path.c_str(), xyzi.data(), capacity, &n)) != B200REG_OK) return rc;
  n = std::min(n, capacity);  // the file may have changed between the two calls
  cloud.points.resize(n);
  for (size_t i = 0; i < n; i++) {
    cloud.points[i].x = xyzi[4 * i];
    cloud.points[i].y = xyzi[4 * i + 1];
    cloud.points[i].z = xyzi[4 * i + 2];
    cloud.points[i].intensity = xyzi[4 * i + 3];
  }
#ifdef B200REG_WITH_PCL
  cloud.width = static_cast<decltype(cloud.width)>(n);
  cloud.height = 1;
#endif
  return B200REG_OK;
}

// ---- frontend session: device-resident map maintenance (b200sm_*, include/b200reg.h) -------------------------------
// What ScanMatcherComponent keeps per node instead of targeted_cloud_ / map_array_msg_.submaps[i].cloud on the host:
// one call per frame (receiveCloud) or the individual steps (setScan / updateMap). `Reg` is any of the registration
// classes above (it only needs the C handle).
class ScanMatcherSession {
 public:
  explicit ScanMatcherSession(int device = 0) {
    b200sm_t s = nullptr;
    if (b200sm_create(device, &s) != B200REG_OK) throw std::runtime_error("b200sm_create: no CUDA device (there is no CPU fallback)");
    s_.reset(s, [](b200sm_t p) { b200sm_destroy(p); });
  }
  void setParams(float vg_size_for_input, float vg_size_for_map, int num_targeted_cloud, double trans_for_mapupdate,
                 bool use_min_max_filter = false, double scan_min_range = 0.1, double scan_max_range = 100.0) {
    check(b200sm_set_params(s_.get(), vg_size_for_input, vg_size_for_map, num_targeted_cloud, trans_for_mapupdate,
                            use_min_max_filter ? 1 : 0, scan_min_range, scan_max_range));
  }
  void setInitialPose(const double position[3], const double quat_xyzw[4]) { check(b200sm_set_initial_pose(s_.get(), position, quat_xyzw)); }
  // cloud_callback's doTransform (sm.cpp:188-199): lookupTransform(robot_frame_id_, msg->header.frame_id, stamp), applied
  // on the device to every later frame; (nullptr, nullptr) turns it off
  void setSensorTransform(const double* translation3, const double* quat_xyzw) {
    check(b200sm_set_sensor_transform(s_.get(), translation3, quat_xyzw));
  }
  // use_odom (sm.cpp:333-348): lookupTransform(odom_frame_id_, robot_frame_id_, stamp) for the next receiveCloud
  void odomNextScan(const double translation3[3], const double quat_xyzw[4]) {
    check(b200sm_odom_next_scan(s_.get(), translation3, quat_xyzw));
  }
  // points: n structs of `stride` bytes with x, y, z floats first and the intensity float at `intensity_offset` (or -1)
  // pose7 = position + quaternion (x, y, z, w); final16 column-major like Eigen::Matrix4f::data()
  bool receiveCloud(b200reg_t reg, const float* points, size_t n, size_t stride, long intensity_offset, double pose7[7], float final16[16]) {
    int updated = 0;
    check(b200sm_receive_cloud(s_.get(), reg, points, n, stride, intensity_offset, pose7, final16, &updated));
    return updated != 0;
  }
  size_t setScan(b200reg_t reg, const float* points, size_t n, size_t stride, long intensity_offset) {
    size_t m = 0;
    check(b200sm_set_scan(s_.get(), reg, points, n, stride, intensity_offset, &m));
    return m;
  }
  void updateMap(b200reg_t reg, const float final16[16], const double position[3], const double quat_xyzw[4], bool adopt_now = true) {
    check(b200sm_update_map(s_.get(), reg, final16, position, quat_xyzw, adopt_now ? 1 : 0));
  }
  size_t numSubmaps() const {
    size_t n = 0;
    b200sm_num_submaps(s_.get(), &n);
    return n;
  }
  // doPoseAdjustment's solve (gbs.cpp:262-319): poses = 16 * numSubmaps() doubles, column-major per submap
  b200sm_pose_adjust_result poseAdjust(const std::vector<b200sm_loop_edge>& loop_edges, std::vector<double>& poses,
                                       int num_adjacent_pose_cnstraints = 5, int max_iterations = 10) {
    poses.resize(16 * numSubmaps());
    b200sm_pose_adjust_result r{};
    check(b200sm_pose_adjust(s_.get(), num_adjacent_pose_cnstraints, loop_edges.data(), (int)loop_edges.size(), max_iterations,
                             poses.data(), &r));
    return r;
  }
  // the map moved by `poses` (nullptr: the submaps' own poses, publishMap); xyzi = 4 floats per point in submap order,
  // offsets = numSubmaps() + 1 prefix sums (modified_map_array's i-th cloud is [offsets[i], offsets[i+1]))
  void assembleMap(const double* poses_colmajor16, std::vector<float>& xyzi, std::vector<size_t>& offsets) {
    size_t n = 0;
    offsets.resize(numSubmaps() + 1);
    check(b200sm_assemble_map(s_.get(), poses_colmajor16, nullptr, 0, &n, offsets.data()));
    xyzi.resize(4 * n);
    check(b200sm_assemble_map(s_.get(), poses_colmajor16, xyzi.data(), n, &n, nullptr));
  }
  // pcl::io::savePCDFileASCII(path, map) of the map assembleMap(poses_colmajor16, ...) builds (the map_save service),
  // formatted on the device; throws like PCL for an empty map or a file that cannot be written. Returns the file size.
  size_t saveMapPCDASCII(const std::string& path, const double* poses_colmajor16 = nullptr) {
    size_t n = 0, bytes = 0;
    check(b200sm_save_map_pcd_ascii(s_.get(), poses_colmajor16, path.c_str(), &n, &bytes));
    return bytes;
  }
  // ---- localisation in a prior map (b200sm_set_prior_map*, b200sm_localize_*): the map stays on the device, each frame is
  // registered against a cut of it around the pose. Returns the map's points.
  size_t setPriorMapPCD(const std::string& path) {
    size_t n = 0;
    check(b200sm_set_prior_map_pcd(s_.get(), path.c_str(), &n));
    return n;
  }
  void setPriorMap(const float* points, size_t n, size_t stride, long intensity_offset) {
    check(b200sm_set_prior_map(s_.get(), points, n, stride, intensity_offset));
  }
  // keep crop_radius >= scan_max_range + recrop_distance
  void setLocalizationParams(double crop_radius, double recrop_distance) {
    check(b200sm_set_localization_params(s_.get(), crop_radius, recrop_distance));
  }
  // one frame; returns true when the target was cut again (the new cut is the target from the next frame on)
  bool localizeCloud(b200reg_t reg, const float* points, size_t n, size_t stride, long intensity_offset, double pose7[7], float final16[16]) {
    int recut = 0;
    check(b200sm_localize_cloud(s_.get(), reg, points, n, stride, intensity_offset, pose7, final16, &recut));
    return recut != 0;
  }
  // NDT: the initial pose from guesses.size() / 16 hypotheses (column-major 4x4 each) in one batch launch; returns the index
  // of the adopted one or -1, rows = one result per guess
  int localizeInit(b200reg_t reg, const float* points, size_t n, size_t stride, long intensity_offset, const std::vector<float>& guesses,
                   std::vector<b200reg_batch_result>& rows) {
    int best = -1;
    rows.resize(guesses.size() / 16);
    check(b200sm_localize_init(s_.get(), reg, points, n, stride, intensity_offset, guesses.data(), (int)rows.size(), rows.data(), &best));
    return best;
  }
  // NDT: the pose without a precise guess (b200sm_localize_global): the (x, y, yaw) grid of `spec` around the current pose
  // scored in one launch, the best spec.top_k refined in one batch launch; returns the adopted row or -1. candidates[r] = the
  // hypothesis of row r, rows = one result per refined hypothesis (as localizeInit's), info (optional) = the search's counts
  int localizeGlobal(b200reg_t reg, const float* points, size_t n, size_t stride, long intensity_offset, const b200sm_global_search& spec,
                     std::vector<int>& candidates, std::vector<b200reg_batch_result>& rows, b200sm_global_result* info = nullptr) {
    const size_t k = spec.top_k > 0 ? (size_t)spec.top_k : 1;
    candidates.assign(k, -1);
    rows.resize(k);
    b200sm_global_result r{};
    check(b200sm_localize_global(s_.get(), reg, points, n, stride, intensity_offset, &spec, candidates.data(), rows.data(), &r));
    candidates.resize((size_t)r.n_refined);
    rows.resize((size_t)r.n_refined);
    if (info) *info = r;
    return r.best;
  }
  // the grid of the last localizeGlobal: 16 floats per hypothesis (column-major), its score and its kept pairs
  void globalSearch(std::vector<float>& poses, std::vector<double>& scores, std::vector<long long>& hits) {
    size_t n = 0;
    check(b200sm_get_global_search(s_.get(), 0, &n, nullptr, nullptr, nullptr));
    poses.resize(16 * n);
    scores.resize(n);
    hits.resize(n);
    check(b200sm_get_global_search(s_.get(), n, &n, poses.data(), scores.data(), hits.data()));
  }
  // relocalisation anywhere in the prior map (b200sm_relocalize; params NULL: the defaults): the refined rows in rank order;
  // returns the adopted row or -1 (pose unchanged)
  int relocalize(b200reg_t reg, const float* points, size_t n, size_t stride, long intensity_offset, const b200sm_relocalize_params* params,
                 std::vector<b200sm_relocalize_row>& rows, b200sm_relocalize_result* info = nullptr) {
    const int top_k = params ? params->top_k : 4;
    rows.resize(top_k > 0 ? (size_t)top_k : 1);
    b200sm_relocalize_result r{};
    check(b200sm_relocalize(s_.get(), reg, points, n, stride, intensity_offset, params, rows.data(), rows.size(), &r));
    rows.resize((size_t)r.n_rows);
    if (info) *info = r;
    return r.best;
  }
  // ---- place recognition (b200sm_search_loop_place): a loop search by Scan Context that does not trust the drifted poses
  void setScanContextParams(const b200sm_scan_context_params* p) { check(b200sm_set_scan_context_params(s_.get(), p)); }
  // descriptor of submap `index`: num_rings * num_sectors floats, ring-major
  void scanContext(size_t index, std::vector<float>& out, int num_rings = 20, int num_sectors = 60) {
    out.resize((size_t)num_rings * num_sectors);
    check(b200sm_get_scan_context(s_.get(), index, out.data(), out.size()));
  }
  // the top_k best candidates under sc_threshold, verified from the descriptors' heading; an accepted row gives the loop
  // edge (row.loop.id_min, numSubmaps() - 1, row.loop.relative_pose). Returns the number of eligible submaps.
  size_t searchLoopPlace(b200reg_t reg, float voxel_leaf_size, double threshold_loop_closure_score, double distance_loop_closure,
                         int search_submap_num, double sc_threshold, int top_k, std::vector<b200sm_place_result>& rows) {
    rows.resize(top_k > 0 ? (size_t)top_k : 1);
    size_t n = 0, scored = 0;
    check(b200sm_search_loop_place(s_.get(), reg, voxel_leaf_size, threshold_loop_closure_score, distance_loop_closure,
                                   search_submap_num, sc_threshold, top_k, rows.data(), rows.size(), &n, &scored));
    rows.resize(n);
    return scored;
  }
  // the last place search's D (NaN: not eligible) and s* (-1) per submap
  void placeScores(std::vector<double>& distances, std::vector<int>& shifts) {
    size_t n = 0;
    check(b200sm_get_place_scores(s_.get(), 0, &n, nullptr, nullptr));
    distances.resize(n);
    shifts.resize(n);
    check(b200sm_get_place_scores(s_.get(), n, &n, distances.data(), shifts.data()));
  }
  // ---- merging a second recording (b200sm_merge_session): `other`'s submaps are appended as a new segment when at least
  // min_inliers consistent matches are found. p nullptr = the defaults; loop_edges in merged numbering (other's submap b is
  // numSubmaps() + b). rows = the verified pairs; poses_out = the joint adjustment's (n_A + n_B) x 16 column-major doubles
  // when merged. Returns the result (result.merged says whether this session changed).
  b200sm_merge_result mergeSession(const ScanMatcherSession& other, b200reg_t reg, std::vector<b200sm_merge_row>& rows,
                                   std::vector<double>& poses_out, const b200sm_merge_params* p = nullptr,
                                   const std::vector<b200sm_loop_edge>& loop_edges = {}) {
    size_t na = 0, nb = 0, n = 0;
    check(b200sm_num_submaps(s_.get(), &na));
    check(b200sm_num_submaps(other.handle(), &nb));
    rows.resize(p ? (size_t)std::max(p->max_verifications, 1) : 64);
    std::vector<double> poses(16 * (na + nb));
    b200sm_merge_result r{};
    check(b200sm_merge_session(s_.get(), other.handle(), reg, p, loop_edges.empty() ? nullptr : loop_edges.data(),
                               (int)loop_edges.size(), rows.data(), rows.size(), &n, poses.data(), &r));
    rows.resize(n);
    if (r.merged) poses_out.swap(poses);
    return r;
  }
  // ---- the session on disk (b200sm_save_session / b200sm_load_session): dir/session.txt, dir/pose_graph.g2o and one binary
  // PCD per submap under dir/submaps. adjusted_poses: empty, or 16 * numSubmaps() doubles column-major (poseAdjust's output)
  b200sm_session_io_info saveSession(const std::string& dir, const std::vector<b200sm_loop_edge>& loop_edges = {},
                                     int num_adjacent_pose_cnstraints = 5, const std::vector<double>& adjusted_poses = {}) {
    b200sm_session_io_info info{};
    if (!adjusted_poses.empty() && adjusted_poses.size() != 16 * numSubmaps())
      throw std::runtime_error("saveSession: adjusted_poses must hold 16 doubles per submap");
    check(b200sm_save_session(s_.get(), dir.c_str(), num_adjacent_pose_cnstraints, loop_edges.empty() ? nullptr : loop_edges.data(),
                              (int)loop_edges.size(), adjusted_poses.empty() ? nullptr : adjusted_poses.data(), &info));
    return info;
  }
  // into this (empty) session; loop_edges, adjusted_poses (empty when saved without) and k: the graph it was saved with
  b200sm_session_io_info loadSession(const std::string& dir, std::vector<b200sm_loop_edge>& loop_edges, std::vector<double>& adjusted_poses,
                                     int& num_adjacent_pose_cnstraints) {
    b200sm_session_io_info info{};
    check(b200sm_load_session(s_.get(), dir.c_str(), &info));
    size_t n = 0;
    loop_edges.resize(info.n_loop_edges);
    adjusted_poses.assign(info.adjusted ? 16 * info.n_submaps : 0, 0.0);
    check(b200sm_get_session_graph(s_.get(), loop_edges.empty() ? nullptr : loop_edges.data(), loop_edges.size(), &n,
                                   adjusted_poses.empty() ? nullptr : adjusted_poses.data(), &num_adjacent_pose_cnstraints));
    return info;
  }
  // ---- occupancy grid for a navigation stack (b200sm_build_occupancy_grid): poses empty = the submaps' own, else 16 doubles
  // per submap, column-major (b200sm_pose_adjust's output); p nullptr = the defaults
  b200sm_occupancy_info buildOccupancyGrid(const std::vector<double>& poses_colmajor16 = {},
                                           const b200sm_occupancy_params* p = nullptr) {
    b200sm_occupancy_info info{};
    check(b200sm_build_occupancy_grid(s_.get(), poses_colmajor16.empty() ? nullptr : poses_colmajor16.data(), p, &info));
    og_cells_ = (size_t)info.width * info.height;
    return info;
  }
  // the last grid as nav_msgs/OccupancyGrid.data (row-major from cell (0, 0)); hits / frees when non-null
  void occupancyGrid(std::vector<signed char>& data, std::vector<unsigned>* hits = nullptr, std::vector<unsigned>* frees = nullptr) {
    data.resize(og_cells_);
    if (hits) hits->resize(og_cells_);
    if (frees) frees->resize(og_cells_);
    check(b200sm_get_occupancy_grid(s_.get(), data.data(), hits ? hits->data() : nullptr, frees ? frees->data() : nullptr,
                                    og_cells_));
  }
  // nav2 map_server's map.pgm + map.yaml of the last grid
  void saveOccupancyMap(const std::string& pgm_path, const std::string& yaml_path) {
    check(b200sm_save_occupancy_map(s_.get(), pgm_path.c_str(), yaml_path.c_str()));
  }
  // ---- elevation / traversability map for non-flat ground (b200sm_build_elevation_map): poses empty = the submaps' own,
  // else 16 doubles per submap, column-major; p nullptr = the defaults
  b200sm_elevation_info buildElevationMap(const std::vector<double>& poses_colmajor16 = {}, const b200sm_elevation_params* p = nullptr) {
    b200sm_elevation_info info{};
    check(b200sm_build_elevation_map(s_.get(), poses_colmajor16.empty() ? nullptr : poses_colmajor16.data(), p, &info));
    el_cells_ = (size_t)info.width * info.height;
    return info;
  }
  // the last map, row-major from cell (0, 0): values (-1, 0..99, 100) and, where asked for, surface heights (fixed point),
  // tangents of the slope, and roughness (metres)
  void elevationMap(std::vector<signed char>& value, std::vector<long long>* h = nullptr, std::vector<float>* tan_slope = nullptr,
                    std::vector<float>* roughness = nullptr) {
    value.resize(el_cells_);
    if (h) h->resize(el_cells_);
    if (tan_slope) tan_slope->resize(el_cells_);
    if (roughness) roughness->resize(el_cells_);
    check(b200sm_get_elevation_map(s_.get(), nullptr, h ? h->data() : nullptr, nullptr, nullptr, tan_slope ? tan_slope->data() : nullptr,
                                   roughness ? roughness->data() : nullptr, value.data(), el_cells_));
  }
  // nav2 map_server's pgm + yaml of the last map, next to the occupancy grid's
  void saveTraversabilityMap(const std::string& pgm_path, const std::string& yaml_path) {
    check(b200sm_save_traversability_map(s_.get(), pgm_path.c_str(), yaml_path.c_str()));
  }
  // ---- static map (b200sm_build_static_map): the map without what moved while it was recorded; poses empty = the
  // submaps' own, else 16 doubles per submap, column-major (b200sm_pose_adjust's output); p nullptr = the defaults
  // ---- map consistency (b200sm_build_map_consistency): MME / MPV of the map, per point and per submap; poses empty = the
  // submaps' own, else 16 doubles per submap, column-major; p nullptr = the defaults
  b200sm_map_consistency_info buildMapConsistency(const std::vector<double>& poses_colmajor16 = {},
                                                  const b200sm_map_consistency_params* p = nullptr) {
    b200sm_map_consistency_info info{};
    check(b200sm_build_map_consistency(s_.get(), poses_colmajor16.empty() ? nullptr : poses_colmajor16.data(), p, &info));
    return info;
  }
  b200sm_static_map_info buildStaticMap(const std::vector<double>& poses_colmajor16 = {}, const b200sm_static_map_params* p = nullptr) {
    b200sm_static_map_info info{};
    check(b200sm_build_static_map(s_.get(), poses_colmajor16.empty() ? nullptr : poses_colmajor16.data(), p, &info));
    sm_sub_ = numSubmaps();
    return info;
  }
  // the last static map, x y z intensity per point; offsets (when non-null) = per-submap prefix sums (submaps at the build + 1)
  void staticMap(std::vector<float>& xyzi, std::vector<size_t>* offsets = nullptr) {
    size_t n = 0;
    check(b200sm_get_static_map(s_.get(), nullptr, 0, &n, nullptr));
    xyzi.resize(4 * n);
    if (offsets) offsets->resize(sm_sub_ + 1);
    check(b200sm_get_static_map(s_.get(), xyzi.data(), n, &n, offsets ? offsets->data() : nullptr));
  }
  // the occupied voxels of the last build in rank order: 3 ints each, hits, frees, dynamic flags
  void mapVoxels(std::vector<int>& ijk3, std::vector<unsigned>& hits, std::vector<unsigned>& frees, std::vector<unsigned char>& dynamic) {
    size_t n = 0;
    check(b200sm_get_map_voxels(s_.get(), nullptr, nullptr, nullptr, nullptr, 0, &n));
    ijk3.resize(3 * n);
    hits.resize(n);
    frees.resize(n);
    dynamic.resize(n);
    check(b200sm_get_map_voxels(s_.get(), ijk3.data(), hits.data(), frees.data(), dynamic.data(), n, &n));
  }
  // PCL's ASCII PCD of the last static map (as saveMapPCDASCII writes the map)
  void saveStaticMapPcd(const std::string& path) { check(b200sm_save_static_map_pcd_ascii(s_.get(), path.c_str(), nullptr, nullptr)); }
  // ---- map changes (b200sm_build_map_changes): what appeared and vanished between the submaps before split_submap and
  // those from it on (-1: the last segment's first submap); poses empty = the submaps' own; p nullptr = the defaults
  b200sm_map_change_info buildMapChanges(const std::vector<double>& poses_colmajor16 = {}, long long split_submap = -1,
                                         const b200sm_static_map_params* p = nullptr) {
    b200sm_map_change_info info{};
    check(b200sm_build_map_changes(s_.get(), poses_colmajor16.empty() ? nullptr : poses_colmajor16.data(), p, split_submap, &info));
    ch_sub_ = numSubmaps();
    return info;
  }
  // the label of every point of the last build (B200SM_CHANGE_*), in map order
  void mapChanges(std::vector<unsigned char>& labels) {
    size_t n = 0;
    check(b200sm_get_map_changes(s_.get(), nullptr, 0, &n));
    labels.resize(n);
    check(b200sm_get_map_changes(s_.get(), labels.data(), n, &n));
  }
  // the occupied voxels of the last build in rank order: 3 ints each, the counts of each epoch, the label
  void changeVoxels(std::vector<int>& ijk3, std::vector<unsigned>& hits_before, std::vector<unsigned>& frees_before,
                    std::vector<unsigned>& hits_after, std::vector<unsigned>& frees_after, std::vector<unsigned char>& label) {
    size_t n = 0;
    check(b200sm_get_change_voxels(s_.get(), nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, &n));
    ijk3.resize(3 * n);
    hits_before.resize(n);
    frees_before.resize(n);
    hits_after.resize(n);
    frees_after.resize(n);
    label.resize(n);
    check(b200sm_get_change_voxels(s_.get(), ijk3.data(), hits_before.data(), frees_before.data(), hits_after.data(), frees_after.data(),
                                   label.data(), n, &n));
  }
  // the last updated map, x y z intensity per point; offsets (when non-null) = per-submap prefix sums (submaps at the build + 1)
  void updatedMap(std::vector<float>& xyzi, std::vector<size_t>* offsets = nullptr) {
    size_t n = 0;
    check(b200sm_get_updated_map(s_.get(), nullptr, 0, &n, nullptr));
    xyzi.resize(4 * n);
    if (offsets) offsets->resize(ch_sub_ + 1);
    check(b200sm_get_updated_map(s_.get(), xyzi.data(), n, &n, offsets ? offsets->data() : nullptr));
  }
  // PCL's ASCII PCD of the last updated map: the prior map for setPriorMapPcd next time
  void saveUpdatedMapPcd(const std::string& path) { check(b200sm_save_updated_map_pcd_ascii(s_.get(), path.c_str(), nullptr, nullptr)); }

  // ---- surface mesh (b200sm_build_mesh): a TSDF of every submap's rays, extracted by surface nets; poses empty = the
  // submaps' own; p nullptr = the defaults
  b200sm_mesh_info buildMesh(const std::vector<double>& poses_colmajor16 = {}, const b200sm_mesh_params* p = nullptr) {
    b200sm_mesh_info info{};
    check(b200sm_build_mesh(s_.get(), poses_colmajor16.empty() ? nullptr : poses_colmajor16.data(), p, &info));
    return info;
  }
  // the last mesh: x y z per vertex (map frame), three vertex ids per face (counter-clockwise seen from free space)
  void mesh(std::vector<float>& xyz, std::vector<unsigned>& faces3) {
    size_t nv = 0, nf = 0;
    check(b200sm_get_mesh(s_.get(), nullptr, 0, &nv, nullptr, 0, &nf));
    xyz.resize(3 * nv);
    faces3.resize(3 * nf);
    check(b200sm_get_mesh(s_.get(), xyz.data(), nv, &nv, faces3.data(), nf, &nf));
  }
  // the last build's band voxels in rank order: 3 ints each, the fused signed-distance sum and the ray count
  void meshVoxels(std::vector<int>& ijk3, std::vector<long long>& sdf_sum, std::vector<unsigned>& weight) {
    size_t n = 0;
    check(b200sm_get_mesh_voxels(s_.get(), nullptr, nullptr, nullptr, 0, &n));
    ijk3.resize(3 * n);
    sdf_sum.resize(n);
    weight.resize(n);
    check(b200sm_get_mesh_voxels(s_.get(), ijk3.data(), sdf_sum.data(), weight.data(), n, &n));
  }
  // the last mesh as binary PLY; returns the file's bytes
  size_t saveMeshPly(const std::string& path) {
    size_t n = 0;
    check(b200sm_save_mesh_ply(s_.get(), path.c_str(), &n));
    return n;
  }

  // ---- OctoMap (b200sm_build_octomap): free and occupied voxels of every submap's rays, pruned into OctoMap's key tree;
  // poses empty = the submaps' own; p nullptr = the static map's defaults
  b200sm_octomap_info buildOctoMap(const std::vector<double>& poses_colmajor16 = {}, const b200sm_static_map_params* p = nullptr) {
    b200sm_octomap_info info{};
    check(b200sm_build_octomap(s_.get(), poses_colmajor16.empty() ? nullptr : poses_colmajor16.data(), p, &info));
    return info;
  }
  // the last OctoMap as an OctoMap .bt file (octomap_server, MoveIt, rviz); returns the file's bytes
  size_t saveOctoMapBt(const std::string& path) {
    size_t n = 0;
    check(b200sm_save_octomap_bt(s_.get(), path.c_str(), &n));
    return n;
  }
  b200sm_localize_stats localizeStats() const {
    b200sm_localize_stats st{};
    check(b200sm_get_localize_stats(s_.get(), &st));
    return st;
  }
  void cutCloud(std::vector<float>& xyzi) {
    size_t n = 0;
    check(b200sm_get_cut(s_.get(), nullptr, 0, &n));
    xyzi.resize(4 * n);
    check(b200sm_get_cut(s_.get(), xyzi.data(), n, &n));
  }
  b200sm_t handle() const { return s_.get(); }

 private:
  void check(int rc) const {
    if (rc != B200REG_OK) throw std::runtime_error(std::string("b200sm: ") + b200sm_last_error(s_.get()));
  }
  std::shared_ptr<b200sm_session> s_;
  size_t og_cells_ = 0;  // cells of the last grid this adapter built
  size_t el_cells_ = 0;  // cells of the last elevation map this adapter built
  size_t sm_sub_ = 0;    // submaps at the last static-map build of this adapter
  size_t ch_sub_ = 0;    // submaps at the last map-change build of this adapter
};

}  // namespace b200reg
