// IMU de-skew of a spinning-LiDAR scan on the GPU (SURVEY.md §8f row 4).
// Replaces scanmatcher/include/scanmatcher/lidar_undistortion.hpp: LidarUndistortion::getImu :52-106 (host state machine,
// one call per IMU message) and adjustDistortion :110-226 (per-point work -> kernels, deskew.cu).
#pragma once
#include <cuda_runtime.h>

#include "engine.hpp"

namespace b200 {

constexpr int IMU_QUE = 200;  // imu_que_length_ (lidar_undistortion.hpp:242)

struct ImuSample {  // one ring entry as the kernels read it
  double time;
  float roll, pitch, yaw;
  float shift[3];
  float velo[3];
  float pad;
};

class ImuDeskew {
 public:
  double scan_period = 0.1;  // scan_period_ (setScanPeriod)
  // ring buffer state (members of LidarUndistortion)
  int ptr_front = 0, ptr_last = -1, ptr_last_iter = 0;
  double time[IMU_QUE] = {};
  float roll[IMU_QUE] = {}, pitch[IMU_QUE] = {}, yaw[IMU_QUE] = {};
  float velo[IMU_QUE][3] = {}, shift[IMU_QUE][3] = {}, ang_rot[IMU_QUE][3] = {};
  int launches = 0;

  // getImu (:52-106): angular velocity, linear acceleration, orientation quaternion (x, y, z, w), stamp [s]
  void get_imu(const float* angular_velo3, const float* acc3, const float* quat_xyzw, double imu_time);
  // adjustDistortion (:110-226) in place on a device-resident scan of n float4 (x, y, z, intensity) in firing order.
  // first_xy / last_xy: x, y of the first and the last point (the host has them: it uploaded the scan).
  // Synchronises the stream (the carried ring pointers come back to the host).
  void adjust_distortion(float4* d_cloud, size_t n, const float* first_xy, const float* last_xy, double scan_time, cudaStream_t s);
  // The last adjust_distortion's per-point scratch: relative time, time stamp, imu_ptr_front_ (ring index) and the
  // stable skip flag of min(capacity, n) points, the half-turn index and the fix-point passes. Returns n (0 when the
  // kernels did not run). Synchronises the stream.
  size_t get_trace(size_t capacity, float* rel_time, double* t, int* front, unsigned char* skip, int* k_first, int* rounds,
                   cudaStream_t s);

 private:
  int trace_n = 0, trace_base = 0, trace_k_first = 0, trace_rounds = 0;
  DeviceBuffer<float> d_ori, d_a, d_rel;
  DeviceBuffer<double> d_t;
  DeviceBuffer<int> d_lb, d_front;
  DeviceBuffer<unsigned char> d_skip;  // 2 x n (double-buffered by the fix-point iteration)
  DeviceBuffer<unsigned char> d_small;  // DeskewShared
  PinnedBuffer<int> h_out;
};

}  // namespace b200
