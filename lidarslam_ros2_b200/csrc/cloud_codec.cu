// Point-cloud wire format -> device layout (SURVEY.md §8f row 3). The reference hands clouds around as arrays of
// fixed-size records — pcl::PointCloud<PointXYZI> (32-byte points) or the data block of a sensor_msgs/PointCloud2
// (point_step bytes per point, x/y/z/intensity float32 fields at their offsets; pcl::fromROSMsg,
// scanmatcher_component.cpp:202, 457) — and re-packs them on the CPU. Here the raw records go to the GPU in ONE bulk
// copy (straight from the caller's buffer when it is pinned, else through a pinned staging copy made with memcpy) and a
// kernel unpacks them into the float4 (x, y, z, w) layout every other kernel reads.
#include <algorithm>
#include <cstring>
#include <thread>

#include "engine.hpp"
#include "grid_index.cuh"

namespace b200 {

namespace {
__global__ void unpack_points_kernel(const unsigned char* __restrict__ raw, size_t n, size_t stride, long w_off, float w_default,
                                     float4* __restrict__ dst) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned char* p = raw + i * stride;  // records are 4-byte aligned (float fields)
  const float* f = reinterpret_cast<const float*>(p);
  float4 v;
  v.x = f[0];
  v.y = f[1];
  v.z = f[2];
  v.w = w_off >= 0 ? *reinterpret_cast<const float*>(p + w_off) : w_default;
  dst[i] = v;
}
// same + min/max of the finite points (the NDT voxel grid and the NN grid of a target are sized from them): one pass less
// over the cloud and no separate round trip for the bounds.
// kTransform: x, y, z go through T (transform_point) before the store, and the bounds are those of the transformed points
// — tf2::doTransform of the frontend's cloud callback (scanmatcher_component.cpp:188-199) in the pass that reads the
// records anyway. .w is copied untouched. The <false> instantiation has no transform code at all.
template <bool kTransform>
__global__ void unpack_points_bounds_kernel(const unsigned char* __restrict__ raw, size_t n, size_t stride, long w_off, float w_default,
                                            float4* __restrict__ dst, unsigned* __restrict__ out6, Mat34f T) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  if (i < n) {
    const unsigned char* p = raw + i * stride;
    const float* f = reinterpret_cast<const float*>(p);
    float4 v;
    v.x = f[0];
    v.y = f[1];
    v.z = f[2];
    v.w = w_off >= 0 ? *reinterpret_cast<const float*>(p + w_off) : w_default;
    if (kTransform) {
      const float3 r = transform_point(T.m, v);
      v.x = r.x;
      v.y = r.y;
      v.z = r.z;
    }
    dst[i] = v;
    if (isfinite(v.x) && isfinite(v.y) && isfinite(v.z)) {
      mn[0] = mx[0] = v.x;
      mn[1] = mx[1] = v.y;
      mn[2] = mx[2] = v.z;
    }
  }
  block_bounds_merge(mn, mx, out6);
}
// host -> device copy of `bytes`. Pinned memory goes out in one DMA; pageable memory (a pcl::PointCloud, a numpy array) is
// staged through the pinned buffer in 2 MB pieces, each piece's DMA enqueued as soon as it is staged, so that the copy
// engine works on piece k while the CPU copies piece k + 1 (the staging buffer holds the whole cloud: no piece is reused).
void staged_h2d(void* d_dst, const void* host, size_t bytes, bool pinned, unsigned char* staging, cudaStream_t s) {
  if (pinned) {
    B200_CUDA(cudaMemcpyAsync(d_dst, host, bytes, cudaMemcpyHostToDevice, s));
    return;
  }
  constexpr size_t PIECE = (size_t)2 << 20;
  const unsigned char* src = static_cast<const unsigned char*>(host);
  unsigned char* dst = static_cast<unsigned char*>(d_dst);
  const size_t n_pieces = (bytes + PIECE - 1) / PIECE;
  auto stage_piece = [&](size_t k) -> cudaError_t {
    const size_t off = k * PIECE, len = std::min(PIECE, bytes - off);
    std::memcpy(staging + off, src + off, len);
    return cudaMemcpyAsync(dst + off, staging + off, len, cudaMemcpyHostToDevice, s);
  };
  if (bytes >= ((size_t)8 << 20)) {
    // a big pageable cloud (a 1 M-point map is 12 - 32 MB): one CPU thread copies at 5 - 8 GB/s, well below the DMA rate, so
    // four threads stage interleaved pieces (each enqueues its own piece's DMA; the pieces are disjoint, their order is free)
    constexpr int T = 4;
    cudaError_t errs[T];
    std::thread th[T - 1];
    auto work = [&](int t) {
      errs[t] = cudaSuccess;
      int dev = 0;
      for (size_t k = (size_t)t; k < n_pieces && errs[t] == cudaSuccess; k += T) errs[t] = stage_piece(k);
      (void)dev;
    };
    int device = 0;
    cudaGetDevice(&device);
    for (int t = 1; t < T; t++)
      th[t - 1] = std::thread([&, t, device]() {
        cudaSetDevice(device);
        work(t);
      });
    work(0);
    for (int t = 1; t < T; t++) th[t - 1].join();
    for (int t = 0; t < T; t++) B200_CUDA(errs[t]);
    return;
  }
  for (size_t k = 0; k < n_pieces; k++) B200_CUDA(stage_piece(k));
}
}  // namespace

// upload + bounds: the result is valid after the caller has synchronised the stream (finish_bounds)
void CloudUploader::upload_with_bounds(const void* host, size_t n, size_t stride, long w_off, float w_default, float4* dst,
                                       cudaStream_t s, const Mat34f* T) {
  if (n == 0) return;
  const size_t bytes = n * stride;
  raw.ensure(bytes);
  bounds_dev.ensure(8);
  bounds_host.ensure(8);
  const bool pinned = is_pinned(host);
  if (!pinned) staging.ensure(bytes);
  const unsigned init[6] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u};
  std::memcpy(bounds_host.ptr, init, sizeof(init));
  B200_CUDA(cudaMemcpyAsync(bounds_dev.ptr, bounds_host.ptr, sizeof(init), cudaMemcpyHostToDevice, s));
  staged_h2d(raw.ptr, host, bytes, pinned, staging.ptr, s);
  const int blocks = (int)((n + 255) / 256);
  if (T)
    unpack_points_bounds_kernel<true><<<blocks, 256, 0, s>>>(raw.ptr, n, stride, w_off, w_default, dst, bounds_dev.ptr, *T);
  else
    unpack_points_bounds_kernel<false><<<blocks, 256, 0, s>>>(raw.ptr, n, stride, w_off, w_default, dst, bounds_dev.ptr, Mat34f{});
  B200_CUDA(cudaGetLastError());
  B200_CUDA(cudaMemcpyAsync(bounds_host.ptr, bounds_dev.ptr, sizeof(init), cudaMemcpyDeviceToHost, s));
  launches += 1;
}
Bounds CloudUploader::finish_bounds() const {
  return decode_bounds(bounds_host.ptr);
}

void CloudUploader::upload(const void* host, size_t n, size_t stride, long w_off, float w_default, float4* dst, cudaStream_t s) {
  if (n == 0) return;
  const size_t bytes = n * stride;
  raw.ensure(bytes);
  const bool pinned = is_pinned(host);
  if (!pinned) staging.ensure(bytes);
  staged_h2d(raw.ptr, host, bytes, pinned, staging.ptr, s);
  unpack_points_kernel<<<(int)((n + 255) / 256), 256, 0, s>>>(raw.ptr, n, stride, w_off, w_default, dst);
  B200_CUDA(cudaGetLastError());
  launches += 1;
}

// Batched form: `reserve` sizes the raw device buffer (and the pinned staging copy when some input is pageable) for
// the whole batch once, `upload_at` then enqueues copy + unpack of one cloud at its byte offset — no synchronisation
// between the clouds of a batch, the copy engine streams them back to back.
void CloudUploader::reserve(size_t raw_bytes, bool need_staging) {
  raw.ensure(raw_bytes);
  if (need_staging) staging.ensure(raw_bytes);
}
bool CloudUploader::is_pinned(const void* host) {
  cudaPointerAttributes attr{};
  const bool pinned = cudaPointerGetAttributes(&attr, host) == cudaSuccess && attr.type == cudaMemoryTypeHost;
  if (!pinned) cudaGetLastError();
  return pinned;
}
// host -> raw device buffer only (no unpack): the batch solver reads the records as they are
void CloudUploader::copy_at(const void* host, bool pinned, size_t bytes, size_t byte_offset, cudaStream_t s) {
  if (bytes == 0) return;
  staged_h2d(raw.ptr + byte_offset, host, bytes, pinned, staging.ptr + byte_offset, s);
}
void CloudUploader::upload_at(const void* host, bool pinned, size_t n, size_t stride, long w_off, float w_default, float4* dst,
                              size_t byte_offset, cudaStream_t s) {
  if (n == 0) return;
  const size_t bytes = n * stride;
  staged_h2d(raw.ptr + byte_offset, host, bytes, pinned, staging.ptr + byte_offset, s);
  unpack_points_kernel<<<(int)((n + 255) / 256), 256, 0, s>>>(raw.ptr + byte_offset, n, stride, w_off, w_default, dst);
  B200_CUDA(cudaGetLastError());
  launches += 1;
}

void upload_cloud(const float* base, size_t n, size_t stride_bytes, DeviceBuffer<float4>& dst, CloudUploader& up, cudaStream_t s) {
  dst.ensure(n);
  up.upload(base, n, stride_bytes, -1, 1.0f, dst.ptr, s);
}

}  // namespace b200
