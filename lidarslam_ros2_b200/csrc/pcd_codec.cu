// Device -> ASCII PCD text (pcl::io::savePCDFileASCII, graph_based_slam_component.cpp:369): every float of a float4
// (x, y, z, intensity) cloud formatted on the GPU by pcd_format.cuh, byte for byte what PCL's writeASCII prints.
//
// Two passes over tiles of PCD_TILE points. Pass 1 (pcd_measure_kernel) formats a tile's lines and writes the tile's byte
// count; counter_scan_async turns the counts of each chunk of PCD_CHUNK_POINTS points into tile offsets and the chunk's
// total. Pass 2 (pcd_encode_kernel) formats the tile again into shared memory at its in-tile offsets and copies the
// contiguous block out, with 16-byte stores for the aligned middle and byte stores for the head and tail. A chunk's text is
// at most PCD_CHUNK_POINTS * PCD_LINE_MAX_CHARS bytes, so the unsigned offsets inside a chunk cannot overflow.
#include <cstdio>
#include <string>

#include "engine.hpp"
#include "grid_index.cuh"
#include "pcd_format.cuh"

namespace b200 {

namespace {

constexpr int PCD_TILE = 256;  // points (= threads) per tile
constexpr size_t PCD_TILES_PER_CHUNK = PCD_CHUNK_POINTS / PCD_TILE;
static_assert(PCD_CHUNK_POINTS % PCD_TILE == 0, "a chunk is whole tiles");
static_assert(PCD_CHUNK_POINTS * PCD_LINE_MAX_CHARS < ((size_t)1 << 32), "offsets inside a chunk are unsigned");

// counts of chunk c start at c * (PCD_TILES_PER_CHUNK + 1): each chunk's scan leaves its total right after its tiles
__global__ void __launch_bounds__(PCD_TILE) pcd_measure_kernel(const float4* __restrict__ pts, size_t n, unsigned* __restrict__ counts) {
  const size_t tile = blockIdx.x;
  const size_t i = tile * PCD_TILE + threadIdx.x;
  unsigned len = 0;
  if (i < n) {
    char line[PCD_LINE_MAX_CHARS];
    const float4 p = pts[i];
    len = (unsigned)pcd_format_line(p.x, p.y, p.z, p.w, line);
  }
  unsigned total;
  block_exclusive_scan<PCD_TILE>(len, total);
  if (threadIdx.x == 0) counts[(tile / PCD_TILES_PER_CHUNK) * (PCD_TILES_PER_CHUNK + 1) + tile % PCD_TILES_PER_CHUNK] = total;
}

// one chunk: pts = its first point, n = its points, tile_off = its scanned counts, out = its text (16-byte aligned)
__global__ void __launch_bounds__(PCD_TILE) pcd_encode_kernel(const float4* __restrict__ pts, unsigned n,
                                                              const unsigned* __restrict__ tile_off, char* __restrict__ out) {
  __shared__ uint4 buf[PCD_TILE * PCD_LINE_MAX_CHARS / 16 + 1];
  const unsigned i = blockIdx.x * PCD_TILE + threadIdx.x;
  char line[PCD_LINE_MAX_CHARS];
  unsigned len = 0;
  if (i < n) {
    const float4 p = pts[i];
    len = (unsigned)pcd_format_line(p.x, p.y, p.z, p.w, line);
  }
  unsigned total;
  const unsigned pos = block_exclusive_scan<PCD_TILE>(len, total);
  const unsigned off = tile_off[blockIdx.x], end = off + total;
  // output byte g sits at buf byte g - (off & ~15): the shared copy has the output's alignment
  const unsigned shift = off & ~15u;
  char* sb = reinterpret_cast<char*>(buf);
  for (unsigned j = 0; j < len; j++) sb[(off & 15u) + pos + j] = line[j];
  __syncthreads();
  const unsigned a0 = (off + 15u) & ~15u, a1 = end & ~15u;
  if (a0 >= a1) {  // no whole 16-byte word inside the tile's text
    for (unsigned g = off + threadIdx.x; g < end; g += PCD_TILE) out[g] = sb[g - shift];
    return;
  }
  for (unsigned g = off + threadIdx.x; g < a0; g += PCD_TILE) out[g] = sb[g - shift];
  for (unsigned g = a1 + threadIdx.x; g < end; g += PCD_TILE) out[g] = sb[g - shift];
  const uint4* src = buf + (a0 - shift) / 16;
  uint4* dst = reinterpret_cast<uint4*>(out + a0);
  for (unsigned w = threadIdx.x; w < (a1 - a0) / 16; w += PCD_TILE) dst[w] = src[w];
}

}  // namespace

std::string pcd_ascii_header(size_t n) {
  char tail[160];
  snprintf(tail, sizeof tail, "WIDTH %zu\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS %zu\nDATA ascii\n", n, n);
  return std::string("# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z intensity\nSIZE 4 4 4 4\n"
                     "TYPE F F F F\nCOUNT 1 1 1 1\n") + tail;
}

void PcdEncoder::measure(const float4* pts, size_t n, cudaStream_t s) {
  const size_t tiles = (n + PCD_TILE - 1) / PCD_TILE;
  const size_t chunks = (n + PCD_CHUNK_POINTS - 1) / PCD_CHUNK_POINTS;
  const size_t words = chunks * (PCD_TILES_PER_CHUNK + 1);
  counts.ensure(words);
  h_counts.ensure(words);
  chunk_bytes.assign(chunks, 0);
  if (n == 0) return;
  pcd_measure_kernel<<<(unsigned)tiles, PCD_TILE, 0, s>>>(pts, n, counts.ptr);
  B200_CUDA(cudaGetLastError());
  launches += 1;
  for (size_t c = 0; c < chunks; c++) {
    counter_scan_async(counts.ptr + c * (PCD_TILES_PER_CHUNK + 1), std::min(PCD_TILES_PER_CHUNK, tiles - c * PCD_TILES_PER_CHUNK),
                       scan_tmp, s);
    launches += 3;
  }
  B200_CUDA(cudaMemcpyAsync(h_counts.ptr, counts.ptr, words * sizeof(unsigned), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  size_t most = 0;
  for (size_t c = 0; c < chunks; c++) {
    chunk_bytes[c] = h_counts.ptr[c * (PCD_TILES_PER_CHUNK + 1) + std::min(PCD_TILES_PER_CHUNK, tiles - c * PCD_TILES_PER_CHUNK)];
    most = std::max(most, chunk_bytes[c]);
  }
  text.ensure(most);
}

void PcdEncoder::encode_chunk(const float4* pts, size_t n, size_t c, cudaStream_t s) {
  const size_t first = c * PCD_CHUNK_POINTS, m = std::min(PCD_CHUNK_POINTS, n - first);
  pcd_encode_kernel<<<(unsigned)((m + PCD_TILE - 1) / PCD_TILE), PCD_TILE, 0, s>>>(
      pts + first, (unsigned)m, counts.ptr + c * (PCD_TILES_PER_CHUNK + 1), text.ptr);
  B200_CUDA(cudaGetLastError());
  launches += 1;
}

}  // namespace b200

using namespace b200;

// a host cloud: uploaded once, measured, then each chunk encoded and copied to its place in `out` (up to capacity)
extern "C" int b200reg_encode_pcd_ascii(int device, const float* base, size_t n, size_t stride_bytes, long intensity_offset_bytes,
                                        char* out, size_t capacity, size_t* n_bytes) {
  // the file's intensity column is always written, so the records must carry one
  if (!base || n == 0 || !n_bytes || (!out && capacity) || intensity_offset_bytes < 0 ||
      !valid_record_layout(stride_bytes, intensity_offset_bytes))
    return B200REG_ERR_ARG;
  struct State {
    cudaStream_t stream = nullptr;
    CloudUploader uploader;
    DeviceBuffer<float4> points;
    PcdEncoder encoder;
  };
  static std::mutex mu;
  static State* states[64] = {nullptr};
  std::lock_guard<std::mutex> lock(mu);
  try {
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) {
      cudaGetLastError();
      return B200REG_ERR_CUDA;
    }
    if (device >= 64) return B200REG_ERR_ARG;
    B200_CUDA(cudaSetDevice(device));
    if (!states[device]) {
      states[device] = new State();
      B200_CUDA(cudaStreamCreateWithFlags(&states[device]->stream, cudaStreamNonBlocking));
    }
    State& S = *states[device];
    S.points.ensure(n);
    S.uploader.upload(base, n, stride_bytes, intensity_offset_bytes, 0.0f, S.points.ptr, S.stream);
    S.encoder.measure(S.points.ptr, n, S.stream);
    const std::string header = pcd_ascii_header(n);
    size_t pos = header.size();
    for (size_t b : S.encoder.chunk_bytes) pos += b;
    *n_bytes = pos;
    if (capacity) std::memcpy(out, header.data(), std::min(header.size(), capacity));
    pos = header.size();
    for (size_t c = 0; c < S.encoder.chunk_bytes.size() && pos < capacity; c++) {
      S.encoder.encode_chunk(S.points.ptr, n, c, S.stream);
      const size_t k = std::min(S.encoder.chunk_bytes[c], capacity - pos);
      B200_CUDA(cudaMemcpyAsync(out + pos, S.encoder.text.ptr, k, cudaMemcpyDeviceToHost, S.stream));
      B200_CUDA(cudaStreamSynchronize(S.stream));
      pos += S.encoder.chunk_bytes[c];
    }
    return B200REG_OK;
  } catch (const CudaError&) {
    cudaGetLastError();
    return B200REG_ERR_CUDA;
  }
}
