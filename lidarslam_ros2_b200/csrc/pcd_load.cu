// PCD file -> float4 (x, y, z, intensity) on the device: pcl::io::loadPCDFile (apps/align.cpp:54-61) for the map that
// b200sm_save_map_pcd_ascii writes, and for any PCD v0.7 cloud whose x, y, z (and intensity) are 4-byte floats.
//
// DATA ascii: the body moves in pieces of B200REG_PCD_LOAD_PIECE_BYTES, each ending at its last '\n' (the tail carries to
// the next piece). The calling thread freads piece k + 1 into one pinned buffer while piece k, in the other, is copied and
// parsed on the stream. Per piece, two passes over tiles of LOAD_TILE bytes: pass 1 (pcd_line_count_kernel) counts the
// starts of non-empty lines of each tile from 16-byte loads, counter_scan_async turns the counts into tile offsets; pass 2
// (pcd_parse_kernel) stages the tile and LOAD_SPILL bytes after it in shared memory, and each thread parses the lines that
// start in its 16 bytes (pcd_parse.cuh) and stores their points at the running line offset, which stays on the device.
// Points past POINTS are dropped, and reading stops about one piece after the POINTS-th line; a bad line leaves its file
// offset in a flag (the first one wins); the host reads the flag and the line count once, at the end. POINTS is checked
// against the size of the body before any buffer is sized from it.
// DATA binary: the body is read whole into pinned memory and unpacked by the upload path (CloudUploader, cloud_codec.cu).
#include <algorithm>
#include <cerrno>
#include <cstdio>
#include <cstring>
#include <string>

#include <sys/stat.h>

#include "engine.hpp"
#include "grid_index.cuh"

namespace b200 {

namespace {

constexpr int LOAD_THREADS = 256;
constexpr size_t LOAD_TILE = LOAD_THREADS * 16;  // bytes of text per CTA: 16 per thread
constexpr size_t LOAD_SPILL = 4096;              // staged past the tile: a line that starts in it and ends there
constexpr size_t PIECE = B200REG_PCD_LOAD_PIECE_BYTES;
constexpr unsigned long long NO_ERROR = ~0ull;
static_assert(PIECE % LOAD_TILE == 0 && PIECE < ((size_t)1 << 32), "offsets inside a piece are unsigned");

// bit k set when byte k of the 16 in v starts a non-empty line (prev: the byte before them; bytes at or past len: none)
__device__ __forceinline__ unsigned line_starts16(uint4 v, char prev, size_t pos0, size_t len) {
  const unsigned w[4] = {v.x, v.y, v.z, v.w};
  const unsigned n = len - pos0 < 16 ? (unsigned)(len - pos0) : 16u;
  unsigned m = 0;
#pragma unroll
  for (int k = 0; k < 16; k++) {
    const char c = (char)((w[k >> 2] >> (8 * (k & 3))) & 0xffu);
    if (prev == '\n' && c != '\n' && (unsigned)k < n) m |= 1u << k;
    prev = c;
  }
  return m;
}

__global__ void __launch_bounds__(LOAD_THREADS) pcd_line_count_kernel(const char* __restrict__ text, size_t len,
                                                                      unsigned* __restrict__ counts) {
  const size_t pos0 = (blockIdx.x * (size_t)LOAD_THREADS + threadIdx.x) * 16;
  unsigned c = 0;
  if (pos0 < len) {
    const uint4 v = *reinterpret_cast<const uint4*>(text + pos0);
    c = __popc(line_starts16(v, pos0 ? text[pos0 - 1] : '\n', pos0, len));
  }
  c = __reduce_add_sync(0xffffffffu, c);
  __shared__ unsigned warp_sum[LOAD_THREADS / 32];
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned t = 0;
    for (int w = 0; w < LOAD_THREADS / 32; w++) t += warp_sum[w];
    counts[blockIdx.x] = t;
  }
}

// text: the piece, readable LOAD_TILE + LOAD_SPILL bytes past any tile start; tile_off: scanned counts;
// state[0]: non-empty lines of the earlier pieces; state[1]: first failing line (file offset << 2 | PcdLineStatus)
__global__ void __launch_bounds__(LOAD_THREADS) pcd_parse_kernel(const char* __restrict__ text, size_t len,
                                                                 const unsigned* __restrict__ tile_off, PcdLineLayout L,
                                                                 unsigned long long n_points, unsigned long long file_off,
                                                                 float4* __restrict__ out, unsigned long long* state) {
  __shared__ uint4 stage[(LOAD_TILE + LOAD_SPILL) / 16];
  const size_t tile0 = blockIdx.x * LOAD_TILE;
  const unsigned long long base = state[0] + tile_off[blockIdx.x];
  if (base >= n_points) return;  // every line of the tile is past POINTS
  const uint4* src = reinterpret_cast<const uint4*>(text + tile0);
  for (int i = threadIdx.x; i < (int)((LOAD_TILE + LOAD_SPILL) / 16); i += LOAD_THREADS) stage[i] = src[i];
  __syncthreads();
  const char* sb = reinterpret_cast<const char*>(stage);
  const size_t win = len - tile0 < LOAD_TILE + LOAD_SPILL ? len - tile0 : LOAD_TILE + LOAD_SPILL;  // staged bytes of the piece
  const unsigned k0 = threadIdx.x * 16;
  unsigned mask = 0;
  if (tile0 + k0 < len) mask = line_starts16(stage[threadIdx.x], k0 ? sb[k0 - 1] : (tile0 ? text[tile0 - 1] : '\n'), tile0 + k0, len);
  unsigned total;
  unsigned long long idx = base + block_exclusive_scan<LOAD_THREADS>(__popc(mask), total);
  for (; mask && idx < n_points; mask &= mask - 1, idx++) {
    const unsigned at = k0 + (unsigned)(__ffs(mask) - 1);
    float v[4];
    const char* stop;
    int st = pcd_parse_line(sb + at, sb + win, L, v, &stop);
    if (stop == sb + win && tile0 + win < len)  // the line runs past the staged bytes: parse it from global memory
      st = pcd_parse_line(text + tile0 + at, text + len, L, v, &stop);
    if (st == PCD_LINE_OK) out[idx] = make_float4(v[0], v[1], v[2], v[3]);
    else atomicMin(&state[1], ((file_off + tile0 + at) << 2) | (unsigned long long)st);
  }
}

__global__ void pcd_advance_kernel(unsigned long long* state, const unsigned* piece_lines) { state[0] += *piece_lines; }

// 1-based line number of the file at byte offset `off`
size_t line_of_offset(const char* path, unsigned long long off) {
  FILE* fp = std::fopen(path, "rb");
  if (!fp) return 0;
  size_t line = 1;
  char buf[1 << 16];
  while (off > 0) {
    const size_t got = std::fread(buf, 1, (size_t)std::min<unsigned long long>(off, sizeof buf), fp);
    if (got == 0) break;
    line += (size_t)std::count(buf, buf + got, '\n');
    off -= got;
  }
  std::fclose(fp);
  return line;
}

int format_error(std::string& err, const std::string& why) {
  err = why;
  return B200REG_ERR_FORMAT;
}

}  // namespace

int read_pcd_header(FILE* fp, PcdHeader& h, std::string& err) {
  std::string text, line;
  for (;;) {
    line.clear();
    int c;
    while ((c = std::getc(fp)) != EOF && c != '\n') line.push_back((char)c);
    if (std::ferror(fp)) return err = std::string("reading the header: ") + std::strerror(errno), B200REG_ERR_IO;
    text += line;
    text += '\n';
    const size_t i = line.find_first_not_of(" \t\r");
    if (i != std::string::npos && line.compare(i, 4, "DATA") == 0 && (line.size() == i + 4 || pcdparse::is_sep(line[i + 4])))
      break;
    if (c == EOF) return format_error(err, "no DATA line");
    if (text.size() > ((size_t)1 << 20)) return format_error(err, "no DATA line in the first MiB");
  }
  if (!pcd_parse_header(text, h, err)) return B200REG_ERR_FORMAT;
  // POINTS against what the body can hold, before anything is sized from it: an ASCII point takes at least one character
  // per token, one separator between tokens and a '\n' (none after the last), a binary point exactly one record
  struct stat st;
  const long body_at = std::ftell(fp);
  if (body_at >= 0 && fstat(fileno(fp), &st) == 0 && S_ISREG(st.st_mode)) {
    const unsigned long long body = st.st_size > body_at ? (unsigned long long)(st.st_size - body_at) : 0ull;
    const unsigned long long most = h.data == PCD_DATA_ASCII    ? (body + 1) / (2ull * (unsigned)h.layout.n_tokens)
                                    : h.data == PCD_DATA_BINARY ? body / h.record_bytes
                                                                : ~0ull;
    if (h.points > most)
      return format_error(err, "POINTS " + std::to_string(h.points) + ": the body of " + std::to_string(body) +
                                   " bytes holds at most " + std::to_string(most));
  }
  return B200REG_OK;
}

int PcdLoader::load(const char* path, DeviceBuffer<float4>& dst, size_t* n, std::string& err, cudaStream_t s) {
  FILE* fp = std::fopen(path, "rb");
  if (!fp) return err = std::string("cannot open ") + path + ": " + std::strerror(errno), B200REG_ERR_IO;
  cudaEvent_t done[2] = {nullptr, nullptr};
  struct Cleanup {  // on every return: no copy out of the pinned pieces left in flight, the file closed
    FILE* fp;
    cudaEvent_t* ev;
    cudaStream_t s;
    ~Cleanup() {
      cudaStreamSynchronize(s);
      for (int b = 0; b < 2; b++)
        if (ev[b]) cudaEventDestroy(ev[b]);
      std::fclose(fp);
    }
  } cleanup{fp, done, s};
  PcdHeader h;
  int rc = read_pcd_header(fp, h, err);
  if (rc != B200REG_OK) return rc;
  *n = h.points;
  if (h.data == PCD_DATA_BINARY_COMPRESSED) return format_error(err, "DATA binary_compressed is not supported");
  dst.ensure(std::max<size_t>(h.points, 1));
  if (h.data == PCD_DATA_BINARY) {
    const long ox = h.offset[0], oi = h.offset[3];
    const size_t rec = h.record_bytes;
    if (h.offset[1] != ox + 4 || h.offset[2] != ox + 8) return format_error(err, "binary: x, y and z are not consecutive");
    if (rec % 4 || ox % 4 || (oi >= 0 && (oi % 4 || oi < ox)))
      return format_error(err, "binary: the record size and the offsets of x and intensity must be multiples of 4, intensity after x");
    if (h.points == 0) return B200REG_OK;
    if (h.points > (((size_t)1 << 46) / rec)) return format_error(err, "binary: POINTS too large");
    const size_t bytes = h.points * rec;
    body.ensure(bytes + rec);  // the upload starts at x's offset: it reads that many bytes past the last record
    const size_t got = std::fread(body.ptr, 1, bytes, fp);
    if (got != bytes) {
      if (std::ferror(fp)) return err = std::string("reading ") + path + ": " + std::strerror(errno), B200REG_ERR_IO;
      return format_error(err, "binary: the body has " + std::to_string(got) + " bytes, the header says " + std::to_string(bytes));
    }
    uploader.upload(body.ptr + ox, h.points, rec, oi >= 0 ? oi - ox : -1, 0.0f, dst.ptr, s);
    launches += 1;
    B200_CUDA(cudaStreamSynchronize(s));
    return B200REG_OK;
  }
  // DATA ascii. Like PCL's loop, reading stops once POINTS lines are in: the line count of each piece comes back to
  // h_state[2 + buffer] behind its kernels, and is looked at when that buffer is needed again (one piece later).
  if (h.points == 0) return B200REG_OK;
  text.ensure(PIECE + LOAD_TILE + LOAD_SPILL);
  counts.ensure(PIECE / LOAD_TILE + 1);
  state.ensure(2);
  h_state.ensure(4);
  for (auto& p : pieces) p.ensure(PIECE);
  for (cudaEvent_t& e : done) B200_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  h_state.ptr[0] = 0;
  h_state.ptr[1] = NO_ERROR;
  B200_CUDA(cudaMemcpyAsync(state.ptr, h_state.ptr, 2 * sizeof(unsigned long long), cudaMemcpyHostToDevice, s));
  unsigned long long file_off = (unsigned long long)std::ftell(fp);
  size_t carry = 0;
  const char* carry_src = nullptr;
  bool used[2] = {false, false};
  for (int b = 0;; b ^= 1) {
    if (used[b]) {
      B200_CUDA(cudaEventSynchronize(done[b]));  // the piece it held has been copied and parsed
      if (h_state.ptr[2 + b] >= h.points) break;
    }
    char* buf = pieces[b].ptr;
    if (carry) std::memcpy(buf, carry_src, carry);  // from the other buffer, whose copy only reads it
    const size_t want = PIECE - carry, got = std::fread(buf + carry, 1, want, fp);
    if (got < want && std::ferror(fp)) return err = std::string("reading ") + path + ": " + std::strerror(errno), B200REG_ERR_IO;
    const bool last = got < want;
    size_t len = carry + got;
    if (len == 0) break;
    if (!last) {
      const char* nl = static_cast<const char*>(memrchr(buf, '\n', len));
      if (!nl) {  // a line longer than a piece: an error unless POINTS lines came before it
        B200_CUDA(cudaMemcpyAsync(h_state.ptr + 2 + b, state.ptr, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
        B200_CUDA(cudaStreamSynchronize(s));
        if (h_state.ptr[2 + b] >= h.points) break;
        return format_error(err, "a line longer than " + std::to_string(PIECE) + " bytes at line " +
                                     std::to_string(line_of_offset(path, file_off)));
      }
      const size_t whole = (size_t)(nl - buf) + 1;
      carry = len - whole;
      carry_src = buf + whole;
      len = whole;
    } else {
      carry = 0;
    }
    B200_CUDA(cudaMemcpyAsync(text.ptr, buf, len, cudaMemcpyHostToDevice, s));
    used[b] = true;
    const unsigned tiles = (unsigned)((len + LOAD_TILE - 1) / LOAD_TILE);
    pcd_line_count_kernel<<<tiles, LOAD_THREADS, 0, s>>>(text.ptr, len, counts.ptr);
    B200_CUDA(cudaGetLastError());
    counter_scan_async(counts.ptr, tiles, scan_tmp, s);
    pcd_parse_kernel<<<tiles, LOAD_THREADS, 0, s>>>(text.ptr, len, counts.ptr, h.layout, h.points, file_off, dst.ptr, state.ptr);
    B200_CUDA(cudaGetLastError());
    pcd_advance_kernel<<<1, 1, 0, s>>>(state.ptr, counts.ptr + tiles);
    B200_CUDA(cudaGetLastError());
    B200_CUDA(cudaMemcpyAsync(h_state.ptr + 2 + b, state.ptr, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    B200_CUDA(cudaEventRecord(done[b], s));
    launches += 6;
    file_off += len;
    if (last) break;
  }
  B200_CUDA(cudaMemcpyAsync(h_state.ptr, state.ptr, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  B200_CUDA(cudaStreamSynchronize(s));
  const unsigned long long lines = h_state.ptr[0], bad = h_state.ptr[1];
  if (bad != NO_ERROR) {
    const std::string where = "line " + std::to_string(line_of_offset(path, bad >> 2));
    if ((bad & 3u) == PCD_LINE_COUNT)
      return format_error(err, where + ": the token count is not " + std::to_string(h.layout.n_tokens) + " (the sum of COUNT)");
    return format_error(err, where + ": a field of x, y, z or intensity is not a number");
  }
  if (lines < h.points)
    return format_error(err, std::to_string(lines) + " data lines, POINTS says " + std::to_string(h.points));
  return B200REG_OK;
}

}  // namespace b200

using namespace b200;

// one loader per device, like b200reg_encode_pcd_ascii's encoder
extern "C" int b200reg_load_pcd(int device, const char* path, float* out_xyzi, size_t capacity, size_t* n_points) {
  if (!path || !n_points || (!out_xyzi && capacity)) return B200REG_ERR_ARG;
  std::string err;
  if (capacity == 0) {
    FILE* fp = std::fopen(path, "rb");
    if (!fp) return B200REG_ERR_IO;
    PcdHeader h;
    const int rc = read_pcd_header(fp, h, err);
    std::fclose(fp);
    if (rc == B200REG_OK) *n_points = h.points;
    return rc;
  }
  struct State {
    cudaStream_t stream = nullptr;
    PcdLoader loader;
    DeviceBuffer<float4> points;
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
    size_t n = 0;
    const int rc = S.loader.load(path, S.points, &n, err, S.stream);
    if (rc != B200REG_OK) return rc;
    *n_points = n;
    if (n) {
      B200_CUDA(cudaMemcpyAsync(out_xyzi, S.points.ptr, std::min(n, capacity) * sizeof(float4), cudaMemcpyDeviceToHost, S.stream));
      B200_CUDA(cudaStreamSynchronize(S.stream));
    }
    return B200REG_OK;
  } catch (const CudaError&) {
    cudaGetLastError();
    return B200REG_ERR_CUDA;
  }
}
