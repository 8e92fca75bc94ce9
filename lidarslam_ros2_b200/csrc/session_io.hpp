// A mapping session on disk (b200sm_save_session / b200sm_load_session): the manifest's format, its writer and its strict
// parser, the binary PCD header of a submap file, and the pose graph as the reference's optimizer.save("pose_graph.g2o")
// writes it (graph_based_slam_component.cpp:319). Header-only and free of CUDA so that a CPU harness
// (tests/hostmath/session_io_host.cpp, g++ -ffp-contract=off) compiles it as scanmatcher.cu does.
//
// The directory:
//   <dir>/session.txt          the manifest below; the load reads only this and the submap files
//   <dir>/pose_graph.g2o       the graph (an export; never read back)
//   <dir>/submaps/000000.pcd   one binary PCD per submap, sensor frame, in submap order (name: the index as %06zu)
//
// The manifest is line-oriented text: single spaces between tokens, every line ended by '\n', every double printed with
// %.17g (strtod gives the same bits back, -0, subnormals and the largest finite values included). In this order:
//   b200sm_session 1
//   scan_context <num_rings> <num_sectors> <max_radius> <lidar_height>
//   submaps <n>
//   segments <m> <first_0> ... <first_m-1>
//   submap <i> <points> <distance> <pose: 16 doubles, column-major>      n lines, i = 0 .. n-1
//   odometry <k>                                                          num_adjacent_pose_cnstraints of the graph
//   loops <L>
//   loop <from> <to> <relative_pose: 16 doubles, column-major>            L lines
//   adjusted <0|1>
//   pose <i> <16 doubles, column-major>                                   n lines when adjusted is 1
//
// pose_graph.g2o is *g2o*'s OptimizableGraph::save restated (g2o is not vendored in the reference, so this cannot be
// checked against its source; see pose_graph.hpp): per submap in id order "VERTEX_SE3:QUAT id x y z qx qy qz qw " and, after
// vertex 0, "FIX 0"; then per edge in build_edges' order "EDGE_SE3:QUAT from to x y z qx qy qz qw " followed by the upper
// triangle of the identity information matrix row by row, each number followed by a space. Quaternions are
// matrix_to_quat_d's (Eigen's Quaterniond(Matrix3d)) normalised, with no sign change (toVectorQT). Numbers are printed
// like an ostream at its default precision (%g). Vertex estimates are the adjusted poses when given, the submaps' own
// otherwise; edge measurements are those b200sm_pose_adjust optimises: P_from^-1 P_to of the submaps' own poses for the
// odometry edges of every segment, then the loop edges as given.
#pragma once
#include <cerrno>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "pose_graph.hpp"
#include "scan_context.hpp"

namespace b200 {
namespace sio {

constexpr unsigned long long MAX_SUBMAP_POINTS = 1ull << 40;  // 16 TiB of records: byte counts never overflow

struct LoopEdge {
  int from, to;
  double rel[16];  // column-major
};

// Everything the manifest holds. Poses are column-major 4x4 doubles.
struct Manifest {
  ScParams sc;
  std::vector<int> seg_first{0};
  std::vector<unsigned long long> points;  // per submap
  std::vector<double> distance;            // per submap
  std::vector<double> pose;                // 16 per submap
  int k = 5;
  std::vector<LoopEdge> loops;
  bool adjusted = false;
  std::vector<double> adjusted_pose;  // 16 per submap when adjusted
  size_t n() const { return points.size(); }
};

inline std::string submap_name(size_t i) {
  char b[32];
  std::snprintf(b, sizeof b, "%06zu.pcd", i);
  return b;
}

// pcl::io::savePCDFileBinary's header for a dense PointXYZI cloud of n points (generateHeader, then "DATA binary")
inline std::string pcd_binary_header(unsigned long long n) {
  char tail[160];
  std::snprintf(tail, sizeof tail, "WIDTH %llu\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS %llu\nDATA binary\n", n, n);
  return std::string("# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z intensity\nSIZE 4 4 4 4\n"
                     "TYPE F F F F\nCOUNT 1 1 1 1\n") + tail;
}

inline void put_exact(std::string& s, double v) {
  char b[40];
  std::snprintf(b, sizeof b, " %.17g", v);
  s += b;
}

inline std::string write_manifest(const Manifest& m) {
  std::string s = "b200sm_session 1\n";
  char b[96];
  std::snprintf(b, sizeof b, "scan_context %d %d", m.sc.num_rings, m.sc.num_sectors);
  s += b;
  put_exact(s, m.sc.max_radius);
  put_exact(s, m.sc.lidar_height);
  std::snprintf(b, sizeof b, "\nsubmaps %zu\nsegments %zu", m.n(), m.seg_first.size());
  s += b;
  for (int f : m.seg_first) s += " " + std::to_string(f);
  s += "\n";
  for (size_t i = 0; i < m.n(); i++) {
    std::snprintf(b, sizeof b, "submap %zu %llu", i, m.points[i]);
    s += b;
    put_exact(s, m.distance[i]);
    for (int c = 0; c < 16; c++) put_exact(s, m.pose[16 * i + c]);
    s += "\n";
  }
  std::snprintf(b, sizeof b, "odometry %d\nloops %zu\n", m.k, m.loops.size());
  s += b;
  for (const LoopEdge& e : m.loops) {
    std::snprintf(b, sizeof b, "loop %d %d", e.from, e.to);
    s += b;
    for (int c = 0; c < 16; c++) put_exact(s, e.rel[c]);
    s += "\n";
  }
  s += m.adjusted ? "adjusted 1\n" : "adjusted 0\n";
  if (m.adjusted)
    for (size_t i = 0; i < m.n(); i++) {
      s += "pose " + std::to_string(i);
      for (int c = 0; c < 16; c++) put_exact(s, m.adjusted_pose[16 * i + c]);
      s += "\n";
    }
  return s;
}

// ---- the parser: any deviation from the format is an error naming its 1-based line ----
namespace detail {

struct Lines {
  std::vector<std::string> lines;
  size_t at = 0;  // the next line to read (0-based)
};

inline bool fail(std::string& err, size_t line, const std::string& why) {
  err = "line " + std::to_string(line) + ": " + why;
  return false;
}

// the tokens of a line: exactly one space between tokens, none leading or trailing
inline bool split(const std::string& line, std::vector<std::string>& tok) {
  tok.clear();
  size_t p = 0;
  for (;;) {
    const size_t q = line.find(' ', p);
    const std::string t = line.substr(p, q == std::string::npos ? std::string::npos : q - p);
    if (t.empty()) return false;
    tok.push_back(t);
    if (q == std::string::npos) return true;
    p = q + 1;
  }
}

// a decimal integer as printf writes it: digits only, no sign, no leading zero
inline bool parse_count(const std::string& t, unsigned long long most, unsigned long long* v) {
  if (t.empty() || t.size() > 19 || (t.size() > 1 && t[0] == '0')) return false;
  unsigned long long x = 0;
  for (char c : t) {
    if (c < '0' || c > '9') return false;
    x = x * 10 + (unsigned long long)(c - '0');
  }
  if (x > most) return false;
  *v = x;
  return true;
}

// a finite double that strtod consumes whole
inline bool parse_double(const std::string& t, double* v) {
  if (t.empty()) return false;
  char* end = nullptr;
  errno = 0;
  const double x = std::strtod(t.c_str(), &end);
  if (end != t.c_str() + t.size() || !std::isfinite(x)) return false;
  *v = x;
  return true;
}

// the next line: its keyword must be `key` and it must have `n_tok` tokens (0: any number)
inline bool next(Lines& L, const char* key, size_t n_tok, std::vector<std::string>& tok, size_t* line_no, std::string& err) {
  *line_no = L.at + 1;
  if (L.at >= L.lines.size()) return fail(err, *line_no, std::string("missing, expected '") + key + "'");
  const std::string& line = L.lines[L.at++];
  if (!split(line, tok)) return fail(err, *line_no, "tokens must be separated by single spaces");
  if (tok[0] != key) return fail(err, *line_no, std::string("expected '") + key + "', found '" + tok[0] + "'");
  if (n_tok && tok.size() != n_tok)
    return fail(err, *line_no, std::string("'") + key + "' takes " + std::to_string(n_tok - 1) + " values, found " + std::to_string(tok.size() - 1));
  return true;
}

inline bool doubles(const std::vector<std::string>& tok, size_t first, size_t count, double* out, size_t line, std::string& err) {
  for (size_t c = 0; c < count; c++)
    if (!parse_double(tok[first + c], out + c)) return fail(err, line, "'" + tok[first + c] + "' is not a finite number");
  return true;
}

}  // namespace detail

// The whole manifest, or false with err = "line N: why". m is only meaningful on success.
inline bool parse_manifest(const std::string& text, Manifest& m, std::string& err) {
  using namespace detail;
  Lines L;
  size_t p = 0;
  while (p < text.size()) {
    const size_t q = text.find('\n', p);
    if (q == std::string::npos) return fail(err, L.lines.size() + 1, "the last line has no '\\n'");
    L.lines.push_back(text.substr(p, q - p));
    p = q + 1;
  }
  std::vector<std::string> tok;
  size_t ln = 0;
  unsigned long long v = 0;
  if (!next(L, "b200sm_session", 2, tok, &ln, err)) return false;
  if (tok[1] != "1") return fail(err, ln, "version '" + tok[1] + "', this reader knows version 1");
  if (!next(L, "scan_context", 5, tok, &ln, err)) return false;
  if (!parse_count(tok[1], SC_MAX_RINGS, &v)) return fail(err, ln, "num_rings '" + tok[1] + "'");
  m.sc.num_rings = (int)v;
  if (!parse_count(tok[2], SC_MAX_SECTORS, &v)) return fail(err, ln, "num_sectors '" + tok[2] + "'");
  m.sc.num_sectors = (int)v;
  if (!doubles(tok, 3, 1, &m.sc.max_radius, ln, err) || !doubles(tok, 4, 1, &m.sc.lidar_height, ln, err)) return false;
  if (!sc_params_valid(m.sc)) return fail(err, ln, "Scan Context parameters out of range");
  if (!next(L, "submaps", 2, tok, &ln, err)) return false;
  if (!parse_count(tok[1], INT_MAX, &v) || v == 0) return fail(err, ln, "the submap count '" + tok[1] + "' is not in 1 .. 2^31 - 1");
  const size_t n = (size_t)v;
  if (!next(L, "segments", 0, tok, &ln, err)) return false;
  if (tok.size() < 2 || !parse_count(tok[1], n, &v) || v == 0) return fail(err, ln, "the segment count must be in 1 .. submaps");
  if (tok.size() != 2 + v) return fail(err, ln, "'segments' lists " + std::to_string(tok.size() - 2) + " firsts, the count says " + tok[1]);
  m.seg_first.assign(v, 0);
  for (size_t s = 0; s < m.seg_first.size(); s++) {
    if (!parse_count(tok[2 + s], INT_MAX, &v)) return fail(err, ln, "segment first '" + tok[2 + s] + "'");
    m.seg_first[s] = (int)v;
    if (s == 0 && v != 0) return fail(err, ln, "the first segment must start at submap 0");
    if (s > 0 && (int)v <= m.seg_first[s - 1]) return fail(err, ln, "segment firsts must be strictly increasing");
    if (v >= n) return fail(err, ln, "a segment starts at or past the last submap");
  }
  m.points.assign(n, 0);
  m.distance.assign(n, 0.0);
  m.pose.assign(16 * n, 0.0);
  for (size_t i = 0; i < n; i++) {
    if (!next(L, "submap", 20, tok, &ln, err)) return false;
    if (!parse_count(tok[1], ~0ull, &v) || v != i) return fail(err, ln, "submap index '" + tok[1] + "', expected " + std::to_string(i));
    if (!parse_count(tok[2], MAX_SUBMAP_POINTS, &m.points[i])) return fail(err, ln, "point count '" + tok[2] + "'");
    if (!doubles(tok, 3, 1, &m.distance[i], ln, err) || !doubles(tok, 4, 16, &m.pose[16 * i], ln, err)) return false;
  }
  if (!next(L, "odometry", 2, tok, &ln, err)) return false;
  if (!parse_count(tok[1], INT_MAX, &v) || v == 0) return fail(err, ln, "num_adjacent_pose_cnstraints '" + tok[1] + "' is not >= 1");
  m.k = (int)v;
  if (!next(L, "loops", 2, tok, &ln, err)) return false;
  if (!parse_count(tok[1], INT_MAX, &v)) return fail(err, ln, "loop edge count '" + tok[1] + "'");
  const size_t n_loops = (size_t)v;
  if (n_loops > L.lines.size()) return fail(err, ln, "more loop edges than lines in the file");
  m.loops.assign(n_loops, LoopEdge{});
  for (size_t l = 0; l < n_loops; l++) {
    if (!next(L, "loop", 19, tok, &ln, err)) return false;
    unsigned long long f = 0, t = 0;
    if (!parse_count(tok[1], n - 1, &f) || !parse_count(tok[2], n - 1, &t)) return fail(err, ln, "a loop edge end outside [0, submaps)");
    if (f == t) return fail(err, ln, "a loop edge with from == to");
    m.loops[l].from = (int)f;
    m.loops[l].to = (int)t;
    if (!doubles(tok, 3, 16, m.loops[l].rel, ln, err)) return false;
  }
  if (!next(L, "adjusted", 2, tok, &ln, err)) return false;
  if (tok[1] != "0" && tok[1] != "1") return fail(err, ln, "'adjusted' must be 0 or 1");
  m.adjusted = tok[1] == "1";
  m.adjusted_pose.clear();
  if (m.adjusted) {
    m.adjusted_pose.assign(16 * n, 0.0);
    for (size_t i = 0; i < n; i++) {
      if (!next(L, "pose", 18, tok, &ln, err)) return false;
      if (!parse_count(tok[1], ~0ull, &v) || v != i) return fail(err, ln, "pose index '" + tok[1] + "', expected " + std::to_string(i));
      if (!doubles(tok, 2, 16, &m.adjusted_pose[16 * i], ln, err)) return false;
    }
  }
  if (L.at != L.lines.size()) return fail(err, L.at + 1, "a line after the end of the manifest");
  return true;
}

// ---- pose_graph.g2o ----
struct GraphEdge {
  int from, to;
  pg::Iso Z;  // the measurement (build_edges keeps its inverse)
};

// build_edges' edges with their measurements: odometry per segment from the submaps' own poses X, then the loop edges
inline std::vector<GraphEdge> graph_edges(const std::vector<pg::Iso>& X, int k, const std::vector<int>& seg_first,
                                          const std::vector<LoopEdge>& loops) {
  std::vector<GraphEdge> E;
  const int n = (int)X.size();
  for (size_t s = 0; s < seg_first.size(); s++) {
    const int f0 = seg_first[s], f1 = s + 1 < seg_first.size() ? seg_first[s + 1] : n;
    for (int i = k + 1; i < f1 - f0; i++)
      for (int j = 0; j < k; j++) {
        const int f = f0 + i - k + j, t = f0 + i;
        E.push_back({f, t, pg::compose(pg::inverse(X[f]), X[t])});
      }
  }
  for (const LoopEdge& e : loops) E.push_back({e.from, e.to, pg::iso_from_colmajor16(e.rel)});
  return E;
}

// *g2o* internal::toVectorQT: x y z, then Quaterniond(R) normalised (qx qy qz qw), each followed by a space
inline void put_qt(std::string& s, const pg::Iso& a) {
  double q[4];
  matrix_to_quat_d(a.R, q);
  const double nq = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const double v[7] = {a.t[0], a.t[1], a.t[2], q[0] / nq, q[1] / nq, q[2] / nq, q[3] / nq};
  char b[40];
  for (double x : v) {
    std::snprintf(b, sizeof b, "%g ", x);
    s += b;
  }
}

inline std::string write_g2o(const Manifest& m) {
  const size_t n = m.n();
  std::vector<pg::Iso> X(n);
  for (size_t i = 0; i < n; i++) X[i] = pg::iso_from_colmajor16(&m.pose[16 * i]);
  std::string s;
  for (size_t i = 0; i < n; i++) {
    s += "VERTEX_SE3:QUAT " + std::to_string(i) + " ";
    put_qt(s, m.adjusted ? pg::iso_from_colmajor16(&m.adjusted_pose[16 * i]) : X[i]);
    s += "\n";
    if (i == 0) s += "FIX 0\n";
  }
  for (const GraphEdge& e : graph_edges(X, m.k, m.seg_first, m.loops)) {
    s += "EDGE_SE3:QUAT " + std::to_string(e.from) + " " + std::to_string(e.to) + " ";
    put_qt(s, e.Z);
    for (int r = 0; r < 6; r++)
      for (int c = r; c < 6; c++) s += r == c ? "1 " : "0 ";
    s += "\n";
  }
  return s;
}

}  // namespace sio
}  // namespace b200
