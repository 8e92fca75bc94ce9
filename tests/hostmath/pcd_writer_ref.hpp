// TEST REFERENCE: pcl::io::savePCDFileASCII(path, pcl::PointCloud<pcl::PointXYZI>) restated with the standard library.
// PCL is not vendored by the reference (graph_based_slam_component.cpp:369 calls it); this follows upstream PCL 1.12's
// PCDWriter::writeASCII<PointT> and generateHeader<PointT> with savePCDFileASCII's precision 8: the header of a dense
// cloud (WIDTH = points, HEIGHT 1, default sensor origin and orientation), then per point the four FLOAT32 fields through
// an std::ostringstream at precision 8 in the classic locale, a NaN as "nan", one space between fields, the line trimmed
// (boost::trim) and ended by '\n'. Single-threaded, like PCL: it is both the byte-level checker of the device encoder and
// the CPU timing of the reference's write.
#pragma once
#include <cmath>
#include <cstddef>
#include <locale>
#include <ostream>
#include <sstream>
#include <string>

namespace pcdref {

inline std::string header_xyzi(size_t n) {
  std::ostringstream oss;
  oss.imbue(std::locale::classic());
  oss << "# .PCD v0.7 - Point Cloud Data file format"
         "\nVERSION 0.7"
         "\nFIELDS x y z intensity"
         "\nSIZE 4 4 4 4"
         "\nTYPE F F F F"
         "\nCOUNT 1 1 1 1";
  oss << "\nWIDTH " << n << "\nHEIGHT " << 1 << "\n";
  oss << "VIEWPOINT " << 0 << " " << 0 << " " << 0 << " " << 1 << " " << 0 << " " << 0 << " " << 0 << "\n";
  oss << "POINTS " << n << "\n";
  return oss.str();
}

inline void trim(std::string& s) {  // boost::trim with the classic locale's whitespace
  const char* ws = " \t\n\v\f\r";
  const size_t b = s.find_first_not_of(ws);
  if (b == std::string::npos) {
    s.clear();
    return;
  }
  s = s.substr(b, s.find_last_not_of(ws) - b + 1);
}

// xyzi: n points of (x, y, z, intensity). Returns false for an empty cloud (PCL throws "Input point cloud has no data!").
inline bool write_ascii_xyzi(std::ostream& fs, const float* xyzi, size_t n) {
  if (n == 0) return false;
  fs.precision(8);
  fs.imbue(std::locale::classic());
  fs << header_xyzi(n) << "DATA ascii\n";
  std::ostringstream stream;
  stream.precision(8);
  stream.imbue(std::locale::classic());
  for (size_t i = 0; i < n; i++) {
    for (int d = 0; d < 4; d++) {
      const float value = xyzi[4 * i + d];
      if (std::isnan(value)) stream << "nan";
      else stream << value;
      if (d < 3) stream << " ";
    }
    std::string result = stream.str();
    trim(result);
    stream.str("");
    fs << result << "\n";
  }
  return true;
}

}  // namespace pcdref
