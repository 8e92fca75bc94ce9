// TEST REFERENCE: pcl::io::loadPCDFile(path, pcl::PointCloud<pcl::PointXYZI>) of a DATA ascii file, restated with the
// standard library after upstream PCL 1.12's PCDReader::readHeader / readBodyASCII and copyStringValue<float>: every line
// through std::getline, empty lines skipped, tokens from pcl::split(st, line, "\r\t ") (runs of separators compressed, no
// empty tokens), and each float token compared with "nan" ignoring case (quiet_NaN), else read by `istringstream >> float`
// in the classic locale with atof as the fallback when the stream fails. Reading stops after POINTS points.
// Two choices follow the device reader rather than PCL, because PCL's handling differs between releases: a line whose
// token count is not the sum of COUNT is an error (not a skipped point), and so is a file with fewer lines than POINTS.
// Built with the local libstdc++, so the number parsing is the real num_get / strtof. Single-threaded, like PCL: it is
// both the checker of the device reader and the CPU timing of the reference's load.
#pragma once
#include <cctype>
#include <cmath>
#include <cstdlib>
#include <istream>
#include <limits>
#include <locale>
#include <sstream>
#include <string>
#include <vector>

namespace pcdref {

// pcl::split: the maximal runs of characters not in `delims`
inline void split(std::vector<std::string>& out, const std::string& in, const char* delims) {
  out.clear();
  size_t b = in.find_first_not_of(delims);
  while (b != std::string::npos) {
    const size_t e = in.find_first_of(delims, b);
    out.push_back(in.substr(b, e == std::string::npos ? std::string::npos : e - b));
    b = e == std::string::npos ? e : in.find_first_not_of(delims, e);
  }
}

inline bool iequals_nan(const std::string& s) {  // boost::iequals(s, "nan")
  if (s.size() != 3) return false;
  const char* n = "nan";
  for (int i = 0; i < 3; i++)
    if (std::tolower(static_cast<unsigned char>(s[i])) != n[i]) return false;
  return true;
}

// copyStringValue<float>
inline float copy_string_value(const std::string& st, std::istringstream& is) {
  float value;
  if (iequals_nan(st)) {
    value = std::numeric_limits<float>::quiet_NaN();
  } else {
    is.str(st);
    is.clear();
    if (!(is >> value)) value = static_cast<float>(std::atof(st.c_str()));
  }
  return value;
}

enum { READ_OK = 0, READ_HEADER = -1, READ_TOKEN_COUNT = -2, READ_TOO_FEW = -3 };

// xyzi receives 4 floats per point (intensity 0 when the file has none). *bad_line = 1-based line number of the file
// at a READ_TOKEN_COUNT error.
inline int read_ascii_xyzi(std::istream& fs, std::vector<float>& xyzi, size_t* bad_line) {
  std::string line;
  std::vector<std::string> st, fields;
  std::vector<int> count;
  size_t nr_points = 0, line_no = 0;
  bool data = false;
  while (!data && std::getline(fs, line)) {
    line_no++;
    split(st, line, "\r\t ");
    if (st.empty() || st[0][0] == '#') continue;
    if (st[0] == "FIELDS") fields.assign(st.begin() + 1, st.end());
    else if (st[0] == "COUNT") {
      count.clear();
      for (size_t i = 1; i < st.size(); i++) count.push_back(std::atoi(st[i].c_str()));
    } else if (st[0] == "POINTS") nr_points = std::strtoull(st[1].c_str(), nullptr, 10);
    else if (st[0] == "DATA") data = st.size() > 1 && st[1] == "ascii";
  }
  if (!data) return READ_HEADER;
  if (count.empty()) count.assign(fields.size(), 1);
  int tok[4] = {-1, -1, -1, -1}, elems_per_line = 0;
  const char* names[4] = {"x", "y", "z", "intensity"};
  for (size_t f = 0; f < fields.size() && f < count.size(); f++) {
    for (int k = 0; k < 4; k++)
      if (fields[f] == names[k] && tok[k] < 0) tok[k] = elems_per_line;
    elems_per_line += count[f];
  }
  if (tok[0] < 0 || tok[1] < 0 || tok[2] < 0) return READ_HEADER;
  xyzi.assign(4 * nr_points, 0.0f);
  std::istringstream is;
  is.imbue(std::locale::classic());
  size_t idx = 0;
  while (idx < nr_points && !fs.eof()) {
    std::getline(fs, line);
    line_no++;
    if (line.empty()) continue;
    split(st, line, "\r\t ");
    if (st.size() != (size_t)elems_per_line) {
      if (bad_line) *bad_line = line_no;
      return READ_TOKEN_COUNT;
    }
    for (int k = 0; k < 4; k++)
      if (tok[k] >= 0) xyzi[4 * idx + k] = copy_string_value(st[tok[k]], is);
    idx++;
  }
  return idx == nr_points ? READ_OK : READ_TOO_FEW;
}

}  // namespace pcdref
