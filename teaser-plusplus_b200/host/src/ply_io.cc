// teaser::PLYReader / PLYWriter without tinyply (reference: teaser/src/ply_io.cc:22-130).
#include "teaser/ply_io.h"

#include <cstdint>
#include <cstring>
#include <fstream>
#include <iostream>
#include <sstream>
#include <vector>

namespace teaser {

namespace {

struct Prop {
  std::string name;
  int bytes = 0;     // size of a scalar property, 0 for a list
  char kind = 'f';   // 'f' float, 'i' signed, 'u' unsigned
  int list_count_bytes = 0, list_item_bytes = 0;
};

bool scalar_type(const std::string& t, int* bytes, char* kind) {
  static const struct {
    const char* name;
    int bytes;
    char kind;
  } table[] = {{"char", 1, 'i'},   {"int8", 1, 'i'},    {"uchar", 1, 'u'},  {"uint8", 1, 'u'},  {"short", 2, 'i'},
               {"int16", 2, 'i'},  {"ushort", 2, 'u'},  {"uint16", 2, 'u'}, {"int", 4, 'i'},    {"int32", 4, 'i'},
               {"uint", 4, 'u'},   {"uint32", 4, 'u'},  {"float", 4, 'f'},  {"float32", 4, 'f'}, {"double", 8, 'f'},
               {"float64", 8, 'f'}};
  for (const auto& e : table)
    if (t == e.name) {
      *bytes = e.bytes;
      *kind = e.kind;
      return true;
    }
  return false;
}

bool host_is_little_endian() {
  const uint16_t one = 1;
  return *reinterpret_cast<const uint8_t*>(&one) == 1;
}

double decode(const unsigned char* p, int bytes, char kind, bool swap) {
  unsigned char b[8];
  for (int i = 0; i < bytes; ++i) b[i] = swap ? p[bytes - 1 - i] : p[i];
  switch (kind) {
    case 'f':
      if (bytes == 4) {
        float f;
        std::memcpy(&f, b, 4);
        return f;
      } else {
        double d;
        std::memcpy(&d, b, 8);
        return d;
      }
    case 'i':
      if (bytes == 1) return static_cast<int8_t>(b[0]);
      if (bytes == 2) {
        int16_t v;
        std::memcpy(&v, b, 2);
        return v;
      } else {
        int32_t v;
        std::memcpy(&v, b, 4);
        return v;
      }
    default:
      if (bytes == 1) return b[0];
      if (bytes == 2) {
        uint16_t v;
        std::memcpy(&v, b, 2);
        return v;
      } else {
        uint32_t v;
        std::memcpy(&v, b, 4);
        return v;
      }
  }
}

// Both PLYReader::read overloads: the vertex element's x, y, z into cloud and, with colors, its red, green and blue
// divided by 255 (Open3D's ReadColorCallback) into colors.  A file without the channels asked for appends nothing.
int read_vertices(const std::string& file_name, PointCloud& cloud, ColorCloud* colors) {
  std::ifstream f(file_name, std::ios::binary);
  if (!f) {
    std::cerr << "Failed to open " << file_name << std::endl;
    return -1;
  }
  std::string line;
  if (!std::getline(f, line) || line.substr(0, 3) != "ply") return -1;
  enum { ASCII, LE, BE } fmt = ASCII;
  struct Element {
    std::string name;
    long count = 0;
    std::vector<Prop> props;
  };
  std::vector<Element> elements;
  bool header_done = false;
  while (std::getline(f, line)) {
    if (!line.empty() && line.back() == '\r') line.pop_back();
    std::istringstream is(line);
    std::string key;
    is >> key;
    if (key == "format") {
      std::string v;
      is >> v;
      if (v == "ascii") fmt = ASCII;
      else if (v == "binary_little_endian") fmt = LE;
      else if (v == "binary_big_endian") fmt = BE;
      else return -1;
    } else if (key == "element") {
      Element e;
      is >> e.name >> e.count;
      elements.push_back(e);
    } else if (key == "property") {
      if (elements.empty()) return -1;
      Prop p;
      std::string t;
      is >> t;
      if (t == "list") {
        std::string ct, it;
        is >> ct >> it >> p.name;
        char k;
        if (!scalar_type(ct, &p.list_count_bytes, &k) || !scalar_type(it, &p.list_item_bytes, &k)) return -1;
      } else {
        if (!scalar_type(t, &p.bytes, &p.kind)) return -1;
        is >> p.name;
      }
      elements.back().props.push_back(p);
    } else if (key == "end_header") {
      header_done = true;
      break;
    }
  }
  if (!header_done) return -1;
  const bool swap = (fmt == LE) != host_is_little_endian();
  bool found_vertices = false;
  for (const Element& e : elements) {
    // slot of every property: 0 ... 2 x, y, z, 3 ... 5 red, green, blue, -1 skipped
    static const char* const names[6] = {"x", "y", "z", "red", "green", "blue"};
    std::vector<int> slot(e.props.size(), -1);
    bool seen[6] = {false, false, false, false, false, false};
    for (size_t k = 0; k < e.props.size(); ++k)
      for (int c = 0; c < (colors ? 6 : 3); ++c)
        if (e.props[k].name == names[c]) {
          slot[k] = c;
          seen[c] = true;
        }
    const bool is_vertex = e.name == "vertex";
    if (is_vertex && !(seen[0] && seen[1] && seen[2] && (!colors || (seen[3] && seen[4] && seen[5])))) return -1;
    for (long r = 0; r < e.count; ++r) {
      double xyz[6] = {0, 0, 0, 0, 0, 0};
      if (fmt == ASCII) {
        if (!std::getline(f, line)) return -1;
        std::istringstream is(line);
        for (size_t k = 0; k < e.props.size(); ++k) {
          const Prop& p = e.props[k];
          if (p.bytes == 0) {  // list: count followed by the items
            long cnt = 0;
            is >> cnt;
            double skip;
            for (long q = 0; q < cnt; ++q) is >> skip;
          } else {
            double v = 0;
            is >> v;
            if (slot[k] >= 0) xyz[slot[k]] = v;
          }
        }
        if (is_vertex && !is) return -1;
      } else {
        unsigned char buf[8];
        for (size_t k = 0; k < e.props.size(); ++k) {
          const Prop& p = e.props[k];
          if (p.bytes == 0) {
            if (!f.read(reinterpret_cast<char*>(buf), p.list_count_bytes)) return -1;
            const long cnt = static_cast<long>(decode(buf, p.list_count_bytes, 'u', swap));
            f.seekg(static_cast<std::streamoff>(cnt) * p.list_item_bytes, std::ios::cur);
          } else {
            if (!f.read(reinterpret_cast<char*>(buf), p.bytes)) return -1;
            const double v = decode(buf, p.bytes, p.kind, swap);
            if (slot[k] >= 0) xyz[slot[k]] = v;
          }
        }
      }
      if (is_vertex) {
        cloud.push_back({static_cast<float>(xyz[0]), static_cast<float>(xyz[1]), static_cast<float>(xyz[2])});
        if (colors)
          colors->push_back({static_cast<float>(xyz[3] / 255.0), static_cast<float>(xyz[4] / 255.0),
                             static_cast<float>(xyz[5] / 255.0)});
      }
    }
    if (is_vertex) {
      found_vertices = true;
      break;  // nothing after the vertices is needed
    }
  }
  return found_vertices ? 0 : -1;
}

}  // namespace

int PLYReader::read(const std::string& file_name, PointCloud& cloud) { return read_vertices(file_name, cloud, nullptr); }

int PLYReader::read(const std::string& file_name, PointCloud& cloud, ColorCloud& colors) {
  return read_vertices(file_name, cloud, &colors);
}

int PLYWriter::write(const std::string& file_name, const PointCloud& cloud, bool binary_mode) {
  std::ofstream f(file_name, std::ios::binary);
  if (!f) {
    std::cerr << "Failed to open " << file_name << " for writing" << std::endl;
    return -1;
  }
  const bool le = host_is_little_endian();
  f << "ply\nformat " << (binary_mode ? (le ? "binary_little_endian" : "binary_big_endian") : "ascii") << " 1.0\n"
    << "element vertex " << cloud.size() << "\nproperty float x\nproperty float y\nproperty float z\nend_header\n";
  if (binary_mode) {
    for (const PointXYZ& p : cloud) f.write(reinterpret_cast<const char*>(&p.x), 3 * sizeof(float));
  } else {
    f.precision(9);  // enough digits to round-trip a float
    for (const PointXYZ& p : cloud) f << p.x << " " << p.y << " " << p.z << "\n";
  }
  return f ? 0 : -1;
}

}  // namespace teaser
