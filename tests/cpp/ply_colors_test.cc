// teaser::PLYReader::read(file, cloud, colors): the vertices' red, green and blue, divided by 255, from ASCII,
// binary little-endian and binary big-endian files with uchar, ushort and float channels, alpha, normals and other
// properties between them; a file without colours returns -1 and appends nothing.  The points equal the points-only
// reader's.  Host only.
// usage: ply_colors_test <scratch dir>   (prints "ok")
#include <cmath>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <iostream>
#include <string>
#include <vector>

#include "teaser/ply_io.h"

#define CHECK(c)                                                                  \
  do {                                                                            \
    if (!(c)) {                                                                   \
      std::cerr << "CHECK failed: " #c " at line " << __LINE__ << std::endl;     \
      return 1;                                                                   \
    }                                                                             \
  } while (0)

namespace {

struct Prop {
  const char* type;
  const char* name;
};

// one vertex row: a value per property, in order
using Row = std::vector<double>;

int type_bytes(const std::string& t) {
  if (t == "uchar" || t == "char") return 1;
  if (t == "ushort" || t == "short") return 2;
  if (t == "double") return 8;
  return 4;
}

void put(std::ofstream& f, const std::string& t, double v, bool big) {
  unsigned char b[8];
  const int n = type_bytes(t);
  if (t == "uchar") {
    b[0] = static_cast<uint8_t>(v);
  } else if (t == "ushort") {
    const uint16_t x = static_cast<uint16_t>(v);
    std::memcpy(b, &x, 2);
  } else if (t == "int") {
    const int32_t x = static_cast<int32_t>(v);
    std::memcpy(b, &x, 4);
  } else if (t == "double") {
    std::memcpy(b, &v, 8);
  } else {
    const float x = static_cast<float>(v);
    std::memcpy(b, &x, 4);
  }
  const uint16_t one = 1;
  const bool host_little = *reinterpret_cast<const uint8_t*>(&one) == 1;
  if (big == host_little)
    for (int i = 0; i < n / 2; ++i) std::swap(b[i], b[n - 1 - i]);
  f.write(reinterpret_cast<const char*>(b), n);
}

// a vertex element (props, rows) and, after it, a face element with one list per row
void write_ply(const std::string& path, const std::string& format, const std::vector<Prop>& props,
               const std::vector<Row>& rows) {
  std::ofstream f(path, std::ios::binary);
  f << "ply\nformat " << format << " 1.0\ncomment written by ply_colors_test\nelement vertex " << rows.size() << "\n";
  for (const Prop& p : props) f << "property " << p.type << " " << p.name << "\n";
  f << "element face 1\nproperty list uchar int vertex_indices\nend_header\n";
  const bool ascii = format == "ascii", big = format == "binary_big_endian";
  for (const Row& r : rows) {
    for (size_t k = 0; k < props.size(); ++k) {
      if (ascii) {
        f.precision(9);
        f << (k ? " " : "") << r[k];
      } else {
        put(f, props[k].type, r[k], big);
      }
    }
    if (ascii) f << "\n";
  }
  if (ascii) {
    f << "3 0 1 2\n";
  } else {
    put(f, "uchar", 3, big);
    for (int i = 0; i < 3; ++i) put(f, "int", i, big);
  }
}

}  // namespace

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  const std::string dir = argv[1];
  const int n = 5;
  const char* formats[] = {"ascii", "binary_little_endian", "binary_big_endian"};
  const char* channel_types[] = {"uchar", "ushort", "float"};
  int files = 0;
  for (const char* fmt : formats) {
    for (const char* ct : channel_types) {
      // x, y, z, a normal, red, alpha, green, an int and a double between the channels, blue, curvature
      const std::vector<Prop> props{{"float", "x"},  {"float", "y"},     {"float", "z"},      {"float", "nx"},
                                    {ct, "red"},     {ct, "alpha"},      {ct, "green"},       {"int", "label"},
                                    {"double", "q"}, {ct, "blue"},       {"float", "curvature"}};
      std::vector<Row> rows;
      std::vector<teaser::ColorRGB> want;
      for (int i = 0; i < n; ++i) {
        const double x = 0.25 * i - 1.0, y = 0.5 + 0.125 * i, z = -2.0 + 0.0625 * i;
        double r, g, b;
        if (std::string(ct) == "float") {
          r = 0.125 * i, g = 255.0, b = 1.5;  // exact in float and in the ASCII text
        } else {
          r = 40.0 * i, g = 255.0, b = std::string(ct) == "ushort" ? 1000.0 + i : 7.0 * i;
        }
        rows.push_back({x, y, z, 0.5, r, 200.0, g, -3.0, 1e-3, b, 0.25});
        want.push_back({static_cast<float>(static_cast<double>(static_cast<float>(r)) / 255.0),
                        static_cast<float>(static_cast<double>(static_cast<float>(g)) / 255.0),
                        static_cast<float>(static_cast<double>(static_cast<float>(b)) / 255.0)});
      }
      const std::string path = dir + "/colors_" + std::to_string(files++) + ".ply";
      write_ply(path, fmt, props, rows);
      teaser::PLYReader reader;
      teaser::PointCloud pts_only, pts;
      teaser::ColorCloud colors;
      pts.push_back({9.f, 9.f, 9.f});  // both overloads append
      colors.push_back({1.f, 2.f, 3.f});
      CHECK(reader.read(path, pts_only) == 0);
      CHECK(reader.read(path, pts, colors) == 0);
      CHECK(pts_only.size() == static_cast<size_t>(n) && pts.size() == static_cast<size_t>(n) + 1);
      CHECK(colors.size() == static_cast<size_t>(n) + 1 && colors[0].r == 1.f && colors[0].b == 3.f);
      for (int i = 0; i < n; ++i) {
        CHECK(pts[i + 1] == pts_only[i]);
        CHECK(pts_only[i].x == static_cast<float>(rows[i][0]) && pts_only[i].z == static_cast<float>(rows[i][2]));
        CHECK(colors[i + 1].r == want[i].r && colors[i + 1].g == want[i].g && colors[i + 1].b == want[i].b);
      }
      if (std::string(ct) == "uchar") CHECK(colors[1 + 1].g == 1.0f && colors[1 + 1].r == static_cast<float>(40.0 / 255.0));
    }
  }
  // no colours, or only some of the channels: -1 and nothing appended; the points-only reader still reads the file
  for (const char* fmt : formats) {
    const std::vector<std::vector<Prop>> variants{
        {{"float", "x"}, {"float", "y"}, {"float", "z"}},
        {{"float", "x"}, {"float", "y"}, {"float", "z"}, {"uchar", "red"}, {"uchar", "green"}, {"uchar", "alpha"}}};
    for (const auto& props : variants) {
      std::vector<Row> rows;
      for (int i = 0; i < n; ++i) {
        Row r{0.1 * i, 0.2 * i, 0.3 * i};
        while (r.size() < props.size()) r.push_back(10.0 * i);
        rows.push_back(r);
      }
      const std::string path = dir + "/plain_" + std::to_string(files++) + ".ply";
      write_ply(path, fmt, props, rows);
      teaser::PLYReader reader;
      teaser::PointCloud pts, pts_only;
      teaser::ColorCloud colors;
      CHECK(reader.read(path, pts, colors) == -1);
      CHECK(pts.empty() && colors.empty());
      CHECK(reader.read(path, pts_only) == 0 && pts_only.size() == static_cast<size_t>(n));
    }
  }
  // a missing file
  {
    teaser::PLYReader reader;
    teaser::PointCloud pts;
    teaser::ColorCloud colors;
    CHECK(reader.read(dir + "/no_such_file.ply", pts, colors) == -1 && pts.empty() && colors.empty());
  }
  std::cout << "ok" << std::endl;
  return 0;
}
