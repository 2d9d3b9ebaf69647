// PLY reader / writer of the TEASER++ public API (mirrors teaser/include/teaser/ply_io.h:15-49 of the reference, which
// wraps tinyply).  Self-contained: parses the `vertex` element of ASCII, binary_little_endian and binary_big_endian
// files with scalar properties of any PLY type and takes x, y, z as floats; other elements are ignored.
#pragma once
#include <string>

#include "teaser/geometry.h"

namespace teaser {

class PLYReader {
 public:
  PLYReader() {}
  /// Reads the vertices of a PLY file into `cloud` (appending).  Returns 0 on success, -1 on failure (ply_io.cc:22-81).
  int read(const std::string& file_name, PointCloud& cloud);
  /// The same, plus the vertices' red, green and blue (any scalar type, each divided by 255 as Open3D reads them, so
  /// uchar colours land in [0, 1]) appended to `colors`, one per point.  A vertex element without all three channels
  /// returns -1 and appends nothing.
  int read(const std::string& file_name, PointCloud& cloud, ColorCloud& colors);
};

class PLYWriter {
 public:
  PLYWriter() {}
  /// Writes `cloud` as float x, y, z vertices; binary_mode selects binary_little_endian.  Returns 0 on success.
  int write(const std::string& file_name, const PointCloud& cloud, bool binary_mode = false);
};

}  // namespace teaser
