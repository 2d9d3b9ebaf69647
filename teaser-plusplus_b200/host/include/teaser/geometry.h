// Point containers of the TEASER++ public API (mirrors teaser/include/teaser/geometry.h:15-70 of the
// reference: PointXYZ is three floats, PointCloud is a std::vector-like container of them).
#pragma once
#include <cstddef>
#include <vector>

namespace teaser {

struct PointXYZ {
  float x, y, z;
  friend bool operator==(const PointXYZ& a, const PointXYZ& b) { return a.x == b.x && a.y == b.y && a.z == b.z; }
  friend bool operator!=(const PointXYZ& a, const PointXYZ& b) { return !(a == b); }
};

// One point's colour (r, g, b as floats, any range; Open3D uses [0, 1]): coloured ICP and voxel downsampling with
// colours (teaser/icp.h, teaser/voxel.h).
struct ColorRGB {
  float r, g, b;
};
using ColorCloud = std::vector<ColorRGB>;

class PointCloud {
 public:
  using value_type = PointXYZ;
  using reference = PointXYZ&;
  using const_reference = const PointXYZ&;
  using storage = std::vector<PointXYZ>;
  using difference_type = storage::difference_type;
  using size_type = storage::size_type;
  using iterator = storage::iterator;
  using const_iterator = storage::const_iterator;

  PointCloud() = default;
  iterator begin() { return pts_.begin(); }
  iterator end() { return pts_.end(); }
  const_iterator begin() const { return pts_.begin(); }
  const_iterator end() const { return pts_.end(); }
  std::size_t size() const { return pts_.size(); }
  void reserve(std::size_t n) { pts_.reserve(n); }
  bool empty() const { return pts_.empty(); }
  PointXYZ& operator[](std::size_t i) { return pts_[i]; }
  const PointXYZ& operator[](std::size_t i) const { return pts_[i]; }
  PointXYZ& at(std::size_t i) { return pts_.at(i); }
  const PointXYZ& at(std::size_t i) const { return pts_.at(i); }
  PointXYZ& front() { return pts_.front(); }
  const PointXYZ& front() const { return pts_.front(); }
  PointXYZ& back() { return pts_.back(); }
  const PointXYZ& back() const { return pts_.back(); }
  void push_back(const PointXYZ& p) { pts_.push_back(p); }
  void clear() { pts_.clear(); }

 private:
  storage pts_;
};

}  // namespace teaser
