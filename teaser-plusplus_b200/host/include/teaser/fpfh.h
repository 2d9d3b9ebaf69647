// Descriptor containers of the TEASER++ public API (mirrors teaser/include/teaser/fpfh.h:19-21 of the reference, where
// FPFHCloud is pcl::PointCloud<pcl::FPFHSignature33>).  PCL is not a dependency of the GPU path: the two types below
// have the layout the matcher needs (33 floats per point, `histogram` member like pcl::FPFHSignature33, a
// std::vector-like cloud), so code that fills or iterates descriptors compiles unchanged.  FPFHEstimation keeps the
// reference's computeFPFHFeatures / getNormals (fpfh.h:23-57); the work (PCL's NormalEstimationOMP + FPFHEstimationOMP
// in the reference, fpfh.cc:15-43) runs on the GPU through tzr_compute_fpfh.  getImplPointer() (the raw PCL estimator)
// has no counterpart.
#pragma once
#include <cstddef>
#include <memory>
#include <vector>

#include "teaser/geometry.h"

namespace teaser {

struct FPFHSignature33 {
  float histogram[33];
  static int descriptorSize() { return 33; }
};

class FPFHCloud {
 public:
  using value_type = FPFHSignature33;
  using storage = std::vector<FPFHSignature33>;
  using iterator = storage::iterator;
  using const_iterator = storage::const_iterator;

  iterator begin() { return pts_.begin(); }
  iterator end() { return pts_.end(); }
  const_iterator begin() const { return pts_.begin(); }
  const_iterator end() const { return pts_.end(); }
  std::size_t size() const { return pts_.size(); }
  bool empty() const { return pts_.empty(); }
  void resize(std::size_t n) { pts_.resize(n); }
  void reserve(std::size_t n) { pts_.reserve(n); }
  void push_back(const FPFHSignature33& f) { pts_.push_back(f); }
  void clear() { pts_.clear(); }
  FPFHSignature33& operator[](std::size_t i) { return pts_[i]; }
  const FPFHSignature33& operator[](std::size_t i) const { return pts_[i]; }
  const float* data() const { return pts_.empty() ? nullptr : pts_[0].histogram; }  // size() x 33 row-major floats

 private:
  storage pts_;
};

using FPFHCloudPtr = std::shared_ptr<FPFHCloud>;

/// Layout-compatible stand-in for pcl::Normal's public fields.
struct Normal {
  float normal_x, normal_y, normal_z, curvature;
};
using NormalCloud = std::vector<Normal>;



class FPFHEstimation {
 public:
  FPFHEstimation() = default;

  /**
   * Compute FPFH features (fpfh.h:39-41, same defaults).
   * @param normal_search_radius Radius for estimating normals
   * @param fpfh_search_radius Radius for calculating FPFH (needs to be at least normalSearchRadius)
   */
  FPFHCloudPtr computeFPFHFeatures(const PointCloud& input_cloud, double normal_search_radius = 0.03,
                                   double fpfh_search_radius = 0.05);

  /// The normal vectors of the input cloud that were used in the calculation of FPFH (fpfh.h:55).
  NormalCloud getNormals() { return normals_; }

 private:
  NormalCloud normals_;
};

}  // namespace teaser
