// teaser::Matcher — same public surface as teaser/include/teaser/matcher.h:18-61 of the reference; the work
// (normalizePoints, both nearest-neighbour passes, cross check, tuple test, sort/unique: matcher.cc:21-297) runs on
// the GPU through tzr_match_correspondences (include/teaser_b200.h).
#pragma once
#include <cstdint>
#include <utility>
#include <vector>

#include "teaser/fpfh.h"
#include "teaser/geometry.h"

namespace teaser {

class Matcher {
 public:
  Matcher() = default;

  /**
   * Calculate correspondences based on given features and point clouds (matcher.h:39-43: same argument order and
   * defaults).  Returns sorted unique (source index, target index) pairs.
   */
  std::vector<std::pair<int, int>> calculateCorrespondences(const teaser::PointCloud& source_points,
                                                            const teaser::PointCloud& target_points,
                                                            const teaser::FPFHCloud& source_features,
                                                            const teaser::FPFHCloud& target_features,
                                                            bool use_absolute_scale = true, bool use_crosscheck = true,
                                                            bool use_tuple_test = true, float tuple_scale = 0);

  /// Same, for descriptors of any dimension (row-major n x dim floats).
  std::vector<std::pair<int, int>> calculateCorrespondences(const teaser::PointCloud& source_points,
                                                            const teaser::PointCloud& target_points,
                                                            const float* source_features, const float* target_features,
                                                            int dim, bool use_absolute_scale = true,
                                                            bool use_crosscheck = true, bool use_tuple_test = true,
                                                            float tuple_scale = 0);

  /**
   * calculateCorrespondences on B cloud pairs (source_points[b], target_points[b] and their descriptors) in one
   * device call.  Pair b uses the tuple seed the b-th of B consecutive single calls would use, so the result, the
   * seed afterwards and getGlobalScale() (the last non-empty pair's) are those of the B consecutive calls.
   */
  std::vector<std::vector<std::pair<int, int>>> calculateCorrespondencesBatch(
      const std::vector<teaser::PointCloud>& source_points, const std::vector<teaser::PointCloud>& target_points,
      const std::vector<teaser::FPFHCloudPtr>& source_features,
      const std::vector<teaser::FPFHCloudPtr>& target_features, bool use_absolute_scale = true,
      bool use_crosscheck = true, bool use_tuple_test = true, float tuple_scale = 0);

  /// The reference seeds the tuple test with time(NULL) (matcher.cc:225); here the seed is explicit and every call
  /// advances it, so two Matcher objects with the same seed produce the same sequence of results.
  void setTupleSeed(uint64_t seed) { tuple_seed_ = seed; }
  uint64_t getTupleSeed() const { return tuple_seed_; }

  /// Matcher::global_scale_ of the last call (matcher.cc:97-101).
  float getGlobalScale() const { return global_scale_; }

 private:
  std::vector<std::pair<int, int>> corres_;
  float global_scale_ = 1.0f;
  uint64_t tuple_seed_ = 0x7ea5e2ull;
};

}  // namespace teaser
