// teaser::Matcher façade: forwards to the C-ABI (no CPU implementation behind it).
#include "teaser/matcher.h"

#include <stdexcept>
#include <string>

#include "teaser_b200.h"

namespace teaser {

tzr_ctx* b200_context();  // registration.cc: one context per host thread

std::vector<std::pair<int, int>> Matcher::calculateCorrespondences(const PointCloud& source_points,
                                                                   const PointCloud& target_points,
                                                                   const FPFHCloud& source_features,
                                                                   const FPFHCloud& target_features,
                                                                   bool use_absolute_scale, bool use_crosscheck,
                                                                   bool use_tuple_test, float tuple_scale) {
  if (source_features.size() != source_points.size() || target_features.size() != target_points.size())
    throw std::invalid_argument("teaser::Matcher: one descriptor per point is required");
  return calculateCorrespondences(source_points, target_points, source_features.data(), target_features.data(), 33,
                                  use_absolute_scale, use_crosscheck, use_tuple_test, tuple_scale);
}

std::vector<std::pair<int, int>> Matcher::calculateCorrespondences(const PointCloud& source_points,
                                                                   const PointCloud& target_points,
                                                                   const float* source_features,
                                                                   const float* target_features, int dim,
                                                                   bool use_absolute_scale, bool use_crosscheck,
                                                                   bool use_tuple_test, float tuple_scale) {
  corres_.clear();
  const int ns = static_cast<int>(source_points.size()), nd = static_cast<int>(target_points.size());
  if (ns == 0 || nd == 0) return corres_;
  static_assert(sizeof(PointXYZ) == 3 * sizeof(float), "PointXYZ must be three packed floats");
  tzr_ctx* ctx = b200_context();
  std::vector<int32_t> pairs(2 * (static_cast<size_t>(ns) + nd));
  int64_t n_pairs = 0;
  const int rc = tzr_match_correspondences(ctx, &source_points[0].x, ns, &target_points[0].x, nd, source_features,
                                           target_features, dim, use_absolute_scale, use_crosscheck, use_tuple_test,
                                           tuple_scale, tuple_seed_, pairs.data(), static_cast<int64_t>(ns) + nd,
                                           &n_pairs, &global_scale_);
  if (rc != TZR_OK)
    throw std::runtime_error(std::string("teaser::Matcher (GPU): ") + tzr_status_string(rc) + " (" +
                             tzr_last_error(ctx) + ")");
  tuple_seed_ += 0x9E3779B97F4A7C15ull;  // a fresh stream for the next call, like successive time(NULL) seeds
  corres_.reserve(static_cast<size_t>(n_pairs));
  for (int64_t c = 0; c < n_pairs; ++c) corres_.emplace_back(pairs[2 * c], pairs[2 * c + 1]);
  return corres_;
}

FPFHCloudPtr FPFHEstimation::computeFPFHFeatures(const PointCloud& input_cloud, double normal_search_radius,
                                                 double fpfh_search_radius) {
  FPFHCloudPtr descriptors(new FPFHCloud());
  normals_.clear();
  const int n = static_cast<int>(input_cloud.size());
  if (n == 0) return descriptors;
  static_assert(sizeof(FPFHSignature33) == 33 * sizeof(float), "FPFHSignature33 must be 33 packed floats");
  static_assert(sizeof(Normal) == 4 * sizeof(float), "Normal must be 4 packed floats");
  descriptors->resize(n);
  normals_.resize(n);
  tzr_ctx* ctx = b200_context();
  const int rc = tzr_compute_fpfh(ctx, &input_cloud[0].x, n, normal_search_radius, fpfh_search_radius,
                                  (*descriptors)[0].histogram, &normals_[0].normal_x);
  if (rc != TZR_OK)
    throw std::runtime_error(std::string("teaser::FPFHEstimation (GPU): ") + tzr_status_string(rc) + " (" +
                             tzr_last_error(ctx) + ")");
  return descriptors;
}

}  // namespace teaser
