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

std::vector<std::vector<std::pair<int, int>>> Matcher::calculateCorrespondencesBatch(
    const std::vector<PointCloud>& source_points, const std::vector<PointCloud>& target_points,
    const std::vector<FPFHCloudPtr>& source_features, const std::vector<FPFHCloudPtr>& target_features,
    bool use_absolute_scale, bool use_crosscheck, bool use_tuple_test, float tuple_scale) {
  const size_t B = source_points.size();
  if (target_points.size() != B || source_features.size() != B || target_features.size() != B)
    throw std::invalid_argument("teaser::Matcher: one point cloud and one descriptor cloud per side and pair");
  std::vector<std::vector<std::pair<int, int>>> result(B);
  // pairs with an empty side return no correspondences and leave the seed alone, like the single call
  std::vector<int32_t> ns, nd;
  std::vector<const float *> sp, dp, sf, df;
  std::vector<uint64_t> seeds;
  std::vector<size_t> which;
  for (size_t b = 0; b < B; ++b) {
    if (!source_features[b] || !target_features[b] || source_features[b]->size() != source_points[b].size() ||
        target_features[b]->size() != target_points[b].size())
      throw std::invalid_argument("teaser::Matcher: one descriptor per point is required");
    if (source_points[b].empty() || target_points[b].empty()) continue;
    which.push_back(b);
    ns.push_back(static_cast<int32_t>(source_points[b].size()));
    nd.push_back(static_cast<int32_t>(target_points[b].size()));
    sp.push_back(&source_points[b][0].x);
    dp.push_back(&target_points[b][0].x);
    sf.push_back(source_features[b]->data());
    df.push_back(target_features[b]->data());
    seeds.push_back(tuple_seed_ + 0x9E3779B97F4A7C15ull * (uint64_t)seeds.size());
  }
  corres_.clear();
  const int nb = static_cast<int>(which.size());
  if (nb == 0) return result;
  std::vector<std::vector<int32_t>> pairs(nb);
  std::vector<int32_t*> pair_ptrs(nb);
  std::vector<int64_t> capacity(nb), n_pairs(nb);
  std::vector<float> scales(nb);
  for (int k = 0; k < nb; ++k) {
    capacity[k] = static_cast<int64_t>(ns[k]) + nd[k];
    pairs[k].resize(2 * static_cast<size_t>(capacity[k]));
    pair_ptrs[k] = pairs[k].data();
  }
  tzr_ctx* ctx = b200_context();
  const int rc = tzr_match_correspondences_batch(ctx, nb, ns.data(), sp.data(), nd.data(), dp.data(), sf.data(),
                                                 df.data(), 33, use_absolute_scale, use_crosscheck, use_tuple_test,
                                                 tuple_scale, seeds.data(), pair_ptrs.data(), capacity.data(),
                                                 n_pairs.data(), scales.data());
  if (rc != TZR_OK)
    throw std::runtime_error(std::string("teaser::Matcher (GPU): ") + tzr_status_string(rc) + " (" +
                             tzr_last_error(ctx) + ")");
  tuple_seed_ += 0x9E3779B97F4A7C15ull * (uint64_t)nb;
  global_scale_ = scales[nb - 1];
  for (int k = 0; k < nb; ++k) {
    auto& out = result[which[k]];
    out.reserve(static_cast<size_t>(n_pairs[k]));
    for (int64_t c = 0; c < n_pairs[k]; ++c) out.emplace_back(pairs[k][2 * c], pairs[k][2 * c + 1]);
  }
  corres_ = result[B - 1];
  return result;
}

std::vector<FPFHCloudPtr> FPFHEstimation::computeFPFHFeaturesBatch(const std::vector<PointCloud>& clouds,
                                                                   double normal_search_radius,
                                                                   double fpfh_search_radius) {
  const size_t B = clouds.size();
  std::vector<FPFHCloudPtr> result(B);
  std::vector<NormalCloud> normals(B);
  std::vector<int32_t> n;
  std::vector<const float*> pts;
  std::vector<float*> out, nor;
  for (size_t b = 0; b < B; ++b) {
    result[b].reset(new FPFHCloud());
    if (clouds[b].empty()) continue;  // an empty cloud has no descriptors, like the single call
    result[b]->resize(clouds[b].size());
    normals[b].resize(clouds[b].size());
    n.push_back(static_cast<int32_t>(clouds[b].size()));
    pts.push_back(&clouds[b][0].x);
    out.push_back((*result[b])[0].histogram);
    nor.push_back(&normals[b][0].normal_x);
  }
  if (!n.empty()) {
    tzr_ctx* ctx = b200_context();
    const int rc = tzr_compute_fpfh_batch(ctx, static_cast<int>(n.size()), n.data(), pts.data(), normal_search_radius,
                                          fpfh_search_radius, out.data(), nor.data(), nullptr);
    if (rc != TZR_OK)
      throw std::runtime_error(std::string("teaser::FPFHEstimation (GPU): ") + tzr_status_string(rc) + " (" +
                               tzr_last_error(ctx) + ")");
  }
  if (B) normals_ = normals[B - 1];
  return result;
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
