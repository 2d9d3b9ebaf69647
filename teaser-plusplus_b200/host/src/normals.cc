// teaser::estimateNormals (teaser/normals.h) on top of the C-ABI: marshalling only, the search runs in libteaser_b200.so.
#include "teaser/normals.h"

#include <stdexcept>
#include <string>

#include "teaser_b200.h"

namespace teaser {

tzr_ctx* b200_context();  // registration.cc: one context per host thread

NormalCloud estimateNormals(const PointCloud& cloud, double normal_search_radius) {
  return estimateNormalsBatch({cloud}, normal_search_radius)[0];
}

std::vector<NormalCloud> estimateNormalsBatch(const std::vector<PointCloud>& clouds, double normal_search_radius) {
  static_assert(sizeof(PointXYZ) == 3 * sizeof(float), "PointXYZ must be three packed floats");
  static_assert(sizeof(Normal) == 4 * sizeof(float), "Normal must be 4 packed floats");
  const size_t B = clouds.size();
  std::vector<NormalCloud> out(B);
  // empty clouds have no normals; the others go to the device in one call
  std::vector<int32_t> n;
  std::vector<const float*> pts;
  std::vector<float*> nor;
  for (size_t b = 0; b < B; ++b) {
    if (clouds[b].empty()) continue;
    out[b].resize(clouds[b].size());
    n.push_back(static_cast<int32_t>(clouds[b].size()));
    pts.push_back(&clouds[b][0].x);
    nor.push_back(&out[b][0].normal_x);
  }
  if (n.empty()) return out;
  tzr_ctx* ctx = b200_context();
  const int rc = n.size() == 1
                     ? tzr_estimate_normals(ctx, pts[0], n[0], normal_search_radius, nor[0])
                     : tzr_estimate_normals_batch(ctx, static_cast<int>(n.size()), n.data(), pts.data(),
                                                  normal_search_radius, nor.data(), nullptr);
  if (rc != TZR_OK)
    throw std::runtime_error(std::string("estimateNormals: ") + tzr_status_string(rc) + " (" + tzr_last_error(ctx) +
                             ")");
  return out;
}

std::vector<std::array<double, 3>> estimateColorGradients(const PointCloud& cloud, const NormalCloud& normals,
                                                          const ColorCloud& colors, double radius) {
  return estimateColorGradientsBatch({cloud}, {normals}, {colors}, radius)[0];
}

std::vector<std::vector<std::array<double, 3>>> estimateColorGradientsBatch(const std::vector<PointCloud>& clouds,
                                                                          const std::vector<NormalCloud>& normals,
                                                                          const std::vector<ColorCloud>& colors,
                                                                          double radius) {
  static_assert(sizeof(ColorRGB) == 3 * sizeof(float), "ColorRGB must be three packed floats");
  static_assert(sizeof(std::array<double, 3>) == 3 * sizeof(double), "a gradient must be three packed doubles");
  const size_t B = clouds.size();
  if (normals.size() != B || colors.size() != B)
    throw std::invalid_argument("estimateColorGradients: one normal cloud and one colour cloud per cloud");
  std::vector<std::vector<std::array<double, 3>>> out(B);
  std::vector<int32_t> n;
  std::vector<const float*> pts, nor, col;
  std::vector<double*> grad;
  for (size_t b = 0; b < B; ++b) {
    if (normals[b].size() != clouds[b].size() || colors[b].size() != clouds[b].size())
      throw std::invalid_argument("estimateColorGradients: one normal and one colour per point");
    if (clouds[b].empty()) continue;
    out[b].resize(clouds[b].size());
    n.push_back(static_cast<int32_t>(clouds[b].size()));
    pts.push_back(&clouds[b][0].x);
    nor.push_back(&normals[b][0].normal_x);
    col.push_back(&colors[b][0].r);
    grad.push_back(out[b][0].data());
  }
  if (n.empty()) return out;
  tzr_ctx* ctx = b200_context();
  const int rc = n.size() == 1 ? tzr_estimate_color_gradients(ctx, pts[0], n[0], nor[0], col[0], radius, grad[0])
                               : tzr_estimate_color_gradients_batch(ctx, static_cast<int>(n.size()), n.data(),
                                                                    pts.data(), nor.data(), col.data(), radius,
                                                                    grad.data(), nullptr);
  if (rc != TZR_OK)
    throw std::runtime_error(std::string("estimateColorGradients: ") + tzr_status_string(rc) + " (" +
                             tzr_last_error(ctx) + ")");
  return out;
}

}  // namespace teaser
