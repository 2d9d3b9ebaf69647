// teaser::voxelDownSample (teaser/voxel.h) on top of the C-ABI: marshalling only, the grid runs in libteaser_b200.so.
#include "teaser/voxel.h"

#include <cmath>
#include <stdexcept>
#include <string>

#include "teaser_b200.h"

namespace teaser {

tzr_ctx* b200_context();  // registration.cc: one context per host thread

PointCloud voxelDownSample(const PointCloud& cloud, double voxel_size, std::vector<int>* voxel_of) {
  std::vector<std::vector<int>> trace;
  std::vector<PointCloud> out = voxelDownSampleBatch({cloud}, voxel_size, voxel_of ? &trace : nullptr);
  if (voxel_of) *voxel_of = std::move(trace[0]);
  return std::move(out[0]);
}

namespace {

// both overloads: colors / colors_out null for points only
std::vector<PointCloud> voxel_batch(const std::vector<PointCloud>& clouds, const std::vector<ColorCloud>* colors,
                                    double voxel_size, std::vector<ColorCloud>* colors_out,
                                    std::vector<std::vector<int>>* voxel_of) {
  if (!(voxel_size > 0) || !std::isfinite(voxel_size))
    throw std::invalid_argument("voxelDownSample: the voxel size must be finite and > 0");
  static_assert(sizeof(PointXYZ) == 3 * sizeof(float), "PointXYZ must be three packed floats");
  static_assert(sizeof(ColorRGB) == 3 * sizeof(float), "ColorRGB must be three packed floats");
  static_assert(sizeof(int) == sizeof(int32_t), "voxel_of is filled as int32");
  const size_t B = clouds.size();
  if (colors && colors->size() != B) throw std::invalid_argument("voxelDownSample: one colour cloud per cloud");
  std::vector<PointCloud> out(B);
  if (voxel_of) voxel_of->assign(B, {});
  if (colors_out) colors_out->assign(B, {});
  // empty clouds have nothing to downsample; the others go to the device in one call
  std::vector<size_t> which;
  for (size_t b = 0; b < B; ++b) {
    if (colors && (*colors)[b].size() != clouds[b].size())
      throw std::invalid_argument("voxelDownSample: one colour per point");
    if (!clouds[b].empty()) which.push_back(b);
  }
  if (which.empty()) return out;
  const size_t K = which.size();
  std::vector<int32_t> n(K), n_out(K), status(K);
  std::vector<const float*> in(K), cin(K, nullptr);
  std::vector<std::vector<float>> buf(K), cbuf(K);
  std::vector<float*> out_p(K), cout_p(K, nullptr);
  std::vector<int32_t*> vo_p(K, nullptr);
  for (size_t k = 0; k < K; ++k) {
    const PointCloud& c = clouds[which[k]];
    n[k] = static_cast<int32_t>(c.size());
    in[k] = &c[0].x;
    buf[k].resize(3 * c.size());
    out_p[k] = buf[k].data();
    if (colors) {
      cin[k] = &(*colors)[which[k]][0].r;
      cbuf[k].resize(3 * c.size());
      cout_p[k] = cbuf[k].data();
    }
    if (voxel_of) {
      (*voxel_of)[which[k]].resize(c.size());
      vo_p[k] = reinterpret_cast<int32_t*>((*voxel_of)[which[k]].data());
    }
  }
  tzr_ctx* ctx = b200_context();
  const int Ki = static_cast<int>(K);
  int rc;
  if (colors)
    rc = K == 1 ? tzr_voxel_downsample_colors(ctx, in[0], n[0], voxel_size, out_p[0], n_out.data(), vo_p[0], cin[0],
                                              cout_p[0])
                : tzr_voxel_downsample_colors_batch(ctx, Ki, n.data(), in.data(), voxel_size, out_p.data(),
                                                    n_out.data(), vo_p.data(), status.data(), cin.data(),
                                                    cout_p.data());
  else
    rc = K == 1 ? tzr_voxel_downsample(ctx, in[0], n[0], voxel_size, out_p[0], n_out.data(), vo_p[0])
                : tzr_voxel_downsample_batch(ctx, Ki, n.data(), in.data(), voxel_size, out_p.data(), n_out.data(),
                                             vo_p.data(), status.data());
  if (rc != TZR_OK)
    throw std::runtime_error(std::string("voxelDownSample: ") + tzr_status_string(rc) + " (" + tzr_last_error(ctx) + ")");
  for (size_t k = 0; k < K; ++k) {
    PointCloud& pc = out[which[k]];
    pc.reserve(static_cast<size_t>(n_out[k]));
    for (int32_t r = 0; r < n_out[k]; ++r) pc.push_back({buf[k][3 * r], buf[k][3 * r + 1], buf[k][3 * r + 2]});
    if (colors_out) {
      ColorCloud& cc = (*colors_out)[which[k]];
      for (int32_t r = 0; r < n_out[k]; ++r) cc.push_back({cbuf[k][3 * r], cbuf[k][3 * r + 1], cbuf[k][3 * r + 2]});
    }
  }
  return out;
}

}  // namespace

std::vector<PointCloud> voxelDownSampleBatch(const std::vector<PointCloud>& clouds, double voxel_size,
                                             std::vector<std::vector<int>>* voxel_of) {
  return voxel_batch(clouds, nullptr, voxel_size, nullptr, voxel_of);
}

PointCloud voxelDownSample(const PointCloud& cloud, const ColorCloud& colors, double voxel_size, ColorCloud* colors_out,
                           std::vector<int>* voxel_of) {
  std::vector<std::vector<int>> trace;
  std::vector<ColorCloud> cols;
  const std::vector<ColorCloud> in{colors};
  std::vector<PointCloud> out = voxel_batch({cloud}, &in, voxel_size, &cols, voxel_of ? &trace : nullptr);
  if (voxel_of) *voxel_of = std::move(trace[0]);
  if (colors_out) *colors_out = std::move(cols[0]);
  return std::move(out[0]);
}

std::vector<PointCloud> voxelDownSampleBatch(const std::vector<PointCloud>& clouds,
                                             const std::vector<ColorCloud>& colors, double voxel_size,
                                             std::vector<ColorCloud>* colors_out,
                                             std::vector<std::vector<int>>* voxel_of) {
  std::vector<ColorCloud> cols;
  std::vector<PointCloud> out = voxel_batch(clouds, &colors, voxel_size, &cols, voxel_of);
  if (colors_out) *colors_out = std::move(cols);
  return out;
}

}  // namespace teaser
