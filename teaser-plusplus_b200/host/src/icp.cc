// teaser::PointToPointICP, teaser::PointToPlaneICP and teaser::GeneralizedICP (teaser/icp.h) on top of the C-ABI:
// marshalling only, the loop runs in libteaser_b200.so.
#include "teaser/icp.h"

#include <cstring>
#include <stdexcept>
#include <string>

#include "teaser_b200.h"

namespace teaser {

tzr_ctx* b200_context();  // registration.cc: one context per host thread

namespace {

tzr_icp_params to_c(const PointToPointICPParams& p) {
  tzr_icp_params c;
  tzr_icp_params_default(&c);
  c.max_correspondence_distance = p.max_correspondence_distance;
  c.max_iteration = p.max_iteration;
  c.relative_fitness = p.relative_fitness;
  c.relative_rmse = p.relative_rmse;
  return c;
}

tzr_similarity to_c(const RegistrationSolution& s) {
  tzr_similarity c;
  c.scale = s.scale;
  std::memcpy(c.rotation, s.rotation.data(), sizeof(c.rotation));
  for (int k = 0; k < 3; ++k) c.translation[k] = s.translation(k);
  return c;
}

}  // namespace

// shared with registration.cc's solveCloudPairs overload
void icp_result_from_c(const tzr_icp_result& r, const int32_t* corr, PointToPointICPResult* out) {
  out->solution.valid = true;
  out->solution.scale = r.transform.scale;
  std::memcpy(out->solution.rotation.data(), r.transform.rotation, sizeof(r.transform.rotation));
  for (int k = 0; k < 3; ++k) out->solution.translation(k) = r.transform.translation[k];
  out->fitness = r.fitness;
  out->inlier_rmse = r.inlier_rmse;
  out->iterations = r.iterations;
  out->converged = r.converged != 0;
  out->correspondences.clear();
  if (corr)
    for (int c = 0; c < r.n_correspondences; ++c) out->correspondences.emplace_back(corr[2 * c], corr[2 * c + 1]);
}

namespace {

// every class's refineBatch: point-to-point when dst_normals is null, generalized when src_normals is given (with
// epsilon), point-to-plane otherwise; a kernel other than L2 goes through the robust batch entries
std::vector<PointToPointICPResult> refine_batch(const char* who, const PointToPointICPParams& params,
                                                const std::vector<PointCloud>& src, const std::vector<PointCloud>& dst,
                                                const std::vector<NormalCloud>* dst_normals,
                                                const std::vector<RegistrationSolution>& init,
                                                const std::vector<NormalCloud>* src_normals = nullptr,
                                                double epsilon = 0, const RobustKernel* kernel = nullptr) {
  const size_t B = src.size();
  if (dst.size() != B || init.size() != B || (dst_normals && dst_normals->size() != B) ||
      (src_normals && src_normals->size() != B))
    throw std::invalid_argument(std::string(who) + ": one target and seed (and normal cloud) per source");
  std::vector<PointToPointICPResult> out(B);
  if (B == 0) return out;
  static_assert(sizeof(PointXYZ) == 3 * sizeof(float), "PointXYZ must be three packed floats");
  static_assert(sizeof(Normal) == 4 * sizeof(float), "Normal must be 4 packed floats");
  std::vector<int32_t> ns(B), nd(B);
  std::vector<const float*> sp(B), dp(B), np(B, nullptr), snp(B, nullptr);
  std::vector<tzr_similarity> seeds(B);
  std::vector<std::vector<int32_t>> corr(B);
  std::vector<int32_t*> corr_p(B);
  for (size_t b = 0; b < B; ++b) {
    if (src[b].empty() || dst[b].empty()) throw std::invalid_argument(std::string(who) + ": clouds must be non-empty");
    ns[b] = static_cast<int32_t>(src[b].size());
    nd[b] = static_cast<int32_t>(dst[b].size());
    sp[b] = &src[b][0].x;
    dp[b] = &dst[b][0].x;
    if (dst_normals) {
      if ((*dst_normals)[b].size() != dst[b].size())
        throw std::invalid_argument(std::string(who) + ": one normal per target point");
      np[b] = &(*dst_normals)[b][0].normal_x;
    }
    if (src_normals) {
      if ((*src_normals)[b].size() != src[b].size())
        throw std::invalid_argument(std::string(who) + ": one normal per source point");
      snp[b] = &(*src_normals)[b][0].normal_x;
    }
    seeds[b] = to_c(init[b]);
    corr[b].resize(2 * src[b].size());
    corr_p[b] = corr[b].data();
  }
  const tzr_icp_params p = to_c(params);
  std::vector<tzr_icp_result> res(B);
  tzr_ctx* ctx = b200_context();
  const int Bi = static_cast<int>(B);
  int rc;
  if (kernel && kernel->type != RobustKernel::kL2) {
    tzr_robust_kernel k;
    std::memset(&k, 0, sizeof(k));
    k.type = static_cast<int32_t>(kernel->type);
    k.k = kernel->k;
    rc = src_normals ? tzr_icp_generalized_robust_batch(ctx, &p, epsilon, Bi, ns.data(), sp.data(), snp.data(),
                                                        nd.data(), dp.data(), np.data(), seeds.data(), res.data(),
                                                        corr_p.data(), &k)
                     : tzr_icp_point_to_plane_robust_batch(ctx, &p, Bi, ns.data(), sp.data(), nd.data(), dp.data(),
                                                           np.data(), seeds.data(), res.data(), corr_p.data(), &k);
  } else if (src_normals)
    rc = B == 1 ? tzr_icp_generalized(ctx, &p, epsilon, sp[0], ns[0], snp[0], dp[0], nd[0], np[0], seeds.data(),
                                      res.data(), corr_p[0])
                : tzr_icp_generalized_batch(ctx, &p, epsilon, Bi, ns.data(), sp.data(), snp.data(), nd.data(),
                                            dp.data(), np.data(), seeds.data(), res.data(), corr_p.data());
  else if (!dst_normals)
    rc = B == 1 ? tzr_icp(ctx, &p, sp[0], ns[0], dp[0], nd[0], seeds.data(), res.data(), corr_p[0])
                : tzr_icp_batch(ctx, &p, Bi, ns.data(), sp.data(), nd.data(), dp.data(), seeds.data(), res.data(),
                                corr_p.data());
  else
    rc = B == 1 ? tzr_icp_point_to_plane(ctx, &p, sp[0], ns[0], dp[0], nd[0], np[0], seeds.data(), res.data(),
                                         corr_p[0])
                : tzr_icp_point_to_plane_batch(ctx, &p, Bi, ns.data(), sp.data(), nd.data(), dp.data(), np.data(),
                                               seeds.data(), res.data(), corr_p.data());
  if (rc != TZR_OK)
    throw std::runtime_error(std::string(who) + ": " + tzr_status_string(rc) + " (" + tzr_last_error(ctx) + ")");
  for (size_t b = 0; b < B; ++b) icp_result_from_c(res[b], corr[b].data(), &out[b]);
  return out;
}

}  // namespace

PointToPointICP::Result PointToPointICP::refine(const PointCloud& src, const PointCloud& dst,
                                                const RegistrationSolution& init) const {
  return refineBatch({src}, {dst}, {init})[0];
}

std::vector<PointToPointICP::Result> PointToPointICP::refineBatch(const std::vector<PointCloud>& src,
                                                                  const std::vector<PointCloud>& dst,
                                                                  const std::vector<RegistrationSolution>& init) const {
  return refine_batch("PointToPointICP", params_, src, dst, nullptr, init);
}

PointToPlaneICP::Result PointToPlaneICP::refine(const PointCloud& src, const PointCloud& dst,
                                                const NormalCloud& dst_normals,
                                                const RegistrationSolution& init) const {
  return refineBatch({src}, {dst}, {dst_normals}, {init})[0];
}

std::vector<PointToPlaneICP::Result> PointToPlaneICP::refineBatch(const std::vector<PointCloud>& src,
                                                                  const std::vector<PointCloud>& dst,
                                                                  const std::vector<NormalCloud>& dst_normals,
                                                                  const std::vector<RegistrationSolution>& init) const {
  return refine_batch("PointToPlaneICP", params_, src, dst, &dst_normals, init, nullptr, 0, &kernel_);
}

GeneralizedICP::Result GeneralizedICP::refine(const PointCloud& src, const PointCloud& dst,
                                              const NormalCloud& src_normals, const NormalCloud& dst_normals,
                                              const RegistrationSolution& init) const {
  return refineBatch({src}, {dst}, {src_normals}, {dst_normals}, {init})[0];
}

std::vector<GeneralizedICP::Result> GeneralizedICP::refineBatch(const std::vector<PointCloud>& src,
                                                                const std::vector<PointCloud>& dst,
                                                                const std::vector<NormalCloud>& src_normals,
                                                                const std::vector<NormalCloud>& dst_normals,
                                                                const std::vector<RegistrationSolution>& init) const {
  return refine_batch("GeneralizedICP", params_, src, dst, &dst_normals, init, &src_normals, params_.epsilon,
                      &kernel_);
}

ColoredICP::Result ColoredICP::refine(const PointCloud& src, const PointCloud& dst, const NormalCloud& dst_normals,
                                      const ColorCloud& src_colors, const ColorCloud& dst_colors,
                                      const RegistrationSolution& init) const {
  return refineBatch({src}, {dst}, {dst_normals}, {src_colors}, {dst_colors}, {init})[0];
}

std::vector<ColoredICP::Result> ColoredICP::refineBatch(const std::vector<PointCloud>& src,
                                                        const std::vector<PointCloud>& dst,
                                                        const std::vector<NormalCloud>& dst_normals,
                                                        const std::vector<ColorCloud>& src_colors,
                                                        const std::vector<ColorCloud>& dst_colors,
                                                        const std::vector<RegistrationSolution>& init) const {
  const size_t B = src.size();
  if (dst.size() != B || init.size() != B || dst_normals.size() != B || src_colors.size() != B ||
      dst_colors.size() != B)
    throw std::invalid_argument("ColoredICP: one target, normal cloud, colour clouds and seed per source");
  std::vector<Result> out(B);
  if (B == 0) return out;
  static_assert(sizeof(ColorRGB) == 3 * sizeof(float), "ColorRGB must be three packed floats");
  std::vector<int32_t> ns(B), nd(B);
  std::vector<const float*> sp(B), dp(B), np(B), scp(B), dcp(B);
  std::vector<tzr_similarity> seeds(B);
  std::vector<std::vector<int32_t>> corr(B);
  std::vector<int32_t*> corr_p(B);
  for (size_t b = 0; b < B; ++b) {
    if (src[b].empty() || dst[b].empty()) throw std::invalid_argument("ColoredICP: clouds must be non-empty");
    if (dst_normals[b].size() != dst[b].size() || dst_colors[b].size() != dst[b].size() ||
        src_colors[b].size() != src[b].size())
      throw std::invalid_argument("ColoredICP: one normal per target point and one colour per point");
    ns[b] = static_cast<int32_t>(src[b].size());
    nd[b] = static_cast<int32_t>(dst[b].size());
    sp[b] = &src[b][0].x;
    dp[b] = &dst[b][0].x;
    np[b] = &dst_normals[b][0].normal_x;
    scp[b] = &src_colors[b][0].r;
    dcp[b] = &dst_colors[b][0].r;
    seeds[b] = to_c(init[b]);
    corr[b].resize(2 * src[b].size());
    corr_p[b] = corr[b].data();
  }
  const tzr_icp_params p = to_c(params_);
  tzr_robust_kernel k;
  std::memset(&k, 0, sizeof(k));
  k.type = static_cast<int32_t>(kernel_.type);
  k.k = kernel_.k;
  const tzr_robust_kernel* kp = kernel_.type == RobustKernel::kL2 ? nullptr : &k;
  std::vector<tzr_icp_result> res(B);
  tzr_ctx* ctx = b200_context();
  const int rc = B == 1 ? tzr_icp_colored(ctx, &p, sp[0], ns[0], dp[0], nd[0], np[0], seeds.data(), res.data(),
                                          corr_p[0], scp[0], dcp[0], params_.lambda_geometric, kp)
                        : tzr_icp_colored_batch(ctx, &p, static_cast<int>(B), ns.data(), sp.data(), nd.data(),
                                                dp.data(), np.data(), seeds.data(), res.data(), corr_p.data(),
                                                scp.data(), dcp.data(), params_.lambda_geometric, kp);
  if (rc != TZR_OK)
    throw std::runtime_error(std::string("ColoredICP: ") + tzr_status_string(rc) + " (" + tzr_last_error(ctx) + ")");
  for (size_t b = 0; b < B; ++b) icp_result_from_c(res[b], corr[b].data(), &out[b]);
  return out;
}

MultiScaleICP::Result MultiScaleICP::refineBatch(const std::vector<PointCloud>& clouds,
                                                 const std::vector<ColorCloud>& colors,
                                                 const std::vector<std::pair<int, int>>& pairs,
                                                 const std::vector<RegistrationSolution>& init,
                                                 bool information) const {
  const size_t K = clouds.size(), P = pairs.size(), S = params_.scales.size();
  const bool colored = params_.method == kColored;
  if (init.size() != P) throw std::invalid_argument("MultiScaleICP: one seed per pair");
  if (colored && colors.size() != K) throw std::invalid_argument("MultiScaleICP: one colour cloud per cloud");
  static_assert(sizeof(ColorRGB) == 3 * sizeof(float), "ColorRGB must be three packed floats");
  std::vector<int32_t> n(K), pc(2 * P);
  std::vector<const float*> pts(K), cols(colored ? K : 0);
  for (size_t c = 0; c < K; ++c) {
    if (clouds[c].empty()) throw std::invalid_argument("MultiScaleICP: clouds must be non-empty");
    if (colored && colors[c].size() != clouds[c].size())
      throw std::invalid_argument("MultiScaleICP: one colour per point");
    n[c] = static_cast<int32_t>(clouds[c].size());
    pts[c] = &clouds[c][0].x;
    if (colored) cols[c] = &colors[c][0].r;
  }
  std::vector<tzr_similarity> seeds(P);
  for (size_t p = 0; p < P; ++p) {
    pc[2 * p] = pairs[p].first;
    pc[2 * p + 1] = pairs[p].second;
    seeds[p] = to_c(init[p]);
  }
  std::vector<tzr_icp_scale> sc(S);
  for (size_t s = 0; s < S; ++s) {
    const ICPScale& x = params_.scales[s];
    sc[s] = tzr_icp_scale{x.voxel_size, x.max_correspondence_distance, x.normal_search_radius, x.relative_fitness,
                          x.relative_rmse, x.max_iteration, 0};
  }
  tzr_robust_kernel k;
  std::memset(&k, 0, sizeof(k));
  k.type = static_cast<int32_t>(params_.kernel.type);
  k.k = params_.kernel.k;
  const tzr_robust_kernel* kp = params_.kernel.type == RobustKernel::kL2 ? nullptr : &k;
  std::vector<tzr_icp_result> res(P * S);
  std::vector<int32_t> nd(K * S), st(K * S), cnt(information ? P : 0);
  std::vector<double> info(information ? 36 * P : 0);
  tzr_ctx* ctx = b200_context();
  const int rc = tzr_icp_multiscale_batch(
      ctx, static_cast<int>(params_.method), static_cast<int>(S), sc.data(), static_cast<int>(K), n.data(),
      pts.data(), colored ? cols.data() : nullptr, static_cast<int>(P), pc.data(), seeds.data(), params_.epsilon,
      params_.lambda_geometric, kp, res.data(), nd.data(), st.data(), information ? info.data() : nullptr,
      information ? cnt.data() : nullptr);
  if (rc != TZR_OK && rc != TZR_ERR_TOO_LARGE)
    throw std::runtime_error(std::string("MultiScaleICP: ") + tzr_status_string(rc) + " (" + tzr_last_error(ctx) +
                             ")");
  Result out;
  out.too_large = rc == TZR_ERR_TOO_LARGE;
  out.records.assign(P, std::vector<PointToPointICPResult>(S));
  for (size_t p = 0; p < P; ++p)
    for (size_t s = 0; s < S; ++s) {
      const tzr_icp_result& r = res[p * S + s];
      icp_result_from_c(r, nullptr, &out.records[p][s]);
      out.records[p][s].solution.valid = r.transform.scale != 0;
    }
  out.n_down.assign(K, std::vector<int>(S));
  out.status.assign(K, std::vector<int>(S));
  for (size_t c = 0; c < K; ++c)
    for (size_t s = 0; s < S; ++s) {
      out.n_down[c][s] = nd[c * S + s];
      out.status[c][s] = st[c * S + s];
    }
  if (information) {
    out.information.resize(P);
    for (size_t p = 0; p < P; ++p)
      for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) out.information[p](r, c) = info[36 * p + 6 * r + c];
    out.info_counts.assign(cnt.begin(), cnt.end());
  }
  return out;
}

}  // namespace teaser
