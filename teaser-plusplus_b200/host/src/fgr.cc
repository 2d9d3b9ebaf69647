// teaser::FastGlobalRegistration (teaser/fgr.h) on top of the C-ABI: marshalling only, FGR runs in libteaser_b200.so.
#include "teaser/fgr.h"

#include <cstring>
#include <stdexcept>
#include <string>

#include "teaser_b200.h"

namespace teaser {

tzr_ctx* b200_context();  // registration.cc: one context per host thread
void icp_result_from_c(const tzr_icp_result& r, const int32_t* corr, PointToPointICPResult* out);  // icp.cc

namespace {

tzr_fgr_params to_c(const FastGlobalRegistrationParams& p) {
  tzr_fgr_params c;
  tzr_fgr_params_default(&c);
  c.division_factor = p.division_factor;
  c.use_absolute_scale = p.use_absolute_scale ? 1 : 0;
  c.decrease_mu = p.decrease_mu ? 1 : 0;
  c.maximum_correspondence_distance = p.maximum_correspondence_distance;
  c.iteration_number = p.iteration_number;
  return c;
}

[[noreturn]] void fail(tzr_ctx* ctx, int rc) {
  throw std::runtime_error(std::string("FastGlobalRegistration: ") + tzr_status_string(rc) + " (" +
                           tzr_last_error(ctx) + ")");
}

}  // namespace

FastGlobalRegistration::Result FastGlobalRegistration::registerPair(
    const PointCloud& src, const PointCloud& dst, const std::vector<std::pair<int, int>>& corr) const {
  if (src.empty() || dst.empty()) throw std::invalid_argument("FastGlobalRegistration: clouds must be non-empty");
  std::vector<int32_t> rows(2 * corr.size()), ev(2 * src.size());
  for (size_t k = 0; k < corr.size(); ++k) {
    rows[2 * k] = corr[k].first;
    rows[2 * k + 1] = corr[k].second;
  }
  const tzr_fgr_params p = to_c(params_);
  tzr_icp_result res;
  tzr_ctx* ctx = b200_context();
  const int rc = tzr_fgr(ctx, &p, &src[0].x, static_cast<int>(src.size()), &dst[0].x, static_cast<int>(dst.size()),
                         static_cast<int>(corr.size()), rows.data(), &res, ev.data());
  if (rc != TZR_OK) fail(ctx, rc);
  Result out;
  icp_result_from_c(res, ev.data(), &out);
  return out;
}

std::vector<FastGlobalRegistration::Result> FastGlobalRegistration::registerBatch(
    const std::vector<PointCloud>& src, const std::vector<PointCloud>& dst,
    const std::vector<std::vector<std::pair<int, int>>>& corr) const {
  const size_t B = src.size();
  if (dst.size() != B || corr.size() != B)
    throw std::invalid_argument("FastGlobalRegistration: one target and one correspondence list per source");
  std::vector<Result> out(B);
  if (B == 0) return out;
  std::vector<int32_t> ns(B), nd(B), nc(B);
  std::vector<const float*> sp(B), dp(B);
  std::vector<std::vector<int32_t>> rows(B), ev(B);
  std::vector<const int32_t*> rows_p(B);
  std::vector<int32_t*> ev_p(B);
  for (size_t b = 0; b < B; ++b) {
    if (src[b].empty() || dst[b].empty())
      throw std::invalid_argument("FastGlobalRegistration: clouds must be non-empty");
    ns[b] = static_cast<int32_t>(src[b].size());
    nd[b] = static_cast<int32_t>(dst[b].size());
    nc[b] = static_cast<int32_t>(corr[b].size());
    sp[b] = &src[b][0].x;
    dp[b] = &dst[b][0].x;
    rows[b].resize(2 * corr[b].size() + 2);  // never empty: the row pointer stays valid
    for (size_t k = 0; k < corr[b].size(); ++k) {
      rows[b][2 * k] = corr[b][k].first;
      rows[b][2 * k + 1] = corr[b][k].second;
    }
    rows_p[b] = rows[b].data();
    ev[b].resize(2 * src[b].size());
    ev_p[b] = ev[b].data();
  }
  const tzr_fgr_params p = to_c(params_);
  std::vector<tzr_icp_result> res(B);
  tzr_ctx* ctx = b200_context();
  const int rc = tzr_fgr_batch(ctx, &p, static_cast<int>(B), ns.data(), sp.data(), nd.data(), dp.data(), nc.data(),
                               rows_p.data(), res.data(), ev_p.data());
  if (rc != TZR_OK) fail(ctx, rc);
  for (size_t b = 0; b < B; ++b) icp_result_from_c(res[b], ev[b].data(), &out[b]);
  return out;
}

std::vector<FastGlobalRegistration::CloudPairResult> FastGlobalRegistration::registerCloudPairs(
    const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs,
    const CloudPairParams& cp) const {
  const int K = static_cast<int>(clouds.size()), P = static_cast<int>(pairs.size());
  std::vector<CloudPairResult> out(P);
  if (P == 0) return out;
  if (K == 0) throw std::invalid_argument("FastGlobalRegistration: registerCloudPairs needs clouds");
  std::vector<int32_t> n(K), pc(2 * P), status(P);
  std::vector<const float*> pts(K);
  for (int c = 0; c < K; ++c) {
    if (clouds[c].empty()) throw std::invalid_argument("FastGlobalRegistration: clouds must be non-empty");
    n[c] = static_cast<int32_t>(clouds[c].size());
    pts[c] = &clouds[c][0].x;
  }
  std::vector<uint64_t> seeds(P);
  std::vector<std::vector<int32_t>> corr(P);
  std::vector<int32_t*> corr_p(P);
  for (int p = 0; p < P; ++p) {
    const int a = pairs[p].first, b = pairs[p].second;
    if (a < 0 || a >= K || b < 0 || b >= K)
      throw std::invalid_argument("FastGlobalRegistration: registerCloudPairs: no such cloud");
    pc[2 * p] = a;
    pc[2 * p + 1] = b;
    seeds[p] = cp.tuple_seed + 0x9E3779B97F4A7C15ull * static_cast<uint64_t>(p);  // solveCloudPairs' seeds
    corr[p].resize(2 * (static_cast<size_t>(n[a]) + n[b]));
    corr_p[p] = corr[p].data();
  }
  tzr_frontend_params f;
  tzr_frontend_params_default(&f);
  f.normal_search_radius = cp.normal_search_radius;
  f.fpfh_search_radius = cp.fpfh_search_radius;
  f.use_absolute_scale = cp.use_absolute_scale ? 1 : 0;
  f.use_crosscheck = cp.use_crosscheck ? 1 : 0;
  f.use_tuple_test = cp.use_tuple_test ? 1 : 0;
  f.tuple_scale = cp.tuple_scale;
  const tzr_fgr_params prm = to_c(params_);
  std::vector<int64_t> cnt(P);
  std::vector<float> gs(P);
  std::vector<tzr_icp_result> res(P);
  tzr_ctx* ctx = b200_context();
  const int rc = tzr_register_cloud_pairs_fgr(ctx, &f, &prm, K, n.data(), pts.data(), P, pc.data(), seeds.data(),
                                              status.data(), cnt.data(), corr_p.data(), gs.data(), res.data());
  if (rc != TZR_OK && rc != TZR_ERR_TOO_LARGE) fail(ctx, rc);
  for (int p = 0; p < P; ++p) {
    CloudPairResult& r = out[p];
    r.status = status[p];
    r.global_scale = gs[p];
    for (int64_t k = 0; k < cnt[p]; ++k) r.correspondences.emplace_back(corr[p][2 * k], corr[p][2 * k + 1]);
    r.registered = status[p] == TZR_OK;
    if (r.registered) icp_result_from_c(res[p], nullptr, &r.fgr);
  }
  return out;
}

}  // namespace teaser
