// teaser::RANSACRegistration (teaser/ransac.h) on top of the C-ABI: marshalling only, RANSAC runs in libteaser_b200.so.
#include "teaser/ransac.h"

#include <cstring>
#include <stdexcept>
#include <string>

#include "teaser_b200.h"

namespace teaser {

tzr_ctx* b200_context();  // registration.cc: one context per host thread
void icp_result_from_c(const tzr_icp_result& r, const int32_t* corr, PointToPointICPResult* out);  // icp.cc

namespace {

tzr_ransac_params to_c(const RANSACRegistrationParams& p) {
  tzr_ransac_params c;
  tzr_ransac_params_default(&c);
  c.max_correspondence_distance = p.max_correspondence_distance;
  c.ransac_n = p.ransac_n;
  c.max_iteration = p.max_iteration;
  c.confidence = p.confidence;
  c.check_edge_length = p.check_edge_length ? 1 : 0;
  c.edge_length_similarity = p.edge_length_similarity;
  c.check_distance = p.check_distance ? 1 : 0;
  c.distance_threshold = p.distance_threshold;
  c.check_normal = p.check_normal ? 1 : 0;
  c.normal_angle_threshold = p.normal_angle_threshold;
  return c;
}

RANSACInfo info_of(const tzr_ransac_info& c) {
  RANSACInfo i;
  i.drawn = c.drawn;
  i.passed = c.passed;
  i.winner = c.winner;
  i.inliers = c.inliers;
  i.usable = c.usable;
  i.rmse = c.rmse;
  return i;
}

[[noreturn]] void fail(tzr_ctx* ctx, int rc) {
  throw std::runtime_error(std::string("RANSACRegistration: ") + tzr_status_string(rc) + " (" + tzr_last_error(ctx) +
                           ")");
}

const float* normals_of(const NormalCloud* n, size_t points) {
  if (!n) return nullptr;
  if (n->size() != points) throw std::invalid_argument("RANSACRegistration: one normal per point is required");
  return n->empty() ? nullptr : &(*n)[0].normal_x;
}

}  // namespace

RANSACRegistration::Result RANSACRegistration::registerPair(const PointCloud& src, const PointCloud& dst,
                                                            const std::vector<std::pair<int, int>>& corr,
                                                            uint64_t seed, const NormalCloud* src_normals,
                                                            const NormalCloud* dst_normals, RANSACInfo* info) const {
  std::vector<RANSACInfo> infos;
  std::vector<NormalCloud> sn, dn;
  if (src_normals) sn.push_back(*src_normals);
  if (dst_normals) dn.push_back(*dst_normals);
  const std::vector<Result> r = registerBatch({src}, {dst}, {corr}, {seed}, sn, dn, info ? &infos : nullptr);
  if (info) *info = infos[0];
  return r[0];
}

std::vector<RANSACRegistration::Result> RANSACRegistration::registerBatch(
    const std::vector<PointCloud>& src, const std::vector<PointCloud>& dst,
    const std::vector<std::vector<std::pair<int, int>>>& corr, const std::vector<uint64_t>& seeds,
    const std::vector<NormalCloud>& src_normals, const std::vector<NormalCloud>& dst_normals,
    std::vector<RANSACInfo>* info) const {
  const size_t B = src.size();
  if (dst.size() != B || corr.size() != B)
    throw std::invalid_argument("RANSACRegistration: one target and one correspondence list per source");
  if (!seeds.empty() && seeds.size() != B) throw std::invalid_argument("RANSACRegistration: one seed per problem");
  if ((!src_normals.empty() && src_normals.size() != B) || (!dst_normals.empty() && dst_normals.size() != B))
    throw std::invalid_argument("RANSACRegistration: one normal cloud per problem");
  std::vector<Result> out(B);
  if (info) info->assign(B, RANSACInfo());
  if (B == 0) return out;
  std::vector<int32_t> ns(B), nd(B), nc(B);
  std::vector<const float*> sp(B), dp(B), snp(B), dnp(B);
  std::vector<std::vector<int32_t>> rows(B), ev(B);
  std::vector<const int32_t*> rows_p(B);
  std::vector<int32_t*> ev_p(B);
  for (size_t b = 0; b < B; ++b) {
    if (src[b].empty() || dst[b].empty()) throw std::invalid_argument("RANSACRegistration: clouds must be non-empty");
    ns[b] = static_cast<int32_t>(src[b].size());
    nd[b] = static_cast<int32_t>(dst[b].size());
    nc[b] = static_cast<int32_t>(corr[b].size());
    sp[b] = &src[b][0].x;
    dp[b] = &dst[b][0].x;
    if (!src_normals.empty()) snp[b] = normals_of(&src_normals[b], src[b].size());
    if (!dst_normals.empty()) dnp[b] = normals_of(&dst_normals[b], dst[b].size());
    rows[b].resize(2 * corr[b].size() + 2);  // never empty: the row pointer stays valid
    for (size_t k = 0; k < corr[b].size(); ++k) {
      rows[b][2 * k] = corr[b][k].first;
      rows[b][2 * k + 1] = corr[b][k].second;
    }
    rows_p[b] = rows[b].data();
    ev[b].resize(2 * src[b].size());
    ev_p[b] = ev[b].data();
  }
  const tzr_ransac_params p = to_c(params_);
  std::vector<tzr_icp_result> res(B);
  std::vector<tzr_ransac_info> inf(B);
  tzr_ctx* ctx = b200_context();
  const int rc = tzr_ransac_batch(ctx, &p, static_cast<int>(B), ns.data(), sp.data(), nd.data(), dp.data(), nc.data(),
                                  rows_p.data(), seeds.empty() ? nullptr : seeds.data(),
                                  src_normals.empty() ? nullptr : snp.data(),
                                  dst_normals.empty() ? nullptr : dnp.data(), res.data(), inf.data(), ev_p.data());
  if (rc != TZR_OK) fail(ctx, rc);
  for (size_t b = 0; b < B; ++b) {
    icp_result_from_c(res[b], ev[b].data(), &out[b]);
    if (info) (*info)[b] = info_of(inf[b]);
  }
  return out;
}

std::vector<RANSACRegistration::CloudPairResult> RANSACRegistration::registerCloudPairs(
    const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& cp,
    const std::vector<uint64_t>& ransac_seeds) const {
  const int K = static_cast<int>(clouds.size()), P = static_cast<int>(pairs.size());
  std::vector<CloudPairResult> out(P);
  if (P == 0) return out;
  if (K == 0) throw std::invalid_argument("RANSACRegistration: registerCloudPairs needs clouds");
  if (!ransac_seeds.empty() && ransac_seeds.size() != pairs.size())
    throw std::invalid_argument("RANSACRegistration: one RANSAC seed per pair");
  std::vector<int32_t> n(K), pc(2 * P), status(P);
  std::vector<const float*> pts(K);
  for (int c = 0; c < K; ++c) {
    if (clouds[c].empty()) throw std::invalid_argument("RANSACRegistration: clouds must be non-empty");
    n[c] = static_cast<int32_t>(clouds[c].size());
    pts[c] = &clouds[c][0].x;
  }
  std::vector<uint64_t> seeds(P);
  std::vector<std::vector<int32_t>> corr(P);
  std::vector<int32_t*> corr_p(P);
  for (int p = 0; p < P; ++p) {
    const int a = pairs[p].first, b = pairs[p].second;
    if (a < 0 || a >= K || b < 0 || b >= K)
      throw std::invalid_argument("RANSACRegistration: registerCloudPairs: no such cloud");
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
  const tzr_ransac_params prm = to_c(params_);
  std::vector<int64_t> cnt(P);
  std::vector<float> gs(P);
  std::vector<tzr_icp_result> res(P);
  std::vector<tzr_ransac_info> inf(P);
  tzr_ctx* ctx = b200_context();
  const int rc = tzr_register_cloud_pairs_ransac(ctx, &f, &prm, K, n.data(), pts.data(), P, pc.data(), seeds.data(),
                                                 ransac_seeds.empty() ? nullptr : ransac_seeds.data(), status.data(),
                                                 cnt.data(), corr_p.data(), gs.data(), res.data(), inf.data());
  if (rc != TZR_OK && rc != TZR_ERR_TOO_LARGE) fail(ctx, rc);
  for (int p = 0; p < P; ++p) {
    CloudPairResult& r = out[p];
    r.status = status[p];
    r.global_scale = gs[p];
    for (int64_t k = 0; k < cnt[p]; ++k) r.correspondences.emplace_back(corr[p][2 * k], corr[p][2 * k + 1]);
    r.registered = status[p] == TZR_OK;
    if (r.registered) {
      icp_result_from_c(res[p], nullptr, &r.ransac);
      r.info = info_of(inf[p]);
    }
  }
  return out;
}

}  // namespace teaser
