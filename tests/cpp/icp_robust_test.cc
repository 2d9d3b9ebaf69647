// teaser::RobustKernel with PointToPlaneICP and GeneralizedICP, and the robust overloads of
// RobustRegistrationSolver::solveCloudPairsPointToPlane / solveCloudPairsGeneralizedICP, against the C-ABI: refine /
// refineBatch equal tzr_icp_point_to_plane_robust_batch and tzr_icp_generalized_robust_batch on each problem alone, bit
// for bit; the default (L2) kernel equals the unweighted classes; the chained overloads equal solveCloudPairs followed
// by estimateNormalsBatch and refineBatch over the pairs with a valid solution.
// usage: icp_robust_test   (needs a GPU; prints "ok")
#include <cmath>
#include <cstdint>
#include <cstring>
#include <iostream>
#include <stdexcept>
#include <utility>
#include <vector>

#include "teaser/icp.h"
#include "teaser/normals.h"
#include "teaser/registration.h"
#include "teaser_b200.h"

#define CHECK(c)                                                                  \
  do {                                                                            \
    if (!(c)) {                                                                   \
      std::cerr << "CHECK failed: " #c " at line " << __LINE__ << std::endl;     \
      return 1;                                                                   \
    }                                                                             \
  } while (0)

static uint64_t rng_state = 0x7654321ull;
static float uniform() {  // [-1, 1)
  rng_state = rng_state * 6364136223846793005ull + 1442695040888963407ull;
  return (float)((rng_state >> 40) * (1.0 / 16777216.0)) * 2.0f - 1.0f;
}

// a wavy surface patch; `from` (may be null) lends its first points, then the cloud is rotated by `angle` and shifted
static teaser::PointCloud scan(int n, const teaser::PointCloud* from, float shift, float angle) {
  teaser::PointCloud raw;
  const int keep = from ? std::min<int>(static_cast<int>(from->size()), n - n / 3) : 0;
  for (int i = 0; i < keep; ++i) raw.push_back((*from)[i]);
  for (int i = keep; i < n; ++i) {
    const float u = uniform(), v = uniform();
    raw.push_back({u, v, 0.3f * std::sin(3 * u) * std::cos(2 * v) + 0.003f * uniform() + 2.0f});
  }
  teaser::PointCloud pc;
  const float c = std::cos(angle), s = std::sin(angle);
  for (int i = n - 1; i >= 0; --i) {
    const teaser::PointXYZ p = raw[i];
    pc.push_back({c * p.x - s * p.y + shift, s * p.x + c * p.y, p.z});
  }
  return pc;
}

using Result = teaser::PointToPointICPResult;

static bool same(const Result& a, const Result& b) {
  return a.solution.scale == b.solution.scale &&
         std::memcmp(a.solution.rotation.data(), b.solution.rotation.data(), 9 * sizeof(double)) == 0 &&
         std::memcmp(a.solution.translation.data(), b.solution.translation.data(), 3 * sizeof(double)) == 0 &&
         a.fitness == b.fitness && a.inlier_rmse == b.inlier_rmse && a.iterations == b.iterations &&
         a.converged == b.converged && a.correspondences == b.correspondences;
}

static bool same_c(const Result& one, const tzr_icp_result& r, const std::vector<int32_t>& corr) {
  if (std::memcmp(one.solution.rotation.data(), r.transform.rotation, sizeof(r.transform.rotation)) != 0) return false;
  if (std::memcmp(one.solution.translation.data(), r.transform.translation, sizeof(r.transform.translation)) != 0)
    return false;
  if (!(one.fitness == r.fitness && one.inlier_rmse == r.inlier_rmse && one.iterations == r.iterations)) return false;
  if ((int)one.correspondences.size() != r.n_correspondences || r.n_correspondences <= 100) return false;
  for (int c = 0; c < r.n_correspondences; ++c)
    if (one.correspondences[c].first != corr[2 * c] || one.correspondences[c].second != corr[2 * c + 1]) return false;
  return true;
}

int main() {
  std::vector<teaser::PointCloud> clouds;
  clouds.push_back(scan(600, nullptr, 0.f, 0.f));
  clouds.push_back(scan(1500, &clouds[0], 0.03f, 0.04f));
  clouds.push_back(scan(500, &clouds[1], 0.05f, 0.03f));
  const auto nb = teaser::estimateNormalsBatch(clouds, 0.15);
  teaser::GeneralizedICP::Params ip;
  ip.max_correspondence_distance = 0.05;
  ip.epsilon = 0.01;
  const teaser::RobustKernel tukey_plane(teaser::RobustKernel::kTukey, 0.03);
  const teaser::RobustKernel cauchy_gicp(teaser::RobustKernel::kCauchy, 0.2);
  const teaser::PointToPlaneICP plane(ip, tukey_plane);
  const teaser::GeneralizedICP gicp(ip, cauchy_gicp);
  CHECK(plane.getKernel().type == teaser::RobustKernel::kTukey && gicp.getKernel().k == 0.2);
  CHECK(teaser::PointToPlaneICP(ip).getKernel().type == teaser::RobustKernel::kL2);
  teaser::RegistrationSolution seed;
  seed.scale = 1;
  seed.rotation.setIdentity();
  seed.translation << -0.03, 0.0, 0.0;
  const std::vector<std::pair<int, int>> probs = {{0, 1}, {1, 2}, {2, 0}};
  std::vector<teaser::PointCloud> S, D;
  std::vector<teaser::NormalCloud> SN, DN;
  std::vector<teaser::RegistrationSolution> I;
  for (const auto& pr : probs) {
    S.push_back(clouds[pr.first]);
    D.push_back(clouds[pr.second]);
    SN.push_back(nb[pr.first]);
    DN.push_back(nb[pr.second]);
    I.push_back(seed);
  }
  const auto pb = plane.refineBatch(S, D, DN, I);
  const auto gb = gicp.refineBatch(S, D, SN, DN, I);
  tzr_ctx* ctx = nullptr;
  CHECK(tzr_ctx_create(-1, &ctx) == TZR_OK);
  tzr_icp_params cp;
  tzr_icp_params_default(&cp);
  cp.max_correspondence_distance = 0.05;
  tzr_similarity cs;
  cs.scale = 1;
  std::memcpy(cs.rotation, seed.rotation.data(), sizeof(cs.rotation));
  for (int k = 0; k < 3; ++k) cs.translation[k] = seed.translation(k);
  tzr_robust_kernel kt, kc;
  std::memset(&kt, 0, sizeof(kt));
  std::memset(&kc, 0, sizeof(kc));
  kt.type = TZR_LOSS_TUKEY;
  kt.k = 0.03;
  kc.type = TZR_LOSS_CAUCHY;
  kc.k = 0.2;
  for (size_t b = 0; b < probs.size(); ++b) {
    const auto p1 = plane.refine(S[b], D[b], DN[b], I[b]);
    const auto g1 = gicp.refine(S[b], D[b], SN[b], DN[b], I[b]);
    CHECK(same(p1, pb[b]) && same(g1, gb[b]));
    const int32_t ns = (int32_t)S[b].size(), nd = (int32_t)D[b].size();
    const float* sp = &S[b][0].x;
    const float* dp = &D[b][0].x;
    const float* snp = &SN[b][0].normal_x;
    const float* dnp = &DN[b][0].normal_x;
    tzr_icp_result r;
    std::vector<int32_t> corr(2 * S[b].size());
    int32_t* corr_p = corr.data();
    CHECK(tzr_icp_point_to_plane_robust_batch(ctx, &cp, 1, &ns, &sp, &nd, &dp, &dnp, &cs, &r, &corr_p, &kt) == TZR_OK);
    CHECK(same_c(p1, r, corr));
    CHECK(tzr_icp_generalized_robust_batch(ctx, &cp, ip.epsilon, 1, &ns, &sp, &snp, &nd, &dp, &dnp, &cs, &r, &corr_p,
                                           &kc) == TZR_OK);
    CHECK(same_c(g1, r, corr));
  }
  tzr_ctx_destroy(ctx);
  // the default kernel is L2: the unweighted classes, bit for bit
  const auto l2p = teaser::PointToPlaneICP(ip, teaser::RobustKernel()).refine(S[0], D[0], DN[0], I[0]);
  CHECK(same(l2p, teaser::PointToPlaneICP(ip).refine(S[0], D[0], DN[0], I[0])));
  teaser::GeneralizedICP g2(ip);
  g2.setKernel(teaser::RobustKernel(teaser::RobustKernel::kL2));
  CHECK(same(g2.refine(S[0], D[0], SN[0], DN[0], I[0]), teaser::GeneralizedICP(ip).refine(S[0], D[0], SN[0], DN[0], I[0])));
  // a bad k is refused
  bool threw = false;
  try {
    teaser::PointToPlaneICP(ip, teaser::RobustKernel(teaser::RobustKernel::kHuber, 0.0)).refine(S[0], D[0], DN[0], I[0]);
  } catch (const std::runtime_error&) {
    threw = true;
  }
  CHECK(threw);
  // the chained overloads against solveCloudPairs + estimateNormalsBatch + refineBatch
  teaser::RobustRegistrationSolver::Params params;
  params.noise_bound = 0.01;
  params.estimate_scaling = false;
  params.rotation_cost_threshold = 1e-12;
  teaser::RobustRegistrationSolver::CloudPairParams fp;
  fp.normal_search_radius = 0.1;
  fp.fpfh_search_radius = 0.15;
  fp.use_absolute_scale = false;
  fp.use_tuple_test = false;
  teaser::RobustRegistrationSolver solver(params);
  const std::vector<std::pair<int, int>> pairs = {{0, 1}, {1, 2}, {2, 1}, {1, 0}};
  const auto plain = solver.solveCloudPairs(clouds, pairs, fp);
  const auto fnb = teaser::estimateNormalsBatch(clouds, fp.normal_search_radius);
  for (int method = 1; method <= 2; ++method) {
    const auto chained = method == 1 ? solver.solveCloudPairsPointToPlane(clouds, pairs, fp, ip, tukey_plane)
                                     : solver.solveCloudPairsGeneralizedICP(clouds, pairs, fp, ip, cauchy_gicp);
    CHECK(plain.size() == chained.size());
    std::vector<teaser::PointCloud> S2, D2;
    std::vector<teaser::NormalCloud> SN2, DN2;
    std::vector<teaser::RegistrationSolution> I2;
    std::vector<size_t> which;
    for (size_t p = 0; p < pairs.size(); ++p) {
      const auto& a = plain[p];
      const auto& b = chained[p];
      CHECK(a.status == b.status && a.correspondences == b.correspondences && a.max_clique == b.max_clique);
      CHECK(b.refined == (a.status == 0 && a.solution.valid));
      if (b.refined) {
        S2.push_back(clouds[pairs[p].first]);
        D2.push_back(clouds[pairs[p].second]);
        SN2.push_back(fnb[pairs[p].first]);
        DN2.push_back(fnb[pairs[p].second]);
        I2.push_back(a.solution);
        which.push_back(p);
      }
    }
    CHECK(!which.empty());
    auto ref = method == 1 ? plane.refineBatch(S2, D2, DN2, I2) : gicp.refineBatch(S2, D2, SN2, DN2, I2);
    for (size_t k = 0; k < which.size(); ++k) {
      ref[k].correspondences.clear();  // the chained call returns no ICP correspondences
      CHECK(same(ref[k], chained[which[k]].icp));
    }
  }
  std::cout << "ok" << std::endl;
  return 0;
}
