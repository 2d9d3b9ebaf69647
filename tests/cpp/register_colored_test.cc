// RobustRegistrationSolver::solveCloudPairsColoredICP and the coloured solveMultiway against the C-ABI: each equals
// tzr_register_cloud_pairs_icp_colored / tzr_register_cloud_pairs_multiway_colored on the same inputs bit for bit,
// with and without a robust kernel and with Open3D's tutorial rule for the uncertain flags.
// usage: register_colored_test   (needs a GPU; prints "ok")
#include <cmath>
#include <cstdint>
#include <cstring>
#include <iostream>
#include <utility>
#include <vector>

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

// a wavy textured surface patch; `from` (may be null) lends its first points and their colours, then the cloud is
// rotated by `angle` and shifted
static void scan(int n, const teaser::PointCloud* from, const teaser::ColorCloud* from_c, float shift, float angle,
                 teaser::PointCloud* pc, teaser::ColorCloud* cc) {
  teaser::PointCloud raw;
  teaser::ColorCloud rc;
  const int keep = from ? std::min<int>(static_cast<int>(from->size()), n - n / 3) : 0;
  for (int i = 0; i < keep; ++i) {
    raw.push_back((*from)[i]);
    rc.push_back((*from_c)[i]);
  }
  for (int i = keep; i < n; ++i) {
    const float u = uniform(), v = uniform();
    raw.push_back({u, v, 0.3f * std::sin(3 * u) * std::cos(2 * v) + 0.003f * uniform() + 2.0f});
    const float a = 0.5f + 0.4f * std::sin(9 * u) * std::cos(7 * v), b = 0.5f + 0.4f * std::cos(5 * u + 3 * v);
    rc.push_back({a, b, 0.5f * (a + b)});
  }
  const float c = std::cos(angle), s = std::sin(angle);
  for (int i = n - 1; i >= 0; --i) {
    const teaser::PointXYZ p = raw[i];
    pc->push_back({c * p.x - s * p.y + shift, s * p.x + c * p.y, p.z});
    cc->push_back(rc[i]);
  }
}

static bool same_record(const teaser::RobustRegistrationSolver::CloudPairICPResult& r, const tzr_icp_result& c) {
  if (!r.refined) return c.transform.scale == 0;
  return r.icp.solution.scale == c.transform.scale &&
         std::memcmp(r.icp.solution.rotation.data(), c.transform.rotation, 9 * sizeof(double)) == 0 &&
         std::memcmp(r.icp.solution.translation.data(), c.transform.translation, 3 * sizeof(double)) == 0 &&
         r.icp.fitness == c.fitness && r.icp.inlier_rmse == c.inlier_rmse && r.icp.iterations == c.iterations &&
         r.icp.converged == (c.converged != 0);
}

static bool same_pose(const Eigen::Matrix4d& T, const tzr_similarity& s) {
  for (int r = 0; r < 3; ++r) {
    for (int k = 0; k < 3; ++k)
      if (T(r, k) != s.rotation[3 * k + r]) return false;
    if (T(r, 3) != s.translation[r]) return false;
  }
  return true;
}

int main() {
  tzr_ctx* ctx = teaser::b200_context();
  std::vector<teaser::PointCloud> clouds(1);
  std::vector<teaser::ColorCloud> colors(1);
  scan(700, nullptr, nullptr, 0, 0, &clouds[0], &colors[0]);
  for (int k = 1; k < 5; ++k) {
    teaser::PointCloud pc;
    teaser::ColorCloud cc;
    scan(700, &clouds.back(), &colors.back(), 0.04f, 0.03f, &pc, &cc);
    clouds.push_back(pc);
    colors.push_back(cc);
  }
  const double r = 0.05;
  const std::vector<std::pair<int, int>> pairs{{0, 1}, {1, 2}, {2, 3}, {3, 4}, {4, 0}, {3, 1}};
  const int K = 5, P = 6;

  teaser::RobustRegistrationSolver::Params sp;
  sp.noise_bound = 0.01;
  sp.estimate_scaling = false;
  sp.rotation_cost_threshold = 1e-12;
  teaser::RobustRegistrationSolver solver(sp);
  teaser::RobustRegistrationSolver::CloudPairParams cp;
  cp.normal_search_radius = 0.1;
  cp.fpfh_search_radius = 0.15;
  cp.use_absolute_scale = false;
  cp.use_tuple_test = false;
  teaser::ColoredICPParams ip;
  ip.max_correspondence_distance = r;
  ip.lambda_geometric = 0.9;
  teaser::PoseGraphParams pg;
  pg.max_correspondence_distance = r;

  // the C-ABI's inputs
  std::vector<int32_t> n(K, 700), pc, unc;
  std::vector<const float*> pts, cols;
  for (int k = 0; k < K; ++k) {
    pts.push_back(&clouds[k][0].x);
    cols.push_back(&colors[k][0].r);
  }
  std::vector<uint64_t> seeds;
  for (int p = 0; p < P; ++p) {
    pc.push_back(pairs[p].first);
    pc.push_back(pairs[p].second);
    unc.push_back(pairs[p].second == pairs[p].first + 1 ? 0 : 1);
    seeds.push_back(cp.tuple_seed + 0x9E3779B97F4A7C15ull * static_cast<uint64_t>(p));
  }
  tzr_frontend_params f;
  tzr_frontend_params_default(&f);
  f.normal_search_radius = cp.normal_search_radius;
  f.fpfh_search_radius = cp.fpfh_search_radius;
  f.use_absolute_scale = 0;
  f.use_crosscheck = 1;
  f.use_tuple_test = 0;
  tzr_params tp;
  tzr_params_default(&tp);
  tp.noise_bound = 0.01;
  tp.estimate_scaling = 0;
  tp.rotation_cost_threshold = 1e-12;
  tzr_icp_params icp;
  tzr_icp_params_default(&icp);
  icp.max_correspondence_distance = r;
  tzr_pose_graph_params pgc;
  tzr_pose_graph_params_default(&pgc);
  pgc.max_correspondence_distance = r;

  // the chained call, without and with a kernel
  for (int with_kernel = 0; with_kernel < 2; ++with_kernel) {
    const teaser::RobustKernel rk = with_kernel ? teaser::RobustKernel(teaser::RobustKernel::kHuber, 0.02)
                                                : teaser::RobustKernel();
    const auto res = solver.solveCloudPairsColoredICP(clouds, colors, pairs, cp, ip, rk);
    CHECK(res.size() == static_cast<size_t>(P));
    std::vector<int32_t> status(P), index(P);
    std::vector<tzr_solution> sols(P);
    std::vector<int64_t> n_corr(P);
    std::vector<tzr_icp_result> ir(P);
    tzr_robust_kernel k;
    std::memset(&k, 0, sizeof(k));
    k.type = TZR_LOSS_HUBER;
    k.k = 0.02;
    CHECK(tzr_register_cloud_pairs_icp_colored(ctx, &f, &tp, K, n.data(), pts.data(), P, pc.data(), seeds.data(),
                                               sols.data(), status.data(), index.data(), n_corr.data(), nullptr,
                                               nullptr, nullptr, &icp, cols.data(), ip.lambda_geometric,
                                               with_kernel ? &k : nullptr, ir.data()) == TZR_OK);
    int refined = 0;
    for (int p = 0; p < P; ++p) {
      CHECK(res[p].status == status[p] && res[p].solution.valid == (sols[p].valid != 0));
      CHECK(same_record(res[p], ir[p]));
      refined += res[p].refined;
    }
    CHECK(refined >= 5);
  }
  // a colour cloud that does not match its cloud is refused
  {
    std::vector<teaser::ColorCloud> bad = colors;
    bad[2].pop_back();
    bool threw = false;
    try {
      solver.solveCloudPairsColoredICP(clouds, bad, pairs, cp, ip);
    } catch (const std::invalid_argument&) {
      threw = true;
    }
    CHECK(threw);
  }

  // multiway, tutorial rule, without and with a kernel
  for (int with_kernel = 0; with_kernel < 2; ++with_kernel) {
    const teaser::RobustKernel rk = with_kernel ? teaser::RobustKernel(teaser::RobustKernel::kCauchy, 0.02)
                                                : teaser::RobustKernel();
    const auto mw = solver.solveMultiway(clouds, colors, pairs, cp, ip, pg, rk);
    CHECK(mw.pose_graph_status == TZR_OK && mw.poses.size() == clouds.size());
    std::vector<int32_t> status(P), index(P), counts_c(P), pg_status(1);
    std::vector<tzr_solution> sols(P);
    std::vector<int64_t> n_corr(P);
    std::vector<tzr_icp_result> ir(P);
    std::vector<double> info(36 * P), w(P);
    std::vector<uint8_t> mask(P);
    std::vector<tzr_similarity> poses(K);
    tzr_pose_graph_summary summ;
    tzr_robust_kernel k;
    std::memset(&k, 0, sizeof(k));
    k.type = TZR_LOSS_CAUCHY;
    k.k = 0.02;
    const int rc = tzr_register_cloud_pairs_multiway_colored(
        ctx, &f, &tp, K, n.data(), pts.data(), P, pc.data(), seeds.data(), sols.data(), status.data(), index.data(),
        n_corr.data(), nullptr, nullptr, nullptr, &icp, cols.data(), ip.lambda_geometric, with_kernel ? &k : nullptr,
        ir.data(), unc.data(), &pgc, info.data(), counts_c.data(), w.data(), mask.data(), poses.data(), &summ,
        pg_status.data());
    CHECK(rc == TZR_OK && pg_status[0] == mw.pose_graph_status);
    for (int q = 0; q < K; ++q) CHECK(same_pose(mw.poses[q], poses[q]));
    for (int p = 0; p < P; ++p) {
      CHECK(same_record(mw.pairs[p], ir[p]));
      CHECK(mw.edge_weights[p] == w[p] && mw.edge_inliers[p] == (mask[p] != 0));
      CHECK(mw.information_counts[p] == counts_c[p]);
      for (int a = 0; a < 6; ++a)
        for (int b = 0; b < 6; ++b) CHECK(mw.information[p](a, b) == info[36 * p + 6 * a + b]);
    }
    CHECK(mw.iterations == summ.iterations && mw.inner_iterations == summ.inner_iterations && mw.cost == summ.cost);
  }
  // explicit flags: every pair certain
  const auto all = solver.solveMultiway(clouds, colors, pairs, cp, ip, pg, std::vector<bool>(pairs.size(), false));
  CHECK(all.pose_graph_status == TZR_OK && all.iterations == 1);
  std::cout << "ok" << std::endl;
  return 0;
}
