// teaser::GlobalOptimization and the line-process overloads of RobustRegistrationSolver::solveMultiway against the
// C-ABI: solveMultiway equals tzr_register_cloud_pairs_multiway_line_process with Open3D's tutorial rule ((k, k + 1)
// certain), and GlobalOptimization::optimize equals tzr_pose_graph_optimize_line_process, bit for bit.
// usage: line_process_test   (needs a GPU; prints "ok")
#include <cmath>
#include <cstdint>
#include <cstring>
#include <iostream>
#include <utility>
#include <vector>

#include "teaser/pose_graph.h"
#include "teaser/registration.h"
#include "teaser_b200.h"

#define CHECK(c)                                                                  \
  do {                                                                            \
    if (!(c)) {                                                                   \
      std::cerr << "CHECK failed: " #c " at line " << __LINE__ << std::endl;     \
      return 1;                                                                   \
    }                                                                             \
  } while (0)

static uint64_t rng_state = 0x1234567ull;
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

static tzr_similarity sim(const teaser::Matrix6d*, const Eigen::Matrix4d& T) {
  tzr_similarity c;
  c.scale = 1.0;
  for (int r = 0; r < 3; ++r) {
    for (int k = 0; k < 3; ++k) c.rotation[3 * k + r] = T(r, k);
    c.translation[r] = T(r, 3);
  }
  return c;
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
  std::vector<teaser::PointCloud> clouds{scan(700, nullptr, 0, 0)};
  for (int k = 1; k < 5; ++k) clouds.push_back(scan(700, &clouds.back(), 0.04f, 0.03f));
  const double r = 0.05;

  // the chained call, with the tutorial rule, against the C-ABI entry
  const std::vector<std::pair<int, int>> pairs{{0, 1}, {1, 2}, {2, 3}, {3, 4}, {4, 0}, {3, 1}};
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
  teaser::PointToPointICPParams ip;
  ip.max_correspondence_distance = r;
  teaser::GlobalOptimization::Params go;
  go.max_correspondence_distance = r;
  const auto mw = solver.solveMultiway(clouds, pairs, cp, ip, go);
  CHECK(mw.pose_graph_status == TZR_OK && mw.poses.size() == clouds.size());
  {
    const int K = 5, P = 6;
    std::vector<int32_t> n(K, 700), pc, status(P), index(P), unc, counts_c(P), lp_status(1);
    std::vector<const float*> pts;
    for (const auto& c : clouds) pts.push_back(&c[0].x);
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
    tzr_line_process_params lpc;
    tzr_line_process_params_default(&lpc);
    lpc.max_correspondence_distance = r;
    std::vector<tzr_solution> sols(P);
    std::vector<int64_t> n_corr(P);
    std::vector<tzr_icp_result> ir(P);
    std::vector<double> info(36 * P), l(P);
    std::vector<uint8_t> kept(P);
    std::vector<tzr_similarity> poses(K);
    tzr_line_process_summary summ;
    const int rc = tzr_register_cloud_pairs_multiway_line_process(
        ctx, &f, &tp, K, n.data(), pts.data(), P, pc.data(), seeds.data(), sols.data(), status.data(), index.data(),
        n_corr.data(), nullptr, nullptr, nullptr, &icp, nullptr, 0.0, nullptr, ir.data(), unc.data(), &lpc,
        info.data(), counts_c.data(), l.data(), kept.data(), poses.data(), &summ, lp_status.data());
    CHECK(rc == TZR_OK && lp_status[0] == mw.pose_graph_status);
    for (int k = 0; k < K; ++k) CHECK(same_pose(mw.poses[k], poses[k]));
    for (int p = 0; p < P; ++p) {
      CHECK(mw.edge_weights[p] == l[p] && mw.edge_inliers[p] == (kept[p] != 0));
      CHECK(mw.information_counts[p] == counts_c[p]);
      for (int a = 0; a < 6; ++a)
        for (int b = 0; b < 6; ++b) CHECK(mw.information[p](a, b) == info[36 * p + 6 * a + b]);
    }
    for (int q = 0; q < 2; ++q)
      CHECK(mw.line_process.trials[q] == summ.trials[q] && mw.line_process.iterations[q] == summ.iterations[q] &&
            mw.line_process.stop_reason[q] == summ.stop_reason[q] && mw.line_process.mu[q] == summ.mu[q]);
    CHECK(mw.line_process.pruned == summ.pruned && mw.line_process.residual == summ.residual);
  }

  // GlobalOptimization::optimize against tzr_pose_graph_optimize_line_process on the refined pairs
  std::vector<teaser::GlobalOptimization::Edge> edges;
  for (size_t p = 0; p < pairs.size(); ++p) {
    if (!mw.pairs[p].refined) continue;
    teaser::GlobalOptimization::Edge e;
    e.source = pairs[p].first;
    e.target = pairs[p].second;
    e.transform = Eigen::Matrix4d::Identity();
    for (int a = 0; a < 3; ++a) {
      for (int b = 0; b < 3; ++b) e.transform(a, b) = mw.pairs[p].icp.solution.rotation(a, b);
      e.transform(a, 3) = mw.pairs[p].icp.solution.translation(a);
    }
    e.information = mw.information[p];
    e.uncertain = pairs[p].second != pairs[p].first + 1;
    edges.push_back(e);
  }
  CHECK(edges.size() >= 5);
  const teaser::GlobalOptimization graph(go);
  const teaser::GlobalOptimization::Result res = graph.optimize(5, edges);
  {
    const int E = static_cast<int>(edges.size());
    std::vector<int32_t> ends, unc;
    std::vector<tzr_similarity> tr;
    std::vector<double> info;
    for (const auto& e : edges) {
      ends.push_back(e.source);
      ends.push_back(e.target);
      unc.push_back(e.uncertain ? 1 : 0);
      tr.push_back(sim(nullptr, e.transform));
      for (int a = 0; a < 6; ++a)
        for (int b = 0; b < 6; ++b) info.push_back(e.information(a, b));
    }
    tzr_line_process_params lpc;
    tzr_line_process_params_default(&lpc);
    lpc.max_correspondence_distance = r;
    std::vector<tzr_similarity> poses(5);
    std::vector<double> l(E), rz(E);
    std::vector<uint8_t> kept(E);
    tzr_line_process_summary summ;
    CHECK(tzr_pose_graph_optimize_line_process(ctx, &lpc, 5, E, ends.data(), tr.data(), info.data(), unc.data(),
                                               nullptr, poses.data(), l.data(), kept.data(), rz.data(),
                                               &summ) == TZR_OK);
    for (int k = 0; k < 5; ++k) CHECK(same_pose(res.poses[k], poses[k]));
    for (int e = 0; e < E; ++e)
      CHECK(res.confidence[e] == l[e] && res.residuals[e] == rz[e] && res.kept[e] == (kept[e] != 0));
    for (int q = 0; q < 2; ++q)
      CHECK(res.summary.trials[q] == summ.trials[q] && res.summary.stop_reason[q] == summ.stop_reason[q]);
    CHECK(res.summary.residual == summ.residual && res.summary.pruned == summ.pruned);
    // the same graph as solveMultiway's
    for (int k = 0; k < 5; ++k) CHECK(same_pose(mw.poses[k], poses[k]));
  }
  // a disconnected graph and a parameter out of range throw
  bool threw = false;
  try {
    graph.optimize(6, edges);
  } catch (const std::runtime_error&) {
    threw = true;
  }
  CHECK(threw);
  threw = false;
  teaser::GlobalOptimization::Params bad = go;
  bad.edge_prune_threshold = 2.0;
  try {
    teaser::GlobalOptimization(bad).optimize(5, edges);
  } catch (const std::runtime_error&) {
    threw = true;
  }
  CHECK(threw);
  std::cout << "ok" << std::endl;
  return 0;
}
