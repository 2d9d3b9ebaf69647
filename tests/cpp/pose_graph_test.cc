// teaser::informationMatrix(Batch), teaser::PoseGraph and RobustRegistrationSolver::solveMultiway against the C-ABI:
// informationMatrix equals tzr_information_matrix and each batch entry the single call, bit for bit; PoseGraph::optimize
// equals tzr_pose_graph_optimize; solveMultiway equals tzr_register_cloud_pairs_multiway with Open3D's tutorial rule
// ((k, k + 1) certain) and with explicit flags.
// usage: pose_graph_test   (needs a GPU; prints "ok")
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

  // information matrices
  teaser::RegistrationSolution T;
  T.scale = 1.0;
  T.rotation.setIdentity();
  T.translation.setZero();
  T.translation(0) = 0.04;
  int count = 0;
  const teaser::Matrix6d L = teaser::informationMatrix(clouds[0], clouds[1], T, r, &count);
  tzr_similarity ts;
  ts.scale = 1.0;
  std::memcpy(ts.rotation, T.rotation.data(), sizeof(ts.rotation));
  for (int k = 0; k < 3; ++k) ts.translation[k] = T.translation(k);
  double Lc[36];
  int32_t cc = 0;
  CHECK(tzr_information_matrix(ctx, &clouds[0][0].x, 700, &clouds[1][0].x, 700, &ts, r, Lc, &cc) == TZR_OK);
  CHECK(count == cc && count > 0 && L(5, 5) == count);
  for (int a = 0; a < 6; ++a)
    for (int b = 0; b < 6; ++b) CHECK(L(a, b) == Lc[6 * a + b]);
  std::vector<int> counts;
  const std::vector<teaser::Matrix6d> LB =
      teaser::informationMatrixBatch({clouds[2], clouds[0]}, {clouds[3], clouds[1]}, {T, T}, r, &counts);
  CHECK(LB.size() == 2 && counts[1] == count);
  for (int a = 0; a < 6; ++a)
    for (int b = 0; b < 6; ++b) CHECK(LB[1](a, b) == L(a, b));

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
  teaser::PoseGraphParams pg;
  pg.max_correspondence_distance = r;
  const auto mw = solver.solveMultiway(clouds, pairs, cp, ip, pg);
  CHECK(mw.pose_graph_status == TZR_OK && mw.poses.size() == clouds.size());
  {
    const int K = 5, P = 6;
    std::vector<int32_t> n(K, 700), pc, status(P), index(P), unc, counts_c(P), pg_status(1);
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
    tzr_pose_graph_params pgc;
    tzr_pose_graph_params_default(&pgc);
    pgc.max_correspondence_distance = r;
    std::vector<tzr_solution> sols(P);
    std::vector<int64_t> n_corr(P);
    std::vector<tzr_icp_result> ir(P);
    std::vector<double> info(36 * P), w(P);
    std::vector<uint8_t> mask(P);
    std::vector<tzr_similarity> poses(K);
    tzr_pose_graph_summary summ;
    const int rc = tzr_register_cloud_pairs_multiway(ctx, &f, &tp, K, n.data(), pts.data(), P, pc.data(), seeds.data(),
                                                     sols.data(), status.data(), index.data(), n_corr.data(), nullptr,
                                                     nullptr, nullptr, &icp, ir.data(), unc.data(), &pgc, info.data(),
                                                     counts_c.data(), w.data(), mask.data(), poses.data(), &summ,
                                                     pg_status.data());
    CHECK(rc == TZR_OK && pg_status[0] == mw.pose_graph_status);
    for (int k = 0; k < K; ++k) CHECK(same_pose(mw.poses[k], poses[k]));
    for (int p = 0; p < P; ++p) {
      CHECK(mw.edge_weights[p] == w[p] && mw.edge_inliers[p] == (mask[p] != 0));
      CHECK(mw.information_counts[p] == counts_c[p]);
      for (int a = 0; a < 6; ++a)
        for (int b = 0; b < 6; ++b) CHECK(mw.information[p](a, b) == info[36 * p + 6 * a + b]);
    }
    CHECK(mw.iterations == summ.iterations && mw.inner_iterations == summ.inner_iterations && mw.cost == summ.cost);
  }
  // explicit flags: every pair certain
  const auto all = solver.solveMultiway(clouds, pairs, cp, ip, pg, std::vector<bool>(pairs.size(), false));
  CHECK(all.pose_graph_status == TZR_OK && all.iterations == 1);

  // PoseGraph::optimize against tzr_pose_graph_optimize on the refined pairs
  std::vector<teaser::PoseGraph::Edge> edges;
  for (size_t p = 0; p < pairs.size(); ++p) {
    if (!mw.pairs[p].refined) continue;
    teaser::PoseGraph::Edge e;
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
  const teaser::PoseGraph graph(pg);
  const teaser::PoseGraph::Result res = graph.optimize(5, edges);
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
    tzr_pose_graph_params pgc;
    tzr_pose_graph_params_default(&pgc);
    pgc.max_correspondence_distance = r;
    std::vector<tzr_similarity> poses(5);
    std::vector<double> w(E), rb(E);
    std::vector<uint8_t> mask(E);
    tzr_pose_graph_summary summ;
    CHECK(tzr_pose_graph_optimize(ctx, &pgc, 5, E, ends.data(), tr.data(), info.data(), unc.data(), nullptr,
                                  poses.data(), w.data(), mask.data(), rb.data(), &summ) == TZR_OK);
    for (int k = 0; k < 5; ++k) CHECK(same_pose(res.poses[k], poses[k]));
    for (int e = 0; e < E; ++e) CHECK(res.weights[e] == w[e] && res.residuals[e] == rb[e] && res.inliers[e] == (mask[e] != 0));
    CHECK(res.iterations == summ.iterations && res.cost == summ.cost);
    // the same graph as solveMultiway's
    for (int k = 0; k < 5; ++k) CHECK(same_pose(mw.poses[k], poses[k]));
  }
  // a disconnected graph throws
  bool threw = false;
  try {
    graph.optimize(6, edges);
  } catch (const std::runtime_error&) {
    threw = true;
  }
  CHECK(threw);
  std::cout << "ok" << std::endl;
  return 0;
}
