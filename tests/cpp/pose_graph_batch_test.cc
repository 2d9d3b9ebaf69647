// teaser::PoseGraph::optimizeBatch against tzr_pose_graph_optimize_batch, bit for bit, on a batch of synthetic graphs:
// fragment-shaped graphs of both routes (K <= 128 and K = 140), one with given initial poses, and a disconnected graph
// whose status the façade reports.
// usage: pose_graph_batch_test   (needs a GPU; prints "ok")
#include <cmath>
#include <cstdint>
#include <iostream>
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

static uint64_t rng_state = 0x2545f491ull;
static double uniform() {  // [-1, 1)
  rng_state = rng_state * 6364136223846793005ull + 1442695040888963407ull;
  return (double)(rng_state >> 11) * (2.0 / 9007199254740992.0) - 1.0;
}

// a rigid motion: rotation by Rodrigues' formula about a random axis (angle up to about `angle`), random shift
static Eigen::Matrix4d motion(double angle, double shift) {
  double w[3] = {uniform(), uniform(), uniform()};
  const double n = std::sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]), th = angle * n;
  for (double& x : w) x /= n;
  const double c = std::cos(th), s = std::sin(th);
  Eigen::Matrix4d T = Eigen::Matrix4d::Identity();
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) T(a, b) = (a == b ? c : 0.0) + (1.0 - c) * w[a] * w[b];
  T(0, 1) -= s * w[2];
  T(0, 2) += s * w[1];
  T(1, 0) += s * w[2];
  T(1, 2) -= s * w[0];
  T(2, 0) -= s * w[1];
  T(2, 1) += s * w[0];
  for (int a = 0; a < 3; ++a) T(a, 3) = shift * uniform();
  return T;
}

static Eigen::Matrix4d inverse(const Eigen::Matrix4d& T) {
  Eigen::Matrix4d I = Eigen::Matrix4d::Identity();
  for (int a = 0; a < 3; ++a) {
    for (int b = 0; b < 3; ++b) I(a, b) = T(b, a);
  }
  for (int a = 0; a < 3; ++a) I(a, 3) = -(I(a, 0) * T(0, 3) + I(a, 1) * T(1, 3) + I(a, 2) * T(2, 3));
  return I;
}

// odometry (k, k + 1), closures between keyframes (every 5th node) up to 10 apart, one wrong far closure
static teaser::PoseGraph::Graph fragment(int K, bool wrong) {
  std::vector<Eigen::Matrix4d> gt{Eigen::Matrix4d::Identity()};
  for (int k = 1; k < K; ++k) gt.push_back(motion(0.3, 0.5));
  std::vector<std::pair<int, int>> pairs;
  for (int k = 0; k + 1 < K; ++k) pairs.push_back({k, k + 1});
  for (int a = 0; a < K; a += 5)
    for (int b = a + 5; b < K && b <= a + 10; b += 5) pairs.push_back({a, b});
  if (wrong && K > 20) pairs.push_back({0, 20});
  teaser::PoseGraph::Graph g;
  g.num_nodes = K;
  for (size_t j = 0; j < pairs.size(); ++j) {
    teaser::PoseGraph::Edge e;
    e.source = pairs[j].first;
    e.target = pairs[j].second;
    const bool bad = wrong && j + 1 == pairs.size();
    e.transform = (bad ? motion(0.5, 1.0) : motion(0.004, 0.004)) * inverse(gt[e.target]) * gt[e.source];
    teaser::Matrix6d L = teaser::Matrix6d::Zero();
    for (int i = 0; i < 150; ++i) {
      const double q[3] = {uniform(), uniform(), uniform()};
      // G = [-[q]x | I]
      Eigen::Matrix<double, 3, 6> G = Eigen::Matrix<double, 3, 6>::Zero();
      G(0, 1) = q[2];
      G(0, 2) = -q[1];
      G(1, 0) = -q[2];
      G(1, 2) = q[0];
      G(2, 0) = q[1];
      G(2, 1) = -q[0];
      for (int a = 0; a < 3; ++a) G(a, 3 + a) = 1.0;
      L = L + G.transpose() * G;
    }
    e.information = L;
    e.uncertain = e.target != e.source + 1;
    g.edges.push_back(e);
  }
  return g;
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
  std::vector<teaser::PoseGraph::Graph> gs{fragment(60, true), fragment(140, true), fragment(25, false),
                                           fragment(100, true)};
  for (int k = 0; k < gs[2].num_nodes; ++k) gs[2].initial_poses.push_back(motion(0.02, 0.02));
  gs.push_back(fragment(12, false));
  gs.back().num_nodes = 13;  // node 12 has no edge
  teaser::PoseGraph::Params prm;
  prm.max_correspondence_distance = 0.05;
  prm.reference_node = 3;
  const teaser::PoseGraph pg(prm);
  std::vector<int> status;
  const auto res = pg.optimizeBatch(gs, &status);
  CHECK(res.size() == gs.size() && status.size() == gs.size());

  // the same batch through the C ABI
  const size_t G = gs.size();
  tzr_pose_graph_params p;
  tzr_pose_graph_params_default(&p);
  p.max_correspondence_distance = 0.05;
  p.reference_node = 3;
  std::vector<int32_t> K(G), E(G), st(G);
  std::vector<std::vector<int32_t>> ends(G), unc(G);
  std::vector<std::vector<tzr_similarity>> tr(G), init(G), poses(G);
  std::vector<std::vector<double>> L(G), w(G), r(G);
  std::vector<std::vector<uint8_t>> mask(G);
  std::vector<const int32_t*> ep(G), up(G);
  std::vector<const tzr_similarity*> tp(G), ip(G);
  std::vector<const double*> Lp(G);
  std::vector<tzr_similarity*> pp(G);
  std::vector<double*> wp(G), rp(G);
  std::vector<uint8_t*> mp(G);
  auto sim = [](const Eigen::Matrix4d& T) {
    tzr_similarity c;
    c.scale = 1.0;
    for (int a = 0; a < 3; ++a) {
      for (int b = 0; b < 3; ++b) c.rotation[3 * b + a] = T(a, b);
      c.translation[a] = T(a, 3);
    }
    return c;
  };
  for (size_t g = 0; g < G; ++g) {
    K[g] = gs[g].num_nodes;
    E[g] = (int32_t)gs[g].edges.size();
    for (const auto& e : gs[g].edges) {
      ends[g].push_back(e.source);
      ends[g].push_back(e.target);
      unc[g].push_back(e.uncertain ? 1 : 0);
      tr[g].push_back(sim(e.transform));
      for (int a = 0; a < 6; ++a)
        for (int b = 0; b < 6; ++b) L[g].push_back(e.information(a, b));
    }
    for (const auto& T : gs[g].initial_poses) init[g].push_back(sim(T));
    poses[g].resize(K[g]);
    w[g].resize(E[g]);
    r[g].resize(E[g]);
    mask[g].resize(E[g]);
    ep[g] = ends[g].data();
    up[g] = unc[g].data();
    tp[g] = tr[g].data();
    Lp[g] = L[g].data();
    ip[g] = init[g].empty() ? nullptr : init[g].data();
    pp[g] = poses[g].data();
    wp[g] = w[g].data();
    rp[g] = r[g].data();
    mp[g] = mask[g].data();
  }
  std::vector<tzr_pose_graph_summary> s(G);
  CHECK(tzr_pose_graph_optimize_batch(teaser::b200_context(), &p, (int)G, K.data(), E.data(), ep.data(), tp.data(),
                                      Lp.data(), up.data(), ip.data(), pp.data(), wp.data(), mp.data(), rp.data(),
                                      s.data(), st.data()) == TZR_OK);
  for (size_t g = 0; g < G; ++g) {
    CHECK(status[g] == st[g]);
    if (st[g] != TZR_OK) {
      CHECK(res[g].poses.empty());
      continue;
    }
    CHECK(res[g].poses.size() == (size_t)K[g]);
    for (int k = 0; k < K[g]; ++k) CHECK(same_pose(res[g].poses[k], poses[g][k]));
    for (int e = 0; e < E[g]; ++e) {
      CHECK(res[g].weights[e] == w[g][e] && res[g].residuals[e] == r[g][e]);
      CHECK(res[g].inliers[e] == (mask[g][e] != 0));
    }
    CHECK(res[g].iterations == s[g].iterations && res[g].inner_iterations == s[g].inner_iterations);
    CHECK(res[g].cost == s[g].cost);
  }
  CHECK(st[0] == TZR_OK && st[1] == TZR_OK && st[2] == TZR_OK && st[3] == TZR_OK && st[4] == TZR_ERR_INVALID_ARG);
  bool threw = false;
  try {
    pg.optimizeBatch({});
  } catch (const std::runtime_error&) {
    threw = true;
  }
  CHECK(threw);
  std::cout << "ok" << std::endl;
  return 0;
}
