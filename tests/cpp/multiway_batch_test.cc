// RobustRegistrationSolver::solveMultiwayBatch against the C-ABI: both overloads (GNC-TLS with a fused map, the line
// process without one) equal tzr_register_cloud_pairs_multiway(_line_process)_batch on the flattened table, each
// sequence's pairs seeded as solveMultiway seeds them on that sequence alone, bit for bit.
// usage: multiway_batch_test   (needs a GPU; prints "ok")
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
  const double r = 0.05, vox = 0.02;
  std::vector<teaser::RobustRegistrationSolver::MultiwaySequence> seqs(2);
  for (int g = 0; g < 2; ++g) {
    const int K = g ? 4 : 5, n = g ? 600 : 700;
    seqs[g].clouds.push_back(scan(n, nullptr, 0, 0));
    for (int k = 1; k < K; ++k) seqs[g].clouds.push_back(scan(n, &seqs[g].clouds.back(), 0.04f, 0.03f));
    for (int k = 0; k + 1 < K; ++k) seqs[g].pairs.emplace_back(k, k + 1);
    seqs[g].pairs.emplace_back(K - 1, 0);
  }
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
  teaser::PoseGraphParams pg;
  pg.max_correspondence_distance = r;
  teaser::LineProcessParams lpp;
  lpp.max_correspondence_distance = r;

  // the flat table, as the façade builds it
  std::vector<int32_t> n, pc, unc, off{0};
  std::vector<const float*> pts;
  std::vector<uint64_t> seeds;
  std::vector<int> pair_lo{0};
  std::vector<size_t> total(2, 0);
  for (int g = 0; g < 2; ++g) {
    for (const auto& c : seqs[g].clouds) {
      n.push_back(static_cast<int32_t>(c.size()));
      pts.push_back(&c[0].x);
      total[g] += c.size();
    }
    for (size_t j = 0; j < seqs[g].pairs.size(); ++j) {
      pc.push_back(off.back() + seqs[g].pairs[j].first);
      pc.push_back(off.back() + seqs[g].pairs[j].second);
      unc.push_back(seqs[g].pairs[j].second == seqs[g].pairs[j].first + 1 ? 0 : 1);
      seeds.push_back(cp.tuple_seed + 0x9E3779B97F4A7C15ull * static_cast<uint64_t>(j));
    }
    off.push_back(off.back() + static_cast<int32_t>(seqs[g].clouds.size()));
    pair_lo.push_back(static_cast<int>(unc.size()));
  }
  const int K = off.back(), P = static_cast<int>(unc.size());
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

  for (int lp = 0; lp < 2; ++lp) {
    const double v = lp ? 0.0 : vox;
    const auto mw = lp ? solver.solveMultiwayBatch(seqs, cp, ip, lpp) : solver.solveMultiwayBatch(seqs, cp, ip, pg, v);
    CHECK(mw.size() == 2);
    std::vector<int32_t> status(P), index(P), counts(P), pg_status(2), map_counts(2);
    std::vector<tzr_solution> sols(P);
    std::vector<int64_t> n_corr(P);
    std::vector<tzr_icp_result> ir(P);
    std::vector<double> info(36 * P), w(P);
    std::vector<uint8_t> mask(P);
    std::vector<tzr_similarity> poses(K);
    std::vector<tzr_pose_graph_summary> summ(2);
    std::vector<tzr_line_process_summary> lsumm(2);
    std::vector<std::vector<float>> maps{std::vector<float>(3 * total[0]), std::vector<float>(3 * total[1])};
    float* map_p[2] = {maps[0].data(), maps[1].data()};
    int rc;
    if (lp) {
      tzr_line_process_params lc;
      tzr_line_process_params_default(&lc);
      lc.max_correspondence_distance = r;
      rc = tzr_register_cloud_pairs_multiway_line_process_batch(
          ctx, &f, &tp, K, n.data(), pts.data(), P, pc.data(), seeds.data(), sols.data(), status.data(), index.data(),
          n_corr.data(), nullptr, nullptr, nullptr, &icp, nullptr, 0.0, nullptr, ir.data(), unc.data(), &lc,
          info.data(), counts.data(), w.data(), mask.data(), poses.data(), lsumm.data(), pg_status.data(), 2,
          off.data(), 0.0, nullptr, nullptr, nullptr);
    } else {
      tzr_pose_graph_params pgc;
      tzr_pose_graph_params_default(&pgc);
      pgc.max_correspondence_distance = r;
      rc = tzr_register_cloud_pairs_multiway_batch(
          ctx, &f, &tp, K, n.data(), pts.data(), P, pc.data(), seeds.data(), sols.data(), status.data(), index.data(),
          n_corr.data(), nullptr, nullptr, nullptr, &icp, nullptr, 0.0, nullptr, ir.data(), unc.data(), &pgc,
          info.data(), counts.data(), w.data(), mask.data(), poses.data(), summ.data(), pg_status.data(), 2, off.data(),
          v, map_p, map_counts.data(), nullptr);
    }
    CHECK(rc == TZR_OK);
    for (int g = 0; g < 2; ++g) {
      const auto& m = mw[g];
      CHECK(pg_status[g] == TZR_OK && m.pose_graph_status == TZR_OK);
      CHECK(m.poses.size() == seqs[g].clouds.size() && m.pairs.size() == seqs[g].pairs.size());
      for (int k = off[g]; k < off[g + 1]; ++k) CHECK(same_pose(m.poses[k - off[g]], poses[k]));
      for (int p = pair_lo[g]; p < pair_lo[g + 1]; ++p) {
        const int j = p - pair_lo[g];
        CHECK(m.pairs[j].status == status[p] && m.pairs[j].solution.valid == (sols[p].valid != 0));
        CHECK(m.edge_weights[j] == w[p] && m.edge_inliers[j] == (mask[p] != 0));
        CHECK(m.information_counts[j] == counts[p]);
        for (int a = 0; a < 6; ++a)
          for (int b = 0; b < 6; ++b) CHECK(m.information[j](a, b) == info[36 * p + 6 * a + b]);
        if (m.pairs[j].refined) CHECK(m.pairs[j].icp.fitness == ir[p].fitness);
      }
      if (lp) {
        CHECK(m.line_process.pruned == lsumm[g].pruned && m.line_process.residual == lsumm[g].residual);
        for (int q = 0; q < 2; ++q)
          CHECK(m.line_process.iterations[q] == lsumm[g].iterations[q] && m.line_process.mu[q] == lsumm[g].mu[q]);
        CHECK(m.map.empty());
      } else {
        CHECK(m.iterations == summ[g].iterations && m.inner_iterations == summ[g].inner_iterations &&
              m.cost == summ[g].cost);
        CHECK(map_counts[g] > 0 && static_cast<int>(m.map.size()) == map_counts[g] && m.map_colors.empty());
        CHECK(std::memcmp(&m.map[0].x, maps[g].data(), 12 * static_cast<size_t>(map_counts[g])) == 0);
      }
    }
  }
  // a single sequence: its pairs' records equal solveMultiway on it alone
  const auto one = solver.solveMultiway(seqs[1].clouds, seqs[1].pairs, cp, ip, pg);
  const auto both = solver.solveMultiwayBatch(seqs, cp, ip, pg);
  for (size_t j = 0; j < one.pairs.size(); ++j) {
    CHECK(one.pairs[j].status == both[1].pairs[j].status && one.pairs[j].refined == both[1].pairs[j].refined);
    CHECK(one.information_counts[j] == both[1].information_counts[j]);
    CHECK(one.pairs[j].icp.fitness == both[1].pairs[j].icp.fitness &&
          one.pairs[j].icp.inlier_rmse == both[1].pairs[j].icp.inlier_rmse &&
          one.pairs[j].icp.solution.translation(0) == both[1].pairs[j].icp.solution.translation(0));
  }
  CHECK(one.edge_inliers == both[1].edge_inliers && one.iterations == both[1].iterations);
  std::cout << "ok" << std::endl;
  return 0;
}
