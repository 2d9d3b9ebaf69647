// RobustRegistrationSolver::solveCloudPairs against the façade chain it replaces: FPFHEstimation::
// computeFPFHFeaturesBatch over the clouds, Matcher::calculateCorrespondencesBatch over the pairs with the same tuple
// seed, then solve(src_cloud, dst_cloud, correspondences) per pair on a second solver with the same Params.
// usage: register_pairs_test   (needs a GPU; prints "ok")
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <iostream>
#include <utility>
#include <vector>

#include "teaser/fpfh.h"
#include "teaser/matcher.h"
#include "teaser/registration.h"

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
  for (int i = n - 1; i >= 0; --i) {  // reversed: the kept points do not keep their indices
    const teaser::PointXYZ p = raw[i];
    pc.push_back({c * p.x - s * p.y + shift, s * p.x + c * p.y, p.z});
  }
  return pc;
}

int main() {
  std::vector<teaser::PointCloud> clouds;
  clouds.push_back(scan(600, nullptr, 0.f, 0.f));
  clouds.push_back(scan(700, &clouds[0], 0.03f, 0.04f));
  clouds.push_back(scan(500, &clouds[1], 0.05f, 0.03f));
  clouds.push_back(scan(650, &clouds[0], -0.02f, -0.05f));
  const std::vector<std::pair<int, int>> pairs = {{0, 1}, {1, 2}, {2, 1}, {0, 3}, {3, 3}, {1, 0}};
  const double rn = 0.1, rf = 0.15;
  teaser::RobustRegistrationSolver::Params params;
  params.noise_bound = 0.01;
  params.estimate_scaling = false;
  params.rotation_cost_threshold = 1e-12;

  for (int flags = 0; flags < 2; ++flags) {
    teaser::RobustRegistrationSolver::CloudPairParams cp;
    cp.normal_search_radius = rn;
    cp.fpfh_search_radius = rf;
    cp.use_absolute_scale = false;
    cp.use_tuple_test = flags == 1;
    cp.tuple_scale = 0.9f;
    cp.tuple_seed = 4242 + flags;
    teaser::RobustRegistrationSolver batch(params);
    const auto got = batch.solveCloudPairs(clouds, pairs, cp);
    CHECK(got.size() == pairs.size());

    teaser::FPFHEstimation est;
    const auto feats = est.computeFPFHFeaturesBatch(clouds, rn, rf);
    std::vector<teaser::PointCloud> src, dst;
    std::vector<teaser::FPFHCloudPtr> fs, fd;
    for (const auto& p : pairs) {
      src.push_back(clouds[p.first]);
      dst.push_back(clouds[p.second]);
      fs.push_back(feats[p.first]);
      fd.push_back(feats[p.second]);
    }
    teaser::Matcher matcher;
    matcher.setTupleSeed(cp.tuple_seed);
    const auto corr = matcher.calculateCorrespondencesBatch(src, dst, fs, fd, cp.use_absolute_scale,
                                                            cp.use_crosscheck, cp.use_tuple_test, cp.tuple_scale);
    int solved = 0;
    for (size_t p = 0; p < pairs.size(); ++p) {
      CHECK(got[p].correspondences == corr[p]);
      if (corr[p].empty()) {
        CHECK(got[p].status != 0 && !got[p].solution.valid && got[p].max_clique.empty());
        continue;
      }
      CHECK(got[p].status == 0);
      teaser::RobustRegistrationSolver one(params);
      const teaser::RegistrationSolution s = one.solve(src[p], dst[p], corr[p]);
      const teaser::RegistrationSolution& g = got[p].solution;
      CHECK(g.valid == s.valid && g.scale == s.scale);
      CHECK(std::memcmp(g.rotation.data(), s.rotation.data(), 9 * sizeof(double)) == 0);
      for (int k = 0; k < 3; ++k) CHECK(g.translation(k) == s.translation(k));
      CHECK(got[p].max_clique == one.getInlierMaxClique());
      ++solved;
    }
    CHECK(solved > 0);
    // the last pair's global scale is the Matcher's getGlobalScale() after the batch
    const float g1 = got.back().global_scale, g2 = matcher.getGlobalScale();
    CHECK(std::memcmp(&g1, &g2, sizeof(float)) == 0);
  }
  std::cout << "ok" << std::endl;
  return 0;
}
