// The façade's batch methods against consecutive single calls: FPFHEstimation::computeFPFHFeaturesBatch and
// Matcher::calculateCorrespondencesBatch must return, bit for bit, what B calls of computeFPFHFeatures /
// calculateCorrespondences return, and leave the same state behind (normals, tuple seed, global scale).
// usage: frontend_batch_test   (needs a GPU; prints "ok")
#include <cmath>
#include <cstdint>
#include <cstring>
#include <iostream>
#include <vector>

#include "teaser/fpfh.h"
#include "teaser/matcher.h"

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

// a wavy surface patch, shifted and slightly rotated per cloud
static teaser::PointCloud surface(int n, float shift, float angle) {
  teaser::PointCloud pc;
  const float c = std::cos(angle), s = std::sin(angle);
  for (int i = 0; i < n; ++i) {
    const float u = uniform(), v = uniform();
    const float x = u, y = v, z = 0.3f * std::sin(3 * u) * std::cos(2 * v) + 0.003f * uniform();
    pc.push_back({c * x - s * y + shift, s * x + c * y, z + 2.0f});
  }
  return pc;
}

static bool same_bytes(const void* a, const void* b, size_t n) { return n == 0 || std::memcmp(a, b, n) == 0; }

int main() {
  std::vector<teaser::PointCloud> src = {surface(800, 0.f, 0.f), teaser::PointCloud(), surface(5000, 0.5f, 0.1f),
                                         surface(3, 0.f, 0.f)};
  std::vector<teaser::PointCloud> dst = {surface(700, 0.01f, 0.05f), surface(20, 0.f, 0.f),
                                         surface(4500, 0.51f, 0.12f), surface(5, 0.f, 0.f)};
  const double rn = 0.08, rf = 0.12;

  // descriptors: one batch over all eight clouds against eight single calls
  std::vector<teaser::PointCloud> all(src);
  all.insert(all.end(), dst.begin(), dst.end());
  teaser::FPFHEstimation batch_est, single_est;
  const auto feats = batch_est.computeFPFHFeaturesBatch(all, rn, rf);
  CHECK(feats.size() == all.size());
  for (size_t b = 0; b < all.size(); ++b) {
    const auto one = single_est.computeFPFHFeatures(all[b], rn, rf);
    CHECK(one->size() == feats[b]->size());
    CHECK(same_bytes(one->data(), feats[b]->data(), one->size() * 33 * sizeof(float)));
  }
  const auto n1 = batch_est.getNormals(), n2 = single_est.getNormals();
  CHECK(n1.size() == n2.size() && same_bytes(n1.data(), n2.data(), n1.size() * sizeof(teaser::Normal)));

  // correspondences: the batch on one Matcher against consecutive single calls on another with the same seed
  std::vector<teaser::FPFHCloudPtr> fs(feats.begin(), feats.begin() + src.size()),
      fd(feats.begin() + src.size(), feats.end());
  for (int flags = 0; flags < 4; ++flags) {
    const bool crosscheck = flags & 1, tuple = flags & 2;
    teaser::Matcher mb, ms;
    mb.setTupleSeed(99 + flags);
    ms.setTupleSeed(99 + flags);
    const auto got = mb.calculateCorrespondencesBatch(src, dst, fs, fd, false, crosscheck, tuple, 0.9f);
    CHECK(got.size() == src.size());
    for (size_t b = 0; b < src.size(); ++b) {
      const auto want = ms.calculateCorrespondences(src[b], dst[b], *fs[b], *fd[b], false, crosscheck, tuple, 0.9f);
      CHECK(want == got[b]);
    }
    CHECK(mb.getTupleSeed() == ms.getTupleSeed());
    const float g1 = mb.getGlobalScale(), g2 = ms.getGlobalScale();
    CHECK(same_bytes(&g1, &g2, sizeof(float)));
  }
  CHECK(!teaser::Matcher().calculateCorrespondencesBatch(src, dst, fs, fd)[2].empty());
  std::cout << "ok" << std::endl;
  return 0;
}
