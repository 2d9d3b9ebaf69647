// teaser::MultiScaleICP against the C-ABI: refineBatch equals tzr_icp_multiscale_batch on the same inputs bit for bit
// (records, sizes, statuses, information matrices and counts), for point-to-plane with a kernel and for coloured ICP.
// usage: icp_multiscale_test   (needs a GPU; prints "ok")
#include <cmath>
#include <cstdint>
#include <cstring>
#include <iostream>
#include <stdexcept>
#include <vector>

#include "teaser/icp.h"
#include "teaser/registration.h"
#include "teaser_b200.h"

#define CHECK(c)                                                                  \
  do {                                                                            \
    if (!(c)) {                                                                   \
      std::cerr << "CHECK failed: " #c " at line " << __LINE__ << std::endl;     \
      return 1;                                                                   \
    }                                                                             \
  } while (0)

static uint64_t rng_state = 0x2468aceull;
static float uniform() {  // [-1, 1)
  rng_state = rng_state * 6364136223846793005ull + 1442695040888963407ull;
  return (float)((rng_state >> 40) * (1.0 / 16777216.0)) * 2.0f - 1.0f;
}

// a wavy textured surface patch, shifted along x by `shift`; colours from the unshifted (u, v)
static void scan(int n, float shift, teaser::PointCloud* pc, teaser::ColorCloud* cc) {
  for (int i = 0; i < n; ++i) {
    const float u = uniform(), v = uniform();
    pc->push_back({u + shift, v, 0.3f * std::sin(3 * u) * std::cos(2 * v) + 2.0f});
    const float a = 0.5f + 0.4f * std::sin(9 * u) * std::cos(7 * v), b = 0.5f + 0.4f * std::cos(5 * u + 3 * v);
    cc->push_back({a, b, 0.5f * (a + b)});
  }
}

int main() {
  std::vector<teaser::PointCloud> clouds(3);
  std::vector<teaser::ColorCloud> colors(3);
  scan(3000, 0.0f, &clouds[0], &colors[0]);
  scan(6000, 0.02f, &clouds[1], &colors[1]);
  scan(2500, -0.015f, &clouds[2], &colors[2]);
  const std::vector<std::pair<int, int>> pairs = {{0, 1}, {2, 1}, {1, 2}};
  std::vector<teaser::RegistrationSolution> init(3);
  for (int p = 0; p < 3; ++p) {
    init[p].valid = true;
    init[p].scale = p == 1 ? 1.01 : 1.0;
    init[p].rotation.setIdentity();
    init[p].translation.setZero();
  }
  tzr_ctx* ctx = nullptr;
  CHECK(tzr_ctx_create(0, &ctx) == TZR_OK);
  for (int m = 0; m < 2; ++m) {
    teaser::MultiScaleICP::Params prm;
    const double vox[3] = {0.08, 0.04, 0.02};
    const int iters[3] = {8, 5, 3};
    for (int s = 0; s < 3; ++s) prm.scales.push_back(teaser::ICPScale(vox[s], 1.5 * vox[s], iters[s]));
    prm.method = m ? teaser::MultiScaleICP::kColored : teaser::MultiScaleICP::kPointToPlane;
    prm.kernel = teaser::RobustKernel(teaser::RobustKernel::kHuber, 0.02);
    prm.lambda_geometric = 0.9;
    const teaser::MultiScaleICP icp(prm);
    const teaser::MultiScaleICP::Result r = icp.refineBatch(clouds, m ? colors : std::vector<teaser::ColorCloud>{},
                                                            pairs, init, true);
    const int K = 3, P = 3, S = 3;
    std::vector<tzr_icp_scale> sc(S);
    for (int s = 0; s < S; ++s) sc[s] = tzr_icp_scale{vox[s], 1.5 * vox[s], 2 * vox[s], 1e-6, 1e-6, iters[s], 0};
    std::vector<int32_t> n(K), pc = {0, 1, 2, 1, 1, 2}, nd(K * S), st(K * S), cnt(P);
    std::vector<const float*> pts(K), cols(K);
    for (int c = 0; c < K; ++c) {
      n[c] = (int32_t)clouds[c].size();
      pts[c] = &clouds[c][0].x;
      cols[c] = &colors[c][0].r;
    }
    std::vector<tzr_similarity> seeds(P);
    for (int p = 0; p < P; ++p) {
      std::memset(&seeds[p], 0, sizeof(tzr_similarity));
      seeds[p].scale = init[p].scale;
      seeds[p].rotation[0] = seeds[p].rotation[4] = seeds[p].rotation[8] = 1.0;
    }
    tzr_robust_kernel k;
    std::memset(&k, 0, sizeof(k));
    k.type = TZR_LOSS_HUBER;
    k.k = 0.02;
    std::vector<tzr_icp_result> res(P * S);
    std::vector<double> info(36 * P);
    CHECK(tzr_icp_multiscale_batch(ctx, m ? TZR_ICP_COLORED : TZR_ICP_POINT_TO_PLANE, S, sc.data(), K, n.data(),
                                   pts.data(), m ? cols.data() : nullptr, P, pc.data(), seeds.data(), 1e-3, 0.9, &k,
                                   res.data(), nd.data(), st.data(), info.data(), cnt.data()) == TZR_OK);
    CHECK(!r.too_large && r.records.size() == (size_t)P && r.information.size() == (size_t)P);
    for (int p = 0; p < P; ++p) {
      for (int s = 0; s < S; ++s) {
        const tzr_icp_result& c = res[p * S + s];
        const teaser::PointToPointICPResult& x = r.records[p][s];
        CHECK(x.solution.valid && x.solution.scale == c.transform.scale);
        CHECK(std::memcmp(x.solution.rotation.data(), c.transform.rotation, 9 * sizeof(double)) == 0);
        CHECK(std::memcmp(x.solution.translation.data(), c.transform.translation, 3 * sizeof(double)) == 0);
        CHECK(x.fitness == c.fitness && x.inlier_rmse == c.inlier_rmse && x.iterations == c.iterations &&
              x.converged == (c.converged != 0) && c.n_correspondences > 0);
      }
      for (int a = 0; a < 6; ++a)
        for (int b = 0; b < 6; ++b) CHECK(r.information[p](a, b) == info[36 * p + 6 * a + b]);
      CHECK(r.info_counts[p] == cnt[p] && cnt[p] > 0);
    }
    for (int c = 0; c < K; ++c)
      for (int s = 0; s < S; ++s) CHECK(r.n_down[c][s] == nd[c * S + s] && r.status[c][s] == st[c * S + s]);
  }
  bool threw = false;
  try {
    teaser::MultiScaleICP::Params prm;
    prm.scales = {teaser::ICPScale(0.08, 0.0, 3)};  // a distance of 0 is refused by the library
    teaser::MultiScaleICP(prm).refineBatch(clouds, {}, pairs, init);
  } catch (const std::runtime_error&) {
    threw = true;
  }
  CHECK(threw);
  threw = false;
  try {
    teaser::MultiScaleICP::Params prm;
    prm.scales = {teaser::ICPScale(0.08, 0.12, 3)};
    prm.method = teaser::MultiScaleICP::kColored;
    teaser::MultiScaleICP(prm).refineBatch(clouds, {}, pairs, init);  // coloured without colours
  } catch (const std::invalid_argument&) {
    threw = true;
  }
  CHECK(threw);
  tzr_ctx_destroy(ctx);
  std::cout << "ok" << std::endl;
  return 0;
}
