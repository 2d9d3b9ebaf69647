// teaser::ColoredICP, teaser::estimateColorGradients(Batch) and the colour overloads of teaser::voxelDownSample(Batch)
// against the C-ABI: each equals tzr_icp_colored, tzr_estimate_color_gradients and tzr_voxel_downsample_colors on the
// same inputs bit for bit, and the batch forms equal the single calls.
// usage: icp_colored_test   (needs a GPU; prints "ok")
#include <cmath>
#include <cstdint>
#include <cstring>
#include <iostream>
#include <stdexcept>
#include <vector>

#include "teaser/icp.h"
#include "teaser/normals.h"
#include "teaser/registration.h"
#include "teaser/voxel.h"
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

// a wavy textured surface patch, shifted along x by `shift`; colours from the unshifted (u, v)
static void scan(int n, float shift, teaser::PointCloud* pc, teaser::ColorCloud* cc) {
  for (int i = 0; i < n; ++i) {
    const float u = uniform(), v = uniform();
    pc->push_back({u + shift, v, 0.3f * std::sin(3 * u) * std::cos(2 * v) + 2.0f});
    const float a = 0.5f + 0.4f * std::sin(9 * u) * std::cos(7 * v), b = 0.5f + 0.4f * std::cos(5 * u + 3 * v);
    cc->push_back({a, b, 0.5f * (a + b)});
  }
}

static bool same(const teaser::ColoredICP::Result& a, const teaser::ColoredICP::Result& b) {
  return a.solution.scale == b.solution.scale &&
         std::memcmp(a.solution.rotation.data(), b.solution.rotation.data(), 9 * sizeof(double)) == 0 &&
         std::memcmp(a.solution.translation.data(), b.solution.translation.data(), 3 * sizeof(double)) == 0 &&
         a.fitness == b.fitness && a.inlier_rmse == b.inlier_rmse && a.iterations == b.iterations &&
         a.converged == b.converged && a.correspondences == b.correspondences;
}

int main() {
  teaser::PointCloud src, dst;
  teaser::ColorCloud sc, dc;
  scan(1500, 0.0f, &src, &sc);
  scan(1800, 0.01f, &dst, &dc);
  const teaser::NormalCloud dn = teaser::estimateNormals(dst, 0.15);
  tzr_ctx* ctx = nullptr;
  CHECK(tzr_ctx_create(0, &ctx) == TZR_OK);

  // gradients
  const double R = 0.05;
  const auto g = teaser::estimateColorGradients(dst, dn, dc, 2 * R);
  std::vector<double> gc(3 * dst.size());
  CHECK(tzr_estimate_color_gradients(ctx, &dst[0].x, (int)dst.size(), &dn[0].normal_x, &dc[0].r, 2 * R, gc.data()) ==
        TZR_OK);
  CHECK(g.size() == dst.size() && std::memcmp(g[0].data(), gc.data(), gc.size() * sizeof(double)) == 0);
  const auto gb = teaser::estimateColorGradientsBatch({src, dst}, {teaser::estimateNormals(src, 0.15), dn}, {sc, dc},
                                                      2 * R);
  CHECK(gb.size() == 2 && std::memcmp(gb[1][0].data(), gc.data(), gc.size() * sizeof(double)) == 0);

  // coloured ICP, with and without a kernel
  teaser::RegistrationSolution init;
  init.valid = true;
  init.scale = 1.0;
  init.rotation.setIdentity();
  init.translation.setZero();
  for (int kk = 0; kk < 2; ++kk) {
    teaser::ColoredICP::Params p;
    p.max_correspondence_distance = R;
    p.lambda_geometric = 0.9;
    const teaser::RobustKernel kern = kk ? teaser::RobustKernel(teaser::RobustKernel::kTukey, 0.03)
                                         : teaser::RobustKernel();
    const teaser::ColoredICP icp(p, kern);
    const teaser::ColoredICP::Result r = icp.refine(src, dst, dn, sc, dc, init);
    tzr_icp_params cp;
    tzr_icp_params_default(&cp);
    cp.max_correspondence_distance = R;
    tzr_similarity s;
    std::memset(&s, 0, sizeof(s));
    s.scale = 1.0;
    s.rotation[0] = s.rotation[4] = s.rotation[8] = 1.0;
    tzr_robust_kernel k;
    std::memset(&k, 0, sizeof(k));
    k.type = TZR_LOSS_TUKEY;
    k.k = 0.03;
    tzr_icp_result cr;
    std::vector<int32_t> corr(2 * src.size());
    CHECK(tzr_icp_colored(ctx, &cp, &src[0].x, (int)src.size(), &dst[0].x, (int)dst.size(), &dn[0].normal_x, &s, &cr,
                          corr.data(), &sc[0].r, &dc[0].r, 0.9, kk ? &k : nullptr) == TZR_OK);
    CHECK(std::memcmp(r.solution.rotation.data(), cr.transform.rotation, 9 * sizeof(double)) == 0);
    CHECK(std::memcmp(r.solution.translation.data(), cr.transform.translation, 3 * sizeof(double)) == 0);
    CHECK(r.fitness == cr.fitness && r.inlier_rmse == cr.inlier_rmse && r.iterations == cr.iterations);
    CHECK((int)r.correspondences.size() == cr.n_correspondences);
    for (int c = 0; c < cr.n_correspondences; ++c)
      CHECK(r.correspondences[c].first == corr[2 * c] && r.correspondences[c].second == corr[2 * c + 1]);
    CHECK(r.iterations > 1);
    const auto rb = icp.refineBatch({dst, src}, {src, dst}, {teaser::estimateNormals(src, 0.15), dn}, {dc, sc},
                                    {sc, dc}, {init, init});
    CHECK(rb.size() == 2 && same(rb[1], r));
  }
  bool threw = false;
  try {
    teaser::ColoredICP::Params p;
    p.max_correspondence_distance = R;
    p.lambda_geometric = std::nan("");
    teaser::ColoredICP(p).refine(src, dst, dn, sc, dc, init);
  } catch (const std::runtime_error&) {
    threw = true;
  }
  CHECK(threw);

  // voxels with colours
  std::vector<int> trace;
  teaser::ColorCloud vc;
  const teaser::PointCloud vp = teaser::voxelDownSample(dst, dc, 0.05, &vc, &trace);
  const teaser::PointCloud vplain = teaser::voxelDownSample(dst, 0.05);
  CHECK(vp.size() == vplain.size() && vc.size() == vp.size() && vp.size() < dst.size());
  CHECK(std::memcmp(&vp[0].x, &vplain[0].x, vp.size() * sizeof(teaser::PointXYZ)) == 0);
  std::vector<float> po(3 * dst.size()), co(3 * dst.size());
  std::vector<int32_t> vo(dst.size());
  int32_t m = 0;
  CHECK(tzr_voxel_downsample_colors(ctx, &dst[0].x, (int)dst.size(), 0.05, po.data(), &m, vo.data(), &dc[0].r,
                                    co.data()) == TZR_OK);
  CHECK(m == (int32_t)vc.size() && std::memcmp(&vc[0].r, co.data(), vc.size() * sizeof(teaser::ColorRGB)) == 0);
  for (size_t i = 0; i < dst.size(); ++i) CHECK(trace[i] == vo[i]);
  std::vector<teaser::ColorCloud> vcb;
  const auto vpb = teaser::voxelDownSampleBatch({src, dst}, {sc, dc}, 0.05, &vcb);
  CHECK(vpb.size() == 2 && vcb.size() == 2 && vcb[1].size() == vc.size());
  CHECK(std::memcmp(&vcb[1][0].r, &vc[0].r, vc.size() * sizeof(teaser::ColorRGB)) == 0);
  CHECK(std::memcmp(&vpb[1][0].x, &vp[0].x, vp.size() * sizeof(teaser::PointXYZ)) == 0);

  tzr_ctx_destroy(ctx);
  std::cout << "ok" << std::endl;
  return 0;
}
