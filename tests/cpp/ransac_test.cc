// teaser::RANSACRegistration against the C-ABI: registerPair equals tzr_ransac, registerBatch equals tzr_ransac_batch
// and each registerPair, and registerCloudPairs equals tzr_register_cloud_pairs_ransac with solveCloudPairs' seeds, bit
// for bit (transform, evaluation, iterations, converged, correspondences, the loop summary, statuses and global scales;
// registerCloudPairs returns the matched correspondences, not the evaluation's).
// usage: ransac_test   (needs a GPU; prints "ok")
#include <cmath>
#include <cstdint>
#include <cstring>
#include <iostream>
#include <stdexcept>
#include <utility>
#include <vector>

#include "teaser/ransac.h"
#include "teaser_b200.h"

#define CHECK(c)                                                                  \
  do {                                                                            \
    if (!(c)) {                                                                   \
      std::cerr << "CHECK failed: " #c " at line " << __LINE__ << std::endl;     \
      return 1;                                                                   \
    }                                                                             \
  } while (0)

static uint64_t rng_state = 0x5eed1234ull;
static float uniform() {  // [-1, 1)
  rng_state = rng_state * 6364136223846793005ull + 1442695040888963407ull;
  return (float)((rng_state >> 40) * (1.0 / 16777216.0)) * 2.0f - 1.0f;
}
static int below(int n) { return (int)((uniform() * 0.5f + 0.5f) * n) % n; }

// a wavy surface patch, and the same points rotated by `a` about z and shifted
static void scan_pair(int n, float a, teaser::PointCloud* src, teaser::PointCloud* dst) {
  for (int i = 0; i < n; ++i) {
    const float u = uniform(), v = uniform();
    src->push_back({u, v, 0.3f * std::sin(3 * u) * std::cos(2 * v) + 2.0f});
  }
  const float c = std::cos(a), s = std::sin(a);
  for (int i = 0; i < n; ++i) {
    const teaser::PointXYZ& p = (*src)[i];
    dst->push_back({c * p.x - s * p.y + 0.1f, s * p.x + c * p.y - 0.05f, p.z + 0.02f});
  }
}

static std::vector<std::pair<int, int>> rows(int n, int K, double outliers) {
  std::vector<std::pair<int, int>> c;
  for (int k = 0; k < K; ++k) {
    const int i = below(n);
    c.emplace_back(i, (uniform() * 0.5f + 0.5f) < outliers ? below(n) : i);
  }
  return c;
}

using Result = teaser::RANSACRegistration::Result;

static bool same_c(const Result& a, const tzr_icp_result& r, const std::vector<int32_t>* ev) {
  if (!(a.solution.scale == r.transform.scale &&
        std::memcmp(a.solution.rotation.data(), r.transform.rotation, 9 * sizeof(double)) == 0 &&
        std::memcmp(a.solution.translation.data(), r.transform.translation, 3 * sizeof(double)) == 0 &&
        std::memcmp(&a.fitness, &r.fitness, 8) == 0 && std::memcmp(&a.inlier_rmse, &r.inlier_rmse, 8) == 0 &&
        a.iterations == r.iterations && a.converged == (r.converged != 0)))
    return false;
  if (!ev) return true;
  if ((int)a.correspondences.size() != r.n_correspondences) return false;
  for (int k = 0; k < r.n_correspondences; ++k)
    if (a.correspondences[k].first != (*ev)[2 * k] || a.correspondences[k].second != (*ev)[2 * k + 1]) return false;
  return true;
}

static bool same(const Result& a, const Result& b) {
  return a.solution.scale == b.solution.scale &&
         std::memcmp(a.solution.rotation.data(), b.solution.rotation.data(), 9 * sizeof(double)) == 0 &&
         std::memcmp(a.solution.translation.data(), b.solution.translation.data(), 3 * sizeof(double)) == 0 &&
         a.fitness == b.fitness && a.inlier_rmse == b.inlier_rmse && a.iterations == b.iterations &&
         a.converged == b.converged && a.correspondences == b.correspondences;
}

static bool same_info(const teaser::RANSACInfo& a, const tzr_ransac_info& c) {
  return a.drawn == c.drawn && a.passed == c.passed && a.winner == c.winner && a.inliers == c.inliers &&
         a.usable == c.usable && std::memcmp(&a.rmse, &c.rmse, 8) == 0;
}

static teaser::NormalCloud normals(const teaser::PointCloud& pc, float a) {  // rotated by `a` about z from src's
  teaser::NormalCloud n;
  const float c = std::cos(a), s = std::sin(a);
  for (size_t i = 0; i < pc.size(); ++i) {
    const float nx = std::sin(3.0f * i), ny = std::cos(5.0f * i), nz = 0.5f;
    n.push_back({c * nx - s * ny, s * nx + c * ny, nz, 0.f});
  }
  return n;
}

int main() {
  tzr_ctx* ctx = nullptr;
  CHECK(tzr_ctx_create(0, &ctx) == TZR_OK);
  teaser::RANSACRegistration::Params prm;
  prm.max_correspondence_distance = 0.02;
  prm.check_edge_length = true;
  prm.check_normal = true;
  prm.normal_angle_threshold = 0.6;
  const teaser::RANSACRegistration rs(prm);
  tzr_ransac_params cp;
  tzr_ransac_params_default(&cp);
  cp.max_correspondence_distance = 0.02;
  cp.check_edge_length = 1;
  cp.check_normal = 1;
  cp.normal_angle_threshold = 0.6;

  // three problems: an ordinary one, one below ransac_n, one with duplicated rows; normals for the normal checker
  std::vector<teaser::PointCloud> S(3), D(3);
  std::vector<teaser::NormalCloud> SN(3), DN(3);
  std::vector<std::vector<std::pair<int, int>>> C(3);
  const float ang[3] = {0.4f, -0.2f, 0.8f};
  scan_pair(1500, ang[0], &S[0], &D[0]);
  scan_pair(300, ang[1], &S[1], &D[1]);
  scan_pair(2500, ang[2], &S[2], &D[2]);
  C[0] = rows(1500, 3000, 0.6);
  C[1] = rows(300, 2, 0.0);
  C[2] = rows(2500, 800, 0.3);
  for (int k = 0; k < 200; ++k) C[2].push_back(C[2][k]);
  const std::vector<uint64_t> seeds = {3, 4, 0xffffffffffffffffull};
  for (int b = 0; b < 3; ++b) {
    SN[b] = normals(S[b], 0.0f);
    DN[b] = normals(D[b], ang[b]);
  }

  std::vector<teaser::RANSACInfo> binfo;
  const std::vector<Result> batch = rs.registerBatch(S, D, C, seeds, SN, DN, &binfo);
  CHECK(batch.size() == 3 && binfo.size() == 3);
  for (int b = 0; b < 3; ++b) {
    teaser::RANSACInfo oinfo;
    const Result one = rs.registerPair(S[b], D[b], C[b], seeds[b], &SN[b], &DN[b], &oinfo);
    CHECK(same(one, batch[b]));
    std::vector<int32_t> r;
    for (const auto& c : C[b]) {
      r.push_back(c.first);
      r.push_back(c.second);
    }
    std::vector<int32_t> ev(2 * S[b].size());
    tzr_icp_result res;
    tzr_ransac_info info;
    CHECK(tzr_ransac(ctx, &cp, &S[b][0].x, (int)S[b].size(), &D[b][0].x, (int)D[b].size(), (int)C[b].size(), r.data(),
                     seeds[b], &SN[b][0].normal_x, &DN[b][0].normal_x, &res, &info, ev.data()) == TZR_OK);
    CHECK(same_c(one, res, &ev));
    CHECK(same_info(oinfo, info) && same_info(binfo[b], info));
  }
  CHECK(binfo[1].drawn == 0 && binfo[1].winner == -1);
  CHECK(binfo[0].winner >= 0 && binfo[0].passed < binfo[0].drawn);

  // the cloud table: a sequence of three scans and a pair in the other direction
  std::vector<teaser::PointCloud> clouds(3);
  scan_pair(1200, 0.3f, &clouds[0], &clouds[1]);
  teaser::PointCloud tmp;
  scan_pair(1200, -0.3f, &clouds[2], &tmp);
  const std::vector<std::pair<int, int>> pairs = {{0, 1}, {1, 2}, {1, 0}};
  teaser::RANSACRegistration::CloudPairParams fp;
  fp.normal_search_radius = 0.1;
  fp.fpfh_search_radius = 0.15;
  fp.use_absolute_scale = false;
  fp.use_tuple_test = false;
  const std::vector<uint64_t> rseeds = {7, 8, 9};
  const auto got = rs.registerCloudPairs(clouds, pairs, fp, rseeds);
  CHECK(got.size() == 3);
  const int P = 3;
  std::vector<int32_t> n = {1200, 1200, 1200}, pc = {0, 1, 1, 2, 1, 0}, status(P);
  std::vector<const float*> pts = {&clouds[0][0].x, &clouds[1][0].x, &clouds[2][0].x};
  std::vector<uint64_t> tseeds(P);
  std::vector<std::vector<int32_t>> corr(P, std::vector<int32_t>(2 * 2400));
  std::vector<int32_t*> corr_p(P);
  for (int p = 0; p < P; ++p) {
    tseeds[p] = fp.tuple_seed + 0x9E3779B97F4A7C15ull * (uint64_t)p;
    corr_p[p] = corr[p].data();
  }
  tzr_frontend_params f;
  tzr_frontend_params_default(&f);
  f.normal_search_radius = 0.1;
  f.fpfh_search_radius = 0.15;
  f.use_absolute_scale = 0;
  f.use_tuple_test = 0;
  std::vector<int64_t> cnt(P);
  std::vector<float> gs(P);
  std::vector<tzr_icp_result> res(P);
  std::vector<tzr_ransac_info> inf(P);
  CHECK(tzr_register_cloud_pairs_ransac(ctx, &f, &cp, 3, n.data(), pts.data(), P, pc.data(), tseeds.data(),
                                        rseeds.data(), status.data(), cnt.data(), corr_p.data(), gs.data(), res.data(),
                                        inf.data()) == TZR_OK);
  for (int p = 0; p < P; ++p) {
    CHECK(got[p].status == status[p] && got[p].registered == (status[p] == TZR_OK));
    CHECK(std::memcmp(&got[p].global_scale, &gs[p], 4) == 0);
    CHECK((int64_t)got[p].correspondences.size() == cnt[p]);
    for (int64_t k = 0; k < cnt[p]; ++k)
      CHECK(got[p].correspondences[k].first == corr[p][2 * k] &&
            got[p].correspondences[k].second == corr[p][2 * k + 1]);
    CHECK(got[p].registered);
    CHECK(same_c(got[p].ransac, res[p], nullptr) && same_info(got[p].info, inf[p]));
  }
  // a refused parameter throws
  teaser::RANSACRegistration::Params bad = prm;
  bad.ransac_n = 2;
  bool threw = false;
  try {
    teaser::RANSACRegistration(bad).registerPair(S[0], D[0], C[0], 0, &SN[0], &DN[0]);
  } catch (const std::runtime_error&) {
    threw = true;
  }
  CHECK(threw);
  tzr_ctx_destroy(ctx);
  std::cout << "ok" << std::endl;
  return 0;
}
