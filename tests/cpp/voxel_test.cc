// teaser::voxelDownSample and voxelDownSampleBatch against the C-ABI: both equal tzr_voxel_downsample on each cloud
// alone, bit for bit (points, count and voxel_of), and an empty cloud comes back empty.
// usage: voxel_test   (needs a GPU; prints "ok")
#include <cmath>
#include <cstdint>
#include <cstring>
#include <iostream>
#include <limits>
#include <vector>

#include "teaser/voxel.h"
#include "teaser_b200.h"

#define CHECK(c)                                                                  \
  do {                                                                            \
    if (!(c)) {                                                                   \
      std::cerr << "CHECK failed: " #c " at line " << __LINE__ << std::endl;     \
      return 1;                                                                   \
    }                                                                             \
  } while (0)

static uint64_t rng_state = 0x9e3779b97f4a7c15ull;
static float uniform() {  // [-1, 1)
  rng_state = rng_state * 6364136223846793005ull + 1442695040888963407ull;
  return (float)((rng_state >> 40) * (1.0 / 16777216.0)) * 2.0f - 1.0f;
}

// a wavy surface patch with a few non-finite rows
static teaser::PointCloud scan(int n) {
  teaser::PointCloud pc;
  for (int i = 0; i < n; ++i) {
    const float u = uniform(), v = uniform();
    pc.push_back({u, v, 0.3f * std::sin(3 * u) * std::cos(2 * v) + 0.003f * uniform() + 2.0f});
  }
  pc[n / 2].y = std::numeric_limits<float>::quiet_NaN();
  pc[n / 3].z = std::numeric_limits<float>::infinity();
  return pc;
}

int main() {
  const double v = 0.05;
  std::vector<teaser::PointCloud> clouds = {scan(20000), scan(1), teaser::PointCloud(), scan(7000)};
  std::vector<std::vector<int>> traces;
  const auto batch = teaser::voxelDownSampleBatch(clouds, v, &traces);
  CHECK(batch.size() == clouds.size() && traces.size() == clouds.size());
  CHECK(batch[2].empty() && traces[2].empty());
  tzr_ctx* ctx = nullptr;
  CHECK(tzr_ctx_create(-1, &ctx) == TZR_OK);
  for (size_t b = 0; b < clouds.size(); ++b) {
    std::vector<int> one_trace;
    const teaser::PointCloud one = teaser::voxelDownSample(clouds[b], v, &one_trace);
    CHECK(one.size() == batch[b].size() && one_trace == traces[b]);
    for (size_t i = 0; i < one.size(); ++i) CHECK(std::memcmp(&one[i], &batch[b][i], sizeof(teaser::PointXYZ)) == 0);
    if (clouds[b].empty()) continue;
    const int n = (int)clouds[b].size();
    std::vector<float> out(3 * (size_t)n);
    std::vector<int32_t> vo((size_t)n);
    int32_t m = -1;
    CHECK(tzr_voxel_downsample(ctx, &clouds[b][0].x, n, v, out.data(), &m, vo.data()) == TZR_OK);
    CHECK(m == (int32_t)one.size() && (n < 100 || m < n));
    CHECK(m == 0 || std::memcmp(out.data(), &one[0].x, (size_t)m * 12) == 0);
    for (int i = 0; i < n; ++i) CHECK(vo[i] == one_trace[i]);
  }
  tzr_ctx_destroy(ctx);
  bool threw = false;
  try {
    teaser::voxelDownSample(clouds[0], 0.0);
  } catch (const std::invalid_argument&) {
    threw = true;
  }
  CHECK(threw);
  std::cout << "ok" << std::endl;
  return 0;
}
