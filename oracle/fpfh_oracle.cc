// TEST INFRASTRUCTURE ONLY — CPU restatement of teaser::FPFHEstimation::computeFPFHFeatures
// (reference: teaser/src/fpfh.cc:15-43), which is a thin wrapper over PCL: NormalEstimationOMP with a radius search,
// then FPFHEstimationOMP with a (larger) radius search on the same KD-tree.  PCL is a system dependency of the
// reference (find_package(PCL 1.8), CMakeLists.txt) and is not part of the reference tree, so the
// algorithm below restates PCL's published sources (pcl/features/impl/normal_3d.hpp, feature.hpp
// solvePlaneParameters, common/impl/centroid.hpp computeMeanAndCovarianceMatrix, common/impl/eigen.hpp
// computeRoots/eigen33, features/src/pfh_tools.cpp computePairFeatures, features/impl/fpfh.hpp
// computePointSPFHSignature / weightPointSPFHSignature) in the same float arithmetic.
//
// PARITY STATUS: pinned to the reference's golden vector test/teaser/data/bunny_fpfh.csv (397 x 33 values, the
// expected output of computeFPFHFeatures(bunny.pcd, 0.03, 0.05) in test/teaser/feature-test.cc:52-90, tolerance
// 1e-4 there); see tests/test_fpfh_cpu.py for how closely this restatement reproduces it.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>

namespace {

struct Nb {
  float d2;
  int idx;
};

// pcl::search::KdTree -> KdTreeFLANN::radiusSearch: squared L2 in float (flann::L2_Simple: sequential sum), strict
// `< r^2`, results sorted by ascending distance (ties: by index here)
void radius_search(const float* pts, int n, int q, float r2, std::vector<Nb>& out) {
  out.clear();
  const float qx = pts[3 * q], qy = pts[3 * q + 1], qz = pts[3 * q + 2];
  for (int i = 0; i < n; ++i) {
    const float dx = qx - pts[3 * i], dy = qy - pts[3 * i + 1], dz = qz - pts[3 * i + 2];
    float d = dx * dx;
    d += dy * dy;
    d += dz * dz;
    if (d < r2) out.push_back({d, i});
  }
  std::sort(out.begin(), out.end(), [](const Nb& a, const Nb& b) { return a.d2 < b.d2 || (a.d2 == b.d2 && a.idx < b.idx); });
}

// ---- deterministic single-precision elementary functions --------------------------------------------------------
// PCL calls the C library's atan2f / cosf / sinf / acosf.  To make the CUDA path comparable BIT FOR BIT with this
// restatement, both sides use the same fixed sequences of IEEE float +, -, *, / and sqrt below (Cephes-style
// minimax polynomials, 1-2 ulp; no FMA contraction on either side) instead of their platform's libm, whose results
// differ in the last ulp between glibc and CUDA.  The csrc/fpfh.cu copies must stay operation-for-operation identical.
constexpr float kPiF = 3.14159265358979323846f;
constexpr float kPio2F = 1.57079632679489661923f;
constexpr float kPio4F = 0.78539816339744830962f;

inline float det_atan_pos(float x) {  // x >= 0
  float y;
  if (x > 2.414213562373095f) {
    y = kPio2F;
    x = -(1.0f / x);
  } else if (x > 0.4142135623730950f) {
    y = kPio4F;
    x = (x - 1.0f) / (x + 1.0f);
  } else {
    y = 0.0f;
  }
  const float z = x * x;
  const float p = (((8.05374449538e-2f * z - 1.38776856032e-1f) * z + 1.99777106478e-1f) * z - 3.33329491539e-1f) * z * x + x;
  return y + p;
}

inline float det_atan2(float y, float x) {
  if (x != x || y != y) return std::numeric_limits<float>::quiet_NaN();
  if (y == 0.0f) return (x < 0.0f) ? kPiF : 0.0f;
  if (x == 0.0f) return y > 0.0f ? kPio2F : -kPio2F;
  float a = det_atan_pos(std::fabs(y) / std::fabs(x));
  if (x < 0.0f) a = kPiF - a;
  return y < 0.0f ? -a : a;
}

inline float det_asin_small(float x) {  // |x| <= 0.5
  const float z = x * x;
  return ((((4.2163199048e-2f * z + 2.4181311049e-2f) * z + 4.5470025998e-2f) * z + 7.4953002686e-2f) * z + 1.6666752422e-1f) * z * x + x;
}

inline float det_acos01(float x) {  // x >= 0; NaN for x > 1 (like acosf)
  if (!(x <= 1.0f)) return std::numeric_limits<float>::quiet_NaN();
  if (x > 0.5f) return 2.0f * det_asin_small(std::sqrt(0.5f * (1.0f - x)));
  return kPio2F - det_asin_small(x);
}

inline float det_sin_q(float x) {  // |x| <= pi/4
  const float z = x * x;
  return ((-1.9515295891e-4f * z + 8.3321608736e-3f) * z - 1.6666654611e-1f) * z * x + x;
}
inline float det_cos_q(float x) {  // |x| <= pi/4
  const float z = x * x;
  return ((2.443315711809948e-5f * z - 1.388731625493765e-3f) * z + 4.166664568298827e-2f) * z * z - 0.5f * z + 1.0f;
}
inline void det_sincos_0_pi2(float t, float* s, float* c) {  // 0 <= t <= pi/2
  if (t <= kPio4F) {
    *s = det_sin_q(t);
    *c = det_cos_q(t);
  } else {
    const float u = kPio2F - t;
    *s = det_cos_q(u);
    *c = det_sin_q(u);
  }
}

// pcl::computeRoots2 / computeRoots (common/impl/eigen.hpp), Scalar = float
void compute_roots2(float b, float c, float* roots) {
  roots[0] = 0.f;
  float d = b * b - 4.0f * c;
  if (d < 0.0f) d = 0.0f;
  const float sd = std::sqrt(d);
  roots[2] = 0.5f * (b + sd);
  roots[1] = 0.5f * (b - sd);
}

void compute_roots(const float m[3][3], float* roots) {
  const float c0 = m[0][0] * m[1][1] * m[2][2] + 2.0f * m[0][1] * m[0][2] * m[1][2] - m[0][0] * m[1][2] * m[1][2] -
                   m[1][1] * m[0][2] * m[0][2] - m[2][2] * m[0][1] * m[0][1];
  const float c1 = m[0][0] * m[1][1] - m[0][1] * m[0][1] + m[0][0] * m[2][2] - m[0][2] * m[0][2] +
                   m[1][1] * m[2][2] - m[1][2] * m[1][2];
  const float c2 = m[0][0] + m[1][1] + m[2][2];
  if (std::fabs(c0) < std::numeric_limits<float>::epsilon()) {
    compute_roots2(c2, c1, roots);
    return;
  }
  const float s_inv3 = 1.0f / 3.0f;
  const float s_sqrt3 = std::sqrt(3.0f);
  const float c2_over_3 = c2 * s_inv3;
  float a_over_3 = (c1 - c2 * c2_over_3) * s_inv3;
  if (a_over_3 > 0.0f) a_over_3 = 0.0f;
  const float half_b = 0.5f * (c0 + c2_over_3 * (2.0f * c2_over_3 * c2_over_3 - c1));
  float q = half_b * half_b + a_over_3 * a_over_3 * a_over_3;
  if (q > 0.0f) q = 0.0f;
  const float rho = std::sqrt(-a_over_3);
  const float theta = det_atan2(std::sqrt(-q), half_b) * s_inv3;  // in [0, pi/3]
  float cos_theta, sin_theta;
  det_sincos_0_pi2(theta, &sin_theta, &cos_theta);
  roots[0] = c2_over_3 + 2.0f * rho * cos_theta;
  roots[1] = c2_over_3 - rho * (cos_theta + s_sqrt3 * sin_theta);
  roots[2] = c2_over_3 - rho * (cos_theta - s_sqrt3 * sin_theta);
  if (roots[0] >= roots[1]) std::swap(roots[0], roots[1]);
  if (roots[1] >= roots[2]) {
    std::swap(roots[1], roots[2]);
    if (roots[0] >= roots[1]) std::swap(roots[0], roots[1]);
  }
  if (roots[0] <= 0.0f) compute_roots2(c2, c1, roots);
}

inline void cross3(const float* a, const float* b, float* o) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}

// pcl::eigen33(mat, eigenvalue, eigenvector): smallest eigenvalue and its eigenvector
void eigen33_smallest(const float cov[3][3], float* eigenvalue, float* vec) {
  float scale = 0.f;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) scale = std::max(scale, std::fabs(cov[r][c]));
  if (scale <= std::numeric_limits<float>::min()) scale = 1.0f;
  float m[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) m[r][c] = cov[r][c] / scale;
  float roots[3];
  compute_roots(m, roots);
  *eigenvalue = roots[0] * scale;
  for (int d = 0; d < 3; ++d) m[d][d] -= roots[0];
  float v1[3], v2[3], v3[3];
  cross3(m[0], m[1], v1);
  cross3(m[0], m[2], v2);
  cross3(m[1], m[2], v3);
  const float l1 = v1[0] * v1[0] + v1[1] * v1[1] + v1[2] * v1[2];
  const float l2 = v2[0] * v2[0] + v2[1] * v2[1] + v2[2] * v2[2];
  const float l3 = v3[0] * v3[0] + v3[1] * v3[1] + v3[2] * v3[2];
  const float* best;
  float len;
  if (l1 >= l2 && l1 >= l3) {
    best = v1;
    len = l1;
  } else if (l2 >= l1 && l2 >= l3) {
    best = v2;
    len = l2;
  } else {
    best = v3;
    len = l3;
  }
  const float s = std::sqrt(len);
  for (int k = 0; k < 3; ++k) vec[k] = best[k] / s;
}

// pcl::computePairFeatures (features/src/pfh_tools.cpp)
bool pair_features(const float* p1, const float* n1, const float* p2, const float* n2, float* f1, float* f2,
                   float* f3, float* f4) {
  float dp[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
  *f4 = std::sqrt(dp[0] * dp[0] + dp[1] * dp[1] + dp[2] * dp[2]);
  if (*f4 == 0.0f) {
    *f1 = *f2 = *f3 = *f4 = 0.0f;
    return false;
  }
  float a[3] = {n1[0], n1[1], n1[2]}, b[3] = {n2[0], n2[1], n2[2]};
  const float angle1 = (a[0] * dp[0] + a[1] * dp[1] + a[2] * dp[2]) / *f4;
  const float angle2 = (b[0] * dp[0] + b[1] * dp[1] + b[2] * dp[2]) / *f4;
  if (det_acos01(std::fabs(angle1)) > det_acos01(std::fabs(angle2))) {
    for (int k = 0; k < 3; ++k) {
      a[k] = n2[k];
      b[k] = n1[k];
      dp[k] *= -1.0f;
    }
    *f3 = -angle2;
  } else {
    *f3 = angle1;
  }
  float v[3];
  cross3(dp, a, v);
  const float vn = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  if (vn == 0.0f) {
    *f1 = *f2 = *f3 = *f4 = 0.0f;
    return false;
  }
  for (int k = 0; k < 3; ++k) v[k] /= vn;
  float w[3];
  cross3(a, v, w);
  *f2 = v[0] * b[0] + v[1] * b[1] + v[2] * b[2];
  *f1 = det_atan2(w[0] * b[0] + w[1] * b[1] + w[2] * b[2], a[0] * b[0] + a[1] * b[1] + a[2] * b[2]);
  return true;
}

}  // namespace

extern "C" {

// normals_out: n x 4 floats (nx, ny, nz, curvature); NaN where fewer than 3 neighbours.  cov_variant: 0 = the
// single-pass float accumulation of PCL <= 1.11 (sum of products minus product of means), 1 = PCL >= 1.12 (same, on
// coordinates shifted by the first neighbour).
void orc_estimate_normals(const float* pts, int n, double radius, int cov_variant, float* normals_out) {
  const float r2 = static_cast<float>(radius * radius);
#pragma omp parallel
  {
    std::vector<Nb> nb;
#pragma omp for schedule(dynamic, 16)
    for (int i = 0; i < n; ++i) {
      float* o = normals_out + 4 * (size_t)i;
      radius_search(pts, n, i, r2, nb);
      if (nb.size() < 3) {
        o[0] = o[1] = o[2] = o[3] = std::numeric_limits<float>::quiet_NaN();
        continue;
      }
      float accu[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
      float K[3] = {0, 0, 0};
      if (cov_variant == 1)
        for (int k = 0; k < 3; ++k) K[k] = pts[3 * (size_t)nb[0].idx + k];
      for (const Nb& e : nb) {
        const float x = pts[3 * (size_t)e.idx] - K[0], y = pts[3 * (size_t)e.idx + 1] - K[1],
                    z = pts[3 * (size_t)e.idx + 2] - K[2];
        accu[0] += x * x;
        accu[1] += x * y;
        accu[2] += x * z;
        accu[3] += y * y;
        accu[4] += y * z;
        accu[5] += z * z;
        accu[6] += x;
        accu[7] += y;
        accu[8] += z;
      }
      const float cnt = static_cast<float>(nb.size());
      for (float& v : accu) v /= cnt;
      float cov[3][3];
      cov[0][0] = accu[0] - accu[6] * accu[6];
      cov[0][1] = accu[1] - accu[6] * accu[7];
      cov[0][2] = accu[2] - accu[6] * accu[8];
      cov[1][1] = accu[3] - accu[7] * accu[7];
      cov[1][2] = accu[4] - accu[7] * accu[8];
      cov[2][2] = accu[5] - accu[8] * accu[8];
      cov[1][0] = cov[0][1];
      cov[2][0] = cov[0][2];
      cov[2][1] = cov[1][2];
      float ev, nv[3];
      eigen33_smallest(cov, &ev, nv);
      const float eig_sum = cov[0][0] + cov[1][1] + cov[2][2];
      const float curvature = eig_sum != 0 ? std::fabs(ev / eig_sum) : 0.f;
      // flipNormalTowardsViewpoint, viewpoint (0, 0, 0)
      const float vx = 0.f - pts[3 * (size_t)i], vy = 0.f - pts[3 * (size_t)i + 1], vz = 0.f - pts[3 * (size_t)i + 2];
      const float cos_theta = vx * nv[0] + vy * nv[1] + vz * nv[2];
      if (cos_theta < 0) {
        nv[0] *= -1;
        nv[1] *= -1;
        nv[2] *= -1;
      }
      o[0] = nv[0];
      o[1] = nv[1];
      o[2] = nv[2];
      o[3] = curvature;
    }
  }
}

// out: n x 33 floats.  normals: n x 4 (as written by orc_estimate_normals).
void orc_fpfh_from_normals(const float* pts, const float* normals, int n, double radius, float* out) {
  const float r2 = static_cast<float>(radius * radius);
  const int nb1 = 11, nb2 = 11, nb3 = 11;
  const float d_pi = 1.0f / (2.0f * static_cast<float>(M_PI));
  std::vector<float> spfh((size_t)n * 33, 0.f);
  std::vector<std::vector<Nb>> nbs(n);
#pragma omp parallel for schedule(dynamic, 16)
  for (int p = 0; p < n; ++p) {
    radius_search(pts, n, p, r2, nbs[p]);
    const std::vector<Nb>& nb = nbs[p];
    if (nb.empty()) continue;
    float* h = spfh.data() + (size_t)p * 33;
    const float hist_incr = 100.0f / static_cast<float>(nb.size() - 1);
    for (const Nb& e : nb) {
      if (e.idx == p) continue;
      float f1, f2, f3, f4;
      if (!pair_features(pts + 3 * (size_t)p, normals + 4 * (size_t)p, pts + 3 * (size_t)e.idx,
                         normals + 4 * (size_t)e.idx, &f1, &f2, &f3, &f4))
        continue;
      // h_index = static_cast<int>(std::floor(nr_bins * ...)), clamped to [0, nr_bins - 1] (fpfh.hpp).  A NaN feature
      // (NaN normal) makes that cast undefined; x86 yields INT_MIN, i.e. bin 0 after the clamp — fixed to bin 0 here.
      auto bin = [](double v, int nbins) {
        if (!(v == v)) return 0;
        const double f = std::floor(v);
        if (f < 0.0) return 0;
        if (f >= (double)nbins) return nbins - 1;
        return (int)f;
      };
      h[bin(nb1 * ((f1 + M_PI) * d_pi), nb1)] += hist_incr;
      h[nb1 + bin(nb2 * ((f2 + 1.0) * 0.5), nb2)] += hist_incr;
      h[nb1 + nb2 + bin(nb3 * ((f3 + 1.0) * 0.5), nb3)] += hist_incr;
    }
  }
#pragma omp parallel for schedule(dynamic, 16)
  for (int p = 0; p < n; ++p) {
    float* o = out + (size_t)p * 33;
    for (int k = 0; k < 33; ++k) o[k] = 0.f;
    float sum[3] = {0, 0, 0};
    for (const Nb& e : nbs[p]) {
      if (e.d2 == 0) continue;
      const float weight = 1.0f / e.d2;
      const float* h = spfh.data() + (size_t)e.idx * 33;
      for (int s = 0; s < 3; ++s)
        for (int k = 0; k < 11; ++k) {
          const float val = h[11 * s + k] * weight;
          sum[s] += val;
          o[11 * s + k] += val;
        }
    }
    for (int s = 0; s < 3; ++s) {
      float sc = sum[s];
      if (sc != 0) sc = static_cast<float>(100.0 / sc);
      for (int k = 0; k < 11; ++k) o[11 * s + k] *= sc;
    }
  }
}

// teaser::FPFHEstimation::computeFPFHFeatures (fpfh.cc:15-43)
void orc_compute_fpfh(const float* pts, int n, double normal_radius, double fpfh_radius, int cov_variant,
                      float* normals_out, float* fpfh_out) {
  std::vector<float> normals((size_t)n * 4);
  orc_estimate_normals(pts, n, normal_radius, cov_variant, normals.data());
  if (normals_out) std::memcpy(normals_out, normals.data(), normals.size() * sizeof(float));
  orc_fpfh_from_normals(pts, normals.data(), n, fpfh_radius, fpfh_out);
}

}  // extern "C"
