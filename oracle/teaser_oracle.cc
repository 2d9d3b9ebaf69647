// =============================================================================
// teaser_oracle.cc — CPU restatement ("oracle") of the TEASER++ solve() hot path.
//
// THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
// and bench.py's cpu_baseline / --impl reference legs may load the library built from
// this file.  The product path (teaser-plusplus_b200/csrc) never links, includes or
// calls anything in oracle/.
//
// Parity status: the true reference is not built alongside this project (it needs Eigen, PMC
// and tinyply, fetched at configure time).  This restatement is pinned against the reference's
// own golden vectors (tests/golden/, data files copied from the reference's test/...):
// tls-test KATs, translation-solver KAT, rotation-solver KAT, scale-solver KATs, the
// six benchmark_* end-to-end fixtures and the PMC toy graphs (tests/test_oracle_*.py).
// The max-clique stage replaces the un-vendored, un-pinned PMC library
// (https://github.com/jingnanshi/pmc.git, fetched at configure time with no tag by
// the reference's teaser/CMakeLists.txt:6-8) by an own exact branch-and-bound that
// follows PMC's published structure (k-core bound -> greedy heuristic -> k-core pruning
// -> greedy-colouring branch and bound).  Its result is a *mathematically* maximum
// clique; it equals PMC's answer as an index set whenever the maximum clique is unique.
// At benchmark scale the reference's tests do not pin the clique: "parity unpinned" there.
//
// Every function cites the reference file:line it restates (paths relative to
// the reference repository).  Build: see oracle/Makefile
//   g++ -O3 -DNDEBUG -fopenmp -ffp-contract=off  (mirrors the reference's Release flags,
//   CMakeLists.txt:11-15; no -march=native => no FMA contraction, SURVEY Q6).
// =============================================================================
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <numeric>
#include <utility>
#include <vector>

#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

using i64 = long long;

double now_ms() {
  using namespace std::chrono;
  return duration<double, std::milli>(steady_clock::now().time_since_epoch()).count();
}

int max_threads() {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

// ----------------------------------------------------------------------------
// 3x3 helpers (column-major, like Eigen::Matrix3d)
// ----------------------------------------------------------------------------
struct M3 {
  double a[9];  // a[c*3+r]
  double& operator()(int r, int c) { return a[c * 3 + r]; }
  double operator()(int r, int c) const { return a[c * 3 + r]; }
};

M3 m3_identity() {
  M3 m;
  for (int i = 0; i < 9; ++i) m.a[i] = 0;
  m(0, 0) = m(1, 1) = m(2, 2) = 1;
  return m;
}

double m3_det(const M3& m) {
  return m(0, 0) * (m(1, 1) * m(2, 2) - m(1, 2) * m(2, 1)) -
         m(0, 1) * (m(1, 0) * m(2, 2) - m(1, 2) * m(2, 0)) +
         m(0, 2) * (m(1, 0) * m(2, 1) - m(1, 1) * m(2, 0));
}

// Plane rotation [c s; -s c] (same convention as a Jacobi/Givens rotation object).
struct Rot {
  double c, s;
};

// A <- J^T-style application on rows p,q:  row_p = c*row_p + s*row_q ; row_q = -s*row_p + c*row_q
void rot_left(M3& A, int p, int q, Rot j) {
  for (int col = 0; col < 3; ++col) {
    double xp = A(p, col), xq = A(q, col);
    A(p, col) = j.c * xp + j.s * xq;
    A(q, col) = -j.s * xp + j.c * xq;
  }
}
// A <- A * J on columns p,q: col_p = c*col_p - s*col_q ; col_q = s*col_p + c*col_q
void rot_right(M3& A, int p, int q, Rot j) {
  for (int row = 0; row < 3; ++row) {
    double xp = A(row, p), xq = A(row, q);
    A(row, p) = j.c * xp - j.s * xq;
    A(row, q) = j.s * xp + j.c * xq;
  }
}

// Two-sided Jacobi SVD of a 3x3 matrix, H = U * diag(S) * V^T, U and V full orthogonal,
// singular values non-negative and sorted descending.  This plays the role of
// Eigen::JacobiSVD<Matrix3d>(H, ComputeFullU|ComputeFullV) used by utils::svdRot
// (teaser/include/teaser/utils.h:121-136).  Eigen itself is not part of the reference
// tree; the algorithm below is the textbook two-sided (Kogbetliantz) Jacobi iteration:
// for every off-diagonal pair, first symmetrise the 2x2 block with a rotation, then
// diagonalise it with a symmetric Jacobi rotation.
void svd3(const M3& H, M3& U, double S[3], M3& V) {
  M3 A = H;
  U = m3_identity();
  V = m3_identity();
  const double eps = std::numeric_limits<double>::epsilon();
  const double tiny = std::numeric_limits<double>::min();
  double max_diag = std::max(std::fabs(A(0, 0)), std::max(std::fabs(A(1, 1)), std::fabs(A(2, 2))));
  for (int sweep = 0; sweep < 64; ++sweep) {
    bool finished = true;
    for (int p = 1; p < 3; ++p) {
      for (int q = 0; q < p; ++q) {
        double thr = std::max(tiny, 2.0 * eps * max_diag);
        if (std::fabs(A(p, q)) > thr || std::fabs(A(q, p)) > thr) {
          finished = false;
          // 2x2 block m = [A(p,p) A(p,q); A(q,p) A(q,q)]
          double m00 = A(p, p), m01 = A(p, q), m10 = A(q, p), m11 = A(q, q);
          // rot1 makes the block symmetric
          Rot rot1;
          double t = m00 + m11, d = m10 - m01;
          if (std::fabs(d) < tiny) {
            rot1.c = 1;
            rot1.s = 0;
          } else {
            double u = t / d;
            double tmp = std::sqrt(1.0 + u * u);
            rot1.s = 1.0 / tmp;
            rot1.c = u / tmp;
          }
          // apply rot1 on the left of the 2x2 block
          double n00 = rot1.c * m00 + rot1.s * m10;
          double n01 = rot1.c * m01 + rot1.s * m11;
          double n11 = -rot1.s * m01 + rot1.c * m11;
          // symmetric Jacobi rotation diagonalising [n00 n01; n01 n11]
          Rot jr;
          double deno = 2.0 * std::fabs(n01);
          if (deno < tiny) {
            jr.c = 1;
            jr.s = 0;
          } else {
            double tau = (n00 - n11) / deno;
            double w = std::sqrt(tau * tau + 1.0);
            double tt = (tau > 0) ? 1.0 / (tau + w) : 1.0 / (tau - w);
            double sign_t = tt > 0 ? 1.0 : -1.0;
            double nn = 1.0 / std::sqrt(tt * tt + 1.0);
            jr.s = -sign_t * (n01 / std::fabs(n01)) * std::fabs(tt) * nn;
            jr.c = nn;
          }
          // j_left = rot1 * jr^T
          Rot jl;
          jl.c = rot1.c * jr.c + rot1.s * jr.s;
          jl.s = rot1.s * jr.c - rot1.c * jr.s;
          rot_left(A, p, q, jl);
          // U <- U * jl^T  (apply transpose on the right)
          Rot jlt{jl.c, -jl.s};
          rot_right(U, p, q, jlt);
          rot_right(A, p, q, jr);
          rot_right(V, p, q, jr);
          max_diag = std::max(max_diag, std::max(std::fabs(A(p, p)), std::fabs(A(q, q))));
        }
      }
    }
    if (finished) break;
  }
  // positive singular values
  for (int i = 0; i < 3; ++i) {
    double a = A(i, i);
    S[i] = std::fabs(a);
    if (a < 0)
      for (int r = 0; r < 3; ++r) U(r, i) = -U(r, i);
  }
  // sort descending (selection sort with column swaps, like Eigen's final ordering pass)
  for (int i = 0; i < 3; ++i) {
    int pos = i;
    for (int k = i + 1; k < 3; ++k)
      if (S[k] > S[pos]) pos = k;
    if (pos != i) {
      std::swap(S[i], S[pos]);
      for (int r = 0; r < 3; ++r) {
        std::swap(U(r, i), U(r, pos));
        std::swap(V(r, i), V(r, pos));
      }
    }
  }
}

// R maximising tr(R H) is invariant under positive scaling of H.  Like Eigen's JacobiSVD, which divides the matrix by
// its largest |entry| first, bring an H whose largest |entry| lies outside [2^-400, 2^400] into [1/2, 1) by an exact
// power of two; entries inside that range keep their bits (rot_trans.cu does the same).
void normalise_scale(double* a, int n) {
  double mx = 0.0;
  for (int i = 0; i < n; ++i) mx = std::max(mx, std::fabs(a[i]));
  if (mx > 0.0 && mx <= std::numeric_limits<double>::max() && (mx < 0x1p-400 || mx > 0x1p400)) {
    int e;
    std::frexp(mx, &e);
    for (int i = 0; i < n; ++i) a[i] = std::ldexp(a[i], -e);
  }
}

// utils::svdRot  (teaser/include/teaser/utils.h:121-136)
//   H = X * diag(W) * Y^T ; SVD ; if det(U)*det(V) < 0 negate V.col(2) ; R = V * U^T
M3 svd_rot(const double* X, const double* Y, const double* W, i64 m) {
  M3 H;
  for (int i = 0; i < 9; ++i) H.a[i] = 0;
  for (i64 j = 0; j < m; ++j) {
    const double w = W[j];
    const double xw0 = X[3 * j + 0] * w, xw1 = X[3 * j + 1] * w, xw2 = X[3 * j + 2] * w;
    const double y0 = Y[3 * j + 0], y1 = Y[3 * j + 1], y2 = Y[3 * j + 2];
    H(0, 0) += xw0 * y0; H(0, 1) += xw0 * y1; H(0, 2) += xw0 * y2;
    H(1, 0) += xw1 * y0; H(1, 1) += xw1 * y1; H(1, 2) += xw1 * y2;
    H(2, 0) += xw2 * y0; H(2, 1) += xw2 * y1; H(2, 2) += xw2 * y2;
  }
  M3 U, V;
  double S[3];
  normalise_scale(H.a, 9);
  svd3(H, U, S, V);
  if (m3_det(U) * m3_det(V) < 0) {
    for (int r = 0; r < 3; ++r) V(r, 2) = -V(r, 2);
  }
  M3 R;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R(r, c) = V(r, 0) * U(c, 0) + V(r, 1) * U(c, 1) + V(r, 2) * U(c, 2);
  return R;
}

// ----------------------------------------------------------------------------
// ScalarTLSEstimator::estimate   (teaser/src/registration.cc:21-88)
// ----------------------------------------------------------------------------
// Two deliberate deviations (DESIGN.md §3.3), shared with every device scalar TLS:
//  * tie order: end points are ordered by (value, payload), payload 2i entering / 2i+1 leaving.  The reference's
//    std::sort on the value alone leaves the order among equal values unspecified; std::stable_sort over end points
//    pushed in payload order gives exactly this order.
//  * exclusion: a measurement whose value or range is not finite (a TIM with d1 = 0, a NaN coordinate) contributes no
//    end points (keys +inf, no term in any sum, ranges.sum() included) and is no inlier.  With no kept measurement the
//    estimate is NaN.
void scalar_tls(const double* X, const double* ranges, i64 N, double* estimate, uint8_t* inliers) {
  auto kept = [&](i64 i) { return std::isfinite(X[i]) && std::isfinite(ranges[i]); };
  std::vector<std::pair<double, i64>> h;
  h.reserve(2 * N);
  const double inf = std::numeric_limits<double>::infinity();
  for (i64 i = 0; i < N; ++i) {  // :35-38
    h.push_back(std::make_pair(kept(i) ? X[i] - ranges[i] : inf, i + 1));
    h.push_back(std::make_pair(kept(i) ? X[i] + ranges[i] : inf, -i - 1));
  }
  // ascending order, compare on value only   :41-42 (stable: ties keep payload order)
  std::stable_sort(h.begin(), h.end(),
                   [](const std::pair<double, i64>& a, const std::pair<double, i64>& b) { return a.first < b.first; });

  // weights = 1 / ranges^2   :45-46
  std::vector<double> weights(N);
  for (i64 i = 0; i < N; ++i) {
    double sq = ranges[i] * ranges[i];
    weights[i] = 1.0 / sq;
  }
  const i64 nr_centers = 2 * N;
  double ranges_inverse_sum = 0;  // ranges.sum()  :51
  for (i64 i = 0; i < N; ++i)
    if (kept(i)) ranges_inverse_sum += ranges[i];
  double dot_X_weights = 0, dot_weights_consensus = 0;
  i64 consensus_set_cardinal = 0;
  double sum_xi = 0, sum_xi_square = 0;

  // running argmin with Eigen minCoeff semantics (first strict minimum; NaN never wins
  // unless it is the first element)   :77-79
  double best_cost = 0, best_xhat = std::numeric_limits<double>::quiet_NaN();
  bool first = true;
  for (i64 i = 0; i < nr_centers; ++i) {  // :58-75
    i64 idx = std::llabs(h[i].second) - 1;
    if (!kept(idx)) continue;
    int epsilon = (h[i].second > 0) ? 1 : -1;
    consensus_set_cardinal += epsilon;
    dot_weights_consensus += epsilon * weights[idx];
    dot_X_weights += epsilon * weights[idx] * X[idx];
    ranges_inverse_sum -= epsilon * ranges[idx];
    sum_xi += epsilon * X[idx];
    sum_xi_square += epsilon * X[idx] * X[idx];

    double x_hat = dot_X_weights / dot_weights_consensus;
    double residual = consensus_set_cardinal * x_hat * x_hat + sum_xi_square - 2 * sum_xi * x_hat;
    double x_cost = residual + ranges_inverse_sum;
    if (first || x_cost < best_cost) {
      best_cost = x_cost;
      best_xhat = x_hat;
      first = false;
    }
  }
  if (estimate) *estimate = best_xhat;
  if (inliers) {  // :86
    for (i64 i = 0; i < N; ++i) inliers[i] = kept(i) && std::fabs(X[i] - best_xhat) <= ranges[i];
  }
}

// column norms: src.array().square().colwise().sum().array().sqrt()  (registration.cc:415-418,
// :434-437).  Summation order (x^2 + y^2) + z^2 (SSE2 packet reduction of the first two rows,
// then the scalar tail) — see DESIGN.md "summation order".
inline double col_norm(const double* p) {
  double xx = p[0] * p[0];
  double yy = p[1] * p[1];
  double zz = p[2] * p[2];
  double s = xx + yy;
  s = s + zz;
  return std::sqrt(s);
}

// ----------------------------------------------------------------------------
// RobustRegistrationSolver::computeTIMs  (teaser/src/registration.cc:512-551)
// ----------------------------------------------------------------------------
void compute_tims(const double* v, i64 N, double* vtilde, int* map) {
#pragma omp parallel for schedule(static)
  for (i64 i = 0; i < N - 1; i++) {
    i64 segment_start_idx = i * N - i * (i + 1) / 2;  // :531
    i64 segment_cols = N - 1 - i;                     // :532
    // temp = v - m * Ones(1,N) for ALL N columns (:536), then the right-most columns are kept (:539)
    std::vector<double> temp(3 * N);
    const double m0 = v[3 * i], m1 = v[3 * i + 1], m2 = v[3 * i + 2];
    for (i64 j = 0; j < N; ++j) {
      temp[3 * j + 0] = v[3 * j + 0] - m0;
      temp[3 * j + 1] = v[3 * j + 1] - m1;
      temp[3 * j + 2] = v[3 * j + 2] - m2;
    }
    std::memcpy(vtilde + 3 * segment_start_idx, temp.data() + 3 * (N - segment_cols),
                sizeof(double) * 3 * segment_cols);
    if (map) {
      // index map (:542-547)
      std::vector<int> map_addition(2 * N);
      for (i64 j = 0; j < N; ++j) {
        map_addition[2 * j + 0] = (int)i;
        map_addition[2 * j + 1] = (int)j;
      }
      std::memcpy(map + 2 * segment_start_idx, map_addition.data() + 2 * (N - segment_cols),
                  sizeof(int) * 2 * segment_cols);
    }
  }
}

// ScaleInliersSelector::solveForScale  (teaser/src/registration.cc:427-443)
void scale_inliers_selector(const double* src, const double* dst, i64 K, double noise_bound, double cbar2,
                            double* scale, uint8_t* inliers) {
  *scale = 1;
  std::vector<double> v1_dist(K), v2_dist(K);
  for (i64 k = 0; k < K; ++k) v1_dist[k] = col_norm(src + 3 * k);
  for (i64 k = 0; k < K; ++k) v2_dist[k] = col_norm(dst + 3 * k);
  double beta = 2 * noise_bound * std::sqrt(cbar2);
  for (i64 k = 0; k < K; ++k) inliers[k] = std::fabs(v1_dist[k] - v2_dist[k]) <= beta;
}

// TLSScaleSolver::solveForScale  (teaser/src/registration.cc:410-425)
void tls_scale_solver(const double* src, const double* dst, i64 K, double noise_bound, double cbar2,
                      double* scale, uint8_t* inliers) {
  std::vector<double> v1_dist(K), v2_dist(K), raw_scales(K), alphas(K);
  for (i64 k = 0; k < K; ++k) v1_dist[k] = col_norm(src + 3 * k);
  for (i64 k = 0; k < K; ++k) v2_dist[k] = col_norm(dst + 3 * k);
  for (i64 k = 0; k < K; ++k) raw_scales[k] = v2_dist[k] / v1_dist[k];
  double beta = 2 * noise_bound * std::sqrt(cbar2);
  for (i64 k = 0; k < K; ++k) alphas[k] = beta * (1.0 / v1_dist[k]);  // beta * v1_dist.cwiseInverse()
  scalar_tls(raw_scales.data(), alphas.data(), K, scale, inliers);
  // a repeated source point (d1 = 0): the pair is an inlier iff d2 <= beta, the fixed-scale rule (DESIGN.md §3.4)
  for (i64 k = 0; k < K; ++k)
    if (v1_dist[k] == 0) inliers[k] = v2_dist[k] <= beta;
}

// TLSTranslationSolver::solveForTranslation  (teaser/src/registration.cc:445-471)
void tls_translation(const double* src, const double* dst, i64 N, double noise_bound, double cbar2,
                     double t[3], uint8_t* inliers) {
  std::vector<double> raw(N), alphas(N);
  double beta = noise_bound * std::sqrt(cbar2);
  for (i64 i = 0; i < N; ++i) alphas[i] = beta * 1.0;
  std::vector<uint8_t> tmp(N);
  if (inliers)
    for (i64 i = 0; i < N; ++i) inliers[i] = 1;
  for (int axis = 0; axis < 3; ++axis) {
    for (i64 i = 0; i < N; ++i) raw[i] = dst[3 * i + axis] - src[3 * i + axis];
    scalar_tls(raw.data(), alphas.data(), N, &t[axis], tmp.data());
    if (inliers)
      for (i64 i = 0; i < N; ++i) inliers[i] = inliers[i] && tmp[i];
  }
}

// ----------------------------------------------------------------------------
// GNCTLSRotationSolver::solveForRotation  (teaser/src/registration.cc:764-866)
// trace (optional): per iteration {mu_used, cost, th1, th2}; weights are not traced.
// ----------------------------------------------------------------------------
struct GncResult {
  M3 R;
  double cost;
  int iterations;  // number of loop bodies entered
};

GncResult gnc_tls(const double* src, const double* dst, i64 match_size, size_t max_iterations,
                  double cost_threshold, double gnc_factor, double noise_bound, uint8_t* inliers,
                  double* trace, int trace_cap, double* weights_out) {
  GncResult res;
  res.R = m3_identity();
  double mu = 1;
  double prev_cost = std::numeric_limits<double>::infinity();
  double cost = std::numeric_limits<double>::infinity();
  double noise_bound_sq = std::pow(noise_bound, 2);
  if (noise_bound_sq < 1e-16) noise_bound_sq = 1e-2;  // :794-796
  std::vector<double> weights(match_size, 1.0), residuals_sq(match_size);
  int it_done = 0;
  for (size_t i = 0; i < max_iterations; ++i) {
    it_done = (int)i + 1;
    res.R = svd_rot(src, dst, weights.data(), match_size);  // :809
    const M3& R = res.R;
    for (i64 j = 0; j < match_size; ++j) {  // :812-813
      const double x = src[3 * j], y = src[3 * j + 1], z = src[3 * j + 2];
      double d0 = dst[3 * j + 0] - (R(0, 0) * x + R(0, 1) * y + R(0, 2) * z);
      double d1 = dst[3 * j + 1] - (R(1, 0) * x + R(1, 1) * y + R(1, 2) * z);
      double d2 = dst[3 * j + 2] - (R(2, 0) * x + R(2, 1) * y + R(2, 2) * z);
      residuals_sq[j] = d0 * d0 + d1 * d1 + d2 * d2;
    }
    if (i == 0) {  // :814-825
      double max_residual = residuals_sq[0];
      for (i64 j = 1; j < match_size; ++j) max_residual = std::max(max_residual, residuals_sq[j]);
      mu = 1 / (2 * max_residual / noise_bound_sq - 1);
      if (mu <= 0) break;
    }
    double th1 = (mu + 1) / mu * noise_bound_sq;  // :828-829
    double th2 = mu / (mu + 1) * noise_bound_sq;
    cost = 0;
    for (i64 j = 0; j < match_size; ++j) {  // :831-844
      cost += weights[j] * residuals_sq[j];
      if (residuals_sq[j] >= th1) {
        weights[j] = 0;
      } else if (residuals_sq[j] <= th2) {
        weights[j] = 1;
      } else {
        weights[j] = std::sqrt(noise_bound_sq * mu * (mu + 1) / residuals_sq[j]) - mu;
      }
    }
    if (trace && (int)i < trace_cap) {
      trace[4 * i + 0] = mu;
      trace[4 * i + 1] = cost;
      trace[4 * i + 2] = th1;
      trace[4 * i + 3] = th2;
    }
    double cost_diff = std::fabs(cost - prev_cost);  // :847
    mu = mu * gnc_factor;                            // :850
    prev_cost = cost;
    if (cost_diff < cost_threshold) break;  // :853
  }
  if (inliers)
    for (i64 j = 0; j < match_size; ++j) inliers[j] = weights[j] >= 0.5;  // :861-865
  if (weights_out)
    for (i64 j = 0; j < match_size; ++j) weights_out[j] = weights[j];
  res.cost = cost;
  res.iterations = it_done;
  return res;
}

// helper for FGR: utils::calculateDiameter (teaser/include/teaser/utils.h:107-112); returns float!
float calculate_diameter(const double* X, i64 n) {
  double cog[3] = {0, 0, 0};
  for (i64 j = 0; j < n; ++j)
    for (int r = 0; r < 3; ++r) cog[r] += X[3 * j + r];
  for (int r = 0; r < 3; ++r) cog[r] = cog[r] / (double)n;
  double mx = -1;
  for (i64 j = 0; j < n; ++j) {
    double a = X[3 * j] - cog[0], b = X[3 * j + 1] - cog[1], c = X[3 * j + 2] - cog[2];
    double t = a * a + b * b + c * c;
    if (t > mx) mx = t;
  }
  return (float)(2 * std::sqrt(mx));
}

// FastGlobalRegistrationSolver::solveForRotation (teaser/src/registration.cc:206-278)
GncResult fgr(const double* src, const double* dst, i64 match_size, size_t max_iterations,
              double cost_threshold, double gnc_factor, double noise_bound, uint8_t* inliers) {
  GncResult res;
  double noise_bound_sq = std::pow(noise_bound, 2);
  double cost = std::numeric_limits<double>::infinity();
  double src_diameter = calculate_diameter(src, match_size);
  double dest_diameter = calculate_diameter(dst, match_size);
  double global_scale = src_diameter > dest_diameter ? src_diameter : dest_diameter;
  global_scale /= noise_bound_sq;
  double mu = std::pow(global_scale, 2) / noise_bound_sq;
  double min_mu = 1.0;
  res.R = m3_identity();
  std::vector<double> l_pq(match_size, 1.0);
  int it_done = 0;
  for (size_t i = 0; i < max_iterations; ++i) {
    it_done = (int)i + 1;
    double scaled_mu = mu * noise_bound_sq;
    const M3 R = res.R;
    for (i64 j = 0; j < match_size; ++j) {
      const double x = src[3 * j], y = src[3 * j + 1], z = src[3 * j + 2];
      double d0 = dst[3 * j + 0] - (R(0, 0) * x + R(0, 1) * y + R(0, 2) * z);
      double d1 = dst[3 * j + 1] - (R(1, 0) * x + R(1, 1) * y + R(1, 2) * z);
      double d2 = dst[3 * j + 2] - (R(2, 0) * x + R(2, 1) * y + R(2, 2) * z);
      double sq = d0 * d0 + d1 * d1 + d2 * d2;
      l_pq[j] = std::pow(scaled_mu / (scaled_mu + sq), 2);
    }
    res.R = svd_rot(src, dst, l_pq.data(), match_size);
    cost = 0;
    for (i64 j = 0; j < match_size; ++j) {
      const M3& Q = res.R;
      const double x = src[3 * j], y = src[3 * j + 1], z = src[3 * j + 2];
      double d0 = dst[3 * j + 0] - (Q(0, 0) * x + Q(0, 1) * y + Q(0, 2) * z);
      double d1 = dst[3 * j + 1] - (Q(1, 0) * x + Q(1, 1) * y + Q(1, 2) * z);
      double d2 = dst[3 * j + 2] - (Q(2, 0) * x + Q(2, 1) * y + Q(2, 2) * z);
      double sq = d0 * d0 + d1 * d1 + d2 * d2;
      cost += (scaled_mu * sq) / (scaled_mu + sq);
    }
    if (cost < cost_threshold || mu < min_mu) break;
    mu /= gnc_factor;
  }
  if (inliers)
    for (i64 j = 0; j < match_size; ++j) inliers[j] = (l_pq[j] != 0.0);  // l_pq.cast<bool>()
  res.cost = cost;
  res.iterations = it_done;
  return res;
}

// utils::svdRot2d  (teaser/include/teaser/utils.h:145-160): H = X diag(W) Y^T (2x2), JacobiSVD, reflection fix on
// V.col(1), R = V U^T.  The 2x2 SVD is one two-sided Jacobi step (symmetrise, then diagonalise).
void svd_rot2d(const double* X, const double* Y, const double* W, i64 m, double R2[4] /* column-major 2x2 */) {
  double h00 = 0, h01 = 0, h10 = 0, h11 = 0;
  for (i64 j = 0; j < m; ++j) {
    const double w = W[j];
    const double x0 = X[3 * j] * w, x1 = X[3 * j + 1] * w;
    const double y0 = Y[3 * j], y1 = Y[3 * j + 1];
    h00 += x0 * y0; h01 += x0 * y1;
    h10 += x1 * y0; h11 += x1 * y1;
  }
  {
    double h[4] = {h00, h01, h10, h11};
    normalise_scale(h, 4);
    h00 = h[0], h01 = h[1], h10 = h[2], h11 = h[3];
  }
  // step 1: G1 = [c1 s1; -s1 c1] such that G1*H is symmetric
  double c1 = 1, s1 = 0;
  const double t = h00 + h11, d = h10 - h01;
  const double tiny = std::numeric_limits<double>::min();
  if (std::fabs(d) >= tiny) {
    const double u = t / d, hh = std::sqrt(1.0 + u * u);
    s1 = 1.0 / hh;
    c1 = u / hh;
  }
  const double n00 = c1 * h00 + s1 * h10, n01 = c1 * h01 + s1 * h11, n11 = c1 * h11 - s1 * h01;
  // step 2: J = [c2 s2; -s2 c2] diagonalising the symmetric block
  double c2 = 1, s2 = 0;
  if (2.0 * std::fabs(n01) >= tiny) {
    const double tau = (n00 - n11) / (2.0 * n01), w = std::sqrt(tau * tau + 1.0);
    const double tt = (tau >= 0) ? -1.0 / (tau + w) : 1.0 / (w - tau);
    c2 = 1.0 / std::sqrt(tt * tt + 1.0);
    s2 = tt * c2;
  }
  // L = J^T G1, D = L H J diagonal;  H = L^T D J^T  => U = L^T, V = J (then sign/sort fixes)
  const double cl = c2 * c1 + s2 * s1, sl = c2 * s1 - s2 * c1;
  double U[4] = {cl, sl, -sl, cl};   // column-major: U = L^T = [cl -sl; sl cl]
  double V[4] = {c2, -s2, s2, c2};   // column-major: V = J   = [c2 s2; -s2 c2]
  double d0 = cl * (h00 * c2 - h01 * s2) + sl * (h10 * c2 - h11 * s2);
  double d1 = -sl * (h00 * s2 + h01 * c2) + cl * (h10 * s2 + h11 * c2);
  if (d0 < 0) { d0 = -d0; U[0] = -U[0]; U[1] = -U[1]; }
  if (d1 < 0) { d1 = -d1; U[2] = -U[2]; U[3] = -U[3]; }
  if (d1 > d0) {  // sort descending
    std::swap(d0, d1);
    std::swap(U[0], U[2]); std::swap(U[1], U[3]);
    std::swap(V[0], V[2]); std::swap(V[1], V[3]);
  }
  const double detU = U[0] * U[3] - U[2] * U[1], detV = V[0] * V[3] - V[2] * V[1];
  if (detU * detV < 0) { V[2] = -V[2]; V[3] = -V[3]; }
  // R = V U^T
  R2[0] = V[0] * U[0] + V[2] * U[2];  // (0,0)
  R2[1] = V[1] * U[0] + V[3] * U[2];  // (1,0)
  R2[2] = V[0] * U[1] + V[2] * U[3];  // (0,1)
  R2[3] = V[1] * U[1] + V[3] * U[3];  // (1,1)
}

// QuatroSolver::solveForRotation (teaser/src/registration.cc:280-408): yaw-only GNC-TLS.  The reference keeps
// the noise bound in function-local statics (:329-330), i.e. the FIRST call's value sticks for the lifetime of
// the process; this restatement uses the solver's current params_.noise_bound (the evident intent).
GncResult quatro(const double* src, const double* dst, i64 match_size, size_t max_iterations, double cost_threshold,
                 double gnc_factor, double noise_bound, uint8_t* inliers) {
  GncResult res;
  res.R = m3_identity();
  double R2[4] = {1, 0, 0, 1};
  double mu = 1;
  double prev_cost = std::numeric_limits<double>::infinity();
  double cost = std::numeric_limits<double>::infinity();
  double noise_bound_sq = std::pow(noise_bound, 2);
  if (noise_bound_sq < 1e-16) noise_bound_sq = 1e-2;
  std::vector<double> weights(match_size, 1.0), residuals_sq(match_size);
  int it_done = 0;
  for (size_t i = 0; i < max_iterations; ++i) {
    it_done = (int)i + 1;
    svd_rot2d(src, dst, weights.data(), match_size, R2);
    for (i64 j = 0; j < match_size; ++j) {
      const double x = src[3 * j], y = src[3 * j + 1];
      const double d0 = dst[3 * j + 0] - (R2[0] * x + R2[2] * y);
      const double d1 = dst[3 * j + 1] - (R2[1] * x + R2[3] * y);
      residuals_sq[j] = d0 * d0 + d1 * d1;
    }
    if (i == 0) {
      double max_residual = residuals_sq[0];
      for (i64 j = 1; j < match_size; ++j) max_residual = std::max(max_residual, residuals_sq[j]);
      mu = 1 / (2 * max_residual / noise_bound_sq - 1);
      if (mu <= 0) break;
    }
    const double th1 = (mu + 1) / mu * noise_bound_sq, th2 = mu / (mu + 1) * noise_bound_sq;
    cost = 0;
    for (i64 j = 0; j < match_size; ++j) {
      cost += weights[j] * residuals_sq[j];
      if (residuals_sq[j] >= th1) weights[j] = 0;
      else if (residuals_sq[j] <= th2) weights[j] = 1;
      else weights[j] = std::sqrt(noise_bound_sq * mu * (mu + 1) / residuals_sq[j]) - mu;
    }
    const double cost_diff = std::fabs(cost - prev_cost);
    mu = mu * gnc_factor;
    prev_cost = cost;
    if (cost_diff < cost_threshold) break;
  }
  if (inliers)
    for (i64 j = 0; j < match_size; ++j) inliers[j] = weights[j] >= 0.4;  // :398-402
  res.R(0, 0) = R2[0]; res.R(1, 0) = R2[1]; res.R(0, 1) = R2[2]; res.R(1, 1) = R2[3];  // :407
  res.cost = cost;
  res.iterations = it_done;
  return res;
}

// ----------------------------------------------------------------------------
// teaser::Graph  (teaser/include/teaser/graph.h:29-207) — adjacency lists; addEdge performs
// the linear duplicate scan of hasEdge (graph.h:74-82,96-104) exactly as the reference does.
// ----------------------------------------------------------------------------
struct Graph {
  std::vector<std::vector<int>> adj;
  size_t num_edges = 0;
  void populateVertices(int n) { adj.resize(n); }
  bool hasEdge(int a, int b) const {
    if (a >= (int)adj.size() || b >= (int)adj.size()) return false;
    const auto& c = adj[a];
    return std::find(c.begin(), c.end(), b) != c.end();
  }
  void addEdge(int a, int b) {
    if (hasEdge(a, b)) return;
    adj[a].push_back(b);
    adj[b].push_back(a);
    num_edges++;
  }
};

// ----------------------------------------------------------------------------
// Max clique: restatement of teaser::MaxCliqueSolver::findMaxClique (teaser/src/graph.cc:12-125)
// with PMC replaced by own code (see file header).
// ----------------------------------------------------------------------------
enum { MODE_PMC_EXACT = 0, MODE_PMC_HEU = 1, MODE_KCORE_HEU = 2 };

// Batagelj–Zaversnik O(n+m) k-core decomposition (what pmc_graph::compute_cores computes;
// graph.cc:58-59).  Returns standard core numbers; max_core = degeneracy (test pin: K5 -> 4,
// test/teaser/graph-test.cc:155-167 expects ub = max_core+1 = 5).
void kcores(const std::vector<i64>& off, const std::vector<int>& edges, int n, std::vector<int>& core,
            std::vector<int>& order) {
  core.assign(n, 0);
  order.assign(n, 0);
  if (n == 0) return;
  std::vector<int> deg(n), pos(n);
  int md = 0;
  for (int v = 0; v < n; ++v) {
    deg[v] = (int)(off[v + 1] - off[v]);
    md = std::max(md, deg[v]);
  }
  std::vector<int> bin(md + 2, 0);
  for (int v = 0; v < n; ++v) bin[deg[v]]++;
  int start = 0;
  for (int d = 0; d <= md; ++d) {
    int num = bin[d];
    bin[d] = start;
    start += num;
  }
  for (int v = 0; v < n; ++v) {
    pos[v] = bin[deg[v]];
    order[pos[v]] = v;
    bin[deg[v]]++;
  }
  for (int d = md; d >= 1; --d) bin[d] = bin[d - 1];
  bin[0] = 0;
  for (int i = 0; i < n; ++i) {
    int v = order[i];
    core[v] = deg[v];
    for (i64 e = off[v]; e < off[v + 1]; ++e) {
      int u = edges[e];
      if (deg[u] > deg[v]) {
        int du = deg[u], pu = pos[u], pw = bin[du], w = order[pw];
        if (u != w) {
          pos[u] = pw;
          order[pu] = w;
          pos[w] = pu;
          order[pw] = u;
        }
        bin[du]++;
        deg[u]--;
      }
    }
  }
}

struct Bits {
  int W = 0;  // 64-bit words per row
  std::vector<uint64_t> d;
  void init(int n_rows, int n_cols) {
    W = (n_cols + 63) / 64;
    d.assign((size_t)n_rows * W, 0);
  }
  uint64_t* row(int r) { return d.data() + (size_t)r * W; }
  const uint64_t* row(int r) const { return d.data() + (size_t)r * W; }
};

struct CliqueScratch {
  // one slot per recursion depth; the outer vectors are sized once (depth <= ub+2) so that
  // growing an inner vector never invalidates pointers held by shallower levels
  std::vector<std::vector<uint64_t>> bits;  // per level: P (W) | Q (W) | R (W)
  std::vector<std::vector<int>> ord;        // per level: (vertex, colour) pairs
  void init(int max_depth, int W) {
    bits.assign(max_depth, std::vector<uint64_t>());
    ord.assign(max_depth, std::vector<int>());
    for (auto& b : bits) b.assign(3 * (size_t)W, 0);
  }
};

struct CliqueSearch {
  const Bits* A;
  int n, W;
  std::atomic<int> best;
  std::vector<int> best_clique;  // in compact labels
  const int* orig = nullptr;     // compact label -> original vertex id (for the canonical tie-break)
  double deadline_ms;
  std::atomic<bool> timed_out;
  std::atomic<i64> nodes;
  double pass_deadline_ms = -1;       // first pass of the two-pass scheme (see find_max_clique); < 0 = none
  std::atomic<bool> budget_out{false};
  int strict = 0;  // 1 after a Nemhauser-Trotter reduction: prune whatever cannot BEAT the incumbent (see find_max_clique)
  int stop_at = 0x7fffffff;  // ... and stop as soon as the incumbent reaches this (the LP upper bound)

  // BBMC-style expansion (Tomita / San Segundo): a greedy sequential colouring of P yields, for the
  // vertices that could still beat the incumbent, a branching order and a colour bound.
  // P lives in S.bits[depth][0..W).
  void expand(std::vector<int>& C, CliqueScratch& S, int depth) {
    i64 nd = nodes.fetch_add(1, std::memory_order_relaxed);
    if ((nd & 0xff) == 0) {
      const double t = now_ms();
      if (t > deadline_ms) timed_out.store(true);
      if (pass_deadline_ms >= 0 && t > pass_deadline_ms) budget_out.store(true);
    }
    if (timed_out.load(std::memory_order_relaxed) || budget_out.load(std::memory_order_relaxed)) return;
    if (best.load(std::memory_order_relaxed) >= stop_at) return;
    uint64_t* P = S.bits[depth].data();
    uint64_t* Q = P + W;
    uint64_t* R = Q + W;
    // Canonical result: ALL maximum cliques are enumerated (branches are cut only when they cannot even
    // tie the incumbent) and the lexicographically smallest sorted index set is kept.  When the maximum
    // clique is unique this is exactly the reference's answer; when it is not, the reference (PMC, multi-
    // threaded) returns an unspecified one of them.
    int pc = 0;
    for (int w = 0; w < W; ++w) pc += __builtin_popcountll(P[w]);
    // Universal vertices (adjacent to every other candidate) belong to every maximum clique of this subproblem:
    // they join C without branching (the device kernel does the same in node_reduce).  Without this, dense
    // subproblems re-branch over interchangeable universal vertices and never finish.
    struct PopGuard {
      std::vector<int>& c;
      size_t n0;
      ~PopGuard() { c.resize(n0); }
    } guard{C, C.size()};
    if (pc >= 32) {
      int absorbed = 0;
      for (int w = 0; w < W; ++w) {
        uint64_t m = P[w];
        while (m) {
          const int bpos = __builtin_ctzll(m);
          m &= m - 1;
          const int v = w * 64 + bpos;
          const uint64_t* nv = A->row(v);
          int d = 0;
          for (int x = 0; x < W; ++x) d += __builtin_popcountll(P[x] & nv[x]);
          if (d == pc - 1) {  // P itself is not modified inside this scan, so the test is against the full candidate set
            C.push_back(v);
            ++absorbed;
          }
        }
      }
      if (absorbed) {
        for (size_t q = guard.n0; q < C.size(); ++q) P[C[q] >> 6] &= ~(1ull << (C[q] & 63));
        pc -= absorbed;
        if (pc == 0) {
          if ((int)C.size() >= best.load(std::memory_order_relaxed)) {
#pragma omp critical(orc_clique_update)
            {
              if ((int)C.size() > best.load()) {
                best_clique = C;
                best.store((int)C.size());
              } else if ((int)C.size() == best.load()) {
                std::vector<int> a(C.size()), b(best_clique.size());
                for (size_t q = 0; q < C.size(); ++q) a[q] = orig[C[q]];
                for (size_t q = 0; q < best_clique.size(); ++q) b[q] = orig[best_clique[q]];
                std::sort(a.begin(), a.end());
                std::sort(b.begin(), b.end());
                if (b.size() != a.size() || a < b) best_clique = C;
              }
            }
          }
          return;
        }
      }
    }
    int kmin = best.load(std::memory_order_relaxed) + strict - (int)C.size();
    if (kmin < 1) kmin = 1;
    std::vector<int>& ord = S.ord[depth];
    if (ord.size() < 2 * (size_t)pc) ord.resize(2 * (size_t)pc);
    std::memcpy(Q, P, sizeof(uint64_t) * W);
    int cnt = 0, k = 1, remaining = pc;
    while (remaining > 0) {
      std::memcpy(R, Q, sizeof(uint64_t) * W);
      for (int w = 0; w < W; ++w) {
        while (R[w]) {
          int b = __builtin_ctzll(R[w]);
          int v = w * 64 + b;
          Q[w] &= ~(1ull << b);
          R[w] &= ~(1ull << b);
          remaining--;
          const uint64_t* nv = A->row(v);
          for (int x = w; x < W; ++x) R[x] &= ~nv[x];
          if (k >= kmin) {
            ord[2 * cnt] = v;
            ord[2 * cnt + 1] = k;
            cnt++;
          }
        }
      }
      k++;
    }
    uint64_t* newP = S.bits[depth + 1].data();
    for (int i = cnt - 1; i >= 0; --i) {
      int v = ord[2 * i];
      int col = ord[2 * i + 1];
      if ((int)C.size() + col < best.load(std::memory_order_relaxed) + strict) return;
      const uint64_t* nv = A->row(v);
      bool any = false;
      for (int w = 0; w < W; ++w) {
        newP[w] = P[w] & nv[w];
        any |= (newP[w] != 0);
      }
      C.push_back(v);
      if (!any) {
        if ((int)C.size() >= best.load(std::memory_order_relaxed)) {
#pragma omp critical(orc_clique_update)
          {
            if ((int)C.size() > best.load()) {
              best_clique = C;
              best.store((int)C.size());
            } else if ((int)C.size() == best.load()) {
              std::vector<int> a(C.size()), b(best_clique.size());
              for (size_t q = 0; q < C.size(); ++q) a[q] = orig[C[q]];
              for (size_t q = 0; q < best_clique.size(); ++q) b[q] = orig[best_clique[q]];
              std::sort(a.begin(), a.end());
              std::sort(b.begin(), b.end());
              if (b.size() != a.size() || a < b) best_clique = C;
            }
          }
        }
      } else {
        expand(C, S, depth + 1);
      }
      C.pop_back();
      P[v >> 6] &= ~(1ull << (v & 63));
      if (timed_out.load(std::memory_order_relaxed)) return;
    }
  }
};

// Greedy heuristic in the spirit of pmc::pmc_heu (graph.cc:88-91): vertices are visited in
// decreasing core order; from each start vertex whose core number can still beat the incumbent,
// a clique is grown by repeatedly taking the candidate with the largest core number (ties: larger
// degree, then smaller index) and intersecting the candidate set with its neighbourhood.
int heuristic_clique(const std::vector<i64>& off, const std::vector<int>& edges, int n,
                     const std::vector<int>& core, const std::vector<int>& order, std::vector<int>& C,
                     int num_threads) {
  std::vector<int> best_c;
  std::atomic<int> best(0);
  const int ub = n ? (*std::max_element(core.begin(), core.end()) + 1) : 0;
#pragma omp parallel num_threads(num_threads)
  {
    std::vector<int> P, P2, cur;
    std::vector<char> mark(n, 0);
#pragma omp for schedule(dynamic, 16)
    for (int oi = n - 1; oi >= 0; --oi) {
      int v = order[oi];
      int b = best.load(std::memory_order_relaxed);
      if (b >= ub) continue;
      if (core[v] + 1 <= b) continue;
      P.clear();
      for (i64 e = off[v]; e < off[v + 1]; ++e) {
        int u = edges[e];
        if (core[u] + 1 > b) P.push_back(u);
      }
      if ((int)P.size() + 1 <= b) continue;
      cur.clear();
      cur.push_back(v);
      while (!P.empty()) {
        if ((int)(cur.size() + P.size()) <= b) break;
        // pick best candidate
        int bi = 0;
        for (int i = 1; i < (int)P.size(); ++i) {
          int a = P[i], c = P[bi];
          if (core[a] > core[c] || (core[a] == core[c] && ((off[a + 1] - off[a]) > (off[c + 1] - off[c]) ||
                                                            ((off[a + 1] - off[a]) == (off[c + 1] - off[c]) && a < c))))
            bi = i;
        }
        int u = P[bi];
        cur.push_back(u);
        for (i64 e = off[u]; e < off[u + 1]; ++e) mark[edges[e]] = 1;
        P2.clear();
        for (int w : P)
          if (w != u && mark[w]) P2.push_back(w);
        for (i64 e = off[u]; e < off[u + 1]; ++e) mark[edges[e]] = 0;
        P.swap(P2);
      }
      if (P.empty() && (int)cur.size() > b) {
#pragma omp critical(orc_heu_update)
        {
          if ((int)cur.size() > best.load()) {
            best_c = cur;
            best.store((int)cur.size());
          }
        }
      }
    }
  }
  C = best_c;
  return best.load();
}

struct CliqueInfo {
  int max_core = 0;
  int lb = 0;
  int ub = 0;
  int exact_ran = 0;
  int timed_out = 0;
  i64 nodes = 0;
  int lp_closed = 0;  // 1: size proven through the vertex-cover LP bound / Nemhauser-Trotter reduction (not canonical)
};

// findMaxClique  (teaser/src/graph.cc:12-125)
std::vector<int> find_max_clique(const std::vector<std::vector<int>>& adj, int mode, double kcore_thr,
                                 double time_limit_s, int num_threads, CliqueInfo* info) {
  const int n = (int)adj.size();
  // CSR flatten  (graph.cc:20-29)
  std::vector<int> edges;
  std::vector<i64> vertices;
  vertices.push_back(0);
  for (int i = 0; i < n; ++i) {
    edges.insert(edges.end(), adj[i].begin(), adj[i].end());
    vertices.push_back((i64)edges.size());
  }
  if (num_threads <= 0) num_threads = max_threads();
  std::vector<int> C;
  std::vector<int> core, order;
  kcores(vertices, edges, n, core, order);  // graph.cc:58
  int max_core = 0;
  for (int v = 0; v < n; ++v) max_core = std::max(max_core, core[v]);  // :59
  if (info) info->max_core = max_core;

  // k-core heuristic shortcut  (graph.cc:66-81)
  if (mode == MODE_KCORE_HEU && kcore_thr != 1 && max_core > (int)(kcore_thr * (double)n)) {
    for (int v = 0; v < n; ++v)
      if (core[v] >= max_core) C.push_back(v);
    return C;
  }
  int ub = max_core + 1;  // :83-85
  int lb = 0;
  if (!edges.empty()) lb = heuristic_clique(vertices, edges, n, core, order, C, num_threads);  // :88-91
  if (info) {
    info->lb = lb;
    info->ub = ub;
  }
  if (lb == 0) return C;   // :93-98  (graph without edges: PMC's heuristic reports 0)
  // graph.cc:100-102 returns the heuristic clique when lb == ub, and :105 skips the exact search unless
  // PMC_EXACT.  In PMC_EXACT mode this restatement ALWAYS runs the enumeration below so that ties between
  // maximum cliques are resolved canonically (lexicographically smallest sorted index set); with a unique
  // maximum clique the result equals the reference's in both branches.
  if (mode != MODE_PMC_EXACT) return C;  // PMC_HEU, or KCORE_HEU below threshold

  // ---- exact search (graph.cc:105-122; pmc::pmcx_maxclique) ----
  if (info) info->exact_ran = 1;
  // k-core pruning: a vertex of a clique of size >= lb has core number >= lb-1
  std::vector<int> keep;
  for (int i = 0; i < n; ++i) {
    int v = order[i];  // ascending core/degeneracy order
    if (core[v] >= lb - 1) keep.push_back(v);
  }
  if (keep.empty()) return C;
  const double t_end_ms = now_ms() + time_limit_s * 1000.0;
  i64 total_nodes = 0;
  bool timed_out = false;
  int best = lb;
  // One search over the vertex list `keep` (compact labels = positions in keep); returns true when it ran to the end.
  auto run_search = [&](const std::vector<int>& kp, double pass_seconds, int strict = 0, int stop_at = 0x7fffffff) -> bool {
    const int nk = (int)kp.size();
    std::vector<int> label(n, -1);
    for (int i = 0; i < nk; ++i) label[kp[i]] = i;
    Bits A;
    A.init(nk, nk);
    for (int i = 0; i < nk; ++i) {
      int v = kp[i];
      uint64_t* r = A.row(i);
      for (i64 e = vertices[v]; e < vertices[v + 1]; ++e) {
        int l = label[edges[e]];
        if (l >= 0) r[l >> 6] |= 1ull << (l & 63);
      }
    }
    CliqueSearch S;
    S.A = &A;
    S.n = nk;
    S.W = A.W;
    S.best.store(best);
    S.orig = kp.data();
    bool inc_ok = true;
    for (int v : C) inc_ok &= label[v] >= 0;
    if (inc_ok)
      for (int v : C) S.best_clique.push_back(label[v]);  // incumbent = first candidate of the tie-break
    S.timed_out.store(false);
    S.nodes.store(0);
    S.deadline_ms = t_end_ms;
    S.pass_deadline_ms = pass_seconds >= 0 ? now_ms() + pass_seconds * 1000.0 : -1;
    S.strict = strict;
    S.stop_at = stop_at;
    const int W = A.W;
    // roots in reverse degeneracy order; root i only sees later vertices (labels > i)
#pragma omp parallel num_threads(num_threads)
    {
      CliqueScratch scratch;
      scratch.init(ub + 3, W);
      std::vector<int> Cc;
#pragma omp for schedule(dynamic, 1)
      for (int ri = 0; ri < nk; ++ri) {
        int i = nk - 1 - ri;
        if (S.timed_out.load() || S.budget_out.load() || S.best.load() >= S.stop_at) continue;
        // P = N(i) ∩ {j > i}
        uint64_t* P = scratch.bits[0].data();
        const uint64_t* r = A.row(i);
        int pc = 0;
        for (int w = 0; w < W; ++w) {
          uint64_t m = r[w];
          int lo = w * 64;
          if (lo + 63 <= i) m = 0;
          else if (lo <= i) m &= ~((2ull << (i - lo)) - 1ull);
          P[w] = m;
          pc += __builtin_popcountll(m);
        }
        if (pc + 1 < S.best.load() + S.strict) continue;
        Cc.clear();
        Cc.push_back(i);
        S.expand(Cc, scratch, 0);
      }
    }
    if ((int)S.best_clique.size() >= best && !S.best_clique.empty()) {
      std::vector<int> Cn;
      for (int l : S.best_clique) Cn.push_back(kp[l]);
      C = Cn;
      best = (int)C.size();
    }
    total_nodes += S.nodes.load();
    timed_out = S.timed_out.load();
    return !S.timed_out.load() && !S.budget_out.load();
  };

  // Pass 1 with a short wall-clock budget: every instance whose canonical enumeration is feasible finishes here
  // (the device path uses 50 ms of GPU time for the same purpose).
  const double kFirstPassSeconds = 3.0;
  bool done = run_search(keep, std::min(kFirstPassSeconds, time_limit_s));
  if (!done && !timed_out && 2 * best >= (int)keep.size()) {
    // Dense graph (the device path does the same in clique_lp_kernel, max_clique.cu K4): max clique of G[A] =
    // |A| - min vertex cover of the complement H[A]; LP relaxation = half the maximum matching of H's bipartite double
    // cover; Nemhauser-Trotter: some maximum clique avoids the vertices with LP value 1.
    const int nk = (int)keep.size();
    std::vector<int> label(n, -1);
    for (int i = 0; i < nk; ++i) label[keep[i]] = i;
    std::vector<std::vector<int>> H(nk);
    {
      std::vector<char> nb(nk);
      for (int i = 0; i < nk; ++i) {
        std::fill(nb.begin(), nb.end(), 0);
        for (i64 e = vertices[keep[i]]; e < vertices[keep[i] + 1]; ++e)
          if (label[edges[e]] >= 0) nb[label[edges[e]]] = 1;
        for (int j = 0; j < nk; ++j)
          if (j != i && !nb[j]) H[i].push_back(j);
      }
    }
    std::vector<int> mateL(nk, -1), mateR(nk, -1), parent(nk, -1), queue;
    std::vector<char> vis(nk, 0);
    int matching = 0;
    for (int u = 0; u < nk; ++u)
      for (int v : H[u])
        if (mateR[v] < 0) {
          mateL[u] = v;
          mateR[v] = u;
          ++matching;
          break;
        }
    auto bfs = [&](bool augment, std::vector<char>* lz) -> int {
      size_t head = 0;
      while (head < queue.size()) {
        const int x = queue[head++];
        for (int v : H[x]) {
          if (vis[v]) continue;
          vis[v] = 1;
          parent[v] = x;
          if (mateR[v] < 0) {
            if (augment) return v;
          } else {
            queue.push_back(mateR[v]);
            if (lz) (*lz)[mateR[v]] = 1;
          }
        }
      }
      return -1;
    };
    for (int u = 0; u < nk; ++u) {
      if (mateL[u] >= 0) continue;
      std::fill(vis.begin(), vis.end(), 0);
      queue.assign(1, u);
      int v = bfs(true, nullptr);
      if (v >= 0) {
        while (v >= 0) {
          const int x = parent[v], nv = mateL[x];
          mateL[x] = v;
          mateR[v] = x;
          v = nv;
        }
        ++matching;
      }
    }
    if (info) info->lp_closed = 1;
    if (nk - (matching + 1) / 2 <= best) {
      done = true;  // the incumbent is a maximum clique
    } else {
      std::vector<char> lz(nk, 0);
      std::fill(vis.begin(), vis.end(), 0);
      queue.clear();
      for (int u = 0; u < nk; ++u)
        if (mateL[u] < 0) {
          queue.push_back(u);
          lz[u] = 1;
        }
      bfs(false, &lz);
      std::vector<int> keep2;
      for (int i = 0; i < nk; ++i)
        if (!(!lz[i] && vis[i])) keep2.push_back(keep[i]);  // drop LP value 1
      // ties no longer matter (and are astronomically many on dense graphs); reaching the LP bound ends the search
      done = run_search(keep2, -1, 1, nk - (matching + 1) / 2);
    }
  } else if (!done && !timed_out) {
    done = run_search(keep, -1);
  }
  if (info) {
    info->timed_out = timed_out ? 1 : 0;
    info->nodes = total_nodes;
  }
  return C;
}

}  // namespace

// =============================================================================
// C API (ctypes-friendly).  Layout of orc_params / orc_solution is identical to
// tzr_params / tzr_solution in include/teaser_b200.h so tests can share structures.
// =============================================================================
extern "C" {

struct orc_params {
  double noise_bound;
  double cbar2;
  int32_t estimate_scaling;
  int32_t rotation_estimation_algorithm;  // 0 GNC_TLS, 1 FGR, 2 QUATRO
  double rotation_gnc_factor;
  uint64_t rotation_max_iterations;
  double rotation_cost_threshold;
  int32_t rotation_tim_graph;     // 0 CHAIN, 1 COMPLETE
  int32_t inlier_selection_mode;  // 0 PMC_EXACT, 1 PMC_HEU, 2 KCORE_HEU, 3 NONE
  double kcore_heuristic_threshold;
  int32_t use_max_clique;
  int32_t max_clique_exact_solution;
  double max_clique_time_limit;
  int32_t max_clique_num_threads;
  int32_t reserved;
};

struct orc_solution {
  int32_t valid;
  int32_t clique_size;
  double scale;
  double translation[3];
  double rotation[9];  // column-major
  int32_t clique_proven_optimal;
  int32_t gnc_iterations;
  double gnc_cost;
  int32_t n_rotation_inliers;
  int32_t n_translation_inliers;
  int64_t n_edges;
  double stage_ms[8];  // 0 tims, 1 scale, 2 graph, 3 clique, 4 rotation, 5 translation, 6 total
};

int orc_num_threads() { return max_threads(); }

// bench.py sets the OpenMP thread count explicitly (torchrun exports OMP_NUM_THREADS=1 to its children)
void orc_set_num_threads(int t) {
#ifdef _OPENMP
  if (t > 0) omp_set_num_threads(t);
#else
  (void)t;
#endif
}

void orc_compute_tims(const double* v, int64_t n, double* tims, int32_t* map) { compute_tims(v, n, tims, map); }

void orc_scale_inliers_selector(const double* src_tims, const double* dst_tims, int64_t K, double noise_bound,
                                double cbar2, double* scale, uint8_t* mask) {
  scale_inliers_selector(src_tims, dst_tims, K, noise_bound, cbar2, scale, mask);
}

void orc_tls_scale_solver(const double* src_tims, const double* dst_tims, int64_t K, double noise_bound,
                          double cbar2, double* scale, uint8_t* mask) {
  tls_scale_solver(src_tims, dst_tims, K, noise_bound, cbar2, scale, mask);
}

void orc_scalar_tls(const double* X, const double* ranges, int64_t M, double* est, uint8_t* inliers) {
  scalar_tls(X, ranges, M, est, inliers);
}

void orc_tls_translation(const double* src, const double* dst, int64_t m, double noise_bound, double cbar2,
                         double* t, uint8_t* inliers) {
  tls_translation(src, dst, m, noise_bound, cbar2, t, inliers);
}

void orc_svd_rot(const double* X, const double* Y, const double* W, int64_t m, double* R) {
  M3 r = svd_rot(X, Y, W, m);
  std::memcpy(R, r.a, sizeof(r.a));
}

void orc_svd3(const double* H, double* U, double* S, double* V) {
  M3 h, u, v;
  std::memcpy(h.a, H, sizeof(h.a));
  svd3(h, u, S, v);
  std::memcpy(U, u.a, sizeof(u.a));
  std::memcpy(V, v.a, sizeof(v.a));
}

// returns iterations executed
int orc_gnc_tls_rotation(const double* src, const double* dst, int64_t m, uint64_t max_iterations,
                         double cost_threshold, double gnc_factor, double noise_bound, double* R, uint8_t* inliers,
                         double* cost, double* trace, int trace_cap, double* weights_out) {
  GncResult r = gnc_tls(src, dst, m, max_iterations, cost_threshold, gnc_factor, noise_bound, inliers, trace,
                        trace_cap, weights_out);
  std::memcpy(R, r.R.a, sizeof(r.R.a));
  if (cost) *cost = r.cost;
  return r.iterations;
}

int orc_fgr_rotation(const double* src, const double* dst, int64_t m, uint64_t max_iterations, double cost_threshold,
                     double gnc_factor, double noise_bound, double* R, uint8_t* inliers, double* cost) {
  GncResult r = fgr(src, dst, m, max_iterations, cost_threshold, gnc_factor, noise_bound, inliers);
  std::memcpy(R, r.R.a, sizeof(r.R.a));
  if (cost) *cost = r.cost;
  return r.iterations;
}

int orc_quatro_rotation(const double* src, const double* dst, int64_t m, uint64_t max_iterations,
                        double cost_threshold, double gnc_factor, double noise_bound, double* R, uint8_t* inliers,
                        double* cost) {
  GncResult r = quatro(src, dst, m, max_iterations, cost_threshold, gnc_factor, noise_bound, inliers);
  std::memcpy(R, r.R.a, sizeof(r.R.a));
  if (cost) *cost = r.cost;
  return r.iterations;
}

// Max clique from CSR adjacency (offsets: n+1 entries).  info[0]=max_core, [1]=lb, [2]=ub, [3]=exact_ran,
// [4]=timed_out, [5]=nodes (clamped to int).  Returns clique size; clique written unsorted (as findMaxClique).
int orc_max_clique_csr(const int64_t* offsets, const int32_t* edges, int n, int mode, double kcore_thr,
                       double time_limit, int num_threads, int32_t* clique_out, int32_t* info) {
  std::vector<std::vector<int>> adj(n);
  for (int v = 0; v < n; ++v) adj[v].assign(edges + offsets[v], edges + offsets[v + 1]);
  CliqueInfo ci;
  std::vector<int> C = find_max_clique(adj, mode, kcore_thr, time_limit, num_threads, &ci);
  for (size_t i = 0; i < C.size(); ++i) clique_out[i] = C[i];
  if (info) {
    info[0] = ci.max_core; info[1] = ci.lb; info[2] = ci.ub; info[3] = ci.exact_ran; info[4] = ci.timed_out;
    info[5] = (int)std::min<i64>(ci.nodes, 2147483647LL);
  }
  return (int)C.size();
}

// Max clique from a packed adjacency bitset (n rows x words_per_row uint64), as produced by the
// product's graph-build stage.  Convenience for cross-checking stages in tests.
int orc_max_clique_bits(const uint64_t* bits, int n, int words_per_row, int mode, double kcore_thr,
                        double time_limit, int num_threads, int32_t* clique_out, int32_t* info) {
  std::vector<std::vector<int>> adj(n);
  for (int v = 0; v < n; ++v) {
    const uint64_t* r = bits + (size_t)v * words_per_row;
    for (int w = 0; w < words_per_row; ++w) {
      uint64_t m = r[w];
      while (m) {
        int b = __builtin_ctzll(m);
        m &= m - 1;
        int u = w * 64 + b;
        if (u < n) adj[v].push_back(u);
      }
    }
  }
  CliqueInfo ci;
  std::vector<int> C = find_max_clique(adj, mode, kcore_thr, time_limit, num_threads, &ci);
  for (size_t i = 0; i < C.size(); ++i) clique_out[i] = C[i];
  if (info) {
    info[0] = ci.max_core; info[1] = ci.lb; info[2] = ci.ub; info[3] = ci.exact_ran; info[4] = ci.timed_out;
    info[5] = (int)std::min<i64>(ci.nodes, 2147483647LL);
  }
  return (int)C.size();
}

// Build the inlier graph exactly as solve() does (registration.cc:599-619) for the FIXED-scale
// selector and return it as a packed bitset + degree vector (for bit-exact comparison with the
// product's graph-build kernel).  bits: n x words_per_row, zero-initialised by the caller.
int64_t orc_build_graph_bits(const double* src, const double* dst, int n, double noise_bound, double cbar2,
                             uint64_t* bits, int words_per_row, int32_t* degree) {
  const i64 N = n, K = N * (N - 1) / 2;
  std::vector<double> st(3 * (size_t)K), dt(3 * (size_t)K);
  std::vector<int> map(2 * (size_t)K);
  compute_tims(src, N, st.data(), map.data());
  compute_tims(dst, N, dt.data(), nullptr);
  std::vector<uint8_t> mask(K);
  double scale;
  scale_inliers_selector(st.data(), dt.data(), K, noise_bound, cbar2, &scale, mask.data());
  i64 e = 0;
  if (degree)
    for (int i = 0; i < n; ++i) degree[i] = 0;
  for (i64 k = 0; k < K; ++k)
    if (mask[k]) {
      int a = map[2 * k], b = map[2 * k + 1];
      bits[(size_t)a * words_per_row + (b >> 6)] |= 1ull << (b & 63);
      bits[(size_t)b * words_per_row + (a >> 6)] |= 1ull << (a & 63);
      if (degree) {
        degree[a]++;
        degree[b]++;
      }
      e++;
    }
  return e;
}

// -----------------------------------------------------------------------------
// RobustRegistrationSolver::solve(src, dst)   (teaser/src/registration.cc:568-737)
// Honours Params (SURVEY Q1 decision).  A fresh "solver" per call (SURVEY Q2).
// Outputs (all optional except sol): clique (sorted, capacity n), rotation inlier mask (capacity =
// number of rotation TIMs), translation inlier mask (capacity = clique size), adjacency bitset.
// -----------------------------------------------------------------------------
int orc_solve(const orc_params* p, const double* src, const double* dst, int n, orc_solution* sol,
              int32_t* clique_out, uint8_t* rot_inliers_out, uint8_t* trans_inliers_out, uint64_t* adj_bits_out,
              int words_per_row) {
  std::memset(sol, 0, sizeof(*sol));
  sol->valid = 1;
  const double t_start = now_ms();
  const i64 N = n, K = N * (N - 1) / 2;
  int inlier_selection_mode = p->inlier_selection_mode;
  if (!p->use_max_clique) inlier_selection_mode = 3;             // :574-578
  if (!p->max_clique_exact_solution) inlier_selection_mode = 1;  // :579-583

  // TIMs  (:599-600)
  double t0 = now_ms();
  std::vector<double> src_tims(3 * (size_t)K), dst_tims(3 * (size_t)K);
  std::vector<int> src_map(2 * (size_t)K), dst_map(2 * (size_t)K);
  compute_tims(src, N, src_tims.data(), src_map.data());
  compute_tims(dst, N, dst_tims.data(), dst_map.data());
  sol->stage_ms[0] = now_ms() - t0;

  // scale  (:603)
  t0 = now_ms();
  std::vector<uint8_t> scale_mask(K);
  double scale = 1;
  if (p->estimate_scaling)
    tls_scale_solver(src_tims.data(), dst_tims.data(), K, p->noise_bound, p->cbar2, &scale, scale_mask.data());
  else
    scale_inliers_selector(src_tims.data(), dst_tims.data(), K, p->noise_bound, p->cbar2, &scale, scale_mask.data());
  sol->scale = scale;
  sol->stage_ms[1] = now_ms() - t0;

  std::vector<int> max_clique;
  if (inlier_selection_mode != 3) {
    // inlier graph  (:614-619)
    t0 = now_ms();
    Graph g;
    g.populateVertices(n);
    for (i64 k = 0; k < K; ++k)
      if (scale_mask[k]) g.addEdge(src_map[2 * k], src_map[2 * k + 1]);
    sol->n_edges = (int64_t)g.num_edges;
    sol->stage_ms[2] = now_ms() - t0;
    if (adj_bits_out) {
      for (int a = 0; a < n; ++a)
        for (int b : g.adj[a]) adj_bits_out[(size_t)a * words_per_row + (b >> 6)] |= 1ull << (b & 63);
    }
    // max clique  (:621-636)
    t0 = now_ms();
    int mode = inlier_selection_mode == 0 ? MODE_PMC_EXACT : (inlier_selection_mode == 1 ? MODE_PMC_HEU : MODE_KCORE_HEU);
    CliqueInfo ci;
    max_clique = find_max_clique(g.adj, mode, p->kcore_heuristic_threshold, p->max_clique_time_limit,
                                 p->max_clique_num_threads, &ci);
    std::sort(max_clique.begin(), max_clique.end());
    sol->stage_ms[3] = now_ms() - t0;
    sol->clique_proven_optimal = (mode == MODE_PMC_EXACT && !ci.timed_out) ? (ci.lp_closed ? 2 : 1) : 0;
    if (max_clique.size() <= 1) {  // :643-647
      sol->valid = 0;
      sol->clique_size = (int)max_clique.size();
      if (clique_out)
        for (size_t i = 0; i < max_clique.size(); ++i) clique_out[i] = max_clique[i];
      sol->stage_ms[6] = now_ms() - t_start;
      return 0;
    }
  } else {
    for (int i = 0; i < n; ++i) max_clique.push_back(i);  // :650-653
  }
  const i64 m = (i64)max_clique.size();
  sol->clique_size = (int)m;
  if (clique_out)
    for (i64 i = 0; i < m; ++i) clique_out[i] = max_clique[i];
  if (scale != scale) {  // no TIM was finite (every source point identical): nothing to register (DESIGN.md §3.3)
    sol->valid = 0;
    sol->stage_ms[6] = now_ms() - t_start;
    return 0;
  }

  // pruned TIMs  (:657-694)
  t0 = now_ms();
  std::vector<double> pruned_src, pruned_dst;
  i64 n_rot = 0;
  if (p->rotation_tim_graph == 0) {
    n_rot = m;
    pruned_src.resize(3 * m);
    pruned_dst.resize(3 * m);
    for (i64 i = 0; i < m; ++i) {
      int root = max_clique[i];
      int leaf = (i != m - 1) ? max_clique[i + 1] : max_clique[0];
      for (int r = 0; r < 3; ++r) {
        pruned_src[3 * i + r] = src[3 * (i64)leaf + r] - src[3 * (i64)root + r];
        pruned_dst[3 * i + r] = dst[3 * (i64)leaf + r] - dst[3 * (i64)root + r];
      }
    }
  } else {
    std::vector<double> si(3 * m), di(3 * m);
    for (i64 i = 0; i < m; ++i)
      for (int r = 0; r < 3; ++r) {
        si[3 * i + r] = src[3 * (i64)max_clique[i] + r];
        di[3 * i + r] = dst[3 * (i64)max_clique[i] + r];
      }
    n_rot = m * (m - 1) / 2;
    pruned_src.resize(3 * (size_t)n_rot);
    pruned_dst.resize(3 * (size_t)n_rot);
    compute_tims(di.data(), m, pruned_dst.data(), nullptr);
    compute_tims(si.data(), m, pruned_src.data(), nullptr);
  }
  // remove scaling (:697); rotation noise bound (:702-704)
  const double inv_scale = 1 / scale;
  for (size_t i = 0; i < pruned_dst.size(); ++i) pruned_dst[i] *= inv_scale;
  const double rot_noise_bound = p->noise_bound * (2 / scale);

  // rotation (:708)
  std::vector<uint8_t> rot_mask(n_rot);
  GncResult gr;
  if (p->rotation_estimation_algorithm == 1)
    gr = fgr(pruned_src.data(), pruned_dst.data(), n_rot, p->rotation_max_iterations, p->rotation_cost_threshold,
             p->rotation_gnc_factor, rot_noise_bound, rot_mask.data());
  else if (p->rotation_estimation_algorithm == 2)
    gr = quatro(pruned_src.data(), pruned_dst.data(), n_rot, p->rotation_max_iterations, p->rotation_cost_threshold,
                p->rotation_gnc_factor, rot_noise_bound, rot_mask.data());
  else
    gr = gnc_tls(pruned_src.data(), pruned_dst.data(), n_rot, p->rotation_max_iterations,
                 p->rotation_cost_threshold, p->rotation_gnc_factor, rot_noise_bound, rot_mask.data(), nullptr, 0,
                 nullptr);
  std::memcpy(sol->rotation, gr.R.a, sizeof(gr.R.a));
  sol->gnc_cost = gr.cost;
  sol->gnc_iterations = gr.iterations;
  int nri = 0;
  for (i64 i = 0; i < n_rot; ++i) nri += rot_mask[i];
  sol->n_rotation_inliers = nri;
  if (rot_inliers_out) std::memcpy(rot_inliers_out, rot_mask.data(), (size_t)n_rot);
  sol->stage_ms[4] = now_ms() - t0;

  // translation (:717-731)
  t0 = now_ms();
  std::vector<double> rs(3 * m), rd(3 * m);
  const M3& R = gr.R;
  for (i64 i = 0; i < m; ++i) {
    const double* s = src + 3 * (i64)max_clique[i];
    // (scale * R) * src : the 3x3 is scaled first (Eigen evaluates scalar*matrix, then the product)
    double x = s[0], y = s[1], z = s[2];
    rs[3 * i + 0] = (scale * R(0, 0)) * x + (scale * R(0, 1)) * y + (scale * R(0, 2)) * z;
    rs[3 * i + 1] = (scale * R(1, 0)) * x + (scale * R(1, 1)) * y + (scale * R(1, 2)) * z;
    rs[3 * i + 2] = (scale * R(2, 0)) * x + (scale * R(2, 1)) * y + (scale * R(2, 2)) * z;
    for (int r = 0; r < 3; ++r) rd[3 * i + r] = dst[3 * (i64)max_clique[i] + r];
  }
  std::vector<uint8_t> tmask(m);
  tls_translation(rs.data(), rd.data(), m, p->noise_bound, p->cbar2, sol->translation, tmask.data());
  int nti = 0;
  for (i64 i = 0; i < m; ++i) nti += tmask[i];
  sol->n_translation_inliers = nti;
  if (trans_inliers_out) std::memcpy(trans_inliers_out, tmask.data(), (size_t)m);
  sol->stage_ms[5] = now_ms() - t0;
  sol->valid = 1;
  sol->stage_ms[6] = now_ms() - t_start;
  return 0;
}

}  // extern "C"
