// 3x3 helpers shared by the rotation stage (rot_trans.cu) and ICP (icp.cu): column-major matrices, the two-sided
// Jacobi SVD and the Procrustes rotation with the reflection fix.  Internal linkage in every TU that includes it.
#pragma once

#include "tzr_internal.cuh"

namespace tzr {

namespace {

// ---- 3x3 helpers (column-major like Eigen::Matrix3d) -------------------------------------------
struct M3 {
  double a[9];
  __device__ double& operator()(int r, int c) { return a[c * 3 + r]; }
  __device__ double operator()(int r, int c) const { return a[c * 3 + r]; }
};

__device__ inline void m3_identity(M3& m) {
#pragma unroll
  for (int i = 0; i < 9; ++i) m.a[i] = 0.0;
  m.a[0] = m.a[4] = m.a[8] = 1.0;
}

__device__ inline double m3_det(const M3& m) {
  return m(0, 0) * (m(1, 1) * m(2, 2) - m(1, 2) * m(2, 1)) - m(0, 1) * (m(1, 0) * m(2, 2) - m(1, 2) * m(2, 0)) +
         m(0, 2) * (m(1, 0) * m(2, 1) - m(1, 1) * m(2, 0));
}

// rows p,q <- [c s; -s c] * rows
__device__ inline void rot_rows(M3& A, int p, int q, double c, double s) {
#pragma unroll
  for (int col = 0; col < 3; ++col) {
    const double xp = A(p, col), xq = A(q, col);
    A(p, col) = c * xp + s * xq;
    A(q, col) = c * xq - s * xp;
  }
}
// cols p,q <- cols * [c s; -s c]
__device__ inline void rot_cols(M3& A, int p, int q, double c, double s) {
#pragma unroll
  for (int row = 0; row < 3; ++row) {
    const double xp = A(row, p), xq = A(row, q);
    A(row, p) = c * xp - s * xq;
    A(row, q) = s * xp + c * xq;
  }
}

// Two-sided Jacobi (Kogbetliantz) SVD, H = U diag(S) V^T, singular values sorted descending,
// U and V full orthogonal — the role Eigen::JacobiSVD<Matrix3d>(ComputeFullU|ComputeFullV) plays in
// utils::svdRot (utils.h:126).
__device__ void svd3(const M3& H, M3& U, double S[3], M3& V) {
  M3 A = H;
  m3_identity(U);
  m3_identity(V);
  const double eps = 2.220446049250313e-16, tiny = 2.2250738585072014e-308;
  double max_diag = fmax(fabs(A(0, 0)), fmax(fabs(A(1, 1)), fabs(A(2, 2))));
  for (int sweep = 0; sweep < 64; ++sweep) {
    bool finished = true;
    for (int p = 1; p < 3; ++p) {
      for (int q = 0; q < p; ++q) {
        const double thr = fmax(tiny, 2.0 * eps * max_diag);
        if (fabs(A(p, q)) > thr || fabs(A(q, p)) > thr) {
          finished = false;
          const double m00 = A(p, p), m01 = A(p, q), m10 = A(q, p), m11 = A(q, q);
          // step 1: rotation that symmetrises the 2x2 block
          double c1, s1;
          const double t = m00 + m11, d = m10 - m01;
          if (fabs(d) < tiny) {
            c1 = 1.0;
            s1 = 0.0;
          } else {
            const double u = t / d;
            const double h = sqrt(1.0 + u * u);
            s1 = 1.0 / h;
            c1 = u / h;
          }
          const double n00 = c1 * m00 + s1 * m10;
          const double n01 = c1 * m01 + s1 * m11;
          const double n11 = c1 * m11 - s1 * m01;
          // step 2: symmetric Jacobi rotation  t^2 - 2*tau*t - 1 = 0, smaller root
          double c2, s2;
          if (2.0 * fabs(n01) < tiny) {
            c2 = 1.0;
            s2 = 0.0;
          } else {
            const double tau = (n00 - n11) / (2.0 * n01);
            const double w = sqrt(tau * tau + 1.0);
            const double tt = (tau >= 0.0) ? -1.0 / (tau + w) : 1.0 / (w - tau);
            c2 = 1.0 / sqrt(tt * tt + 1.0);
            s2 = tt * c2;
          }
          // left rotation L = J2^T * G1
          const double cl = c2 * c1 + s2 * s1;
          const double sl = c2 * s1 - s2 * c1;
          rot_rows(A, p, q, cl, sl);
          rot_cols(U, p, q, cl, -sl);  // U <- U * L^T
          rot_cols(A, p, q, c2, s2);
          rot_cols(V, p, q, c2, s2);
          max_diag = fmax(max_diag, fmax(fabs(A(p, p)), fabs(A(q, q))));
        }
      }
    }
    if (finished) break;
  }
  for (int i = 0; i < 3; ++i) {
    const double a = A(i, i);
    S[i] = fabs(a);
    if (a < 0.0)
      for (int r = 0; r < 3; ++r) U(r, i) = -U(r, i);
  }
  for (int i = 0; i < 3; ++i) {
    int pos = i;
    for (int k = i + 1; k < 3; ++k)
      if (S[k] > S[pos]) pos = k;
    if (pos != i) {
      double ts = S[i];
      S[i] = S[pos];
      S[pos] = ts;
      for (int r = 0; r < 3; ++r) {
        double tu = U(r, i);
        U(r, i) = U(r, pos);
        U(r, pos) = tu;
        double tv = V(r, i);
        V(r, i) = V(r, pos);
        V(r, pos) = tv;
      }
    }
  }
}

// R maximising tr(R H) does not change when H is scaled by a positive number.  If H's largest |entry| lies outside
// [2^-400, 2^400], scale the n entries by the power of two that brings it into [1/2, 1): exact, and it keeps the Jacobi
// threshold (tiny / eps*max_diag) and the squares of the planar closed form clear of underflow and overflow.  Entries
// already in that range keep their bits, so ordinary inputs are untouched.
__device__ inline void normalise_scale(double* a, int n) {
  double mx = 0.0;
  for (int i = 0; i < n; ++i) mx = fmax(mx, fabs(a[i]));
  if (mx > 0.0 && mx <= 1.7976931348623157e308 && (mx < 0x1p-400 || mx > 0x1p400)) {
    int e;
    frexp(mx, &e);
    for (int i = 0; i < n; ++i) a[i] = ldexp(a[i], -e);
  }
}

// R = V * U^T with the reflection fix (utils.h:130-135)
__device__ void rotation_from_H(const M3& H0, M3& R) {
  M3 H = H0, U, V;
  double S[3];
  normalise_scale(H.a, 9);
  svd3(H, U, S, V);
  if (m3_det(U) * m3_det(V) < 0.0) {
    for (int r = 0; r < 3; ++r) V(r, 2) = -V(r, 2);
  }
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R(r, c) = V(r, 0) * U(c, 0) + V(r, 1) * U(c, 1) + V(r, 2) * U(c, 2);
}

}  // namespace

}  // namespace tzr
