// Stages 3 and 4 of solve(): GNC-TLS rotation and per-axis TLS translation; one CTA per problem,
// all iterations on chip.
//
// Replaces (reference):
//   chain-TIM rebuild + de-scaling                       teaser/src/registration.cc:657-704
//   GNCTLSRotationSolver::solveForRotation               teaser/src/registration.cc:764-866
//   utils::svdRot (weighted 3x3 covariance + SVD)        teaser/include/teaser/utils.h:121-136
//   TLSTranslationSolver::solveForTranslation            teaser/src/registration.cc:445-471
//   ScalarTLSEstimator::estimate                         teaser/src/registration.cc:21-88
//
// Not a dense contraction (m = clique size, 3x3 outputs): warp-shuffle reductions + a 3x3 Jacobi
// SVD in registers; no tensor cores.  All arithmetic is FP64 (tolerance vs the oracle: 1e-4 rad /
// 1e-4 m; observed ~1e-12).  The TU is compiled with -fmad=false so that the scalar sweeps round
// like the reference's non-contracted x86-64 build.
#include "tzr_internal.cuh"
#include "tls_device.cuh"

namespace tzr {

namespace {

constexpr int kRTThreads = 128;  // 128 regs x 128 threads: 4 CTAs/SM (256 threads: 2)
constexpr int kRTWarps = kRTThreads / 32;

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

// ---- block reductions (256 threads) -------------------------------------------------------------
template <int K>
__device__ void block_sum(double (&v)[K], double* s_buf /* kRTWarps*K + K */) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < K; ++k)
    for (int o = 16; o; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  __syncthreads();
  if (lane == 0)
    for (int k = 0; k < K; ++k) s_buf[w * K + k] = v[k];
  __syncthreads();
  if (threadIdx.x < K) {
    double s = 0.0;
    for (int q = 0; q < kRTWarps; ++q) s += s_buf[q * K + threadIdx.x];
    s_buf[kRTWarps * K + threadIdx.x] = s;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = s_buf[kRTWarps * K + k];
}

__device__ double block_max(double v, double* s_buf) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) s_buf[w] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = s_buf[0];
    for (int q = 1; q < kRTWarps; ++q) s = fmax(s, s_buf[q]);
    s_buf[kRTWarps] = s;
  }
  __syncthreads();
  return s_buf[kRTWarps];
}

// ---- rotation TIM sets --------------------------------------------------------------------------------
// CHAIN (registration.cc:657-680): m TIMs materialised in ps/pd (pd already de-scaled, :697).
// COMPLETE (registration.cc:681-694): all m(m-1)/2 differences of the clique points, in computeTIMs order
// k = i*m - i(i+1)/2 + (j-i-1); they are recomputed from the m clique points on every pass instead of being
// materialised (only the per-TIM weight has to persist between GNC iterations).
struct TimSrc {
  int complete;
  int m;                // chain: number of TIMs; complete: number of clique points
  long long count;      // number of TIMs
  const double* a;      // chain: src TIMs (3*m)        complete: clique src points (3*m)
  const double* b;      // chain: dst TIMs, de-scaled   complete: clique dst points (3*m)
  double inv_scale;     // complete only: 1/scale applied to dst differences
};

template <class F>
__device__ __forceinline__ void for_each_tim(const TimSrc& t, F&& f) {
  if (!t.complete) {
    for (int k = threadIdx.x; k < t.m; k += kRTThreads)
      f((long long)k, t.a[3 * k], t.a[3 * k + 1], t.a[3 * k + 2], t.b[3 * k], t.b[3 * k + 1], t.b[3 * k + 2]);
  } else {
    for (int i = 0; i + 1 < t.m; ++i) {
      const long long base = (long long)i * t.m - (long long)i * (i + 1) / 2 - i - 1;
      const double sx = t.a[3 * i], sy = t.a[3 * i + 1], sz = t.a[3 * i + 2];
      const double dx = t.b[3 * i], dy = t.b[3 * i + 1], dz = t.b[3 * i + 2];
      for (int j = i + 1 + threadIdx.x; j < t.m; j += kRTThreads)
        f(base + j, t.a[3 * j] - sx, t.a[3 * j + 1] - sy, t.a[3 * j + 2] - sz, (t.b[3 * j] - dx) * t.inv_scale,
          (t.b[3 * j + 1] - dy) * t.inv_scale, (t.b[3 * j + 2] - dz) * t.inv_scale);
    }
  }
}

struct GncOut {
  M3 R;
  double cost;
  int iters;
};

// weighted covariance H = X diag(w) Y^T (utils.h:125) reduced over the block, then R on one thread
__device__ void rotation_step(const TimSrc& ts, const double* __restrict__ wgt, bool planar, double* s_buf, M3* s_R) {
  double h[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) h[k] = 0.0;
  for_each_tim(ts, [&](long long k, double x0, double x1, double x2, double y0, double y1, double y2) {
    const double w = wgt[k];
    const double a0 = x0 * w, a1 = x1 * w, a2 = x2 * w;
    h[0] += a0 * y0; h[1] += a1 * y0; h[2] += a2 * y0;
    h[3] += a0 * y1; h[4] += a1 * y1; h[5] += a2 * y1;
    h[6] += a0 * y2; h[7] += a1 * y2; h[8] += a2 * y2;
  });
  block_sum<9>(h, s_buf);
  if (threadIdx.x == 0) {
    M3 R;
    if (!planar) {
      M3 H;
#pragma unroll
      for (int k = 0; k < 9; ++k) H.a[k] = h[k];
      rotation_from_H(H, R);
    } else {
      // utils::svdRot2d (utils.h:145-160): the proper rotation maximising tr(R H2) for the 2x2 block
      // H2 = [h00 h01; h10 h11] is R = [c -s; s c] with (c, s) ~ (h00 + h11, h01 - h10)  (closed form of V U^T)
      double h2[4] = {h[0], h[1], h[3], h[4]};
      normalise_scale(h2, 4);
      const double ca = h2[0] + h2[3], sb = h2[2] - h2[1];
      const double nrm = sqrt(ca * ca + sb * sb);
      m3_identity(R);
      if (nrm > 0.0) {
        const double c = ca / nrm, sn = sb / nrm;
        R(0, 0) = c; R(0, 1) = -sn; R(1, 0) = sn; R(1, 1) = c;
      }
    }
    *s_R = R;
  }
  __syncthreads();
}

// ---- GNC-TLS (registration.cc:764-866) and Quatro (registration.cc:280-408; planar = yaw only), whole CTA ----
__device__ void gnc_tls_block(const TimSrc& ts, bool planar, unsigned long long max_iterations, double cost_threshold,
                              double gnc_factor, double noise_bound, double* __restrict__ wgt,
                              uint8_t* __restrict__ mask, GncOut& out, double* s_buf, M3* s_R) {
  double mu = 1.0;
  double prev_cost = 1.0 / 0.0, cost = 1.0 / 0.0;
  double nbsq = noise_bound * noise_bound;  // std::pow(x, 2)
  if (nbsq < 1e-16) nbsq = 1e-2;            // :794-796
  for (long long j = threadIdx.x; j < ts.count; j += kRTThreads) wgt[j] = 1.0;
  m3_identity(out.R);
  int it_done = 0;
  __syncthreads();
  for (unsigned long long i = 0; i < max_iterations; ++i) {
    it_done = (int)i + 1;
    rotation_step(ts, wgt, planar, s_buf, s_R);
    const M3 R = *s_R;
    out.R = R;
    auto residual = [&](double x, double y, double z, double p0, double p1, double p2) {
      const double d0 = p0 - (R(0, 0) * x + R(0, 1) * y + R(0, 2) * z);
      const double d1 = p1 - (R(1, 0) * x + R(1, 1) * y + R(1, 2) * z);
      if (planar) return d0 * d0 + d1 * d1;  // :349-350 (x,y rows only)
      const double d2 = p2 - (R(2, 0) * x + R(2, 1) * y + R(2, 2) * z);
      return d0 * d0 + d1 * d1 + d2 * d2;  // :812-813
    };
    if (i == 0) {  // :814-825
      double rmax = 0.0;
      for_each_tim(ts, [&](long long, double x, double y, double z, double p0, double p1, double p2) {
        rmax = fmax(rmax, residual(x, y, z, p0, p1, p2));
      });
      const double max_residual = block_max(rmax, s_buf);
      mu = 1.0 / (2.0 * max_residual / nbsq - 1.0);
      if (mu <= 0.0) break;
    }
    const double th1 = (mu + 1.0) / mu * nbsq;  // :828-829
    const double th2 = mu / (mu + 1.0) * nbsq;
    double c1[1] = {0.0};
    for_each_tim(ts, [&](long long k, double x, double y, double z, double p0, double p1, double p2) {
      const double r2 = residual(x, y, z, p0, p1, p2);
      c1[0] += wgt[k] * r2;  // cost with the previous weights (:834)
      double wn;
      if (r2 >= th1)
        wn = 0.0;
      else if (r2 <= th2)
        wn = 1.0;
      else
        wn = sqrt(nbsq * mu * (mu + 1.0) / r2) - mu;
      wgt[k] = wn;
    });
    block_sum<1>(c1, s_buf);
    cost = c1[0];
    const double cost_diff = fabs(cost - prev_cost);  // :847
    mu = mu * gnc_factor;                             // :850
    prev_cost = cost;
    if (cost_diff < cost_threshold) break;  // :853
  }
  __syncthreads();
  const double thr = planar ? 0.4 : 0.5;  // :400 / :863
  if (mask)
    for (long long j = threadIdx.x; j < ts.count; j += kRTThreads) mask[j] = wgt[j] >= thr;
  out.cost = cost;
  out.iters = it_done;
}

// ---- FGR rotation (registration.cc:206-278), whole CTA ----------------------------------------------------
// utils::calculateDiameter (utils.h:107-112) returns a float: 2*sqrt(max ||x - mean||^2) rounded to single.
__device__ double tim_diameter(const TimSrc& ts, bool dst_side, double* s_buf) {
  double c[3] = {0.0, 0.0, 0.0};
  for_each_tim(ts, [&](long long, double x, double y, double z, double p0, double p1, double p2) {
    c[0] += dst_side ? p0 : x;
    c[1] += dst_side ? p1 : y;
    c[2] += dst_side ? p2 : z;
  });
  block_sum<3>(c, s_buf);
  const double n = (double)ts.count;
  const double g0 = c[0] / n, g1 = c[1] / n, g2 = c[2] / n;
  double mx = 0.0;
  for_each_tim(ts, [&](long long, double x, double y, double z, double p0, double p1, double p2) {
    const double a = (dst_side ? p0 : x) - g0, b = (dst_side ? p1 : y) - g1, cc = (dst_side ? p2 : z) - g2;
    mx = fmax(mx, a * a + b * b + cc * cc);
  });
  mx = block_max(mx, s_buf);
  return (double)(float)(2.0 * sqrt(mx));
}

__device__ void fgr_block(const TimSrc& ts, unsigned long long max_iterations, double cost_threshold,
                          double gnc_factor, double noise_bound, double* __restrict__ wgt, uint8_t* __restrict__ mask,
                          GncOut& out, double* s_buf, M3* s_R) {
  const double nbsq = noise_bound * noise_bound;
  double cost = 1.0 / 0.0;
  const double sd = tim_diameter(ts, false, s_buf), dd = tim_diameter(ts, true, s_buf);
  double global_scale = sd > dd ? sd : dd;  // :226
  global_scale /= nbsq;
  double mu = global_scale * global_scale / nbsq;  // :228
  const double min_mu = 1.0;
  for (long long j = threadIdx.x; j < ts.count; j += kRTThreads) wgt[j] = 1.0;
  M3 R;
  m3_identity(R);
  int it_done = 0;
  __syncthreads();
  for (unsigned long long i = 0; i < max_iterations; ++i) {
    it_done = (int)i + 1;
    const double scaled_mu = mu * nbsq;
    for_each_tim(ts, [&](long long k, double x, double y, double z, double p0, double p1, double p2) {
      const double d0 = p0 - (R(0, 0) * x + R(0, 1) * y + R(0, 2) * z);
      const double d1 = p1 - (R(1, 0) * x + R(1, 1) * y + R(1, 2) * z);
      const double d2 = p2 - (R(2, 0) * x + R(2, 1) * y + R(2, 2) * z);
      const double q = scaled_mu / (scaled_mu + (d0 * d0 + d1 * d1 + d2 * d2));
      wgt[k] = q * q;  // :250
    });
    __syncthreads();
    rotation_step(ts, wgt, false, s_buf, s_R);  // :254
    R = *s_R;
    double c1[1] = {0.0};
    for_each_tim(ts, [&](long long, double x, double y, double z, double p0, double p1, double p2) {
      const double d0 = p0 - (R(0, 0) * x + R(0, 1) * y + R(0, 2) * z);
      const double d1 = p1 - (R(1, 0) * x + R(1, 1) * y + R(1, 2) * z);
      const double d2 = p2 - (R(2, 0) * x + R(2, 1) * y + R(2, 2) * z);
      const double sq = d0 * d0 + d1 * d1 + d2 * d2;
      c1[0] += (scaled_mu * sq) / (scaled_mu + sq);  // :257-260
    });
    block_sum<1>(c1, s_buf);
    cost = c1[0];
    if (cost < cost_threshold || mu < min_mu) break;  // :263
    mu /= gnc_factor;                                 // :272
  }
  __syncthreads();
  if (mask)
    for (long long j = threadIdx.x; j < ts.count; j += kRTThreads) mask[j] = wgt[j] != 0.0;  // l_pq.cast<bool>() :276
  out.R = R;
  out.cost = cost;
  out.iters = it_done;
}

// dispatch on ROTATION_ESTIMATION_ALGORITHM (registration.h:382-386)
__device__ void rotation_block(int alg, const TimSrc& ts, unsigned long long max_iterations, double cost_threshold,
                               double gnc_factor, double noise_bound, double* wgt, uint8_t* mask, GncOut& out,
                               double* s_buf, M3* s_R) {
  if (alg == 1)
    fgr_block(ts, max_iterations, cost_threshold, gnc_factor, noise_bound, wgt, mask, out, s_buf, s_R);
  else
    gnc_tls_block(ts, alg == 2, max_iterations, cost_threshold, gnc_factor, noise_bound, wgt, mask, out, s_buf, s_R);
}

// ---- TLS translation (registration.cc:445-471), whole CTA ---------------------------------------------------------
// raw: axis-major raw[ax*m + i]; key/idx: 3 * next_pow2(2m) entries.  s_t (shared, 3) receives the estimate of each
// axis; mask[i] = measurement i is an inlier on all three axes.  Returns the number of inliers on every thread.
__device__ int tls_translation(const double* __restrict__ raw, int m, double beta, double* key, int32_t* idx,
                               uint8_t* __restrict__ mask, double* s_t, int* s_cnt) {
  if (threadIdx.x == 0) *s_cnt = 0;
  tls_block(raw, nullptr, beta, m, 3, key, idx, s_t);
  int c = 0;
  for (int i = threadIdx.x; i < m; i += kRTThreads) {
    bool in = true;
#pragma unroll
    for (int ax = 0; ax < 3; ++ax) in = in && tls_inlier(raw[(size_t)ax * m + i], beta, s_t[ax]);  // :86, :469
    mask[i] = in;
    c += in;
  }
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(s_cnt, c);
  __syncthreads();
  return *s_cnt;
}

}  // namespace

// =================================================================================================
// batch kernel: clique finalisation + chain TIMs + GNC-TLS + TLS translation
// =================================================================================================
__global__ void __launch_bounds__(kRTThreads) rot_trans_kernel(Batch bt, tzr_params p, int use_clique, int exact_mode) {
  const int b = blockIdx.x;
  const int n = bt.n;
  const int tid = threadIdx.x;
  __shared__ double s_buf[kRTWarps * 9 + 9];
  __shared__ M3 s_R;
  __shared__ int s_scan[34];
  __shared__ double s_t[3];
  __shared__ int s_cnt[2];
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t* cbits = reinterpret_cast<uint32_t*>(smem_raw);  // pitch32(n) words

  tzr_solution* sol = bt.sol + b;
  int32_t* sc = bt.sorted_clq + (size_t)b * n;
  const double* src = bt.src + (size_t)b * n * 3;
  const double* dst = bt.dst + (size_t)b * n * 3;
  int m;
  if (use_clique) {
    // ---- sort the clique through a bitset (registration.cc:636)
    const int W = pitch32(n);
    m = bt.L[b];
    for (int x = tid; x < W; x += kRTThreads) cbits[x] = 0u;
    __syncthreads();
    const int32_t* cq = bt.clq + (size_t)b * n;
    for (int i = tid; i < m; i += kRTThreads) atomicOr(&cbits[cq[i] >> 5], 1u << (cq[i] & 31));
    __syncthreads();
    int base = 0;
    for (int x0 = 0; x0 < W; x0 += kRTThreads) {
      const int x = x0 + tid;
      const uint32_t wv = x < W ? cbits[x] : 0u;
      // exclusive scan of popcounts over the block
      const int lane = tid & 31, w = tid >> 5;
      int inc = __popc(wv);
      const int mine = inc;
      for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
      }
      __syncthreads();
      if (lane == 31) s_scan[w] = inc;
      __syncthreads();
      if (tid == 0) {
        int acc = 0;
        for (int q = 0; q < kRTWarps; ++q) {
          int t = s_scan[q];
          s_scan[q] = acc;
          acc += t;
        }
        s_scan[33] = acc;
      }
      __syncthreads();
      int pos = base + s_scan[w] + inc - mine;
      uint32_t mm = wv;
      while (mm) {
        const int bit = __ffs(mm) - 1;
        mm &= mm - 1;
        sc[pos++] = x * 32 + bit;
      }
      base += s_scan[33];
      __syncthreads();
    }
  } else {
    m = n;  // inlier selection NONE: every measurement is "in the clique" (registration.cc:650-653)
    for (int i = tid; i < n; i += kRTThreads) sc[i] = i;
  }
  __syncthreads();
  const double scale = sol->scale;
  if (tid == 0) {
    sol->clique_size = m;
    sol->n_edges = (int64_t)(bt.n_edges2[b] / 2ull);
    // 1: enumeration complete (canonical tie-break); 2: maximum size proven through the vertex-cover LP bound /
    // Nemhauser-Trotter reduction after the first search budget (max_clique.cu K4); 0: budget hit, incumbent returned
    sol->clique_proven_optimal = (use_clique && exact_mode && !(bt.flags[b] & 1)) ? ((bt.flags[b] & 12) ? 2 : 1) : 0;
    sol->valid = 1;
  }
  // registration.cc:643-647; a NaN scale: no TIM was finite (every source point identical), nothing to register
  if ((use_clique && m <= 1) || scale != scale) {
    if (tid == 0) sol->valid = 0;
    return;
  }
  // ---- rotation TIMs (registration.cc:657-694), de-scale dst (:697), rotation noise bound (:702-704)
  double* ps = bt.ps + (size_t)b * n * 3;
  double* pd = bt.pd + (size_t)b * n * 3;
  const double inv_scale = 1.0 / scale;
  TimSrc ts;
  ts.complete = p.rotation_tim_graph == 1;
  ts.m = m;
  ts.a = ps;
  ts.b = pd;
  ts.inv_scale = inv_scale;
  if (!ts.complete) {
    ts.count = m;
    for (int i = tid; i < m; i += kRTThreads) {
      const int root = sc[i];
      const int leaf = (i != m - 1) ? sc[i + 1] : sc[0];
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        ps[3 * i + r] = src[3 * (size_t)leaf + r] - src[3 * (size_t)root + r];
        pd[3 * i + r] = (dst[3 * (size_t)leaf + r] - dst[3 * (size_t)root + r]) * inv_scale;
      }
    }
  } else {
    ts.count = (long long)m * (m - 1) / 2;
    for (int i = tid; i < m; i += kRTThreads) {
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        ps[3 * i + r] = src[3 * (size_t)sc[i] + r];
        pd[3 * i + r] = dst[3 * (size_t)sc[i] + r];
      }
    }
  }
  if (ts.count > bt.rot_cap) {  // COMPLETE graph larger than the workspace: report, never compute garbage
    if (tid == 0) {
      sol->valid = 0;
      sol->clique_proven_optimal = -2;
    }
    return;
  }
  __syncthreads();
  const double rot_nb = p.noise_bound * (2.0 / scale);
  GncOut g;
  uint8_t* rmask = bt.rot_mask + (size_t)b * bt.rot_cap;
  rotation_block(p.rotation_estimation_algorithm, ts, p.rotation_max_iterations, p.rotation_cost_threshold,
                 p.rotation_gnc_factor, rot_nb, bt.wgt + (size_t)b * bt.rot_cap, rmask, g, s_buf, &s_R);
  __syncthreads();
  if (tid == 0) s_cnt[0] = 0;
  __syncthreads();
  {
    int c = 0;
    for (long long j = tid; j < ts.count; j += kRTThreads) c += rmask[j];
    c = __reduce_add_sync(0xffffffffu, c);
    if ((tid & 31) == 0 && c) atomicAdd(&s_cnt[0], c);
  }
  // ---- translation (registration.cc:717-731): raw = dst - (s*R)*src over the clique
  const M3 R = g.R;
  double sR[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) sR[k] = scale * R.a[k];
  double* raw = ps;  // reuse: axis-major raw[ax*m + i]
  __syncthreads();
  const double beta = p.noise_bound * sqrt(p.cbar2);
  // gather first (ps is overwritten by raw): compute into registers per i, then store
  for (int i0 = 0; i0 < m; i0 += kRTThreads) {
    const int i = i0 + tid;
    double v0 = 0, v1 = 0, v2 = 0;
    if (i < m) {
      const double* s = src + 3 * (size_t)sc[i];
      const double* d = dst + 3 * (size_t)sc[i];
      const double x = s[0], y = s[1], z = s[2];
      v0 = d[0] - (sR[0] * x + sR[3] * y + sR[6] * z);
      v1 = d[1] - (sR[1] * x + sR[4] * y + sR[7] * z);
      v2 = d[2] - (sR[2] * x + sR[5] * y + sR[8] * z);
    }
    __syncthreads();
    if (i < m) {
      raw[0 * (size_t)m + i] = v0;
      raw[1 * (size_t)m + i] = v1;
      raw[2 * (size_t)m + i] = v2;
    }
  }
  __syncthreads();
  // per-axis key capacity sort_cap = next_pow2(2n) >= next_pow2(2m)
  const int n_trans = tls_translation(raw, m, beta, bt.skey + (size_t)b * 3 * bt.sort_cap,
                                      bt.sidx + (size_t)b * 3 * bt.sort_cap, bt.trans_mask + (size_t)b * n, s_t,
                                      &s_cnt[1]);
  if (tid == 0) {
#pragma unroll
    for (int k = 0; k < 9; ++k) sol->rotation[k] = R.a[k];
    sol->translation[0] = s_t[0];
    sol->translation[1] = s_t[1];
    sol->translation[2] = s_t[2];
    sol->gnc_cost = g.cost;
    sol->gnc_iterations = g.iters;
    sol->n_rotation_inliers = s_cnt[0];
    sol->n_translation_inliers = n_trans;
    sol->valid = 1;
  }
}

void launch_rot_trans(const Batch& bt, const tzr_params& p, int use_clique, cudaStream_t st) {
  static bool attr_done_dev[64] = {};  // per device: a process may hold contexts on several GPUs
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr_done_dev[dev & 63]) {
    cudaFuncSetAttribute(rot_trans_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
    attr_done_dev[dev & 63] = true;
  }
  int mode = p.inlier_selection_mode;
  if (!p.use_max_clique) mode = 3;
  if (!p.max_clique_exact_solution) mode = 1;
  rot_trans_kernel<<<bt.B, kRTThreads, (size_t)pitch32(bt.n) * 4 + 16, st>>>(bt, p, use_clique, mode == 0 ? 1 : 0);
}

// =================================================================================================
// stand-alone stage kernels (per-stage C-ABI entry points)
// =================================================================================================
__global__ void __launch_bounds__(kRTThreads) gnc_only_kernel(int alg, const double* src, const double* dst, int m,
                                                               double noise_bound, double gnc_factor,
                                                               unsigned long long max_iter, double cost_thr,
                                                               double* wgt, double* res, double* out_R, uint8_t* mask,
                                                               double* out_cost, int* out_iters) {
  __shared__ double s_buf[kRTWarps * 9 + 9];
  __shared__ M3 s_R;
  (void)res;
  GncOut g;
  TimSrc ts;
  ts.complete = 0;
  ts.m = m;
  ts.count = m;
  ts.a = src;
  ts.b = dst;
  ts.inv_scale = 1.0;
  rotation_block(alg, ts, max_iter, cost_thr, gnc_factor, noise_bound, wgt, mask, g, s_buf, &s_R);
  if (threadIdx.x == 0) {
    for (int k = 0; k < 9; ++k) out_R[k] = g.R.a[k];
    *out_cost = g.cost;
    *out_iters = g.iters;
  }
}

void launch_gnc_only(int alg, const double* src, const double* dst, int m, double noise_bound, double gnc_factor,
                     unsigned long long max_iter, double cost_thr, double* wgt, double* res, double* out_R,
                     uint8_t* mask, double* out_cost, int* out_iters, cudaStream_t st) {
  gnc_only_kernel<<<1, kRTThreads, 0, st>>>(alg, src, dst, m, noise_bound, gnc_factor, max_iter, cost_thr, wgt, res,
                                            out_R, mask, out_cost, out_iters);
}

// translation: raw = dst - src per axis, TLS with constant range beta
__global__ void __launch_bounds__(kRTThreads) translation_only_kernel(const double* src, const double* dst, int m,
                                                                       double beta, double* key, int32_t* idx,
                                                                       double* raw, double* out_t, uint8_t* mask) {
  __shared__ double s_t[3];
  __shared__ int s_cnt;
  for (int i = threadIdx.x; i < m; i += kRTThreads)
    for (int ax = 0; ax < 3; ++ax) raw[(size_t)ax * m + i] = dst[3 * (size_t)i + ax] - src[3 * (size_t)i + ax];  // :455
  __syncthreads();
  tls_translation(raw, m, beta, key, idx, mask, s_t, &s_cnt);
  if (threadIdx.x < 3) out_t[threadIdx.x] = s_t[threadIdx.x];
}

void launch_translation_only(const double* src, const double* dst, int m, double beta, double* key, int32_t* idx,
                             double* raw, double* out_t, uint8_t* mask, cudaStream_t st) {
  translation_only_kernel<<<1, kRTThreads, 0, st>>>(src, dst, m, beta, key, idx, raw, out_t, mask);
}

}  // namespace tzr
