// Device-side scalar TLS (adaptive voting) shared by the translation, scale and stand-alone kernels.
// ScalarTLSEstimator::estimate  (teaser/src/registration.cc:21-88)
#pragma once
#include "tzr_internal.cuh"

namespace tzr {
namespace {

// ---- scalar TLS (registration.cc:21-88): bitonic sort of the 2M interval endpoints + sweep --------
// Arrays for `nax` independent estimators are processed together.  key/idx: nax * npad entries.
// payload idx: 2*i (lower endpoint, enters the consensus set) or 2*i+1 (upper endpoint, leaves it).
__device__ inline bool key_less(double ka, int ia, double kb, int ib) { return ka < kb || (ka == kb && ia < ib); }

__device__ void bitonic_sort_block(double* key, int* idx, int npad, int nax) {
  const int half = npad >> 1;
  for (int k = 2; k <= npad; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < half * nax; t += blockDim.x) {
        const int ax = t / half, q = t - ax * half;
        const int lo = 2 * q - (q & (j - 1));  // index with bit j cleared
        const int hi = lo + j;
        double* kk = key + (size_t)ax * npad;
        int* ii = idx + (size_t)ax * npad;
        const bool up = ((lo & k) == 0);
        const double ka = kk[lo], kb = kk[hi];
        const int ia = ii[lo], ib = ii[hi];
        const bool sw = up ? key_less(kb, ib, ka, ia) : key_less(ka, ia, kb, ib);
        if (sw) {
          kk[lo] = kb;
          kk[hi] = ka;
          ii[lo] = ib;
          ii[hi] = ia;
        }
      }
      __syncthreads();
    }
  }
}

// Excluded measurements (DESIGN.md §3.3): a measurement whose value or range is not finite (a TIM with d1 = 0, a NaN
// coordinate) contributes no end points.  Both its keys are +inf, so they sort after every kept end point and before the
// padding (payload 0x7fffffff), no NaN ever reaches a sort, and the sweeps skip them; the payloads of the kept
// measurements, hence their tie order (value, then payload), do not change.
__device__ __forceinline__ bool tls_kept(double x, double r) { return isfinite(x) && isfinite(r); }
// sort key of end point q (payload q: 2i enters, 2i+1 leaves) of measurement i = q >> 1   (registration.cc:36-37)
__device__ __forceinline__ double tls_key(double x, double r, long long q) {
  if (!tls_kept(x, r)) return 1.0 / 0.0;
  return (q & 1) ? x + r : x - r;
}

// Sequential sweep over the sorted endpoints (one thread), exactly the reference's accumulation order.
// X: measurements, ranges: per-measurement range (or nullptr -> const_range).
// Returns NaN when no measurement is kept.
__device__ double tls_sweep(const double* __restrict__ X, const double* __restrict__ ranges, double const_range,
                            long long M, const int* __restrict__ idx) {
  double ranges_inverse_sum = 0.0;
  for (long long i = 0; i < M; ++i) {  // ranges.sum() :51, over the kept measurements
    const double r = ranges ? ranges[i] : const_range;
    if (tls_kept(X[i], r)) ranges_inverse_sum += r;
  }
  double dot_X_weights = 0.0, dot_weights_consensus = 0.0;
  long long consensus = 0;
  double sum_xi = 0.0, sum_xi_square = 0.0;
  double best_cost = 0.0, best_xhat = 0.0 / 0.0;
  bool first = true;
  const long long nr = 2 * M;
  for (long long i = 0; i < nr; ++i) {  // :58-75
    const int e = idx[i];
    const long long id = e >> 1;
    const double r = ranges ? ranges[id] : const_range;
    const double x = X[id];
    if (!tls_kept(x, r)) continue;
    const double eps = (e & 1) ? -1.0 : 1.0;
    const double w = 1.0 / (r * r);
    consensus += (e & 1) ? -1 : 1;
    dot_weights_consensus += eps * w;
    dot_X_weights += eps * w * x;
    ranges_inverse_sum -= eps * r;
    sum_xi += eps * x;
    sum_xi_square += eps * x * x;
    const double x_hat = dot_X_weights / dot_weights_consensus;
    const double residual = (double)consensus * x_hat * x_hat + sum_xi_square - 2.0 * sum_xi * x_hat;
    const double x_cost = residual + ranges_inverse_sum;
    if (first || x_cost < best_cost) {  // minCoeff: first strict minimum, NaN never wins after the first end point
      best_cost = x_cost;
      best_xhat = x_hat;
      first = false;
    }
  }
  return best_xhat;
}

// Inlier flag of a measurement against the estimate (registration.cc:86); false for an excluded measurement.
// By reference, so that operands in memory are read where the expression uses them (the range only for a finite value,
// the estimate only for a kept measurement), as the inline expression did.
__device__ __forceinline__ bool tls_inlier(const double& x, const double& r, const double& est) {
  return tls_kept(x, r) && fabs(x - est) <= r;
}

// Scalar TLS of `nax` independent estimators in one CTA.  Estimator ax has the m measurements x[ax*m + i] with ranges
// r[ax*m + i], or the constant range c_range when r is nullptr.  key/idx: nax * next_pow2(2m) entries of scratch.
// The end points of each estimator are padded to a power of two with (+inf, 0x7fffffff), which sorts after every real
// one, and sorted together; thread 32*ax then sweeps estimator ax.  On return est[ax] (shared memory) holds its estimate
// on every thread.
__device__ __forceinline__ void tls_block(const double* __restrict__ x, const double* __restrict__ r, double c_range,
                                          int m, int nax, double* key, int* idx, double* est) {
  const int npad = next_pow2(2 * m);
  for (int t = threadIdx.x; t < nax * npad; t += blockDim.x) {
    const int ax = t / npad, q = t - ax * npad;
    if (q < 2 * m) {
      const size_t i = (size_t)ax * m + (q >> 1);
      key[t] = tls_key(x[i], r ? r[i] : c_range, q);  // registration.cc:36-37
      idx[t] = q;
    } else {
      key[t] = 1.0 / 0.0;
      idx[t] = 0x7fffffff;
    }
  }
  __syncthreads();
  bitonic_sort_block(key, idx, npad, nax);
  if ((threadIdx.x & 31) == 0 && (threadIdx.x >> 5) < nax) {
    const int ax = threadIdx.x >> 5;
    est[ax] = tls_sweep(x + (size_t)ax * m, r ? r + (size_t)ax * m : nullptr, c_range, m, idx + (size_t)ax * npad);
  }
  __syncthreads();
}

}  // namespace
}  // namespace tzr
