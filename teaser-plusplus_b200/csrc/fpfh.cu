// Descriptor estimation upstream of the matcher: teaser::FPFHEstimation::computeFPFHFeatures (reference
// teaser/src/fpfh.cc:15-43), i.e. PCL's NormalEstimationOMP + FPFHEstimationOMP with radius searches, on the device.
//
//   normals_kernel   one CTA per point: brute-force radius search (float squared distances in flann::L2_Simple's
//                    order, strict `< r^2`), neighbours sorted by (distance, index) like the sorted KD-tree result,
//                    single-pass float mean/covariance in that order (PCL <= 1.11 computeMeanAndCovarianceMatrix),
//                    pcl::eigen33's analytic smallest eigenpair, flip towards the viewpoint (0,0,0).
//   spfh_kernel      one CTA per point: radius search again (larger radius), one thread per neighbour computes
//                    pcl::computePairFeatures and bins f1/f2/f3 (11 bins each); the `+= hist_incr` float additions are
//                    replayed per bin from the integer counts (adding the same constant c times does not depend on
//                    which neighbour came first).
//   fpfh_kernel      one CTA per point: radius search + sort, then pcl's weightPointSPFHSignature as written: three
//                    threads (one per sub-histogram) run the sequential 1/d^2-weighted float sums in neighbour order
//                    and normalise to 100.
//
// Elementary functions: the det_* routines below are operation-for-operation copies of oracle/fpfh_oracle.cc's
// (IEEE float + - * / sqrt only, -fmad=false), so the device output is comparable bit for bit with the restatement.
// Radius search: brute force below kGridMinN points (n^2 float distance tests from L2-resident points cost well under a
// millisecond there); above, a hashed uniform grid with cell edge = the larger radius * (1 + 1e-5): points are sorted
// by bucket (CUB radix sort — library call, like the matcher's), every query visits the <= 27 distinct buckets of its
// 3x3x3 cell neighbourhood and applies the SAME float distance test, so the neighbour sets — and everything downstream —
// are identical to the brute-force ones (a point two cells away is farther than the radius by more than the float
// error of the test; hash collisions only add candidates that fail it).  A cloud with a finite point too far from its
// bounding-box minimum for an accurate double cell index (kCellIndexMax) is searched by brute force.  Debug flags
// 4194304 / 8388608 force brute force / the grid for every cloud.
//
// Batches: every kernel runs over B clouds stored back to back (one CTA per point of the whole batch); a CTA finds its
// cloud from the per-cloud FpfhCloud table and searches only inside it.  Each grid cloud owns the bucket range
// [base, base + T_b); one radix sort on base + hash orders the points of all of them, and the table (origin, 1/h, mask,
// base, brute-force fallback) stays on the device, so nothing is read back before the three descriptor kernels.  A
// single cloud is the B = 1 case of the same launches.
#include <math_constants.h>

#include <cub/cub.cuh>

#include <algorithm>

#include "tzr_internal.cuh"

namespace tzr {

namespace {

constexpr int kFpfhThreads = 256;
constexpr int kNbCap = 4096;  // neighbours per point held in shared memory (32 KB of 64-bit keys)

constexpr float kPiF = 3.14159265358979323846f;
constexpr float kPio2F = 1.57079632679489661923f;
constexpr float kPio4F = 0.78539816339744830962f;

__device__ __forceinline__ float det_atan_pos(float x) {  // x >= 0
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

// std::atan2's special values: atan2(+-0, x) is +-0 for x >= +0 and +-pi for x <= -0; both infinite: +-pi/4, +-3pi/4
__device__ __forceinline__ float det_atan2(float y, float x) {
  if (x != x || y != y) return CUDART_NAN_F;
  if (y == 0.0f) return signbit(x) ? copysignf(kPiF, y) : y;
  if (x == 0.0f) return y > 0.0f ? kPio2F : -kPio2F;
  if (isinf(x) && isinf(y)) return copysignf(x > 0.0f ? kPio4F : 3.0f * kPio4F, y);
  float a = det_atan_pos(fabsf(y) / fabsf(x));
  if (x < 0.0f) a = kPiF - a;
  return y < 0.0f ? -a : a;
}

// computeRoots' angle: y = sqrtf(-q) is +0 or -0 (sqrtf(-0) = -0) when q = 0, and both zeros give pi for x < 0 and 0
// otherwise, so that theta stays in det_sincos_0_pi2's domain [0, pi/3]
__device__ __forceinline__ float det_atan2_roots(float y, float x) {
  if (y == 0.0f && x == x) return (x < 0.0f) ? kPiF : 0.0f;
  return det_atan2(y, x);
}

__device__ __forceinline__ float det_asin_small(float x) {  // |x| <= 0.5
  const float z = x * x;
  return ((((4.2163199048e-2f * z + 2.4181311049e-2f) * z + 4.5470025998e-2f) * z + 7.4953002686e-2f) * z + 1.6666752422e-1f) * z * x + x;
}

__device__ __forceinline__ float det_acos01(float x) {  // x >= 0; NaN for x > 1 or NaN
  if (!(x <= 1.0f)) return CUDART_NAN_F;
  if (x > 0.5f) return 2.0f * det_asin_small(sqrtf(0.5f * (1.0f - x)));
  return kPio2F - det_asin_small(x);
}

__device__ __forceinline__ float det_sin_q(float x) {
  const float z = x * x;
  return ((-1.9515295891e-4f * z + 8.3321608736e-3f) * z - 1.6666654611e-1f) * z * x + x;
}
__device__ __forceinline__ float det_cos_q(float x) {
  const float z = x * x;
  return ((2.443315711809948e-5f * z - 1.388731625493765e-3f) * z + 4.166664568298827e-2f) * z * z - 0.5f * z + 1.0f;
}
__device__ __forceinline__ void det_sincos_0_pi2(float t, float* s, float* c) {
  if (t <= kPio4F) {
    *s = det_sin_q(t);
    *c = det_cos_q(t);
  } else {
    const float u = kPio2F - t;
    *s = det_cos_q(u);
    *c = det_sin_q(u);
  }
}

// pcl::computeRoots2 / computeRoots (common/impl/eigen.hpp), float
__device__ void compute_roots2(float b, float c, float* roots) {
  roots[0] = 0.f;
  float d = b * b - 4.0f * c;
  if (d < 0.0f) d = 0.0f;
  const float sd = sqrtf(d);
  roots[2] = 0.5f * (b + sd);
  roots[1] = 0.5f * (b - sd);
}

__device__ void compute_roots(const float m[3][3], float* roots) {
  const float c0 = m[0][0] * m[1][1] * m[2][2] + 2.0f * m[0][1] * m[0][2] * m[1][2] - m[0][0] * m[1][2] * m[1][2] -
                   m[1][1] * m[0][2] * m[0][2] - m[2][2] * m[0][1] * m[0][1];
  const float c1 = m[0][0] * m[1][1] - m[0][1] * m[0][1] + m[0][0] * m[2][2] - m[0][2] * m[0][2] +
                   m[1][1] * m[2][2] - m[1][2] * m[1][2];
  const float c2 = m[0][0] + m[1][1] + m[2][2];
  if (fabsf(c0) < 1.1920928955078125e-07f) {  // std::numeric_limits<float>::epsilon()
    compute_roots2(c2, c1, roots);
    return;
  }
  const float s_inv3 = 1.0f / 3.0f;
  const float s_sqrt3 = sqrtf(3.0f);
  const float c2_over_3 = c2 * s_inv3;
  float a_over_3 = (c1 - c2 * c2_over_3) * s_inv3;
  if (a_over_3 > 0.0f) a_over_3 = 0.0f;
  const float half_b = 0.5f * (c0 + c2_over_3 * (2.0f * c2_over_3 * c2_over_3 - c1));
  float q = half_b * half_b + a_over_3 * a_over_3 * a_over_3;
  if (q > 0.0f) q = 0.0f;
  const float rho = sqrtf(-a_over_3);
  const float theta = det_atan2_roots(sqrtf(-q), half_b) * s_inv3;
  float cos_theta, sin_theta;
  det_sincos_0_pi2(theta, &sin_theta, &cos_theta);
  roots[0] = c2_over_3 + 2.0f * rho * cos_theta;
  roots[1] = c2_over_3 - rho * (cos_theta + s_sqrt3 * sin_theta);
  roots[2] = c2_over_3 - rho * (cos_theta - s_sqrt3 * sin_theta);
  float t;
  if (roots[0] >= roots[1]) { t = roots[0]; roots[0] = roots[1]; roots[1] = t; }
  if (roots[1] >= roots[2]) {
    t = roots[1]; roots[1] = roots[2]; roots[2] = t;
    if (roots[0] >= roots[1]) { t = roots[0]; roots[0] = roots[1]; roots[1] = t; }
  }
  if (roots[0] <= 0.0f) compute_roots2(c2, c1, roots);
}

__device__ __forceinline__ void cross3(const float* a, const float* b, float* o) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}

// pcl::eigen33(mat, eigenvalue, eigenvector)
__device__ void eigen33_smallest(const float cov[3][3], float* eigenvalue, float* vec) {
  float scale = 0.f;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) scale = fmaxf(scale, fabsf(cov[r][c]));
  if (scale <= 1.17549435e-38f) scale = 1.0f;  // std::numeric_limits<float>::min()
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
  const float s = sqrtf(len);
  for (int k = 0; k < 3; ++k) vec[k] = best[k] / s;
}

// pcl::computePairFeatures (features/src/pfh_tools.cpp)
__device__ bool pair_features(const float* p1, const float* n1, const float* p2, const float* n2, float* f1,
                              float* f2, float* f3) {
  float dp[3] = {p2[0] - p1[0], p2[1] - p1[1], p2[2] - p1[2]};
  const float f4 = sqrtf(dp[0] * dp[0] + dp[1] * dp[1] + dp[2] * dp[2]);
  if (f4 == 0.0f) return false;
  float a[3] = {n1[0], n1[1], n1[2]}, b[3] = {n2[0], n2[1], n2[2]};
  const float angle1 = (a[0] * dp[0] + a[1] * dp[1] + a[2] * dp[2]) / f4;
  const float angle2 = (b[0] * dp[0] + b[1] * dp[1] + b[2] * dp[2]) / f4;
  if (det_acos01(fabsf(angle1)) > det_acos01(fabsf(angle2))) {
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
  const float vn = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  if (vn == 0.0f) return false;
  for (int k = 0; k < 3; ++k) v[k] /= vn;
  float w[3];
  cross3(a, v, w);
  *f2 = v[0] * b[0] + v[1] * b[1] + v[2] * b[2];
  *f1 = det_atan2(w[0] * b[0] + w[1] * b[1] + w[2] * b[2], a[0] * b[0] + a[1] * b[1] + a[2] * b[2]);
  return true;
}

constexpr int kGridMinN = 4096;

// the cloud of flat point p: the last c with clouds[c].lo <= p (every cloud has at least one point)
__device__ __forceinline__ int cloud_of(const FpfhCloud* __restrict__ clouds, int B, int p) {
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (clouds[mid].lo <= p) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

struct Grid {           // the radius search of one cloud; n_sorted == 0 means brute force over [lo, lo + n)
  const int* sorted;    // flat point indices of the batch sorted by bucket
  const int* bstart;    // [buckets] first position of every bucket in sorted
  const int* bend;      // [buckets] one past the last
  int lo, n;
  int n_sorted;
  unsigned int mask;    // T_b - 1
  unsigned int base;    // first bucket of the cloud
  double ox, oy, oz;    // grid origin (bounding-box minimum)
  double inv_h;         // 1 / cell edge
};

__device__ __forceinline__ unsigned int cell_hash(long long ix, long long iy, long long iz, unsigned int mask) {
  return ((unsigned int)(ix * 73856093ll) ^ (unsigned int)(iy * 19349663ll) ^ (unsigned int)(iz * 83492791ll)) & mask;
}

// Largest cell index the grid uses.  The index is u = fl(fl(x - o) * fl(1/h)) with x and the origin o floats (exact in
// double): the subtraction and the product each round by at most 2^-53 relative, and fl(1/h) and h = r (1 + 1e-5)
// carry two more such roundings, so |u - (x - o)/h| <= |u| 2^-51 (to first order).  Two points that pass the float
// test d^2 < r^2 are at most r (1 + 2^-20) apart per axis (the test's own rounding is a few 2^-24 relative), so their
// exact indices differ by at most (1 + 2^-20) / (1 + 1e-5) < 1 - 9e-6.  Their floors then differ by at most 1, which
// is what the 3x3x3 search needs, while the two index errors sum to less than 9e-6.  With |u| < 2^32 each error is at
// most 2^-19 < 1.91e-6, well inside that margin.  The bound grows with the extent and passes half the margin (4.5e-6)
// near 1e10 cells, about 2^33 (one far point at 1e11 with r = 0.01 is 2^43 cells: true neighbours land two cells
// apart), so a cloud
// with a finite point outside the range is searched by brute force.
constexpr double kCellIndexMax = 4294967296.0;  // 2^32

__device__ __forceinline__ bool cell_of(const Grid& g, float x, float y, float z, long long* ix, long long* iy,
                                        long long* iz) {
  if (!(x == x) || !(y == y) || !(z == z)) return false;
  const double fx = floor(((double)x - g.ox) * g.inv_h), fy = floor(((double)y - g.oy) * g.inv_h),
               fz = floor(((double)z - g.oz) * g.inv_h);
  // +-inf coordinates, and finite ones too far from the origin for an accurate index
  if (!(fabs(fx) < kCellIndexMax) || !(fabs(fy) < kCellIndexMax) || !(fabs(fz) < kCellIndexMax)) return false;
  *ix = (long long)fx;
  *iy = (long long)fy;
  *iz = (long long)fz;
  return true;
}

// bounding-box minimum over finite coordinates (ordered-int encoding of floats)
__device__ __forceinline__ int f2ord(float f) {
  const int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

// The search of cloud c: the grid when the cloud has one and every finite point of it found a cell, else brute force.
__device__ __forceinline__ Grid grid_of(const FpfhCloud& cl, const int* sorted, const int* bstart, const int* bend) {
  Grid g{};
  g.lo = cl.lo;
  g.n = cl.n;
  if (!cl.grid || cl.mins[3]) return g;
  g.sorted = sorted;
  g.bstart = bstart;
  g.bend = bend;
  g.n_sorted = cl.n;
  g.mask = cl.mask;
  g.base = cl.base;
  g.ox = (double)ord2f(cl.mins[0]);
  g.oy = (double)ord2f(cl.mins[1]);
  g.oz = (double)ord2f(cl.mins[2]);
  g.inv_h = cl.inv_h;
  return g;
}

// per-cloud minimum of the grid clouds' points; a warp whose lanes share one cloud reduces before its atomics
__global__ void bbox_min_kernel(const float* __restrict__ pts, int N, FpfhCloud* clouds, int B) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int m[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff};
  int c = -1;
  if (i < N) {
    c = cloud_of(clouds, B, i);
    if (clouds[c].grid)
      for (int k = 0; k < 3; ++k) {
        const float v = pts[3 * (size_t)i + k];
        if (isfinite(v)) m[k] = f2ord(v);
      }
  }
  const bool uniform = __all_sync(0xffffffffu, c == __shfl_sync(0xffffffffu, c, 0));
  for (int k = 0; k < 3; ++k) {
    if (uniform)
      for (int off = 16; off; off >>= 1) m[k] = min(m[k], __shfl_xor_sync(0xffffffffu, m[k], off));
    if ((!uniform || (threadIdx.x & 31) == 0) && m[k] != 0x7fffffff) atomicMin(&clouds[c].mins[k], m[k]);
  }
}

// key = the cloud's first bucket + cell hash; `buckets` (a bucket nobody visits) for non-finite points and for the
// points of brute-force clouds
__global__ void bucket_kernel(const float* __restrict__ pts, int N, FpfhCloud* clouds, int B, unsigned int buckets,
                              unsigned int* __restrict__ keys, int* __restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  idx[i] = i;
  const int c = cloud_of(clouds, B, i);
  FpfhCloud& cl = clouds[c];
  if (!cl.grid) {
    keys[i] = buckets;
    return;
  }
  Grid g{};
  g.ox = (double)ord2f(cl.mins[0]);
  g.oy = (double)ord2f(cl.mins[1]);
  g.oz = (double)ord2f(cl.mins[2]);
  g.inv_h = cl.inv_h;
  long long ix, iy, iz;
  const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
  const bool ok = cell_of(g, x, y, z, &ix, &iy, &iz);
  keys[i] = ok ? cl.base + cell_hash(ix, iy, iz, cl.mask) : buckets;
  // a finite point the grid cannot index accurately (kCellIndexMax cells or more from the origin): this cloud falls
  // back to brute force
  if (!ok && isfinite(x) && isfinite(y) && isfinite(z)) cl.mins[3] = 1;
}

__global__ void bucket_bounds_kernel(const unsigned int* __restrict__ keys, int n, unsigned int buckets,
                                     int* __restrict__ bstart, int* __restrict__ bend) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned int k = keys[i];
  if (k >= buckets) return;
  if (i == 0 || keys[i - 1] != k) bstart[k] = i;
  if (i == n - 1 || keys[i + 1] != k) bend[k] = i + 1;
}

// Block-wide radius search of point q inside its cloud: keys[] (shared, kNbCap) receives (d2 bits << 32 | index) of
// every point with d2 < r2, unordered; indices are flat, so their order within the cloud is the cloud-local one.
// Returns the count (may exceed kNbCap: overflow, caller flags it).  Contains __syncthreads.
__device__ int collect_neighbors(const float* __restrict__ pts, int q, float r2, unsigned long long* keys,
                                 int* s_count, const Grid& g) {
  __shared__ int s_rs[28], s_re[28], s_pref[28];
  if (threadIdx.x == 0) *s_count = 0;
  const float qx = pts[3 * (size_t)q], qy = pts[3 * (size_t)q + 1], qz = pts[3 * (size_t)q + 2];
  auto test = [&](int i) {
    const float dx = qx - pts[3 * (size_t)i], dy = qy - pts[3 * (size_t)i + 1], dz = qz - pts[3 * (size_t)i + 2];
    float d = dx * dx;
    d += dy * dy;
    d += dz * dz;
    if (d < r2) {
      const int pos = atomicAdd(s_count, 1);
      if (pos < kNbCap) keys[pos] = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned int)i;
    }
  };
  if (g.n_sorted == 0) {  // brute force
    __syncthreads();
    for (int i = g.lo + threadIdx.x; i < g.lo + g.n; i += blockDim.x) test(i);
    __syncthreads();
    return *s_count;
  }
  // the <= 27 distinct buckets of the 3x3x3 cell neighbourhood
  if (threadIdx.x < 27) {
    long long ix, iy, iz;
    int rs = 0, re = 0;
    if (cell_of(g, qx, qy, qz, &ix, &iy, &iz)) {
      const int t = threadIdx.x;
      const unsigned int b = cell_hash(ix + (t % 3) - 1, iy + ((t / 3) % 3) - 1, iz + (t / 9) - 1, g.mask);
      bool dup = false;
      for (int u = 0; u < t; ++u)
        dup |= cell_hash(ix + (u % 3) - 1, iy + ((u / 3) % 3) - 1, iz + (u / 9) - 1, g.mask) == b;
      if (!dup) {
        rs = g.bstart[g.base + b];
        re = g.bend[g.base + b];
      }
    }
    s_rs[threadIdx.x] = rs;
    s_re[threadIdx.x] = re;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int t = 0; t < 27; ++t) {
      s_pref[t] = acc;
      acc += s_re[t] - s_rs[t];
    }
    s_pref[27] = acc;
  }
  __syncthreads();
  const int total = s_pref[27];
  for (int c = threadIdx.x; c < total; c += blockDim.x) {
    int t = 0;
    while (c >= s_pref[t + 1]) ++t;
    test(g.sorted[s_rs[t] + (c - s_pref[t])]);
  }
  __syncthreads();
  return *s_count;
}

// ascending bitonic sort of keys[0..count) in shared memory (padded with ~0 to a power of two <= kNbCap)
__device__ void sort_keys(unsigned long long* keys, int count) {
  int np = 1;
  while (np < count) np <<= 1;
  for (int i = count + threadIdx.x; i < np; i += blockDim.x) keys[i] = ~0ull;
  __syncthreads();
  for (int k = 2; k <= np; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < np; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = keys[i], b = keys[ixj];
          const bool up = (i & k) == 0;
          if ((a > b) == up) {
            keys[i] = b;
            keys[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
}

// The arguments every descriptor kernel shares: the flat points, the cloud table and the batch's grid arrays.
struct Clouds {
  const float* pts;
  const FpfhCloud* clouds;
  int B;
  const int* sorted;
  const int* bstart;
  const int* bend;
  __device__ __forceinline__ int cloud(int p) const { return cloud_of(clouds, B, p); }
  __device__ __forceinline__ Grid grid(int c) const { return grid_of(clouds[c], sorted, bstart, bend); }
};

__global__ void __launch_bounds__(kFpfhThreads) normals_kernel(Clouds cs, float r2, float4* __restrict__ normals,
                                                              int* overflow) {
  __shared__ unsigned long long keys[kNbCap];
  __shared__ int s_count;
  const float* __restrict__ pts = cs.pts;
  const int p = blockIdx.x;
  const int c = cs.cloud(p);
  const int cnt = collect_neighbors(pts, p, r2, keys, &s_count, cs.grid(c));
  if (cnt > kNbCap) {
    if (threadIdx.x == 0) {
      atomicExch(&overflow[c], 1);
      normals[p] = make_float4(CUDART_NAN_F, CUDART_NAN_F, CUDART_NAN_F, CUDART_NAN_F);
    }
    return;
  }
  sort_keys(keys, cnt);
  if (threadIdx.x != 0) return;
  if (cnt < 3) {  // computePointNormal fails -> NaN normal (normal_3d.hpp)
    normals[p] = make_float4(CUDART_NAN_F, CUDART_NAN_F, CUDART_NAN_F, CUDART_NAN_F);
    return;
  }
  float accu[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int e = 0; e < cnt; ++e) {
    const int i = (int)(unsigned int)keys[e];
    const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
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
  const float fc = (float)cnt;
  for (int k = 0; k < 9; ++k) accu[k] /= fc;
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
  const float curvature = eig_sum != 0 ? fabsf(ev / eig_sum) : 0.f;
  const float vx = 0.f - pts[3 * (size_t)p], vy = 0.f - pts[3 * (size_t)p + 1], vz = 0.f - pts[3 * (size_t)p + 2];
  const float cos_theta = vx * nv[0] + vy * nv[1] + vz * nv[2];
  if (cos_theta < 0) {
    nv[0] *= -1;
    nv[1] *= -1;
    nv[2] *= -1;
  }
  normals[p] = make_float4(nv[0], nv[1], nv[2], curvature);
}

__device__ __forceinline__ int bin11(double v) {  // static_cast<int>(floor(v)) clamped to [0, 10]; NaN -> 0
  if (!(v == v)) return 0;
  const double f = floor(v);
  if (f < 0.0) return 0;
  if (f >= 11.0) return 10;
  return (int)f;
}

__global__ void __launch_bounds__(kFpfhThreads) spfh_kernel(Clouds cs, const float4* __restrict__ normals, float r2,
                                                           float* __restrict__ spfh, int* overflow) {
  __shared__ unsigned long long keys[kNbCap];
  __shared__ int s_count;
  __shared__ int s_bins[33];
  const float* __restrict__ pts = cs.pts;
  const int p = blockIdx.x;
  const int c = cs.cloud(p);
  if (threadIdx.x < 33) s_bins[threadIdx.x] = 0;
  const int cnt = collect_neighbors(pts, p, r2, keys, &s_count, cs.grid(c));  // its barriers also publish s_bins
  if (cnt > kNbCap) {
    if (threadIdx.x == 0) atomicExch(&overflow[c], 1);
    if (threadIdx.x < 33) spfh[(size_t)p * 33 + threadIdx.x] = 0.f;
    return;
  }
  const float d_pi = 1.0f / (2.0f * 3.14159265358979323846f);
  const float4 np4 = normals[p];
  const float pp[3] = {pts[3 * (size_t)p], pts[3 * (size_t)p + 1], pts[3 * (size_t)p + 2]};
  const float np_[3] = {np4.x, np4.y, np4.z};
  for (int e = threadIdx.x; e < cnt; e += blockDim.x) {
    const int i = (int)(unsigned int)keys[e];
    if (i == p) continue;
    const float4 nq4 = normals[i];
    const float pq[3] = {pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2]};
    const float nq[3] = {nq4.x, nq4.y, nq4.z};
    float f1, f2, f3;
    if (!pair_features(pp, np_, pq, nq, &f1, &f2, &f3)) continue;
    atomicAdd(&s_bins[bin11(11 * (((double)f1 + 3.14159265358979323846) * (double)d_pi))], 1);
    atomicAdd(&s_bins[11 + bin11(11 * (((double)f2 + 1.0) * 0.5))], 1);
    atomicAdd(&s_bins[22 + bin11(11 * (((double)f3 + 1.0) * 0.5))], 1);
  }
  __syncthreads();
  if (threadIdx.x < 33) {
    const float hist_incr = 100.0f / (float)(cnt - 1);
    float v = 0.f;
    for (int k = s_bins[threadIdx.x]; k > 0; --k) v += hist_incr;  // the reference's repeated `+= hist_incr`
    spfh[(size_t)p * 33 + threadIdx.x] = v;
  }
}

__global__ void __launch_bounds__(kFpfhThreads) fpfh_kernel(Clouds cs, const float* __restrict__ spfh, float r2,
                                                           float* __restrict__ out, int* overflow) {
  __shared__ unsigned long long keys[kNbCap];
  __shared__ int s_count;
  const int p = blockIdx.x;
  const int c = cs.cloud(p);
  const int cnt = collect_neighbors(cs.pts, p, r2, keys, &s_count, cs.grid(c));
  if (cnt > kNbCap) {
    if (threadIdx.x == 0) atomicExch(&overflow[c], 1);
    if (threadIdx.x < 33) out[(size_t)p * 33 + threadIdx.x] = 0.f;
    return;
  }
  sort_keys(keys, cnt);
  if (threadIdx.x >= 3) return;
  const int s = threadIdx.x;  // sub-histogram
  float acc[11];
#pragma unroll
  for (int k = 0; k < 11; ++k) acc[k] = 0.f;
  float sum = 0.f;
  for (int e = 0; e < cnt; ++e) {
    const unsigned long long key = keys[e];
    const float d2 = __uint_as_float((unsigned int)(key >> 32));
    if (d2 == 0) continue;
    const float weight = 1.0f / d2;
    const float* h = spfh + (size_t)(unsigned int)key * 33 + 11 * s;
#pragma unroll
    for (int k = 0; k < 11; ++k) {
      const float val = h[k] * weight;
      sum += val;
      acc[k] += val;
    }
  }
  float sc = sum;
  if (sc != 0) sc = (float)(100.0 / (double)sc);
#pragma unroll
  for (int k = 0; k < 11; ++k) out[(size_t)p * 33 + 11 * s + k] = acc[k] * sc;
}

// tzr_fpfh_pair_features / tzr_fpfh_smallest_eigenpair: the production device functions, one item per thread
__global__ void pair_features_kernel(int n, const float* __restrict__ p1, const float* __restrict__ n1,
                                     const float* __restrict__ p2, const float* __restrict__ n2, float* __restrict__ f,
                                     int32_t* __restrict__ ok) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float f1, f2, f3;
  const size_t o = 3 * (size_t)i;
  const bool good = pair_features(p1 + o, n1 + o, p2 + o, n2 + o, &f1, &f2, &f3);
  f[o] = good ? f1 : 0.f;
  f[o + 1] = good ? f2 : 0.f;
  f[o + 2] = good ? f3 : 0.f;
  ok[i] = good;
}

__global__ void smallest_eigenpair_kernel(int n, const float* __restrict__ cov, float* __restrict__ ev,
                                          float* __restrict__ vec) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float m[3][3], v[3];
  for (int k = 0; k < 9; ++k) m[k / 3][k % 3] = cov[9 * (size_t)i + k];
  eigen33_smallest(m, &ev[i], v);
  for (int k = 0; k < 3; ++k) vec[3 * (size_t)i + k] = v[k];
}

size_t radix_bytes(int n, int bits) {
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const unsigned int*)nullptr, (unsigned int*)nullptr,
                                  (const int*)nullptr, (int*)nullptr, n, 0, bits);
  return cub_bytes;
}

int key_bits(unsigned int buckets) {  // keys go up to `buckets` (the sentinel)
  int bits = 1;
  while (bits < 32 && (1ull << bits) <= buckets) ++bits;
  return bits;
}

}  // namespace

int fpfh_plan(int B, const int32_t* n, double normal_radius, double fpfh_radius, int route, FpfhCloud* clouds,
              FpfhPlan* plan) {
  const double h = std::max(normal_radius, fpfh_radius) * (1.0 + 1e-5);
  long long lo = 0, buckets = 0;
  bool any_grid = false;
  for (int c = 0; c < B; ++c) {
    FpfhCloud& cl = clouds[c];
    cl = FpfhCloud{};
    cl.lo = (int)lo;
    cl.n = n[c];
    cl.grid = route == kFpfhRouteBrute ? 0 : route == kFpfhRouteGrid ? 1 : n[c] >= kGridMinN;
    cl.mins[0] = cl.mins[1] = cl.mins[2] = 0x7fffffff;
    cl.mins[3] = 0;
    cl.inv_h = 1.0 / h;
    if (cl.grid) {
      unsigned int T = 1024;
      while (T < 2u * (unsigned int)n[c]) T <<= 1;
      cl.mask = T - 1;
      cl.base = (unsigned int)buckets;
      buckets += T;
      any_grid = true;
    }
    lo += n[c];
  }
  if (lo > 0x7fffffffll || buckets >= 0xffffffffll) return TZR_ERR_TOO_LARGE;
  plan->B = B;
  plan->N = (int)lo;
  plan->any_grid = any_grid;
  plan->buckets = (unsigned int)buckets;
  plan->grid_bytes = any_grid ? 4 * (size_t)lo * 4 + 2 * (size_t)buckets * 4 +
                                    radix_bytes(plan->N, key_bits(plan->buckets)) + 1024
                              : 0;
  return TZR_OK;
}

int launch_fpfh(const FpfhPlan& plan, const float* pts, FpfhCloud* clouds, double normal_radius, double fpfh_radius,
                float4* normals, float* spfh, float* out, int* overflow, void* grid_scratch, cudaStream_t st) {
  const float r2n = (float)(normal_radius * normal_radius);
  const float r2f = (float)(fpfh_radius * fpfh_radius);
  const int N = plan.N, B = plan.B;
  int nl = 0;
  cudaMemsetAsync(overflow, 0, (size_t)B * sizeof(int), st);
  Clouds cs{pts, clouds, B, nullptr, nullptr, nullptr};
  if (plan.any_grid) {
    const unsigned int T = plan.buckets;
    char* w = (char*)grid_scratch;
    unsigned int* keys = (unsigned int*)w;  w += (size_t)N * 4;
    unsigned int* keys2 = (unsigned int*)w; w += (size_t)N * 4;
    int* idx = (int*)w;                     w += (size_t)N * 4;
    int* idx2 = (int*)w;                    w += (size_t)N * 4;
    int* bstart = (int*)w;                  w += (size_t)T * 4;
    int* bend = (int*)w;                    w += (size_t)T * 4;
    const int bits = key_bits(T);
    size_t cub_bytes = radix_bytes(N, bits);
    cudaMemsetAsync(bstart, 0, 2 * (size_t)T * 4, st);
    bbox_min_kernel<<<(N + 255) / 256, 256, 0, st>>>(pts, N, clouds, B);
    bucket_kernel<<<(N + 255) / 256, 256, 0, st>>>(pts, N, clouds, B, T, keys, idx);
    cub::DeviceRadixSort::SortPairs((void*)w, cub_bytes, keys, keys2, idx, idx2, N, 0, bits, st);
    bucket_bounds_kernel<<<(N + 255) / 256, 256, 0, st>>>(keys2, N, T, bstart, bend);
    nl += 4;
    cs.sorted = idx2;
    cs.bstart = bstart;
    cs.bend = bend;
  }
  normals_kernel<<<N, kFpfhThreads, 0, st>>>(cs, r2n, normals, overflow);
  spfh_kernel<<<N, kFpfhThreads, 0, st>>>(cs, normals, r2f, spfh, overflow);
  fpfh_kernel<<<N, kFpfhThreads, 0, st>>>(cs, spfh, r2f, out, overflow);
  return nl + 3;
}

void launch_fpfh_pair_features(int n, const float* p1, const float* n1, const float* p2, const float* n2, float* f,
                               int32_t* ok, cudaStream_t st) {
  pair_features_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, p1, n1, p2, n2, f, ok);
}

void launch_fpfh_smallest_eigenpair(int n, const float* cov, float* ev, float* vec, cudaStream_t st) {
  smallest_eigenpair_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, cov, ev, vec);
}

}  // namespace tzr
