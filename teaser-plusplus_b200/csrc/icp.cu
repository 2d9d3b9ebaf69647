// Point-to-point ICP (the refinement step of the reference's FPFH + TEASER++ + ICP tutorial, DESIGN.md §3.11): Open3D's
// RegistrationICP with TransformationEstimationPointToPoint and ICPConvergenceCriteria, written out as this project's
// own definition in include/teaser_b200.h, for B problems at once.  Point-to-plane ICP (DESIGN.md §3.13) shares the
// search, the evaluation and the loop, and replaces the covariance and update pair with icp_plane_system_kernel (the
// centred 6 x 6 Gauss-Newton system) and icp_plane_update_kernel (its pivoted solve and the Euler rotation).
// Generalized ICP (DESIGN.md §3.14) replaces only the system, with icp_gicp_system_kernel (plane-to-plane covariances
// from both clouds' normals, the same 27 sums), and shares icp_plane_update_kernel.  Robust kernels (DESIGN.md §3.15)
// are the <true> instances of both system kernels: weighted sums, the same layout; the <false> instances are the
// unweighted systems and run for TZR_LOSS_L2.  Coloured ICP (DESIGN.md §3.17) replaces only the system, with
// icp_colored_system_kernel (a geometric and a photometric row per correspondence, the same 27 sums), after the
// targets' colour-gradient pass (fpfh.cu's launch_color_gradients).
//
//   icp_nn_kernel      one CTA per chunk of kIcpChunk source points: p = s (R x) + t in float64 (icp_transform), the
//                      nearest target with d^2 < r^2 (lowest index among equal d^2), by brute force through shared
//                      memory or through the target's hashed grid; writes the match per point and the chunk's sums
//                      (count, sum p, sum q, sum d^2).
//   icp_eval_kernel    one warp per problem: combines the chunk sums in a fixed order, evaluates fitness and rmse,
//                      applies the convergence test and clears the active flag.
//   icp_cov_kernel     one CTA per chunk: the centred cross-covariance sum (p - mu_p)(q - mu_q)^T of its matches.
//   icp_update_kernel  one warp per problem: combines it, runs rotation_from_H (the rotation stage's SVD and reflection
//                      fix), and composes the update into (R, t).
//
// Information matrices (DESIGN.md §3.16) reuse the grid build and icp_nn_kernel as they are, then sum the 21 entries of
// G^T G per correspondence in icp_info_kernel and combine them per problem in icp_info_combine_kernel.
//
// Every reduction runs in an order fixed by the problem's own points (chunk k of a problem always holds its points
// [256 k, 256 k + 256), and the chunks of a problem are combined by lane k mod 32 then a butterfly), so a problem's
// bits do not depend on the batch it runs in.  Finished problems return at once from every kernel.  The iterations are
// enqueued back to back without a host synchronisation; the launch count depends on max_iteration only.
#include <algorithm>

#include "rot3.cuh"
#include "tzr_internal.cuh"

namespace tzr {

namespace {

constexpr int kIcpThreads = kIcpChunk;

// p = s * (R x) + t, each row (R(r,0) x + R(r,1) y) + R(r,2) z, with -fmad=false: tests/icp_reference.py reproduces it
// bit for bit
__device__ __forceinline__ void icp_transform(const IcpProb& pr, const float* __restrict__ src, int i, double p[3]) {
  const double x = src[3 * (size_t)i], y = src[3 * (size_t)i + 1], z = src[3 * (size_t)i + 2];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double rx = (pr.R[r] * x + pr.R[3 + r] * y) + pr.R[6 + r] * z;
    p[r] = pr.s * rx + pr.t[r];
  }
}

__device__ __forceinline__ double icp_d2(const double p[3], double qx, double qy, double qz) {
  const double dx = p[0] - qx, dy = p[1] - qy, dz = p[2] - qz;
  return (dx * dx + dy * dy) + dz * dz;
}

// keep the lexicographically smallest (d2, j); *best starts at r^2 with *bj = INT_MAX (no match), and d2 = r^2 is no
// match (the bound is strict)
__device__ __forceinline__ void icp_keep(double d2, int j, double* best, int* bj) {
  if (d2 < *best || (d2 == *best && j < *bj && *bj != 0x7fffffff)) {
    *best = d2;
    *bj = j;
  }
}

// Fixed-order sum over a CTA of kIcpThreads threads: butterfly inside each warp (every lane ends with the same bits),
// then the warp sums in warp order by one thread.  Result in s_out[0..K).
template <int K>
__device__ void icp_block_sum(double (&v)[K], double* s_buf /* (kIcpThreads/32) * K */, double* s_out) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < K; ++k)
    for (int o = 16; o; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < K; ++k) s_buf[w * K + k] = v[k];
  __syncthreads();
  if (threadIdx.x < K) {
    double s = 0.0;
    for (int q = 0; q < kIcpThreads / 32; ++q) s += s_buf[q * K + threadIdx.x];
    s_out[threadIdx.x] = s;
  }
}

// Fixed-order sum of the problem's nc chunk partials (K of the S doubles each: S = 9 for the nearest-neighbour sums and
// the covariance, 27 for the point-to-plane system) over one warp: lane l takes chunks l, l + 32, ..., then a
// butterfly; every lane returns the same bits.
template <int K, int S = 9>
__device__ void icp_warp_combine(const double* __restrict__ partial, int c_lo, int nc, double (&v)[K]) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = 0.0;
  for (int c = lane; c < nc; c += 32)
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] += partial[S * (size_t)(c_lo + c) + k];
#pragma unroll
  for (int k = 0; k < K; ++k)
    for (int o = 16; o; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
}

struct IcpArgs {
  const float* src;
  const float* dst;
  IcpProb* probs;
  const FpfhCloud* clouds;
  const int* chunk_prob;
  int* match;
  double* partial;
  const int* sorted;    // the target grid (nullptr without grid targets)
  const int* bstart;
  const int* bend;
  double r2;
};

// Nearest target of p over all targets of the problem, read from global memory (a grid problem's query that the grid
// cannot index)
__device__ void icp_nn_scan(const float* __restrict__ dst, int d_lo, int nd, const double p[3], double* best,
                            int* bj) {
  for (int j = 0; j < nd; ++j) {
    const size_t o = 3 * (size_t)(d_lo + j);
    icp_keep(icp_d2(p, dst[o], dst[o + 1], dst[o + 2]), j, best, bj);
  }
}

__global__ void __launch_bounds__(kIcpThreads) icp_nn_kernel(IcpArgs a) {
  __shared__ double s_t[3][kIcpThreads];
  __shared__ double s_buf[(kIcpThreads / 32) * 8];
  const int c = blockIdx.x;
  const int b = a.chunk_prob[c];
  const IcpProb& pr = a.probs[b];
  if (!pr.active) return;
  const int i = (c - pr.c_lo) * kIcpChunk + threadIdx.x;  // source point inside the problem
  const bool have = i < pr.ns;
  double p[3] = {0.0, 0.0, 0.0};
  bool query = false;
  if (have) {
    icp_transform(pr, a.src, pr.s_lo + i, p);
    query = isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]);
  }
  double best = a.r2;  // strict d^2 < r^2: a candidate must be smaller than r^2 itself
  int bj = 0x7fffffff;
  const FpfhCloud& cl = a.clouds[pr.tc];
  if (!cl.grid || cl.mins[3]) {
    // brute force, the problem's targets tiled through shared memory
    for (int t0 = 0; t0 < pr.nd; t0 += kIcpThreads) {
      const int m = min(kIcpThreads, pr.nd - t0);
      __syncthreads();
      if (threadIdx.x < m) {
        const size_t o = 3 * (size_t)(pr.d_lo + t0 + threadIdx.x);
        s_t[0][threadIdx.x] = a.dst[o];
        s_t[1][threadIdx.x] = a.dst[o + 1];
        s_t[2][threadIdx.x] = a.dst[o + 2];
      }
      __syncthreads();
      if (query)
        for (int k = 0; k < m; ++k) {
          const double d2 = icp_d2(p, s_t[0][k], s_t[1][k], s_t[2][k]);
          if (d2 < best) {  // ascending j: the first of equal d^2 stays
            best = d2;
            bj = t0 + k;
          }
        }
    }
  } else if (query) {
    // the cell of the float64 query in the target's grid (DESIGN.md §3.11); out of the accurate range: brute force
    const double fx = floor((p[0] - (double)ord2f(cl.mins[0])) * cl.inv_h);
    const double fy = floor((p[1] - (double)ord2f(cl.mins[1])) * cl.inv_h);
    const double fz = floor((p[2] - (double)ord2f(cl.mins[2])) * cl.inv_h);
    if (fabs(fx) < kCellIndexMax && fabs(fy) < kCellIndexMax && fabs(fz) < kCellIndexMax) {
      const long long ix = (long long)fx, iy = (long long)fy, iz = (long long)fz;
      for (int t = 0; t < 27; ++t) {
        const unsigned int h = cl.base + cell_hash(ix + (t % 3) - 1, iy + ((t / 3) % 3) - 1, iz + (t / 9) - 1, cl.mask);
        const int e = a.bend[h];
        for (int k = a.bstart[h]; k < e; ++k) {
          const int j = a.sorted[k];
          const size_t o = 3 * (size_t)j;
          icp_keep(icp_d2(p, a.dst[o], a.dst[o + 1], a.dst[o + 2]), j - pr.d_lo, &best, &bj);
        }
      }
    } else {
      icp_nn_scan(a.dst, pr.d_lo, pr.nd, p, &best, &bj);
    }
  }
  const bool hit = query && bj != 0x7fffffff;
  if (have) a.match[pr.m_lo + i] = hit ? bj : -1;
  double v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (hit) {
    const size_t o = 3 * (size_t)(pr.d_lo + bj);
    v[0] = 1.0;
    v[1] = p[0];
    v[2] = p[1];
    v[3] = p[2];
    v[4] = a.dst[o];
    v[5] = a.dst[o + 1];
    v[6] = a.dst[o + 2];
    v[7] = best;
  }
  icp_block_sum<8>(v, s_buf, a.partial + 9 * (size_t)c);
}

__global__ void icp_eval_kernel(IcpArgs a, int max_iteration, double relative_fitness, double relative_rmse) {
  IcpProb& pr = a.probs[blockIdx.x];
  if (!pr.active) return;
  const int nc = (pr.ns + kIcpChunk - 1) / kIcpChunk;
  double v[8];
  icp_warp_combine<8>(a.partial, pr.c_lo, nc, v);
  if (threadIdx.x != 0) return;
  const int count = (int)v[0];
  const double fitness = count ? (double)count / (double)pr.ns : 0.0;
  const double rmse = count ? sqrt(v[7] / (double)count) : 0.0;
  if (pr.iterations > 0 && fabs(pr.fitness - fitness) < relative_fitness && fabs(pr.rmse - rmse) < relative_rmse)
    pr.converged = 1;
  if (pr.converged || pr.iterations >= max_iteration) pr.active = 0;
  pr.count = count;
  pr.fitness = fitness;
  pr.rmse = rmse;
  const double inv = count ? 1.0 / (double)count : 0.0;
  for (int k = 0; k < 3; ++k) {
    pr.mup[k] = v[1 + k] * inv;
    pr.muq[k] = v[4 + k] * inv;
  }
}

__global__ void __launch_bounds__(kIcpThreads) icp_cov_kernel(IcpArgs a) {
  __shared__ double s_buf[(kIcpThreads / 32) * 9];
  const int c = blockIdx.x;
  const int b = a.chunk_prob[c];
  const IcpProb& pr = a.probs[b];
  if (!pr.active || pr.count < 3) return;  // the update of fewer than 3 correspondences reads no covariance
  const int i = (c - pr.c_lo) * kIcpChunk + threadIdx.x;
  double h[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  const int j = i < pr.ns ? a.match[pr.m_lo + i] : -1;
  if (j >= 0) {
    double p[3];
    icp_transform(pr, a.src, pr.s_lo + i, p);
    const size_t o = 3 * (size_t)(pr.d_lo + j);
    const double u[3] = {p[0] - pr.mup[0], p[1] - pr.mup[1], p[2] - pr.mup[2]};
    const double w[3] = {(double)a.dst[o] - pr.muq[0], (double)a.dst[o + 1] - pr.muq[1],
                         (double)a.dst[o + 2] - pr.muq[2]};
#pragma unroll
    for (int cc = 0; cc < 3; ++cc)
#pragma unroll
      for (int r = 0; r < 3; ++r) h[3 * cc + r] = u[r] * w[cc];  // H(r, c) column-major
  }
  icp_block_sum<9>(h, s_buf, a.partial + 9 * (size_t)c);
}

// R <- Ru R, t <- Ru t + tu, and one more iteration (both update kernels)
__device__ __forceinline__ void icp_compose(IcpProb& pr, const M3& Ru, const double tu[3]) {
  double R[9], t[3];
  for (int r = 0; r < 3; ++r) {
    for (int cc = 0; cc < 3; ++cc)
      R[3 * cc + r] = (Ru(r, 0) * pr.R[3 * cc] + Ru(r, 1) * pr.R[3 * cc + 1]) + Ru(r, 2) * pr.R[3 * cc + 2];
    t[r] = ((Ru(r, 0) * pr.t[0] + Ru(r, 1) * pr.t[1]) + Ru(r, 2) * pr.t[2]) + tu[r];
  }
  for (int k = 0; k < 9; ++k) pr.R[k] = R[k];
  for (int k = 0; k < 3; ++k) pr.t[k] = t[k];
  pr.iterations += 1;
}

__global__ void icp_update_kernel(IcpArgs a) {
  IcpProb& pr = a.probs[blockIdx.x];
  if (!pr.active) return;
  const int nc = (pr.ns + kIcpChunk - 1) / kIcpChunk;
  double h[9];
  if (pr.count >= 3) icp_warp_combine<9>(a.partial, pr.c_lo, nc, h);
  if (threadIdx.x != 0) return;
  M3 Ru;
  m3_identity(Ru);
  double tu[3] = {0.0, 0.0, 0.0};
  if (pr.count >= 3) {
    M3 H;
    for (int k = 0; k < 9; ++k) H.a[k] = h[k];
    rotation_from_H(H, Ru);
    for (int r = 0; r < 3; ++r) tu[r] = pr.muq[r] - ((Ru(r, 0) * pr.mup[0] + Ru(r, 1) * pr.mup[1]) + Ru(r, 2) * pr.mup[2]);
  } else if (pr.count > 0) {
    for (int r = 0; r < 3; ++r) tu[r] = pr.muq[r] - pr.mup[r];
  }
  icp_compose(pr, Ru, tu);
}

// ---- robust kernels (DESIGN.md §3.15) ----------------------------------------------------------------------------------
// The weight rho'(r) / r of the kernel TZR_LOSS_* with parameter k, from e = |r| (include/teaser_b200.h writes out each
// one).  L1 at e = 0 gives +inf: the callers drop a correspondence whose weight is not finite.
__device__ __forceinline__ double icp_robust_weight(int loss, double k, double r) {
  const double e = fabs(r);
  if (loss == TZR_LOSS_L1) return 1.0 / e;
  if (loss == TZR_LOSS_HUBER) return k / fmax(e, k);
  if (loss == TZR_LOSS_CAUCHY) {
    const double q = e / k;
    return 1.0 / (1.0 + q * q);
  }
  if (loss == TZR_LOSS_GM) {
    const double t = k + e * e;
    return k / (t * t);
  }
  if (loss == TZR_LOSS_TUKEY) {
    if (e > k) return 0.0;
    const double q = e / k, t = 1.0 - q * q;
    return t * t;
  }
  return 1.0;
}

// ---- point-to-plane (DESIGN.md §3.13) ----------------------------------------------------------------------------------
// One CTA per chunk: each correspondence (i, j) whose target normal n has three finite components adds J J^T (the 21
// entries of the upper triangle, row by row) and J r (6), with u = p - c (c = mu_p of the current correspondences),
// J = (u x n, n) and r = ((p0 - q0) n0 + (p1 - q1) n1) + (p2 - q2) n2.  Flipping n negates J and r exactly, so the sums do
// not depend on the normal's sign.  The partials of this pass use 27 doubles per chunk; the nearest-neighbour pass that
// follows writes its 8 sums over them with stride 9 only after the update has read them.
// kRobust (DESIGN.md §3.15): the correspondence adds (w J_a) J_b and (w J_a) r with w = icp_robust_weight(loss, loss_k,
// r), and nothing when w is not finite.  The instance without it ignores loss and loss_k.
template <bool kRobust>
__global__ void __launch_bounds__(kIcpThreads) icp_plane_system_kernel(IcpArgs a, const float4* __restrict__ normals,
                                                                       int loss, double loss_k) {
  __shared__ double s_buf[(kIcpThreads / 32) * kIcpPlaneSums];
  const int c = blockIdx.x;
  const int b = a.chunk_prob[c];
  const IcpProb& pr = a.probs[b];
  if (!pr.active || pr.count == 0) return;  // the update of no correspondence reads no system
  const int i = (c - pr.c_lo) * kIcpChunk + threadIdx.x;
  double v[kIcpPlaneSums];
#pragma unroll
  for (int k = 0; k < kIcpPlaneSums; ++k) v[k] = 0.0;
  const int j = i < pr.ns ? a.match[pr.m_lo + i] : -1;
  if (j >= 0) {
    const float4 nf = normals[pr.n_lo + j];
    const double n[3] = {nf.x, nf.y, nf.z};
    if (isfinite(n[0]) && isfinite(n[1]) && isfinite(n[2])) {
      double p[3];
      icp_transform(pr, a.src, pr.s_lo + i, p);
      const size_t o = 3 * (size_t)(pr.d_lo + j);
      const double u[3] = {p[0] - pr.mup[0], p[1] - pr.mup[1], p[2] - pr.mup[2]};
      const double J[6] = {u[1] * n[2] - u[2] * n[1], u[2] * n[0] - u[0] * n[2], u[0] * n[1] - u[1] * n[0],
                           n[0], n[1], n[2]};
      const double r = ((p[0] - (double)a.dst[o]) * n[0] + (p[1] - (double)a.dst[o + 1]) * n[1]) +
                       (p[2] - (double)a.dst[o + 2]) * n[2];
      if constexpr (kRobust) {
        const double w = icp_robust_weight(loss, loss_k, r);
        if (isfinite(w)) {
          double wJ[6];
#pragma unroll
          for (int row = 0; row < 6; ++row) wJ[row] = w * J[row];
          int k = 0;
#pragma unroll
          for (int row = 0; row < 6; ++row)
#pragma unroll
            for (int col = row; col < 6; ++col) v[k++] = wJ[row] * J[col];
#pragma unroll
          for (int row = 0; row < 6; ++row) v[21 + row] = wJ[row] * r;
        }
      } else {
        int k = 0;
#pragma unroll
        for (int row = 0; row < 6; ++row)
#pragma unroll
          for (int col = row; col < 6; ++col) v[k++] = J[row] * J[col];
#pragma unroll
        for (int row = 0; row < 6; ++row) v[21 + row] = J[row] * r;
      }
    }
  }
  icp_block_sum<kIcpPlaneSums>(v, s_buf, a.partial + kIcpPlaneSums * (size_t)c);
}

// ---- generalized ICP (DESIGN.md §3.14) --------------------------------------------------------------------------------
// C(v) = I - (k v_a) v_b with k = (1 - eps) / ((v0 v0 + v1 v1) + v2 v2): the upper triangle (00, 01, 02, 11, 12, 22).
// Negating v negates k v_a and v_b, so the entries keep their bits.
__device__ __forceinline__ void gicp_cov(const double v[3], double k, double c[6]) {
  c[0] = 1.0 - (k * v[0]) * v[0];
  c[1] = 0.0 - (k * v[0]) * v[1];
  c[2] = 0.0 - (k * v[0]) * v[2];
  c[3] = 1.0 - (k * v[1]) * v[1];
  c[4] = 0.0 - (k * v[1]) * v[2];
  c[5] = 1.0 - (k * v[2]) * v[2];
}

// (v0 v0 + v1 v1) + v2 v2 of a normal with three finite components, or 0 (the correspondence adds nothing) otherwise
__device__ __forceinline__ double gicp_len2(const double v[3]) {
  if (!(isfinite(v[0]) && isfinite(v[1]) && isfinite(v[2]))) return 0.0;
  return (v[0] * v[0] + v[1] * v[1]) + v[2] * v[2];
}

// a x b
__device__ __forceinline__ void gicp_cross(const double a[3], const double b[3], double o[3]) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}

// S v for a symmetric S held as its upper triangle (00, 01, 02, 11, 12, 22), row r: (S(r,0) v0 + S(r,1) v1) + S(r,2) v2
__device__ __forceinline__ void gicp_symv(const double S[6], const double v[3], double o[3]) {
  o[0] = (S[0] * v[0] + S[1] * v[1]) + S[2] * v[2];
  o[1] = (S[1] * v[0] + S[3] * v[1]) + S[4] * v[2];
  o[2] = (S[2] * v[0] + S[4] * v[1]) + S[5] * v[2];
}

// The 27 sums of one correspondence: J^T A J (21 entries, the plane system's order) and J^T A d (6), with
// J = [e_k x u (k = 0..2), I], evaluated as include/teaser_b200.h writes them
__device__ __forceinline__ void gicp_add(const double A[6], const double u[3], const double d[3],
                                         double (&v)[kIcpPlaneSums]) {
  // ww[l] = u x A (e_l x u), wt[l] = u x A e_l: column l of the omega-omega and omega-tau blocks
  double ww[3][3], wt[3][3];
#pragma unroll
  for (int l = 0; l < 3; ++l) {
    const double e[3] = {l == 0 ? 1.0 : 0.0, l == 1 ? 1.0 : 0.0, l == 2 ? 1.0 : 0.0};
    double eu[3], Aeu[3], Ae[3];
    gicp_cross(e, u, eu);
    gicp_symv(A, eu, Aeu);
    gicp_cross(u, Aeu, ww[l]);
    Ae[0] = A[l == 0 ? 0 : l == 1 ? 1 : 2];
    Ae[1] = A[l == 0 ? 1 : l == 1 ? 3 : 4];
    Ae[2] = A[l == 0 ? 2 : l == 1 ? 4 : 5];
    gicp_cross(u, Ae, wt[l]);
  }
  int k = 0;
#pragma unroll
  for (int row = 0; row < 3; ++row) {
#pragma unroll
    for (int col = row; col < 3; ++col) v[k++] = ww[col][row];
#pragma unroll
    for (int col = 0; col < 3; ++col) v[k++] = wt[col][row];
  }
  v[k++] = A[0];
  v[k++] = A[1];
  v[k++] = A[2];
  v[k++] = A[3];
  v[k++] = A[4];
  v[k++] = A[5];
  double w[3], uw[3];
  gicp_symv(A, d, w);
  gicp_cross(u, w, uw);
  v[21] = uw[0];
  v[22] = uw[1];
  v[23] = uw[2];
  v[24] = w[0];
  v[25] = w[1];
  v[26] = w[2];
}

// The robust information matrix A~ = W diag(w) W (upper triangle) with W = M^-1/2 = V diag(1 / sqrt(sigma)) V^T from
// svd3 of the symmetric M (upper triangle) and w_k the weight of the whitened residual r_k = W_k . d (DESIGN.md §3.15,
// include/teaser_b200.h writes out every sum and its order).  False, and A~ unset, when some sigma is not > 0 or not
// finite, or some weight is not finite.
__device__ __forceinline__ bool gicp_robust_info(const double M[6], const double d[3], int loss, double loss_k,
                                                 double At[6]) {
  M3 H, U, V;
  H.a[0] = M[0];
  H.a[1] = M[1];
  H.a[2] = M[2];
  H.a[3] = M[1];
  H.a[4] = M[3];
  H.a[5] = M[4];
  H.a[6] = M[2];
  H.a[7] = M[4];
  H.a[8] = M[5];
  double S[3], q[3];
  svd3(H, U, S, V);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (!(S[k] > 0.0 && isfinite(S[k]))) return false;
    q[k] = 1.0 / sqrt(S[k]);
  }
  double W[3][3], w[3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c)
      W[r][c] = ((V(r, 0) * q[0]) * V(c, 0) + (V(r, 1) * q[1]) * V(c, 1)) + (V(r, 2) * q[2]) * V(c, 2);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    w[k] = icp_robust_weight(loss, loss_k, (W[k][0] * d[0] + W[k][1] * d[1]) + W[k][2] * d[2]);
    if (!isfinite(w[k])) return false;
  }
  int e = 0;
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = r; c < 3; ++c)
      At[e++] = ((w[0] * W[0][r]) * W[0][c] + (w[1] * W[1][r]) * W[1][c]) + (w[2] * W[2][r]) * W[2][c];
  return true;
}

// One CTA per chunk: each correspondence (i, j) whose source normal m and target normal n are finite and of non-zero
// length adds J^T A J (21 entries, the plane system's order) and J^T A d (6), with u = p - c, d = p - q,
// J = [e_k x u (k = 0..2), I] and A = (s^2 C(R m) + C(n))^-1 by the symmetric adjugate (include/teaser_b200.h writes
// out every formula and its order).  The 27 sums and their layout are the plane system's, so icp_plane_update_kernel
// solves them unchanged.
// kRobust (DESIGN.md §3.15): A~ of gicp_robust_info (loss, loss_k) in place of A, from the same M; the instance without
// it ignores loss and loss_k.
template <bool kRobust>
__global__ void __launch_bounds__(kIcpThreads) icp_gicp_system_kernel(IcpArgs a, const float4* __restrict__ src_normals,
                                                                      const float4* __restrict__ dst_normals,
                                                                      double epsilon, int loss, double loss_k) {
  __shared__ double s_buf[(kIcpThreads / 32) * kIcpPlaneSums];
  const int c = blockIdx.x;
  const int b = a.chunk_prob[c];
  const IcpProb& pr = a.probs[b];
  if (!pr.active || pr.count == 0) return;  // the update of no correspondence reads no system
  const int i = (c - pr.c_lo) * kIcpChunk + threadIdx.x;
  double v[kIcpPlaneSums];
#pragma unroll
  for (int k = 0; k < kIcpPlaneSums; ++k) v[k] = 0.0;
  const int j = i < pr.ns ? a.match[pr.m_lo + i] : -1;
  if (j >= 0) {
    const float4 mf = src_normals[pr.sn_lo + i], nf = dst_normals[pr.n_lo + j];
    const double m0[3] = {mf.x, mf.y, mf.z}, n[3] = {nf.x, nf.y, nf.z};
    const double lm = gicp_len2(m0), ln = gicp_len2(n);
    if (lm > 0.0 && ln > 0.0) {
      double m[3];  // R m, without the scale
#pragma unroll
      for (int r = 0; r < 3; ++r) m[r] = (pr.R[r] * m0[0] + pr.R[3 + r] * m0[1]) + pr.R[6 + r] * m0[2];
      double Cm[6], Cn[6], M[6];
      gicp_cov(m, (1.0 - epsilon) / ((m[0] * m[0] + m[1] * m[1]) + m[2] * m[2]), Cm);
      gicp_cov(n, (1.0 - epsilon) / ln, Cn);
      const double s2 = pr.s * pr.s;
#pragma unroll
      for (int k = 0; k < 6; ++k) M[k] = s2 * Cm[k] + Cn[k];
      if constexpr (kRobust) {
        double p[3];
        icp_transform(pr, a.src, pr.s_lo + i, p);
        const size_t o = 3 * (size_t)(pr.d_lo + j);
        const double d[3] = {p[0] - (double)a.dst[o], p[1] - (double)a.dst[o + 1], p[2] - (double)a.dst[o + 2]};
        double At[6];
        if (gicp_robust_info(M, d, loss, loss_k, At)) {
          const double u[3] = {p[0] - pr.mup[0], p[1] - pr.mup[1], p[2] - pr.mup[2]};
          gicp_add(At, u, d, v);
        }
      } else {
        // cofactors of M = [M0 M1 M2; M1 M3 M4; M2 M4 M5]
        const double c00 = M[3] * M[5] - M[4] * M[4], c01 = M[2] * M[4] - M[1] * M[5],
                     c02 = M[1] * M[4] - M[2] * M[3];
        const double c11 = M[0] * M[5] - M[2] * M[2], c12 = M[1] * M[2] - M[0] * M[4],
                     c22 = M[0] * M[3] - M[1] * M[1];
        const double det = (M[0] * c00 + M[1] * c01) + M[2] * c02;
        if (det > 0.0 && isfinite(det)) {
          const double A[6] = {c00 / det, c01 / det, c02 / det, c11 / det, c12 / det, c22 / det};
          double p[3];
          icp_transform(pr, a.src, pr.s_lo + i, p);
          const size_t o = 3 * (size_t)(pr.d_lo + j);
          const double u[3] = {p[0] - pr.mup[0], p[1] - pr.mup[1], p[2] - pr.mup[2]};
          const double d[3] = {p[0] - (double)a.dst[o], p[1] - (double)a.dst[o + 1], p[2] - (double)a.dst[o + 2]};
          // gicp_add written out: the form this instance has always had, so its code does not move
          double ww[3][3], wt[3][3];
#pragma unroll
          for (int l = 0; l < 3; ++l) {
            const double e[3] = {l == 0 ? 1.0 : 0.0, l == 1 ? 1.0 : 0.0, l == 2 ? 1.0 : 0.0};
            double eu[3], Aeu[3], Ae[3];
            gicp_cross(e, u, eu);
            gicp_symv(A, eu, Aeu);
            gicp_cross(u, Aeu, ww[l]);
            Ae[0] = A[l == 0 ? 0 : l == 1 ? 1 : 2];
            Ae[1] = A[l == 0 ? 1 : l == 1 ? 3 : 4];
            Ae[2] = A[l == 0 ? 2 : l == 1 ? 4 : 5];
            gicp_cross(u, Ae, wt[l]);
          }
          int k = 0;
#pragma unroll
          for (int row = 0; row < 3; ++row) {
#pragma unroll
            for (int col = row; col < 3; ++col) v[k++] = ww[col][row];
#pragma unroll
            for (int col = 0; col < 3; ++col) v[k++] = wt[col][row];
          }
          v[k++] = A[0];
          v[k++] = A[1];
          v[k++] = A[2];
          v[k++] = A[3];
          v[k++] = A[4];
          v[k++] = A[5];
          double w[3], uw[3];
          gicp_symv(A, d, w);
          gicp_cross(u, w, uw);
          v[21] = uw[0];
          v[22] = uw[1];
          v[23] = uw[2];
          v[24] = w[0];
          v[25] = w[1];
          v[26] = w[2];
        }
      }
    }
  }
  icp_block_sum<kIcpPlaneSums>(v, s_buf, a.partial + kIcpPlaneSums * (size_t)c);
}

// ---- coloured ICP (DESIGN.md §3.17) ---------------------------------------------------------------------------------
// The terms of one row (J, r) with weight w (kRobust) into v: (w J_a) J_b (21) and (w J_a) r (6); without kRobust J_a J_b
// and J_a r, point-to-plane's unweighted products.  add: v += the terms, else v = the terms.
template <bool kRobust>
__device__ __forceinline__ void icp_row_terms(const double J[6], double r, double w, bool add,
                                              double (&v)[kIcpPlaneSums]) {
  double wJ[6];
#pragma unroll
  for (int row = 0; row < 6; ++row) wJ[row] = kRobust ? w * J[row] : J[row];
  int k = 0;
#pragma unroll
  for (int row = 0; row < 6; ++row)
#pragma unroll
    for (int col = row; col < 6; ++col) {
      const double t = wJ[row] * J[col];
      v[k] = add ? v[k] + t : t;
      ++k;
    }
#pragma unroll
  for (int row = 0; row < 6; ++row) v[21 + row] = add ? v[21 + row] + wJ[row] * r : wJ[row] * r;
}

// One CTA per chunk: each correspondence (i, j) whose target normal n has three finite components adds a geometric row
// J_G = sqrt(lambda) (u x n, n), r_G = sqrt(lambda) r (r: point-to-plane's residual) and then a photometric row
// J_I = sqrt(1 - lambda) (u x m, m), r_I = sqrt(1 - lambda) (i_s - i_hat) with m = -(I - n n^T) g, g the target's
// colour gradient and i_hat = g . (p - s n - q) + i_t (include/teaser_b200.h writes out every expression and its
// order).  A row adds nothing when its factor is 0 or its weight is not finite; the photometric row adds nothing when
// a colour or g has a non-finite component.  The 27 sums and their layout are the plane system's, so
// icp_plane_update_kernel solves them unchanged; with lambda = 1 they are icp_plane_system_kernel's bit for bit.
// kRobust (DESIGN.md §3.15): each row has its own weight, icp_robust_weight(loss, loss_k, r_row).
template <bool kRobust>
__global__ void __launch_bounds__(kIcpThreads) icp_colored_system_kernel(IcpArgs a, const float4* __restrict__ normals,
                                                                         const float* __restrict__ src_colors,
                                                                         const float* __restrict__ dst_colors,
                                                                         const double* __restrict__ grad,
                                                                         double lambda, int loss, double loss_k) {
  __shared__ double s_buf[(kIcpThreads / 32) * kIcpPlaneSums];
  const int c = blockIdx.x;
  const int b = a.chunk_prob[c];
  const IcpProb& pr = a.probs[b];
  if (!pr.active || pr.count == 0) return;  // the update of no correspondence reads no system
  const int i = (c - pr.c_lo) * kIcpChunk + threadIdx.x;
  double v[kIcpPlaneSums];
#pragma unroll
  for (int k = 0; k < kIcpPlaneSums; ++k) v[k] = 0.0;
  const int j = i < pr.ns ? a.match[pr.m_lo + i] : -1;
  if (j >= 0) {
    const float4 nf = normals[pr.n_lo + j];
    const double n[3] = {nf.x, nf.y, nf.z};
    if (isfinite(n[0]) && isfinite(n[1]) && isfinite(n[2])) {
      const double sg = sqrt(lambda), si = sqrt(1.0 - lambda);
      double p[3];
      icp_transform(pr, a.src, pr.s_lo + i, p);
      const size_t o = 3 * (size_t)(pr.d_lo + j);
      const double q[3] = {a.dst[o], a.dst[o + 1], a.dst[o + 2]};
      const double u[3] = {p[0] - pr.mup[0], p[1] - pr.mup[1], p[2] - pr.mup[2]};
      const double r = ((p[0] - q[0]) * n[0] + (p[1] - q[1]) * n[1]) + (p[2] - q[2]) * n[2];
      bool any = false;
      if (sg != 0.0) {
        const double J[6] = {sg * (u[1] * n[2] - u[2] * n[1]), sg * (u[2] * n[0] - u[0] * n[2]),
                             sg * (u[0] * n[1] - u[1] * n[0]), sg * n[0], sg * n[1], sg * n[2]};
        const double rg = sg * r;
        const double w = kRobust ? icp_robust_weight(loss, loss_k, rg) : 1.0;
        if (isfinite(w)) {
          icp_row_terms<kRobust>(J, rg, w, false, v);
          any = true;
        }
      }
      const size_t ks = (size_t)(pr.s_lo + i), kt = (size_t)(pr.d_lo + j), kg = 3 * (size_t)(pr.n_lo + j);
      const double g[3] = {grad[kg], grad[kg + 1], grad[kg + 2]};
      const double cs[3] = {src_colors[3 * ks], src_colors[3 * ks + 1], src_colors[3 * ks + 2]};
      const double ct[3] = {dst_colors[3 * kt], dst_colors[3 * kt + 1], dst_colors[3 * kt + 2]};
      bool fin = true;
#pragma unroll
      for (int k = 0; k < 3; ++k) fin &= isfinite(g[k]) && isfinite(cs[k]) && isfinite(ct[k]);
      if (si != 0.0 && fin) {
        const double is = ((cs[0] + cs[1]) + cs[2]) / 3.0, it = ((ct[0] + ct[1]) + ct[2]) / 3.0;
        const double d[3] = {(p[0] - r * n[0]) - q[0], (p[1] - r * n[1]) - q[1], (p[2] - r * n[2]) - q[2]};
        const double ihat = ((g[0] * d[0] + g[1] * d[1]) + g[2] * d[2]) + it;
        double m[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double M0 = (k == 0 ? 1.0 : 0.0) - n[0] * n[k], M1 = (k == 1 ? 1.0 : 0.0) - n[1] * n[k],
                       M2 = (k == 2 ? 1.0 : 0.0) - n[2] * n[k];
          m[k] = -((g[0] * M0 + g[1] * M1) + g[2] * M2);
        }
        const double J[6] = {si * (u[1] * m[2] - u[2] * m[1]), si * (u[2] * m[0] - u[0] * m[2]),
                             si * (u[0] * m[1] - u[1] * m[0]), si * m[0], si * m[1], si * m[2]};
        const double ri = si * (is - ihat);
        const double w = kRobust ? icp_robust_weight(loss, loss_k, ri) : 1.0;
        if (isfinite(w)) icp_row_terms<kRobust>(J, ri, w, any, v);
      }
    }
  }
  icp_block_sum<kIcpPlaneSums>(v, s_buf, a.partial + kIcpPlaneSums * (size_t)c);
}

__global__ void icp_plane_update_kernel(IcpArgs a) {
  IcpProb& pr = a.probs[blockIdx.x];
  if (!pr.active) return;
  const int nc = (pr.ns + kIcpChunk - 1) / kIcpChunk;
  double v[kIcpPlaneSums];
  if (pr.count > 0) icp_warp_combine<kIcpPlaneSums, kIcpPlaneSums>(a.partial, pr.c_lo, nc, v);
  if (threadIdx.x != 0) return;
  M3 Ru;
  m3_identity(Ru);
  double tu[3] = {0.0, 0.0, 0.0};
  if (pr.count > 0) {
    double x[6];
    ldlt_solve<6>(v, v + 21, x);
    bool finite = true;
    for (int k = 0; k < 6; ++k) finite &= isfinite(x[k]) != 0;
    if (finite) {
      // Ru = Rz(x2) Ry(x1) Rx(x0)
      double sa, ca, sb, cb, sg, cg;
      sincos(x[0], &sa, &ca);
      sincos(x[1], &sb, &cb);
      sincos(x[2], &sg, &cg);
      Ru(0, 0) = cg * cb;
      Ru(0, 1) = (cg * sb) * sa - sg * ca;
      Ru(0, 2) = (cg * sb) * ca + sg * sa;
      Ru(1, 0) = sg * cb;
      Ru(1, 1) = (sg * sb) * sa + cg * ca;
      Ru(1, 2) = (sg * sb) * ca - cg * sa;
      Ru(2, 0) = -sb;
      Ru(2, 1) = cb * sa;
      Ru(2, 2) = cb * ca;
      for (int r = 0; r < 3; ++r)
        tu[r] = (pr.mup[r] + x[3 + r]) - ((Ru(r, 0) * pr.mup[0] + Ru(r, 1) * pr.mup[1]) + Ru(r, 2) * pr.mup[2]);
    }
  }
  icp_compose(pr, Ru, tu);
}

__global__ void icp_seed_kernel(IcpProb* probs, int B, const tzr_solution* __restrict__ sol) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const tzr_solution& s = sol[b];
  IcpProb& pr = probs[b];
  bool ok = s.valid && isfinite(s.scale) && s.scale > 0.0;
  for (int k = 0; k < 9; ++k) ok &= isfinite(s.rotation[k]) != 0;
  for (int k = 0; k < 3; ++k) ok &= isfinite(s.translation[k]) != 0;
  pr.active = pr.seeded = ok ? 1 : 0;
  if (!ok) return;
  pr.s = s.scale;
  for (int k = 0; k < 9; ++k) pr.R[k] = s.rotation[k];
  for (int k = 0; k < 3; ++k) pr.t[k] = s.translation[k];
}

// ---- information matrices (DESIGN.md §3.16) -----------------------------------------------------------------------
// Open3D's GetInformationMatrixFromPointClouds: one CTA per chunk; each correspondence (i, j) of the stored matches adds
// G^T G with q = y_j (the target point) and G = [-[q]x | I] (3 x 6, ordering (omega, tau)), its 21 upper entries row by
// row, each ((G(0,a) G(0,b) + G(1,a) G(1,b)) + G(2,a) G(2,b)).  Entry 20 (Lambda(5,5)) is the correspondence count.
// A problem that was not seeded (a chained pair without a valid record) adds nothing.
__global__ void __launch_bounds__(kIcpThreads) icp_info_kernel(IcpArgs a) {
  __shared__ double s_buf[(kIcpThreads / 32) * kIcpInfoSums];
  const int c = blockIdx.x;
  const IcpProb& pr = a.probs[a.chunk_prob[c]];
  if (!pr.seeded) return;
  const int i = (c - pr.c_lo) * kIcpChunk + threadIdx.x;
  double v[kIcpInfoSums];
#pragma unroll
  for (int k = 0; k < kIcpInfoSums; ++k) v[k] = 0.0;
  const int j = i < pr.ns ? a.match[pr.m_lo + i] : -1;
  if (j >= 0) {
    const size_t o = 3 * (size_t)(pr.d_lo + j);
    const double x = a.dst[o], y = a.dst[o + 1], z = a.dst[o + 2];
    const double G[3][6] = {{0.0, z, -y, 1.0, 0.0, 0.0}, {-z, 0.0, x, 0.0, 1.0, 0.0}, {y, -x, 0.0, 0.0, 0.0, 1.0}};
    int k = 0;
#pragma unroll
    for (int row = 0; row < 6; ++row)
#pragma unroll
      for (int col = row; col < 6; ++col)
        v[k++] = (G[0][row] * G[0][col] + G[1][row] * G[1][col]) + G[2][row] * G[2][col];
  }
  icp_block_sum<kIcpInfoSums>(v, s_buf, a.partial + kIcpInfoSums * (size_t)c);
}

// One warp per problem: the chunk sums in ICP's fixed order, mirrored into 36 doubles (row-major, symmetric), and the
// count; zeros for a problem that was not seeded
__global__ void icp_info_combine_kernel(IcpArgs a, double* __restrict__ info, int* __restrict__ counts) {
  const IcpProb& pr = a.probs[blockIdx.x];
  double v[kIcpInfoSums];
  if (pr.seeded) {
    icp_warp_combine<kIcpInfoSums, kIcpInfoSums>(a.partial, pr.c_lo, (pr.ns + kIcpChunk - 1) / kIcpChunk, v);
  } else {
#pragma unroll
    for (int k = 0; k < kIcpInfoSums; ++k) v[k] = 0.0;
  }
  if (threadIdx.x != 0) return;
  double* L = info + 36 * (size_t)blockIdx.x;
  int k = 0;
  for (int row = 0; row < 6; ++row)
    for (int col = row; col < 6; ++col) {
      L[6 * row + col] = v[k];
      L[6 * col + row] = v[k];
      ++k;
    }
  counts[blockIdx.x] = (int)v[kIcpInfoSums - 1];
}

// a chained call's problems run their search once more after ICP finished them: active again where seeded
__global__ void icp_info_seed_kernel(IcpProb* probs, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) probs[b].active = probs[b].seeded;
}

// ---- multi-scale schedule (DESIGN.md §3.19) ---------------------------------------------------------------------------
// Problem b of a scale starts from the pose of its pair pair_of[b]: the seed, or the pair's transform after the previous
// scale.  Sets active = seeded = 1.
__global__ void icp_pose_load_kernel(IcpProb* probs, int B, const int* __restrict__ pair_of,
                                     const tzr_similarity* __restrict__ pose) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const tzr_similarity& x = pose[pair_of[b]];
  IcpProb& pr = probs[b];
  pr.active = pr.seeded = 1;
  pr.s = x.scale;
  for (int k = 0; k < 9; ++k) pr.R[k] = x.rotation[k];
  for (int k = 0; k < 3; ++k) pr.t[k] = x.translation[k];
}

// Pair p's record of a scale at rec[p * stride]: a refined pair (prob_of[p] >= 0) gets its problem's result, whose
// transform also becomes the pair's pose; any other pair carries its pose with every other field 0
__global__ void icp_pose_store_kernel(const IcpProb* __restrict__ probs, int P, const int* __restrict__ prob_of,
                                      tzr_similarity* __restrict__ pose, tzr_icp_result* __restrict__ rec, int stride) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  tzr_similarity& x = pose[p];
  tzr_icp_result r;
  r.fitness = r.inlier_rmse = 0.0;
  r.iterations = r.n_correspondences = r.converged = r.reserved = 0;
  const int k = prob_of[p];
  if (k >= 0) {
    const IcpProb& pr = probs[k];
    x.scale = pr.s;
    for (int q = 0; q < 9; ++q) x.rotation[q] = pr.R[q];
    for (int q = 0; q < 3; ++q) x.translation[q] = pr.t[q];
    r.fitness = pr.fitness;
    r.inlier_rmse = pr.rmse;
    r.iterations = pr.iterations;
    r.n_correspondences = pr.count;
    r.converged = pr.converged;
  }
  r.transform = x;
  rec[(size_t)p * stride] = r;
}

}  // namespace

int launch_icp_pose_load(IcpProb* probs, int B, const int* pair_of, const tzr_similarity* pose, cudaStream_t st) {
  icp_pose_load_kernel<<<(B + 127) / 128, 128, 0, st>>>(probs, B, pair_of, pose);
  return 1;
}

int launch_icp_pose_store(const IcpProb* probs, int P, const int* prob_of, tzr_similarity* pose, tzr_icp_result* rec,
                          int stride, cudaStream_t st) {
  icp_pose_store_kernel<<<(P + 127) / 128, 128, 0, st>>>(probs, P, prob_of, pose, rec, stride);
  return 1;
}

int icp_plan(int B, const int32_t* ns, const int32_t* s_lo, const int32_t* tc, int T, const int32_t* nt, double r,
             int route, const tzr_similarity* init, IcpPlan* plan, std::vector<FpfhCloud>* clouds,
             std::vector<IcpProb>* probs, std::vector<int>* chunk_prob) {
  long long NS = 0, chunks = 0;
  for (int b = 0; b < B; ++b) {
    NS += ns[b];
    chunks += (ns[b] + kIcpChunk - 1) / kIcpChunk;
  }
  clouds->resize((size_t)T);
  if (NS > 0x7fffffffll || fpfh_plan(T, nt, r, r, route, clouds->data(), &plan->grid, kIcpGridMinN) != TZR_OK)
    return TZR_ERR_TOO_LARGE;
  plan->B = B;
  plan->NS = (int)NS;
  plan->ND = plan->grid.N;
  plan->chunks = (int)chunks;
  plan->r2 = r * r;
  probs->assign((size_t)B, IcpProb{});
  chunk_prob->resize((size_t)chunks);
  int m_lo = 0, c_lo = 0;
  for (int b = 0; b < B; ++b) {
    IcpProb& pr = (*probs)[b];
    const FpfhCloud& t = (*clouds)[tc ? tc[b] : b];
    pr.s_lo = s_lo ? s_lo[b] : m_lo;
    pr.ns = ns[b];
    pr.d_lo = t.lo;
    pr.nd = t.n;
    pr.c_lo = c_lo;
    pr.m_lo = m_lo;
    pr.tc = tc ? tc[b] : b;
    pr.n_lo = t.lo;
    pr.sn_lo = pr.s_lo;
    if (init) {
      pr.active = pr.seeded = 1;
      pr.s = init[b].scale;
      for (int k = 0; k < 9; ++k) pr.R[k] = init[b].rotation[k];
      for (int k = 0; k < 3; ++k) pr.t[k] = init[b].translation[k];
    }
    const int nc = (ns[b] + kIcpChunk - 1) / kIcpChunk;
    for (int c = 0; c < nc; ++c) (*chunk_prob)[c_lo + c] = b;
    m_lo += ns[b];
    c_lo += nc;
  }
  return TZR_OK;
}

IcpLayout icp_layout(const IcpPlan& plan, size_t base, bool information) {
  const int stride = std::max(icp_partial_stride(plan.mode), information ? kIcpInfoSums : 0);
  IcpLayout L;
  L.probs = base;
  L.clouds = L.probs + al256((size_t)plan.B * sizeof(IcpProb));
  L.chunks = L.clouds + al256((size_t)plan.grid.B * sizeof(FpfhCloud));
  L.match = L.chunks + al256((size_t)plan.chunks * 4);
  L.partial = L.match + al256((size_t)plan.NS * 4);
  L.grid = L.partial + al256((size_t)plan.chunks * stride * 8);
  const bool colored = plan.mode == kIcpColored;
  const size_t grid_bytes = colored ? std::max(plan.grid.grid_bytes, plan.ggrid.grid_bytes) : plan.grid.grid_bytes;
  L.info = L.counts = L.end = L.grid + grid_bytes;
  if (information) {
    L.info = al256(L.end);
    L.counts = L.info + al256((size_t)plan.B * 36 * 8);
    L.end = L.counts + (size_t)plan.B * 4;
  }
  L.gclouds = L.grad = L.end;
  if (colored) {
    L.gclouds = al256(L.end);
    L.grad = L.gclouds + al256((size_t)plan.ggrid.B * sizeof(FpfhCloud));
    L.end = L.grad + (size_t)plan.ND * 3 * 8;
  }
  return L;
}

IcpBuffers icp_buffers(char* d, const IcpLayout& L) {
  IcpBuffers b{nullptr, nullptr, nullptr, nullptr, (IcpProb*)(d + L.probs), (FpfhCloud*)(d + L.clouds),
               (const int*)(d + L.chunks), (int*)(d + L.match), (double*)(d + L.partial), d + L.grid,
               (double*)(d + L.info), (int*)(d + L.counts), nullptr, nullptr, nullptr, nullptr};
  if (L.grad != L.end) {
    b.gclouds = (FpfhCloud*)(d + L.gclouds);
    b.grad = (double*)(d + L.grad);
  }
  return b;
}

int launch_icp_information(const IcpPlan& plan, const IcpBuffers& buf, bool reseed, cudaStream_t st,
                           const IcpGrid* grid) {
  int nl = 0;
  IcpArgs a{buf.src, buf.dst, buf.probs, buf.clouds, buf.chunk_prob, buf.match, buf.partial, nullptr, nullptr, nullptr,
            plan.r2};
  if (reseed) {
    icp_info_seed_kernel<<<(plan.B + 127) / 128, 128, 0, st>>>(buf.probs, plan.B);
    ++nl;
  }
  if (grid) {  // launch_icp's grid over the same targets, still in grid_scratch
    a.sorted = grid->sorted;
    a.bstart = grid->bstart;
    a.bend = grid->bend;
  } else if (plan.grid.any_grid) {
    nl += launch_fpfh_grid(plan.grid, buf.dst, buf.clouds, buf.grid_scratch, st, &a.sorted, &a.bstart, &a.bend);
  }
  icp_nn_kernel<<<plan.chunks, kIcpThreads, 0, st>>>(a);
  icp_info_kernel<<<plan.chunks, kIcpThreads, 0, st>>>(a);
  icp_info_combine_kernel<<<plan.B, 32, 0, st>>>(a, buf.info, buf.counts);
  return nl + 3;
}

int launch_icp_seed(IcpProb* probs, int B, const tzr_solution* sol, cudaStream_t st) {
  icp_seed_kernel<<<(B + 127) / 128, 128, 0, st>>>(probs, B, sol);
  return 1;
}

int launch_icp(const IcpPlan& plan, const IcpBuffers& buf, cudaStream_t st, IcpGrid* grid_out) {
  int nl = 0;
  IcpArgs a{buf.src, buf.dst, buf.probs, buf.clouds, buf.chunk_prob, buf.match, buf.partial, nullptr, nullptr, nullptr,
            plan.r2};
  if (plan.mode == kIcpColored)  // the targets' gradients, before ICP's own grid reuses the scratch
    nl += launch_color_gradients(plan.ggrid, buf.dst, buf.gclouds, plan.grad_r, buf.dst_normals, buf.dst_colors,
                                 buf.grad, buf.grid_scratch, st);
  if (plan.grid.any_grid)
    nl += launch_fpfh_grid(plan.grid, buf.dst, buf.clouds, buf.grid_scratch, st, &a.sorted, &a.bstart, &a.bend);
  if (grid_out) *grid_out = IcpGrid{a.sorted, a.bstart, a.bend};
  icp_nn_kernel<<<plan.chunks, kIcpThreads, 0, st>>>(a);
  icp_eval_kernel<<<plan.B, 32, 0, st>>>(a, plan.max_iteration, plan.relative_fitness, plan.relative_rmse);
  nl += 2;
  for (int it = 0; it < plan.max_iteration; ++it) {
    if (plan.mode == kIcpPointToPlane) {
      if (plan.loss == TZR_LOSS_L2)
        icp_plane_system_kernel<false><<<plan.chunks, kIcpThreads, 0, st>>>(a, buf.dst_normals, 0, 0.0);
      else
        icp_plane_system_kernel<true><<<plan.chunks, kIcpThreads, 0, st>>>(a, buf.dst_normals, plan.loss,
                                                                           plan.loss_k);
      icp_plane_update_kernel<<<plan.B, 32, 0, st>>>(a);
    } else if (plan.mode == kIcpGeneralized) {
      if (plan.loss == TZR_LOSS_L2)
        icp_gicp_system_kernel<false><<<plan.chunks, kIcpThreads, 0, st>>>(a, buf.src_normals, buf.dst_normals,
                                                                           plan.epsilon, 0, 0.0);
      else
        icp_gicp_system_kernel<true><<<plan.chunks, kIcpThreads, 0, st>>>(a, buf.src_normals, buf.dst_normals,
                                                                          plan.epsilon, plan.loss, plan.loss_k);
      icp_plane_update_kernel<<<plan.B, 32, 0, st>>>(a);
    } else if (plan.mode == kIcpColored) {
      if (plan.loss == TZR_LOSS_L2)
        icp_colored_system_kernel<false><<<plan.chunks, kIcpThreads, 0, st>>>(
            a, buf.dst_normals, buf.src_colors, buf.dst_colors, buf.grad, plan.lambda_geometric, 0, 0.0);
      else
        icp_colored_system_kernel<true><<<plan.chunks, kIcpThreads, 0, st>>>(
            a, buf.dst_normals, buf.src_colors, buf.dst_colors, buf.grad, plan.lambda_geometric, plan.loss,
            plan.loss_k);
      icp_plane_update_kernel<<<plan.B, 32, 0, st>>>(a);
    } else {
      icp_cov_kernel<<<plan.chunks, kIcpThreads, 0, st>>>(a);
      icp_update_kernel<<<plan.B, 32, 0, st>>>(a);
    }
    icp_nn_kernel<<<plan.chunks, kIcpThreads, 0, st>>>(a);
    icp_eval_kernel<<<plan.B, 32, 0, st>>>(a, plan.max_iteration, plan.relative_fitness, plan.relative_rmse);
    nl += 4;
  }
  return nl;
}

}  // namespace tzr
