// Fast Global Registration (Zhou, Park and Koltun, ECCV 2016; Open3D's FastGlobalRegistration, DESIGN.md §3.20): the
// normalisation and the Geman-McClure Gauss-Newton loop of B problems, written out as this project's own definition in
// include/teaser_b200.h.  The evaluation is ICP's (launch_icp with max_iteration = 0), seeded by fgr_kernel.
//
//   fgr_prep_kernel  one CTA per problem: the means of both clouds' finite points (fixed-order sums), sigma (a max, exact
//                    in any order), scale_global and mu_start, then the usable correspondences compacted in input order
//                    and written once as float64 rows (p, q) of the normalised frame.
//   fgr_kernel       one CTA per problem, every iteration inside it: each thread sums the 27 terms of the weighted 6 x 6
//                    system over rows l, l + 256, ... of its problem, a fixed-order block sum, the solve and the update
//                    on one thread, T broadcast through shared memory; then the result in the input frame, into the
//                    FGR table and the ICP problem that evaluates it.
//
// The order of every sum depends only on the problem's own clouds and rows (and the fixed block size), so a problem's bits
// do not depend on the batch it runs in.  The rows are read from global memory on every iteration (not staged in shared
// memory): DESIGN.md §3.20 records the measurements behind that choice.
#include "tzr_internal.cuh"

namespace tzr {

namespace {

constexpr int kFgrThreads = kIcpChunk;  // icp_block_sum's block

struct FgrArgs {
  const float* src;
  const float* dst;
  IcpProb* icp;
  FgrProb* probs;
  const int2* corr;
  double* pq;
  double division_factor, max_dist;
  int use_absolute_scale, decrease_mu, iteration_number;
};

__device__ __forceinline__ bool fgr_finite(double x, double y, double z) {
  return isfinite(x) && isfinite(y) && isfinite(z);
}

// mean of the finite points of pts[lo, lo + n) into m[0..3) (every thread); NaN without a finite point
__device__ void fgr_mean(const float* __restrict__ pts, int lo, int n, double* s_buf, double* s_sum, double m[3]) {
  double v[4] = {0.0, 0.0, 0.0, 0.0};
  for (int i = threadIdx.x; i < n; i += kFgrThreads) {
    const size_t o = 3 * (size_t)(lo + i);
    const double x = pts[o], y = pts[o + 1], z = pts[o + 2];
    if (fgr_finite(x, y, z)) {
      v[0] += x;
      v[1] += y;
      v[2] += z;
      v[3] += 1.0;
    }
  }
  icp_block_sum<4>(v, s_buf, s_sum);
  __syncthreads();
  for (int k = 0; k < 3; ++k) m[k] = s_sum[k] / s_sum[3];
  __syncthreads();  // s_sum and s_buf are reused
}

// this thread's largest ||x - m|| over its finite points of pts[lo, lo + n) (0 without one)
__device__ double fgr_radius(const float* __restrict__ pts, int lo, int n, const double m[3]) {
  double r = 0.0;
  for (int i = threadIdx.x; i < n; i += kFgrThreads) {
    const size_t o = 3 * (size_t)(lo + i);
    const double x = pts[o], y = pts[o + 1], z = pts[o + 2];
    if (!fgr_finite(x, y, z)) continue;
    const double dx = x - m[0], dy = y - m[1], dz = z - m[2];
    r = fmax(r, sqrt((dx * dx + dy * dy) + dz * dz));
  }
  return r;
}

__global__ void __launch_bounds__(kFgrThreads) fgr_prep_kernel(FgrArgs a) {
  __shared__ double s_buf[(kFgrThreads / 32) * 4];
  __shared__ double s_sum[4];
  __shared__ double s_max[kFgrThreads / 32];
  __shared__ int s_cnt[kFgrThreads / 32];
  const int b = blockIdx.x;
  const IcpProb& ip = a.icp[b];
  FgrProb& fp = a.probs[b];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double ms[3], mt[3];
  fgr_mean(a.src, ip.s_lo, ip.ns, s_buf, s_sum, ms);
  fgr_mean(a.dst, ip.d_lo, ip.nd, s_buf, s_sum, mt);
  double r = fmax(fgr_radius(a.src, ip.s_lo, ip.ns, ms), fgr_radius(a.dst, ip.d_lo, ip.nd, mt));
  for (int o = 16; o; o >>= 1) r = fmax(r, __shfl_xor_sync(0xffffffffu, r, o));
  if (lane == 0) s_max[w] = r;
  __syncthreads();
  double sigma = 0.0;
  for (int q = 0; q < kFgrThreads / 32; ++q) sigma = fmax(sigma, s_max[q]);
  const double sg = a.use_absolute_scale || sigma == 0.0 ? 1.0 : sigma;
  // the usable rows, in input order: a block-wide exclusive scan of the flags per round of 256 rows
  const int2* corr = a.corr + fp.c_lo;
  double* pq = a.pq + 6 * fp.c_lo;
  const int K = fp.K;
  int kv = 0;
  for (int k0 = 0; k0 < K; k0 += kFgrThreads) {
    const int k = k0 + threadIdx.x;
    double p[3] = {0.0, 0.0, 0.0}, q[3] = {0.0, 0.0, 0.0};
    bool ok = false;
    if (k < K) {
      const int2 c = corr[k];
      const size_t os = 3 * (size_t)(ip.s_lo + c.x), od = 3 * (size_t)(ip.d_lo + c.y);
      const double x[3] = {a.src[os], a.src[os + 1], a.src[os + 2]};
      const double y[3] = {a.dst[od], a.dst[od + 1], a.dst[od + 2]};
      ok = fgr_finite(x[0], x[1], x[2]) && fgr_finite(y[0], y[1], y[2]);
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        p[d] = (x[d] - ms[d]) / sg;
        q[d] = (y[d] - mt[d]) / sg;
      }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) s_cnt[w] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
    for (int q2 = 0; q2 < kFgrThreads / 32; ++q2) {
      before += q2 < w ? s_cnt[q2] : 0;
      total += s_cnt[q2];
    }
    if (ok) {
      double* row = pq + 6 * (size_t)(kv + before + __popc(bal & ((1u << lane) - 1u)));
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        row[d] = p[d];
        row[3 + d] = q[d];
      }
    }
    kv += total;
    __syncthreads();  // s_cnt is rewritten by the next round
  }
  if (threadIdx.x == 0) {
    fp.Kv = kv;
    fp.scale_global = sg;
    fp.mu0 = a.use_absolute_scale ? sigma : 1.0;
    fp.sigma = sigma;
    for (int d = 0; d < 3; ++d) {
      fp.mean_s[d] = ms[d];
      fp.mean_t[d] = mt[d];
    }
  }
}

__global__ void __launch_bounds__(kFgrThreads) fgr_kernel(FgrArgs a) {
  __shared__ double s_buf[(kFgrThreads / 32) * kIcpPlaneSums];
  __shared__ double s_sum[kIcpPlaneSums];
  __shared__ double s_T[12];  // R (column-major), t
  const int b = blockIdx.x;
  FgrProb& fp = a.probs[b];
  const int K = fp.Kv;
  const bool run = K >= kFgrMinCorr && a.iteration_number > 0;
  if (threadIdx.x < 12) s_T[threadIdx.x] = threadIdx.x == 0 || threadIdx.x == 4 || threadIdx.x == 8 ? 1.0 : 0.0;
  __syncthreads();
  const double* pq = a.pq + 6 * fp.c_lo;
  double mu = fp.mu0;
  for (int itr = 0; run && itr < a.iteration_number; ++itr) {
    if (a.decrease_mu && itr % 4 == 0 && mu > a.max_dist) mu = mu / a.division_factor;
    double R[9], t[3];
#pragma unroll
    for (int k = 0; k < 9; ++k) R[k] = s_T[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) t[k] = s_T[9 + k];
    double v[kIcpPlaneSums];
#pragma unroll
    for (int k = 0; k < kIcpPlaneSums; ++k) v[k] = 0.0;
    for (int k = threadIdx.x; k < K; k += kFgrThreads) {
      const double* row = pq + 6 * (size_t)k;
      double qq[3], r[3];
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        qq[d] = ((R[d] * row[3] + R[3 + d] * row[4]) + R[6 + d] * row[5]) + t[d];
        r[d] = row[d] - qq[d];
      }
      double w = mu / (((r[0] * r[0] + r[1] * r[1]) + r[2] * r[2]) + mu);
      w = w * w;
      const double Jx[6] = {0.0, -qq[2], qq[1], -1.0, 0.0, 0.0};
      const double Jy[6] = {qq[2], 0.0, -qq[0], 0.0, -1.0, 0.0};
      const double Jz[6] = {-qq[1], qq[0], 0.0, 0.0, 0.0, -1.0};
      icp_row_terms<true>(Jx, r[0], w, true, v);
      icp_row_terms<true>(Jy, r[1], w, true, v);
      icp_row_terms<true>(Jz, r[2], w, true, v);
    }
    icp_block_sum<kIcpPlaneSums>(v, s_buf, s_sum);
    __syncthreads();
    if (threadIdx.x == 0) {
      double x[6];
      ldlt_solve<6>(s_sum, s_sum + 21, x);
      bool finite = true;
      for (int k = 0; k < 6; ++k) finite &= isfinite(x[k]) != 0;
      if (finite) {
        // Delta R = Rz(x2) Ry(x1) Rx(x0), as icp_plane_update_kernel writes R_u
        double sa, ca, sb, cb, sgm, cg;
        sincos(x[0], &sa, &ca);
        sincos(x[1], &sb, &cb);
        sincos(x[2], &sgm, &cg);
        double D[9];  // column-major
        D[0] = cg * cb;
        D[3] = (cg * sb) * sa - sgm * ca;
        D[6] = (cg * sb) * ca + sgm * sa;
        D[1] = sgm * cb;
        D[4] = (sgm * sb) * sa + cg * ca;
        D[7] = (sgm * sb) * ca - cg * sa;
        D[2] = -sb;
        D[5] = cb * sa;
        D[8] = cb * ca;
        double Rn[9], tn[3];
        for (int rr = 0; rr < 3; ++rr) {
          for (int cc = 0; cc < 3; ++cc)
            Rn[3 * cc + rr] = (D[rr] * R[3 * cc] + D[3 + rr] * R[3 * cc + 1]) + D[6 + rr] * R[3 * cc + 2];
          tn[rr] = ((D[rr] * t[0] + D[3 + rr] * t[1]) + D[6 + rr] * t[2]) + x[3 + rr];
        }
        for (int k = 0; k < 9; ++k) s_T[k] = Rn[k];
        for (int k = 0; k < 3; ++k) s_T[9 + k] = tn[k];
      }
    }
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  double Ro[9] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0}, to[3] = {0.0, 0.0, 0.0};
  if (run) {
    const double* R = s_T;
    const double* t = s_T + 9;
    double tp[3];  // t' = (-(R mu_t) + scale_global t) + mu_s
    for (int rr = 0; rr < 3; ++rr) {
      const double Rm = (R[rr] * fp.mean_t[0] + R[3 + rr] * fp.mean_t[1]) + R[6 + rr] * fp.mean_t[2];
      tp[rr] = (-Rm + fp.scale_global * t[rr]) + fp.mean_s[rr];
    }
    for (int rr = 0; rr < 3; ++rr) {
      for (int cc = 0; cc < 3; ++cc) Ro[3 * cc + rr] = R[3 * rr + cc];  // R^T
      to[rr] = -((R[3 * rr] * tp[0] + R[3 * rr + 1] * tp[1]) + R[3 * rr + 2] * tp[2]);
    }
  }
  fp.iterations = run ? a.iteration_number : 0;
  fp.converged = run ? 1 : 0;
  IcpProb& ip = a.icp[b];
  ip.s = 1.0;
  ip.active = ip.seeded = 1;
  for (int k = 0; k < 9; ++k) fp.R[k] = ip.R[k] = Ro[k];
  for (int k = 0; k < 3; ++k) fp.t[k] = ip.t[k] = to[k];
}

}  // namespace

int launch_fgr(const tzr_fgr_params& prm, int B, FgrProb* probs, IcpProb* icp, const float* src, const float* dst,
               const int2* corr, double* pq, cudaStream_t st) {
  const FgrArgs a{src, dst, icp, probs, corr, pq, prm.division_factor, prm.maximum_correspondence_distance,
                  prm.use_absolute_scale ? 1 : 0, prm.decrease_mu ? 1 : 0, prm.iteration_number};
  fgr_prep_kernel<<<B, kFgrThreads, 0, st>>>(a);
  fgr_kernel<<<B, kFgrThreads, 0, st>>>(a);
  return 2;
}

}  // namespace tzr
