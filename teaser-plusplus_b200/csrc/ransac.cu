// RANSAC on correspondences (Open3D's registration_ransac_based_on_correspondence, DESIGN.md §3.21): the sequential loop
// of include/teaser_b200.h, with every hypothesis of a round drawn, checked and scored at once for B problems.  The
// evaluation is ICP's (launch_icp with max_iteration = 0), seeded by ransac_seed_kernel.
//
//   ransac_prep_kernel    one CTA per problem: the usable rows (both ends finite) compacted in input order as float
//                         rows (x, y), and their normals when the normal checker is on; the loop's state.
//   ransac_hyp_kernel     one thread per hypothesis, one CTA per tile of 256: the draws, the edge-length check, the
//                         Kabsch estimate (rotation_from_H), the distance and normal checks; the passing hypotheses of
//                         the tile compacted in index order, and their count.
//   ransac_score_kernel   one CTA per (problem, segment of kRansacSeg rows, tile of 256 passing hypotheses of the round):
//                         the segment staged in shared memory as float64, each thread one hypothesis's (R, t) in
//                         registers, walking the rows in ascending order: the inlier count and sum d^2 of the segment.
//   ransac_select_kernel  one warp per problem: per passing hypothesis in index order, the segments combined in
//                         ascending order, then the sequential rule (a prefix "best so far" and a prefix minimum of the
//                         exit bounds across the warp); the best, the exit bound, the passed count and the stop flag.
//   ransac_seed_kernel    one thread per problem: the hypotheses drawn, and the winner (or the identity) written into
//                         its ICP problem for the evaluation.
//
// Every sum runs in an order fixed by the problem's own rows, and the rule is applied in hypothesis order, so a
// problem's bits depend neither on the batch it runs in nor on the round schedule.
#include <math_constants.h>

#include <algorithm>

#include "rot3.cuh"
#include "tzr_internal.cuh"

namespace tzr {

namespace {

constexpr int kTileWords = kRansacThreads / 32;

__device__ __forceinline__ bool ransac_finite(double x, double y, double z) {
  return isfinite(x) && isfinite(y) && isfinite(z);
}

// draw j of hypothesis itr: mulhi64(splitmix64(seed + n itr + j), Kv), a row of [0, Kv)
__device__ __forceinline__ int ransac_draw(unsigned long long seed, int n, int itr, int j, int Kv) {
  const uint64_t h = splitmix64(seed + (uint64_t)n * (uint64_t)itr + (uint64_t)j);
  return (int)__umul64hi(h, (uint64_t)Kv);
}

__device__ __forceinline__ void ransac_load(const float* __restrict__ rows, int k, double x[3], double y[3]) {
  const float* r = rows + 6 * (size_t)k;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    x[d] = r[d];
    y[d] = r[3 + d];
  }
}

__device__ __forceinline__ double ransac_norm(const double a[3], const double b[3]) {
  const double dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
  return sqrt((dx * dx + dy * dy) + dz * dz);
}

// d^2 = ||R x + t - y||^2, each row (R(r,0) x0 + R(r,1) x1) + R(r,2) x2, then + t(r) (icp_transform's order at s = 1)
__device__ __forceinline__ double ransac_d2(const double R[9], const double t[3], const double* x, const double* y) {
  double d2 = 0.0;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double p = ((R[r] * x[0] + R[3 + r] * x[1]) + R[6 + r] * x[2]) + t[r];
    const double dd = p - y[r];
    d2 = r == 0 ? dd * dd : d2 + dd * dd;
  }
  return d2;
}

// Hypothesis itr of problem pr: the draws, the edge-length check, the estimate (R, t), the distance and normal checks.
// Returns whether it passed every enabled checker.
__device__ bool ransac_hypothesis(const RansacArgs& a, const RansacProb& pr, int itr, double R[9], double t[3]) {
  const int n = a.n, Kv = pr.Kv;
  const float* rows = a.rows + 6 * pr.c_lo;
  double x[3], y[3], x2[3], y2[3];
  if (a.check_edge) {  // it reads the sample only, so it runs before the estimate; every pair i < j
    for (int i = 0; i < n; ++i) {
      ransac_load(rows, ransac_draw(pr.seed, n, itr, i, Kv), x, y);
      for (int j = i + 1; j < n; ++j) {
        ransac_load(rows, ransac_draw(pr.seed, n, itr, j, Kv), x2, y2);
        const double ds = ransac_norm(x, x2), dt = ransac_norm(y, y2);
        if (ds < dt * a.edge_sim || dt < ds * a.edge_sim) return false;
      }
    }
  }
  double mp[3] = {0.0, 0.0, 0.0}, mq[3] = {0.0, 0.0, 0.0};
  for (int j = 0; j < n; ++j) {
    ransac_load(rows, ransac_draw(pr.seed, n, itr, j, Kv), x, y);
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      mp[d] += x[d];
      mq[d] += y[d];
    }
  }
  const double dn = (double)n;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    mp[d] = mp[d] / dn;
    mq[d] = mq[d] / dn;
  }
  M3 H;
#pragma unroll
  for (int k = 0; k < 9; ++k) H.a[k] = 0.0;
  for (int j = 0; j < n; ++j) {
    ransac_load(rows, ransac_draw(pr.seed, n, itr, j, Kv), x, y);
    const double u[3] = {x[0] - mp[0], x[1] - mp[1], x[2] - mp[2]};
    const double w[3] = {y[0] - mq[0], y[1] - mq[1], y[2] - mq[2]};
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int r = 0; r < 3; ++r) H.a[3 * c + r] += u[r] * w[c];  // H(r, c) column-major
  }
  M3 Rm;
  rotation_from_H(H, Rm);
#pragma unroll
  for (int k = 0; k < 9; ++k) R[k] = Rm.a[k];
#pragma unroll
  for (int r = 0; r < 3; ++r) t[r] = mq[r] - ((R[r] * mp[0] + R[3 + r] * mp[1]) + R[6 + r] * mp[2]);
  if (a.check_dist) {
    for (int j = 0; j < n; ++j) {
      ransac_load(rows, ransac_draw(pr.seed, n, itr, j, Kv), x, y);
      if (sqrt(ransac_d2(R, t, x, y)) > a.dist_thr) return false;
    }
  }
  if (a.check_normal) {
    const float* nrows = a.nrows + 6 * pr.c_lo;
    for (int j = 0; j < n; ++j) {
      ransac_load(nrows, ransac_draw(pr.seed, n, itr, j, Kv), x, y);  // (source normal, target normal)
      double rn[3];
#pragma unroll
      for (int r = 0; r < 3; ++r) rn[r] = (R[r] * x[0] + R[3 + r] * x[1]) + R[6 + r] * x[2];
      if ((y[0] * rn[0] + y[1] * rn[1]) + y[2] * rn[2] < a.cos_normal) return false;
    }
  }
  return true;
}

__global__ void __launch_bounds__(kRansacThreads) ransac_prep_kernel(RansacArgs a) {
  __shared__ int s_cnt[kTileWords];
  const int b = blockIdx.x;
  const IcpProb& ip = a.icp[b];
  RansacProb& pr = a.probs[b];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int2* corr = a.corr + pr.c_lo;
  float* rows = a.rows + 6 * pr.c_lo;
  float* nrows = a.check_normal ? a.nrows + 6 * pr.c_lo : nullptr;
  const int K = pr.K;
  int kv = 0;
  for (int k0 = 0; k0 < K; k0 += kRansacThreads) {  // a block-wide exclusive scan of the flags per round of 256 rows
    const int k = k0 + threadIdx.x;
    float x[3] = {0.f, 0.f, 0.f}, y[3] = {0.f, 0.f, 0.f};
    int2 c = make_int2(0, 0);
    bool ok = false;
    if (k < K) {
      c = corr[k];
      const size_t os = 3 * (size_t)(ip.s_lo + c.x), od = 3 * (size_t)(ip.d_lo + c.y);
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        x[d] = a.src[os + d];
        y[d] = a.dst[od + d];
      }
      ok = ransac_finite(x[0], x[1], x[2]) && ransac_finite(y[0], y[1], y[2]);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) s_cnt[w] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
    for (int q = 0; q < kTileWords; ++q) {
      before += q < w ? s_cnt[q] : 0;
      total += s_cnt[q];
    }
    if (ok) {
      const size_t o = 6 * (size_t)(kv + before + __popc(bal & ((1u << lane) - 1u)));
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        rows[o + d] = x[d];
        rows[o + 3 + d] = y[d];
      }
      if (nrows) {
        const float4 ns = a.src_normals[ip.s_lo + c.x], nd = a.dst_normals[ip.d_lo + c.y];
        nrows[o] = ns.x;
        nrows[o + 1] = ns.y;
        nrows[o + 2] = ns.z;
        nrows[o + 3] = nd.x;
        nrows[o + 4] = nd.y;
        nrows[o + 5] = nd.z;
      }
    }
    kv += total;
    __syncthreads();  // s_cnt is rewritten by the next round
  }
  if (threadIdx.x == 0) {
    pr.Kv = kv;
    pr.done = kv < a.n || a.max_iteration == 0;
    pr.passed = 0;
    pr.best = -1;
    pr.best_count = 0;
    pr.drawn = pr.converged = 0;
    pr.exit = (double)a.max_iteration;
    pr.best_fit = pr.best_rmse = 0.0;
    for (int k = 0; k < 9; ++k) pr.R[k] = k % 4 == 0 ? 1.0 : 0.0;
    for (int k = 0; k < 3; ++k) pr.t[k] = 0.0;
  }
}

__global__ void __launch_bounds__(kRansacThreads) ransac_hyp_kernel(RansacArgs a, int start, int span) {
  __shared__ int s_cnt[kTileWords];
  const int b = blockIdx.x, g = blockIdx.y;
  const RansacProb& pr = a.probs[b];
  if (pr.done) return;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = g * kRansacThreads + threadIdx.x;
  const long long itr = (long long)start + h;
  // hypotheses at or past the bound as the round starts are never drawn (the bound only comes down)
  bool ok = h < span && (double)itr < fmin((double)a.max_iteration, pr.exit);
  double R[9], t[3];
  if (ok) ok = ransac_hypothesis(a, pr, (int)itr, R, t);
  const unsigned bal = __ballot_sync(0xffffffffu, ok);
  if (lane == 0) s_cnt[w] = __popc(bal);
  __syncthreads();
  int before = 0, total = 0;
  for (int q = 0; q < kTileWords; ++q) {
    before += q < w ? s_cnt[q] : 0;
    total += s_cnt[q];
  }
  if (ok) {
    RansacHyp& hy = a.hyps[(size_t)b * a.cap + g * kRansacThreads + before + __popc(bal & ((1u << lane) - 1u))];
#pragma unroll
    for (int k = 0; k < 9; ++k) hy.R[k] = R[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) hy.t[k] = t[k];
    hy.itr = (int)itr;
  }
  if (threadIdx.x == 0) a.tile_cnt[(size_t)b * (a.cap / kRansacThreads) + g] = total;
}

// exclusive prefix of the round's tile counts of problem b into s_pre (tiles <= kRansacThreads), returns the total
__device__ int ransac_tile_prefix(const RansacArgs& a, int b, int tiles, int* s_pre, int* s_warp) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = threadIdx.x < tiles ? a.tile_cnt[(size_t)b * (a.cap / kRansacThreads) + threadIdx.x] : 0;
  int v = c;
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  if (lane == 31) s_warp[w] = v;
  __syncthreads();
  int before = 0, total = 0;
  for (int q = 0; q < kTileWords; ++q) {
    before += q < w ? s_warp[q] : 0;
    total += s_warp[q];
  }
  s_pre[threadIdx.x] = before + v - c;
  __syncthreads();
  return total;
}

__global__ void __launch_bounds__(kRansacThreads) ransac_score_kernel(RansacArgs a, int tiles) {
  __shared__ double s_rows[kRansacSeg * 6];
  __shared__ int s_pre[kRansacThreads];
  __shared__ int s_warp[kTileWords];
  const int b = blockIdx.x / a.nseg, s = blockIdx.x % a.nseg, cg = blockIdx.y;
  const RansacProb& pr = a.probs[b];
  const int r0 = s * kRansacSeg;
  if (pr.done || r0 >= pr.Kv) return;
  const int total = ransac_tile_prefix(a, b, tiles, s_pre, s_warp);
  if (cg * kRansacThreads >= total) return;
  const int m = min(kRansacSeg, pr.Kv - r0);
  const float* rows = a.rows + 6 * (pr.c_lo + r0);
  for (int k = threadIdx.x; k < 6 * m; k += kRansacThreads) s_rows[k] = rows[k];
  __syncthreads();
  const int pos = cg * kRansacThreads + threadIdx.x;
  if (pos >= total) return;
  int lo = 0, hi = tiles - 1;  // the last tile whose prefix is <= pos: the one holding it
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (s_pre[mid] <= pos) lo = mid;
    else hi = mid - 1;
  }
  const RansacHyp& hy = a.hyps[(size_t)b * a.cap + lo * kRansacThreads + (pos - s_pre[lo])];
  double R[9], t[3];
#pragma unroll
  for (int k = 0; k < 9; ++k) R[k] = hy.R[k];
#pragma unroll
  for (int k = 0; k < 3; ++k) t[k] = hy.t[k];
  const double r2 = a.r2;
  int count = 0;
  double sum = 0.0;
  for (int k = 0; k < m; ++k) {
    const double* row = s_rows + 6 * k;
    const double d2 = ransac_d2(R, t, row, row + 3);
    if (d2 < r2) {
      ++count;
      sum += d2;
    }
  }
  a.partial[((size_t)b * a.nseg + s) * a.cap + pos] = make_double2((double)count, sum);
}

// a better than b: a higher fitness, or the same fitness and a smaller rmse
__device__ __forceinline__ bool ransac_better(double fa, double ra, double fb, double rb) {
  return fa > fb || (fa == fb && ra < rb);
}

// ceil(log(1 - confidence) / log(1 - f^n)), f^n as ((f f) f) ...; +inf where it is NaN or -inf (no bound)
__device__ __forceinline__ double ransac_bound(double log1mc, double f, int n) {
  double fn = f;
  for (int k = 1; k < n; ++k) fn = fn * f;
  const double b = ceil(log1mc / log(1.0 - fn));
  return b >= 0.0 ? b : CUDART_INF;
}

__global__ void __launch_bounds__(32) ransac_select_kernel(RansacArgs a, int start, int span, int tiles) {
  const int b = blockIdx.x, lane = threadIdx.x;
  RansacProb& pr = a.probs[b];
  if (pr.done) return;
  const int Kv = pr.Kv, nseg = (Kv + kRansacSeg - 1) / kRansacSeg;
  double exit = pr.exit, bf = pr.best_fit, brm = pr.best_rmse;
  int passed = pr.passed;
  bool stop = false;
  int base = 0;
  for (int g = 0; g < tiles && !stop; ++g) {
    const int c = a.tile_cnt[(size_t)b * (a.cap / kRansacThreads) + g];
    for (int k0 = 0; k0 < c && !stop; k0 += 32) {
      const int j = k0 + lane;
      const bool v = j < c;
      const size_t slot = (size_t)b * a.cap + g * kRansacThreads + j;
      int itr = 0x7fffffff, cnt = 0;
      double f = -1.0, rm = 0.0;
      if (v) {
        itr = a.hyps[slot].itr;
        double sum = 0.0;
        for (int s = 0; s < nseg; ++s) {
          const double2 q = a.partial[((size_t)b * a.nseg + s) * a.cap + base + j];
          cnt += (int)q.x;
          sum += q.y;
        }
        f = cnt > 0 ? (double)cnt / (double)Kv : 0.0;
        rm = cnt > 0 ? sqrt(sum / (double)cnt) : 0.0;
      }
      // the best of lanes 0..lane (the earlier lane on ties), then of the lanes before this one and the best so far
      double pf = f, pe = rm;
      for (int o = 1; o < 32; o <<= 1) {
        const double of = __shfl_up_sync(0xffffffffu, pf, o), oe = __shfl_up_sync(0xffffffffu, pe, o);
        if (lane >= o && !ransac_better(pf, pe, of, oe)) {
          pf = of;
          pe = oe;
        }
      }
      double xf = __shfl_up_sync(0xffffffffu, pf, 1), xe = __shfl_up_sync(0xffffffffu, pe, 1);
      if (lane == 0 || !ransac_better(xf, xe, bf, brm)) {
        xf = bf;
        xe = brm;
      }
      const bool imp = v && ransac_better(f, rm, xf, xe);
      const double bd = imp ? ransac_bound(a.log1mc, f, a.n) : CUDART_INF;
      double mn = bd;  // the smallest bound of lanes 0..lane
      for (int o = 1; o < 32; o <<= 1) {
        const double u = __shfl_up_sync(0xffffffffu, mn, o);
        if (lane >= o) mn = fmin(mn, u);
      }
      double ex = __shfl_up_sync(0xffffffffu, mn, 1);
      ex = lane == 0 ? exit : fmin(exit, ex);  // the bound as hypothesis j comes up
      const unsigned undrawn = __ballot_sync(0xffffffffu, v && (double)itr >= ex);
      const int first = undrawn ? __ffs(undrawn) - 1 : 32;
      const unsigned drawn = first == 32 ? 0xffffffffu : (1u << first) - 1u;
      passed += __popc(__ballot_sync(0xffffffffu, v) & drawn);
      const unsigned imps = __ballot_sync(0xffffffffu, imp) & drawn;
      if (imps) {
        const int win = 31 - __clz(imps);
        bf = __shfl_sync(0xffffffffu, f, win);
        brm = __shfl_sync(0xffffffffu, rm, win);
        if (lane == win) {
          pr.best = itr;
          pr.best_count = cnt;
          const RansacHyp& hy = a.hyps[slot];
          for (int k = 0; k < 9; ++k) pr.R[k] = hy.R[k];
          for (int k = 0; k < 3; ++k) pr.t[k] = hy.t[k];
        }
      }
      exit = first == 32 ? fmin(exit, __shfl_sync(0xffffffffu, mn, 31)) : __shfl_sync(0xffffffffu, ex, first);
      stop = first < 32;
    }
    base += c;
  }
  __syncwarp();
  if (lane == 0) {
    pr.exit = exit;
    pr.best_fit = bf;
    pr.best_rmse = brm;
    pr.passed = passed;
    pr.done = stop || (double)((long long)start + span) >= fmin((double)a.max_iteration, exit);
  }
}

__global__ void ransac_seed_kernel(RansacArgs a, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  RansacProb& pr = a.probs[b];
  const bool ran = pr.Kv >= a.n && a.max_iteration > 0;
  int drawn = 0;
  if (ran) {  // the loop stops at the first hypothesis at or past min(max_iteration, exit), and never before the winner
    drawn = (int)fmin((double)a.max_iteration, pr.exit);
    if (pr.best >= 0) drawn = max(drawn, pr.best + 1);
  }
  pr.drawn = drawn;
  pr.converged = ran && drawn < a.max_iteration;
  IcpProb& ip = a.icp[b];
  ip.s = 1.0;
  ip.active = ip.seeded = 1;
  for (int k = 0; k < 9; ++k) ip.R[k] = pr.R[k];
  for (int k = 0; k < 3; ++k) ip.t[k] = pr.t[k];
}

}  // namespace

void ransac_schedule(int max_iteration, long long k_max, std::vector<int>* spans, int* cap, int* nseg) {
  *nseg = (int)std::max(1ll, (k_max + kRansacSeg - 1) / kRansacSeg);
  int c = kRansacMaxRound;
  while (c > kRansacMinRound && (long long)c * *nseg > kRansacPartialBudget) c >>= 1;
  *cap = c;
  spans->clear();
  long long start = 0;
  for (int r = kRansacMinRound; start < max_iteration; r = std::min(2 * r, c)) {
    const int span = std::min(r, c);
    spans->push_back(span);
    start += span;
  }
  // the largest round actually run (the spans only grow); no round (max_iteration = 0) keeps the smallest tables
  *cap = spans->empty() ? kRansacMinRound : spans->back();
}

int launch_ransac(const RansacArgs& a, int B, const std::vector<int>& spans, cudaStream_t st) {
  ransac_prep_kernel<<<B, kRansacThreads, 0, st>>>(a);
  long long start = 0;
  for (int span : spans) {
    const int tiles = (span + kRansacThreads - 1) / kRansacThreads;
    ransac_hyp_kernel<<<dim3(B, tiles), kRansacThreads, 0, st>>>(a, (int)start, span);
    ransac_score_kernel<<<dim3(B * a.nseg, tiles), kRansacThreads, 0, st>>>(a, tiles);
    ransac_select_kernel<<<B, 32, 0, st>>>(a, (int)start, span, tiles);
    start += span;
  }
  ransac_seed_kernel<<<(B + 127) / 128, 128, 0, st>>>(a, B);
  return 2 + 3 * (int)spans.size();
}

}  // namespace tzr
