// The two device handoffs of tzr_register_cloud_pairs (DESIGN.md §3.10): FPFH over a table of clouds, matching over a
// list of cloud pairs and the ragged solve over the pairs that can be solved, with nothing crossing PCIe between the
// stages but one small read-back of counts.
//
//   pair_rows_kernel     clouds -> the matcher's flat layout: every pair's source and target points (a copy: the
//                        matcher normalises its points in place) and 33-float descriptors at MatchPair::s_off / d_off,
//                        read from the FPFH stage's input points and output descriptors.
//   corr_gather_kernel   matcher output -> solve input: each pair's sorted unique index rows (slot s_off + d_off of the
//                        matcher's output) become float64 rows of the original float points (an exact conversion) at
//                        the pair's row of the solve's flat layout, and the same rows as index pairs compacted back to
//                        back, so that the read-back moves sum n_corr rows and not sum (ns + nd) slots.
#include <algorithm>

#include "tzr_internal.cuh"

namespace tzr {

namespace {

// the pair of flat matcher row r: the last pair whose source (or target) rows start at or before r
__device__ __forceinline__ int pair_of_flat_row(const MatchPair* __restrict__ P, int B, int r, bool dst) {
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if ((dst ? P[mid].d_off : P[mid].s_off) <= r) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// One thread per output float of [source points 3 NS | target points 3 ND | source descriptors 33 NS | target
// descriptors 33 ND]: consecutive threads write consecutive floats and read consecutive floats of one cloud.
__global__ void __launch_bounds__(256) pair_rows_kernel(const MatchPair* __restrict__ P,
                                                        const int2* __restrict__ cloud_lo, int B, int NS, int ND,
                                                        const float* __restrict__ pts, const float* __restrict__ feat,
                                                        float* __restrict__ src_pts, float* __restrict__ dst_pts,
                                                        float* __restrict__ src_feat, float* __restrict__ dst_feat) {
  const long long rows = (long long)NS + ND, E = 36LL * rows;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < E; e += (long long)gridDim.x * blockDim.x) {
    long long x = e;
    const bool desc = x >= 3 * rows;
    if (desc) x -= 3 * rows;
    const int width = desc ? 33 : 3;
    const bool dst = x >= (long long)width * NS;
    if (dst) x -= (long long)width * NS;
    const int r = (int)(x / width), k = (int)(x - (long long)r * width);
    const int b = pair_of_flat_row(P, B, r, dst);
    const int i = r - (dst ? P[b].d_off : P[b].s_off);
    const int lo = dst ? cloud_lo[b].y : cloud_lo[b].x;
    const float v = (desc ? feat : pts)[(size_t)(lo + i) * width + k];
    float* out = desc ? (dst ? dst_feat : src_feat) : (dst ? dst_pts : src_pts);
    out[x] = v;
  }
}

// blockIdx.x: one entry of the gather table; blockIdx.y and the threads stride over its rows
__global__ void __launch_bounds__(256) corr_gather_kernel(const PairGather* __restrict__ G,
                                                          const int32_t* __restrict__ pairs,
                                                          const float* __restrict__ pts, int2* __restrict__ corr,
                                                          double* __restrict__ src, double* __restrict__ dst) {
  const PairGather g = G[blockIdx.x];
  const int2* rows = reinterpret_cast<const int2*>(pairs) + g.slot;
  for (int i = blockIdx.y * blockDim.x + threadIdx.x; i < g.count; i += gridDim.y * blockDim.x) {
    const int2 q = rows[i];
    if (g.corr_row >= 0) corr[g.corr_row + i] = q;
    if (g.solve_row >= 0) {
      const float* a = pts + 3 * ((size_t)g.src_lo + q.x);
      const float* b = pts + 3 * ((size_t)g.dst_lo + q.y);
      double* s = src + 3 * (size_t)(g.solve_row + i);
      double* d = dst + 3 * (size_t)(g.solve_row + i);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        s[k] = (double)a[k];
        d[k] = (double)b[k];
      }
    }
  }
}

}  // namespace

int launch_pair_rows(const MatchPlan& plan, const MatchPair* pairs, const int2* cloud_lo, const float* pts,
                     const float* feat, float* src_pts, float* dst_pts, float* src_feat, float* dst_feat, int num_sms,
                     cudaStream_t st) {
  const long long E = 36LL * ((long long)plan.NS + plan.ND);
  const int grid = (int)std::min<long long>((E + 255) / 256, 32LL * num_sms);
  pair_rows_kernel<<<grid, 256, 0, st>>>(pairs, cloud_lo, plan.B, plan.NS, plan.ND, pts, feat, src_pts, dst_pts,
                                         src_feat, dst_feat);
  return 1;
}

int launch_corr_gather(const PairGather* table, int n_entries, int max_count, const int32_t* pairs, const float* pts,
                       int2* corr, double* src, double* dst, cudaStream_t st) {
  const dim3 grid((unsigned)n_entries, (unsigned)std::max(1, std::min(64, (max_count + 255) / 256)));
  corr_gather_kernel<<<grid, 256, 0, st>>>(table, pairs, pts, corr, src, dst);
  return 1;
}

}  // namespace tzr
