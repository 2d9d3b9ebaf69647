// Unknown-scale variant of stage 1 (Params::estimate_scaling = true, the reference's default):
//   TLSScaleSolver::solveForScale         teaser/src/registration.cc:410-425
//   ScalarTLSEstimator::estimate over K   teaser/src/registration.cc:21-88
// Per TIM k=(i,j), i<j in the reference's order k = i*N - i(i+1)/2 + (j-i-1) (registration.cc:531):
//   ratio_k = ||dst_j-dst_i|| / ||src_j-src_i||,  alpha_k = beta * (1/||src_j-src_i||)
// then a scalar TLS over the K ratios gives the scale; the inlier predicate |ratio - s| <= alpha is
// re-evaluated (identically) by the graph tile kernel when it emits the bitset.
//
// Two implementations, selected by size:
//  * n <= kScaleSmallN: one CTA per problem sorts the 2K interval end points with a bitonic network and one
//    thread sweeps them in the reference's accumulation order (bit-exact vs the oracle up to tied end points).
//  * larger n (C2: K = 12.5 M, 25 M end points): stable LSD radix sort of (key, payload) pairs — the one library
//    call on this path, cub::DeviceRadixSort, flagged as such in DESIGN.md — over stored ratios and ranges up to
//    n = 8192, above it in chunks of at most 2^27 end points whose ratios and ranges are regenerated from the points
//    (no K-sized array; any n <= 65536), followed by hand-written,
//    DETERMINISTIC two-level scans (fixed summation trees, no decoupled look-back) of the six running sums of
//    registration.cc:58-68, the cost of :70-74 at every end point and a first-minimum arg-min (:77-79).  The
//    running sums are associated differently from the reference's sequential sweep (relative differences
//    ~1e-13 in the estimate), which is why the scale is compared with a tolerance at these sizes.
#include <cub/device/device_radix_sort.cuh>

#include "tls_device.cuh"
#include "tzr_internal.cuh"

namespace tzr {

__global__ void __launch_bounds__(256) scale_pairs_kernel(Batch bt, double* X, double* Rg) {
  const int i = blockIdx.x, b = blockIdx.y;
  const int n = bt.n;
  const int nv = bt.nb ? bt.nb[b] : n;  // ragged size class: the problem's own TIMs, packed in its own order
  const long long K = (long long)n * (n - 1) / 2;
  const double* src = bt.src + (size_t)b * n * 3;
  const double* dst = bt.dst + (size_t)b * n * 3;
  double* x = X + (size_t)b * K;
  double* r = Rg + (size_t)b * K;
  const long long seg = (long long)i * nv - (long long)i * (i + 1) / 2;  // registration.cc:531
  for (int j = i + 1 + threadIdx.x; j < nv; j += blockDim.x) {
    const double d1 = tim_norm_exact(src, i, j);
    const double d2 = tim_norm_exact(dst, i, j);
    const long long k = seg + (j - i - 1);
    x[k] = __ddiv_rn(d2, d1);                        // raw_scales = v2_dist / v1_dist        :420
    r[k] = __dmul_rn(bt.beta, __ddiv_rn(1.0, d1));   // alphas = beta * v1_dist.cwiseInverse() :422
  }
}

// small path: one CTA per problem (n <= kScaleSmallN, so K and its end-point count fit an int)
__global__ void __launch_bounds__(1024) scale_tls_kernel(Batch bt, const double* X, const double* Rg, double* key,
                                                          int32_t* idx) {
  const int b = blockIdx.x;
  const int K = bt.n * (bt.n - 1) / 2;
  const int npad = next_pow2(2 * K);
  const int nv = bt.nb ? bt.nb[b] : bt.n;
  if (nv < 2) return;  // no TIM: the scale stays 1, as launch_scale_estimation leaves it for n < 2
  const int Kb = nv * (nv - 1) / 2;
  __shared__ double s_est;
  tls_block(X + (size_t)b * K, Rg + (size_t)b * K, 0.0, Kb, 1, key + (size_t)b * npad, idx + (size_t)b * npad, &s_est);
  if (threadIdx.x == 0) bt.sol[b].scale = s_est;
}

// tzr_scalar_tls on the small path: one CTA
__global__ void __launch_bounds__(1024) scalar_tls_kernel(const double* x, const double* ranges, long long m,
                                                           double* key, int32_t* idx, double* out_est,
                                                           uint8_t* inliers) {
  __shared__ double s_est;
  tls_block(x, ranges, 0.0, (int)m, 1, key, idx, &s_est);
  const double est = s_est;
  for (long long i = threadIdx.x; i < m; i += blockDim.x) inliers[i] = tls_inlier(x[i], ranges[i], est);
  if (threadIdx.x == 0) *out_est = est;
}

// ---------------------------------------------------------------------------------------------------------------
// large-K path
// ---------------------------------------------------------------------------------------------------------------
namespace {

constexpr int kTileThreads = 256;
constexpr int kPerThread = 8;
constexpr int kTileElems = kTileThreads * kPerThread;  // 2048 end points per tile

struct Sums {  // running sums of the sweep (registration.cc:51-56)
  double card, w, wx, r, x, xx, rplus;  // rplus: sum of ranges over entering end points (== ranges.sum() in total)
};
__device__ __forceinline__ Sums sums_zero() { return Sums{0, 0, 0, 0, 0, 0, 0}; }
__device__ __forceinline__ Sums sums_add(const Sums& a, const Sums& b) {
  return Sums{a.card + b.card, a.w + b.w, a.wx + b.wx, a.r + b.r, a.x + b.x, a.xx + b.xx, a.rplus + b.rplus};
}
// Where a measurement's value and range come from.  ArrayTls: arrays (tzr_scalar_tls).  TimTls: regenerated from the
// points, as scale_pairs_kernel computes them (the same bits), for TIM t of a problem of nv points in its packed order.
struct ArrayTls {
  const double* X;
  const double* Rg;
  // read-only loads, as from __restrict__ kernel parameters (a struct member's __restrict__ does not give them)
  __device__ __forceinline__ void at(long long t, double* x, double* r) const {
    *r = __ldg(Rg + t);
    *x = __ldg(X + t);
  }
};
struct TimTls {
  const double* __restrict__ src;
  const double* __restrict__ dst;
  int nv;
  double beta;
  // (i, j) of TIM t: the largest i with i*nv - i(i+1)/2 <= t (registration.cc:531), from a double estimate and an exact
  // integer correction
  __device__ __forceinline__ void pair(long long t, int* i, int* j) const {
    const double b = 2.0 * nv - 1.0;
    int a = (int)((b - sqrt(fmax(b * b - 8.0 * (double)t, 0.0))) * 0.5);
    a = max(0, min(a, nv - 2));
    auto seg = [&](long long v) { return v * nv - v * (v + 1) / 2; };
    while (a > 0 && seg(a) > t) --a;
    while (a + 1 < nv - 1 && seg(a + 1) <= t) ++a;
    *i = a;
    *j = (int)(t - seg(a)) + a + 1;
  }
  __device__ __forceinline__ void at(long long t, double* x, double* r) const {
    int i, j;
    pair(t, &i, &j);
    const double d1 = tim_norm_exact(src, i, j);
    const double d2 = tim_norm_exact(dst, i, j);
    *x = __ddiv_rn(d2, d1);
    *r = __dmul_rn(beta, __ddiv_rn(1.0, d1));
  }
};

template <class Src, class Idx>
__device__ __forceinline__ Sums endpoint_terms(Idx e, const Src& s, bool* kept) {
  const long long id = e >> 1;
  const double eps = (e & 1) ? -1.0 : 1.0;
  double x, r;
  s.at(id, &x, &r);
  *kept = tls_kept(x, r);
  if (!*kept) return sums_zero();  // excluded measurement: no contribution to any sum, ranges.sum() included
  const double w = 1.0 / (r * r);
  return Sums{eps, eps * w, eps * w * x, eps * r, eps * x, eps * x * x, (e & 1) ? 0.0 : r};
}
__device__ __forceinline__ Sums warp_shfl_up(const Sums& v, int o) {
  return Sums{__shfl_up_sync(0xffffffffu, v.card, o), __shfl_up_sync(0xffffffffu, v.w, o),
              __shfl_up_sync(0xffffffffu, v.wx, o),   __shfl_up_sync(0xffffffffu, v.r, o),
              __shfl_up_sync(0xffffffffu, v.x, o),    __shfl_up_sync(0xffffffffu, v.xx, o),
              __shfl_up_sync(0xffffffffu, v.rplus, o)};
}

// inclusive scan of one Sums per thread over the block (fixed tree: Hillis-Steele inside warps, sequential over
// the 8 warp totals) -> returns the EXCLUSIVE prefix of this thread; *total = block sum
__device__ Sums block_excl_scan_sums(const Sums& v, Sums* s_warp /* kTileThreads/32 + 1 */, Sums* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  Sums inc = v;
  for (int o = 1; o < 32; o <<= 1) {
    const Sums t = warp_shfl_up(inc, o);
    if (lane >= o) inc = sums_add(t, inc);
  }
  __syncthreads();
  if (lane == 31) s_warp[w] = inc;
  __syncthreads();
  if (threadIdx.x == 0) {
    Sums acc = sums_zero();
    for (int q = 0; q < kTileThreads / 32; ++q) {
      const Sums t = s_warp[q];
      s_warp[q] = acc;
      acc = sums_add(acc, t);
    }
    s_warp[kTileThreads / 32] = acc;
  }
  __syncthreads();
  *total = s_warp[kTileThreads / 32];
  // exclusive prefix = warp offset + (inclusive - own)
  Sums excl = s_warp[w];
  const Sums prev = warp_shfl_up(inc, 1);
  if (lane > 0) excl = sums_add(excl, prev);
  return excl;
}

__global__ void __launch_bounds__(256) make_endpoints_kernel(const double* __restrict__ X,
                                                              const double* __restrict__ Rg, long long K,
                                                              double* __restrict__ key, int* __restrict__ val) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= 2 * K) return;
  const long long t = q >> 1;
  key[q] = tls_key(X[t], Rg[t], q);  // registration.cc:36-37
  val[q] = (int)q;
}

template <class Src, class Idx>
__global__ void __launch_bounds__(kTileThreads) tile_sums_kernel(const Idx* __restrict__ val, long long M, Src s,
                                                                 Sums* tile_sum) {
  __shared__ Sums s_warp[kTileThreads / 32 + 1];
  const long long base = (long long)blockIdx.x * kTileElems + (long long)threadIdx.x * kPerThread;
  Sums acc = sums_zero();
  for (int k = 0; k < kPerThread; ++k) {
    const long long q = base + k;
    bool kept;
    if (q < M) acc = sums_add(acc, endpoint_terms(val[q], s, &kept));
  }
  Sums total;
  block_excl_scan_sums(acc, s_warp, &total);
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

// exclusive scan of the tile sums, sequential on one thread (deterministic; <= a few hundred thousand tiles), leaving
// the running total in *acc_out.  kChained (the regenerating route): starting from *acc_in (nullptr: zero), so that the
// tiles of consecutive chunks scan as one sequence.
template <bool kChained>
__global__ void tile_scan_kernel(Sums* tile_sum, long long n_tiles, const Sums* acc_in, Sums* acc_out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  Sums acc = (kChained && acc_in) ? *acc_in : sums_zero();
  for (long long t = 0; t < n_tiles; ++t) {
    const Sums v = tile_sum[t];
    tile_sum[t] = acc;
    acc = sums_add(acc, v);
  }
  *acc_out = acc;
}

struct Best {
  double cost, xhat;
  long long pos;
};
__device__ __forceinline__ bool best_less(const Best& a, const Best& b) {  // first strict minimum; NaN never wins
  if (a.pos < 0) return false;
  if (b.pos < 0) return true;
  return (a.cost < b.cost) || (a.cost == b.cost && a.pos < b.pos);
}

// positions are relative to val[0] (final_argmin_kernel makes them global)
template <class Src, class Idx>
__global__ void __launch_bounds__(kTileThreads) tile_cost_kernel(const Idx* __restrict__ val, long long M, Src s,
                                                                 const Sums* __restrict__ tile_off,
                                                                 const Sums* __restrict__ grand, Best* tile_best) {
  __shared__ Sums s_warp[kTileThreads / 32 + 1];
  __shared__ Best s_best[kTileThreads / 32];
  const long long base = (long long)blockIdx.x * kTileElems + (long long)threadIdx.x * kPerThread;
  Sums terms[kPerThread];
  bool kept[kPerThread];
  Sums acc = sums_zero();
  for (int k = 0; k < kPerThread; ++k) {
    const long long q = base + k;
    kept[k] = false;
    terms[k] = (q < M) ? endpoint_terms(val[q], s, &kept[k]) : sums_zero();
    acc = sums_add(acc, terms[k]);
  }
  Sums total;
  Sums run = sums_add(tile_off[blockIdx.x], block_excl_scan_sums(acc, s_warp, &total));
  const double r_total = grand->rplus;  // ranges.sum()  (registration.cc:51)
  Best best{0.0, 0.0, -1};
  for (int k = 0; k < kPerThread; ++k) {
    const long long q = base + k;
    if (q >= M) break;
    if (!kept[k]) continue;  // excluded end points (key +inf, after every kept one) are no candidate state
    run = sums_add(run, terms[k]);
    const double x_hat = run.wx / run.w;                                                 // :70
    const double residual = run.card * x_hat * x_hat + run.xx - 2.0 * run.x * x_hat;   // :72-73
    const double cost = residual + (r_total - run.r);                                    // :74
    if (cost == cost && (best.pos < 0 || cost < best.cost)) best = Best{cost, x_hat, q};  // NaN never wins
  }
  // block arg-min (lexicographic on (cost, position))
  for (int o = 16; o; o >>= 1) {
    Best t{__shfl_xor_sync(0xffffffffu, best.cost, o), __shfl_xor_sync(0xffffffffu, best.xhat, o),
           __shfl_xor_sync(0xffffffffu, best.pos, o)};
    if (best_less(t, best)) best = t;
  }
  if ((threadIdx.x & 31) == 0) s_best[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    Best bb = s_best[0];
    for (int q = 1; q < kTileThreads / 32; ++q)
      if (best_less(s_best[q], bb)) bb = s_best[q];
    tile_best[blockIdx.x] = bb;
  }
}

// arg-min over the tiles.  kChained (the regenerating route): their positions offset by pos0 (the global position of
// the chunk's first tile), on from *run_in (nullptr: none yet), the best so far of earlier chunks, left in *run_out.
template <bool kChained>
__global__ void final_argmin_kernel(const Best* tile_best, long long n_tiles, long long pos0, const Best* run_in,
                                    Best* run_out, double* out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  Best bb;
  if constexpr (kChained) {
    bb = run_in ? *run_in : Best{0.0, 0.0, -1};
    for (long long t = 0; t < n_tiles; ++t) {
      Best c = tile_best[t];
      if (c.pos >= 0) c.pos += pos0;
      if (best_less(c, bb)) bb = c;
    }
    *run_out = bb;
  } else {
    bb = tile_best[0];
    for (long long t = 1; t < n_tiles; ++t)
      if (best_less(tile_best[t], bb)) bb = tile_best[t];
  }
  *out = bb.pos < 0 ? 0.0 / 0.0 : bb.xhat;  // no kept measurement (or no non-NaN cost): NaN, as tls_sweep
}

__global__ void tls_inliers_kernel(const double* __restrict__ X, const double* __restrict__ Rg, long long K,
                                   const double* __restrict__ est, uint8_t* __restrict__ inliers) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < K) inliers[i] = tls_inlier(X[i], Rg[i], *est);
}

size_t tls_large_scratch_bytes(long long K) {
  const long long M = 2 * K;
  size_t temp = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, temp, (const double*)nullptr, (double*)nullptr, (const int*)nullptr,
                                  (int*)nullptr, (int)M);
  const long long n_tiles = (M + kTileElems - 1) / kTileElems;
  return (size_t)M * (8 + 8 + 4 + 4) + temp + (size_t)n_tiles * (sizeof(Sums) + sizeof(Best)) + sizeof(Sums) +
         1024;
}

// Scalar TLS over K measurements with the radix sort + tiled scans + first-minimum arg-min; writes the estimate to
// *out (device).  scratch: tls_large_scratch_bytes(K) bytes, 2K < 2^31.  Returns the number of launches (approximate:
// the radix sort's internal kernels are counted as 8).
int launch_tls_large(const double* X, const double* Rg, long long K, void* scratch, double* out, cudaStream_t st) {
  const long long M = 2 * K;
  const long long n_tiles = (M + kTileElems - 1) / kTileElems;
  size_t temp = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, temp, (const double*)nullptr, (double*)nullptr, (const int*)nullptr,
                                  (int*)nullptr, (int)M);
  char* p = (char*)scratch;
  double* key_in = (double*)p;  p += (size_t)M * 8;
  double* key_out = (double*)p; p += (size_t)M * 8;
  int* val_in = (int*)p;        p += (size_t)M * 4;
  int* val_out = (int*)p;       p += (size_t)M * 4;
  p = (char*)(((uintptr_t)p + 255) & ~(uintptr_t)255);
  Sums* tile_sum = (Sums*)p;    p += (size_t)n_tiles * sizeof(Sums);
  Sums* grand = (Sums*)p;       p += sizeof(Sums);
  Best* tile_best = (Best*)p;   p += (size_t)n_tiles * sizeof(Best);
  p = (char*)(((uintptr_t)p + 255) & ~(uintptr_t)255);
  void* cub_temp = p;
  const ArrayTls s{X, Rg};
  make_endpoints_kernel<<<(unsigned)((M + 255) / 256), 256, 0, st>>>(X, Rg, K, key_in, val_in);
  cub::DeviceRadixSort::SortPairs(cub_temp, temp, key_in, key_out, val_in, val_out, (int)M, 0, 64, st);
  tile_sums_kernel<<<(unsigned)n_tiles, kTileThreads, 0, st>>>(val_out, M, s, tile_sum);
  tile_scan_kernel<false><<<1, 32, 0, st>>>(tile_sum, n_tiles, nullptr, grand);
  tile_cost_kernel<<<(unsigned)n_tiles, kTileThreads, 0, st>>>(val_out, M, s, tile_sum, grand, tile_best);
  final_argmin_kernel<false><<<1, 32, 0, st>>>(tile_best, n_tiles, 0LL, nullptr, nullptr, out);
  return 5 + 8;
}

size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

// ---------------------------------------------------------------------------------------------------------------
// regenerating route of the unknown-scale stage (DESIGN.md §3.4): no ratio or range is stored.  The 2K end points, in
// the order of the stable radix sort above, are cut into chunks of at most C consecutive ones; each chunk is generated
// in ascending q, sorted by cub::DeviceRadixSort and swept by the tile kernels with TimTls, its trailing partial tile
// carried into the next chunk, so that tiles, offsets and the arg-min are those of the sort of all 2K at once.
// ---------------------------------------------------------------------------------------------------------------
using u128 = unsigned __int128;
constexpr long long kChunkAuto = 1LL << 27;  // end points per chunk: 3 GiB of keys and payloads, double-buffered
constexpr int kMaxChunks = 4096;             // a forced capacity is raised until the end points fit this many chunks
constexpr int kGenThreads = 256;
constexpr int kGenRounds = 32;
constexpr long long kGenTims = (long long)kGenThreads * kGenRounds;  // TIMs per block of the generating kernels
constexpr int kCountWindow = 32;              // chunks whose per-block counts one counting pass takes
constexpr int kSelGroup = 32;                 // boundary prefixes one histogram block takes
constexpr int kSelPasses = 12;                // 96-bit (key, q) in 8-bit digits

// The sort order as an unsigned integer: the key's bits as CUB's radix sort orders doubles (-0.0 as +0.0), then q.
__device__ __forceinline__ u128 sort_pos(double key, long long q) {
  unsigned long long b = __double_as_longlong(key);
  if (b == 0x8000000000000000ull) b = 0;
  b ^= (b >> 63) ? ~0ull : 0x8000000000000000ull;
  return ((u128)b << 32) | (u128)(unsigned long long)q;
}
// chunk of an end point: the number of chunk boundaries at or below it
__device__ __forceinline__ int chunk_of(u128 v, const u128* __restrict__ bnd, int nb) {
  int lo = 0, hi = nb;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (bnd[mid] <= v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// selection of the boundaries: target j (rank (j+1) C of the sorted sequence) is known to `bits` leading bits; one
// histogram of the next 8 bits per distinct known prefix
__global__ void __launch_bounds__(kGenThreads) sel_hist_kernel(TimTls s, long long K, int bits,
                                                               const u128* __restrict__ uniq,
                                                               const int* __restrict__ n_uniq,
                                                               unsigned long long* __restrict__ hist) {
  __shared__ u128 s_u[kSelGroup];
  __shared__ unsigned s_h[kSelGroup * 256];
  const int u0 = blockIdx.y * kSelGroup;
  const int nu = *n_uniq;
  if (u0 >= nu) return;
  const int ng = min(kSelGroup, nu - u0);
  for (int k = threadIdx.x; k < kSelGroup * 256; k += blockDim.x) s_h[k] = 0;
  if (threadIdx.x < ng) s_u[threadIdx.x] = uniq[u0 + threadIdx.x];
  __syncthreads();
  const int sh = 96 - bits;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < K; t += (long long)gridDim.x * blockDim.x) {
    double x, r;
    s.at(t, &x, &r);
    for (int e = 0; e < 2; ++e) {
      const long long q = 2 * t + e;
      const u128 v = sort_pos(tls_key(x, r, q), q);
      const u128 pre = v >> sh;
      int lo = 0, hi = ng;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (s_u[mid] < pre) lo = mid + 1; else hi = mid;
      }
      if (lo < ng && s_u[lo] == pre) atomicAdd(&s_h[lo * 256 + (int)((v >> (sh - 8)) & 255)], 1u);
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < ng * 256; k += blockDim.x)
    if (s_h[k]) atomicAdd(&hist[(size_t)(u0 + (k >> 8)) * 256 + (k & 255)], (unsigned long long)s_h[k]);
}

// one thread: start (prefix 0, rank (j+1) C) or extend every target by the digit its histogram puts its rank in, then
// list the distinct prefixes (the targets are in rank order, so their prefixes are non-decreasing)
__global__ void sel_update_kernel(u128* tpre, unsigned long long* trank, int* tu, int T, long long C, u128* uniq,
                                  int* n_uniq, const unsigned long long* __restrict__ hist, bool start) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int nu = 0;
  for (int j = 0; j < T; ++j) {
    if (start) {
      tpre[j] = 0;
      trank[j] = (unsigned long long)(j + 1) * (unsigned long long)C;
    } else {
      const unsigned long long* h = hist + (size_t)tu[j] * 256;
      unsigned long long cum = 0;
      int d = 0;
      while (d < 255 && cum + h[d] <= trank[j]) cum += h[d++];
      tpre[j] = (tpre[j] << 8) | (u128)d;
      trank[j] -= cum;
    }
    if (nu == 0 || uniq[nu - 1] != tpre[j]) uniq[nu++] = tpre[j];
    tu[j] = nu - 1;
  }
  *n_uniq = nu;
}

// count[(c - c0) * nblk + block]: end points of chunk c (c0 <= c < c0 + kCountWindow) among the block's TIMs
__global__ void __launch_bounds__(kGenThreads) chunk_count_kernel(TimTls s, long long K, const u128* __restrict__ bnd,
                                                                  int nb, int c0, unsigned long long* count) {
  __shared__ unsigned s_c[kCountWindow];
  if (threadIdx.x < kCountWindow) s_c[threadIdx.x] = 0;
  __syncthreads();
  const long long t0 = (long long)blockIdx.x * kGenTims;
  for (int rd = 0; rd < kGenRounds; ++rd) {
    const long long t = t0 + (long long)rd * kGenThreads + threadIdx.x;
    if (t >= K) break;
    double x, r;
    s.at(t, &x, &r);
    for (int e = 0; e < 2; ++e) {
      const int c = chunk_of(sort_pos(tls_key(x, r, 2 * t + e), 2 * t + e), bnd, nb) - c0;
      if (c >= 0 && c < kCountWindow) atomicAdd(&s_c[c], 1u);
    }
  }
  __syncthreads();
  if (threadIdx.x < kCountWindow) count[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = s_c[threadIdx.x];
}

// exclusive scan of each chunk's per-block counts in place (one CTA per chunk; integer sums, exact in any order)
__global__ void __launch_bounds__(256) chunk_offsets_kernel(unsigned long long* count, long long nblk) {
  __shared__ unsigned long long s_t[256];
  unsigned long long* c = count + (size_t)blockIdx.x * nblk;
  const long long per = (nblk + 255) / 256;
  const long long lo = min(nblk, per * threadIdx.x), hi = min(nblk, lo + per);
  unsigned long long sum = 0;
  for (long long k = lo; k < hi; ++k) sum += c[k];
  s_t[threadIdx.x] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long acc = 0;
    for (int k = 0; k < 256; ++k) {
      const unsigned long long v = s_t[k];
      s_t[k] = acc;
      acc += v;
    }
  }
  __syncthreads();
  unsigned long long acc = s_t[threadIdx.x];
  for (long long k = lo; k < hi; ++k) {
    const unsigned long long v = c[k];
    c[k] = acc;
    acc += v;
  }
}

// the end points of chunk c (nb == 0: all of them) in ascending q: each block compacts its TIMs' members in order and
// writes them at its offset (off: the chunk's row of chunk_offsets_kernel; nullptr: every end point is a member)
__global__ void __launch_bounds__(kGenThreads) chunk_gen_kernel(TimTls s, long long K, const u128* __restrict__ bnd,
                                                                int nb, int c, const unsigned long long* __restrict__ off,
                                                                double* __restrict__ key, uint32_t* __restrict__ val) {
  __shared__ unsigned s_w[kGenThreads / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const long long t0 = (long long)blockIdx.x * kGenTims;
  unsigned long long at = off ? off[blockIdx.x] : (unsigned long long)(2 * t0);
  for (int rd = 0; rd < kGenRounds; ++rd) {
    const long long t = t0 + (long long)rd * kGenThreads + threadIdx.x;
    if (t0 + (long long)rd * kGenThreads >= K) break;  // uniform over the block
    double kk[2] = {0.0, 0.0};
    bool in[2] = {false, false};
    if (t < K) {
      double x, r;
      s.at(t, &x, &r);
      for (int e = 0; e < 2; ++e) {
        kk[e] = tls_key(x, r, 2 * t + e);
        in[e] = nb == 0 || chunk_of(sort_pos(kk[e], 2 * t + e), bnd, nb) == c;
      }
    }
    const unsigned b0 = __ballot_sync(0xffffffffu, in[0]), b1 = __ballot_sync(0xffffffffu, in[1]);
    const unsigned lt = (1u << lane) - 1u;
    const unsigned mine = __popc(b0 & lt) + __popc(b1 & lt);
    if (lane == 0) s_w[w] = __popc(b0) + __popc(b1);
    __syncthreads();
    unsigned before = 0, total = 0;
    for (int k = 0; k < kGenThreads / 32; ++k) {
      if (k < w) before += s_w[k];
      total += s_w[k];
    }
    unsigned long long o = at + before + mine;
    for (int e = 0; e < 2; ++e)
      if (in[e]) {
        key[o] = kk[e];
        val[o] = (uint32_t)(2 * t + e);
        ++o;
      }
    at += total;
    __syncthreads();
  }
}

struct StreamPlan {
  long long M, C;  // end points, chunk capacity
  int nch;         // chunks
  long long nblk;  // blocks of the generating kernels
};
StreamPlan stream_plan(long long K, long long chunk) {
  StreamPlan pl;
  pl.M = 2 * K;
  long long C = kChunkAuto;
  if (chunk >= kTileElems) C = std::min(C, std::max(chunk, (pl.M + kMaxChunks - 1) / kMaxChunks));
  pl.C = std::min(C, std::max(pl.M, 1LL));
  pl.nch = (int)((pl.M + pl.C - 1) / pl.C);
  pl.nblk = (K + kGenTims - 1) / kGenTims;
  return pl;
}

struct StreamLayout {
  double* key[2];
  uint32_t* val[2];  // kTileElems slots ahead of each: the carried partial tile
  uint32_t* carry;
  Sums *tile_sum, *acc, *grand;
  Best *tile_best, *best;
  u128 *tpre, *uniq;
  unsigned long long *trank, *hist, *count;
  int *tu, *n_uniq;
  void* cub_temp;
  size_t cub_bytes, total;
};
// pointers into base (nullptr: sizes only)
StreamLayout stream_layout(const StreamPlan& pl, char* base) {
  StreamLayout L{};
  const long long C = pl.C, T = pl.nch - 1, ntile = C / kTileElems + 2;
  cub::DoubleBuffer<double> dk(nullptr, nullptr);
  cub::DoubleBuffer<uint32_t> dv(nullptr, nullptr);
  cub::DeviceRadixSort::SortPairs(nullptr, L.cub_bytes, dk, dv, (int)C, 0, 64);
  size_t off = 0;
  auto carve = [&](auto*& ptr, size_t bytes) {
    ptr = base ? (std::remove_reference_t<decltype(ptr)>)(base + off) : nullptr;
    off = align256(off + bytes);
  };
  for (int b = 0; b < 2; ++b) carve(L.key[b], (size_t)C * 8);
  for (int b = 0; b < 2; ++b) {
    carve(L.val[b], (size_t)(C + kTileElems) * 4);
    if (L.val[b]) L.val[b] += kTileElems;
  }
  carve(L.carry, (size_t)kTileElems * 4);
  carve(L.tile_sum, (size_t)ntile * sizeof(Sums));
  carve(L.tile_best, (size_t)ntile * sizeof(Best));
  carve(L.acc, sizeof(Sums));
  carve(L.grand, sizeof(Sums));
  carve(L.best, sizeof(Best));
  if (T > 0) {
    carve(L.tpre, (size_t)T * sizeof(u128));
    carve(L.uniq, (size_t)T * sizeof(u128));
    carve(L.trank, (size_t)T * 8);
    carve(L.tu, (size_t)T * 4);
    carve(L.n_uniq, 4);
    carve(L.hist, (size_t)T * 256 * 8);
    carve(L.count, (size_t)kCountWindow * pl.nblk * 8);
  }
  carve(L.cub_temp, L.cub_bytes);
  L.total = off;
  return L;
}

// The unknown-scale TLS of one problem by the regenerating route; writes the estimate to *out.  Returns the launches
// (the radix sort's internal kernels counted as 8 per call) and the chunk count in *nch.
int launch_tls_stream(const TimTls& s, long long K, long long chunk, void* scratch, double* out, int* nch,
                      cudaStream_t st) {
  const StreamPlan pl = stream_plan(K, chunk);
  const StreamLayout L = stream_layout(pl, (char*)scratch);
  const int T = pl.nch - 1;
  const unsigned gblk = (unsigned)pl.nblk;
  int launches = 0;
  *nch = pl.nch;
  if (T > 0) {  // boundaries: the end points at ranks C, 2C, ... of the sorted sequence, 8 bits per pass
    const unsigned hblk = (unsigned)std::min<long long>(pl.nblk, 4LL * 132 * 8);
    for (int pass = 0; pass <= kSelPasses; ++pass) {
      if (pass > 0) {
        cudaMemsetAsync(L.hist, 0, (size_t)T * 256 * 8, st);
        sel_hist_kernel<<<dim3(hblk, (unsigned)((T + kSelGroup - 1) / kSelGroup)), kGenThreads, 0, st>>>(
            s, K, 8 * (pass - 1), L.uniq, L.n_uniq, L.hist);
      }
      sel_update_kernel<<<1, 32, 0, st>>>(L.tpre, L.trank, L.tu, T, pl.C, L.uniq, L.n_uniq, L.hist, pass == 0);
      launches += pass > 0 ? 2 : 1;
    }
  }
  const u128* bnd = L.tpre;  // after the last pass: the boundaries' full (key, q) positions
  int window = -1;
  for (int sweep = 0; sweep < 2; ++sweep) {  // 0: the grand total (ranges.sum()), 1: offsets again and the arg-min
    long long carry = 0, pos = 0;
    for (int c = 0; c < pl.nch; ++c) {
      const unsigned long long* off = nullptr;
      if (T > 0) {
        if (c / kCountWindow != window) {
          window = c / kCountWindow;
          chunk_count_kernel<<<gblk, kGenThreads, 0, st>>>(s, K, bnd, T, window * kCountWindow, L.count);
          chunk_offsets_kernel<<<(unsigned)std::min(kCountWindow, pl.nch - window * kCountWindow), 256, 0, st>>>(
              L.count, pl.nblk);
          launches += 2;
        }
        off = L.count + (size_t)(c % kCountWindow) * pl.nblk;
      }
      const long long m = (c + 1 < pl.nch) ? pl.C : pl.M - (long long)c * pl.C;
      chunk_gen_kernel<<<gblk, kGenThreads, 0, st>>>(s, K, bnd, T, c, off, L.key[0], L.val[0]);
      cub::DoubleBuffer<double> dk(L.key[0], L.key[1]);
      cub::DoubleBuffer<uint32_t> dv(L.val[0], L.val[1]);
      size_t temp = L.cub_bytes;
      cub::DeviceRadixSort::SortPairs(L.cub_temp, temp, dk, dv, (int)m, 0, 64, st);
      const uint32_t* seq = dv.Current() - carry;
      if (carry) cudaMemcpyAsync((void*)seq, L.carry, (size_t)carry * 4, cudaMemcpyDeviceToDevice, st);
      const long long len = carry + m;
      const bool last = c + 1 == pl.nch;
      const long long nt = last ? (len + kTileElems - 1) / kTileElems : len / kTileElems;
      if (nt > 0) {
        tile_sums_kernel<<<(unsigned)nt, kTileThreads, 0, st>>>(seq, len, s, L.tile_sum);
        tile_scan_kernel<true><<<1, 32, 0, st>>>(L.tile_sum, nt, pos ? L.acc : nullptr, L.acc);
        launches += 2;
        if (sweep == 1) {
          tile_cost_kernel<<<(unsigned)nt, kTileThreads, 0, st>>>(seq, len, s, L.tile_sum, L.grand, L.tile_best);
          final_argmin_kernel<true><<<1, 32, 0, st>>>(L.tile_best, nt, pos, pos ? L.best : nullptr, L.best, out);
          launches += 2;
        }
      }
      carry = len - nt * kTileElems;
      if (!last && carry)
        cudaMemcpyAsync(L.carry, seq + nt * kTileElems, (size_t)carry * 4, cudaMemcpyDeviceToDevice, st);
      pos += nt * kTileElems;
      launches += 1 + 8;
    }
    if (sweep == 0) cudaMemcpyAsync(L.grand, L.acc, sizeof(Sums), cudaMemcpyDeviceToDevice, st);
  }
  return launches;
}

}  // namespace

constexpr int kScaleSmallN = 256;  // single-CTA bitonic sort + sequential one-thread sweep up to here (bit-exact vs the
                                   // reference's order; ~1 ms at 256), radix-sort + parallel-scan pipeline above
// Up to here the pipeline sorts stored ratios and ranges at once (64 B per TIM, 2.1 GB at 8192: faster than
// regenerating them, DESIGN.md §3.4); above it, or with a forced chunk capacity, the regenerating chunked route.
constexpr int kScaleArrayMaxN = 8192;
bool scale_stream(int n, long long chunk) { return n > kScaleArrayMaxN || chunk != 0; }
// debug flag 262144: the large path at every size (same results within the rounding of its summation tree)
bool scale_large(int n, uint32_t flags) { return n > kScaleSmallN || (flags & 262144u); }

size_t tls_scratch_bytes(long long m, int count, bool large) {
  if (2 * m >= (1LL << 31)) return 0;  // end-point payloads are ints
  if (large) return tls_large_scratch_bytes(m);
  return (size_t)count * next_pow2((int)(2 * m)) * (sizeof(double) + sizeof(int32_t));
}

// scratch: tls_scratch_bytes(m, 1, large) bytes (small path: the keys, then the payloads)
int launch_scalar_tls(const double* x, const double* ranges, long long m, bool large, void* scratch, double* out_est,
                      uint8_t* inliers, cudaStream_t st) {
  if (!large) {
    double* key = (double*)scratch;
    scalar_tls_kernel<<<1, 1024, 0, st>>>(x, ranges, m, key, (int32_t*)(key + next_pow2((int)(2 * m))), out_est,
                                          inliers);
    return 1;
  }
  const int nl = launch_tls_large(x, ranges, m, scratch, out_est, st);
  tls_inliers_kernel<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(x, ranges, m, out_est, inliers);
  return nl + 1;
}

// Layout: ratios X and ranges Rg (K doubles per problem), then the sort scratch (256-byte aligned).  The small path holds
// every problem of the batch, the large path one problem at a time (its sort uses the whole GPU).  The regenerating
// route: its chunks' scratch for one problem at a time, at most stream_layout of kChunkAuto end points.
size_t scale_scratch_bytes(int B, int n, uint32_t flags, long long chunk) {
  const bool large = scale_large(n, flags);
  const long long K = (long long)n * (n - 1) / 2;
  if (large && scale_stream(n, chunk)) return stream_layout(stream_plan(K, chunk), nullptr).total;
  const int sets = large ? 1 : B;
  return align256((size_t)sets * K * 16) + tls_scratch_bytes(K, sets, large);
}

int launch_scale_estimation(const Batch& bt, uint32_t flags, long long chunk, void* scratch, int* chunks,
                            cudaStream_t st) {
  const int n = bt.n;
  if (n < 2) return 0;
  const long long K = (long long)n * (n - 1) / 2;
  if (!scale_large(n, flags)) {
    double* X = (double*)scratch;
    double* Rg = X + (size_t)bt.B * K;
    double* key = (double*)((char*)scratch + align256((size_t)bt.B * K * 16));
    scale_pairs_kernel<<<dim3((unsigned)(n - 1), (unsigned)bt.B), 256, 0, st>>>(bt, X, Rg);
    scale_tls_kernel<<<bt.B, 1024, 0, st>>>(bt, X, Rg, key, (int32_t*)(key + (size_t)bt.B * next_pow2((int)(2 * K))));
    return 2;
  }
  const bool stream = scale_stream(n, chunk);  // from the class's n: every problem of a class takes one route
  double* X = (double*)scratch;
  double* Rg = X + (size_t)K;
  char* sort = (char*)scratch + align256((size_t)K * 16);
  int launches = 0;
  for (int b = 0; b < bt.B; ++b) {
    Batch one = bt;  // view of problem b (its own size in a ragged class)
    one.B = 1;
    one.n = bt.nb_host ? bt.nb_host[b] : n;
    one.nb = nullptr;
    one.src = bt.src + (size_t)b * n * 3;
    one.dst = bt.dst + (size_t)b * n * 3;
    if (one.n < 2) continue;
    const long long Kb = (long long)one.n * (one.n - 1) / 2;
    int nch = 1;
    if (stream) {
      launches += launch_tls_stream(TimTls{one.src, one.dst, one.n, bt.beta}, Kb, chunk, scratch, &bt.sol[b].scale,
                                    &nch, st);
    } else {
      scale_pairs_kernel<<<(unsigned)(one.n - 1), 256, 0, st>>>(one, X, Rg);
      launches += 1 + launch_tls_large(X, Rg, Kb, sort, &bt.sol[b].scale, st);
    }
    *chunks = std::max(*chunks, nch);
  }
  return launches;
}

}  // namespace tzr
