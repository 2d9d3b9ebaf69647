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
//    call on this path, cub::DeviceRadixSort, flagged as such in DESIGN.md — followed by hand-written,
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
__device__ __forceinline__ Sums endpoint_terms(int e, const double* __restrict__ X, const double* __restrict__ Rg,
                                               bool* kept) {
  const long long id = e >> 1;
  const double eps = (e & 1) ? -1.0 : 1.0;
  const double r = Rg[id], x = X[id];
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

__global__ void __launch_bounds__(kTileThreads) tile_sums_kernel(const int* __restrict__ val, long long M,
                                                                 const double* __restrict__ X,
                                                                 const double* __restrict__ Rg, Sums* tile_sum) {
  __shared__ Sums s_warp[kTileThreads / 32 + 1];
  const long long base = (long long)blockIdx.x * kTileElems + (long long)threadIdx.x * kPerThread;
  Sums acc = sums_zero();
  for (int k = 0; k < kPerThread; ++k) {
    const long long q = base + k;
    bool kept;
    if (q < M) acc = sums_add(acc, endpoint_terms(val[q], X, Rg, &kept));
  }
  Sums total;
  block_excl_scan_sums(acc, s_warp, &total);
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

// exclusive scan of the tile sums, sequential on one thread (deterministic; <= a few hundred thousand tiles)
__global__ void tile_scan_kernel(Sums* tile_sum, long long n_tiles, Sums* grand_total) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  Sums acc = sums_zero();
  for (long long t = 0; t < n_tiles; ++t) {
    const Sums v = tile_sum[t];
    tile_sum[t] = acc;
    acc = sums_add(acc, v);
  }
  *grand_total = acc;
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

__global__ void __launch_bounds__(kTileThreads) tile_cost_kernel(const int* __restrict__ val, long long M,
                                                                 const double* __restrict__ X,
                                                                 const double* __restrict__ Rg,
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
    terms[k] = (q < M) ? endpoint_terms(val[q], X, Rg, &kept[k]) : sums_zero();
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

__global__ void final_argmin_kernel(const Best* tile_best, long long n_tiles, double* out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  Best bb = tile_best[0];
  for (long long t = 1; t < n_tiles; ++t)
    if (best_less(tile_best[t], bb)) bb = tile_best[t];
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
  return (size_t)M * (8 + 8 + 4 + 4) + temp + (size_t)n_tiles * (sizeof(Sums) + sizeof(Best)) + sizeof(Sums) + 1024;
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
  make_endpoints_kernel<<<(unsigned)((M + 255) / 256), 256, 0, st>>>(X, Rg, K, key_in, val_in);
  cub::DeviceRadixSort::SortPairs(cub_temp, temp, key_in, key_out, val_in, val_out, (int)M, 0, 64, st);
  tile_sums_kernel<<<(unsigned)n_tiles, kTileThreads, 0, st>>>(val_out, M, X, Rg, tile_sum);
  tile_scan_kernel<<<1, 32, 0, st>>>(tile_sum, n_tiles, grand);
  tile_cost_kernel<<<(unsigned)n_tiles, kTileThreads, 0, st>>>(val_out, M, X, Rg, tile_sum, grand, tile_best);
  final_argmin_kernel<<<1, 32, 0, st>>>(tile_best, n_tiles, out);
  return 5 + 8;
}

size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

}  // namespace

constexpr int kScaleSmallN = 256;  // single-CTA bitonic sort + sequential one-thread sweep up to here (bit-exact vs the
                                   // reference's order; ~1 ms at 256), radix-sort + parallel-scan pipeline above
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
// every problem of the batch, the large path one problem at a time (its sort uses the whole GPU).
size_t scale_scratch_bytes(int B, int n, uint32_t flags) {
  const bool large = scale_large(n, flags);
  const long long K = (long long)n * (n - 1) / 2;
  const int sets = large ? 1 : B;
  const size_t sort = tls_scratch_bytes(K, sets, large);
  return sort ? align256((size_t)sets * K * 16) + sort : 0;
}

int launch_scale_estimation(const Batch& bt, uint32_t flags, void* scratch, cudaStream_t st) {
  const int n = bt.n;
  if (n < 2) return 0;
  const bool large = scale_large(n, flags);
  const long long K = (long long)n * (n - 1) / 2;
  const int sets = large ? 1 : bt.B;
  double* X = (double*)scratch;
  double* Rg = X + (size_t)sets * K;
  char* sort = (char*)scratch + align256((size_t)sets * K * 16);
  if (!large) {
    double* key = (double*)sort;
    scale_pairs_kernel<<<dim3((unsigned)(n - 1), (unsigned)bt.B), 256, 0, st>>>(bt, X, Rg);
    scale_tls_kernel<<<bt.B, 1024, 0, st>>>(bt, X, Rg, key, (int32_t*)(key + (size_t)bt.B * next_pow2((int)(2 * K))));
    return 2;
  }
  int launches = 0;
  for (int b = 0; b < bt.B; ++b) {
    Batch one = bt;  // view of problem b (its own size in a ragged class) for the pairs kernel
    one.B = 1;
    one.n = bt.nb_host ? bt.nb_host[b] : n;
    one.nb = nullptr;
    one.src = bt.src + (size_t)b * n * 3;
    one.dst = bt.dst + (size_t)b * n * 3;
    if (one.n < 2) continue;
    scale_pairs_kernel<<<(unsigned)(one.n - 1), 256, 0, st>>>(one, X, Rg);
    launches += 1 + launch_tls_large(X, Rg, (long long)one.n * (one.n - 1) / 2, sort, &bt.sol[b].scale, st);
  }
  return launches;
}

}  // namespace tzr
