// Correspondence generation upstream of solve(): teaser::Matcher::calculateCorrespondences
// (reference teaser/src/matcher.cc:21-337) on the device.
//
//   nn_kernel            exact FP32 1-NN of every query feature among a database of features, brute force, with
//                        flann::L2<float>'s accumulation order (groups of four, then the tail) so that distances —
//                        and therefore the argmin — are the ones the reference's exact KD-tree search compares.
//                        Result merged across database segments with one 64-bit atomicMin on (distance bits, index):
//                        the lowest index wins among equal distances.
//   mean/normalize       normalizePoints (matcher.cc:55-113): float, sequential accumulation for the mean.
//   corres_kernel        i_to_j / corres_ij ++ corres_ji / cross check (matcher.cc:152-215) with an ordered compaction.
//   tuple_kernel         the tuple test (matcher.cc:223-281), one thread per trial, counter-based draws.
//   finalize             swap back, sort (CUB radix sort, the only library call), unique (matcher.cc:283-297).
//
// The kNN over 33-D descriptors is 0.8 G multiply-adds at 5000 x 5000: microseconds on the FP32 pipes and exact,
// which the tensor-core route (TF32/BF16 products) is not — it would need the same "filter + exact recheck" split as
// the graph stage for no measurable gain at these sizes.
//
// Batches: every kernel works over B pairs stored back to back (flat source and target arrays, a MatchPair table with
// each pair's offsets); a single call is the B = 1 case of the same launches, and the number of launches does not
// depend on B.  Pair b owns the slots [s_off + d_off, s_off + d_off + ns + nd) of every per-slot array.
#include <algorithm>

#include <cub/cub.cuh>

#include "tzr_internal.cuh"

namespace tzr {

namespace {

constexpr int kNnTile = 64;      // queries per CTA and database points per smem tile
constexpr int kNnThreads = 256;  // 16 x 16 threads, 4 x 4 pairs each

__device__ __forceinline__ unsigned long long pack_dist(float d, int idx) {
  unsigned int bits = (d != d) ? 0x7fc00000u : __float_as_uint(d);  // distances are >= 0: bit order == value order
  return ((unsigned long long)bits << 32) | (unsigned int)idx;
}

// One CTA per work item: 64 query rows against one database segment.  dynamic smem: Qs[dim][64] | Ds[dim][64]
__global__ void __launch_bounds__(kNnThreads) nn_kernel(const NnWork* __restrict__ work,
                                                        const float* __restrict__ feat_a,
                                                        const float* __restrict__ feat_b, int dim,
                                                        unsigned long long* __restrict__ best_a,
                                                        unsigned long long* __restrict__ best_b) {
  extern __shared__ float nn_smem[];
  float* Qs = nn_smem;
  float* Ds = nn_smem + (size_t)dim * kNnTile;
  const NnWork wk = work[blockIdx.x];
  const float* __restrict__ query = wk.dir ? feat_b : feat_a;
  const float* __restrict__ db = wk.dir ? feat_a : feat_b;
  unsigned long long* __restrict__ best = wk.dir ? best_b : best_a;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int q0 = wk.q0, nq = wk.q_end;
  const int seg_lo = wk.seg_lo, seg_hi = wk.seg_hi;
  // transposing loads: consecutive threads take consecutive points (conflict-free smem stores; the strided global
  // reads of one 64 x dim tile stay within 64*dim*4 contiguous bytes and are served by L1 after the first touch)
  for (int e = tid; e < dim * kNnTile; e += kNnThreads) {
    const int k = e / kNnTile, q = e - k * kNnTile;
    Qs[e] = (q0 + q < nq) ? query[(size_t)(q0 + q) * dim + k] : 0.f;
  }
  unsigned long long mine[4] = {~0ull, ~0ull, ~0ull, ~0ull};
  const int dim4 = dim & ~3;
  for (int d0 = seg_lo; d0 < seg_hi; d0 += kNnTile) {
    __syncthreads();
    for (int e = tid; e < dim * kNnTile; e += kNnThreads) {
      const int k = e / kNnTile, p = e - k * kNnTile;
      Ds[e] = (d0 + p < seg_hi) ? db[(size_t)(d0 + p) * dim + k] : 0.f;
    }
    __syncthreads();
    float acc[4][4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int v = 0; v < 4; ++v) acc[u][v] = 0.f;
    for (int k = 0; k < dim4; k += 4) {
      float g[4][4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const float4 qv = *reinterpret_cast<const float4*>(Qs + (k + kk) * kNnTile + ty * 4);
        const float4 dv = *reinterpret_cast<const float4*>(Ds + (k + kk) * kNnTile + tx * 4);
        const float qa[4] = {qv.x, qv.y, qv.z, qv.w}, da[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int v = 0; v < 4; ++v) {
            const float df = __fsub_rn(qa[u], da[v]);
            const float sq = __fmul_rn(df, df);
            g[u][v] = (kk == 0) ? sq : __fadd_rn(g[u][v], sq);  // ((d0^2 + d1^2) + d2^2) + d3^2
          }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) acc[u][v] = __fadd_rn(acc[u][v], g[u][v]);
    }
    for (int k = dim4; k < dim; ++k) {
      const float4 qv = *reinterpret_cast<const float4*>(Qs + k * kNnTile + ty * 4);
      const float4 dv = *reinterpret_cast<const float4*>(Ds + k * kNnTile + tx * 4);
      const float qa[4] = {qv.x, qv.y, qv.z, qv.w}, da[4] = {dv.x, dv.y, dv.z, dv.w};
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          const float df = __fsub_rn(qa[u], da[v]);
          acc[u][v] = __fadd_rn(acc[u][v], __fmul_rn(df, df));
        }
    }
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int p = d0 + tx * 4 + v;
      if (p < seg_hi) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const unsigned long long key = pack_dist(acc[u][v], p - wk.db_lo);
          mine[u] = key < mine[u] ? key : mine[u];
        }
      }
    }
  }
  // the 16 threads sharing ty are 16 consecutive lanes of one warp
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    unsigned long long m = mine[u];
#pragma unroll
    for (int off = 8; off >= 1; off >>= 1) {
      const unsigned long long o = __shfl_xor_sync(0xffffffffu, m, off);
      m = o < m ? o : m;
    }
    const int q = q0 + ty * 4 + u;
    if (tx == 0 && q < nq) atomicMin(&best[q], m);
  }
}

__global__ void fill_u64_kernel(unsigned long long* p, long long n, unsigned long long v) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    p[i] = v;
}

// the pair of flat row r of the target (dst) or source arrays: the last b whose rows start at or before r
__device__ __forceinline__ int pair_of_row(const MatchPair* __restrict__ P, int B, int r, bool dst) {
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if ((dst ? P[mid].d_off : P[mid].s_off) <= r) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// the pair of slot c (pair b's slots start at s_off + d_off)
__device__ __forceinline__ int pair_of_slot(const MatchPair* __restrict__ P, int B, int c) {
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (P[mid].s_off + P[mid].d_off <= c) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// One CTA of two warps per pair, warp c for cloud c (source, target): the sequential float sum of every coordinate in
// index order, then / n (matcher.cc:62-72).  The lanes load 32 points at a time (the next 32 are in flight while the
// current ones are summed) and every lane runs the same three addition chains over them through shuffles, so the
// loop waits on the FP32 adds rather than on one load after another.
__global__ void __launch_bounds__(64) mean_kernel(const MatchPair* __restrict__ P, const float* src,
                                                  const float* dst, float* mean) {
  const int b = blockIdx.x, c = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const MatchPair pr = P[b];
  const float* p = c ? dst + 3 * (size_t)pr.d_off : src + 3 * (size_t)pr.s_off;
  const int n = c ? pr.nd : pr.ns;
  auto load = [&](int i, float* v) {
    v[0] = v[1] = v[2] = 0.f;
    if (i < n)
      for (int k = 0; k < 3; ++k) v[k] = p[3 * (size_t)i + k];
  };
  float s[3] = {0.f, 0.f, 0.f}, cur[3], nxt[3];
  load(lane, cur);
  for (int i = 0; i < n; i += 32) {
    load(i + 32 + lane, nxt);
    const int m = min(32, n - i);
#pragma unroll
    for (int u = 0; u < 32; ++u) {
      float v[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) v[k] = __shfl_sync(0xffffffffu, cur[k], u);
      if (u < m)
#pragma unroll
        for (int k = 0; k < 3; ++k) s[k] = __fadd_rn(s[k], v[k]);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) cur[k] = nxt[k];
  }
  if (lane < 3) mean[6 * (size_t)b + 3 * c + lane] = __fdiv_rn(lane == 0 ? s[0] : lane == 1 ? s[1] : s[2], (float)n);
}

// subtract the pair's mean in place and fold max ||p|| into the pair's scale_bits (non-negative floats: uint order ==
// float order); a warp whose lanes share one pair reduces before its atomic
__global__ void center_kernel(const MatchPair* __restrict__ P, int B, int NS, int ND, float* src, float* dst,
                              const float* mean, unsigned int* scale_bits) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float t = 0.f;
  int b = -1;
  if (i < NS + ND) {
    const int c = i >= NS;
    const int r = c ? i - NS : i;
    b = pair_of_row(P, B, r, c);
    float* p = (c ? dst : src) + 3 * (size_t)r;
    const float* m = mean + 6 * (size_t)b + 3 * c;
    const float x = __fsub_rn(p[0], m[0]), y = __fsub_rn(p[1], m[1]), z = __fsub_rn(p[2], m[2]);
    p[0] = x;
    p[1] = y;
    p[2] = z;
    t = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
    if (!(t == t)) t = 0.f;  // NaN never wins `temp > max_scale`
  }
  const bool uniform = __all_sync(0xffffffffu, b == __shfl_sync(0xffffffffu, b, 0));
  if (uniform) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, off));
  }
  if ((!uniform || (threadIdx.x & 31) == 0) && t > 0.f) atomicMax(&scale_bits[b], __float_as_uint(t));
}

__global__ void rescale_kernel(const MatchPair* __restrict__ P, int B, int NS, int ND, float* src, float* dst,
                               const unsigned int* scale_bits, int use_absolute_scale, float* gscale_out) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= 3ll * (NS + ND)) return;
  const int c = e >= 3ll * NS;
  const long long ec = c ? e - 3ll * NS : e;
  const int b = pair_of_row(P, B, (int)(ec / 3), c);
  const float g = use_absolute_scale ? 1.0f : __uint_as_float(scale_bits[b]);
  if (!c && ec == 3ll * P[b].s_off) gscale_out[b] = g;
  if (g == 1.0f) return;
  float* p = c ? dst : src;
  p[ec] = __fdiv_rn(p[ec], g);
}

// Block-wide ordered compaction helper: returns the exclusive prefix of `flag` over the CTA's threads and the total.
__device__ int block_excl_scan(int flag, int* total, int* s_warp /*[33]*/) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const unsigned int bal = __ballot_sync(0xffffffffu, flag);
  const int in_warp = __popc(bal & ((1u << lane) - 1u));
  __syncthreads();
  if (lane == 0) s_warp[wid] = __popc(bal);
  __syncthreads();
  if (wid == 0) {
    int v = lane < nw ? s_warp[lane] : 0;
    int incl = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += o;
    }
    s_warp[lane] = incl - v;
    if (lane == 31) s_warp[32] = incl;
  }
  __syncthreads();
  *total = s_warp[32];
  return s_warp[wid] + in_warp;
}

// hit[i] of every pair (zeroed before): some j has i as its nearest neighbour.  One thread per row of the batch; the
// j rows are the target rows of a pair, or its source rows when the target cloud is the larger ("i").
__global__ void hit_kernel(const MatchPair* __restrict__ P, int B, int NS, int ND, const unsigned long long* best,
                           uint8_t* hit_all) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= NS + ND) return;
  const int c = row >= NS;
  const MatchPair pr = P[pair_of_row(P, B, c ? row - NS : row, c)];
  if ((c == 1) == (pr.nd > pr.ns)) return;  // an i row
  hit_all[(size_t)pr.s_off + pr.d_off + (unsigned int)best[row]] = 1;
}

// One CTA per pair.  Slots (matcher.cc:152-215): without cross check,
// slot i < n_i is (i, i_to_j[i]) when i was hit, slot n_i + j is (nn_of_j[j], j); with cross check, slot i is
// (i, i_to_j[i]) when hit and nn_of_j[i_to_j[i]] == i.  corres[] receives the valid slots in slot order (the order the
// reference's vectors have), ncorr their number.
__global__ void __launch_bounds__(1024) corres_kernel(const MatchPair* __restrict__ P,
                                                      const unsigned long long* best_src,
                                                      const unsigned long long* best_dst, uint8_t* hit_all,
                                                      int crosscheck, int2* corres_all, int* ncorr) {
  __shared__ int s_warp[33];
  const MatchPair pr = P[blockIdx.x];
  const bool swapped = pr.nd > pr.ns;  // the larger cloud is "i" (matcher.cc:121-126)
  const int n_i = swapped ? pr.nd : pr.ns, n_j = swapped ? pr.ns : pr.nd;
  // best_j: NN of every j among the i features; best_i: NN of every i among the j features
  const unsigned long long* best_j = swapped ? best_src + pr.s_off : best_dst + pr.d_off;
  const unsigned long long* best_i = swapped ? best_dst + pr.d_off : best_src + pr.s_off;
  const size_t so = (size_t)pr.s_off + pr.d_off;
  const uint8_t* hit = hit_all + so;
  int2* corres = corres_all + so;
  const int slots = crosscheck ? n_i : n_i + n_j;
  int base = 0;
  for (int s0 = 0; s0 < slots; s0 += blockDim.x) {
    const int s = s0 + threadIdx.x;
    int flag = 0;
    int2 pc = make_int2(0, 0);
    if (s < slots) {
      if (s < n_i) {
        if (hit[s]) {
          const int j = (int)(unsigned int)best_i[s];
          pc = make_int2(s, j);
          flag = crosscheck ? ((int)(unsigned int)best_j[j] == s) : 1;
        }
      } else {
        const int j = s - n_i;
        pc = make_int2((int)(unsigned int)best_j[j], j);
        flag = 1;
      }
    }
    int total;
    const int pos = block_excl_scan(flag, &total, s_warp);
    if (flag) corres[base + pos] = pc;
    base += total;
  }
  if (threadIdx.x == 0) ncorr[blockIdx.x] = base;
}

__device__ __forceinline__ float dist3(const float* a, const float* b) {
  const float x = __fsub_rn(a[0], b[0]), y = __fsub_rn(a[1], b[1]), z = __fsub_rn(a[2], b[2]);
  return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}

// matcher.cc:223-281: 100 * ncorr_b trials per pair; a passing triple keeps its three correspondences.  The trials of
// all pairs form one sequence dealt round-robin over the grid's threads (pair b's trial t is that sequence's entry
// sum_{b' < b} trials_b' + t), so a batch of small pairs spreads as evenly as one large pair.
__global__ void tuple_kernel(const MatchPair* __restrict__ P, int B, const int2* corres_all, const int* ncorr,
                             const float* src, const float* dst, float scale, uint8_t* keep_all) {
  const long long gt = blockIdx.x * (long long)blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
  long long before = 0;
  for (int b = 0; b < B; ++b) {
    const long long nc = ncorr[b];
    const long long trials = nc * 100;
    long long t = (gt - before % stride) % stride;
    if (t < 0) t += stride;
    before += trials;
    if (t >= trials) continue;
    const MatchPair pr = P[b];
    const bool swapped = pr.nd > pr.ns;
    const float* pts_i = swapped ? dst + 3 * (size_t)pr.d_off : src + 3 * (size_t)pr.s_off;
    const float* pts_j = swapped ? src + 3 * (size_t)pr.s_off : dst + 3 * (size_t)pr.d_off;
    const size_t so = (size_t)pr.s_off + pr.d_off;
    const int2* corres = corres_all + so;
    uint8_t* keep = keep_all + so;
    for (; t < trials; t += stride) {
      long long r[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) r[k] = (long long)(splitmix64(pr.seed + 3ull * (uint64_t)t + k) >> 33) % nc;
      const int2 c0 = corres[r[0]], c1 = corres[r[1]], c2 = corres[r[2]];
      const float *a0 = pts_i + 3 * (size_t)c0.x, *a1 = pts_i + 3 * (size_t)c1.x, *a2 = pts_i + 3 * (size_t)c2.x;
      const float *b0 = pts_j + 3 * (size_t)c0.y, *b1 = pts_j + 3 * (size_t)c1.y, *b2 = pts_j + 3 * (size_t)c2.y;
      const float li0 = dist3(a0, a1), li1 = dist3(a1, a2), li2 = dist3(a2, a0);
      const float lj0 = dist3(b0, b1), lj1 = dist3(b1, b2), lj2 = dist3(b2, b0);
      if ((__fmul_rn(li0, scale) < lj0) && (lj0 < __fdiv_rn(li0, scale)) && (__fmul_rn(li1, scale) < lj1) &&
          (lj1 < __fdiv_rn(li1, scale)) && (__fmul_rn(li2, scale) < lj2) && (lj2 < __fdiv_rn(li2, scale))) {
        keep[r[0]] = 1;
        keep[r[1]] = 1;
        keep[r[2]] = 1;
      }
    }
  }
}

// keys[c] = pair << (bits_a + bits_b) | first << bits_b | second for kept correspondences, in the caller's (src, dst)
// order; pair << (bits_a + bits_b) | all ones (after every kept key of the pair) elsewhere.  One sort over the bits
// orders every pair inside its own slot range.
__global__ void keys_kernel(const MatchPair* __restrict__ P, int B, int C, const int2* corres, const int* ncorr,
                            const uint8_t* keep, int use_keep, int bits_a, int bits_b, unsigned long long* keys) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int b = pair_of_slot(P, B, c);
  const MatchPair pr = P[b];
  const int ab = bits_a + bits_b;
  unsigned long long k = ((unsigned long long)b << ab) | ((1ull << ab) - 1);
  if (c - (pr.s_off + pr.d_off) < ncorr[b] && (!use_keep || keep[c])) {
    const int2 q = corres[c];
    const bool swapped = pr.nd > pr.ns;
    const unsigned int first = swapped ? q.y : q.x, second = swapped ? q.x : q.y;
    k = ((unsigned long long)b << ab) | ((unsigned long long)first << bits_b) | second;
  }
  keys[c] = k;
}

// One CTA per pair: std::unique over the pair's sorted keys (matcher.cc:295-296) -> rows from the pair's first slot
// of out_pairs; counts[b].
__global__ void __launch_bounds__(1024) unique_kernel(const MatchPair* __restrict__ P,
                                                      const unsigned long long* keys_sorted, int bits_a, int bits_b,
                                                      int32_t* out_pairs, int* counts) {
  __shared__ int s_warp[33];
  const MatchPair pr = P[blockIdx.x];
  const size_t so = (size_t)pr.s_off + pr.d_off;
  const int cap = pr.ns + pr.nd;
  const unsigned long long* keys = keys_sorted + so;
  int32_t* pairs = out_pairs + 2 * so;
  const unsigned long long low = (1ull << (bits_a + bits_b)) - 1;
  int base = 0;
  for (int s0 = 0; s0 < cap; s0 += blockDim.x) {
    const int s = s0 + threadIdx.x;
    int flag = 0;
    unsigned long long k = ~0ull;
    if (s < cap) {
      k = keys[s];
      flag = ((k & low) != low) && (s == 0 || keys[s - 1] != k);
    }
    int total;
    const int pos = block_excl_scan(flag, &total, s_warp);
    if (flag) {
      pairs[2 * (size_t)(base + pos)] = (int32_t)((k >> bits_b) & ((1ull << bits_a) - 1));
      pairs[2 * (size_t)(base + pos) + 1] = (int32_t)(k & ((1ull << bits_b) - 1));
    }
    base += total;
  }
  if (threadIdx.x == 0) counts[blockIdx.x] = base;
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

int bits_for(long long x) {  // bits that hold every value in [0, x]
  int b = 0;
  while (b < 63 && (1ll << b) <= x) ++b;
  return b;
}

}  // namespace

int nn_tiles_per_seg(long long tile_pairs, int ctas) {
  return (int)std::max<long long>(1, (tile_pairs + ctas - 1) / ctas);
}

void nn_work_append(std::vector<NnWork>* work, int dir, int q_lo, int nq, int db_lo, int ndb, int tiles_per_seg) {
  const int db_tiles = (ndb + kNnTile - 1) / kNnTile;
  const int segs = (db_tiles + tiles_per_seg - 1) / tiles_per_seg;
  const int seg_rows = (db_tiles + segs - 1) / segs * kNnTile;  // equal segments: the longest one sets the time
  for (int q0 = q_lo; q0 < q_lo + nq; q0 += kNnTile)
    for (int s = db_lo; s < db_lo + ndb; s += seg_rows)
      work->push_back(NnWork{dir, q0, q_lo + nq, db_lo, s, std::min(db_lo + ndb, s + seg_rows)});
}

// best_a (and best_b, when the work list has direction 1) are n_best contiguous entries, reset here.
int launch_feature_nn(const NnWork* work, int n_work, const float* feat_a, const float* feat_b, int dim,
                      unsigned long long* best_a, unsigned long long* best_b, long long n_best, cudaStream_t st) {
  const size_t smem = (size_t)2 * dim * kNnTile * sizeof(float);
  if (smem > 48 * 1024)  // per device and cheap: no process-wide "already set" flag (one context per GPU is allowed)
    cudaFuncSetAttribute(nn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * kMatchMaxDim * kNnTile * 4);
  fill_u64_kernel<<<(int)std::min<long long>(1024, (n_best + 255) / 256), 256, 0, st>>>(best_a, n_best, ~0ull);
  nn_kernel<<<n_work, kNnThreads, smem, st>>>(work, feat_a, feat_b, dim, best_a, best_b);
  return 2;
}

int match_plan(int B, const int32_t* ns, const int32_t* nd, const uint64_t* seeds, int num_sms,
               std::vector<MatchPair>* pairs, std::vector<NnWork>* work, MatchPlan* plan) {
  long long S = 0, D = 0, tile_pairs = 0;
  int ns_max = 0, nd_max = 0;
  pairs->resize(B);
  for (int b = 0; b < B; ++b) {
    (*pairs)[b] = MatchPair{(int)S, ns[b], (int)D, nd[b], seeds[b]};
    S += ns[b];
    D += nd[b];
    if (S + D > 0x7fffffffll) return TZR_ERR_TOO_LARGE;
    ns_max = std::max(ns_max, ns[b]);
    nd_max = std::max(nd_max, nd[b]);
    tile_pairs += 2ll * ((ns[b] + kNnTile - 1) / kNnTile) * ((nd[b] + kNnTile - 1) / kNnTile);
  }
  plan->B = B;
  plan->NS = (int)S;
  plan->ND = (int)D;
  plan->bits_a = bits_for(ns_max);  // every source index is below ns_max: the all-ones field is free for the filler
  plan->bits_b = bits_for(nd_max);
  plan->bits = bits_for(B - 1) + plan->bits_a + plan->bits_b;
  if (plan->bits > 64) return TZR_ERR_TOO_LARGE;
  // both directions of every pair in one launch, about 8 CTAs per SM in all (4 per direction for a single pair)
  const int tps = nn_tiles_per_seg(tile_pairs, 8 * num_sms);
  work->clear();
  for (const MatchPair& p : *pairs) {
    nn_work_append(work, 0, p.s_off, p.ns, p.d_off, p.nd, tps);  // every source row among the pair's targets
    nn_work_append(work, 1, p.d_off, p.nd, p.s_off, p.ns, tps);  // every target row among the pair's sources
  }
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, cub_bytes, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                 (int)(S + D), 0, plan->bits);
  plan->cub_bytes = cub_bytes;
  return TZR_OK;
}

// Scratch layout (all device; C = NS + ND slots): best[C] u64 (sources, then targets) | keys[C] u64 |
// keys_sorted[C] u64 | corres[C] int2 | hit[C] | keep[C] | mean[6B] f32 | scale_bits[B] | ncorr[B] | cub temp
size_t match_scratch_bytes(const MatchPlan& plan) {
  const size_t C = (size_t)plan.NS + plan.ND, B = plan.B;
  return 4 * align256(C * 8) + 2 * align256(C) + align256(6 * B * 4) + 2 * align256(B * 4) +
         align256(plan.cub_bytes) + 1024;
}

int launch_match(const MatchPlan& plan, const MatchPair* pairs, const NnWork* work, int n_work, float* src_pts,
                 float* dst_pts, const float* src_feat, const float* dst_feat, int dim, int use_absolute_scale,
                 int use_crosscheck, int use_tuple_test, float tuple_scale, void* scratch, int32_t* out_pairs,
                 int* counts, float* gscale, int num_sms, cudaStream_t st) {
  const int B = plan.B, NS = plan.NS, ND = plan.ND, C = NS + ND;
  char* w = (char*)scratch;
  auto take = [&](size_t bytes) {
    char* p = w;
    w += align256(bytes);
    return p;
  };
  unsigned long long* best = (unsigned long long*)take((size_t)C * 8);
  unsigned long long* keys = (unsigned long long*)take((size_t)C * 8);
  unsigned long long* keys_sorted = (unsigned long long*)take((size_t)C * 8);
  int2* corres = (int2*)take((size_t)C * 8);
  uint8_t* hit = (uint8_t*)take((size_t)C);
  uint8_t* keep = (uint8_t*)take((size_t)C);
  float* mean = (float*)take((size_t)6 * B * 4);
  unsigned int* scale_bits = (unsigned int*)take((size_t)B * 4);
  int* ncorr = (int*)take((size_t)B * 4);
  void* cub_temp = (void*)w;
  size_t cub_bytes = plan.cub_bytes;
  int nl = 0;
  const bool tuple = use_tuple_test && tuple_scale != 0.f;
  // normalizePoints only feeds the tuple test, but global_scale_ is part of the observable state: always computed
  cudaMemsetAsync(scale_bits, 0, (size_t)B * 4, st);
  cudaMemsetAsync(hit, 0, (size_t)C, st);
  mean_kernel<<<B, 64, 0, st>>>(pairs, src_pts, dst_pts, mean);
  center_kernel<<<(C + 255) / 256, 256, 0, st>>>(pairs, B, NS, ND, src_pts, dst_pts, mean, scale_bits);
  rescale_kernel<<<(int)((3ll * C + 255) / 256), 256, 0, st>>>(pairs, B, NS, ND, src_pts, dst_pts, scale_bits,
                                                               use_absolute_scale, gscale);
  nl += 3;
  // NN of every source row among its pair's targets and of every target row among its pair's sources, in one launch;
  // the reference searches the reverse NN lazily for hit i only (:157-161), the unused ones are ignored by corres_kernel
  nl += launch_feature_nn(work, n_work, src_feat, dst_feat, dim, best, best + NS, C, st);
  hit_kernel<<<(C + 255) / 256, 256, 0, st>>>(pairs, B, NS, ND, best, hit);
  corres_kernel<<<B, 1024, 0, st>>>(pairs, best, best + NS, hit, use_crosscheck, corres, ncorr);
  nl += 2;
  if (tuple) {
    cudaMemsetAsync(keep, 0, (size_t)C, st);
    tuple_kernel<<<num_sms * 8, 256, 0, st>>>(pairs, B, corres, ncorr, src_pts, dst_pts, tuple_scale, keep);
    nl += 1;
  }
  keys_kernel<<<(C + 255) / 256, 256, 0, st>>>(pairs, B, C, corres, ncorr, keep, tuple ? 1 : 0, plan.bits_a,
                                               plan.bits_b, keys);
  cub::DeviceRadixSort::SortKeys(cub_temp, cub_bytes, keys, keys_sorted, C, 0, plan.bits, st);
  unique_kernel<<<B, 1024, 0, st>>>(pairs, keys_sorted, plan.bits_a, plan.bits_b, out_pairs, counts);
  nl += 3;
  return nl;
}

}  // namespace tzr
