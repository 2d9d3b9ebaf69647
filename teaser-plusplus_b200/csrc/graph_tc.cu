// Stage 1 of solve() on the tensor cores (Hopper warpgroup MMA): TIMs + scale-consistency test + inlier graph.
//
// Replaces (reference), exactly like graph_build.cu:
//   RobustRegistrationSolver::computeTIMs            teaser/src/registration.cc:512-551  (x2)
//   ScaleInliersSelector::solveForScale              teaser/src/registration.cc:427-443
//   inlier_graph_.addEdge loop                       teaser/src/registration.cc:614-619
//
// The CUDA-core kernel (graph_build.cu) spends ~20 issue slots per pair: twelve FP32 operations for the two squared
// TIM norms, two MUFU.SQRT, compares, ballots.  Here the squared norms come from the tensor cores instead:
//     a_ij = |s_i - s_j|^2 = n_i + n_j - 2 s_i.s_j      (and b_ij for the destination cloud)
// is a K = 3 (+2 for the norms) contraction.  Every centred coordinate (and every norm) is split into three tf32
// pieces h + m + l (11 significant bits each, so the split carries 33 bits of the FP64 value), and the products
// hh', hm', mh', mm', hl', lh' plus the six norm pieces are laid out as a K = 24 tf32 GEMM (three K = 8 wgmma steps
// per cloud): one 128x64 tile of a and of b is computed by two consumer warpgroups (64 rows each) into registers.  The
// operand tiles (tc_prep_kernel writes them once per problem in the exact shared-memory image the MMA descriptor
// wants: no-swizzle K-major planes) are staged by the TMA engine (cp.async.bulk -> UBLKCP) into a shared-memory ring
// by one producer warp, completion on mbarriers; two CTAs per SM overlap one CTA's MMAs with the other's epilogue.
//
// Epilogue (in the MMA's register fragments): with t = a-b, s = a+b, g = |sqrt a - sqrt b|, w = (sqrt a + sqrt b)^2
//     f = t^2 - 2 beta^2 s + beta^4 = (g^2 - beta^2)(w - beta^2)          edge  <=>  s <= beta^2  or  f <= 0
// a polynomial in the tensor-core values: no square root, no division, and its error is a Lipschitz bound
// (|f' - f| <= 2 E |t'| + E^2 + 2 beta^2 E for |a' - a| + |b' - b| <= E), so there are no guards for tiny norms.  Per pair:
// t, s, P = t^2 + beta^4, d = P - 2 beta^2 s, band = kap P + c0, d + band, d - band = 7 FP32 operations; the two sign
// bits go into the words whi (surely an edge) and wlo (not surely a non-edge) — no compare, no MUFU.  The four lanes
// that share a fragment row combine their bits so that each lane ends up owning one (row, 32-column) word.  whi is the
// tentative row word; wlo & ~whi are the pairs inside the error band (prep_kernel, DESIGN.md §3.1): they are queued and
// tc_patch_kernel re-evaluates them with the reference's exact FP64 sequence.  The transposed half of the bitset goes
// through a small shared-memory buffer and a warp bit transpose.
// Output (packed symmetric bitset, fused degrees) is bit-identical to graph_build.cu's and to the oracle's.
#include "tc_ptx.cuh"
#include "tzr_internal.cuh"

namespace tzr {

using namespace tc;

constexpr int kTcEpiWarps = 8;                        // two consumer warpgroups (MMA + epilogue): 64 rows of a tile each
constexpr int kTcThreads = 32 * (kTcEpiWarps + 1);    // + 1 producer warp (TMA issue by one elected lane)
constexpr int kTcN = 64;                              // columns of one tile (MMA N)
constexpr int kTcPlaneA = 128 * 16;                   // A role: 128 rows x 4 tf32 per plane
constexpr int kTcPlaneB = kTcN * 16;                  // B role: 64 rows x 4 tf32 per plane
constexpr int kTcCloudA = 6 * kTcPlaneA, kTcCloudB = 6 * kTcPlaneB;   // 6 planes = K 24
constexpr int kTcTileA = 2 * kTcCloudA;               // src + dst: 24 KB per 128-row block
constexpr int kTcTileB = 2 * kTcCloudB;               // 12 KB per 64-column block
constexpr int kTcBStages = 4;
constexpr int kTcTrBytes = 2 * kTile * 2 * 4;         // row words of a tile for the transposed half, double-buffered
constexpr int kTcSmemBytes = 2 * kTcTileA + kTcBStages * kTcTileB + 256 + kTcTrBytes;   // 98 KB: two CTAs per SM

__host__ __device__ inline size_t tc_a_bytes(int n) { return (size_t)((n + 127) / 128) * kTcTileA; }
// 64-column blocks per problem: the whole padded row pitch (2 per 128-block), so that every word of the bitset rows is
// written (all-zero operands past n give masked, i.e. zero, words)
__host__ __device__ inline int tc_nt64(int n) { return 2 * ((n + 127) / 128); }
__host__ __device__ inline size_t tc_b_bytes(int n) { return (size_t)tc_nt64(n) * kTcTileB; }
size_t tc_operand_bytes(int B, int n) { return (size_t)B * (tc_a_bytes(n) + tc_b_bytes(n)); }

// ------------------------------------------------------------------------------------------------
// operand tiles.  One thread per point; block (blk, b) covers 128 points.  Per problem: all A-role blocks (128 rows
// each), then all B-role blocks (64 rows each).
// A-role plane p of a cloud holds [c_x, c_y, c_z, w] per row with (piece, w) = (h,N0) (h,N1) (m,N2) (m,1) (h,1) (l,1);
// B-role: -2 x pieces (h,m,h,m,l,h) with w = 1,1,1,N0,N1,N2, so that sum_k A_ik B_jk = N_i + N_j - 2 (hh'+hm'+mh'+mm'+hl'+lh').
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float tf32_trunc(float f) { return __uint_as_float(__float_as_uint(f) & 0xFFFFE000u); }
__device__ __forceinline__ void split3(double v, float& h, float& m, float& l) {
  h = tf32_trunc((float)v);
  const double r1 = v - (double)h;
  m = tf32_trunc((float)r1);
  const double r2 = r1 - (double)m;
  l = tf32_trunc((float)r2);
}

__global__ void __launch_bounds__(128) tc_prep_kernel(Batch bt) {
  const int b = blockIdx.y, blk = blockIdx.x, r = threadIdx.x;
  const GraphConsts* gc = bt.gc + b;
  if (!gc->use_tc) return;
  const int n = bt.n;
  const int j = blk * kTile + r;
  uint8_t* base = reinterpret_cast<uint8_t*>(bt.opnd) + (size_t)b * (tc_a_bytes(n) + tc_b_bytes(n));
  float4* outA = reinterpret_cast<float4*>(base + (size_t)blk * kTcTileA);
  float4* outB = reinterpret_cast<float4*>(base + tc_a_bytes(n) + (size_t)(2 * blk + (r >> 6)) * kTcTileB);
  const int rb = r & 63;
  const double* src = bt.src + (size_t)b * n * 3;
  const double* dst = bt.dst + (size_t)b * n * 3;
#pragma unroll
  for (int cloud = 0; cloud < 2; ++cloud) {
    float c[3][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
    double nrm = 0;
    if (j < n) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double v = cloud == 0 ? (src[3 * j + k] - gc->cs[k]) * gc->s_hat : (dst[3 * j + k] - gc->cd[k]);
        split3(v, c[k][0], c[k][1], c[k][2]);
        const double rep = ((double)c[k][0] + (double)c[k][1]) + (double)c[k][2];
        nrm += rep * rep;
      }
    }
    float N0, N1, N2;
    split3(nrm, N0, N1, N2);
    float4* A = outA + cloud * (kTcCloudA / 16);
    float4* Bq = outB + cloud * (kTcCloudB / 16);
    const float one = j < n ? 1.f : 0.f;  // rows past n: all-zero operands (finite results, masked later)
    A[0 * 128 + r] = make_float4(c[0][0], c[1][0], c[2][0], N0);
    A[1 * 128 + r] = make_float4(c[0][0], c[1][0], c[2][0], N1);
    A[2 * 128 + r] = make_float4(c[0][1], c[1][1], c[2][1], N2);
    A[3 * 128 + r] = make_float4(c[0][1], c[1][1], c[2][1], one);
    A[4 * 128 + r] = make_float4(c[0][0], c[1][0], c[2][0], one);
    A[5 * 128 + r] = make_float4(c[0][2], c[1][2], c[2][2], one);
    {
      Bq[0 * kTcN + rb] = make_float4(-2.f * c[0][0], -2.f * c[1][0], -2.f * c[2][0], one);
      Bq[1 * kTcN + rb] = make_float4(-2.f * c[0][1], -2.f * c[1][1], -2.f * c[2][1], one);
      Bq[2 * kTcN + rb] = make_float4(-2.f * c[0][0], -2.f * c[1][0], -2.f * c[2][0], one);
      Bq[3 * kTcN + rb] = make_float4(-2.f * c[0][1], -2.f * c[1][1], -2.f * c[2][1], N0);
      Bq[4 * kTcN + rb] = make_float4(-2.f * c[0][2], -2.f * c[1][2], -2.f * c[2][2], N1);
      Bq[5 * kTcN + rb] = make_float4(-2.f * c[0][0], -2.f * c[1][0], -2.f * c[2][0], N2);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// tile schedule: a work item is a strip = (problem b, row block I of 128, S consecutive 64-column blocks J of the
// upper triangle, J >= 2I).  CTA c walks items c, c + gridDim.x, ...; the producer lane and the epilogue warps iterate
// the same sequence.
// ------------------------------------------------------------------------------------------------
struct TileIter {
  int item, step, total, spp, S, nt, nt64;
  int b, I, J, J1;
  bool first;
  __device__ __forceinline__ void init(int start, int step_, int total_, int spp_, int S_, int n) {
    item = start - step_;
    step = step_;
    total = total_;
    spp = spp_;
    S = S_;
    nt = (n + kTile - 1) / kTile;
    nt64 = tc_nt64(n);
    b = I = 0;
    J = J1 = 0;
    first = false;
  }
  __device__ __forceinline__ bool next() {
    if (J + 1 < J1) {
      ++J;
      first = false;
      return true;
    }
    item += step;
    if (item >= total) return false;
    b = item / spp;
    int p = item - b * spp;
    I = 0;
    while (true) {
      const int ng = (nt64 - 2 * I + S - 1) / S;
      if (p < ng) break;
      p -= ng;
      ++I;
    }
    J = 2 * I + p * S;
    J1 = min(nt64, J + S);
    first = true;
    return true;
  }
  __device__ __forceinline__ bool last_of_strip() const { return J + 1 == J1; }
};

__host__ __device__ inline int tc_strips_per_problem(int n, int S) {
  const int nt = (n + kTile - 1) / kTile, nt64 = tc_nt64(n);
  int total = 0;
  for (int I = 0; I < nt; ++I) total += (nt64 - 2 * I + S - 1) / S;
  return total;
}

struct TcConsts {
  float nc2, b4, kap, c0;  // -2 beta^2, beta^4, band slope, band offset (prep_kernel; DESIGN.md §3.1)
};

// The pair test on the 32 accumulator values of this thread (d[4 i + 2 r + c] = row r0 + 8 r, column 8 i + 2 (lane % 4)
// + c of the 64-column tile).  Per pair:
//   t = a - b, s = a + b, P = t^2 + beta^4, d = P - 2 beta^2 s  [= (g^2 - beta^2)(w - beta^2)],  band = kap P + c0,
//   d_hi = d + band  (sign bit 1: surely an edge),   d_lo = d - band  (sign bit 0: surely not an edge)
// = 7 FP32 operations, no MUFU, no compare.  whi[r][h] / wlo[r][h] bit k: this lane's sign bits of column 32 h + k.
__device__ __forceinline__ void tc_sweep(const float (&a)[32], const float (&b)[32], const TcConsts& k, int lane,
                                         uint32_t (&whi)[2][2], uint32_t (&wlo)[2][2]) {
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int h = 0; h < 2; ++h) whi[r][h] = wlo[r][h] = 0u;
#pragma unroll
  for (int e = 0; e < 32; ++e) {
    const int i = e >> 2, r = (e >> 1) & 1, pos = 8 * (i & 3) + (e & 1);
    const float t = __fsub_rn(a[e], b[e]), s = __fadd_rn(a[e], b[e]);
    const float P = __fmaf_rn(t, t, k.b4);
    const float d = __fmaf_rn(s, k.nc2, P);
    const float bd = __fmaf_rn(P, k.kap, k.c0);
    whi[r][i >> 2] |= (__float_as_uint(__fadd_rn(d, bd)) >> 31) << pos;
    wlo[r][i >> 2] |= (__float_as_uint(__fsub_rn(d, bd)) >> 31) << pos;
  }
  const int sh = 2 * (lane & 3);
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      whi[r][h] <<= sh;
      wlo[r][h] <<= sh;
    }
}

// The four lanes of a quad hold disjoint bits of the same four words (2 rows x 2 column halves).  Reduce-scatter in two
// exchanges: lane (lane & 3) = 2 mr + mh ends up with the complete word of row r0 + 8 mr, column half mh.
__device__ __forceinline__ uint32_t tc_quad_word(const uint32_t (&w)[2][2], int lane) {
  const int mr = (lane >> 1) & 1, mh = lane & 1;
  const uint32_t k0 = (mr ? w[1][0] : w[0][0]) | __shfl_xor_sync(0xffffffffu, mr ? w[0][0] : w[1][0], 2);
  const uint32_t k1 = (mr ? w[1][1] : w[0][1]) | __shfl_xor_sync(0xffffffffu, mr ? w[0][1] : w[1][1], 2);
  return (mh ? k1 : k0) | __shfl_xor_sync(0xffffffffu, mh ? k0 : k1, 1);
}

// 32x32 bit transpose across the lanes of a warp (lane l passes row l, receives column l)
__device__ __forceinline__ uint32_t tc_transpose32(uint32_t x, int lane) {
#pragma unroll
  for (int st = 0; st < 5; ++st) {
    const int j = 16 >> st;
    const uint32_t m = st == 0 ? 0x0000FFFFu : st == 1 ? 0x00FF00FFu : st == 2 ? 0x0F0F0F0Fu : st == 3 ? 0x33333333u
                                                                                                       : 0x55555555u;
    const uint32_t y = __shfl_xor_sync(0xffffffffu, x, j);
    if ((lane & j) == 0)
      x ^= (((x >> j) ^ y) & m) << j;
    else
      x ^= ((y >> j) ^ x) & m;
  }
  return x;
}

// barrier slots in shared memory
enum {
  kBarAFull = 0,                          // [2]  TMA -> MMA: A tile of the strip landed
  kBarAEmpty = 2,                         // [2]  consumer warps (8 arrivals) -> TMA: the strip's A tile was read for the last time
  kBarBFull = 4,                          // [kTcBStages]  TMA -> MMA
  kBarBEmpty = kBarBFull + kTcBStages,    // [kTcBStages]  consumer warps (8 arrivals) -> TMA: stage may be overwritten
  kNumBars = kBarBEmpty + kTcBStages
};

// 112 registers: two 288-thread CTAs per SM (64 512 of the 65 536 registers); the 64 accumulators of a thread fit without
// spills (at the 96 registers a (288, 2) launch bound gives, ptxas spills).
template <bool kVerify>
__global__ void __maxnreg__(112) graph_tc_kernel(Batch bt, int S, int spp, int total_items) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 2 * kTcTileA + kTcBStages * kTcTileB);
  uint32_t* s_tr = reinterpret_cast<uint32_t*>(smem + 2 * kTcTileA + kTcBStages * kTcTileB + 256);
  const uint32_t sA0 = smem_u32(smem), sB0 = smem_u32(smem + 2 * kTcTileA);
  const uint32_t bar0 = smem_u32(bars);
  auto bar = [&](int i) { return bar0 + 8u * (uint32_t)i; };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n = bt.n;
  if (tid == 0) {
    for (int i = 0; i < kNumBars; ++i)
      mbar_init(bar(i), (i >= kBarBEmpty || (i >= kBarAEmpty && i < kBarBFull)) ? kTcEpiWarps : 1);
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == kTcEpiWarps) {
    // ================= producer: TMA loads, up to kTcBStages tiles and two strips ahead of the MMAs =================
    if (lane == 0) {
      const uint8_t* opnd = reinterpret_cast<const uint8_t*>(bt.opnd);
      const size_t per_problem = tc_a_bytes(n) + tc_b_bytes(n), a_bytes = tc_a_bytes(n);
      TileIter ld;
      ld.init(blockIdx.x, gridDim.x, total_items, spp, S, n);
      uint32_t n_loaded = 0, n_strips_loaded = 0;
      int tc_b = -1;
      bool tc_ok = false;
      while (ld.next()) {
        if (ld.b != tc_b) {  // only tiles of problems that take the tensor-core path
          tc_b = ld.b;
          tc_ok = bt.gc[ld.b].use_tc != 0;
        }
        if (!tc_ok) continue;
        const uint32_t st = n_loaded % kTcBStages, use = n_loaded / kTcBStages;
        if (use > 0) mbar_wait(bar(kBarBEmpty + st), (use - 1) & 1u);  // the MMAs that read this stage are complete
        const uint8_t* pb = opnd + (size_t)ld.b * per_problem;
        if (ld.first) {
          // A buffer (strip index & 1): wait until the strip that used it two strips ago has been read completely
          const uint32_t a = n_strips_loaded & 1u;
          if (n_strips_loaded >= 2) mbar_wait(bar(kBarAEmpty + a), ((n_strips_loaded >> 1) - 1) & 1u);
          mbar_arrive_expect_tx(bar(kBarAFull + a), kTcTileA);
          bulk_g2s(sA0 + a * kTcTileA, pb + (size_t)ld.I * kTcTileA, kTcTileA, bar(kBarAFull + a));
          ++n_strips_loaded;
        }
        mbar_arrive_expect_tx(bar(kBarBFull + st), kTcTileB);
        bulk_g2s(sB0 + st * kTcTileB, pb + a_bytes + (size_t)ld.J * kTcTileB, kTcTileB, bar(kBarBFull + st));
        ++n_loaded;
      }
    }
    __syncwarp();
  } else {
    // ================= consumers: warpgroup g = warp / 4 computes rows 64 g .. 64 g + 63 of the 128-row block =========
    const int g = warp >> 2;
    const int mr = (lane >> 1) & 1, h = lane & 1;
    const int rloc = 64 * g + 16 * (warp & 3) + (lane >> 2) + 8 * mr;  // the row whose (32-column) word this lane owns
    TileIter ti;
    ti.init(blockIdx.x, gridDim.x, total_items, spp, S, n);
    uint32_t n_t = 0, n_strips = 0, n_tr = 0, ap = 0;
    int rdeg = 0;
    const int P32 = pitch32(n);
    TcConsts kc{0.f, 0.f, 0.f, 0.f};
    const GraphConsts* gcp = bt.gc;
    bool use_tc = false;
    uint32_t* adj32 = nullptr;  // bitset of the strip's problem
    uint32_t* rowp = nullptr;   // row i of it
    int* degp = nullptr;
    int i = 0;
    bool row_ok = false, row_edge = false;
    float acc[2][32];
#pragma unroll
    for (int e = 0; e < 32; ++e) acc[0][e] = acc[1][e] = 0.f;
    while (ti.next()) {
      if (ti.first) {  // per strip, not per tile
        gcp = bt.gc + ti.b;
        use_tc = gcp->use_tc != 0;
      }
      if (!use_tc) continue;
      const int I = ti.I, J = ti.J;
      if (ti.first) {
        kc.nc2 = -gcp->tc_c2;
        kc.b4 = gcp->tc_b4;
        kc.kap = gcp->tc_kap;
        kc.c0 = gcp->tc_c0;
        i = I * kTile + rloc;
        adj32 = reinterpret_cast<uint32_t*>(bt.adj) + (size_t)ti.b * n * P32;
        rowp = adj32 + (size_t)i * P32;
        degp = bt.deg + (size_t)ti.b * n;
        row_ok = i < n;
        row_edge = I * kTile + kTile > n;  // some rows of the block lie past n
        ap = n_strips & 1u;
        mbar_wait(bar(kBarAFull + ap), (n_strips >> 1) & 1u);
        ++n_strips;
      }
      const int j0 = J * kTcN + 32 * h;
      const uint32_t st = n_t % kTcBStages, use = n_t / kTcBStages;
      mbar_wait(bar(kBarBFull + st), use & 1u);
      // ---- a and b of the 64 x 64 sub-tile: K-major, no swizzle: leading byte offset = distance of the two 16-byte
      // K-chunks (planes), stride byte offset = distance of consecutive 8-row groups (128 B)
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        acc_fence(acc[0][e]);
        acc_fence(acc[1][e]);
      }
      wgmma_fence();
#pragma unroll
      for (int cloud = 0; cloud < 2; ++cloud)
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const uint64_t da = make_smem_desc(sA0 + ap * kTcTileA + cloud * kTcCloudA + s * 2 * kTcPlaneA + g * 64 * 16,
                                             kTcPlaneA, 128);
          const uint64_t db = make_smem_desc(sB0 + st * kTcTileB + cloud * kTcCloudB + s * 2 * kTcPlaneB, kTcPlaneB, 128);
          wgmma_m64n64k8_tf32(acc[cloud], da, db, s > 0);
        }
      wgmma_commit();
      wgmma_wait_all();
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        acc_fence(acc[0][e]);
        acc_fence(acc[1][e]);
      }
      __syncwarp();
      if (lane == 0) {  // this warp's reads of the B stage (and, at the end of a strip, of the A tile) are complete
        mbar_arrive(bar(kBarBEmpty + st));
        if (ti.last_of_strip()) mbar_arrive(bar(kBarAEmpty + ap));
      }
      // ---- sweep: whi bit k = pair (i, j0+k) surely an edge, wlo bit k = not surely a non-edge
      uint32_t whi, wlo;
      {
        uint32_t qh[2][2], ql[2][2];
        tc_sweep(acc[0], acc[1], kc, lane, qh, ql);
        whi = tc_quad_word(qh, lane);
        wlo = tc_quad_word(ql, lane);
      }
      // validity of the pairs of this thread: columns < n, row < n, i != j (interior tiles: everything valid)
      uint32_t vmask = 0xffffffffu;
      const bool diag = (J >> 1) == I;
      if (row_edge || diag || j0 + 32 > n) {
        vmask = j0 + 32 <= n ? 0xffffffffu : (j0 >= n ? 0u : ((1u << (n - j0)) - 1u));
        if (!row_ok) vmask = 0u;
        if (i >= j0 && i < j0 + 32) vmask &= ~(1u << (i - j0));
      }
      uint32_t word = whi & vmask;             // tentative classification: undecided pairs keep bit 0
      uint32_t fmask = wlo & ~whi & vmask;     // undecided: inside the error band of the tensor-core norms
      if (kVerify || __any_sync(0xffffffffu, fmask != 0u)) {
        // ---- the undecided pairs are queued for tc_patch_kernel, which evaluates the reference's exact FP64 sequence
        // and sets the bits of the edges among them — so no warp of this kernel waits for double-precision square roots.
        // (Queue full: evaluated here.)
        const int b = ti.b;
        const double* src = bt.src + (size_t)b * n * 3;
        const double* dst = bt.dst + (size_t)b * n * 3;
        const double beta = gcp->beta;
        const bool scale_mode = bt.scale_mode != 0;
        const double s_hat = scale_mode ? bt.sol[b].scale : 1.0;
        if (kVerify) {  // every DECIDED pair is re-evaluated exactly; disagreements are counted (must stay 0)
          uint32_t vm = vmask & ~fmask;
          int bad = 0;
          while (vm) {
            const int k = __ffs(vm) - 1;
            vm &= vm - 1;
            const bool ex = scale_mode ? edge_exact_scale(src, dst, i, j0 + k, beta, s_hat) : edge_exact(src, dst, i, j0 + k, beta);
            bad += (ex != (((word >> k) & 1u) != 0u));
          }
          if (bad) atomicAdd(bt.mismatches, (unsigned long long)bad);
        }
        const int cnt = __popc(fmask);
        int incl = cnt;  // inclusive warp scan
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int v = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += v;
        }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        if (total) {
          unsigned int base = 0;
          if (lane == 0) base = atomicAdd(bt.tc_list_count, (unsigned int)total);
          base = __shfl_sync(0xffffffffu, base, 0);
          if (base + (unsigned int)total <= bt.tc_list_cap) {
            unsigned int pos = base + (unsigned int)(incl - cnt);
            while (fmask) {
              const int k = __ffs(fmask) - 1;
              fmask &= fmask - 1;
              bt.tc_list[pos++] = make_uint2((unsigned int)b, ((unsigned int)i << 16) | (unsigned int)(j0 + k));
            }
          } else {  // queue full (the count keeps growing; the patch kernel clamps it): exact evaluation in place
            // the first warp that does not fit leaves [base, cap) unwritten: void entries (b = ~0) for the patch kernel
            for (unsigned int e = base + (unsigned int)lane; e < bt.tc_list_cap; e += 32u) bt.tc_list[e] = make_uint2(0xffffffffu, 0u);
            int nre = 0;
            while (fmask) {
              const int k = __ffs(fmask) - 1;
              fmask &= fmask - 1;
              const bool ex = scale_mode ? edge_exact_scale(src, dst, i, j0 + k, beta, s_hat) : edge_exact(src, dst, i, j0 + k, beta);
              word |= (ex ? 1u : 0u) << k;
              ++nre;
            }
            if (bt.rechecks) {
              nre = __reduce_add_sync(0xffffffffu, nre);
              if (lane == 0 && nre) atomicAdd(bt.rechecks, (unsigned long long)nre);
            }
          }
        }
      }
      rdeg += __popc(word);
      if (row_ok) rowp[2 * J + h] = word;
      if (!diag) {  // transposed half: warp w transposes rows I*128 + 32 (w & 3) .. +31 of column half w >> 2
        uint32_t* buf = s_tr + (n_tr & 1u) * (2 * kTile);
        buf[2 * rloc + h] = word;
        named_bar_sync(1, 32 * kTcEpiWarps);
        const int q = warp & 3, hh = warp >> 2;
        const uint32_t colw = tc_transpose32(buf[2 * (32 * q + lane) + hh], lane);
        const int jc = J * kTcN + 32 * hh + lane;
        if (jc < n) {
          adj32[(size_t)jc * P32 + 4 * I + q] = colw;
          if (colw) atomicAdd(degp + jc, __popc(colw));
        }
        ++n_tr;  // the next transposed tile uses the other buffer: its barrier orders these reads before the rewrite
      }
      if (ti.last_of_strip()) {
        if (row_ok && rdeg) atomicAdd(degp + i, rdeg);
        rdeg = 0;
      }
      ++n_t;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// exact re-check of the queued pairs: one thread per entry.  The bit written by graph_tc_kernel is the tentative
// classification; if the reference's FP64 sequence disagrees the bit (and its mirror, unless both directions live in the
// same diagonal 128-block and were queued separately) is flipped and the degrees are adjusted.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) tc_patch_kernel(Batch bt) {
  const unsigned int count = min(*bt.tc_list_count, bt.tc_list_cap);
  if (blockIdx.x == 0 && threadIdx.x == 0 && bt.rechecks) atomicAdd(bt.rechecks, (unsigned long long)count);
  const int n = bt.n, P32 = pitch32(n);
  const bool scale_mode = bt.scale_mode != 0;
  for (unsigned int e = blockIdx.x * blockDim.x + threadIdx.x; e < count; e += gridDim.x * blockDim.x) {
    const uint2 ent = bt.tc_list[e];
    if (ent.x == 0xffffffffu) continue;  // gap left by the first warp that found the queue full
    const int b = (int)ent.x, i = (int)(ent.y >> 16), j = (int)(ent.y & 0xffffu);
    const double* src = bt.src + (size_t)b * n * 3;
    const double* dst = bt.dst + (size_t)b * n * 3;
    const double beta = bt.gc[b].beta;
    const bool ex = scale_mode ? edge_exact_scale(src, dst, i, j, beta, bt.sol[b].scale) : edge_exact(src, dst, i, j, beta);
    uint32_t* adj32 = reinterpret_cast<uint32_t*>(bt.adj) + (size_t)b * n * P32;
    const bool cur = (adj32[(size_t)i * P32 + (j >> 5)] >> (j & 31)) & 1u;
    if (ex != cur) {
      int* degp = bt.deg + (size_t)b * n;
      const int dd = ex ? 1 : -1;
      atomicXor(adj32 + (size_t)i * P32 + (j >> 5), 1u << (j & 31));
      atomicAdd(degp + i, dd);
      if ((i >> 7) != (j >> 7)) {  // off-diagonal block: the transposed bit came from the same evaluation
        atomicXor(adj32 + (size_t)j * P32 + (i >> 5), 1u << (i & 31));
        atomicAdd(degp + j, dd);
      }
    }
  }
}

int launch_graph_tc(const Batch& bt, cudaStream_t st, int num_sms) {
  static bool attr_done_dev[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr_done_dev[dev & 63]) {
    cudaFuncSetAttribute(graph_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTcSmemBytes);
    cudaFuncSetAttribute(graph_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTcSmemBytes);
    attr_done_dev[dev & 63] = true;
  }
  const int nt = (bt.n + kTile - 1) / kTile;
  dim3 pg((unsigned)nt, (unsigned)bt.B);
  cudaMemsetAsync(bt.tc_list_count, 0, sizeof(unsigned int), st);
  tc_prep_kernel<<<pg, 128, 0, st>>>(bt);
  // strip length (in 64-column tiles): long strips amortise the A tile, short ones balance small batches
  const int ctas = 2 * num_sms;
  int S = 16;
  while (S > 1 && (long long)bt.B * tc_strips_per_problem(bt.n, S) < 4LL * ctas) S >>= 1;
  const int spp = tc_strips_per_problem(bt.n, S);
  const long long total = (long long)bt.B * spp;
  const int grid = (int)(total < ctas ? total : ctas);
  if (bt.flags_dbg & 2u)
    graph_tc_kernel<true><<<grid, kTcThreads, kTcSmemBytes, st>>>(bt, S, spp, (int)total);
  else
    graph_tc_kernel<false><<<grid, kTcThreads, kTcSmemBytes, st>>>(bt, S, spp, (int)total);
  tc_patch_kernel<<<4 * num_sms, 256, 0, st>>>(bt);
  cudaMemsetAsync(bt.tc_list_count, 0, sizeof(unsigned int), st);  // the strip kernel (other problems) queues next
  return 3;
}

void launch_graph_patch(const Batch& bt, cudaStream_t st, int num_sms) { tc_patch_kernel<<<4 * num_sms, 256, 0, st>>>(bt); }

// entries of the re-check queue for a (B, n) batch: 1/256 of the pairs (the band is ~1e-4), at least 1 Mi, at most 64 Mi
size_t tc_list_entries(int B, int n) {
  const double pairs = 0.5 * (double)B * (double)n * (double)n;
  double c = pairs / 256.0;
  if (c < 1048576.0) c = 1048576.0;
  if (c > 67108864.0) c = 67108864.0;
  return (size_t)c;
}

}  // namespace tzr
