// Stage 1 of solve(): TIMs + scale-consistency test + inlier graph, fused.
//
// Replaces (reference):
//   RobustRegistrationSolver::computeTIMs            teaser/src/registration.cc:512-551  (x2)
//   ScaleInliersSelector::solveForScale              teaser/src/registration.cc:427-443
//   inlier_graph_.addEdge loop                       teaser/src/registration.cc:614-619
//
// The reference materialises 2 x (3 x K) doubles of TIMs, 2 x K norms and a K-byte mask
// (K = N(N-1)/2; 65 B per pair).  Here a pair is a register-resident predicate and the only
// output is one bit in a packed symmetric adjacency bitset.
//
// Predicate (must be bit-identical to the reference's IEEE-double evaluation without FMA
// contraction, SURVEY Q6):  | sqrt(|s_j-s_i|^2) - sqrt(|d_j-d_i|^2) | <= beta.
// FP64 sqrt makes a pure-double kernel FP64-issue-bound, so every pair is first classified by a
// sqrt-free FP32 interval test on centred single-precision copies of the points:
//     with a=|ds|^2, b=|dd|^2, t=a-b, s=a+b:   |sqrt(a)-sqrt(b)| <= g  <=>  t^2 <= 2 g^2 s - g^4   (s >= g^2)
// evaluated for g = beta-delta ("surely an edge") and g = beta+delta ("surely not"), where delta
// bounds every FP32 error of the pipeline (conversion, differences, squares; DESIGN.md §graph).
// Only pairs inside the 2*delta band (typically < 1e-4 of all pairs) are re-evaluated with the
// exact double sequence, so the bitset is identical to a pure-FP64 evaluation (verified on device
// by the TZR_FLAG_VERIFY mode and against the oracle in tests/).
#include "tzr_internal.cuh"

namespace tzr {

// ------------------------------------------------------------------------------------------------
// prep: bounding boxes, centred float copies, filter constants.  One CTA per problem.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_min(double v) {
  for (int o = 16; o; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
  for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// launch_graph sends the problems prep_kernel marked use_tc to graph_tc_kernel only under debug flag 1024 without an A/B
// flag (8-256) or the interval-test flag 512
__host__ __device__ __forceinline__ bool tc_path_active(uint32_t flags) {
  return (flags & 1024u) && !(flags & (8u | 16u | 32u | 64u | 128u | 256u | 512u));
}

__global__ void __launch_bounds__(256) prep_kernel(Batch bt) {
  const int b = blockIdx.x;
  const int n = bt.n;
  const double* src = bt.src + (size_t)b * n * 3;
  const double* dst = bt.dst + (size_t)b * n * 3;
  __shared__ double s_red[8][12];
  __shared__ int s_bad[8];
  __shared__ double s_c[7];
  double mn[6], mx[6];
  for (int k = 0; k < 6; ++k) {
    mn[k] = 1.0 / 0.0;
    mx[k] = -1.0 / 0.0;
  }
  int bad = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    for (int k = 0; k < 3; ++k) {
      const double a = src[3 * i + k], c = dst[3 * i + k];
      bad |= !isfinite(a) | !isfinite(c);
      mn[k] = fmin(mn[k], a);
      mx[k] = fmax(mx[k], a);
      mn[3 + k] = fmin(mn[3 + k], c);
      mx[3 + k] = fmax(mx[3 + k], c);
    }
  }
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = 0; k < 6; ++k) {
    mn[k] = warp_min(mn[k]);
    mx[k] = warp_max(mx[k]);
  }
  bad = __any_sync(0xffffffffu, bad);
  if (lane == 0) {
    for (int k = 0; k < 6; ++k) {
      s_red[w][k] = mn[k];
      s_red[w][6 + k] = mx[k];
    }
    s_bad[w] = bad;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int anybad = 0;
    for (int k = 0; k < 6; ++k) {
      double a = s_red[0][k], c = s_red[0][6 + k];
      for (int q = 1; q < 8; ++q) {
        a = fmin(a, s_red[q][k]);
        c = fmax(c, s_red[q][6 + k]);
      }
      mn[k] = a;
      mx[k] = c;
    }
    for (int q = 0; q < 8; ++q) anybad |= s_bad[q];
    double Ms = 0, Md = 0;
    GraphConsts gc;
    for (int k = 0; k < 3; ++k) {
      gc.cs[k] = 0.5 * (mn[k] + mx[k]);
      gc.cd[k] = 0.5 * (mn[3 + k] + mx[3 + k]);
      Ms = fmax(Ms, 0.5 * (mx[k] - mn[k]));
      Md = fmax(Md, 0.5 * (mx[3 + k] - mn[3 + k]));
      s_c[k] = gc.cs[k];
      s_c[3 + k] = gc.cd[k];
    }
    const double beta = bt.beta;
    gc.beta = beta;
    // Unknown scale: |d2/d1 - s| <= beta/d1  <=>  |d2 - s*d1| <= beta (d1 > 0), i.e. the fixed-scale test on a
    // source cloud scaled by s: the float copies are pre-scaled, the exact re-check keeps the reference's
    // division-based sequence (its rounding differs from the real-number predicate by ~1e-16 relative, far
    // inside delta).
    double s_hat = 1.0;
    if (bt.scale_mode) {
      s_hat = bt.sol[b].scale;
      if (!(s_hat > 1e-6) || !(s_hat < 1e6)) {
        s_hat = 1.0;
        anybad = 1;  // degenerate estimate: exact path for every pair
      }
      Ms *= s_hat;
    }
    s_c[6] = s_hat;
    // delta: bound on the FP32 error of |D1 - D2| (DESIGN.md: <= ~70 u32 (Ms+Md)); 256 u32 (...) used.
    const double u32 = 5.9604644775390625e-08;  // 2^-24
    const double delta = 256.0 * u32 * (Ms + Md + beta);
    const double gam1 = beta - delta, gam2 = beta + delta;
    const double up = 1.0 + 9.5367431640625e-07, dn = 1.0 - 9.5367431640625e-07;  // 1 +- 2^-20
    int use64 = anybad || !(Ms < 1e8) || !(Md < 1e8) || !(gam2 > 1e-8) || !isfinite(beta) || (bt.flags_dbg & 1u);
    // sure edge: x <= b1; sure non-edge: x > b2.  Exact path for everything: b1 = -1 (x >= 0), b2 = +inf.
    gc.b1 = (use64 || !(gam1 > 0)) ? -1.0f : (float)(gam1 * dn);
    gc.b2 = use64 ? __int_as_float(0x7f800000) : (float)(gam2 * up);
    gc.use_fp64 = use64;
    gc.s_hat = s_hat;
    // ---- v7 strip kernel (graph_strip3_kernel): d_hi = t^2 - (beta^2 - K) w < 0 proves an edge, d_lo = t^2 -
    // (beta^2 + K) w >= 0 proves a non-edge, K = dt (2 beta + dt) + 32 u beta^2 relative to w = (sqrt a + sqrt b)^2.
    // dt bounds |g' - g|: float conversion of the centred coordinates (<= u M each), the differences, squares and sums
    // give |sqrt a' - sqrt a| <= ~15 u M per cloud; 64 u (Ms + Md) is used, plus the bias eps of the squared norms.
    {
      const double d3 = 64.0 * u32 * (Ms + Md);
      const double eps = fmax((d3 / 16.0) * (d3 / 16.0), 1e-36);
      const double dt = 1.125 * d3;
      const double K = dt * (2.0 * beta + dt) + 32.0 * u32 * beta * beta;
      const double b2v = beta * beta;
      gc.f3_eps = (float)eps;
      if (use64) {  // exact path for every pair (the kernel also overrides the words: NaN inputs have no sign)
        gc.f3_nlo = -__int_as_float(0x7f800000);
        gc.f3_nhi = __int_as_float(0x7f800000);
      } else {
        gc.f3_nlo = (float)(-(b2v + K) * up);
        gc.f3_nhi = (b2v - K > 0) ? (float)(-(b2v - K) * dn) : (float)((K - b2v) * up + 1e-37);
      }
      gc.pad2 = 0;
    }
    // ---- tensor-core filter constants (graph_tc.cu; derivation in DESIGN.md §3.1).  a' = |ds|^2 and b' = |dd|^2 come
    // out of the tensor core with |a' - a| <= ea, |b' - b| <= eb (E = ea + eb).  With t = a - b, s = a + b,
    //   f(a, b) = t^2 - 2 beta^2 s + beta^4 = (g^2 - beta^2)(w - beta^2),  g = |sqrt a - sqrt b|,  w = (sqrt a + sqrt b)^2 >= s
    // so   edge  <=>  s <= beta^2  or  f <= 0   — a polynomial, no square root, no division:
    //   |f(a', b') - f(a, b)| <= 2 E |t'| + E^2 + 2 beta^2 E                      (tensor-core error)
    //   |d^ - f(a', b')|      <= 8 u (t'^2 + 2 beta^2 s' + beta^4)                 (FP32 evaluation of d^: 4 roundings + 2 constants)
    // and for s <= beta^2 (where the sign of f says nothing)  f <= (beta^2 - s)^2 <= beta^4.  The kernel decides by the
    // signs of d^ +- band, band = kap (t'^2 + beta^4) + c0 with 2 E |t'| <= (E/lam) t'^2 + E lam (lam = the typical |t| at the
    // threshold, 0.75 beta D): kap = E/lam + 8 u, c0 = E lam + E^2 + 2 beta^2 E + 16 u beta^2 Smax + 8 u beta^4 + beta^4.
    // (8 u t'^2 needs no case split: it is part of kap.)  d^ + band < 0 proves f < 0 (an edge whatever s is); d^ - band >= 0
    // proves f > beta^4, hence s > beta^2 and a non-edge; everything else goes to the exact FP64 re-check.
    {
      double Ds2 = 0, Dd2 = 0;  // largest possible squared distance inside each (scaled) cloud
      for (int k = 0; k < 3; ++k) {
        const double es = (mx[k] - mn[k]) * s_hat, ed = mx[3 + k] - mn[3 + k];
        Ds2 += es * es;
        Dd2 += ed * ed;
      }
      const double kappa = bt.tc_kappa > 0 ? bt.tc_kappa : kTcKappa;
      const double ea = kappa * u32 * Ds2, eb = kappa * u32 * Dd2, E = ea + eb;
      const double b2 = beta * beta, b4 = b2 * b2;
      const double lam = 0.75 * beta * sqrt(0.5 * (Ds2 + Dd2));
      const double Smax = Ds2 + Dd2 + E;
      const double kap = E / lam + 8.0 * u32;
      const double c0 = E * lam + E * E + 2.0 * b2 * E + 16.0 * u32 * b2 * Smax + 8.0 * u32 * b4 + b4;
      // When is the filter worth it (correctness never depends on this)?  beta <= D/8: the beta^4 floor of the band stays
      // below ~1e-3 of the pairs; E / (0.75 D) <= beta / 64: the band in g = |sqrt a - sqrt b| is a small fraction of the
      // threshold (fails when the noise bound is tiny against the extent of a cloud: beta/D below ~3e-4); b4 a normal float.
      const double Dmin = sqrt(fmin(Ds2, Dd2));
      const bool ok = !use64 && (bt.flags_dbg & 1024u) != 0 && (bt.flags_dbg & 512u) == 0 && Ds2 > 0 && Dd2 > 0 && Ds2 < 1e8 && Dd2 < 1e8 &&
                      b4 > 1e-30 && isfinite(E) && isfinite(kap) && 8.0 * beta <= Dmin && 64.0 * E <= 0.75 * Dmin * beta;
      gc.use_tc = ok ? 1 : 0;
      gc.tc_c2 = (float)(2.0 * b2);
      gc.tc_b4 = (float)b4;
      gc.tc_kap = (float)(kap * up);
      gc.tc_c0 = (float)(c0 * up);
      gc.tc_pad = 0.f;
      if (ok && bt.rechecks) atomicAdd(bt.mismatches + 7, 1ull);  // debug counter 7: problems on the tensor-core path
      // ---- Gram-form test of graph_strip2_kernel (derivation in DESIGN.md §3.1).  a' = fl(N_i + N_j - 2 q_i.q_j) from the
      // float copies q (|q| <= R, R^2 <= Ds2 / 4 about the box centre) is within 8 u R^2 (conversion) + 2 u R^2 (rounded
      // norms) + 14 u R^2 (one FADD and three FMA roundings on partial sums of at most 2 R^2 and 4 R^2) of a; 28 u R^2 is
      // used, the rest covers second-order terms and the reference's own FP64 rounding.  With E = ea + eb, k = E / lam,
      // C = E lam + E^2 + 2 beta^2 E and 4 u (t^2 + |m| S + |c|) the FP32 evaluation error of fma(t, t, fma(s, m, c)):
      //   t^2 + mhi s + chi <= 0  =>  (1 + k) t^2 - 2 beta^2 s + beta^4 + C <= 0  =>  f(a, b) <= 0           (edge)
      //   t^2 + mlo s + clo >= 0  =>  (1 - k) t^2 - 2 beta^2 s - C > 0            =>  f(a, b) > beta^4      (s > beta^2: not)
      const double gE = 7.0 * u32 * (Ds2 + Dd2), gk = gE / lam, gS = Ds2 + Dd2 + gE;
      const double gC = gE * lam + gE * gE + 2.0 * b2 * gE;
      gc.g_mhi = (float)(-2.0 * b2 * (1.0 - 4.0 * u32) / (1.0 + gk) * dn);
      gc.g_chi = (float)(((b4 + gC) / (1.0 + gk) + 8.0 * u32 * b2 * gS) * up);
      gc.g_mlo = (float)(-2.0 * b2 * (1.0 + 4.0 * u32) / (1.0 - gk) * up);
      gc.g_clo = (float)(-(gC + 9.0 * u32 * b2 * gS) / (1.0 - gk) * up * up);
      // conditioning guard (same form as use_tc's): beta <= D/8 keeps pairs with s <= beta^2 rare, 64 E <= 0.75 D beta keeps
      // the band narrow against beta (and k <= 1/64).  C1 (outliers moved 5-10 extents away, beta/D ~ 1e-4) fails it.
      gc.use_gram = (!use64 && (bt.flags_dbg & 512u) == 0 && Ds2 > 0 && Dd2 > 0 && Ds2 < 1e8 && Dd2 < 1e8 && b4 > 1e-30 &&
                     isfinite(gE) && 8.0 * beta <= Dmin && 64.0 * gE <= 0.75 * Dmin * beta) ? 1 : 0;
      // debug counter 15: problems graph_strip2_kernel builds with the Gram test (not those graph_tc_kernel or
      // graph_strip3_kernel builds; launch_graph makes the same choice)
      if (gc.use_gram && bt.rechecks && !(ok && tc_path_active(bt.flags_dbg)) && !(bt.flags_dbg & 2048u))
        atomicAdd(bt.mismatches + 15, 1ull);
    }
    bt.gc[b] = gc;
    bt.n_edges2[b] = 0ull;
  }
  __syncthreads();
  float4* sf = bt.sf + (size_t)b * n;
  float4* df = bt.df + (size_t)b * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float4 a, c;
    a.x = (float)((src[3 * i + 0] - s_c[0]) * s_c[6]);
    a.y = (float)((src[3 * i + 1] - s_c[1]) * s_c[6]);
    a.z = (float)((src[3 * i + 2] - s_c[2]) * s_c[6]);
    a.w = (float)((double)a.x * a.x + (double)a.y * a.y + (double)a.z * a.z);  // squares exact in FP64: one rounding
    c.x = (float)(dst[3 * i + 0] - s_c[3]);
    c.y = (float)(dst[3 * i + 1] - s_c[4]);
    c.z = (float)(dst[3 * i + 2] - s_c[5]);
    c.w = (float)((double)c.x * c.x + (double)c.y * c.y + (double)c.z * c.z);
    sf[i] = a;
    df[i] = c;
    bt.deg[(size_t)b * n + i] = 0;  // accumulated by the graph kernel (fused-degree path)
  }
  // pair-interleaved copy for the packed kernel: (point o, point o+32) of every 64-column half block adjacent
  const int npad = npad128(n);
  float* pk = bt.pk + (size_t)b * 6 * npad;
  for (int j = threadIdx.x; j < npad; j += blockDim.x) {
    const int o = j & 127, pos = (j & ~127) + (o >> 6) * 64 + (o & 31) * 2 + ((o >> 5) & 1);
    float v[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (j < n) {
      v[0] = (float)((src[3 * j + 0] - s_c[0]) * s_c[6]);
      v[1] = (float)((src[3 * j + 1] - s_c[1]) * s_c[6]);
      v[2] = (float)((src[3 * j + 2] - s_c[2]) * s_c[6]);
      v[3] = (float)(dst[3 * j + 0] - s_c[3]);
      v[4] = (float)(dst[3 * j + 1] - s_c[4]);
      v[5] = (float)(dst[3 * j + 2] - s_c[5]);
    }
#pragma unroll
    for (int q = 0; q < 6; ++q) pk[(size_t)q * npad + pos] = v[q];
  }
}

// ------------------------------------------------------------------------------------------------
// graph tile kernel: one CTA (4 warps) per 128x128 tile of the upper triangle (I <= J) of one problem.
// Warp w owns rows [32w, 32w+32) x all 128 columns of the tile: lane l keeps the four column points
// (l, l+32, l+64, l+96) in registers and sweeps the 32 row points broadcast from shared memory, i.e. four
// pair predicates per lane per step (amortises the shared-memory loads and the loop overhead).
// Row words come from __ballot_sync; the transposed (column) words are accumulated per lane, so the
// symmetric half of the bitset costs no extra predicate evaluations.  Validity (i,j < n, i != j) is applied
// as word masks after the sweep, not per pair.
// ------------------------------------------------------------------------------------------------
struct PairEval {
  bool sure, decided;
};

__device__ __forceinline__ float sqrt_approx(float x) {  // one MUFU.SQRT (<= 2 ulp); its error is part of delta
  float y;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// FP32 interval classification of one pair:  x = | |ds| - |dd| |  against  beta -/+ delta.
// 12 FP32 ops for the two squared norms, 2 MUFU.SQRT (their own pipe), 1 FADD, 2 FSETP.
__device__ __forceinline__ PairEval classify(const float4 is, const float4 id, const float4 js, const float4 jd,
                                             const float b1, const float b2) {
  const float ax = js.x - is.x, ay = js.y - is.y, az = js.z - is.z;
  const float bx = jd.x - id.x, by = jd.y - id.y, bz = jd.z - id.z;
  const float a = fmaf(az, az, fmaf(ay, ay, ax * ax));
  const float b = fmaf(bz, bz, fmaf(by, by, bx * bx));
  const float x = fabsf(sqrt_approx(a) - sqrt_approx(b));
  PairEval e;
  e.sure = x <= b1;                 // surely an edge      (b1 = beta - delta, or -1: never)
  e.decided = e.sure || (x > b2);   // ... or surely not   (b2 = beta + delta, or +inf: never)
  return e;
}

#ifdef TZR_AB_KERNELS  // superseded designs, kept for A/B runs only (make AB=1)
template <bool kVerify>
__global__ void __launch_bounds__(kGraphThreads, 5) graph_tile_kernel(Batch bt) {
  const int b = blockIdx.y;
  const int n = bt.n;
  const int nt = (n + kTile - 1) / kTile;
  // decode upper-triangular tile index -> (I, J), I <= J
  const int p = blockIdx.x;
  int I = (int)floor(((2.0 * nt + 1.0) - sqrt((2.0 * nt + 1.0) * (2.0 * nt + 1.0) - 8.0 * (double)p)) * 0.5);
  if (I < 0) I = 0;
  while (I > 0 && (long long)I * nt - (long long)I * (I - 1) / 2 > p) --I;
  while ((long long)(I + 1) * nt - (long long)(I + 1) * I / 2 <= p) ++I;
  const int J = I + (p - (int)((long long)I * nt - (long long)I * (I - 1) / 2));

  __shared__ float4 s_is[kTile];
  __shared__ float4 s_id[kTile];
  __shared__ __align__(16) uint32_t s_row[kTile][4];
  __shared__ __align__(16) uint32_t s_col[kTile][4];

  const GraphConsts* gcp = bt.gc + b;
  const float b1 = gcp->b1, b2 = gcp->b2;
  const double beta = gcp->beta;
  const bool scale_mode = bt.scale_mode != 0;
  const double s_hat = scale_mode ? bt.sol[b].scale : 1.0;

  const float4* sf = bt.sf + (size_t)b * n;
  const float4* df = bt.df + (size_t)b * n;
  const double* src = bt.src + (size_t)b * n * 3;
  const double* dst = bt.dst + (size_t)b * n * 3;

  const int tid = threadIdx.x;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  {
    const int i = I * kTile + tid;
    s_is[tid] = (i < n) ? sf[i] : z4;
    s_id[tid] = (i < n) ? df[i] : z4;
  }
  const int w = tid >> 5, lane = tid & 31;
  const int jb = J * kTile + lane;
  float4 js[4], jd[4];
  bool vj[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int j = jb + 32 * c;
    vj[c] = j < n;
    js[c] = vj[c] ? sf[j] : z4;
    jd[c] = vj[c] ? df[j] : z4;
  }
  __syncthreads();

  uint32_t roww[4] = {0u, 0u, 0u, 0u}, colw[4] = {0u, 0u, 0u, 0u};
  const int ibase = I * kTile + 32 * w;
  const int nrows = min(32, n - ibase);  // may be <= 0 for the last row block
  // ---- hot sweep.  Kept SMALL on purpose (unroll 2, ~3.5 KB of SASS): a fully unrolled sweep with the exact
  // path inlined was instruction-fetch bound (ncu: stall_no_instructions dominant).  Steps that contain an
  // undecided pair are only recorded here (warp-uniform bit mask) and revisited after the sweep.
  uint32_t ambmask = 0u;
  uint32_t bit = 1u;
#pragma unroll 2
  for (int ii = 0; ii < nrows; ++ii, bit <<= 1) {
    const float4 is = s_is[32 * w + ii], id = s_id[32 * w + ii];
    bool all_decided = true;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const PairEval e = classify(is, id, js[c], jd[c], b1, b2);
      all_decided = all_decided && e.decided;
      const uint32_t m = __ballot_sync(0xffffffffu, e.sure);
      if (lane == ii) roww[c] = m;
      colw[c] |= e.sure ? bit : 0u;
    }
    if (!__all_sync(0xffffffffu, all_decided)) ambmask |= bit;
  }
  // ---- rare: steps with pairs inside the ambiguous band -> exact FP64 sequence for those lanes
  while (ambmask) {
    const int ii = __ffs(ambmask) - 1;
    ambmask &= ambmask - 1;
    const int i = ibase + ii;
    const float4 is = s_is[32 * w + ii], id = s_id[32 * w + ii];
    int nre = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int j = jb + 32 * c;
      const PairEval e = classify(is, id, js[c], jd[c], b1, b2);
      bool ex = false;
      if (!e.decided && vj[c] && j != i) {
        ex = scale_mode ? edge_exact_scale(src, dst, i, j, beta, s_hat) : edge_exact(src, dst, i, j, beta);
        ++nre;
      }
      const uint32_t mex = __ballot_sync(0xffffffffu, ex);
      if (lane == ii) roww[c] |= mex;
      colw[c] |= ex ? (1u << ii) : 0u;
    }
    if (bt.rechecks) {
      nre = __reduce_add_sync(0xffffffffu, nre);
      if (lane == 0 && nre) atomicAdd(bt.rechecks, (unsigned long long)nre);
    }
  }
  if (kVerify) {
    // debug: every DECIDED pair is re-evaluated exactly; disagreements are counted (must stay 0)
    for (int ii = 0; ii < nrows; ++ii) {
      const int i = ibase + ii;
      const float4 is = s_is[32 * w + ii], id = s_id[32 * w + ii];
      int bad = 0;
      for (int c = 0; c < 4; ++c) {
        const int j = jb + 32 * c;
        const PairEval e = classify(is, id, js[c], jd[c], b1, b2);
        if (e.decided && vj[c] && j != i)
          bad += ((scale_mode ? edge_exact_scale(src, dst, i, j, beta, s_hat) : edge_exact(src, dst, i, j, beta)) != e.sure);
      }
      if (bad) atomicAdd(bt.mismatches, (unsigned long long)bad);
    }
  }
  // ---- validity masks: columns >= n, rows >= n, and the diagonal (i == j) of diagonal tiles
  const uint32_t rmask = nrows >= 32 ? 0xffffffffu : (nrows <= 0 ? 0u : ((1u << nrows) - 1u));
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const uint32_t cm = __ballot_sync(0xffffffffu, vj[c]);
    roww[c] &= cm;
    colw[c] = vj[c] ? (colw[c] & rmask) : 0u;
    if (I == J) {
      // row r = 32w + lane holds columns 32c + [0,32): self bit at column r
      if (c == w) roww[c] &= ~(1u << lane);
      // column 32c + lane holds rows 32w + [0,32): self bit at row 32c + lane
      if (c == w) colw[c] &= ~(1u << lane);
    }
  }
  *reinterpret_cast<uint4*>(&s_row[32 * w + lane][0]) = make_uint4(roww[0], roww[1], roww[2], roww[3]);
#pragma unroll
  for (int c = 0; c < 4; ++c) s_col[32 * c + lane][w] = colw[c];
  __syncthreads();

  uint32_t* adj32 = reinterpret_cast<uint32_t*>(bt.adj) + (size_t)b * n * pitch32(n);
  const int P32 = pitch32(n);
  {
    const int row = I * kTile + tid;
    if (row < n) {
      const uint4 v = *reinterpret_cast<const uint4*>(&s_row[tid][0]);
      *reinterpret_cast<uint4*>(adj32 + (size_t)row * P32 + 4 * J) = v;
    }
  }
  if (I != J) {
    const int row = J * kTile + tid;
    if (row < n) {
      const uint4 v = *reinterpret_cast<const uint4*>(&s_col[tid][0]);
      *reinterpret_cast<uint4*>(adj32 + (size_t)row * P32 + 4 * I) = v;
    }
  }
}

#endif  // TZR_AB_KERNELS

// ------------------------------------------------------------------------------------------------
// graph strip kernel (default): same sweep as graph_tile_kernel, but every WARP is independent — it owns 32 rows
// and walks up to kStripBlocks consecutive 128-column blocks, keeps its 32 row points in a private shared-memory
// slice (only __syncwarp), and stores its row words (16 B per row) and transposed column words (4 B per row)
// straight from registers.  No CTA barrier, the row points and the tile decode are amortised over the strip, and
// a warp waiting for its next column points does not stall its neighbours (ncu on the tile kernel: 12 % of the
// issue slots were lost at the two __syncthreads of the short-lived CTAs).
// ------------------------------------------------------------------------------------------------
constexpr int kStripBlocks = 4;

__host__ __device__ inline int strip_grid(int n) {
  const int nt = (n + kTile - 1) / kTile;
  int total = 0;
  for (int I = 0; I < nt; ++I) total += (nt - I + kStripBlocks - 1) / kStripBlocks;
  return total;
}

// 32x32 bit transpose across the lanes of a warp: lane l passes row l, receives column l (bit i of the result =
// bit l of lane i's input).  5 butterfly stages (shuffle + 4 logic ops each).
__device__ __forceinline__ uint32_t warp_transpose32(uint32_t x, int lane) {
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

#ifdef TZR_AB_KERNELS
template <bool kVerify, int kMinBlocks>
__global__ void __launch_bounds__(kGraphThreads, kMinBlocks) graph_strip_kernel(Batch bt) {
  const int b = blockIdx.y;
  const int n = bt.n;
  const int nt = (n + kTile - 1) / kTile;
  int I = 0, p = blockIdx.x;
  while (true) {
    const int ng = (nt - I + kStripBlocks - 1) / kStripBlocks;
    if (p < ng) break;
    p -= ng;
    ++I;
  }
  const int J0 = I + p * kStripBlocks;
  const int J1 = min(nt, J0 + kStripBlocks);

  __shared__ float4 s_is[kTile];
  __shared__ float4 s_id[kTile];
  __shared__ __align__(16) uint32_t s_rw[kTile][4];  // row words of the current block (warp-private slices)

  const GraphConsts* gcp = bt.gc + b;
  const float b1 = gcp->b1, b2 = gcp->b2;
  const double beta = gcp->beta;
  const bool scale_mode = bt.scale_mode != 0;
  const double s_hat = scale_mode ? bt.sol[b].scale : 1.0;

  const float4* sf = bt.sf + (size_t)b * n;
  const float4* df = bt.df + (size_t)b * n;
  const double* src = bt.src + (size_t)b * n * 3;
  const double* dst = bt.dst + (size_t)b * n * 3;

  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
  const int ibase = I * kTile + 32 * w;
  const int nrows = min(32, n - ibase);
  if (nrows <= 0) return;  // whole warp: there is no CTA-level synchronisation in this kernel
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  {
    const int i = ibase + lane;
    s_is[tid] = (i < n) ? sf[i] : z4;
    s_id[tid] = (i < n) ? df[i] : z4;
  }
  __syncwarp();
  uint32_t* adj32 = reinterpret_cast<uint32_t*>(bt.adj) + (size_t)b * n * pitch32(n);
  const int P32 = pitch32(n);
  const uint32_t rmask = nrows >= 32 ? 0xffffffffu : ((1u << nrows) - 1u);

  for (int J = J0; J < J1; ++J) {
    const int jb = J * kTile + lane;
    float4 js[4], jd[4];
    bool vj[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int j = jb + 32 * c;
      vj[c] = j < n;
      js[c] = vj[c] ? sf[j] : z4;
      jd[c] = vj[c] ? df[j] : z4;
    }
    if (nrows < 32) *reinterpret_cast<uint4*>(&s_rw[tid][0]) = make_uint4(0u, 0u, 0u, 0u);  // rows past n stay empty
    __syncwarp();
    // ---- hot sweep: 4 pair predicates per lane per step; the four ballots of a step are one uniform 16-byte
    // shared-memory store (the warp's row words); column words are recovered afterwards by bit transposition
    uint32_t ambmask = 0u;
    uint32_t bit = 1u;
#pragma unroll 2
    for (int ii = 0; ii < nrows; ++ii, bit <<= 1) {
      const float4 is = s_is[32 * w + ii], id = s_id[32 * w + ii];
      bool all_decided = true;
      uint32_t m[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const PairEval e = classify(is, id, js[c], jd[c], b1, b2);
        all_decided = all_decided && e.decided;
        m[c] = __ballot_sync(0xffffffffu, e.sure);
      }
      *reinterpret_cast<uint4*>(&s_rw[32 * w + ii][0]) = make_uint4(m[0], m[1], m[2], m[3]);
      if (!__all_sync(0xffffffffu, all_decided)) ambmask |= bit;
    }
    __syncwarp();
    // ---- rare: steps with pairs inside the ambiguous band -> exact FP64 sequence for those lanes
    while (ambmask) {
      const int ii = __ffs(ambmask) - 1;
      ambmask &= ambmask - 1;
      const int i = ibase + ii;
      const float4 is = s_is[32 * w + ii], id = s_id[32 * w + ii];
      int nre = 0;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int j = jb + 32 * c;
        const PairEval e = classify(is, id, js[c], jd[c], b1, b2);
        bool ex = false;
        if (!e.decided && vj[c] && j != i) {
          ex = scale_mode ? edge_exact_scale(src, dst, i, j, beta, s_hat) : edge_exact(src, dst, i, j, beta);
          ++nre;
        }
        const uint32_t mex = __ballot_sync(0xffffffffu, ex);
        if (lane == 0 && mex) s_rw[32 * w + ii][c] |= mex;
      }
      if (bt.rechecks) {
        nre = __reduce_add_sync(0xffffffffu, nre);
        if (lane == 0 && nre) atomicAdd(bt.rechecks, (unsigned long long)nre);
      }
    }
    if (kVerify) {
      for (int ii = 0; ii < nrows; ++ii) {
        const int i = ibase + ii;
        const float4 is = s_is[32 * w + ii], id = s_id[32 * w + ii];
        int bad = 0;
        for (int c = 0; c < 4; ++c) {
          const int j = jb + 32 * c;
          const PairEval e = classify(is, id, js[c], jd[c], b1, b2);
          if (e.decided && vj[c] && j != i)
            bad += ((scale_mode ? edge_exact_scale(src, dst, i, j, beta, s_hat) : edge_exact(src, dst, i, j, beta)) !=
                    e.sure);
        }
        if (bad) atomicAdd(bt.mismatches, (unsigned long long)bad);
      }
    }
    __syncwarp();
    // ---- row words of lane's row; masks (columns >= n, i == j on the diagonal block); transposed column words
    const uint4 rw = *reinterpret_cast<const uint4*>(&s_rw[tid][0]);
    uint32_t roww[4] = {rw.x, rw.y, rw.z, rw.w}, colw[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const uint32_t cm = __ballot_sync(0xffffffffu, vj[c]);
      roww[c] &= cm;
      if (I == J && c == w) roww[c] &= ~(1u << lane);
      colw[c] = warp_transpose32(roww[c], lane) & rmask;
    }
    if (lane < nrows)
      *reinterpret_cast<uint4*>(adj32 + (size_t)(ibase + lane) * P32 + 4 * J) =
          make_uint4(roww[0], roww[1], roww[2], roww[3]);
    if (I != J) {
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (vj[c]) adj32[(size_t)(jb + 32 * c) * P32 + 4 * I + w] = colw[c];
    }
    __syncwarp();
  }
}

#endif  // TZR_AB_KERNELS

// ------------------------------------------------------------------------------------------------
// graph strip kernel, paired-FP32 variant (default): identical decomposition and outputs as graph_strip_kernel, with
// two pairs per 64-bit register pair: the twelve FP32 operations per pair run on (x, y) lanes that are loaded with
// one 8-byte access and stay paired end to end, so no re-packing moves are needed.  Every component is the same IEEE
// operation (explicit round-to-nearest, no contraction) as in the scalar kernel, so the classification (and delta) is
// unchanged.  The row point is stored negated and duplicated in shared memory ((-x,-x), ...) so that js - is is one
// paired add.
// ------------------------------------------------------------------------------------------------
typedef unsigned long long f32x2;
__device__ __forceinline__ f32x2 pk2(float lo, float hi) {
  f32x2 r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void upk2(f32x2 v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ f32x2 add2(f32x2 a, f32x2 b) {
  float a0, a1, b0, b1;
  upk2(a, a0, a1);
  upk2(b, b0, b1);
  return pk2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ f32x2 sub2(f32x2 a, f32x2 b) {
  float a0, a1, b0, b1;
  upk2(a, a0, a1);
  upk2(b, b0, b1);
  return pk2(__fsub_rn(a0, b0), __fsub_rn(a1, b1));
}
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) {
  float a0, a1, b0, b1;
  upk2(a, a0, a1);
  upk2(b, b0, b1);
  return pk2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) {
  float a0, a1, b0, b1, c0, c1;
  upk2(a, a0, a1);
  upk2(b, b0, b1);
  upk2(c, c0, c1);
  return pk2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}

struct __align__(16) IPointNeg2 {
  float4 a;  // (-sx,-sx,-sy,-sy)
  float4 b;  // (-sz,-sz,-dx,-dx)
  float4 c;  // (-dy,-dy,-dz,-dz)
};

// Interval test of graph_strip2_kernel, for the problems that fail the Gram test's conditioning guard (and for every
// problem under debug flags 1 and 512).  kFuseDeg: vertex degrees are accumulated here (row part: one atomic per row and
// strip; column part: one 32-lane RED per transposed word) instead of a second pass over the B*n^2/8-byte bitset; deg[] is
// zeroed by prep_kernel.
template <bool kVerify, bool kFuseDeg>
__device__ __forceinline__ void strip_interval(const Batch& bt, const int b, const int I, const int J0, const int J1) {
  const int n = bt.n;
  __shared__ IPointNeg2 s_ip[kTile];
  __shared__ __align__(16) uint32_t s_rw[kTile][4];

  const GraphConsts* gcp = bt.gc + b;
  const float b1 = gcp->b1, b2 = gcp->b2;
  const double beta = gcp->beta;
  const bool scale_mode = bt.scale_mode != 0;
  const double s_hat = scale_mode ? bt.sol[b].scale : 1.0;

  const float4* sf = bt.sf + (size_t)b * n;
  const float4* df = bt.df + (size_t)b * n;
  const double* src = bt.src + (size_t)b * n * 3;
  const double* dst = bt.dst + (size_t)b * n * 3;

  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
  const int ibase = I * kTile + 32 * w;
  const int nrows = min(32, n - ibase);
  if (nrows <= 0) return;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  {
    const int i = ibase + lane;
    const float4 s = (i < n) ? sf[i] : z4, d = (i < n) ? df[i] : z4;
    IPointNeg2 ip;
    ip.a = make_float4(-s.x, -s.x, -s.y, -s.y);
    ip.b = make_float4(-s.z, -s.z, -d.x, -d.x);
    ip.c = make_float4(-d.y, -d.y, -d.z, -d.z);
    s_ip[tid] = ip;
  }
  __syncwarp();
  uint32_t* adj32 = reinterpret_cast<uint32_t*>(bt.adj) + (size_t)b * n * pitch32(n);
  const int P32 = pitch32(n);
  const uint32_t rmask = nrows >= 32 ? 0xffffffffu : ((1u << nrows) - 1u);

  const int npadh = npad128(n) / 2;  // 64-bit elements per packed array
  const f32x2* pkp = reinterpret_cast<const f32x2*>(bt.pk + (size_t)b * 6 * npad128(n));
  int* degp = bt.deg + (size_t)b * n;
  int rdeg = 0;
  for (int J = J0; J < J1; ++J) {
    const int jb = J * kTile + lane;
    // column points, two pairs per 64-bit register: X[k] = (x of point jb+64k, x of point jb+64k+32), loaded as
    // 8-byte words from the pair-interleaved arrays written by prep_kernel (zero-padded past n)
    f32x2 SX[2], SY[2], SZ[2], DX[2], DY[2], DZ[2];
    bool vj[4];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      vj[2 * k] = jb + 64 * k < n;
      vj[2 * k + 1] = jb + 64 * k + 32 < n;
      const size_t e = (size_t)J * 64 + k * 32 + lane;
      SX[k] = pkp[0 * (size_t)npadh + e]; SY[k] = pkp[1 * (size_t)npadh + e]; SZ[k] = pkp[2 * (size_t)npadh + e];
      DX[k] = pkp[3 * (size_t)npadh + e]; DY[k] = pkp[4 * (size_t)npadh + e]; DZ[k] = pkp[5 * (size_t)npadh + e];
    }
    if (nrows < 32) *reinterpret_cast<uint4*>(&s_rw[tid][0]) = make_uint4(0u, 0u, 0u, 0u);
    __syncwarp();
    // pair index c (word c of the row) = point jb + 32*c = packed slot (k = c>>1, component c&1)
    auto classify4 = [&](int ii, bool sure[4], bool dec[4]) {
      // three 16-byte broadcast loads: six (-v,-v) pairs, each already a 64-bit register pair
      const ulonglong2* ipp = reinterpret_cast<const ulonglong2*>(&s_ip[32 * w + ii]);
      const ulonglong2 qa = ipp[0], qb = ipp[1], qc = ipp[2];
      const f32x2 nsx = qa.x, nsy = qa.y, nsz = qb.x, ndx = qb.y, ndy = qc.x, ndz = qc.y;
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const f32x2 ax = add2(SX[k], nsx), ay = add2(SY[k], nsy), az = add2(SZ[k], nsz);
        const f32x2 bx = add2(DX[k], ndx), by = add2(DY[k], ndy), bz = add2(DZ[k], ndz);
        const f32x2 a = fma2(az, az, fma2(ay, ay, mul2(ax, ax)));
        const f32x2 bb = fma2(bz, bz, fma2(by, by, mul2(bx, bx)));
        float a0, a1, c0, c1;
        upk2(a, a0, a1);
        upk2(bb, c0, c1);
        float x0, x1;
        upk2(sub2(pk2(sqrt_approx(a0), sqrt_approx(a1)), pk2(sqrt_approx(c0), sqrt_approx(c1))), x0, x1);
        x0 = fabsf(x0);
        x1 = fabsf(x1);
        sure[2 * k] = x0 <= b1;
        dec[2 * k] = sure[2 * k] || (x0 > b2);
        sure[2 * k + 1] = x1 <= b1;
        dec[2 * k + 1] = sure[2 * k + 1] || (x1 > b2);
      }
    };
    uint32_t ambmask = 0u;
    uint32_t bit = 1u;
#pragma unroll 2
    for (int ii = 0; ii < nrows; ++ii, bit <<= 1) {
      bool sure[4], dec[4];
      classify4(ii, sure, dec);
      // NOTE word order: word c covers columns 32c..32c+31 = points jb + 32c; packed slot k holds points
      // jb + 64k (component x) and jb + 64k + 32 (component y), i.e. words 2k and 2k+1.
      uint32_t m[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) m[c] = __ballot_sync(0xffffffffu, sure[c]);
      *reinterpret_cast<uint4*>(&s_rw[32 * w + ii][0]) = make_uint4(m[0], m[1], m[2], m[3]);
      if (!__all_sync(0xffffffffu, dec[0] && dec[1] && dec[2] && dec[3])) ambmask |= bit;
    }
    __syncwarp();
    while (ambmask) {
      const int ii = __ffs(ambmask) - 1;
      ambmask &= ambmask - 1;
      const int i = ibase + ii;
      bool sure[4], dec[4];
      classify4(ii, sure, dec);
      int nre = 0;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int j = jb + 32 * c;
        bool ex = false;
        if (!dec[c] && vj[c] && j != i) {
          ex = scale_mode ? edge_exact_scale(src, dst, i, j, beta, s_hat) : edge_exact(src, dst, i, j, beta);
          ++nre;
        }
        const uint32_t mex = __ballot_sync(0xffffffffu, ex);
        if (lane == 0 && mex) s_rw[32 * w + ii][c] |= mex;
      }
      if (bt.rechecks) {
        nre = __reduce_add_sync(0xffffffffu, nre);
        if (lane == 0 && nre) atomicAdd(bt.rechecks, (unsigned long long)nre);
      }
    }
    if (kVerify) {
      for (int ii = 0; ii < nrows; ++ii) {
        const int i = ibase + ii;
        bool sure[4], dec[4];
        classify4(ii, sure, dec);
        int bad = 0;
        for (int c = 0; c < 4; ++c) {
          const int j = jb + 32 * c;
          if (dec[c] && vj[c] && j != i)
            bad += ((scale_mode ? edge_exact_scale(src, dst, i, j, beta, s_hat) : edge_exact(src, dst, i, j, beta)) !=
                    sure[c]);
        }
        if (bad) atomicAdd(bt.mismatches, (unsigned long long)bad);
      }
    }
    __syncwarp();
    const uint4 rw = *reinterpret_cast<const uint4*>(&s_rw[tid][0]);
    uint32_t roww[4] = {rw.x, rw.y, rw.z, rw.w}, colw[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const uint32_t cm = __ballot_sync(0xffffffffu, vj[c]);
      roww[c] &= cm;
      if (I == J && c == w) roww[c] &= ~(1u << lane);
      colw[c] = warp_transpose32(roww[c], lane) & rmask;
    }
    if (lane < nrows)
      *reinterpret_cast<uint4*>(adj32 + (size_t)(ibase + lane) * P32 + 4 * J) =
          make_uint4(roww[0], roww[1], roww[2], roww[3]);
    if (kFuseDeg) rdeg += __popc(roww[0]) + __popc(roww[1]) + __popc(roww[2]) + __popc(roww[3]);
    if (I != J) {
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (vj[c]) {
          adj32[(size_t)(jb + 32 * c) * P32 + 4 * I + w] = colw[c];
          if (kFuseDeg && colw[c]) atomicAdd(degp + jb + 32 * c, __popc(colw[c]));
        }
    }
    __syncwarp();
  }
  if (kFuseDeg && lane < nrows && rdeg) atomicAdd(degp + ibase + lane, rdeg);
}

// Gram test of graph_strip2_kernel (problems with gc.use_gram; DESIGN.md §3.1).  Per pair, on the centred float copies:
//   a = fma(z_j, -2 z_i, fma(y_j, -2 y_i, fma(x_j, -2 x_i, N_i + N_j))), b the same on the destination cloud,
//   t = a - b, s = a + b,  d_hi = fma(t, t, fma(s, mhi, chi)),  d_lo = fma(t, t, fma(s, mlo, clo))
// = 14 FP32 operations and two funnel shifts that move the sign bits into the lane's column words: sign(d_hi) = 1 proves
// an edge, sign(d_lo) = 0 a non-edge.  No square root, no compare, no vote.  Column points (x, y, z, N), (u, v, w, M) stay
// in registers; row points are broadcast from a warp-private slice as (-2x, -2y, -2z, N), (-2u, -2v, -2w, M).  The
// undecided pairs (lo & ~hi, a few per million) keep bit 0 and are queued for tc_patch_kernel; a full queue is evaluated
// in place.  Row words come from the warp-shuffle bit transpose of the column words.
template <bool kVerify, bool kFuseDeg>
__device__ __forceinline__ void strip_gram(const Batch& bt, const int b, const int I, const int J0, const int J1) {
  const int n = bt.n;
  __shared__ float4 s_gr[2 * kTile];

  const GraphConsts* gcp = bt.gc + b;
  const float mhi = gcp->g_mhi, chi = gcp->g_chi, mlo = gcp->g_mlo, clo = gcp->g_clo;
  const double beta = gcp->beta;
  const bool scale_mode = bt.scale_mode != 0;
  const double s_hat = scale_mode ? bt.sol[b].scale : 1.0;

  const float4* sf = bt.sf + (size_t)b * n;
  const float4* df = bt.df + (size_t)b * n;
  const double* src = bt.src + (size_t)b * n * 3;
  const double* dst = bt.dst + (size_t)b * n * 3;

  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
  const int ibase = I * kTile + 32 * w;
  const int nrows = min(32, n - ibase);
  if (nrows <= 0) return;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  {
    const int i = ibase + lane;
    const float4 s = (i < n) ? sf[i] : z4, d = (i < n) ? df[i] : z4;
    s_gr[2 * tid] = make_float4(-2.f * s.x, -2.f * s.y, -2.f * s.z, s.w);
    s_gr[2 * tid + 1] = make_float4(-2.f * d.x, -2.f * d.y, -2.f * d.z, d.w);
  }
  __syncwarp();
  uint32_t* adj32 = reinterpret_cast<uint32_t*>(bt.adj) + (size_t)b * n * pitch32(n);
  const int P32 = pitch32(n);
  const uint32_t rmask = nrows >= 32 ? 0xffffffffu : ((1u << nrows) - 1u);
  const float4* rows = s_gr + 2 * 32 * w;

  int* degp = bt.deg + (size_t)b * n;
  int rdeg = 0;
  for (int J = J0; J < J1; ++J) {
    const int jb = J * kTile + lane;
    float4 cs[4], cd[4];
    bool vj[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int j = jb + 32 * c;
      vj[c] = j < n;
      cs[c] = vj[c] ? sf[j] : z4;
      cd[c] = vj[c] ? df[j] : z4;
    }
    // column words of this lane: bit ii = pair (row ibase+ii, column jb + 32c); hi = surely an edge, lo = edge or undecided
    uint32_t hi[4] = {0u, 0u, 0u, 0u}, lo[4] = {0u, 0u, 0u, 0u};
    // rows are visited from the last to the first so that the funnel shift leaves row ii at bit ii
#pragma unroll 4
    for (int ii = 31; ii >= 0; --ii) {
      const float4 rs = rows[2 * ii], rd = rows[2 * ii + 1];
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        float a = __fadd_rn(rs.w, cs[c].w);
        a = __fmaf_rn(cs[c].x, rs.x, a);
        a = __fmaf_rn(cs[c].y, rs.y, a);
        a = __fmaf_rn(cs[c].z, rs.z, a);
        float bb = __fadd_rn(rd.w, cd[c].w);
        bb = __fmaf_rn(cd[c].x, rd.x, bb);
        bb = __fmaf_rn(cd[c].y, rd.y, bb);
        bb = __fmaf_rn(cd[c].z, rd.z, bb);
        const float t = __fsub_rn(a, bb), s = __fadd_rn(a, bb);
        const float dh = __fmaf_rn(t, t, __fmaf_rn(s, mhi, chi));
        const float dl = __fmaf_rn(t, t, __fmaf_rn(s, mlo, clo));
        hi[c] = __funnelshift_l(__float_as_uint(dh), hi[c], 1);
        lo[c] = __funnelshift_l(__float_as_uint(dl), lo[c], 1);
      }
    }
    // ---- validity (rows < n, columns < n, i != j), undecided pairs, tentative column words
    uint32_t colw[4];
    int nflag = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      uint32_t vm = vj[c] ? rmask : 0u;
      if (I == J && c == w) vm &= ~(1u << lane);  // column 32c + lane of the diagonal block meets row 32w + lane
      const uint32_t fm = lo[c] & ~hi[c] & vm;
      colw[c] = hi[c] & vm;
      if (kVerify) {  // every DECIDED pair is re-evaluated exactly; disagreements are counted (must stay 0)
        uint32_t dm = vm & ~fm;
        int bad = 0;
        while (dm) {
          const int ii = __ffs(dm) - 1;
          dm &= dm - 1;
          const int i = ibase + ii, j = jb + 32 * c;
          const bool ex = scale_mode ? edge_exact_scale(src, dst, i, j, beta, s_hat) : edge_exact(src, dst, i, j, beta);
          bad += (ex != (((colw[c] >> ii) & 1u) != 0u));
        }
        if (bad) atomicAdd(bt.mismatches, (unsigned long long)bad);
      }
      lo[c] = fm;  // re-used: undecided mask of column c
      nflag += __popc(fm);
    }
    if (__any_sync(0xffffffffu, nflag != 0)) {
      // ---- rare: queue the undecided pairs for tc_patch_kernel (their tentative bit is 0); queue full: exact here
      int incl = nflag;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      const int total = __shfl_sync(0xffffffffu, incl, 31);
      unsigned int base = 0;
      if (lane == 0) base = atomicAdd(bt.tc_list_count, (unsigned int)total);
      base = __shfl_sync(0xffffffffu, base, 0);
      const bool queued = base + (unsigned int)total <= bt.tc_list_cap;
      unsigned int pos = base + (unsigned int)(incl - nflag);
      if (!queued)  // the first warp that does not fit leaves [base, cap) unwritten: void entries for the patch kernel
        for (unsigned int q = base + (unsigned int)lane; q < bt.tc_list_cap; q += 32u) bt.tc_list[q] = make_uint2(0xffffffffu, 0u);
      int nre = 0;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        uint32_t fm = lo[c];
        const int j = jb + 32 * c;
        while (fm) {
          const int ii = __ffs(fm) - 1;
          fm &= fm - 1;
          const int i = ibase + ii;
          if (queued) {
            // the patch kernel flips bit (i, j) and, off the diagonal block, its mirror; the diagonal block holds both
            // orientations as separate pairs, each queued by the lane that owns its column
            bt.tc_list[pos++] = make_uint2((unsigned int)b, ((unsigned int)i << 16) | (unsigned int)j);
          } else {
            const bool ex = scale_mode ? edge_exact_scale(src, dst, i, j, beta, s_hat) : edge_exact(src, dst, i, j, beta);
            colw[c] |= (ex ? 1u : 0u) << ii;
            ++nre;
          }
        }
      }
      if (bt.rechecks && !queued) {
        nre = __reduce_add_sync(0xffffffffu, nre);
        if (lane == 0 && nre) atomicAdd(bt.rechecks, (unsigned long long)nre);
      }
    }
    // ---- row words (lane = row ibase + lane) by transposition; stores; fused degrees
    uint32_t roww[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) roww[c] = warp_transpose32(colw[c], lane);
    if (lane < nrows)
      *reinterpret_cast<uint4*>(adj32 + (size_t)(ibase + lane) * P32 + 4 * J) =
          make_uint4(roww[0], roww[1], roww[2], roww[3]);
    if (kFuseDeg) rdeg += __popc(roww[0]) + __popc(roww[1]) + __popc(roww[2]) + __popc(roww[3]);
    if (I != J) {
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (vj[c]) {
          adj32[(size_t)(jb + 32 * c) * P32 + 4 * I + w] = colw[c];
          if (kFuseDeg && colw[c]) atomicAdd(degp + jb + 32 * c, __popc(colw[c]));
        }
    }
  }
  if (kFuseDeg && lane < nrows && rdeg) atomicAdd(degp + ibase + lane, rdeg);
}

// graph strip kernel (default): one launch for the whole batch; each problem runs the Gram test or the interval test, as
// prep_kernel chose (CTA-uniform: a strip belongs to one problem).  Undecided pairs of the Gram test are settled by
// tc_patch_kernel afterwards (launch_graph).
template <bool kVerify, int kMinBlocks, bool kFuseDeg>
__global__ void __launch_bounds__(kGraphThreads, kMinBlocks) graph_strip2_kernel(Batch bt) {
  const int b = blockIdx.y;
  const int nt = (bt.n + kTile - 1) / kTile;
  int I = 0, p = blockIdx.x;
  while (true) {
    const int ng = (nt - I + kStripBlocks - 1) / kStripBlocks;
    if (p < ng) break;
    p -= ng;
    ++I;
  }
  const int J0 = I + p * kStripBlocks;
  const int J1 = min(nt, J0 + kStripBlocks);
  const GraphConsts* gcp = bt.gc + b;
  if (bt.tc_active && gcp->use_tc) return;  // built by graph_tc_kernel
  if (gcp->use_gram)
    strip_gram<kVerify, kFuseDeg>(bt, b, I, J0, J1);
  else
    strip_interval<kVerify, kFuseDeg>(bt, b, I, J0, J1);
}

// ------------------------------------------------------------------------------------------------
// graph strip kernel v7 (debug flag 2048): same decomposition, inputs and outputs as graph_strip2_kernel, cheaper pair test.
//   * one MUFU per pair instead of two: with t = a-b, s = a+b, q = sqrt(ab), w = s + 2q = (sqrt a + sqrt b)^2 the pair
//     is an edge iff d = t^2 - beta^2 w <= 0 (d = w (g^2 - beta^2), g = |sqrt a - sqrt b|); both sides of the
//     comparison are equal at the threshold, so the FP32 evaluation error is a few ulp of beta^2 w;
//   * no compares and no ballots: d_hi = t^2 - (beta^2 - K) w and d_lo = t^2 - (beta^2 + K) w are formed with two
//     packed FFMA, their SIGN BITS are funnel-shifted into two per-lane column words (sure edge / edge-or-undecided);
//     K = delta (2 beta + delta) + 32 u beta^2 with delta >= |g' - g| (FP32 error of the centred float pipeline), so
//     sign(d_hi) = 1 proves g < beta and sign(d_lo) = 0 proves g > beta;
//   * undecided pairs = lo & ~hi (~3e-6 of the pairs on C2) keep the tentative bit 0 and are queued for
//     tc_patch_kernel (exact FP64 sequence, flips the bit if needed); queue full -> evaluated in place;
//   * the lane's column words ARE the transposed half of the bitset; the row words come from the same 5-stage
//     warp-shuffle transpose as before.
// Per 32 pairs: 12.5 issue slots + 1 MUFU instead of 20 + 2.  a, b >= eps > 0 (eps is folded into the first FMA of each
// squared norm) so w > 0 and zero-length TIM pairs (duplicate correspondences) are classified like any other pair.
// ------------------------------------------------------------------------------------------------
template <bool kVerify, int kMinBlocks>
__global__ void __launch_bounds__(kGraphThreads, kMinBlocks) graph_strip3_kernel(Batch bt) {
  const int b = blockIdx.y;
  const int n = bt.n;
  const int nt = (n + kTile - 1) / kTile;
  int I = 0, p = blockIdx.x;
  while (true) {
    const int ng = (nt - I + kStripBlocks - 1) / kStripBlocks;
    if (p < ng) break;
    p -= ng;
    ++I;
  }
  const int J0 = I + p * kStripBlocks;
  const int J1 = min(nt, J0 + kStripBlocks);

  __shared__ IPointNeg2 s_ip[kTile];

  const GraphConsts* gcp = bt.gc + b;
  if (bt.tc_active && gcp->use_tc) return;  // built by graph_tc_kernel
  const f32x2 nlo = pk2(gcp->f3_nlo, gcp->f3_nlo), nhi = pk2(gcp->f3_nhi, gcp->f3_nhi), two = pk2(2.f, 2.f);
  const f32x2 eps2 = pk2(gcp->f3_eps, gcp->f3_eps);
  const double beta = gcp->beta;
  const bool scale_mode = bt.scale_mode != 0;
  const double s_hat = scale_mode ? bt.sol[b].scale : 1.0;

  const float4* sf = bt.sf + (size_t)b * n;
  const float4* df = bt.df + (size_t)b * n;
  const double* src = bt.src + (size_t)b * n * 3;
  const double* dst = bt.dst + (size_t)b * n * 3;

  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
  const int ibase = I * kTile + 32 * w;
  const int nrows = min(32, n - ibase);
  if (nrows <= 0) return;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  {
    const int i = ibase + lane;
    const float4 s = (i < n) ? sf[i] : z4, d = (i < n) ? df[i] : z4;
    IPointNeg2 ip;
    ip.a = make_float4(-s.x, -s.x, -s.y, -s.y);
    ip.b = make_float4(-s.z, -s.z, -d.x, -d.x);
    ip.c = make_float4(-d.y, -d.y, -d.z, -d.z);
    s_ip[tid] = ip;
  }
  __syncwarp();
  uint32_t* adj32 = reinterpret_cast<uint32_t*>(bt.adj) + (size_t)b * n * pitch32(n);
  const int P32 = pitch32(n);
  const uint32_t rmask = nrows >= 32 ? 0xffffffffu : ((1u << nrows) - 1u);

  const int npadh = npad128(n) / 2;  // 64-bit elements per packed array
  const f32x2* pkp = reinterpret_cast<const f32x2*>(bt.pk + (size_t)b * 6 * npad128(n));
  int* degp = bt.deg + (size_t)b * n;
  int rdeg = 0;
  for (int J = J0; J < J1; ++J) {
    const int jb = J * kTile + lane;
    f32x2 SX[2], SY[2], SZ[2], DX[2], DY[2], DZ[2];
    bool vj[4];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      vj[2 * k] = jb + 64 * k < n;
      vj[2 * k + 1] = jb + 64 * k + 32 < n;
      const size_t e = (size_t)J * 64 + k * 32 + lane;
      SX[k] = pkp[0 * (size_t)npadh + e]; SY[k] = pkp[1 * (size_t)npadh + e]; SZ[k] = pkp[2 * (size_t)npadh + e];
      DX[k] = pkp[3 * (size_t)npadh + e]; DY[k] = pkp[4 * (size_t)npadh + e]; DZ[k] = pkp[5 * (size_t)npadh + e];
    }
    // column words of this lane: bit ii = pair (row ibase+ii, column jb + 32c); hi = surely an edge, lo = edge or undecided
    uint32_t hi[4] = {0u, 0u, 0u, 0u}, lo[4] = {0u, 0u, 0u, 0u};
    // rows are visited from the last to the first so that the funnel shift leaves row ii at bit ii
#pragma unroll 2
    for (int ii = 31; ii >= 0; --ii) {
      const ulonglong2* ipp = reinterpret_cast<const ulonglong2*>(&s_ip[32 * w + ii]);
      const ulonglong2 qa = ipp[0], qb = ipp[1], qc = ipp[2];
      const f32x2 nsx = qa.x, nsy = qa.y, nsz = qb.x, ndx = qb.y, ndy = qc.x, ndz = qc.y;
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const f32x2 ax = add2(SX[k], nsx), ay = add2(SY[k], nsy), az = add2(SZ[k], nsz);
        const f32x2 bx = add2(DX[k], ndx), by = add2(DY[k], ndy), bz = add2(DZ[k], ndz);
        const f32x2 a = fma2(az, az, fma2(ay, ay, fma2(ax, ax, eps2)));
        const f32x2 bb = fma2(bz, bz, fma2(by, by, fma2(bx, bx, eps2)));
        const f32x2 t = sub2(a, bb), s = add2(a, bb);
        float p0, p1;
        upk2(mul2(a, bb), p0, p1);
        const f32x2 q = pk2(sqrt_approx(p0), sqrt_approx(p1));
        const f32x2 ww = fma2(q, two, s), t2 = mul2(t, t);
        float h0, h1, l0, l1;
        upk2(fma2(ww, nhi, t2), h0, h1);
        upk2(fma2(ww, nlo, t2), l0, l1);
        hi[2 * k] = __funnelshift_l(__float_as_uint(h0), hi[2 * k], 1);
        hi[2 * k + 1] = __funnelshift_l(__float_as_uint(h1), hi[2 * k + 1], 1);
        lo[2 * k] = __funnelshift_l(__float_as_uint(l0), lo[2 * k], 1);
        lo[2 * k + 1] = __funnelshift_l(__float_as_uint(l1), lo[2 * k + 1], 1);
      }
    }
    // ---- validity (rows < n, columns < n, i != j), undecided pairs, tentative column words
    uint32_t colw[4];
    int nflag = 0;
    if (gcp->use_fp64) {  // exact path for every pair (non-finite input, huge range, debug flag 1)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        hi[c] = 0u;
        lo[c] = 0xffffffffu;
      }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      uint32_t vm = vj[c] ? rmask : 0u;
      if (I == J && c == w) vm &= ~(1u << lane);  // column 32c + lane of the diagonal block meets row 32w + lane
      uint32_t fm = lo[c] & ~hi[c] & vm;
      colw[c] = hi[c] & vm;
      if (kVerify) {  // every DECIDED pair is re-evaluated exactly; disagreements are counted (must stay 0)
        uint32_t dm = vm & ~fm;
        int bad = 0;
        while (dm) {
          const int ii = __ffs(dm) - 1;
          dm &= dm - 1;
          const int i = ibase + ii, j = jb + 32 * c;
          const bool ex = scale_mode ? edge_exact_scale(src, dst, i, j, beta, s_hat) : edge_exact(src, dst, i, j, beta);
          bad += (ex != (((colw[c] >> ii) & 1u) != 0u));
        }
        if (bad) atomicAdd(bt.mismatches, (unsigned long long)bad);
      }
      lo[c] = fm;  // re-used: undecided mask of column c
      nflag += __popc(fm);
    }
    if (__any_sync(0xffffffffu, nflag != 0)) {
      // ---- rare: queue the undecided pairs for tc_patch_kernel (their tentative bit is 0); queue full: exact here
      int incl = nflag;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      const int total = __shfl_sync(0xffffffffu, incl, 31);
      unsigned int base = 0;
      if (lane == 0) base = atomicAdd(bt.tc_list_count, (unsigned int)total);
      base = __shfl_sync(0xffffffffu, base, 0);
      const bool queued = base + (unsigned int)total <= bt.tc_list_cap;
      unsigned int pos = base + (unsigned int)(incl - nflag);
      if (!queued)  // the first warp that does not fit leaves [base, cap) unwritten: void entries for the patch kernel
        for (unsigned int q = base + (unsigned int)lane; q < bt.tc_list_cap; q += 32u) bt.tc_list[q] = make_uint2(0xffffffffu, 0u);
      int nre = 0;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        uint32_t fm = lo[c];
        const int j = jb + 32 * c;
        while (fm) {
          const int ii = __ffs(fm) - 1;
          fm &= fm - 1;
          const int i = ibase + ii;
          if (queued) {
            // the patch kernel flips bit (i, j) and, off the diagonal block, its mirror; the diagonal block holds both
            // orientations as separate pairs, each queued by the lane that owns its column
            bt.tc_list[pos++] = make_uint2((unsigned int)b, ((unsigned int)i << 16) | (unsigned int)j);
          } else {
            const bool ex = scale_mode ? edge_exact_scale(src, dst, i, j, beta, s_hat) : edge_exact(src, dst, i, j, beta);
            colw[c] |= (ex ? 1u : 0u) << ii;
            ++nre;
          }
        }
      }
      if (bt.rechecks && !queued) {
        nre = __reduce_add_sync(0xffffffffu, nre);
        if (lane == 0 && nre) atomicAdd(bt.rechecks, (unsigned long long)nre);
      }
    }
    // ---- row words (lane = row ibase + lane) by transposition; stores; fused degrees
    uint32_t roww[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) roww[c] = warp_transpose32(colw[c], lane);
    if (lane < nrows)
      *reinterpret_cast<uint4*>(adj32 + (size_t)(ibase + lane) * P32 + 4 * J) =
          make_uint4(roww[0], roww[1], roww[2], roww[3]);
    rdeg += __popc(roww[0]) + __popc(roww[1]) + __popc(roww[2]) + __popc(roww[3]);
    if (I != J) {
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (vj[c]) {
          adj32[(size_t)(jb + 32 * c) * P32 + 4 * I + w] = colw[c];
          if (colw[c]) atomicAdd(degp + jb + 32 * c, __popc(colw[c]));
        }
    }
  }
  if (lane < nrows && rdeg) atomicAdd(degp + ibase + lane, rdeg);
}

// n_edges2[b] = sum of degrees (the fused-degree path has no degree kernel to do it)
__global__ void __launch_bounds__(256) edge_count_kernel(Batch bt) {
  const int b = blockIdx.x, n = bt.n;
  __shared__ unsigned long long s_sum[8];
  unsigned long long s = 0;
  for (int v = threadIdx.x; v < n; v += 256) s += (unsigned long long)bt.deg[(size_t)b * n + v];
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int q = 0; q < 8; ++q) t += s_sum[q];
    bt.n_edges2[b] = t;
  }
}

// ------------------------------------------------------------------------------------------------
// degree kernel: deg[v] = popcount(row v); n_edges2[b] = sum of degrees.  One warp per row.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) degree_kernel(Batch bt) {
  const int b = blockIdx.y;
  const int n = bt.n;
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  __shared__ int s_sum[8];
  int d = 0;
  if (row < n) {
    const int P = pitch64(n);
    const uint64_t* r = bt.adj + ((size_t)b * n + row) * P;
    for (int x = lane; x < P; x += 32) d += __popcll(r[x]);
    for (int o = 16; o; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    if (lane == 0) bt.deg[(size_t)b * n + row] = d;
  }
  if (lane == 0) s_sum[threadIdx.x >> 5] = d;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int q = 0; q < 8; ++q) s += s_sum[q];
    if (s) atomicAdd(bt.n_edges2 + b, (unsigned long long)s);
  }
}

void launch_prep(const Batch& bt, cudaStream_t st) { prep_kernel<<<bt.B, 256, 0, st>>>(bt); }

int launch_graph(const Batch& bt0, cudaStream_t st, int num_sms) {
  Batch bt = bt0;
  // default: CUDA-core strip kernel.  Debug flag 1024 routes every problem prep_kernel marked use_tc through the
  // tensor-core kernel instead (bit-identical output: DESIGN.md §3.1)
  bt.tc_active = tc_path_active(bt.flags_dbg) ? 1 : 0;
  int launches = 1;  // the CUDA-core strip kernel below (grid covers every problem; TC problems return at once)
  if (bt.tc_active) launches += launch_graph_tc(bt, st, num_sms);
  const int nt = (bt.n + kTile - 1) / kTile;
  dim3 grid((unsigned)(nt * (nt + 1) / 2), (unsigned)bt.B);
#ifdef TZR_AB_KERNELS
  if (bt.flags_dbg & 8u) {  // first design (one CTA per 128x128 tile, staged through shared memory): A/B only
    if (bt.flags_dbg & 2u)
      graph_tile_kernel<true><<<grid, kGraphThreads, 0, st>>>(bt);
    else
      graph_tile_kernel<false><<<grid, kGraphThreads, 0, st>>>(bt);
    return launches;
  }
#endif
  dim3 sgrid((unsigned)strip_grid(bt.n), (unsigned)bt.B);
  if (!bt.tc_active) cudaMemsetAsync(bt.tc_list_count, 0, sizeof(unsigned int), st);  // (launch_graph_tc zeroes it otherwise)
  bool v7 = false;
  if (bt.flags_dbg & 2048u) {  // v7 (one MUFU, sign-bit words, re-check queue): fewer instructions, but FMA-pipe bound
    v7 = true;
    if (bt.flags_dbg & 2u)
      graph_strip3_kernel<true, 5><<<sgrid, kGraphThreads, 0, st>>>(bt);
    else
      graph_strip3_kernel<false, 8><<<sgrid, kGraphThreads, 0, st>>>(bt);
  }
#ifdef TZR_AB_KERNELS
  else if (bt.flags_dbg & 16u)  // occupancy A/B: 6 CTAs/SM (80 registers)
    graph_strip_kernel<false, 6><<<sgrid, kGraphThreads, 0, st>>>(bt);
  else if (bt.flags_dbg & 32u)  // occupancy A/B: 5 CTAs/SM (96 registers)
    graph_strip_kernel<false, 5><<<sgrid, kGraphThreads, 0, st>>>(bt);
  else if (bt.flags_dbg & 64u)  // scalar-FP32 strip kernel (A/B against the paired default)
    graph_strip_kernel<false, 8><<<sgrid, kGraphThreads, 0, st>>>(bt);
  else if (bt.flags_dbg & 128u)  // paired kernel at 6 CTAs/SM
    graph_strip2_kernel<false, 6, false><<<sgrid, kGraphThreads, 0, st>>>(bt);
#endif
  else if (bt.flags_dbg & 2u)
    graph_strip2_kernel<true, 5, false><<<sgrid, kGraphThreads, 0, st>>>(bt);
  else if (bt.flags_dbg & 256u)  // degrees by the separate degree kernel (A/B against the fused default)
    graph_strip2_kernel<false, 8, false><<<sgrid, kGraphThreads, 0, st>>>(bt);
  else  // default: Gram test (interval test where prep_kernel's guard fails), 8 CTAs/SM, degrees fused
    graph_strip2_kernel<false, 8, true><<<sgrid, kGraphThreads, 0, st>>>(bt);
  // exact re-check of the pairs the strip kernel queued (v7, or the Gram test: every problem unless debug flag 512)
  if (v7 || !(bt.flags_dbg & 512u)) {
    launch_graph_patch(bt, st, num_sms);
    ++launches;
  }
  return launches;
}

// fused degrees: the default kernel (not its verify variant), and v7 always
bool graph_fuses_degrees(const Batch& bt) {
  if (bt.flags_dbg & (8u | 16u | 32u | 64u | 128u | 256u)) return false;
  if (bt.flags_dbg & 2048u) return true;
  return (bt.flags_dbg & 2u) == 0;
}

void launch_degree(const Batch& bt, cudaStream_t st, bool bitset_only) {
  if (!bitset_only && graph_fuses_degrees(bt)) {  // degrees were accumulated by the graph kernel; only the edge count is left
    edge_count_kernel<<<bt.B, 256, 0, st>>>(bt);
    return;
  }
  dim3 grid((unsigned)((bt.n + 7) / 8), (unsigned)bt.B);
  degree_kernel<<<grid, 256, 0, st>>>(bt);
}

}  // namespace tzr
