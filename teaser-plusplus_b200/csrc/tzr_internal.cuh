// Internal declarations shared by the CUDA translation units of libteaser_b200.so.
// Product code: nothing here (or in any file of this directory) includes or links oracle/.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <string>
#include <vector>

#include "../../include/teaser_b200.h"

namespace tzr {

// ---- adjacency layout -------------------------------------------------------------------------
// Device-internal adjacency: n rows, pitch64(n) uint64 words per row.  The pitch is padded to whole
// 128-column tiles (2 words) so that every 128x128 tile of the graph kernel maps to one aligned
// 16-byte segment per row.  The ABI layout (ceil(n/64) words per row) is produced by a pitched copy.
__host__ __device__ inline int pitch64(int n) { return 2 * ((n + 127) / 128); }
__host__ __device__ inline int pitch32(int n) { return 2 * pitch64(n); }
__host__ __device__ inline int words64(int n) { return (n + 63) / 64; }
__host__ __device__ inline int npad128(int n) { return 128 * ((n + 127) / 128); }
// smallest power of two >= v: the padded end-point count of the bitonic TLS sort (tls_device.cuh)
__host__ __device__ inline int next_pow2(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}
// byte offsets of workspace regions: every region starts on a 256-byte boundary
inline size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }

constexpr int kTile = 128;          // graph tile edge (pairs per tile = 128*128)
constexpr int kGraphThreads = 128;  // 4 warps, each owns a 32x128 sub-tile (4 pairs per lane per step)
constexpr int kHeurRoots = 4;       // heuristic start vertices per problem (top degrees); a global-peeling
                                    // second chance in the peel kernel covers the cases they all miss
constexpr int kMatchMaxDim = 128;   // feature dimension limit of the matcher's NN kernel (FPFH: 33)
constexpr double kTcKappa = 64.0;   // allowance for the tensor-core Gram error |a' - a| in units of u D^2 (u = 2^-24, D = largest
                                    // distance inside the cloud).  EMPIRICAL, not a proven bound: the 24 tf32 products are
                                    // exact, but the order and rounding of wgmma's FP32 accumulation are not documented, and a
                                    // worst case of one truncation per addition on partial sums of up to ~4 D^2 would allow a
                                    // few hundred u D^2.  The value is backed by debug flag 2, which re-checks every decided
                                    // pair against FP64; tests/test_gpu_round2.py asserts no mismatch on every tensor-core
                                    // case.  A larger value would be safer but sends well-conditioned problems (beta/D ~ 1/250)
                                    // back to the CUDA-core kernel through prep_kernel's 64 E <= 0.75 D beta test.  The path
                                    // is opt-in (debug flag 1024).
constexpr int kMaxN = 32768;        // per-problem size limit of the shared-memory clique kernels (the small route; the
                                    // large route compacts the graph's core to at most this many vertices)
constexpr int kMaxNLarge = 65536;   // per-problem size limit of the whole pipeline (tzr_ctx_set_max_n): the graph kernels'
                                    // re-check queue packs a pair as (i << 16) | j and the heuristic keeps u16 candidate
                                    // lists and in-set degrees, so every vertex index must fit 16 bits
constexpr int kCoreRounds = 48;     // peel rounds (one launch each) per block of the large route's core peel; the host
                                    // runs further blocks while a problem it would search or cap is still shrinking
constexpr int kCoreSlots = kCoreRounds + 1;  // change counters per problem: "peel on" + one per round of a block

// Per-problem constants of the FP32 filter (see graph_build.cu).
struct GraphConsts {
  float b1;       // x = ||ds| - |dd|| <= b1  : surely an edge      (beta - delta; -1 = never)
  float b2;       // x > b2                   : surely not an edge  (beta + delta; +inf = never)
  int use_fp64;   // 1: FP32 filter disabled for this problem (range/NaN guard or debug flag)
  int pad;
  double beta;    // 2*noise_bound*sqrt(cbar2)
  double cs[3], cd[3];  // centres subtracted before the float conversion
  float f3_nlo, f3_nhi;  // graph_strip3_kernel: -(beta^2 + K), -(beta^2 - K)   (K: undecided band relative to w)
  float f3_eps;          // bias of the squared norms (keeps w > 0)
  int pad2;
  double s_hat;   // scale applied to the centred source copies (1 unless estimate_scaling)
  // tensor-core filter (graph_tc.cu): d = (a-b)^2 - 2 beta^2 (a+b) + beta^4 from the Gram-form squared norms (no square root)
  int use_tc;     // 1: this problem goes through graph_tc_kernel, 0: through the CUDA-core strip kernel
  float tc_c2;    // 2 beta^2
  float tc_b4;    // beta^4
  float tc_kap, tc_c0;  // |d| <= kap (t^2 + beta^4) + c0 : undecided -> exact FP64 re-check   (t = a - b)
  float tc_pad;
  // Gram-form test of graph_strip2_kernel (DESIGN.md §3.1): with a', b' the FP32 Gram-form squared norms, t = a' - b',
  // s = a' + b':  t^2 + g_mhi s + g_chi <= 0 proves an edge, t^2 + g_mlo s + g_clo >= 0 proves a non-edge
  int use_gram;   // 1: the conditioning guard holds, the strip kernel runs the Gram test; 0: the sqrt interval test (b1, b2)
  float g_mhi, g_chi, g_mlo, g_clo;  // two-slope form (debug flag 134217728)
  // single-slope form (default), lengths in units of 2 beta (Batch::gq): with u = c_u - a', v = c_v - b' (c_v = c_u + 1/4
  // exactly) and T = v - u, sign(fma(T, T, u)) = 1 proves an edge and sign(fma(T, T, u) + g_dl) = 0 a non-edge
  float g_cu, g_cv, g_dl;
};

// Everything the device kernels need to know about one batch (passed by value).
struct Batch {
  int B;          // problems
  double tc_kappa; // bound on the tensor-core Gram error in units of 2^-24 D^2 (kTcKappa; env TZR_TC_KAPPA for experiments)
  int tc_desc_swap; // debug (env TZR_TC_SWAP): exchange the leading/stride byte offsets of the MMA operand descriptors
  int tc_active;  // 1: problems with gc.use_tc are built by graph_tc_kernel and skipped by the CUDA-core strip kernel
  int scale_mode; // 1: estimate_scaling=true (TLSScaleSolver predicate, scale from sol[b].scale)
  int n;          // correspondences per problem (uniform inside a device batch)
  double beta;    // 2*noise_bound*sqrt(cbar2)  (registration.cc:438)
  const double* src;  // B*n*3
  const double* dst;  // B*n*3
  float4* sf;     // B*n centred float copies; w = their squared norm, rounded to float (Gram-form test)
  float4* df;
  float4* gq;     // B*n*2: the same points in units of 2 beta (x, y, z, squared norm), source at 2i and destination at
                  // 2i+1; written by prep_kernel for the problems that run the single-slope Gram test
  float* opnd;   // B * ceil(n/128) * 2 roles * 2 clouds * 6 planes * 128 rows * 4: tf32-split MMA operand tiles of the
                  // tensor-core graph kernel (graph_tc.cu), written by tc_prep_kernel
  uint2* tc_list;         // re-check queue of the tensor-core graph kernel: (problem, i << 16 | j)
  unsigned int* tc_list_count;  // 1 (may exceed the capacity: writers past it evaluate in place)
  unsigned int tc_list_cap;
  float* pk;      // B*6*npad128(n): the same centred floats, pair-interleaved per 128-column block for the packed
                  // FP32x2 graph kernel (arrays sx,sy,sz,dx,dy,dz; element of point j at blk*128 + k*64 + lane*2 + half)
  GraphConsts* gc;        // B
  uint64_t* adj;          // B*n*pitch64(n)
  int32_t* deg;           // B*n
  unsigned long long* n_edges2;  // B (sum of degrees = 2*edges)
  // clique state
  int32_t* hclq;          // B*kHeurRoots*n heuristic cliques
  int32_t* hsize;         // B*kHeurRoots
  int32_t* clq;           // B*n incumbent clique (unsorted)
  int32_t* L;             // B incumbent size
  uint32_t* alive;        // B*pitch32(n) bitset of vertices surviving the (L-1)-core peel
  uint32_t* best_bits;    // B*pitch32(n) incumbent clique as a bitset (canonical tie-break)
  int32_t* alive_cnt;     // B
  int32_t* root_ctr;      // B work counter for the exact phase
  int32_t* lock;          // B spin lock for incumbent updates
  int32_t* flags;         // B bit0: search incomplete (depth/time budget)
  int32_t* kcore_final;   // B (KCORE_HEU only, else nullptr): 1 = clq/L already final (max-core shortcut)
  // exact-phase scratch
  uint32_t* stack;        // per warp: max_depth * 2 * pitch32 words
  int32_t* cv;            // per warp: n ints (current clique)
  int32_t* centry;        // per warp: max_depth ints
  int max_depth;
  int exact_ctas;         // CTAs of the (persistent) exact-phase grid; scratch above is per warp of that grid
  int exact_conc;         // problems searched at a time (bitsets that fit the L2 together)
  // rotation / translation scratch (per problem)
  double* ps;             // B*3*n chain TIMs src
  double* pd;             // B*3*n chain TIMs dst (de-scaled)
  double* wgt;            // B*rot_cap GNC weights (one per rotation TIM)
  double* res;            // B*n scratch
  long long rot_cap;      // rotation TIMs per problem the workspace can hold (n for CHAIN)
  double* skey;           // B*3*sort_cap sort keys (per axis)
  int32_t* sidx;          // B*3*sort_cap sort payload
  int sort_cap;           // next_pow2(2n): per-axis capacity of skey/sidx
  int32_t* sorted_clq;    // B*n sorted clique (output order)
  uint8_t* rot_mask;      // B*rot_cap
  uint8_t* trans_mask;    // B*n
  tzr_solution* sol;      // B
  // debug
  unsigned long long* mismatches;  // 1
  unsigned long long* rechecks;    // 1
  uint32_t flags_dbg;
  unsigned long long budget_ns;    // time budget of the exact clique search per problem (0 = none), Params::max_clique_time_limit
  unsigned long long* t_start;     // B: %globaltimer when the first search warp of the problem started (0 = not yet)
  // Ragged size class (DESIGN.md §4.2): problem b has nb[b] <= n correspondences in the first nb[b] rows of its padded
  // slot; n stays the size of every pitch and offset.  nullptr for uniform batches.  Kept last so that the fields above
  // keep their parameter offsets in every kernel.
  const int32_t* nb;        // device, B entries
  const int32_t* nb_host;   // host copy of nb (the unknown-scale large path's per-problem host loop)
  int strip_blocks;         // 128-column blocks per strip of graph_strip2_kernel; set by launch_graph from B and n
};

// ---- rotation TIM sets (shared by rot_trans_kernel and the certifier's gather of a retained solve) ----------------------
constexpr int kRTThreads = 128;  // threads of the CTAs that walk a TIM set (rot_trans.cu: 128 regs x 128 threads, 4 CTAs/SM)

// CHAIN (registration.cc:657-680): m TIMs materialised in ps/pd (pd already de-scaled, :697).
// COMPLETE (registration.cc:681-694): all m(m-1)/2 differences of the clique points, in computeTIMs order
// k = i*m - i(i+1)/2 + (j-i-1); they are recomputed from the m clique points on every pass instead of being
// materialised (only the per-TIM weight has to persist between GNC iterations).
struct TimSrc {
  int complete;
  int m;                // chain: number of TIMs; complete: number of clique points
  long long count;      // number of TIMs
  const double* a;      // chain: src TIMs (3*m)        complete: clique src points (3*m)
  const double* b;      // chain: dst TIMs, de-scaled   complete: clique dst points (3*m)
  double inv_scale;     // complete only: 1/scale applied to dst differences
};

// f(k, src TIM xyz, dst TIM xyz) for every TIM of the set, strided over a CTA of kRTThreads threads
template <class F>
__device__ __forceinline__ void for_each_tim(const TimSrc& t, F&& f) {
  if (!t.complete) {
    for (int k = threadIdx.x; k < t.m; k += kRTThreads)
      f((long long)k, t.a[3 * k], t.a[3 * k + 1], t.a[3 * k + 2], t.b[3 * k], t.b[3 * k + 1], t.b[3 * k + 2]);
  } else {
    for (int i = 0; i + 1 < t.m; ++i) {
      const long long base = (long long)i * t.m - (long long)i * (i + 1) / 2 - i - 1;
      const double sx = t.a[3 * i], sy = t.a[3 * i + 1], sz = t.a[3 * i + 2];
      const double dx = t.b[3 * i], dy = t.b[3 * i + 1], dz = t.b[3 * i + 2];
      for (int j = i + 1 + threadIdx.x; j < t.m; j += kRTThreads)
        f(base + j, t.a[3 * j] - sx, t.a[3 * j + 1] - sy, t.a[3 * j + 2] - sz, (t.b[3 * j] - dx) * t.inv_scale,
          (t.b[3 * j + 1] - dy) * t.inv_scale, (t.b[3 * j + 2] - dz) * t.inv_scale);
    }
  }
}

// ||v_j - v_i|| exactly as the reference computes a TIM norm: IEEE double, no FMA contraction,
// src.array().square().colwise().sum() summed as (x^2 + y^2) + z^2   (registration.cc:415-418, :434-437)
__device__ __forceinline__ double tim_norm_exact(const double* __restrict__ p, int i, int j) {
  const double dx = __dsub_rn(p[3 * j + 0], p[3 * i + 0]);
  const double dy = __dsub_rn(p[3 * j + 1], p[3 * i + 1]);
  const double dz = __dsub_rn(p[3 * j + 2], p[3 * i + 2]);
  const double s = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
  return __dsqrt_rn(s);
}

// exact predicate: the reference's operation sequence in IEEE double, no contraction (registration.cc:427-443).
// Deliberately NOT inlined: it runs for ~1e-4 of the pairs; keeping its two DSQRT expansions out of the unrolled
// sweeps keeps the hot loops small enough for the instruction cache.
static __device__ __noinline__ bool edge_exact(const double* __restrict__ src, const double* __restrict__ dst, int i,
                                               int j, double beta) {
  const double d1 = tim_norm_exact(src, i, j);
  const double d2 = tim_norm_exact(dst, i, j);
  return fabs(__dsub_rn(d1, d2)) <= beta;  // (v1_dist - v2_dist).abs() <= beta   registration.cc:442
}

// Unknown-scale predicate (TLSScaleSolver, registration.cc:410-425 + :86): the pair is an inlier iff
// | d2/d1 - s_hat | <= beta * (1/d1), with s_hat the TLS scale estimate; at d1 = 0 iff d2 <= beta.
static __device__ __noinline__ bool edge_exact_scale(const double* __restrict__ src, const double* __restrict__ dst,
                                                     int i, int j, double beta, double s_hat) {
  const double d1 = tim_norm_exact(src, i, j);
  const double d2 = tim_norm_exact(dst, i, j);
  // repeated source point: the fixed-scale rule |d2 - s*d1| <= beta at d1 = 0, which is what the FP32 filter computes
  // on its pre-scaled copies (the reference's inf <= inf would make the pair an edge for every d2; DESIGN.md §3.4)
  if (d1 == 0.0) return d2 <= beta;
  const double ratio = __ddiv_rn(d2, d1);
  const double alpha = __dmul_rn(beta, __ddiv_rn(1.0, d1));
  return fabs(__dsub_rn(ratio, s_hat)) <= alpha;
}

// x with A x = -g by the truncated, diagonally pivoted LDL^T of include/teaser_b200.h (one thread): ICP's 6 x 6 step
// (icp.cu) and the 3 x 3 colour gradients (fpfh.cu, which pass g = -h to solve A x = h; the negation is exact).  A: the
// N (N + 1) / 2 entries of the upper triangle row by row.  tol = 1e-10 max_k A_kk; step k takes the remaining index
// with the largest current diagonal (a NaN diagonal is never the largest; the lowest index on ties) and stops unless
// that diagonal is > tol; every component not reached is 0.
template <int N>
__device__ void ldlt_solve(const double* __restrict__ Aup, const double* __restrict__ g, double x[N]) {
  double S[N][N];
  int k = 0;
  for (int r = 0; r < N; ++r)
    for (int c = r; c < N; ++c) S[r][c] = S[c][r] = Aup[k++];
  double amax = S[0][0];
  for (int r = 1; r < N; ++r) amax = fmax(amax, S[r][r]);
  const double tol = 1e-10 * amax;
  int piv[N];
  bool used[N];
  for (int i = 0; i < N; ++i) used[i] = false;
  double d[N], L[N][N];  // L[i][s]: multiplier of original index i at step s
  int rank = 0;
  for (int s = 0; s < N; ++s) {
    int best = -1;
    for (int i = 0; i < N; ++i)
      if (!used[i] && (best < 0 || S[i][i] > S[best][best] || (S[best][best] != S[best][best] && S[i][i] == S[i][i])))
        best = i;
    if (!(S[best][best] > tol)) break;
    used[best] = true;
    piv[s] = best;
    d[s] = S[best][best];
    rank = s + 1;
    for (int i = 0; i < N; ++i)
      if (!used[i]) L[i][s] = S[i][best] / d[s];
    for (int i = 0; i < N; ++i)
      if (!used[i])
        for (int c = 0; c < N; ++c)
          if (!used[c]) S[i][c] = S[i][c] - L[i][s] * S[best][c];
  }
  double y[N];
  for (int s = 0; s < rank; ++s) {  // L z = -P g, z / d
    double z = -g[piv[s]];
    for (int q = 0; q < s; ++q) z = z - L[piv[s]][q] * y[q];
    y[s] = z;
  }
  for (int s = 0; s < rank; ++s) y[s] = y[s] / d[s];
  for (int s = rank - 1; s >= 0; --s) {  // L^T y = w
    double z = y[s];
    for (int q = s + 1; q < rank; ++q) z = z - L[piv[q]][s] * y[q];
    y[s] = z;
  }
  for (int i = 0; i < N; ++i) x[i] = 0.0;
  for (int s = 0; s < rank; ++s) x[piv[s]] = y[s];
}

// kernels (defined in the .cu files) -------------------------------------------------------------
void launch_prep(const Batch& bt, cudaStream_t st);
// returns the number of kernels launched; strip_blocks (may be NULL): graph_strip2_kernel's strip length, 0 if it did not run
int launch_graph(const Batch& bt, cudaStream_t st, int num_sms, int* strip_blocks = nullptr);
// graph_strip2_kernel's strip order on the host: the (I, J0) of strips 0 ... strips_below(nt, L) - 1 (either may be
// NULL); returns their count, 0 when nt or L is not positive
int strip_schedule(int nt, int L, int32_t* I, int32_t* J0);
// graph_tc.cu: tensor-core path (operand tiles + wgmma kernel) for the problems prep_kernel marked use_tc
int launch_graph_tc(const Batch& bt, cudaStream_t st, int num_sms);
size_t tc_operand_bytes(int B, int n);
size_t tc_list_entries(int B, int n);
void launch_graph_patch(const Batch& bt, cudaStream_t st, int num_sms);  // tc_patch_kernel over the re-check queue
// bitset_only: the adjacency did not come from launch_graph (tzr_max_clique on a caller's bitset): always popcount
void launch_degree(const Batch& bt, cudaStream_t st, bool bitset_only = false);
void launch_clique(const Batch& bt, const tzr_params& p, int mode, cudaStream_t st, int* n_launches);
// scale_tls.cu: the scalar TLS launches with per-measurement ranges (tzr_scalar_tls and the unknown-scale stage).
// The small path sorts in one CTA per estimator (tls_block), the large path with a radix sort and tiled scans.
// tls_scratch_bytes: sort scratch of `count` estimators over m measurements each; 0 when the 2m end points do not fit
// the int payload (TZR_ERR_TOO_LARGE).  The large path runs one estimator at a time.
size_t tls_scratch_bytes(long long m, int count, bool large);
int launch_scalar_tls(const double* x, const double* ranges, long long m, bool large, void* scratch, double* out_est,
                      uint8_t* inliers, cudaStream_t st);
// Unknown-scale stage: TIM ratios, ranges and sort scratch of a batch (0: too large), and its launches.
size_t scale_scratch_bytes(int B, int n, uint32_t flags);
// Which of the two scale paths a problem of n correspondences takes (the large one above 256, or under debug flag 262144).
// The paths differ in the last bits of the estimate, so a ragged size class never mixes them.
bool scale_large(int n, uint32_t flags);
int launch_scale_estimation(const Batch& bt, uint32_t flags, void* scratch, cudaStream_t st);
void launch_rot_trans(const Batch& bt, const tzr_params& p, int use_clique, cudaStream_t st);
// Large route (n > kMaxN or debug flag 524288; DESIGN.md §3.2).  lists: B * kHeurRoots * 2n u16 of heuristic scratch;
// chg: B * kCoreSlots change counters (slot 0: peel this problem in the next block of rounds; slot r + 1: removals in
// round r of the block); new2old / old2new: B * n; core_cnt / route: B.  launch_core starts the peel (alive0 and one
// block), launch_core_rounds runs one more block of kCoreRounds rounds on the problems whose slot 0 the host set, then
// re-lists the survivors.  route[b] (device copy, set by the host once every problem it decides on holds its core):
// > 0 search the compacted core, 0 not searched (result already final), -1 core above the cap (heuristic clique, not
// proven).
void launch_clique_large_front(const Batch& bt, const tzr_params& p, int mode, uint16_t* lists, cudaStream_t st,
                               int* n_launches);
void launch_core(const Batch& bt, int32_t* chg, int32_t* new2old, int32_t* old2new, int32_t* core_cnt, int num_sms,
                 cudaStream_t st, int* n_launches);
void launch_core_rounds(const Batch& bt, int32_t* chg, int32_t* new2old, int32_t* old2new, int32_t* core_cnt,
                        int num_sms, cudaStream_t st, int* n_launches);
void launch_core_compact(const Batch& bt, const Batch& cb, const int32_t* new2old, const int32_t* old2new,
                         const int32_t* core_cnt, const int32_t* route, cudaStream_t st, int* n_launches);
void launch_clique_search(const Batch& cb, cudaStream_t st, int* n_launches);  // peel (mode 0) + the exact passes
void launch_core_map_back(const Batch& bt, const Batch& cb, const int32_t* new2old, const int32_t* route,
                          cudaStream_t st, int* n_launches);
size_t clique_heur_smem(int n);
size_t clique_peel_smem(int n);
size_t clique_exact_smem(int n);
int clique_exact_grid(int n, int num_sms);  // CTAs of the persistent exact-phase grid on the current device

// stand-alone stage helpers used by the per-stage C-ABI entry points
void launch_gnc_only(int alg, const double* src, const double* dst, int m, double noise_bound, double gnc_factor,
                     unsigned long long max_iter, double cost_thr, double* wgt, double* res, double* out_R,
                     uint8_t* mask, double* out_cost, int* out_iters, cudaStream_t st);
// key/idx: 3 * next_pow2(2m) entries, raw: 3m doubles
void launch_translation_only(const double* src, const double* dst, int m, double beta, double* key, int32_t* idx,
                             double* raw, double* out_t, uint8_t* mask, cudaStream_t st);

// fpfh.cu (FPFHEstimation::computeFPFHFeatures, fpfh.cc:15-43), over B clouds stored back to back
struct FpfhCloud {     // one per cloud, filled by fpfh_plan, read by the kernels from device memory
  int lo, n;           // first point of the cloud in the flat array, point count
  int grid;            // 1: radius search through the hashed grid (n >= kGridMinN, or forced), 0: brute force
  unsigned int mask;   // T_b - 1 (T_b buckets, a power of two)
  unsigned int base;   // first bucket of the cloud in the batch's bucket range
  int mins[4];         // bounding-box minimum of the finite coordinates (ordered-int floats; the grid origin); [3] = 1:
                       // a finite point lies outside the grid's accurate index range, the cloud uses brute force
  double inv_h;        // 1 / cell edge
};

// The hashed uniform grid of the radius searches (fpfh.cu) and of ICP's nearest-neighbour search (icp.cu)
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

// bounding-box minimum over finite coordinates (ordered-int encoding of floats)
__device__ __forceinline__ int f2ord(float f) {
  const int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

struct FpfhPlan {
  int B = 0, N = 0;            // clouds, points in all of them
  bool any_grid = false;
  unsigned int buckets = 0;    // sum of T_b over the grid clouds (also the sentinel key of unsorted points)
  size_t grid_bytes = 0;       // device scratch of the grid path (0 without grid clouds)
};
// Radius-search route of every cloud: by size (the grid from kGridMinN points on), or forced by a debug flag pair:
// brute force or the grid at any size, bits 22 / 23 for the descriptor stage and bits 25 / 26 for ICP's target search.
constexpr int kFpfhRouteAuto = 0, kFpfhRouteBrute = 1, kFpfhRouteGrid = 2;
constexpr uint32_t kFlagFpfhBrute = 1u << 22, kFlagFpfhGrid = 1u << 23;
constexpr uint32_t kFlagIcpBrute = 1u << 25, kFlagIcpGrid = 1u << 26;
inline int search_route(uint32_t flags, uint32_t brute, uint32_t grid) {
  return (flags & brute) ? kFpfhRouteBrute : (flags & grid) ? kFpfhRouteGrid : kFpfhRouteAuto;
}
// Fills clouds[0..B) (host copy, to be staged to the device before launch_fpfh) and the plan.  TZR_ERR_TOO_LARGE when
// the points or buckets of the batch do not fit 32-bit indices.  grid_min_n: the size from which kFpfhRouteAuto uses
// the grid (-1: the descriptor stage's own, 4096).
int fpfh_plan(int B, const int32_t* n, double normal_radius, double fpfh_radius, int route, FpfhCloud* clouds,
              FpfhPlan* plan, int grid_min_n = -1);
// The grid build alone (bounding boxes, bucket keys, CUB radix sort, bucket bounds) over plan.any_grid clouds: *sorted
// receives the flat point indices ordered by bucket, *bstart / *bend the bucket ranges (inside grid_scratch).  Returns
// the launches.  launch_fpfh runs it first; icp.cu reuses it on the target clouds.
int launch_fpfh_grid(const FpfhPlan& plan, const float* pts, FpfhCloud* clouds, void* grid_scratch, cudaStream_t st,
                     const int** sorted, const int** bstart, const int** bend);
// pts (plan.N x 3), clouds (device copy of fpfh_plan's table), normals (N float4), spfh (N x 33), out (N x 33),
// overflow (B ints, zeroed here), grid_scratch (plan.grid_bytes): device pointers.  Returns the launches.  Normals only
// (tzr_estimate_normals): spfh and out nullptr, fpfh_radius unused; the grid build (when some cloud uses it) and the
// normals pass alone.  The normals do not depend on the plan's cell edge: the neighbour sets are the same at any cell
// edge of at least the normal radius, and they are sorted by (distance, index) before the covariance is summed.
int launch_fpfh(const FpfhPlan& plan, const float* pts, FpfhCloud* clouds, double normal_radius, double fpfh_radius,
                float4* normals, float* spfh, float* out, int* overflow, void* grid_scratch, cudaStream_t st);
// The descriptor kernels' device functions on their own, one item per thread (device pointers; one launch each).
// pair_features: p1, n1, p2, n2 are n x 3, f (n x 3) receives f1, f2, f3 and ok (n) 1 where pcl::computePairFeatures
// succeeds; f is zero where it does not.  smallest_eigenpair: cov is n x 9 (row-major 3 x 3), ev (n), vec (n x 3).
void launch_fpfh_pair_features(int n, const float* p1, const float* n1, const float* p2, const float* n2, float* f,
                               int32_t* ok, cudaStream_t st);
void launch_fpfh_smallest_eigenpair(int n, const float* cov, float* ev, float* vec, cudaStream_t st);
// Colour gradients (tzr_estimate_color_gradients, DESIGN.md §3.17) of every point of plan's clouds: pts (N x 3 floats),
// clouds (device copy of fpfh_plan's table for this radius), normals (N float4), colors (N x 3 floats), grad (N x 3
// doubles), grid_scratch (plan.grid_bytes): device pointers.  The 30 nearest neighbours by (d^2, index) of a bounded
// selection, so no neighbourhood is too large.  Returns the launches: 1, + 4 for the grid build when some cloud uses it.
int launch_color_gradients(const FpfhPlan& plan, const float* pts, FpfhCloud* clouds, double radius,
                           const float4* normals, const float* colors, double* grad, void* grid_scratch,
                           cudaStream_t st);

// certify.cu (DRSCertifier::certify, certification.cc:40-190)
// Device input of one certify_batch_device problem (tzr_certify_last_solve): its measurements are built on the device
// from a retained solve, exactly as the rotation stage built the TIMs it solved on (rot_trans.cu).
struct CertGatherProb {
  const double* src;     // the problem's points (rows of 3 doubles, device)
  const double* dst;
  const int32_t* clq;    // its sorted clique, m entries
  const uint8_t* rmask;  // its rotation inlier mask, N entries: theta = +1 where set, -1 elsewhere
  double scale;          // solution scale: dst TIMs are multiplied by 1 / scale
  double nbs;            // cbar2 * nb * nb with nb = noise_bound / scale (host arithmetic, in that order)
  int m;                 // clique size
  int complete;          // 1: COMPLETE TIM graph (N = m(m-1)/2), 0: CHAIN (N = m)
  int k_off, v_off;      // set by certify_batch_device: first measurement and first block row inside the group
};

// What certify_batch_device runs: the whole certifier, or one of its building blocks on X_in[b] / into X_out[b]
// (n x n each): the initial matrix (M_init into X_out, mu into mu_out), one nearest-PSD step or one dual projection.
enum class CertMode { kCertify, kSetup, kPsd, kDual };
// B problems (host pointers, validated by the caller) in device-sized groups of one launch sequence each; loop_eig: one
// cusolverDnDsyevd per active problem instead of cusolverDnXsyevBatched (debug flag 2097152).  src, dst, R_cm and
// results / traj (trajectories may be NULL) serve kCertify and kSetup; theta serves those and kDual.  gather (kCertify,
// may be NULL): B device inputs that replace src, dst, theta and the scalar noise bound; gathered[b] then receives 1, or
// 0 where the gathered measurements hold a non-finite value (the problem never reaches the eigensolver; result {0, 0,
// +inf}).  w_out (kPsd, may be NULL, as may its entries): the n ascending eigenvalues of each problem's symmetrised real
// block; they are defined only where the step takes cusolverDnDsyevd on that block, which a call with B = 1 always
// does.  cuSOLVER is loaded only in kCertify and kPsd; without it those return TZR_ERR_UNSUPPORTED.
int certify_batch_device(CertMode mode, const tzr_certifier_params& prm, int B, const int32_t* N, const double* R_cm,
                         const double* const* src, const double* const* dst, const double* const* theta,
                         const CertGatherProb* gather, int32_t* gathered,
                         tzr_certification_result* results, double* const* traj, const int32_t* traj_cap,
                         const double* const* X_in, double* const* X_out, double* const* w_out, double* mu_out,
                         bool loop_eig, void** scratch, size_t* scratch_cap, void** solver_handle, int64_t* launches,
                         cudaStream_t st, std::string* err);
void certify_release(void* solver_handle);

// matcher.cu (Matcher::calculateCorrespondences, matcher.cc:21-337), over B cloud pairs stored back to back
struct MatchPair {      // one per pair, device-resident
  int s_off, ns;        // first row and rows of the source cloud in the flat source arrays
  int d_off, nd;        // same for the target cloud; the pair's slots (ns + nd of them) start at s_off + d_off
  uint64_t seed;        // tuple-test seed
};
struct NnWork {         // one CTA of the nearest-neighbour kernel: a query tile against one database segment
  int dir;              // 0: query rows of feat_a, database rows of feat_b, result in best_a; 1: the reverse
  int q0, q_end;        // query rows [q0, min(q0 + 64, q_end))
  int db_lo;            // first row of the query's database cloud (reported indices are relative to it)
  int seg_lo, seg_hi;   // database rows of this segment
};
struct MatchPlan {
  int B = 0, NS = 0, ND = 0;   // pairs, source rows, target rows (slots: NS + ND)
  int bits_a = 0, bits_b = 0, bits = 0;  // sort key: pair << (bits_a + bits_b) | source << bits_b | target
  size_t cub_bytes = 0;
};
// Appends the NN work items of query rows [q_lo, q_lo + nq) against database rows [db_lo, db_lo + ndb); tiles_per_seg
// database tiles of 64 rows per item.
void nn_work_append(std::vector<NnWork>* work, int dir, int q_lo, int nq, int db_lo, int ndb, int tiles_per_seg);
// database tiles per NN work item that spread `tile_pairs` (query tile x database tile products) over the GPU
int nn_tiles_per_seg(long long tile_pairs, int num_sms);
int launch_feature_nn(const NnWork* work, int n_work, const float* feat_a, const float* feat_b, int dim,
                      unsigned long long* best_a, unsigned long long* best_b, long long n_best, cudaStream_t st);
// Host tables of a batch: pairs (B entries, seeds[b]), NN work list of both directions; TZR_ERR_TOO_LARGE when the
// sort key does not fit 64 bits.
int match_plan(int B, const int32_t* ns, const int32_t* nd, const uint64_t* seeds, int num_sms,
               std::vector<MatchPair>* pairs, std::vector<NnWork>* work, MatchPlan* plan);
size_t match_scratch_bytes(const MatchPlan& plan);
// All inputs device-resident (pairs/work: device copies of match_plan's tables); pts are normalised IN PLACE (pass
// copies).  out_pairs: (NS + ND) x 2 int32, pair b's rows from slot s_off + d_off; counts, gscale: B each.
// Returns the number of kernel launches.
int launch_match(const MatchPlan& plan, const MatchPair* pairs, const NnWork* work, int n_work, float* src_pts,
                 float* dst_pts, const float* src_feat, const float* dst_feat, int dim, int use_absolute_scale,
                 int use_crosscheck, int use_tuple_test, float tuple_scale, void* scratch, int32_t* out_pairs,
                 int* counts, float* gscale, int num_sms, cudaStream_t st);

// register_pairs.cu (tzr_register_cloud_pairs, DESIGN.md §3.10): the handoffs FPFH -> matcher -> ragged solve
struct PairGather {     // one per pair whose matcher rows go on, built on the host from the read-back counts
  int src_lo, dst_lo;   // first point of the pair's source / target cloud in the flat cloud array
  int slot, count;      // first row of the pair in the matcher's output (s_off + d_off), its correspondences
  long long corr_row;   // first row of its compacted index pairs, -1: not written
  long long solve_row;  // first row of its problem in the solve's flat float64 arrays, -1: not solved
};
// Copies every pair's rows of the clouds (pts: flat n x 3, feat: flat n x 33; cloud_lo[b] = first point of pair b's
// source, target cloud) into the matcher's flat source / target arrays of `plan`.  Returns the launches.
int launch_pair_rows(const MatchPlan& plan, const MatchPair* pairs, const int2* cloud_lo, const float* pts,
                     const float* feat, float* src_pts, float* dst_pts, float* src_feat, float* dst_feat, int num_sms,
                     cudaStream_t st);
// For the n_entries pairs of `table` (max_count: their largest count): the matcher's rows `pairs` -> corr (int2) and
// src / dst (float64 rows of pts).  Returns the launches.
int launch_corr_gather(const PairGather* table, int n_entries, int max_count, const int32_t* pairs, const float* pts,
                       int2* corr, double* src, double* dst, cudaStream_t st);

// icp.cu (point-to-point ICP, DESIGN.md §3.11, point-to-plane ICP, §3.13, generalized ICP, §3.14, and coloured ICP,
// §3.17): B problems
// over flat source and target point arrays
constexpr int kIcpChunk = 256;    // source points per chunk: the unit of the fixed-order reductions (one CTA each)
constexpr int kIcpGridMinN = 1024;  // targets from which the nearest-neighbour search goes through the hashed grid
constexpr int kIcpPointToPoint = 0, kIcpPointToPlane = 1, kIcpGeneralized = 2, kIcpColored = 3;  // IcpPlan::mode
// doubles per chunk of the point-to-plane and generalized systems: 21 of the upper triangle of A, 6 of g
constexpr int kIcpPlaneSums = 27;
// doubles per chunk of launch_icp's partial buffer (the point-to-point pass sums 9)
inline int icp_partial_stride(int mode) { return mode == kIcpPointToPoint ? 9 : kIcpPlaneSums; }
struct IcpProb {        // one per problem, device-resident; the host fills the inputs, the kernels the rest
  int s_lo, ns;         // sources: flat points [s_lo, s_lo + ns)
  int d_lo, nd;         // targets: flat points [d_lo, d_lo + nd) (also FpfhCloud tc of the target table)
  int c_lo;             // first chunk of the problem (chunks are consecutive)
  int active;           // 0: finished (converged or max_iteration reached); every kernel skips the problem
  int iterations, converged;
  int count;            // correspondences of the current transform
  int m_lo;             // first entry of the problem in the per-point match array
  int tc;               // its target's entry in the FpfhCloud table of the targets (lo = d_lo)
  int seeded;           // 1: the problem runs (tzr_register_cloud_pairs_icp: 0 for a pair without a valid solution)
  int n_lo;             // point-to-plane and generalized: the normal of target j is dst_normals[n_lo + j]
  int sn_lo;            // generalized: the normal of source i is src_normals[sn_lo + i]
  double s;             // fixed scale
  double R[9], t[3];    // current transform (column-major R)
  double fitness, rmse; // evaluation of the current transform
  double mup[3], muq[3];  // means of the current correspondences (source side transformed)
};
struct IcpPlan {
  int B = 0, NS = 0, ND = 0, chunks = 0;
  int max_iteration = 0;
  int mode = kIcpPointToPoint;
  double r2 = 0, relative_fitness = 0, relative_rmse = 0;
  double epsilon = 0;   // generalized: the covariances' epsilon (finite, > 0)
  // point-to-plane and generalized: the robust kernel (TZR_LOSS_*, DESIGN.md §3.15) and its k; TZR_LOSS_L2 runs the
  // unweighted system kernels
  int loss = 0;
  double loss_k = 0;
  FpfhPlan grid;        // the target grid (fpfh_plan with both radii = r)
  // coloured (DESIGN.md §3.17): lambda_geometric in [0, 1], and the targets' colour-gradient pass at radius grad_r =
  // 2 r with its own plan (fpfh_plan over the same targets, the descriptor stage's route); unused in the other modes
  double lambda_geometric = 0;
  double grad_r = 0;
  FpfhPlan ggrid;
};
constexpr int kIcpInfoSums = 21;  // doubles per chunk of launch_icp_information's partial buffer
// The tables of B problems against T target clouds of nt[0..T) points, back to back in the flat target array: problem
// b refines ns[b] sources from flat point s_lo[b] (s_lo nullptr: the sources back to back) onto target cloud tc[b]
// (tc nullptr: cloud b).  Fills plan's B, NS, ND, chunks, r2 and grid (route: the targets' search route), clouds (T,
// the targets' fpfh_plan table), probs (B; m_lo and c_lo running sums, the normals indexed like the points) and
// chunk_prob (chunks: the problem of every chunk).  init (may be nullptr): the problems' transforms, which makes them
// active and seeded; without it every problem waits for launch_icp_seed.  The other fields of plan are left as they
// are.  TZR_ERR_TOO_LARGE when the sources, the targets or the grid do not fit 32-bit indices.
int icp_plan(int B, const int32_t* ns, const int32_t* s_lo, const int32_t* tc, int T, const int32_t* nt, double r,
             int route, const tzr_similarity* init, IcpPlan* plan, std::vector<FpfhCloud>* clouds,
             std::vector<IcpProb>* probs, std::vector<int>* chunk_prob);
// Byte offsets of an ICP workspace from `base` on: [problems | target clouds | chunks | matches | partials | grid
// scratch | information | counts]; the last two are empty without `information`, whose partials have room for both
// launch_icp's sums and kIcpInfoSums.  In kIcpColored mode two more regions follow: the gradient pass's cloud table
// (plan.ggrid.B entries) and the targets' gradients (ND x 3 doubles), and the grid scratch has room for either grid
// (the gradient pass finishes before ICP builds its own).  end: the workspace's size.
struct IcpLayout {
  size_t probs, clouds, chunks, match, partial, grid, info, counts, end;
  size_t gclouds, grad;  // kIcpColored only (equal to end otherwise)
};
IcpLayout icp_layout(const IcpPlan& plan, size_t base, bool information);
// The device buffers of launch_icp and launch_icp_information.  src (NS x 3 floats), dst (ND x 3 floats), src_normals
// (generalized: the source normals, (nx, ny, nz, curvature) per point; may be nullptr otherwise), dst_normals
// (point-to-plane and generalized: the target normals, same layout; may be nullptr for point-to-point), probs (B),
// clouds (icp_plan's table of the targets), chunk_prob (chunks), match (target index or -1 per source point from m_lo,
// final correspondences), partial (chunks x icp_partial_stride(plan.mode) doubles, kIcpInfoSums for the information
// matrices), grid_scratch (plan.grid.grid_bytes), info (B x 36 doubles) and counts (B ints).
struct IcpBuffers {
  const float* src;
  const float* dst;
  const float4* src_normals;
  const float4* dst_normals;
  IcpProb* probs;
  FpfhCloud* clouds;
  const int* chunk_prob;
  int* match;
  double* partial;
  void* grid_scratch;
  double* info;
  int* counts;
  // kIcpColored: the source and target colours (NS x 3 and ND x 3 floats, set by the caller), the gradient pass's cloud
  // table and the targets' gradients (ND x 3 doubles, written by launch_icp); nullptr in the other modes
  const float* src_colors;
  const float* dst_colors;
  FpfhCloud* gclouds;
  double* grad;
};
// the table and scratch buffers of a workspace at d laid out by L; the points, normals and colours are left nullptr
IcpBuffers icp_buffers(char* d, const IcpLayout& L);
// Enqueues every iteration without synchronising; returns the launches: 4 for the grid build (when some target uses
// it) + 2 + 4 * max_iteration, in every mode; kIcpColored adds the gradient pass first (launch_color_gradients: 1, + 4
// when some target uses its grid).  info and counts are not used.
// grid_out (may be nullptr): the target grid's sorted indices and bucket ranges inside grid_scratch (all nullptr without
// grid targets), for launch_icp_information to reuse.
struct IcpGrid {
  const int* sorted;
  const int* bstart;
  const int* bend;
};
int launch_icp(const IcpPlan& plan, const IcpBuffers& buf, cudaStream_t st, IcpGrid* grid_out = nullptr);
// The seeds of B problems from B solution records (tzr_register_cloud_pairs_icp): a valid record with a finite transform
// and a positive scale sets (s, R, t) and active = seeded = 1, any other leaves the problem inactive.  One launch.
int launch_icp_seed(IcpProb* probs, int B, const tzr_solution* sol, cudaStream_t st);
// Information matrices (tzr_information_matrix_batch, DESIGN.md §3.16) of B problems at their current transforms: the
// grid build (when some target uses it), icp_nn_kernel as launch_icp runs it, then the 21 sums of G^T G per chunk into
// partial and their fixed-order combination into info and counts.  The normals are not used.  reseed: set active =
// seeded first (a chained call, after launch_icp finished its problems); otherwise the problems must be active.  A
// problem that is not seeded gets zeros.  grid (may be nullptr): launch_icp's grid of the same targets, reused instead
// of built again.  Returns the launches: 3, + 1 with reseed, + 4 for the grid build when some target uses the grid and
// grid is nullptr.
int launch_icp_information(const IcpPlan& plan, const IcpBuffers& buf, bool reseed, cudaStream_t st,
                           const IcpGrid* grid = nullptr);
// The multi-scale schedule (tzr_icp_multiscale_batch, DESIGN.md §3.19), around launch_icp at every scale.  Load: problem
// b of B takes the pose of pair pair_of[b] (P poses, device) and becomes active and seeded.  Store: for each of the P
// pairs, prob_of[p] >= 0 writes that problem's result to rec[p * stride] and its transform to pose[p]; -1 writes the
// pose with every other field 0 (probs may then be nullptr when no pair is refined).  One launch each.
int launch_icp_pose_load(IcpProb* probs, int B, const int* pair_of, const tzr_similarity* pose, cudaStream_t st);
int launch_icp_pose_store(const IcpProb* probs, int P, const int* prob_of, tzr_similarity* pose, tzr_icp_result* rec,
                          int stride, cudaStream_t st);

// pose_graph.cu (tzr_pose_graph_optimize, DESIGN.md §3.16): one graph of K nodes and E edges, device-resident
struct PgEdge {         // one per edge; the host fills it, the kernels read it
  int s, d;             // source and target node
  int fs, fd;           // their free-node index (-1: the reference node)
  int uncertain;        // 1: the edge takes part in GNC-TLS
  int pad;
  double R[9], t[3];    // T_sd (column-major R)
  double L[36];         // Lambda_e (row-major)
  double inv_norm;      // 1 / (c^2 Lambda_e(5,5)), 0 when Lambda_e(5,5) = 0
};
struct PgState {        // the solve's device-side state, read back once per GNC iteration
  double lambda;        // Levenberg-Marquardt damping
  double cost;          // sum w_e e^T Lambda_e e at the current poses
  double cand_cost;     // the same at the candidate poses
  double mu, gnc_cost;  // GNC-TLS: the control parameter and the previous weighted residual sum
  int cur;              // which of the two pose / edge-term buffers holds the current poses
  int done;             // 1: the inner solve has stopped
  int inner;            // inner iterations of this GNC iteration
  int stop;             // 1: GNC-TLS has stopped
  int info[2];          // potrf / potrs status of the latest step
};
struct PgPlan {
  int K = 0, E = 0, n = 0;        // nodes, edges, rows of the normal equations (6 (K - 1))
  int blocks = 0;                 // 6 x 6 blocks of H's lower triangle with some contribution
  int max_inner = 0;              // inner iterations enqueued per GNC iteration
  double gnc_factor = 1.4, cost_threshold = 1e-6;
};
struct PgBlock {        // one 6 x 6 block (bi >= bj) of H's lower triangle, or the gradient block bi (bj = -1)
  int bi, bj;
  int lo, hi;           // its contributions [lo, hi) in the plan's term list, ascending edge index
};
struct PgTerm {         // one contribution: edge e with sign +1 / -1
  int e, sign;
};
// The buffers of launch_pose_graph_*: device pointers.  poses: 2 buffers of K x 12 doubles (R column-major, t); eterm:
// 2 buffers of E x kPgTermStride doubles; weight: E; H: n x n column-major; g: n; state: one PgState.
struct PgDev {
  const PgEdge* edges;
  const PgBlock* blocks;
  const PgTerm* terms;
  double* poses;
  double* eterm;
  double* weight;
  double* H;
  double* g;
  PgState* state;
};
constexpr int kPgTermStride = 44;  // doubles per edge in eterm: A^T Lambda A (36), A^T Lambda e (6), e^T Lambda e, r-bar
// Evaluates every edge at the current poses and starts the inner solve (its cost, damping and flags).  Returns the
// launches (2).
int launch_pose_graph_begin(const PgPlan& plan, const PgDev& dv, double cost_floor, cudaStream_t st);
// The damped H (lower triangle, every listed block; the caller clears H first) and the right-hand side -g of one inner
// iteration.  Returns the launches (1).
int launch_pose_graph_assemble(const PgPlan& plan, const PgDev& dv, cudaStream_t st);
// The candidate poses from the solved step, their edge terms and the accept / reject decision.  Returns the launches (3).
int launch_pose_graph_step(const PgPlan& plan, const PgDev& dv, int ref, double cost_floor, cudaStream_t st);
// GNC-TLS weight update after GNC iteration `iter`.  Returns the launches (1).
int launch_pose_graph_gnc(const PgPlan& plan, const PgDev& dv, int iter, cudaStream_t st);
// dense Cholesky through the lazily loaded cuSOLVER (certify.cu): handle and workspace size of an n x n lower factor;
// TZR_ERR_UNSUPPORTED when cuSOLVER cannot be loaded
int dense_cholesky_setup(void** solver_handle, int n, double* A, int* lwork, cudaStream_t st, std::string* err);
// potrf of A (lower, in place) and potrs of b (in place); info[0] / info[1] (device) their status
int dense_cholesky_solve(void* solver_handle, int n, double* A, double* b, double* work, int lwork, int* info,
                         std::string* err);

// voxel.cu (voxel-grid downsampling, DESIGN.md §3.12): B clouds stored back to back
constexpr unsigned long long kVoxNone = 1ull << 62;  // sort key of a point in no voxel: above every voxel key (< 2^62)
constexpr int kVoxKeyBits = 63;                      // key bits the sort looks at
struct VoxCloud {       // one per cloud; the host fills lo, n and the bound sentinels, the kernels the rest
  int lo, n;            // first point of the cloud in the flat array, point count
  int mn[3], mx[3];     // bounds of the finite points (ordered-int floats; INT_MAX / INT_MIN: none yet)
  double vmin[3];       // min - v * 0.5
  long long cy, cz;     // voxels along y and z (the key's strides)
  int status;           // TZR_OK, or TZR_ERR_TOO_LARGE (Open3D's INT_MAX check or the 2^62-cell limit)
  int valid;            // 1: the cloud has a finite point and its grid fits; its finite points get voxel keys
  int out_lo, n_out;    // its first output row in the batch, its voxels
};
struct VoxPlan {
  int B = 0, N = 0;
  size_t scratch_bytes = 0;
};
// Fills clouds[0..B) (host copy, staged to the device before launch_voxel) and the plan; TZR_ERR_TOO_LARGE when the
// batch's points do not fit 32-bit indices.
int voxel_plan(int B, const int32_t* n, VoxCloud* clouds, VoxPlan* plan);
// pts (N x 3 floats), clouds (device copy of voxel_plan's table), scratch (plan.scratch_bytes), out (N x 3 floats: the
// voxels of the batch in cloud order, cloud b's from row out_lo), voxel_of (N ints: the cloud-local output row of every
// point, -1 for a point in no voxel): device pointers.  colors (may be nullptr; N x 3 floats) and colors_out (as out):
// each voxel's colour mean, summed like its point.  Returns the launches (10).
int launch_voxel(const VoxPlan& plan, double voxel_size, const float* pts, VoxCloud* clouds, void* scratch, float* out,
                 int* voxel_of, cudaStream_t st, const float* colors = nullptr, float* colors_out = nullptr);


}  // namespace tzr
