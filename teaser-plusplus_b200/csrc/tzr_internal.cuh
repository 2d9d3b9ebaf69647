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
constexpr int kCoreRounds = 48;     // peel rounds (one launch each) of the large route's core; a set still shrinking
                                    // after them is a superset of the core, which the compacted search peels again

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
  float g_mhi, g_chi, g_mlo, g_clo;
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
  float* opnd;    // B * ceil(n/128) * 2 roles * 2 clouds * 6 planes * 128 rows * 4: tf32-split MMA operand tiles of the
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
};

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

// kernels (defined in the .cu files) -------------------------------------------------------------
void launch_prep(const Batch& bt, cudaStream_t st);
int launch_graph(const Batch& bt, cudaStream_t st, int num_sms);  // returns the number of kernels launched
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
int launch_scale_estimation(const Batch& bt, uint32_t flags, void* scratch, cudaStream_t st);
void launch_rot_trans(const Batch& bt, const tzr_params& p, int use_clique, cudaStream_t st);
// Large route (n > kMaxN or debug flag 524288; DESIGN.md §3.2).  lists: B * kHeurRoots * 2n u16 of heuristic scratch;
// chg: B * kCoreRounds per-round change counters; new2old / old2new: B * n; core_cnt / route: B.  route[b] (device copy,
// set by the host after reading core_cnt): > 0 search the compacted core, 0 not searched (result already final),
// -1 core above the cap (heuristic clique, not proven).
void launch_clique_large_front(const Batch& bt, const tzr_params& p, int mode, uint16_t* lists, cudaStream_t st,
                               int* n_launches);
void launch_core(const Batch& bt, int32_t* chg, int32_t* new2old, int32_t* old2new, int32_t* core_cnt, int num_sms,
                 cudaStream_t st, int* n_launches);
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
struct FpfhPlan {
  int B = 0, N = 0;            // clouds, points in all of them
  bool any_grid = false;
  unsigned int buckets = 0;    // sum of T_b over the grid clouds (also the sentinel key of unsorted points)
  size_t grid_bytes = 0;       // device scratch of the grid path (0 without grid clouds)
};
// Radius-search route of every cloud: by size (the grid from kGridMinN points on), or forced by the debug flags
// 4194304 (brute force) and 8388608 (the grid at any size).
constexpr int kFpfhRouteAuto = 0, kFpfhRouteBrute = 1, kFpfhRouteGrid = 2;
// Fills clouds[0..B) (host copy, to be staged to the device before launch_fpfh) and the plan.  TZR_ERR_TOO_LARGE when
// the points or buckets of the batch do not fit 32-bit indices.
int fpfh_plan(int B, const int32_t* n, double normal_radius, double fpfh_radius, int route, FpfhCloud* clouds,
              FpfhPlan* plan);
// pts (plan.N x 3), clouds (device copy of fpfh_plan's table), normals (N float4), spfh (N x 33), out (N x 33),
// overflow (B ints, zeroed here), grid_scratch (plan.grid_bytes): device pointers.  Returns the launches.
int launch_fpfh(const FpfhPlan& plan, const float* pts, FpfhCloud* clouds, double normal_radius, double fpfh_radius,
                float4* normals, float* spfh, float* out, int* overflow, void* grid_scratch, cudaStream_t st);
// The descriptor kernels' device functions on their own, one item per thread (device pointers; one launch each).
// pair_features: p1, n1, p2, n2 are n x 3, f (n x 3) receives f1, f2, f3 and ok (n) 1 where pcl::computePairFeatures
// succeeds; f is zero where it does not.  smallest_eigenpair: cov is n x 9 (row-major 3 x 3), ev (n), vec (n x 3).
void launch_fpfh_pair_features(int n, const float* p1, const float* n1, const float* p2, const float* n2, float* f,
                               int32_t* ok, cudaStream_t st);
void launch_fpfh_smallest_eigenpair(int n, const float* cov, float* ev, float* vec, cudaStream_t st);

// certify.cu (DRSCertifier::certify, certification.cc:40-190); mode 0 certify, 1 initial matrix, 2 dual projection,
// 3 nearest-PSD step (W_in -> Wd_out, eigenvalues in w_out)
int certify_device(int mode, double noise_bound, double cbar2, double sub_optimality, double max_iterations,
                   double gamma_tau, const double* R_cm, const double* src, const double* dst, const double* theta,
                   int N, int* is_optimal, double* best_subopt, int* n_iters, double* traj, int traj_cap,
                   double* M_init_out, double* mu_out, const double* W_in, double* Wd_out, double* w_out,
                   void** scratch, size_t* scratch_cap, void** solver_handle, int64_t* launches, cudaStream_t st,
                   std::string* err);
// B problems (host pointers, validated by the caller) in device-sized groups of one launch sequence each; loop_eig: one
// cusolverDnDsyevd per active problem instead of cusolverDnXsyevBatched (debug flag 2097152).  mode 0 certify; the
// building blocks run one step of the batch's iteration on X_in[b] (n x n) into X_out[b]: 1 nearest-PSD step, 2 dual
// projection (theta as for mode 0; src, dst, R_cm, results and traj unused)
int certify_batch_device(int mode, const tzr_certifier_params& prm, int B, const int32_t* N, const double* R_cm,
                         const double* const* src, const double* const* dst, const double* const* theta,
                         tzr_certification_result* results, double* const* traj, const int32_t* traj_cap,
                         const double* const* X_in, double* const* X_out, bool loop_eig, void** scratch,
                         size_t* scratch_cap, void** solver_handle, int64_t* launches, cudaStream_t st,
                         std::string* err);
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


}  // namespace tzr
