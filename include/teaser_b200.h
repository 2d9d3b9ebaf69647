/*
 * teaser_b200.h — C-ABI of the GPU-native TEASER++ registration hot path.
 *
 * This is the drop-in boundary: plain C, caller-owned buffers, no STL / Eigen / torch types.
 * The reference has no FFI layer of its own (SURVEY.md §8b); each entry point below names the
 * reference function(s) it replaces (paths relative to the reference tree).  The C++ facade
 * `teaser::RobustRegistrationSolver` (teaser-plusplus_b200/host/include/teaser/registration.h) and the
 * Python module `teaserpp_python` call exactly these symbols; INTEGRATION.md shows the binding a
 * TEASER++ maintainer would add.
 *
 * Conventions
 *   - Points are 3xN column-major double == N contiguous (x,y,z) triples, i.e. the memory of an
 *     Eigen::Matrix<double,3,Dynamic> (teaser/src/registration.cc:568-570).
 *   - 3x3 rotations are column-major (Eigen::Matrix3d).
 *   - The inlier graph is a packed, symmetric adjacency bitset: n rows of `tzr_words_per_row(n)`
 *     little-endian uint64 words; bit j of row i is set iff TIM (i,j) passed the scale test
 *     (replaces teaser::Graph's vector<vector<int>>, teaser/include/teaser/graph.h:29-207).
 *   - Every function returns 0 on success or a negative tzr_status; no exceptions cross the ABI.
 *   - "_dev" variants take DEVICE pointers and enqueue on the context's stream without
 *     synchronising (tzr_ctx_synchronize does); the plain variants take HOST pointers and are
 *     synchronous, host<->device copies included.
 *   - A context owns one CUDA device, one stream and a growable workspace; it is not thread-safe,
 *     distinct contexts are independent.  There is NO CPU fallback: without a usable CUDA device
 *     tzr_ctx_create fails with TZR_ERR_NO_DEVICE.
 */
#ifndef TEASER_B200_H_
#define TEASER_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TZR_ABI_VERSION 2

typedef enum tzr_status {
  TZR_OK = 0,
  TZR_ERR_INVALID_ARG = -1,
  TZR_ERR_NO_DEVICE = -2,
  TZR_ERR_CUDA = -3,
  TZR_ERR_ALLOC = -4,
  TZR_ERR_UNSUPPORTED = -5,
  TZR_ERR_TOO_LARGE = -6
} tzr_status;

/* teaser::RobustRegistrationSolver::Params (teaser/include/teaser/registration.h:419-514).
 * Enum values are the reference's (registration.h:382-412). */
typedef struct tzr_params {
  double noise_bound;                    /* default 0.01 */
  double cbar2;                          /* default 1 */
  int32_t estimate_scaling;              /* default 1 (true) */
  int32_t rotation_estimation_algorithm; /* 0 GNC_TLS (default), 1 FGR, 2 QUATRO */
  double rotation_gnc_factor;            /* default 1.4 */
  uint64_t rotation_max_iterations;      /* default 100 */
  double rotation_cost_threshold;        /* default 1e-6 */
  int32_t rotation_tim_graph;            /* 0 CHAIN (default), 1 COMPLETE */
  int32_t inlier_selection_mode;         /* 0 PMC_EXACT (default), 1 PMC_HEU, 2 KCORE_HEU, 3 NONE */
  double kcore_heuristic_threshold;      /* default 0.5 */
  int32_t use_max_clique;                /* deprecated, default 1 */
  int32_t max_clique_exact_solution;     /* deprecated, default 1 */
  double max_clique_time_limit;          /* seconds, default 3600 */
  int32_t max_clique_num_threads;        /* ignored on the GPU */
  int32_t reserved;
} tzr_params;

/* teaser::RegistrationSolution (registration.h:32-39) plus diagnostics the getters expose. */
typedef struct tzr_solution {
  int32_t valid;                  /* solution_.valid (registration.cc:643-647,734) */
  int32_t clique_size;            /* getInlierMaxClique().size() */
  double scale;
  double translation[3];
  double rotation[9];             /* column-major */
  int32_t clique_proven_optimal;  /* 1: maximum clique proven by complete enumeration (canonical = lexicographically
                                   * smallest among ties); 2: maximum SIZE proven through the vertex-cover LP bound /
                                   * Nemhauser-Trotter reduction after the first 50 ms search pass (dense graphs; a
                                   * maximum clique, not necessarily the canonical one); 0: heuristic mode or budget hit */
  int32_t gnc_iterations;         /* loop bodies entered by the GNC rotation solver */
  double gnc_cost;                /* getGNCRotationCostAtTermination() */
  int32_t n_rotation_inliers;
  int32_t n_translation_inliers;
  int64_t n_edges;                /* edges of the inlier graph */
  double stage_ms[8];             /* filled by tzr_solve only: 0 h2d, 1 graph, 2 clique, 3 rot+trans, 4 d2h, 6 total */
} tzr_solution;

typedef struct tzr_ctx tzr_ctx;

/* ---- context ------------------------------------------------------------------------------- */
int tzr_abi_version(void);
const char* tzr_status_string(int status);
/* Last CUDA error text seen by this context (empty string if none). */
const char* tzr_last_error(const tzr_ctx* ctx);
/* Fill `p` with the reference's Params defaults (registration.h:419-514). */
void tzr_params_default(tzr_params* p);
/* device < 0: current device.  Fails (TZR_ERR_NO_DEVICE) when no CUDA device is usable. */
int tzr_ctx_create(int device, tzr_ctx** out);
int tzr_ctx_destroy(tzr_ctx* ctx);
/* Use an existing CUDA stream (cudaStream_t as void*) instead of the context's own. */
int tzr_ctx_set_stream(tzr_ctx* ctx, void* cuda_stream);
int tzr_ctx_synchronize(tzr_ctx* ctx);
/* Number of kernels this context has launched so far (bench.py's gpu_launches). */
int64_t tzr_ctx_kernel_launches(const tzr_ctx* ctx);
/* 64-bit words per adjacency row: ceil(n/64). */
int tzr_words_per_row(int n);

/* ---- stage 1: TIMs + scale consistency + inlier graph ---------------------------------------
 * Replaces computeTIMs (registration.cc:512-551) x2, ScaleInliersSelector::solveForScale
 * (registration.cc:427-443) and the Graph::addEdge loop (registration.cc:614-619) — fused, the
 * N(N-1)/2 TIMs are never materialised.  beta = 2*noise_bound*sqrt(cbar2).
 * adj_bits: n * tzr_words_per_row(n) uint64 (fully overwritten); degree: n int32 (may be NULL). */
int tzr_graph_build(tzr_ctx* ctx, const double* src_3xN, const double* dst_3xN, int n, double beta,
                    uint64_t* adj_bits, int32_t* degree, int64_t* n_edges);

/* ---- stage 2: maximum clique ----------------------------------------------------------------
 * Replaces teaser::MaxCliqueSolver::findMaxClique (teaser/src/graph.cc:12-125) including the PMC
 * library calls it makes.  mode: 0 PMC_EXACT, 1 PMC_HEU, 2 KCORE_HEU.  clique: capacity n, returned
 * sorted ascending (solve() sorts it, registration.cc:636).  *proven_optimal: 1 / 2 / 0 with the meaning of
 * tzr_solution.clique_proven_optimal.  Input contract: the bitset must be symmetric; diagonal bits and bits at or beyond
 * n in a row's last word are ignored (cleared on the device after the copy).  Entries of clique past *clique_size are
 * set to -1.  This is tzr_max_clique_batch with B = 1. */
int tzr_max_clique(tzr_ctx* ctx, const uint64_t* adj_bits, int n, int mode, double kcore_heuristic_threshold,
                   double time_limit_s, int32_t* clique, int32_t* clique_size, int32_t* proven_optimal);
/* B independent problems of n vertices searched in one launch sequence.  adj_bits: B * n * tzr_words_per_row(n)
 * uint64 (problem-major, same input contract as above).  cliques: B * n int32, row b sorted ascending, -1 past
 * clique_sizes[b].  proven_optimal (B int32, may be NULL): as tzr_max_clique.  search_flags (B int32, may be NULL): the
 * per-problem flags word the search ends with: 1 = result not proven (depth cap or budget hit), 2 = first-pass deadline
 * (set while a problem is still open after the first pass; cleared when the second pass resumes it), 4 = closed by the
 * vertex-cover LP bound, 8 = Nemhauser-Trotter reduction then a second pass that only accepts larger cliques; bits 8 and
 * up hold the LP bound when 8 is set.  A result with proven_optimal 1 is the one tzr_max_clique gives for that problem
 * alone. */
int tzr_max_clique_batch(tzr_ctx* ctx, int B, int n, const uint64_t* adj_bits, int mode,
                         double kcore_heuristic_threshold, double time_limit_s, int32_t* cliques, int32_t* clique_sizes,
                         int32_t* proven_optimal, int32_t* search_flags);
/* Diagnostics of the most recent tzr_max_clique(_batch) call on this context (TZR_ERR_INVALID_ARG once another call has
 * reused the workspace).  geometry3: CTAs of the persistent exact-search grid, problems searched at a time (start groups
 * of the sweep, sized so that their bitsets fit the L2), stack depth.  heuristic_best (B int32, may be NULL): per
 * problem, the largest clique of the root-based greedy heuristic, before the peel kernel's second chance. */
int tzr_ctx_clique_info(tzr_ctx* ctx, int32_t* geometry3, int32_t* heuristic_best);

/* Per-problem size limit of this context: 32768 <= max_n <= 65536 (TZR_ERR_INVALID_ARG otherwise); the default is
 * 32768.  It applies to tzr_graph_build, tzr_max_clique(_batch), tzr_solve, tzr_solve_batch, tzr_solve_batch_dev and
 * tzr_last_graph; a larger problem is TZR_ERR_TOO_LARGE.  65536 is a hard bound: the graph kernels and the clique
 * heuristic keep vertex indices in 16 bits.  tzr_solve_batch_multi keeps 32768 (its contexts are library-internal).
 * Problems of more than 32768 vertices take the large clique route (DESIGN.md 3.2): the heuristic clique (size L) on
 * the full graph, the (L-1)-core of the graph on the device, and the small route's exact search on that core compacted
 * to at most 32768 vertices (the relabelling keeps the index order, so the canonical tie-break is unchanged).  A graph
 * whose core keeps more than 32768 vertices (a dense graph, e.g. most vertices in one large inlier set) is not
 * searched: it returns its heuristic clique, a valid clique with clique_proven_optimal = 0.  estimate_scaling = 1 needs
 * the unknown-scale stage's scratch (tens of GB at these sizes) and is TZR_ERR_TOO_LARGE from n = 46341 (2K end points
 * exceed 2^31).  A buffer that does not fit the device is TZR_ERR_ALLOC (tzr_last_error names the size). */
int tzr_ctx_set_max_n(tzr_ctx* ctx, int max_n);
/* Clique route of each problem of the most recent clique stage on this context (a solve or a max-clique call; B
 * entries; TZR_ERR_INVALID_ARG once another call has reused the workspace): 0 = small route; k > 0 = large route with
 * the core compacted to k vertices, where k equal to the clique size means the core was the clique itself (or a
 * heuristic mode, or a clique of size <= 1) and no search ran; -1 = large route whose core kept more vertices than the
 * cap, the heuristic clique is returned with clique_proven_optimal = 0 (search flags 1 | 16).  k and the cap test
 * always refer to the (L-1)-core itself, never to a superset of it: a graph that peels slowly (long pendant paths)
 * is peeled on until its core is reached. */
int tzr_ctx_clique_route(tzr_ctx* ctx, int32_t* per_problem);

/* ---- stage 3: GNC-TLS rotation --------------------------------------------------------------
 * Replaces GNCTLSRotationSolver::solveForRotation (registration.cc:764-866) + utils::svdRot
 * (teaser/include/teaser/utils.h:121-136).  inlier_mask (m bytes) and the scalar outputs may be NULL. */
int tzr_gnc_tls_rotation(tzr_ctx* ctx, const double* src_3xM, const double* dst_3xM, int m, double noise_bound,
                         double gnc_factor, uint64_t max_iterations, double cost_threshold, double* R_colmajor9,
                         uint8_t* inlier_mask, double* cost_at_termination, int32_t* iterations);

/* Same stage for any of the reference's rotation back-ends on caller-supplied TIMs: algorithm 0 GNC_TLS
 * (registration.cc:764-866), 1 FGR (FastGlobalRegistrationSolver::solveForRotation, registration.cc:206-278),
 * 2 QUATRO (QuatroSolver::solveForRotation, registration.cc:280-408; yaw only).
 * With max_iterations = 0 no iteration runs: R is the identity, the cost +inf, iterations 0 and every mask entry 1
 * (the reference leaves its rotation untouched there).  A GNC-TLS or Quatro run whose first residuals all lie below
 * noise_bound^2 / 2 stops at mu <= 0 after one iteration with the cost still +inf. */
int tzr_rotation_solve(tzr_ctx* ctx, int algorithm, const double* src_3xM, const double* dst_3xM, int m,
                       double noise_bound, double gnc_factor, uint64_t max_iterations, double cost_threshold,
                       double* R_colmajor9, uint8_t* inlier_mask, double* cost_at_termination, int32_t* iterations);

/* ---- stage 4: TLS translation ---------------------------------------------------------------
 * Replaces TLSTranslationSolver::solveForTranslation (registration.cc:445-471): per-axis
 * ScalarTLSEstimator::estimate on dst - src with range noise_bound*sqrt(cbar2). */
int tzr_tls_translation(tzr_ctx* ctx, const double* src_3xM, const double* dst_3xM, int m, double noise_bound,
                        double cbar2, double* t3, uint8_t* inlier_mask);

/* ScalarTLSEstimator::estimate (registration.cc:21-88), standalone.  Ties among end points are ordered by (value,
 * payload); a measurement whose x or range is not finite is excluded (no end points, inlier flag 0); with no kept
 * measurement the estimate is NaN (DESIGN.md 3.3). */
int tzr_scalar_tls(tzr_ctx* ctx, const double* x, const double* ranges, int64_t m, double* estimate,
                   uint8_t* inliers);

/* ---- upstream of solve(): correspondence generation ------------------------------------------
 * Replaces Matcher::calculateCorrespondences (teaser/src/matcher.cc:21-53 -> normalizePoints :55-113 and
 * advancedMatching :114-297).  Host pointers.  src_pts/dst_pts: ns x 3 / nd x 3 float xyz (PointXYZ AoS,
 * geometry.h:15-24); src_feat/dst_feat: row-major ns x dim / nd x dim float descriptors (FPFH: dim = 33,
 * pcl::FPFHSignature33::histogram), 1 <= dim <= 128.  The nearest-neighbour search is exact under
 * flann::L2<float> (what KDTreeSingleIndex with eps = 0 returns), lowest index among equal distances.
 * use_tuple_test + tuple_scale != 0 runs 100 * ncorr trials (:236); the reference seeds rand() with time(NULL),
 * here the draws are splitmix64(tuple_seed + 3 t + k) >> 33 so a seed reproduces a run.
 * pairs: capacity x 2 int32 rows (source index, target index), sorted and unique like the reference's output;
 * capacity >= ns + nd is always enough.  global_scale (optional) receives Matcher::global_scale_. */
int tzr_match_correspondences(tzr_ctx* ctx, const float* src_pts, int ns, const float* dst_pts, int nd,
                              const float* src_feat, const float* dst_feat, int dim, int use_absolute_scale,
                              int use_crosscheck, int use_tuple_test, float tuple_scale, uint64_t tuple_seed,
                              int32_t* pairs, int64_t capacity, int64_t* n_pairs, float* global_scale);

/* Descriptor estimation: replaces FPFHEstimation::computeFPFHFeatures (teaser/src/fpfh.cc:15-43), i.e. PCL's
 * NormalEstimationOMP (radius normal_search_radius, viewpoint at the origin) followed by FPFHEstimationOMP (radius
 * fpfh_search_radius) on the same cloud.  Host pointers.  pts: n x 3 float xyz.  fpfh_out: n x 33 floats
 * (pcl::FPFHSignature33::histogram rows).  normals_out (optional): n x 4 floats (normal_x, normal_y, normal_z,
 * curvature — FPFHEstimation::getNormals(), fpfh.h:55); NaN where a point has fewer than 3 neighbours.
 * TZR_ERR_TOO_LARGE when some point has more than 4096 neighbours inside a radius (downsample the cloud). */
int tzr_compute_fpfh(tzr_ctx* ctx, const float* pts, int n, double normal_search_radius, double fpfh_search_radius,
                     float* fpfh_out, float* normals_out);

/* ---- the front end over many clouds in one call ----------------------------------------------
 * Host pointers, ragged sizes, synchronous like tzr_solve_batch; the number of kernel launches does not depend on B.
 *
 * Descriptors of B clouds: cloud b has n[b] >= 1 points at pts[b] (n[b] x 3 float).  fpfh_out[b]: n[b] x 33 floats.
 * normals_out (may be NULL, or hold NULL entries): n[b] x 4 floats.  status (B int32, may be NULL): per cloud TZR_OK or
 * TZR_ERR_TOO_LARGE (a point with more than 4096 neighbours).  Returns TZR_ERR_TOO_LARGE if any cloud overflowed; every
 * other cloud's outputs are still written.  TZR_ERR_TOO_LARGE also when the batch holds more than 2^31 - 1 points.
 * Per cloud, the outputs are bit-identical to tzr_compute_fpfh on that cloud alone. */
int tzr_compute_fpfh_batch(tzr_ctx* ctx, int B, const int32_t* n, const float* const* pts,
                           double normal_search_radius, double fpfh_search_radius, float* const* fpfh_out,
                           float* const* normals_out, int32_t* status);

/* Normals alone: the first pass of tzr_compute_fpfh (PCL's NormalEstimationOMP, radius normal_search_radius, viewpoint
 * at the origin) without the descriptor passes, e.g. the target normals of point-to-plane ICP.  normals_out: n x 4
 * floats (normal_x, normal_y, normal_z, curvature), bit-identical to tzr_compute_fpfh's normals_out at the same normal
 * radius, whatever its fpfh_search_radius: a point's neighbours are the points with float d^2 < r^2, sorted by
 * (d^2, index) before the covariance is summed, so neither the grid's cell edge nor the search route changes them.
 * NaN where a point has fewer than 3 neighbours.  The search route is tzr_compute_fpfh's (brute force below 4096
 * points, the hashed grid from there; debug flags 4194304 and 8388608).  Arguments, status, TZR_ERR_TOO_LARGE (a point
 * with more than 4096 neighbours; the other clouds are still written) and workspace as tzr_compute_fpfh(_batch): the
 * calls share the front end's buffers, so a retained tzr_solve / tzr_solve_batch stays retained across them.
 * Batch: normals_out[b] (every entry required): n[b] x 4 floats; status (may be NULL): B entries.  Per cloud, the
 * output is bit-identical to tzr_estimate_normals on that cloud alone. */
int tzr_estimate_normals(tzr_ctx* ctx, const float* pts, int n, double normal_search_radius, float* normals_out);
int tzr_estimate_normals_batch(tzr_ctx* ctx, int B, const int32_t* n, const float* const* pts,
                               double normal_search_radius, float* const* normals_out, int32_t* status);

/* Building blocks of tzr_compute_fpfh, exposed so that each can be checked on any input, not only on the ones a cloud
 * produces.  Host pointers, synchronous; each runs the production device function, one item per thread.
 * tzr_fpfh_pair_features: pcl::computePairFeatures (features/src/pfh_tools.cpp) on n point pairs: p1, n1, p2, n2 are
 *   n x 3 floats (points and normals); f_out (n x 3) receives (f1, f2, f3), ok_out (n int32) 1 where the features are
 *   defined and 0 where they are not (coincident points, or a zero cross product); f_out is zero there.
 * tzr_fpfh_smallest_eigenpair: pcl::eigen33's smallest eigenpair (common/impl/eigen.hpp) of n symmetric 3 x 3 float
 *   matrices: cov is n x 9 (row-major); ev_out (n) and vec_out (n x 3, unit length). */
int tzr_fpfh_pair_features(tzr_ctx* ctx, int n, const float* p1, const float* n1, const float* p2, const float* n2,
                           float* f_out, int32_t* ok_out);
int tzr_fpfh_smallest_eigenpair(tzr_ctx* ctx, int n, const float* cov, float* ev_out, float* vec_out);

/* Correspondences of B cloud pairs: pair b has ns[b] source points (src_pts[b], src_feat[b]) and nd[b] target points
 * (dst_pts[b], dst_feat[b]); dim and the flags apply to every pair; tuple_seeds: B seeds.  pairs[b]: capacity[b] x 2
 * int32 rows.  n_pairs[b] (B entries) is always set.  If some pair needs more than capacity[b] rows the call returns
 * TZR_ERR_INVALID_ARG, and the pairs that fit are still written.  global_scale (B floats, may be NULL).
 * TZR_ERR_TOO_LARGE when the batch holds more than 2^31 - 1 points.  Per pair, the outputs are bit-identical to
 * tzr_match_correspondences with the same arguments and seed. */
int tzr_match_correspondences_batch(tzr_ctx* ctx, int B, const int32_t* ns, const float* const* src_pts,
                                    const int32_t* nd, const float* const* dst_pts, const float* const* src_feat,
                                    const float* const* dst_feat, int dim, int use_absolute_scale, int use_crosscheck,
                                    int use_tuple_test, float tuple_scale, const uint64_t* tuple_seeds,
                                    int32_t* const* pairs, const int64_t* capacity, int64_t* n_pairs,
                                    float* global_scale);

/* The matcher's search primitive on its own (Matcher::searchKDTree with nn = 1, matcher.cc:314-335, for every
 * query row): nn_index[q] = argmin_i L2(query[q], db[i]), nn_dist[q] (optional) the squared distance. */
int tzr_feature_nn(tzr_ctx* ctx, const float* query, int nq, const float* db, int ndb, int dim, int32_t* nn_index,
                   float* nn_dist);

/* ---- downstream of solve(): certification ------------------------------------------------------
 * Replaces DRSCertifier::certify (teaser/src/certification.cc:40-190; Params certification.h:70-108).  Host pointers.
 * R: 3x3 column-major rotation estimate; src/dst: 3 x N column-major (the TIMs the rotation was estimated from);
 * theta: N doubles, +1 inlier / -1 outlier (the bool overload of the reference maps true -> +1, :22-38).
 * traj (optional, capacity traj_capacity): the sub-optimality gap of every iteration
 * (CertificationResult::suboptimality_traj).  eig_decomposition_solver is accepted for source compatibility; both
 * values use the device eigensolver. */
typedef struct tzr_certifier_params {
  double noise_bound;     /* 0.01 */
  double cbar2;           /* 1 */
  double sub_optimality;  /* 1e-3 */
  double max_iterations;  /* 2e2 (a double in the reference too) */
  double gamma_tau;       /* 1.999999 */
  int32_t eig_decomposition_solver; /* 0 EIGEN, 1 SPECTRA */
  int32_t reserved;
} tzr_certifier_params;

typedef struct tzr_certification_result {
  int32_t is_optimal;
  int32_t n_iterations;        /* length of the trajectory */
  double best_suboptimality;
} tzr_certification_result;

void tzr_certifier_params_default(tzr_certifier_params* p);

/* tzr_certify and the single building blocks below (tzr_certifier_initial_matrix, tzr_certifier_dual_projection,
 * tzr_certifier_psd_projection) are tzr_certify_batch's path with B = 1: the same kernels, and one cusolverDnDsyevd on
 * the problem's (4n+4)^2 matrix per eigen step, so each result equals the batch entry's on that one problem bit for bit.
 * traj may be NULL (no trajectory).  The trajectory is kept on the device (at most ceil(max_iterations) gaps) and the
 * workspace is checked against free device memory.  Status: TZR_ERR_INVALID_ARG for a NULL pointer, n <= 0 or
 * traj_capacity < 0; TZR_ERR_TOO_LARGE when 4n+4 exceeds 32768; TZR_ERR_ALLOC when the workspace does not fit the
 * device; TZR_ERR_UNSUPPORTED when cuSOLVER cannot be loaded (tzr_certify and the PSD step only). */
int tzr_certify(tzr_ctx* ctx, const tzr_certifier_params* params, const double* R_colmajor9, const double* src_3xN,
                const double* dst_3xN, const double* theta, int n, tzr_certification_result* result, double* traj,
                int traj_capacity);

/* B certifications in one call: problem b has N[b] >= 1 measurements, its rotation at R_colmajor9xB + 9b (column-major),
 * src_3xN[b] / dst_3xN[b] (3 x N[b] column-major) and theta[b] (N[b] doubles, +1 / -1); params apply to every problem.
 * Host pointers, synchronous like tzr_compute_fpfh_batch.  results: B entries, each meaning what tzr_certify's result
 * means for that problem alone (is_optimal, n_iterations, best_suboptimality).  traj (may be NULL, or hold NULL entries):
 * traj[b] receives min(n_iterations, traj_capacity[b]) gaps; traj_capacity (B int32 >= 0) may be NULL when traj is
 * (TZR_ERR_INVALID_ARG when traj is given without it).
 * The problems run together: one launch sequence per iteration for the whole batch, one read-back of the active flags
 * per iteration, the trajectories copied back once at the end.  Finished problems are skipped by every kernel and by the
 * eigensolver.  The eigendecompositions of an iteration are one cusolverDnXsyevBatched call over the active problems'
 * matrices padded to 4 max N + 4 with a multiple of the identity that follows each problem's scale (DESIGN.md 3.9;
 * once some problems have finished, the active
 * ones are gathered into a compact batch first) while at least 8 problems are active, else one cusolverDnDsyevd per
 * active problem; the loop is also taken
 * when the batched symbol is missing, the batched call refuses the size, or debug flag 2097152 is set.
 * tzr_ctx_kernel_launches counts every eigensolver call as one launch.  A batch that does not fit the device is cut into
 * consecutive groups inside the call; the caller need not split it.  TZR_ERR_TOO_LARGE when some 4N[b]+4 exceeds 32768
 * (no result written); TZR_ERR_ALLOC when a single problem's workspace does not fit the device (tzr_last_error names
 * the size); TZR_ERR_UNSUPPORTED when cuSOLVER cannot be loaded. */
int tzr_certify_batch(tzr_ctx* ctx, const tzr_certifier_params* params, int B, const int32_t* N,
                      const double* R_colmajor9xB, const double* const* src_3xN, const double* const* dst_3xN,
                      const double* const* theta, tzr_certification_result* results, double* const* traj,
                      const int32_t* traj_capacity);

/* Building blocks, exposed so that each can be checked against the reference's fixtures
 * (test/teaser/certification-test.cc:355-497):
 * tzr_certifier_initial_matrix: M_init = D^T Q_cost D - mu J - lambda_guess (certification.cc:60-100), dense
 *   (4n+4)^2 column-major, and mu (:92) — covers getQCost, getBlockDiagOmega/getOmega1, getLambdaGuess.
 * tzr_certifier_dual_projection: getOptimalDualProjection (:316-446) with getLinearProjection's inverse map (:531-655)
 *   applied in closed form; W and W_dual are dense (4n+4)^2 column-major, theta as in tzr_certify. */
int tzr_certifier_initial_matrix(tzr_ctx* ctx, const tzr_certifier_params* params, const double* R_colmajor9,
                                 const double* src_3xN, const double* dst_3xN, const double* theta, int n,
                                 double* M_init, double* mu);
int tzr_certifier_dual_projection(tzr_ctx* ctx, const double* W, const double* theta, int n, double* W_dual);
/* tzr_certifier_psd_projection: the nearest-PSD step of one DRS iteration (linalg.h:84-99) on the path tzr_certify
 *   takes: M is any (4n+4)^2 column-major matrix, M_psd receives V+ diag(w+) V+^T of sym(M) = (M + M^T)/2 over its
 *   positive eigenpairs, w the (4n+4) ascending eigenvalues of sym(M).
 * tzr_certifier_batch_psd_projection / tzr_certifier_batch_dual_projection: the same step, and the dual projection, on
 *   B problems of N[b] measurements on tzr_certify_batch's path: its padded layout and, for the PSD step, the
 *   eigensolver route that call would take for B problems (debug flag 2097152 included).  M[b], M_psd[b], W[b],
 *   W_dual[b]: (4N[b]+4)^2 column-major; theta[b]: N[b] doubles.
 * The initial matrix and the dual projections (single and batch) run no eigensolver and do not load cuSOLVER: they
 * work where it cannot be loaded. */
int tzr_certifier_psd_projection(tzr_ctx* ctx, const double* M, int n, double* M_psd, double* w);
int tzr_certifier_batch_psd_projection(tzr_ctx* ctx, int B, const int32_t* N, const double* const* M,
                                       double* const* M_psd);
int tzr_certifier_batch_dual_projection(tzr_ctx* ctx, int B, const int32_t* N, const double* const* W,
                                        const double* const* theta, double* const* W_dual);

/* ---- whole path -----------------------------------------------------------------------------
 * Replaces RobustRegistrationSolver::solve(src, dst) (registration.cc:568-737) for one problem
 * (tzr_solve) or B independent problems (tzr_solve_batch).  All intermediates stay on the device.
 * clique: capacity n, sorted.  rot_inliers: one byte per rotation TIM — clique_size bytes for CHAIN (capacity n
 * is always enough), clique_size*(clique_size-1)/2 for COMPLETE (capacity n*(n-1)/2 is always enough).
 * trans_inliers: clique_size bytes (capacity n).  Optional outputs may be NULL. */
int tzr_solve(tzr_ctx* ctx, const tzr_params* params, const double* src_3xN, const double* dst_3xN, int n,
              tzr_solution* solution, int32_t* clique, uint8_t* rot_inliers, uint8_t* trans_inliers);

/* B problems, problem b has n[b] correspondences at src[b] / dst[b] (host pointers).
 * cliques: B*max_n int32, problem b's clique at cliques + b*max_n (may be NULL).
 * Sizes may differ.  A ragged batch runs as a few padded device batches (size classes, DESIGN.md 4.2): the problems,
 * ordered by n, are cut wherever n falls below the class's largest n divided by sqrt(2); a problem above 32768 is a class
 * of its own, and with estimate_scaling no class mixes problems on both sides of 256 (the two scale paths).  Padding rows
 * are isolated vertices, and every stage uses each problem's own n where the result depends on it, so each solution
 * (every field but stage_ms) and clique are the ones tzr_solve gives for that problem alone.  The classes share one
 * workspace and one host synchronisation. */
int tzr_solve_batch(tzr_ctx* ctx, const tzr_params* params, int B, const int32_t* n, const double* const* src,
                    const double* const* dst, tzr_solution* solutions, int32_t* cliques, int max_n);

/* Device-resident batch of equally sized problems: src_dev/dst_dev hold B*n*3 doubles each
 * (problem-major), solutions_dev B tzr_solution, cliques_dev B*n int32 (may be NULL).  Asynchronous on
 * the context's stream; this is what bench.py's kernel-only timing and the multi-GPU shards drive. */
int tzr_solve_batch_dev(tzr_ctx* ctx, const tzr_params* params, int B, int n, const double* src_dev,
                        const double* dst_dev, tzr_solution* solutions_dev, int32_t* cliques_dev);

/* Device-resident ragged batch: problem b has n[b] >= 1 correspondences (n is a host array).  src_dev/dst_dev hold the
 * problems back to back, sum(n) rows of 3 doubles each, problem b from row sum_{c<b} n[c] (the layout
 * tzr_register_cloud_pairs builds on the device from the matcher's index pairs).  solutions_dev: B tzr_solution in the caller's order.  cliques_dev
 * (sum(n) int32, may be NULL): problem b's sorted clique from the same row offset, -1 past its clique_size.  The size
 * classes of tzr_solve_batch; the results are those of tzr_solve on each problem alone.  Asynchronous on the context's
 * stream like tzr_solve_batch_dev, except that a class above 32768 correspondences reads back its core sizes. */
int tzr_solve_batch_ragged_dev(tzr_ctx* ctx, const tzr_params* params, int B, const int32_t* n, const double* src_dev,
                               const double* dst_dev, tzr_solution* solutions_dev, int32_t* cliques_dev);

/* Retrieve the adjacency bitset / degrees of problem b of the most recent solve on this context
 * (lazy materialisation of getInlierGraph(), registration.h:772; SURVEY a16). Host pointers.  After a ragged batch,
 * problem b (caller's order) has its own n[b] rows of tzr_words_per_row(n[b]) words and n[b] degrees, equal to its
 * single-solve graph. */
int tzr_last_graph(tzr_ctx* ctx, int b, uint64_t* adj_bits, int32_t* degree);
/* What tzr_last_graph would return: batch size and n of the retained solve (0, 0 if none; the largest n after a ragged
 * batch), whether a graph was
 * built (0 after inlier selection NONE: the reference never populates the graph, registration.cc:607-650, and
 * tzr_last_graph then yields an empty adjacency), and a generation counter that changes with every call that
 * rebuilds or invalidates the retained graph — callers that share a context (the C++ facade's per-thread context)
 * compare it with the value they saw after their own solve before trusting tzr_last_graph. */
int tzr_last_graph_info(const tzr_ctx* ctx, int32_t* B, int32_t* n, int32_t* has_graph, uint64_t* generation);

/* ---- certifying the most recent solve ---------------------------------------------------------
 * Every solve entry (tzr_solve, tzr_solve_batch uniform or ragged, tzr_solve_batch_dev, tzr_solve_batch_ragged_dev)
 * leaves each problem's record, clique, inlier masks and inputs in the context's workspace until the next call that
 * reuses it (another solve, tzr_graph_build, tzr_max_clique(_batch)).  tzr_solve_batch_dev reads the caller's src_dev /
 * dst_dev in place and keeps no copy: those buffers must still hold the solve's inputs when tzr_certify_last_solve runs.
 *
 * tzr_last_inliers: masks of problem b (caller's order) of the most recent solve on this context: rot_inliers receives
 * n_rot bytes (clique_size for CHAIN, clique_size*(clique_size-1)/2 for COMPLETE), trans_inliers clique_size bytes;
 * each may be NULL.  n_rot / n_trans (may be NULL) receive the counts; 0 and 0 for a problem whose solution is not
 * valid.  TZR_ERR_INVALID_ARG when no solve is retained (none yet, or a later call reused the workspace) or b is out
 * of range.  Equal, byte for byte, to what tzr_solve returns for that problem alone.  Host-synchronous, like
 * tzr_last_graph; ordered after every kernel of the solve, including those of the asynchronous _dev entries. */
int tzr_last_inliers(tzr_ctx* ctx, int b, uint8_t* rot_inliers, uint8_t* trans_inliers, int64_t* n_rot,
                     int32_t* n_trans);

/* DRSCertifier::certify(R, getMaxCliqueSrcTIMs(), getMaxCliqueDstTIMs(), getRotationInliersMask()) on problems of the
 * most recent solve, on tzr_certify_batch's path.  problems: count indices into the retained solve (duplicates and any
 * order allowed); NULL only when count equals the solve's B, then all problems in order.  Entry j of results, status
 * (may be NULL), traj and traj_capacity belongs to problems[j]; traj and traj_capacity follow tzr_certify_batch.
 * Problem b's inputs are built on the device from the workspace, bitwise the TIMs its rotation was solved on: R =
 * solution.rotation; CHAIN TIM i = src[leaf] - src[root] and (dst[leaf] - dst[root]) * (1.0 / scale) over the sorted
 * clique; COMPLETE TIMs in computeTIMs order with the same de-scaling; theta = +1 where the rotation mask is set, -1
 * elsewhere; N = n_rot.  Noise bound of problem b: noise_bound / scale_b (nbs = cbar2 * nb * nb).  The rotation solver
 * ran with 2 * the solve's noise_bound / scale (registration.cc:702-704): set params->noise_bound to 2 * the solve's
 * noise_bound to certify the problem it solved.  Only the B solution records cross PCIe; no TIM or mask does.
 * status[j]: TZR_OK certified; TZR_ERR_INVALID_ARG the solution is not valid, or a gathered measurement is not finite (inlier selection NONE with a non-finite input row), never certified, result
 * {0, 0, +inf} and no trajectory; TZR_ERR_TOO_LARGE 4N + 4 > 32768 (COMPLETE above 128 clique points), result
 * {0, 0, +inf}.  Every other entry is certified.  Returns TZR_ERR_TOO_LARGE when some entry was too large, TZR_OK
 * otherwise; TZR_ERR_INVALID_ARG (nothing written) when no solve is retained or an argument is out of range.
 * tzr_ctx_kernel_launches counts tzr_certify_batch's launches plus one gather launch per group. */
int tzr_certify_last_solve(tzr_ctx* ctx, const tzr_certifier_params* params, int count, const int32_t* problems,
                           tzr_certification_result* results, int32_t* status, double* const* traj,
                           const int32_t* traj_capacity);

/* ---- registering cloud pairs: descriptors, matching and the robust solve in one call --------------------------
 * What the reference example teaser_cpp_fpfh does per pair (FPFHEstimation::computeFPFHFeatures on both clouds,
 * Matcher::calculateCorrespondences, solve(src_cloud, dst_cloud, correspondences), registration.cc:553-566), for many
 * pairs over a shared table of clouds, with every stage on the device and each cloud's descriptors computed once. */
typedef struct tzr_frontend_params {
  double normal_search_radius;  /* FPFHEstimation::computeFPFHFeatures, default 0.03 */
  double fpfh_search_radius;    /* default 0.05 */
  int32_t use_absolute_scale;   /* Matcher::calculateCorrespondences defaults: 1, 1, 1, 0 */
  int32_t use_crosscheck;
  int32_t use_tuple_test;
  float tuple_scale;
} tzr_frontend_params;

void tzr_frontend_params_default(tzr_frontend_params* p);

/* n_clouds clouds (host pointers): cloud c has n[c] >= 1 points at pts[c] (n[c] x 3 float).  P pairs: pair_clouds is
 * P x 2 int32 (source cloud, target cloud); a cloud may appear in any number of pairs, on either side, and a pair may
 * match a cloud with itself.  tuple_seeds: P seeds of the tuple test (NULL: 0 for every pair).  Synchronous.
 * Per pair p: solutions[p], status[p] and n_corr[p] are always written.  corr[p] (may be NULL, or hold NULL entries;
 * capacity n[src] + n[dst] rows x 2 int32) receives the sorted unique correspondences; cliques[p] (same rules and
 * capacity) the sorted max clique, as rows of corr[p]; global_scale (P floats, may be NULL) Matcher::global_scale_;
 * problem_index (P int32, may be NULL) p's index in the retained solve, -1 when p was not solved.
 * status[p]: TZR_OK solved; TZR_ERR_TOO_LARGE when a point of one of its clouds has more than 4096 neighbours inside a
 * radius (nothing matched, n_corr = 0), or its correspondences exceed the context's max_n, or with estimate_scaling
 * reach 46341 (correspondences written, not solved); TZR_ERR_INVALID_ARG no correspondence.  An unsolved pair gets a
 * zeroed record (valid = 0).  Returns TZR_ERR_TOO_LARGE when some pair was too large (every other pair is complete),
 * TZR_ERR_ALLOC when the batch's buffers do not fit the device (tzr_last_error names the size).
 * For every solved pair the outputs are bit-identical (the record except stage_ms, the clique, the correspondences and
 * the global scale) to tzr_compute_fpfh_batch over the clouds, tzr_match_correspondences_batch over the pairs with the
 * same seeds, the float points at the correspondences converted to float64, then tzr_solve_batch over the solved pairs.
 * The call is a solve entry: tzr_last_inliers, tzr_last_graph and tzr_certify_last_solve then see the solved pairs in
 * ascending pair order (problem_index).  Two host synchronisations (plus the core-size read-back of a class above 32768
 * correspondences): the per-cloud overflow flags, per-pair counts and global scales after matching, from which the
 * solve's size classes are planned, and the records, correspondences and cliques at the end.  DESIGN.md §3.10. */
int tzr_register_cloud_pairs(tzr_ctx* ctx, const tzr_frontend_params* fparams, const tzr_params* params,
                             int n_clouds, const int32_t* n, const float* const* pts,
                             int P, const int32_t* pair_clouds, const uint64_t* tuple_seeds,
                             tzr_solution* solutions, int32_t* status, int32_t* problem_index,
                             int64_t* n_corr, int32_t* const* corr, int32_t* const* cliques, float* global_scale);

/* ---- refining registrations: point-to-point ICP -------------------------------------------------------------
 * The refinement step of the reference's FPFH + TEASER++ + ICP tutorial (examples/teaser_python_fpfh_icp: Open3D's
 * registration_icp with TransformationEstimationPointToPoint, seeded with TEASER's solution), for many problems at once.
 * The loop is Open3D's RegistrationICP with ICPConvergenceCriteria, defined here as follows (DESIGN.md §3.11):
 *   - Inputs: source x (ns float xyz), target y (nd float xyz), both read exactly as float64, and an initial similarity
 *     (s, R0, t0).  s is held fixed (1 for rigid ICP, a solve's scale when seeded from an estimate_scaling solve).
 *   - Transform: p_i = s * (R x_i) + t, row r computed as s * ((R(r,0) x + R(r,1) y) + R(r,2) z) + t(r) from the
 *     original point and the current (R, t), never incrementally (IEEE double, no FMA contraction).
 *   - Correspondence of p_i: the target with the smallest d^2 = (dx dx + dy dy) + dz dz in float64, strictly d^2 < r^2
 *     with r = max_correspondence_distance and r^2 rounded once; the lowest target index among equal d^2; none for a
 *     non-finite p_i, and a non-finite target point is never matched.
 *   - eval(T): count of correspondences, fitness = count / ns (ns includes non-finite points), inlier_rmse =
 *     sqrt(sum d^2 / count); both 0 when count = 0.
 *   - Update (R_u, t_u) from the current correspondences: count >= 3: Kabsch on centred coordinates, H = sum (p - mu_p)
 *     (q - mu_q)^T, R_u the rotation stage's SVD with the reflection fix, t_u = mu_q - R_u mu_p; count 1 or 2: R_u = I,
 *     t_u = mu_q - mu_p; count 0: the identity.
 *   - Loop: r_0 = eval(T_0); for i < max_iteration: R <- R_u R, t <- R_u t + t_u, r_{i+1} = eval(T_{i+1}), iterations =
 *     i + 1, stop with converged = 1 when |delta fitness| < relative_fitness and |delta rmse| < relative_rmse.
 * Host pointers, synchronous.  The iterations are enqueued without a host synchronisation: 2 + 4 * max_iteration kernel
 * launches per call (+ 4 for the grid build when some target has at least 1024 points), whatever B; a finished problem
 * costs nothing in later launches.  The nearest-neighbour search is brute force below 1024 target points and a hashed
 * uniform grid (cell edge r (1 + 1e-5)) from there on; both give the same correspondences (debug flags 33554432 and
 * 67108864).  These calls are not solve entries: they use a workspace of their own, so a retained solve
 * (tzr_last_inliers, tzr_last_graph, tzr_certify_last_solve) stays retained across them. */
typedef struct tzr_icp_params {
  double max_correspondence_distance;  /* no default, as in Open3D: <= 0 or non-finite is TZR_ERR_INVALID_ARG */
  double relative_fitness;             /* 1e-6 (ICPConvergenceCriteria) */
  double relative_rmse;                /* 1e-6 */
  int32_t max_iteration;               /* 30; >= 0 */
  int32_t reserved;
} tzr_icp_params;

typedef struct tzr_similarity {
  double scale;
  double rotation[9];    /* column-major */
  double translation[3];
} tzr_similarity;

typedef struct tzr_icp_result {
  tzr_similarity transform;  /* the last T (scale unchanged) */
  double fitness;
  double inlier_rmse;
  int32_t iterations;
  int32_t n_correspondences;
  int32_t converged;
  int32_t reserved;
} tzr_icp_result;

/* max_correspondence_distance 0 (the caller must set it), relative_fitness 1e-6, relative_rmse 1e-6, max_iteration 30. */
void tzr_icp_params_default(tzr_icp_params* p);

/* One problem.  init may be NULL (identity, scale 1); a non-finite init or a scale <= 0 is TZR_ERR_INVALID_ARG.
 * corr (may be NULL; capacity ns x 2 int32): the final correspondences (source index, target index), ascending by
 * source, result->n_correspondences rows.  With max_iteration = 0 the result is init, its evaluation, 0 iterations and
 * converged = 0.  This is tzr_icp_batch with B = 1. */
int tzr_icp(tzr_ctx* ctx, const tzr_icp_params* params, const float* src, int ns, const float* dst, int nd,
            const tzr_similarity* init, tzr_icp_result* result, int32_t* corr);

/* B ragged problems: problem b has ns[b] >= 1 source points at src[b] and nd[b] >= 1 target points at dst[b], its
 * initial similarity at init[b]; params apply to every problem.  results: B entries.  corr (may be NULL, or hold NULL
 * entries): as tzr_icp's, per problem.  Per problem, every output is bit-identical to tzr_icp on that problem alone:
 * every reduction runs in an order fixed by the problem's own points.  TZR_ERR_TOO_LARGE when the sources or the targets
 * of the batch exceed 2^31 - 1 points; TZR_ERR_ALLOC when the workspace does not fit the device (tzr_last_error names
 * the size). */
int tzr_icp_batch(tzr_ctx* ctx, const tzr_icp_params* params, int B, const int32_t* ns, const float* const* src,
                  const int32_t* nd, const float* const* dst, const tzr_similarity* init, tzr_icp_result* results,
                  int32_t* const* corr);

/* tzr_register_cloud_pairs (same arguments, same outputs bit for bit), then ICP of every solved pair whose solution is
 * valid, on the pair's two clouds (source cloud, target cloud), seeded with (scale, rotation, translation) of its
 * solution.  icp (required) applies to every pair.  icp_results: P entries; a pair that was not refined (not solved,
 * or its solution not valid or not finite) gets a zeroed record, which the caller can tell from status[p] and
 * solutions[p].valid.  Each refined record is bit-identical to tzr_icp_batch over the valid solved pairs seeded with
 * their records.  The clouds and records are already on the device: the refinement adds no host synchronisation and no
 * upload of points, and it runs before the call's second synchronisation.  Launches: tzr_register_cloud_pairs' own plus,
 * when some pair was solved, 1 seed launch and tzr_icp_batch's (2 + 4 * max_iteration, + 4 when some cloud has 1024
 * points or more).  Like tzr_register_cloud_pairs this is a solve entry: tzr_last_inliers, tzr_last_graph and
 * tzr_certify_last_solve see its solve, which the refinement does not touch. */
int tzr_register_cloud_pairs_icp(tzr_ctx* ctx, const tzr_frontend_params* fparams, const tzr_params* params,
                                 int n_clouds, const int32_t* n, const float* const* pts,
                                 int P, const int32_t* pair_clouds, const uint64_t* tuple_seeds,
                                 tzr_solution* solutions, int32_t* status, int32_t* problem_index,
                                 int64_t* n_corr, int32_t* const* corr, int32_t* const* cliques, float* global_scale,
                                 const tzr_icp_params* icp, tzr_icp_result* icp_results);

/* ---- refining registrations: point-to-plane ICP -------------------------------------------------------------
 * Open3D's registration_icp with TransformationEstimationPointToPlane, for many problems at once, defined here as
 * follows (DESIGN.md §3.13):
 *   - Unchanged from tzr_icp: the inputs x, y and (s, R0, t0), the fixed scale, the transform p_i = s (R x_i) + t from the
 *     original point on every iteration, the correspondence search and its routes, eval(T) (fitness and inlier_rmse from
 *     the point distances d^2, as Open3D evaluates point-to-plane runs), the loop, the convergence test and the
 *     composition R <- R_u R, t <- R_u t + t_u.  The target normals play no part in the search or in the evaluation.
 *   - Target normals: nd x 4 floats per target in the library's normals layout (normal_x, normal_y, normal_z,
 *     curvature: tzr_compute_fpfh's and tzr_estimate_normals' normals_out); the fourth float is ignored.  Read exactly as
 *     float64 and used as given: not renormalised, and their sign does not matter (below).
 *   - Update (R_u, t_u) from the current correspondences, in IEEE float64 with no FMA contraction.  count = 0: the
 *     identity.  Otherwise c = mu_p, the mean of the matched transformed sources, and each correspondence (i, j) whose
 *     normal n = n_j has three finite components contributes, with u = p_i - c and q = y_j:
 *       a = u x n:  a0 = u1 n2 - u2 n1,  a1 = u2 n0 - u0 n2,  a2 = u0 n1 - u1 n0
 *       J = (a0, a1, a2, n0, n1, n2),  r = ((p0 - q0) n0 + (p1 - q1) n1) + (p2 - q2) n2
 *     A correspondence with a non-finite normal counts for fitness and rmse but adds nothing here.  A = sum J J^T (its
 *     21 distinct entries) and g = sum J r, summed in the fixed chunk order of tzr_icp's sums; x solves A x = -g by the
 *     6 x 6 solve below.  With ca = cos x0, sa = sin x0, cb = cos x1, sb = sin x1, cg = cos x2, sg = sin x2,
 *     R_u = Rz(x2) Ry(x1) Rx(x0) (Open3D's TransformVector6dToMatrix4d) =
 *       [ cg cb   (cg sb) sa - sg ca   (cg sb) ca + sg sa ]
 *       [ sg cb   (sg sb) sa + cg ca   (sg sb) ca - cg sa ]
 *       [ -sb     cb sa                cb ca              ]
 *     and t_u = (c + tau) - R_u c with tau = (x3, x4, x5), row r: (c(r) + tau(r)) - ((R_u(r,0) c0 + R_u(r,1) c1) +
 *     R_u(r,2) c2).  If any component of x is non-finite the update is the identity.  Flipping n negates J and r
 *     exactly, so A, g and every output are bit-identical under any choice of normal signs.
 *   - The 6 x 6 solve: a truncated LDL^T with diagonal pivoting.  tol = 1e-10 * max_k A_kk (the original diagonal).
 *     Step k picks the remaining index with the largest current diagonal (the lowest index on ties; a NaN diagonal is
 *     never the largest); if that diagonal is not > tol (NaN included), elimination stops and every remaining component
 *     of the permuted solution is 0.  Otherwise it eliminates as usual; then forward substitution, scaling by the
 *     pivots and back substitution over the leading block.  So a flat target (all normals parallel) gets no motion
 *     along its unobservable directions.
 *   - Centred linearisation: Open3D linearises about the origin; this one about c.  The two are the same Gauss-Newton
 *     step up to second order in the rotation angle and have the same fixed points, and the centred one keeps its
 *     digits far from the origin (DESIGN.md §3.13).
 * Launches: 2 + 4 * max_iteration (+ 4 for the grid build when some target has at least 1024 points), whatever B, as
 * tzr_icp_batch.  Workspace: tzr_icp's own, so a retained solve stays retained. */

/* One problem: tzr_icp's arguments plus dst_normals (nd x 4 floats, required).  This is tzr_icp_point_to_plane_batch
 * with B = 1. */
int tzr_icp_point_to_plane(tzr_ctx* ctx, const tzr_icp_params* params, const float* src, int ns, const float* dst,
                           int nd, const float* dst_normals, const tzr_similarity* init, tzr_icp_result* result,
                           int32_t* corr);

/* B ragged problems: tzr_icp_batch's arguments plus dst_normals (B entries, entry b nd[b] x 4 floats; NULL or a NULL
 * entry is TZR_ERR_INVALID_ARG).  Per problem, every output is bit-identical to tzr_icp_point_to_plane on that problem
 * alone. */
int tzr_icp_point_to_plane_batch(tzr_ctx* ctx, const tzr_icp_params* params, int B, const int32_t* ns,
                                 const float* const* src, const int32_t* nd, const float* const* dst,
                                 const float* const* dst_normals, const tzr_similarity* init,
                                 tzr_icp_result* results, int32_t* const* corr);

/* tzr_register_cloud_pairs_icp with point-to-plane ICP: the same arguments and the same outputs, except that each
 * refined record is point-to-plane ICP on the pair's two clouds, using the target cloud's normals from the call's own
 * FPFH stage (normal_search_radius, viewpoint at the origin).  No normal pass, upload or host synchronisation is added.
 * Each refined record is bit-identical to tzr_register_cloud_pairs, then tzr_estimate_normals_batch over the clouds at
 * fparams->normal_search_radius, then tzr_icp_point_to_plane_batch over the valid solved pairs seeded with their
 * records.  Launches: as tzr_register_cloud_pairs_icp. */
int tzr_register_cloud_pairs_icp_point_to_plane(tzr_ctx* ctx, const tzr_frontend_params* fparams,
                                                const tzr_params* params, int n_clouds, const int32_t* n,
                                                const float* const* pts, int P, const int32_t* pair_clouds,
                                                const uint64_t* tuple_seeds, tzr_solution* solutions,
                                                int32_t* status, int32_t* problem_index, int64_t* n_corr,
                                                int32_t* const* corr, int32_t* const* cliques, float* global_scale,
                                                const tzr_icp_params* icp, tzr_icp_result* icp_results);

/* ---- refining registrations: generalized ICP -----------------------------------------------------------------
 * Open3D's registration_generalized_icp (TransformationEstimationForGeneralizedICP, its default L2 loss), for many
 * problems at once, defined here as follows (DESIGN.md §3.14):
 *   - Unchanged from tzr_icp_point_to_plane: the inputs and the fixed scale s, the transform p_i = s (R x_i) + t, the
 *     search and both of its routes, eval(T), the loop, the convergence test, the composition, the 6 x 6 solve of
 *     A x = -g, R_u = Rz(x2) Ry(x1) Rx(x0) and t_u = (c + tau) - R_u c with c = mu_p.  Only the system changes.
 *   - Normals: the source normals (ns x 4 floats) and the target normals (nd x 4 floats), both in the library's normals
 *     layout (curvature ignored), read exactly as float64 and used up to length and sign.
 *   - System, in IEEE float64 with no FMA contraction.  For each correspondence (i, j), with u = p_i - c, d = p_i - y_j,
 *     m = m_i (source normal) and n = n_j (target normal):
 *       m' = R m, row r: (R(r,0) m0 + R(r,1) m1) + R(r,2) m2 with the current R, without the scale.
 *       C(v) = I - (k v_a) v_b, k = (1 - epsilon) / ((v0 v0 + v1 v1) + v2 v2): each of the six upper entries
 *         (00, 01, 02, 11, 12, 22) is delta_ab - (k v_a) v_b, mirrored below.  For a unit v this is Open3D's
 *         Rx diag(epsilon, 1, 1) Rx^T with Rx = GetRotationFromE1ToX(v); dividing by v^T v uses normals up to length,
 *         and a negated v gives the same bits.
 *       M = s2 C(m') + C(n) entry by entry, s2 = s * s rounded once (Open3D's (sR) C (sR)^T plus the target's).
 *       cofactors c00 = M11 M22 - M12 M12, c01 = M02 M12 - M01 M22, c02 = M01 M12 - M02 M11,
 *                 c11 = M00 M22 - M02 M02, c12 = M01 M02 - M00 M12, c22 = M00 M11 - M01 M01;
 *       det = (M00 c00 + M01 c01) + M02 c02, A = M^-1 with A_ab = c_ab / det.
 *       J = [e_k x u (k = 0..2), I] (3 x 6).  The correspondence adds J^T A J (21 entries, the upper triangle row by
 *       row as point-to-plane's) and J^T A d (6) to the fixed-order chunk sums, evaluated as
 *         omega-omega (k <= l): (u x A (e_l x u))_k,  omega-tau: (u x a_l)_k with a_l = column l of A,
 *         tau-tau (k <= l): A_kl,  g = (u x w, w) with w = A d,
 *       where a x b = (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0) and A v row r is (A(r,0) v0 + A(r,1) v1) + A(r,2) v2.
 *     A correspondence adds nothing, but still counts for fitness and rmse, when either normal has a non-finite
 *     component or zero length, or when det is not > 0 or not finite.
 *   - epsilon (Open3D's epsilon, 1e-3 there) must be finite and > 0; anything else is TZR_ERR_INVALID_ARG.  Where R m
 *     is parallel to n, M has the eigenvalue (s2 + 1) epsilon and A loses accuracy like 2^-53 / epsilon, so below
 *     about 1e-9 a step is less accurate than its float inputs, and near 1e-20 the det > 0 rule drops an arbitrary
 *     subset of such correspondences (DESIGN.md §3.14 has the measured errors).
 *   - Relation to Open3D: Open3D forms W = M^-1/2 and sums three weighted rows per correspondence; with the L2 loss
 *     sum rows^T rows = J^T M^-1 J, so no matrix square root is needed.  Open3D's GetRotationFromE1ToX returns the
 *     identity when e1 . n < -0.99, which makes its covariance depend on the normal's sign there; this definition uses
 *     the closed form and does not.  The step is linearised about c, as point-to-plane's (DESIGN.md §3.13).
 * Launches: 2 + 4 * max_iteration (+ 4 for the grid build when some target has at least 1024 points), whatever B, as
 * tzr_icp_batch.  Workspace: tzr_icp's own, so a retained solve stays retained. */

/* One problem: tzr_icp_point_to_plane's arguments plus epsilon and src_normals (ns x 4 floats, required).  This is
 * tzr_icp_generalized_batch with B = 1. */
int tzr_icp_generalized(tzr_ctx* ctx, const tzr_icp_params* params, double epsilon, const float* src, int ns,
                        const float* src_normals, const float* dst, int nd, const float* dst_normals,
                        const tzr_similarity* init, tzr_icp_result* result, int32_t* corr);

/* B ragged problems: tzr_icp_point_to_plane_batch's arguments plus epsilon and src_normals (B entries, entry b ns[b] x 4
 * floats).  Either normals array NULL, or holding a NULL entry, is TZR_ERR_INVALID_ARG.  Per problem, every output is
 * bit-identical to tzr_icp_generalized on that problem alone. */
int tzr_icp_generalized_batch(tzr_ctx* ctx, const tzr_icp_params* params, double epsilon, int B, const int32_t* ns,
                              const float* const* src, const float* const* src_normals, const int32_t* nd,
                              const float* const* dst, const float* const* dst_normals, const tzr_similarity* init,
                              tzr_icp_result* results, int32_t* const* corr);

/* tzr_register_cloud_pairs_icp with generalized ICP: the same arguments plus epsilon, and the same outputs, except that
 * each refined record is generalized ICP on the pair's two clouds, using both clouds' normals from the call's own FPFH
 * stage (normal_search_radius, viewpoint at the origin).  No normal pass, upload or host synchronisation is added.
 * Each refined record is bit-identical to tzr_register_cloud_pairs, then tzr_estimate_normals_batch over the clouds at
 * fparams->normal_search_radius, then tzr_icp_generalized_batch over the valid solved pairs seeded with their records.
 * Launches: as tzr_register_cloud_pairs_icp. */
int tzr_register_cloud_pairs_icp_generalized(tzr_ctx* ctx, const tzr_frontend_params* fparams,
                                             const tzr_params* params, int n_clouds, const int32_t* n,
                                             const float* const* pts, int P, const int32_t* pair_clouds,
                                             const uint64_t* tuple_seeds, tzr_solution* solutions, int32_t* status,
                                             int32_t* problem_index, int64_t* n_corr, int32_t* const* corr,
                                             int32_t* const* cliques, float* global_scale, const tzr_icp_params* icp,
                                             double epsilon, tzr_icp_result* icp_results);

/* ---- refining registrations: robust kernels ------------------------------------------------------------------
 * Open3D's robust kernels (L1Loss, HuberLoss, CauchyLoss, GMLoss, TukeyLoss) for point-to-plane ICP
 * (TransformationEstimationPointToPlane(kernel)) and generalized ICP (TransformationEstimationForGeneralizedICP(epsilon,
 * kernel)), for many problems at once, defined here as follows (DESIGN.md §3.15):
 *   - Unchanged from tzr_icp_point_to_plane and tzr_icp_generalized: the inputs, the search and both of its routes,
 *     eval(T) (fitness and inlier_rmse stay unweighted, as in Open3D), the loop, the convergence test, the 6 x 6 solve,
 *     R_u, t_u and the composition.  Only each correspondence's contribution to the system is weighted.
 *   - Weights, in IEEE float64 with no FMA contraction, from e = |r| (a residual's sign never matters), k = kernel->k:
 *       TZR_LOSS_L2      1
 *       TZR_LOSS_L1      1 / e
 *       TZR_LOSS_HUBER   k / max(e, k)
 *       TZR_LOSS_CAUCHY  q = e / k, then 1 / (1 + q q)
 *       TZR_LOSS_GM      t = k + e e, then k / (t t)  (k in squared residual units, as Open3D's GMLoss)
 *       TZR_LOSS_TUKEY   0 when e > k; otherwise q = e / k, t = 1 - q q, then t t
 *     Each is rho'(r) / r of Open3D's published rho.  A weight that is not finite (L1 at e = 0) removes that residual's
 *     correspondence from the system; it still counts for fitness and rmse.  (Open3D would multiply an infinite weight by
 *     a zero residual and put NaN into its normal equations.)
 *   - Point-to-plane: w = weight(r) with tzr_icp_point_to_plane's r and J; the correspondence adds (w J_a) J_b to the 21
 *     upper entries and (w J_a) r to g.  With w = 1 these are J_a J_b and J_a r bit for bit.
 *   - Generalized: M = s2 C(m') + C(n) as tzr_icp_generalized's.  W = M^-1/2 from the two-sided Jacobi SVD of the
 *     rotation stage (M = V diag(sigma) V^T for the symmetric positive definite M, sigma descending), with
 *     q_k = 1 / sqrt(sigma_k) and W_ab = ((V_a0 q_0) V_b0 + (V_a1 q_1) V_b1) + (V_a2 q_2) V_b2.  The three whitened
 *     residuals r_k = (W_k0 d0 + W_k1 d1) + W_k2 d2 (d = p_i - y_j) give w_k = weight(r_k), and
 *     A~_ab = ((w_0 W_0a) W_0b + (w_1 W_1a) W_1b) + (w_2 W_2a) W_2b, i.e. W diag(w) W, the sum over Open3D's three
 *     weighted rows.  A~ replaces A in tzr_icp_generalized's J^T A J and J^T A d, evaluated as written there.
 *     M and so every output does not depend on either normal's sign.  A correspondence adds nothing, but still counts
 *     for fitness and rmse, when either normal has a non-finite component or zero length, when some sigma_k is not > 0
 *     or not finite, or when some w_k is not finite.
 *   - TZR_LOSS_L2 runs tzr_icp_point_to_plane's or tzr_icp_generalized's own system (the adjugate inverse), so its
 *     results are bit-identical to those entries'.  (W W equals M^-1 only up to rounding.)
 *   - kernel NULL, an unknown type, or a k that is not finite and > 0 for HUBER, CAUCHY, GM and TUKEY (k is ignored for
 *     L2 and L1) is TZR_ERR_INVALID_ARG, checked before any device work.
 * Launches: 2 + 4 * max_iteration (+ 4 for the grid build when some target has at least 1024 points), whatever B, as
 * tzr_icp_batch.  Workspace: tzr_icp's own, so a retained solve stays retained. */
#define TZR_LOSS_L2 0
#define TZR_LOSS_L1 1
#define TZR_LOSS_HUBER 2
#define TZR_LOSS_CAUCHY 3
#define TZR_LOSS_GM 4
#define TZR_LOSS_TUKEY 5

typedef struct tzr_robust_kernel {
  int32_t type;     /* TZR_LOSS_* */
  int32_t reserved; /* 0 */
  double k;         /* finite and > 0 for HUBER, CAUCHY, GM and TUKEY; ignored for L2 and L1 */
} tzr_robust_kernel;

/* B ragged problems: tzr_icp_point_to_plane_batch's arguments plus the kernel.  Per problem, every output is
 * bit-identical to the same call on that problem alone. */
int tzr_icp_point_to_plane_robust_batch(tzr_ctx* ctx, const tzr_icp_params* params, int B, const int32_t* ns,
                                        const float* const* src, const int32_t* nd, const float* const* dst,
                                        const float* const* dst_normals, const tzr_similarity* init,
                                        tzr_icp_result* results, int32_t* const* corr,
                                        const tzr_robust_kernel* kernel);

/* B ragged problems: tzr_icp_generalized_batch's arguments plus the kernel.  Per problem, every output is bit-identical
 * to the same call on that problem alone. */
int tzr_icp_generalized_robust_batch(tzr_ctx* ctx, const tzr_icp_params* params, double epsilon, int B,
                                     const int32_t* ns, const float* const* src, const float* const* src_normals,
                                     const int32_t* nd, const float* const* dst, const float* const* dst_normals,
                                     const tzr_similarity* init, tzr_icp_result* results, int32_t* const* corr,
                                     const tzr_robust_kernel* kernel);

/* tzr_register_cloud_pairs_icp with a robust kernel: the same arguments plus method (1 = point-to-plane, 2 =
 * generalized; anything else is TZR_ERR_INVALID_ARG), epsilon (read for method 2 only) and the kernel, and the same
 * outputs.  The normals are the call's own FPFH stage's, as in tzr_register_cloud_pairs_icp_point_to_plane and
 * tzr_register_cloud_pairs_icp_generalized.  Each refined record is bit-identical to tzr_register_cloud_pairs, then
 * tzr_estimate_normals_batch over the clouds at fparams->normal_search_radius, then
 * tzr_icp_point_to_plane_robust_batch or tzr_icp_generalized_robust_batch over the valid solved pairs seeded with
 * their records.  Launches: as tzr_register_cloud_pairs_icp. */
int tzr_register_cloud_pairs_icp_robust(tzr_ctx* ctx, const tzr_frontend_params* fparams, const tzr_params* params,
                                        int n_clouds, const int32_t* n, const float* const* pts, int P,
                                        const int32_t* pair_clouds, const uint64_t* tuple_seeds,
                                        tzr_solution* solutions, int32_t* status, int32_t* problem_index,
                                        int64_t* n_corr, int32_t* const* corr, int32_t* const* cliques,
                                        float* global_scale, const tzr_icp_params* icp, int32_t method,
                                        double epsilon, const tzr_robust_kernel* kernel,
                                        tzr_icp_result* icp_results);

/* ---- refining registrations: coloured ICP -------------------------------------------------------------------
 * Open3D's registration_colored_icp (TransformationEstimationForColoredICP with InitializePointCloudForColoredICP's
 * colour gradients), for many problems at once, defined here as follows (DESIGN.md §3.17):
 *   - Colours: n x 3 floats (r, g, b) per point, any range (Open3D uses [0, 1]), read exactly as float64.  A point's
 *     intensity is ((r + g) + b) / 3.0.
 *   - Colour gradients of a target cloud (tzr_estimate_color_gradients), in IEEE float64 with no FMA contraction, for
 *     every point k with position v_k, normal n_k (the library's normals layout, curvature ignored) and intensity i_k:
 *       neighbours: the radius search of tzr_estimate_normals (float d^2 < R^2 with R^2 = (float)(R * R), the list
 *         ordered by (d^2, index)), cut to its first nn = min(count, 30) entries (Open3D's KDTreeSearchParamHybrid(R,
 *         30)).  The 30 are chosen by a bounded selection, so no neighbourhood is too large.  nn < 4: the gradient is
 *         (0, 0, 0).
 *       rows: entry 0 is skipped, whatever it is (Open3D's loop starts at 1).  Entry e = 1 ... nn - 1 at point v with
 *         intensity i gives s = ((v0 - vk0) n0 + (v1 - vk1) n1) + (v2 - vk2) n2, a_e(c) = (v(c) - s n(c)) - vk(c)
 *         (v projected onto the tangent plane, minus v_k) and b_e = i - i_k.  One more row c = (nn - 1) n with
 *         right-hand side 0 pins the normal component.
 *       system: M_ab = sum_e a_e(a) a_e(b) + c_a c_b and h_a = sum_e a_e(a) b_e, each summed from 0.0 in list order with
 *         the constraint row last.  If an entry of M or h is not finite, the gradient is (NaN, NaN, NaN).  Otherwise
 *         the gradient x solves M x = h by the truncated, diagonally pivoted LDL^T of the 6 x 6 step below (the same
 *         device code at size 3; tol = 1e-10 max_k M_kk, the lowest index on ties), so a direction the neighbours do
 *         not observe (collinear neighbours) gets 0.  Open3D solves with Eigen's LDLT: the two agree up to rounding,
 *         and only on neighbourhoods that are not degenerate.
 *     The gradient is float64 and does not depend on the normal's sign (n enters as s n, n n^T and c c^T only).
 *   - Step: tzr_icp_point_to_plane's inputs, search, eval(T), loop, convergence test, centring (c = mu_p, u = p - c),
 *     6 x 6 solve, R_u, t_u and composition, unchanged.  Each correspondence (i, j) with p the transformed source
 *     point, q = y_j, n its target normal, g its target's gradient, i_s the source's and i_t the target's intensity,
 *     sg = sqrt(lambda) and si = sqrt(1 - lambda) (lambda = lambda_geometric) gives two rows:
 *       geometric:    J_G = (sg a0, sg a1, sg a2, sg n0, sg n1, sg n2) with a = u x n as in point-to-plane, and
 *                     r_G = sg r, r = ((p0 - q0) n0 + (p1 - q1) n1) + (p2 - q2) n2.
 *       photometric:  d(c) = (p(c) - r n(c)) - q(c) (the projection of p, minus q), i_hat = ((g0 d0 + g1 d1) + g2 d2) +
 *                     i_t, m_k = -((g0 M_0k + g1 M_1k) + g2 M_2k) with M_ab = delta_ab - n_a n_b,
 *                     J_I = (si e0, si e1, si e2, si m0, si m1, si m2) with e = u x m written as point-to-plane's
 *                     a = u x n, and r_I = si (i_s - i_hat).
 *     Each row has its own weight w = weight(r_row) of the TZR_LOSS_* kernel (w = 1 without a kernel) and adds its own
 *     terms, the geometric row first: (w J_a) J_b to the 21 upper entries and (w J_a) r_row to g, as the robust
 *     point-to-plane step (without a kernel, J_a J_b and J_a r_row).  A row adds nothing when its factor (sg or si) is
 *     0 or its weight is not finite; the photometric row adds nothing when the source colour, the target colour or g
 *     has a non-finite component; a correspondence whose normal has a non-finite component adds nothing.  Every such
 *     correspondence still counts for fitness and rmse.
 *     Consequences: with lambda = 1 every output is bit-identical to tzr_icp_point_to_plane_robust_batch with the same
 *     kernel, and with no kernel or TZR_LOSS_L2 to tzr_icp_point_to_plane_batch; flipping any normal changes no bit.
 *   - lambda_geometric: Open3D's default is 0.968.  A value outside [0, 1] is replaced by 0.968, as Open3D's
 *     constructor does; a non-finite value is TZR_ERR_INVALID_ARG.
 *   - Gradients inside the call: from the targets and their normals and colours already uploaded, at radius
 *     2 max_correspondence_distance (RegistrationColoredICP's), bit-identical to tzr_estimate_color_gradients_batch
 *     over the targets at that radius.
 * Launches: tzr_icp_point_to_plane_batch's (2 + 4 * max_iteration, + 4 when some target has 1024 points or more) plus
 * the gradient pass (1, + 4 when some target has 4096 points or more, or under debug flag 8388608), whatever B.
 * Workspace: tzr_icp's own, so a retained solve stays retained. */

/* Colour gradients of one cloud: pts (n x 3 floats), normals (n x 4 floats, nx, ny, nz, curvature), colors (n x 3
 * floats), radius (finite and > 0, else TZR_ERR_INVALID_ARG), grad_out (n x 3 doubles).  The search route is
 * tzr_estimate_normals' (brute force below 4096 points, the hashed grid from there; debug flags 4194304 and 8388608);
 * both routes give the same bits.  Workspace as tzr_estimate_normals: the front end's buffers, so a retained solve
 * stays retained. */
int tzr_estimate_color_gradients(tzr_ctx* ctx, const float* pts, int n, const float* normals, const float* colors,
                                 double radius, double* grad_out);

/* B clouds: entry b of pts, normals, colors and grad_out as the single call's with n[b] points (every entry required).
 * status (may be NULL): B entries, TZR_OK each (no neighbourhood is too large).  TZR_ERR_TOO_LARGE when the batch holds
 * more than 2^31 - 1 points.  Per cloud, the output is bit-identical to tzr_estimate_color_gradients on that cloud
 * alone. */
int tzr_estimate_color_gradients_batch(tzr_ctx* ctx, int B, const int32_t* n, const float* const* pts,
                                       const float* const* normals, const float* const* colors, double radius,
                                       double* const* grad_out, int32_t* status);

/* B ragged problems: tzr_icp_point_to_plane_batch's arguments plus src_colors (B entries, entry b ns[b] x 3 floats),
 * dst_colors (B entries, entry b nd[b] x 3 floats), lambda_geometric and kernel (NULL: no kernel; otherwise checked as
 * tzr_icp_point_to_plane_robust_batch checks it).  A NULL array or entry is TZR_ERR_INVALID_ARG.  Per problem, every
 * output is bit-identical to tzr_icp_colored on that problem alone. */
int tzr_icp_colored_batch(tzr_ctx* ctx, const tzr_icp_params* params, int B, const int32_t* ns,
                          const float* const* src, const int32_t* nd, const float* const* dst,
                          const float* const* dst_normals, const tzr_similarity* init, tzr_icp_result* results,
                          int32_t* const* corr, const float* const* src_colors, const float* const* dst_colors,
                          double lambda_geometric, const tzr_robust_kernel* kernel);

/* One problem: tzr_icp_point_to_plane's arguments plus src_colors (ns x 3 floats), dst_colors (nd x 3 floats),
 * lambda_geometric and kernel (may be NULL).  This is tzr_icp_colored_batch with B = 1. */
int tzr_icp_colored(tzr_ctx* ctx, const tzr_icp_params* params, const float* src, int ns, const float* dst, int nd,
                    const float* dst_normals, const tzr_similarity* init, tzr_icp_result* result, int32_t* corr,
                    const float* src_colors, const float* dst_colors, double lambda_geometric,
                    const tzr_robust_kernel* kernel);

/* tzr_register_cloud_pairs_icp with coloured ICP: the same arguments plus colors, lambda_geometric and kernel, and the
 * same outputs, except that each refined record is coloured ICP (DESIGN.md §3.18).
 *   - Arguments, all checked before any device work: colors (n_clouds entries, entry c n[c] x 3 floats aligned with
 *     pts[c]; a NULL array or entry is TZR_ERR_INVALID_ARG); lambda_geometric (non-finite: TZR_ERR_INVALID_ARG; outside
 *     [0, 1]: 0.968, as tzr_icp_colored_batch); kernel (NULL: L2; otherwise checked as tzr_icp_colored_batch checks it).
 *   - Solve outputs: solutions, status, problem_index, correspondences, cliques, global scales and the retained solve are
 *     tzr_register_cloud_pairs' bit for bit.
 *   - Refinement: each pair p whose solve succeeded with a valid, finite record gets coloured ICP of cloud
 *     pair_clouds[2p] onto cloud pair_clouds[2p + 1], seeded on the device from its record, its scale held fixed.  The
 *     target normals are the call's own FPFH stage's (normal_search_radius, viewpoint at the origin); the target
 *     gradients are taken at 2 max_correspondence_distance, as RegistrationColoredICP takes them.  Each refined record
 *     is bit-identical to tzr_icp_colored_batch on that pair, with the two clouds and their colours,
 *     tzr_estimate_normals_batch(fparams->normal_search_radius) of the target, the pair's solution as init, the same
 *     lambda_geometric and the same kernel.  A pair that is not refined gets a zeroed record.
 *   - Gradients: one batched pass over every cloud of the call (tzr_estimate_color_gradients_batch at that radius, the
 *     descriptor stage's route), so each cloud's gradients are computed once however many pairs name it as target.
 *   - With lambda_geometric = 1 every output equals tzr_register_cloud_pairs_icp_point_to_plane (no kernel) and
 *     tzr_register_cloud_pairs_icp_robust with method 1 and the same kernel, bit for bit.
 * Launches: tzr_register_cloud_pairs_icp_point_to_plane's, plus, when some pair was solved, the gradient pass (1, + 4
 * when some cloud of the call has 4096 points or more, or under debug flag 8388608), whatever P.  Like
 * tzr_register_cloud_pairs this is a solve entry: tzr_last_inliers, tzr_last_graph and tzr_certify_last_solve see its
 * solve, which the refinement does not touch. */
int tzr_register_cloud_pairs_icp_colored(tzr_ctx* ctx, const tzr_frontend_params* fparams, const tzr_params* params,
                                         int n_clouds, const int32_t* n, const float* const* pts, int P,
                                         const int32_t* pair_clouds, const uint64_t* tuple_seeds,
                                         tzr_solution* solutions, int32_t* status, int32_t* problem_index,
                                         int64_t* n_corr, int32_t* const* corr, int32_t* const* cliques,
                                         float* global_scale, const tzr_icp_params* icp, const float* const* colors,
                                         double lambda_geometric, const tzr_robust_kernel* kernel,
                                         tzr_icp_result* icp_results);

/* ---- multiway registration: information matrices ------------------------------------------------------------
 * Open3D's GetInformationMatrixFromPointClouds(source, target, max_correspondence_distance, T) for many pairs at once,
 * defined here as follows (DESIGN.md §3.16):
 *   - Inputs: source x (ns float xyz), target y (nd float xyz), a similarity T = (s, R, t) with s held as tzr_icp holds it
 *     (finite, > 0; R and t finite), and one distance r for the call (finite and > 0, else TZR_ERR_INVALID_ARG).
 *   - Correspondences: exactly tzr_icp's at T: p_i = s (R x_i) + t, the nearest target with d^2 < r^2, the lowest target
 *     index on ties, brute force below 1024 target points and the hashed grid from there (debug flags 33554432 and
 *     67108864 force either route; both give the same correspondences).
 *   - Sum: each correspondence (i, j), with q = y_j = (x, y, z) the target point, adds G^T G with G = [-[q]x | I] (3 x 6,
 *     ordering (omega, tau)), rows (0, z, -y, 1, 0, 0), (-z, 0, x, 0, 1, 0), (y, -x, 0, 0, 0, 1).  Each of the 21 upper
 *     entries (a, b) is ((G(0,a) G(0,b) + G(1,a) G(1,b)) + G(2,a) G(2,b)) in IEEE float64 with no FMA contraction, summed
 *     in tzr_icp's chunk order (chunk k holds source points [256 k, 256 k + 256), a butterfly inside each warp, the
 *     warps in order; the chunks by lane k mod 32, then a butterfly).  Lambda(5,5) is therefore the correspondence count.
 *   - Outputs: Lambda as 36 doubles (row-major, mirrored, so symmetric bit for bit) and the count.
 * Host pointers, synchronous.  Launches: 3 (+ 4 for the grid build when some target has at least 1024 points), whatever
 * B.  Workspace: tzr_icp's own, so a retained solve stays retained. */
int tzr_information_matrix(tzr_ctx* ctx, const float* src, int ns, const float* dst, int nd,
                           const tzr_similarity* transform, double max_correspondence_distance, double* information,
                           int32_t* count);

/* B ragged pairs: pair b has ns[b] >= 1 source points at src[b], nd[b] >= 1 target points at dst[b] and its transform
 * at transforms[b].  information: B x 36 doubles; counts (may be NULL): B.  Per pair, both outputs are bit-identical to
 * tzr_information_matrix on that pair alone.  TZR_ERR_TOO_LARGE when the sources or targets exceed 2^31 - 1 points. */
int tzr_information_matrix_batch(tzr_ctx* ctx, int B, const int32_t* ns, const float* const* src, const int32_t* nd,
                                 const float* const* dst, const tzr_similarity* transforms,
                                 double max_correspondence_distance, double* information, int32_t* counts);

/* ---- refining registrations coarse to fine: multi-scale ICP -------------------------------------------------------
 * Open3D's multi-scale refinement (the coloured-ICP tutorial's schedule, the reconstruction system's multiscale_icp) for
 * many cloud pairs in one call, defined here as follows (DESIGN.md §3.19):
 *   - Methods: TZR_ICP_* below, the `method` values of the chained robust entries plus 3 for coloured ICP.
 *   - Clouds and pairs: n_clouds clouds (n[c] >= 1 float xyz points at pts[c]; colors[c], n[c] x 3 floats, for
 *     TZR_ICP_COLORED only, where colors and every entry are required) and P pairs in tzr_register_cloud_pairs'
 *     convention: pair p refines cloud pair_clouds[2p] (source) onto cloud pair_clouds[2p + 1] (target), starting from
 *     init[p], its scale held fixed throughout.  A cloud named by several pairs is downsampled, and gets its normals and
 *     gradients, once per scale.
 *   - The chain it equals: scale s's record of pair p is bit-identical to this chain of public calls:
 *       1. tzr_voxel_downsample_batch (tzr_voxel_downsample_colors_batch for TZR_ICP_COLORED) of the cloud table at
 *          scales[s].voxel_size; skipped when the size is 0 (the clouds as given).
 *       2. tzr_estimate_normals_batch of those clouds at scales[s].normal_search_radius (point-to-plane, generalized and
 *          coloured only).
 *       3. The method's tzr_icp_*_batch (tzr_icp_batch, tzr_icp_point_to_plane(_robust)_batch,
 *          tzr_icp_generalized(_robust)_batch with epsilon, tzr_icp_colored_batch with lambda_geometric) on the pair's
 *          two clouds from steps 1 and 2, with scales[s]'s distance and criteria and the same kernel.  The seed is init[p]
 *          at s = 0 and the transform of pair p's record at s - 1 otherwise.
 *   - information (P x 36 doubles, may be NULL) and info_counts (P, may be NULL), each on its own:
 *     tzr_information_matrix_batch on the last scale's pair at its final transform and that scale's
 *     max_correspondence_distance (what the reconstruction system's multiscale_icp returns); zero for a pair not refined
 *     at the last scale.  Either one given runs the information pass.
 *   - colors is read for TZR_ICP_COLORED only (NULL or anything for the other methods).
 *   - Arguments, all checked before any device work (TZR_ERR_INVALID_ARG): method outside 0 ... 3; S < 1; a scale whose
 *     voxel_size is not finite and >= 0, whose max_correspondence_distance is not finite and > 0, whose
 *     normal_search_radius is not finite and > 0 for a method with normals, whose max_iteration is < 0 or whose criteria
 *     are NaN; a pair index outside the cloud table; a seed that tzr_icp refuses; a kernel with TZR_ICP_POINT_TO_POINT,
 *     or one tzr_icp_point_to_plane_robust_batch refuses; epsilon as tzr_icp_generalized_batch checks it (method 2 only);
 *     lambda_geometric as tzr_icp_colored_batch handles it (method 3 only: non-finite refused, outside [0, 1] 0.968).
 *   - Empty cloud at a scale: a cloud with no finite point has no voxel; a pair that uses a cloud with n_down 0 is not
 *     refined at that scale, and its record carries its pose in (transform as it entered the scale; fitness, rmse,
 *     iterations, correspondences and converged 0).
 *   - n_down (n_clouds x S, cloud-major, may be NULL): each cloud's points at each scale (n[c] where voxel_size is 0).
 *   - status (n_clouds x S, cloud-major, may be NULL): TZR_OK, or TZR_ERR_TOO_LARGE where
 *       - the cloud's voxel grid fails Open3D's INT_MAX check or the 2^62-cell limit.  This is found before any normals
 *         or ICP run; then nothing else runs, every record and information matrix is zero, and the call returns
 *         TZR_ERR_TOO_LARGE;
 *       - a point of the cloud has more than 4096 neighbours at that scale's normal radius.  This is found at the end of
 *         the call: the records (and information) of every pair that uses the cloud at that scale or later are zeroed,
 *         every other record is still the chain's, and the call returns TZR_ERR_TOO_LARGE.
 * Device flow: one upload of the clouds, every voxel scale back to back, one read-back of the voxel tables (the call's
 * planning synchronisation, only when some voxel_size > 0), one upload of every scale's tables, then everything else
 * enqueued and one read-back at the end: at most two host synchronisations whatever S and P.
 * Launches, per scale: 10 when voxel_size > 0; for the methods with normals the normals pass, 1 (+ 4 when some cloud of
 * the scale has 4096 points or more); 1 pose store; and when some pair is refined at the scale, 1 pose load and the
 * method's tzr_icp_*_batch launches (2 + 4 max_iteration, + 4 when some cloud of the scale has 1024 points or more;
 * coloured: + 1 for the gradient pass, + 4 more when some cloud of the scale has 4096 points or more).  With
 * information or info_counts, 4 more after the last scale when some pair is refined there.  The debug flags of
 * tzr_estimate_normals (4194304, 8388608) and tzr_icp (33554432, 67108864) force the routes here too.  Not a solve
 * entry: the workspace is tzr_icp's, so a retained solve stays retained. */
#define TZR_ICP_POINT_TO_POINT 0
#define TZR_ICP_POINT_TO_PLANE 1
#define TZR_ICP_GENERALIZED 2
#define TZR_ICP_COLORED 3

typedef struct tzr_icp_scale {
  double voxel_size;                   /* > 0: voxel-downsample every cloud at this size; 0: the clouds as given */
  double max_correspondence_distance;  /* finite, > 0 */
  double normal_search_radius;         /* finite, > 0 for the methods that use normals (Open3D: 2 voxel_size) */
  double relative_fitness, relative_rmse;
  int32_t max_iteration;               /* >= 0 */
  int32_t reserved;
} tzr_icp_scale;

/* results: P x S records, pair-major (pair p's record of scale s at p * S + s). */
int tzr_icp_multiscale_batch(tzr_ctx* ctx, int method, int S, const tzr_icp_scale* scales, int n_clouds,
                             const int32_t* n, const float* const* pts, const float* const* colors, int P,
                             const int32_t* pair_clouds, const tzr_similarity* init, double epsilon,
                             double lambda_geometric, const tzr_robust_kernel* kernel, tzr_icp_result* results,
                             int32_t* n_down, int32_t* status, double* information, int32_t* info_counts);

/* ---- multiway registration: robust pose graph ------------------------------------------------------------------
 * The global step of Open3D's multiway registration (global_optimization over a PoseGraph), with GNC-TLS pruning the
 * uncertain edges instead of Open3D's line process.  One graph per call, defined here as follows (DESIGN.md §3.16):
 *   - Nodes: K poses T_k = (R_k, t_k), 2 <= K <= 1024 (K > 1024 is TZR_ERR_TOO_LARGE); T_k maps cloud k into the world
 *     frame.  The node reference_node is held fixed.
 *   - Edges: E >= 1 edges e = (s, d, T_sd, Lambda_e, uncertain_e) in the cloud-pair orientation p_d ~ T_sd p_s, so a
 *     consistent graph has T_s = T_d T_sd.  T_sd is rigid: its scale is ignored, and a rotation that is not orthonormal
 *     to 1e-6 (max |R^T R - I|), has a determinant below 0, or any non-finite entry is TZR_ERR_INVALID_ARG.  Lambda_e: 36
 *     doubles, row-major, finite, Lambda(5,5) >= 0 (tzr_information_matrix's).  s = d is allowed (the edge adds a
 *     constant to the cost).  An edge with Lambda(5,5) = 0 carries no information: it adds nothing and connects nothing.
 *   - Connectivity: if the edges with s != d and Lambda(5,5) > 0 do not connect every node to the reference node, the
 *     call returns TZR_ERR_INVALID_ARG and writes nothing.
 *   - Residual: E = T_d^-1 T_s T_sd^-1 and e = (omega, tau) with omega = log R_E, tau = t_E.  The log: v = vee(R - R^T)
 *     / 2, c = (tr R - 1) / 2, theta = atan2(|v|, c); theta < 1e-5: omega = (1 + theta^2 / 6) v (small-angle branch);
 *     c < -0.9: omega = theta a with a the column of the symmetric part (R + R^T) / 2 - c I of largest diagonal,
 *     normalised, with the sign of v (near pi); otherwise omega = (theta / |v|) v.
 *   - Linearisation: left perturbations T_k <- Exp(delta_k) T_k, delta = (omega, tau), Exp the SE(3) exponential (R =
 *     Rodrigues(omega), t = V(omega) tau); Jacobians J_s = Ad(T_d^-1), J_d = -Ad(T_d^-1), Ad(T) = [[R, 0], [[t]x R, R]].
 *   - Normalised residual: r-bar_e = e^T Lambda_e e / (c^2 Lambda_e(5,5)) with c = max_correspondence_distance (0 where
 *     Lambda_e(5,5) = 0): an edge is an outlier when it moves its overlap by more than c RMS.
 *   - GNC-TLS on the uncertain edges (the rotation stage's schedule): weights start at 1; for i < max_iterations: the
 *     inner solve with the current weights; if no edge is uncertain, stop; at i = 0, mu = 1 / (2 max r-bar - 1) over
 *     the uncertain edges, and stop unless mu is finite and positive (2 max r-bar - 1 <= 0, every uncertain edge an
 *     inlier, stops with weights 1; so does max r-bar = +inf); then, per uncertain edge, w = 0 where r-bar >= (mu + 1) / mu, 1 where
 *     r-bar <= mu / (mu + 1), sqrt(mu (mu + 1) / r-bar) - mu between; cost = sum over the uncertain edges of the
 *     previous w times r-bar; mu <- mu * gnc_factor; stop when |cost - previous cost| < cost_threshold (previous cost
 *     +inf at i = 0).  Certain edges keep weight 1.  inlier = w >= 0.5.
 *   - Inner solve: Levenberg-Marquardt on F = sum_e w_e e^T Lambda_e e over the K - 1 free nodes, n = 6 (K - 1) unknowns.
 *     H = sum w J^T Lambda J and g = sum w J^T Lambda e, assembled per 6 x 6 block in ascending edge index; damping
 *     H_ii <- H_ii + lambda (H_ii + 1), lambda = 1e-4 at the start of every inner solve (the additive part keeps a
 *     node whose every edge has weight 0 solvable: its step is then 0 and the other nodes still move); delta solves H delta = -g by Cholesky
 *     (cuSOLVER potrf / potrs).  Per iteration, with F' the cost at the candidate poses: if the factorisation failed
 *     (a non-positive pivot) or F' is not finite, reject: lambda <- 10 lambda, and stop once lambda > 1e8; else if
 *     |F - F'| <= 1e-10 F + 1e-24 c^2 sum_e Lambda_e(5,5), take the candidate when F' < F and stop; else if F' < F,
 *     accept and lambda <- lambda / 10; else reject as above.  At most max_inner_iterations iterations, all enqueued.
 *   - Initial poses: initial_poses (K, may be NULL; rigid and finite as the edges).  NULL: breadth-first from the
 *     reference node (identity), first over the certain edges, then over all edges (those with s != d and
 *     Lambda(5,5) > 0), each node's edges in ascending index, T_s = T_d T_sd or T_d = T_s T_sd^-1.
 * Outputs: poses (K, scale 1); per edge (each may be NULL): the final weight, the inlier mask and r-bar at the returned
 * poses; summary (may be NULL).  The returned poses come from the last inner solve, the weights from the GNC update
 * after it (as the rotation stage returns them).  Host pointers, synchronous; one host read-back per GNC iteration.
 * Launches: (3 + 4 max_inner_iterations) per GNC iteration, plus 2 cuSOLVER calls per inner iteration.  Workspace of
 * its own (n^2 doubles for H: about 301 MB at K = 1024), so a retained solve stays retained.  TZR_ERR_UNSUPPORTED when
 * cuSOLVER cannot be loaded. */
typedef struct tzr_pose_graph_params {
  double max_correspondence_distance;  /* c: no default; finite and > 0 */
  double gnc_factor;                   /* 1.4; > 1 */
  double cost_threshold;               /* 1e-6 */
  int32_t max_iterations;              /* 100 GNC iterations; >= 1 */
  int32_t max_inner_iterations;        /* 10 Levenberg-Marquardt iterations per GNC iteration; >= 1 */
  int32_t reference_node;              /* 0 */
  int32_t reserved;
} tzr_pose_graph_params;

typedef struct tzr_pose_graph_summary {
  int32_t iterations;        /* GNC iterations (inner solves) run */
  int32_t inner_iterations;  /* Levenberg-Marquardt iterations, summed over them */
  double cost;               /* F of the last inner solve at the returned poses */
} tzr_pose_graph_summary;

/* max_correspondence_distance 0 (the caller must set it), gnc_factor 1.4, cost_threshold 1e-6, max_iterations 100,
 * max_inner_iterations 10, reference_node 0. */
void tzr_pose_graph_params_default(tzr_pose_graph_params* p);

/* edges: E x 2 (s, d); edge_transforms, information (E x 36): per edge; uncertain (E, may be NULL: every edge certain). */
int tzr_pose_graph_optimize(tzr_ctx* ctx, const tzr_pose_graph_params* params, int K, int E, const int32_t* edges,
                            const tzr_similarity* edge_transforms, const double* information, const int32_t* uncertain,
                            const tzr_similarity* initial_poses, tzr_similarity* poses, double* weights,
                            uint8_t* inlier_mask, double* residuals, tzr_pose_graph_summary* summary);

/* tzr_register_cloud_pairs_icp_point_to_plane (same arguments, same outputs bit for bit), then the information matrix
 * of every refined pair (solved, valid and finite record) at its ICP transform and the ICP's
 * max_correspondence_distance, from the clouds and transforms already on the device (no upload), then
 * tzr_pose_graph_optimize over the n_clouds clouds with one edge per refined pair (s, d) = pair_clouds[p], T_sd its ICP
 * transform, Lambda its information matrix and uncertain[p] (P entries, required).  params->estimate_scaling = 1 is
 * TZR_ERR_INVALID_ARG (the pose graph is rigid).  Outputs: information (P x 36) and info_counts (P), zeroed for a pair
 * that was not refined; edge_weights (P doubles) and edge_mask (P bytes), 0 for a pair that is not an edge; poses
 * (n_clouds); pg_summary (may be NULL); *pg_status receives the pose graph's status (TZR_OK, or its error, e.g.
 * TZR_ERR_INVALID_ARG for a disconnected graph; poses, weights and masks are then zero).  Every output equals
 * tzr_register_cloud_pairs_icp_point_to_plane, then tzr_information_matrix_batch over the refined pairs in pair order,
 * then tzr_pose_graph_optimize over them, bit for bit.  Returns what the registration returns.  A solve entry:
 * tzr_last_inliers and tzr_certify_last_solve see its solve. */
int tzr_register_cloud_pairs_multiway(tzr_ctx* ctx, const tzr_frontend_params* fparams, const tzr_params* params,
                                      int n_clouds, const int32_t* n, const float* const* pts, int P,
                                      const int32_t* pair_clouds, const uint64_t* tuple_seeds,
                                      tzr_solution* solutions, int32_t* status, int32_t* problem_index,
                                      int64_t* n_corr, int32_t* const* corr, int32_t* const* cliques,
                                      float* global_scale, const tzr_icp_params* icp, tzr_icp_result* icp_results,
                                      const int32_t* uncertain, const tzr_pose_graph_params* pg, double* information,
                                      int32_t* info_counts, double* edge_weights, uint8_t* edge_mask,
                                      tzr_similarity* poses, tzr_pose_graph_summary* pg_summary, int32_t* pg_status);

/* tzr_register_cloud_pairs_multiway with coloured ICP: its arguments plus colors, lambda_geometric and kernel (checked as
 * tzr_register_cloud_pairs_icp_colored checks them, before any device work).  It runs
 * tzr_register_cloud_pairs_icp_colored, then the information matrix of every refined pair at its coloured ICP
 * transform and max_correspondence_distance (geometric only, as Open3D's GetInformationMatrixFromPointClouds: the
 * colours play no part), then the GNC-TLS pose graph, all in one call as tzr_register_cloud_pairs_multiway.  Every
 * output equals tzr_register_cloud_pairs_icp_colored, then tzr_information_matrix_batch over the refined pairs in pair
 * order, then tzr_pose_graph_optimize over them, bit for bit; with lambda_geometric = 1 and no kernel it equals
 * tzr_register_cloud_pairs_multiway bit for bit.  params->estimate_scaling = 1 is TZR_ERR_INVALID_ARG. */
int tzr_register_cloud_pairs_multiway_colored(
    tzr_ctx* ctx, const tzr_frontend_params* fparams, const tzr_params* params, int n_clouds, const int32_t* n,
    const float* const* pts, int P, const int32_t* pair_clouds, const uint64_t* tuple_seeds, tzr_solution* solutions,
    int32_t* status, int32_t* problem_index, int64_t* n_corr, int32_t* const* corr, int32_t* const* cliques,
    float* global_scale, const tzr_icp_params* icp, const float* const* colors, double lambda_geometric,
    const tzr_robust_kernel* kernel, tzr_icp_result* icp_results, const int32_t* uncertain,
    const tzr_pose_graph_params* pg, double* information, int32_t* info_counts, double* edge_weights,
    uint8_t* edge_mask, tzr_similarity* poses, tzr_pose_graph_summary* pg_summary, int32_t* pg_status);

/* ---- downsampling point clouds: voxel-grid averaging ----------------------------------------------------------
 * The first step of the reference's FPFH + TEASER++ + ICP tutorial (voxel_down_sample on both raw scans), for many
 * clouds at once.  Open3D's PointCloud::VoxelDownSample, points only, with a defined order.  Per cloud, all arithmetic
 * is IEEE float64 with no FMA contraction (DESIGN.md §3.12):
 *   - Inputs: n float xyz points, read exactly as float64, and one voxel_size v for the whole call; v must be finite
 *     and > 0 (anything else is TZR_ERR_INVALID_ARG, as Open3D's voxel_size <= 0 check).
 *   - Finite points only: a point with any non-finite coordinate belongs to no voxel (voxel_of -1) and does not affect
 *     the bounds.  (Open3D's result is undefined there.)
 *   - Bounds: min and max are the component-wise bounds over the finite points; vmin = min - (v * 0.5) and
 *     vmax = max + (v * 0.5).
 *   - Too small a voxel: a cloud with v * INT_MAX < max_k (vmax_k - vmin_k) (Open3D's check) gets TZR_ERR_TOO_LARGE.
 *   - Voxel index: i_k = (int) floor((p_k - vmin_k) / v), a division as Open3D writes it (not a product with 1/v,
 *     which gives a different voxel on some voxel edges).
 *   - Grid-size limit: points are grouped by the exact triple (i_x, i_y, i_z), packed into one 64-bit key; a cloud
 *     whose per-axis voxel counts (i_k of its largest finite coordinate, + 1) multiply to more than 2^62 gets
 *     TZR_ERR_TOO_LARGE.
 *   - Output point: each voxel's point is the sum of its member points, added one at a time in ascending input index
 *     starting from 0.0 (Open3D's AccumulatedPoint), divided by (double) count, the mean rounded once to float.
 *   - Output order: voxels ordered by their first (lowest-index) member.  (Open3D's order is its unordered_map's.)  A
 *     cloud already sparser than the grid comes back unchanged, in the same order.
 *   - Normals are not carried; colours are, by tzr_voxel_downsample_colors(_batch) below.
 * Cost: a voxel of k points costs one thread k dependent additions (the bit-exact sequential sum), so one voxel holding
 * a whole cloud is correct but slow.  Host pointers, synchronous; 10 kernel launches per call (CUB calls counted as
 * one), whatever B.  These calls are not solve entries: they use a workspace of their own, so a retained solve
 * (tzr_last_inliers, tzr_last_graph, tzr_certify_last_solve) stays retained across them. */

/* One cloud of n >= 1 points: tzr_voxel_downsample_batch with B = 1 (its status is the return value). */
int tzr_voxel_downsample(tzr_ctx* ctx, const float* pts, int n, double voxel_size,
                         float* pts_out, int32_t* n_out, int32_t* voxel_of);

/* B clouds: cloud b has n[b] >= 1 points at pts[b].  pts_out[b]: room for n[b] x 3 floats (always enough), receives
 * n_out[b] rows (n_out: B entries).  voxel_of (may be NULL or hold NULL entries): voxel_of[b][i] is the output row of
 * input point i, or -1 (Open3D's VoxelDownSampleAndTrace, in a form that carries labels or colours).  status (may be
 * NULL; B entries): TZR_OK, or TZR_ERR_TOO_LARGE for a cloud whose grid is too large; such a cloud gets n_out = 0 and
 * voxel_of -1, every other cloud's outputs are still written, and the call returns TZR_ERR_TOO_LARGE.  A cloud with no
 * finite point gets n_out = 0 and status TZR_OK.  Per cloud, every output is bit-identical to the call on that cloud
 * alone.  TZR_ERR_TOO_LARGE when the batch holds more than 2^31 - 1 points; TZR_ERR_ALLOC when the workspace does not
 * fit the device (tzr_last_error names the size). */
int tzr_voxel_downsample_batch(tzr_ctx* ctx, int B, const int32_t* n, const float* const* pts, double voxel_size,
                               float* const* pts_out, int32_t* n_out, int32_t* const* voxel_of, int32_t* status);

/* Voxel downsampling with colours (coloured ICP's input, DESIGN.md §3.17): tzr_voxel_downsample(_batch)'s arguments
 * plus colors (n x 3 floats per cloud, read as float64) and colors_out (room for n x 3 floats per cloud; receives
 * n_out rows).  Each voxel's colour is the sum of its members' colours, added one at a time in ascending input index
 * starting from 0.0, divided by (double) count and rounded once to float, exactly like its point.  Points, n_out,
 * voxel_of and status are bit-identical to tzr_voxel_downsample(_batch)'s; a NULL colors or colors_out (or entry) is
 * TZR_ERR_INVALID_ARG.  Launches and workspace as tzr_voxel_downsample(_batch). */
int tzr_voxel_downsample_colors(tzr_ctx* ctx, const float* pts, int n, double voxel_size, float* pts_out,
                                int32_t* n_out, int32_t* voxel_of, const float* colors, float* colors_out);
int tzr_voxel_downsample_colors_batch(tzr_ctx* ctx, int B, const int32_t* n, const float* const* pts,
                                      double voxel_size, float* const* pts_out, int32_t* n_out,
                                      int32_t* const* voxel_of, int32_t* status, const float* const* colors,
                                      float* const* colors_out);

/* Graph-stage timing of the most recent tzr_solve_batch_dev, in milliseconds, measured with CUDA
 * events on the context's stream (for the roofline line in bench.py). Requires a prior synchronize. */
int tzr_last_stage_ms(tzr_ctx* ctx, double* prep_ms, double* graph_ms, double* clique_ms, double* rot_trans_ms);
/* Stage-timing log: while enabled the context keeps the CUDA events of EVERY pipeline call instead of re-using
 * them, so a benchmark loop can run without a host synchronisation per step; tzr_ctx_stage_log_read synchronises
 * once, returns the sums {prep, graph, clique, rot+trans} in ms over all calls since the last read (or enable) and
 * their count, and clears the log. */
int tzr_ctx_stage_log(tzr_ctx* ctx, int enable);
int tzr_ctx_stage_log_read(tzr_ctx* ctx, double* sums_ms4, int32_t* n_calls);

/* ---- multi-GPU ------------------------------------------------------------------------------
 * tzr_solve_batch over several devices of one node from a single host call (SURVEY §8e: independent problems,
 * no exchange step, no collective): the library keeps one context per device, cuts the batch into contiguous
 * shards balanced by sum n_b^2 and drives each shard from its own host thread.  devices == NULL or n_devices <= 0:
 * every visible device.  Same argument meaning as tzr_solve_batch; thread-safe (calls are serialised). */
int tzr_solve_batch_multi(const int32_t* devices, int n_devices, const tzr_params* params, int B, const int32_t* n,
                          const double* const* src, const double* const* dst, tzr_solution* solutions,
                          int32_t* cliques, int max_n);

/* Debug/verification switches: bit 0 (1) = force the pure-FP64 graph predicate (no FP32 filter),
 * bit 1 (2) = verify the FP32 / tensor-core filter against FP64 for every pair and count mismatches,
 * bit 2 (4) = count exact re-checks and clique search nodes, bit 8 (256) = degrees by a separate pass,
 * bit 10 (1024) = build the graph with the tensor-core kernel (wgmma Gram norms; bit-identical to the default CUDA-core
 * kernel: DESIGN.md 3.1; uniform batches only: the size classes of a ragged batch run the default kernel), bit 9 (512) = the square-root interval test for every problem (no Gram test, no tensor-core
 * kernel; bit-identical), bit 11 (2048) = the one-MUFU
 * CUDA-core variant (graph_strip3_kernel; bit-identical; uniform batches only, like bit 10), bit 13 (8192) = exact clique
 * search without the singleton-class path of the colouring (A/B), bit 12 (4096) = without the block colour bound (only
 * present in builds with -DTZR_BLOCK_BOUND), bit 14 (16384) = cap the graph kernels' re-check queue at 64 entries (the
 * buffer keeps its full size), so that the queue-full path (pairs evaluated in place by the graph kernel) runs at test
 * sizes; bit-identical, bit 15 (32768) = a first exact clique pass of 1 ns (the second pass keeps the caller's whole
 * budget), so that every problem that reaches the exact search goes through the vertex-cover LP kernel regardless of
 * machine load (a problem whose whole first pass fits inside one %globaltimer tick, about 1 us or less, would still
 * finish in it), bit 16 (65536) = an exact-search stack of 8 levels, so that the depth cap (result not proven) is
 * reachable at test sizes, bit 17 (131072) = one exact pass with the caller's whole budget instead of 50 ms + LP bound
 * + second pass, so that whether a canonical enumeration finishes does not depend on the wall clock (bit 15 wins when
 * both are set), bit 18 (262144) = the unknown-scale stage and tzr_scalar_tls through the large path (radix sort +
 * tiled scans) at every size instead of the bitonic sort + sequential sweep below 257 points, bit 19 (524288) = the
 * large clique route at every n (tzr_ctx_clique_route), so that the two routes can be compared on the same graphs,
 * bit 20 (1048576) = cap the large route's compacted core at 64 vertices instead of 32768, so that its "core too large"
 * outcome is reachable at test sizes, bit 21 (2097152) = tzr_certify_batch loops cusolverDnDsyevd over the active
 * problems instead of one cusolverDnXsyevBatched call, so that the two eigen routes can be compared on the same batch,
 * bit 22 (4194304) = tzr_compute_fpfh(_batch) searches every cloud's radius neighbours by brute force, bit 23
 * (8388608) = through the hashed grid at any cloud size (DESIGN.md 3.7; a cloud the grid cannot index still falls back
 * to brute force), so that the two routes can be compared on one input; bit 22 wins when both are set, bit 24
 * (16777216) = a ragged batch forms one size class wherever the large-route and scale-path rules allow, however far
 * apart its sizes are, so that tests can pad n = 2 to n = 4000 in one device batch, bit 25 (33554432) = tzr_icp(_batch)
 * and tzr_icp_point_to_plane(_batch) and tzr_icp_generalized(_batch) (and their robust batch entries)
 * searches every target by brute force, bit 26 (67108864) = through the hashed grid at any target size (a target the
 * grid cannot index still falls back to brute force), so that the two routes can be compared on one input; bit 25 wins
 * when both are set, bit 27 (134217728) = the default graph kernel's Gram test in its two-slope form on the unscaled float
 * copies instead of the single-slope form in units of 2 beta (DESIGN.md 3.1; bit-identical; a same-build A/B switch),
 * bits 28 to 31 = a 4-bit field L: 0 lets the default graph kernel choose its strip length from the batch and the SM
 * count (4 or 6 blocks of 128 columns), L = 1 ... 15 forces strips of L blocks in every instance of that kernel
 * (production, verifying, separate degree pass, ragged size class, two-slope form; bit-identical), so that tests reach
 * every strip length whatever the batch and the device; the opt-in kernels of bits 3 to 7, 10 and 11 ignore it.
 * Bits 15 to 26 and 28 to 31 change host code only; bit 27 changes device code. */
int tzr_ctx_set_flags(tzr_ctx* ctx, uint32_t flags);
/* Strip length (blocks of 128 columns) of the default graph kernel's most recent launch on this context (the last size
 * class or sub-chunk of a batch); 0 before any graph build, or when that build ran another kernel (debug bits 3 to 7
 * and 11). */
int tzr_ctx_last_strip_blocks(const tzr_ctx* ctx);
/* The default graph kernel's strip order over nt row blocks of 128 points, as the device decodes it, for strips of L
 * blocks: I[p] (row block) and J0[p] (first column block) of strip p = 0 ... count - 1, strips numbered from row block 0
 * down, each row block's strips left to right.  Host-only, needs no device; I and J0 may be NULL.  Returns the count,
 * or TZR_ERR_INVALID_ARG unless 1 <= nt <= 512 and 1 <= L <= 15. */
int tzr_graph_strip_schedule(int nt, int L, int32_t* I, int32_t* J0);
int64_t tzr_ctx_filter_mismatches(tzr_ctx* ctx);
/* Number of pairs of the most recent graph build that needed the exact FP64 re-check. */
int64_t tzr_ctx_filter_rechecks(tzr_ctx* ctx);
/* Debug counters of the most recent call (flag bit 2 set): [0] filter mismatches, [1] filter re-checks, [2] clique
 * search nodes, [3] reduce rounds, [4] vertices scanned by reduce rounds, [5] colourings, [6] vertices coloured,
 * [7] problems whose graph was built by the tensor-core kernel, [8]-[10] clock cycles of the exact search in the root
 * colour bound / degree rules / colourings, [11] slowest root (ns << 16 | vertex), [12] summed root time (ns),
 * [13] roots above 1 ms, [14] roots closed by the block colour bound, [15] problems whose graph the default CUDA-core
 * kernel built with the Gram-form test (not the interval test, the tensor-core kernel or the flag-2048 kernel). */
int tzr_ctx_debug_counters(tzr_ctx* ctx, int64_t* out16);

#ifdef __cplusplus
}
#endif
#endif /* TEASER_B200_H_ */
