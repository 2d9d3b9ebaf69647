// teaser::RobustRegistrationSolver — the drop-in C++ surface of the GPU path.
//
// Source compatible with the reference header teaser/include/teaser/registration.h (class and member names,
// Params fields and defaults, enum values, getters), but every computation is forwarded to the C-ABI
// (include/teaser_b200.h).  There is no CPU implementation behind this class: without a CUDA device the
// constructor's first use throws std::runtime_error.
//
// Differences from the reference, all deliberate (SURVEY.md §2 quirks):
//   Q1  Params are honoured (the reference never assigns params_ and silently runs PMC_EXACT + CHAIN).
//   Q2  a solver object may be reused: solve() resets per-call state (the reference compounds the rotation
//       noise bound and appends to rotation_inliers_ on a second call).
//   a16 O(N^2) getters (TIMs, maps, scale-inlier mask, adjacency list) are materialised lazily on first
//       access, never inside solve().
#pragma once

#include <cstdint>
#include <memory>
#include <stdexcept>
#include <tuple>
#include <utility>
#include <vector>

#if defined(__has_include)
#if __has_include(<Eigen/Core>)
#include <Eigen/Core>
#define TEASER_B200_HAVE_EIGEN 1
#endif
#endif
#ifndef TEASER_B200_HAVE_EIGEN
#include "teaser/eigen_lite.h"
#endif

#include "teaser/certification.h"
#include "teaser/geometry.h"
#include "teaser/graph.h"

struct tzr_ctx;

namespace teaser {

// teaser/include/teaser/registration.h:32-39
struct RegistrationSolution {
  bool valid = true;
  double scale = 1;
  Eigen::Vector3d translation;
  Eigen::Matrix3d rotation;
  EIGEN_MAKE_ALIGNED_OPERATOR_NEW
};

// Point-to-point ICP (teaser/icp.h, tzr_icp): the parameters and the result of PointToPointICP, declared here so that
// solveCloudPairs can refine its pairs.  Open3D's registration_icp distance and ICPConvergenceCriteria.
struct PointToPointICPParams {
  double max_correspondence_distance = 0;  // no default, as in Open3D: must be set (> 0)
  int max_iteration = 30;
  double relative_fitness = 1e-6;
  double relative_rmse = 1e-6;
};
// Generalized ICP (teaser/icp.h, tzr_icp_generalized): PointToPointICP's parameters plus Open3D's epsilon of the
// plane-to-plane covariances (finite, > 0).
struct GeneralizedICPParams : PointToPointICPParams {
  double epsilon = 1e-3;
};
// Coloured ICP (teaser/icp.h, tzr_icp_colored): PointToPointICP's parameters plus Open3D's lambda_geometric (outside
// [0, 1] it becomes 0.968; a non-finite value is refused).
struct ColoredICPParams : PointToPointICPParams {
  double lambda_geometric = 0.968;
};
// A robust kernel for point-to-plane and generalized ICP (tzr_robust_kernel, DESIGN.md §3.15): Open3D's L2Loss (the
// default, no weighting), L1Loss, HuberLoss(k), CauchyLoss(k), GMLoss(k) and TukeyLoss(k).  k must be finite and > 0 for
// Huber, Cauchy, GM and Tukey; it is ignored for L2 and L1.
struct RobustKernel {
  enum Type { kL2 = 0, kL1 = 1, kHuber = 2, kCauchy = 3, kGM = 4, kTukey = 5 };
  Type type = kL2;
  double k = 1.0;
  RobustKernel() = default;
  RobustKernel(Type type_, double k_ = 1.0) : type(type_), k(k_) {}
};
// The GNC-TLS pose graph of multiway registration (teaser/pose_graph.h, tzr_pose_graph_optimize): the distance c of
// the normalised residual, the GNC-TLS schedule, the inner Levenberg-Marquardt iterations and the fixed node.
struct PoseGraphParams {
  double max_correspondence_distance = 0;  // no default: must be set (> 0), normally the ICP distance
  double gnc_factor = 1.4;
  double cost_threshold = 1e-6;
  int max_iterations = 100;
  int max_inner_iterations = 10;
  int reference_node = 0;
};
struct PointToPointICPResult {
  RegistrationSolution solution;  // the refined transform; scale is the seed's, held fixed
  double fitness = 0;
  double inlier_rmse = 0;
  int iterations = 0;
  bool converged = false;
  std::vector<std::pair<int, int>> correspondences;  // final (source index, target index), ascending by source
  EIGEN_MAKE_ALIGNED_OPERATOR_NEW
};

using Mat3X = Eigen::Matrix<double, 3, Eigen::Dynamic>;
using BoolRow = Eigen::Matrix<bool, 1, Eigen::Dynamic>;
using Map2X = Eigen::Matrix<int, 2, Eigen::Dynamic>;

// registration.h:44-100
class AbstractScaleSolver {
 public:
  virtual ~AbstractScaleSolver() {}
  virtual void solveForScale(const Mat3X& src, const Mat3X& dst, double* scale, BoolRow* inliers) = 0;
};
class AbstractRotationSolver {
 public:
  virtual ~AbstractRotationSolver() {}
  virtual void solveForRotation(const Mat3X& src, const Mat3X& dst, Eigen::Matrix3d* rotation, BoolRow* inliers) = 0;
};
class AbstractTranslationSolver {
 public:
  virtual ~AbstractTranslationSolver() {}
  virtual void solveForTranslation(const Mat3X& src, const Mat3X& dst, Eigen::Vector3d* translation,
                                   BoolRow* inliers) = 0;
};

// registration.h:105-131 — forwards to tzr_scalar_tls
class ScalarTLSEstimator {
 public:
  ScalarTLSEstimator() = default;
  void estimate(const Eigen::RowVectorXd& X, const Eigen::RowVectorXd& ranges, double* estimate, BoolRow* inliers);
};

// registration.h:136-160
class TLSScaleSolver : public AbstractScaleSolver {
 public:
  TLSScaleSolver() = delete;
  explicit TLSScaleSolver(double noise_bound, double cbar2) : noise_bound_(noise_bound), cbar2_(cbar2) {}
  void solveForScale(const Mat3X& src, const Mat3X& dst, double* scale, BoolRow* inliers) override;
  double noise_bound() const { return noise_bound_; }
  double cbar2() const { return cbar2_; }

 private:
  double noise_bound_, cbar2_;
  ScalarTLSEstimator tls_estimator_;
};

// registration.h:167-187
class ScaleInliersSelector : public AbstractScaleSolver {
 public:
  ScaleInliersSelector() = delete;
  explicit ScaleInliersSelector(double noise_bound, double cbar2) : noise_bound_(noise_bound), cbar2_(cbar2) {}
  void solveForScale(const Mat3X& src, const Mat3X& dst, double* scale, BoolRow* inliers) override;

 private:
  double noise_bound_, cbar2_;
};

// registration.h:192-215 — forwards to tzr_tls_translation
class TLSTranslationSolver : public AbstractTranslationSolver {
 public:
  TLSTranslationSolver() = delete;
  explicit TLSTranslationSolver(double noise_bound, double cbar2) : noise_bound_(noise_bound), cbar2_(cbar2) {}
  void solveForTranslation(const Mat3X& src, const Mat3X& dst, Eigen::Vector3d* translation,
                           BoolRow* inliers) override;

 private:
  double noise_bound_, cbar2_;
};

// registration.h:220-247
class GNCRotationSolver : public AbstractRotationSolver {
 public:
  struct Params {
    size_t max_iterations;
    double cost_threshold;
    double gnc_factor;
    double noise_bound;
  };
  explicit GNCRotationSolver(Params params) : params_(params) {}
  Params getParams() { return params_; }
  void setParams(Params params) { params_ = params; }
  double getCostAtTermination() { return cost_; }

 protected:
  Params params_;
  double cost_ = 0;
};

// registration.h:257-278 — forwards to tzr_gnc_tls_rotation
class GNCTLSRotationSolver : public GNCRotationSolver {
 public:
  GNCTLSRotationSolver() = delete;
  explicit GNCTLSRotationSolver(Params params) : GNCRotationSolver(params) {}
  void solveForRotation(const Mat3X& src, const Mat3X& dst, Eigen::Matrix3d* rotation, BoolRow* inliers) override;
};

// registration.h:290-352 — FGR and Quatro (forward to tzr_rotation_solve; inside solve() they run fused on the device)
class FastGlobalRegistrationSolver : public GNCRotationSolver {
 public:
  FastGlobalRegistrationSolver() = delete;
  explicit FastGlobalRegistrationSolver(Params params) : GNCRotationSolver(params) {}
  void solveForRotation(const Mat3X& src, const Mat3X& dst, Eigen::Matrix3d* rotation, BoolRow* inliers) override;
};
class QuatroSolver : public GNCRotationSolver {
 public:
  QuatroSolver() = delete;
  explicit QuatroSolver(Params params) : GNCRotationSolver(params) {}
  void solveForRotation(const Mat3X& src, const Mat3X& dst, Eigen::Matrix3d* rotation, BoolRow* inliers) override;
};

// registration.h:361-957
class RobustRegistrationSolver {
 public:
  EIGEN_MAKE_ALIGNED_OPERATOR_NEW

  enum class ROTATION_ESTIMATION_ALGORITHM { GNC_TLS = 0, FGR = 1, QUATRO = 2 };
  enum class INLIER_SELECTION_MODE { PMC_EXACT = 0, PMC_HEU = 1, KCORE_HEU = 2, NONE = 3 };
  enum class INLIER_GRAPH_FORMULATION { CHAIN = 0, COMPLETE = 1 };

  struct Params {  // defaults: registration.h:419-514
    double noise_bound = 0.01;
    double cbar2 = 1;
    bool estimate_scaling = true;
    ROTATION_ESTIMATION_ALGORITHM rotation_estimation_algorithm = ROTATION_ESTIMATION_ALGORITHM::GNC_TLS;
    double rotation_gnc_factor = 1.4;
    size_t rotation_max_iterations = 100;
    double rotation_cost_threshold = 1e-6;
    INLIER_GRAPH_FORMULATION rotation_tim_graph = INLIER_GRAPH_FORMULATION::CHAIN;
    INLIER_SELECTION_MODE inlier_selection_mode = INLIER_SELECTION_MODE::PMC_EXACT;
    double kcore_heuristic_threshold = 0.5;
    bool use_max_clique = true;             // deprecated
    bool max_clique_exact_solution = true;  // deprecated
    double max_clique_time_limit = 3600;
    int max_clique_num_threads = 0;  // reference: omp_get_max_threads(); ignored on the GPU
  };

  RobustRegistrationSolver();
  RobustRegistrationSolver(double noise_bound, double cbar2, bool estimate_scaling,
                           ROTATION_ESTIMATION_ALGORITHM rotation_estimation_algorithm, double rotation_gnc_factor,
                           size_t rotation_max_iterations, double rotation_cost_threshold,
                           INLIER_GRAPH_FORMULATION rotation_tim_graph, INLIER_SELECTION_MODE inlier_selection_mode,
                           double kcore_heuristic_threshold, bool use_max_clique, bool max_clique_exact_solution,
                           double max_clique_time_limit, int max_clique_num_threads = 0);
  RobustRegistrationSolver(const Params& params);
  ~RobustRegistrationSolver();
  RobustRegistrationSolver(const RobustRegistrationSolver&) = delete;
  RobustRegistrationSolver& operator=(const RobustRegistrationSolver&) = delete;

  // registration.cc:512-551
  Mat3X computeTIMs(const Mat3X& v, Map2X* map);

  // registration.cc:553-566 / 568-737
  RegistrationSolution solve(const teaser::PointCloud& src_cloud, const teaser::PointCloud& dst_cloud,
                             const std::vector<std::pair<int, int>> correspondences);
  RegistrationSolution solve(const Mat3X& src, const Mat3X& dst);

  double solveForScale(const Mat3X& v1, const Mat3X& v2);
  Eigen::Vector3d solveForTranslation(const Mat3X& v1, const Mat3X& v2);
  Eigen::Matrix3d solveForRotation(const Mat3X& v1, const Mat3X& v2);

  double getGNCRotationCostAtTermination() { return gnc_cost_; }
  RegistrationSolution getSolution() { return solution_; }

  void setScaleEstimator(std::unique_ptr<AbstractScaleSolver> estimator) {
    scale_solver_ = std::move(estimator);
    custom_estimators_ = true;
  }
  void setRotationEstimator(std::unique_ptr<GNCRotationSolver> estimator) {
    rotation_solver_ = std::move(estimator);
    custom_estimators_ = true;
  }
  void setTranslationEstimator(std::unique_ptr<AbstractTranslationSolver> estimator) {
    translation_solver_ = std::move(estimator);
    custom_estimators_ = true;
  }

  // ---- getters (registration.h:609-824); O(N^2) ones are materialised lazily
  BoolRow getScaleInliersMask();
  Map2X getScaleInliersMap();
  std::vector<std::tuple<int, int>> getScaleInliers();
  BoolRow getRotationInliersMask() { return rotation_inliers_mask_; }
  Eigen::Matrix<int, 1, Eigen::Dynamic> getRotationInliersMap();
  std::vector<int> getRotationInliers() { return rotation_inliers_; }
  BoolRow getTranslationInliersMask() { return translation_inliers_mask_; }
  Eigen::Matrix<int, 1, Eigen::Dynamic> getTranslationInliersMap();
  std::vector<int> getTranslationInliers() { return translation_inliers_; }
  std::vector<int> getInputOrderedTranslationInliers();
  std::vector<int> getInlierMaxClique() { return max_clique_; }
  std::vector<std::vector<int>> getInlierGraph();
  Mat3X getSrcTIMs();
  Mat3X getDstTIMs();
  Mat3X getMaxCliqueSrcTIMs() { return pruned_src_tims_; }
  Mat3X getMaxCliqueDstTIMs() { return pruned_dst_tims_; }
  Map2X getSrcTIMsMap();
  Map2X getDstTIMsMap();
  Map2X getSrcTIMsMapForRotation() { return src_tims_map_rotation_; }
  Map2X getDstTIMsMapForRotation() { return dst_tims_map_rotation_; }

  void reset(const double noise_bound, const double cbar2, const bool estimate_scaling,
             const ROTATION_ESTIMATION_ALGORITHM rotation_estimation_algorithm, const double rotation_gnc_factor,
             const size_t rotation_max_iterations, const double rotation_cost_threshold,
             const INLIER_GRAPH_FORMULATION rotation_tim_graph, const INLIER_SELECTION_MODE inlier_selection_mode,
             const double kcore_heuristic_threshold, const bool use_max_clique, const bool max_clique_exact_solution,
             const double max_clique_time_limit, const int max_clique_num_threads);
  void reset(const Params& params);
  Params getParams() { return params_; }

  // GPU extras (not in the reference)
  // Many independent problems in one call: the batch is cut into shards and every shard is solved on its own GPU
  // (tzr_solve_batch_multi: one context + host thread per device inside the library, no collective) with this
  // solver's Params.  devices empty = every visible device.  cliques (optional) receives the sorted max-clique index
  // sets.  The per-problem getters of this object are not touched.
  std::vector<RegistrationSolution> solveBatch(
      const std::vector<Mat3X>& src, const std::vector<Mat3X>& dst, std::vector<std::vector<int>>* cliques = nullptr,
      const std::vector<int>& devices = {});
  // One problem of solveAndCertifyBatch: what solve() and the getters give for it alone, and its certification.
  struct SolveCertifyResult {
    RegistrationSolution solution;
    std::vector<int> max_clique;
    BoolRow rotation_inliers_mask;     // getRotationInliersMask()
    BoolRow translation_inliers_mask;  // getTranslationInliersMask()
    bool certified = false;            // false: invalid solution, a non-finite input, or 4N + 4 > 32768
    CertificationResult certification;
  };
  // solve() then DRSCertifier(cert_params).certify(R, getMaxCliqueSrcTIMs(), getMaxCliqueDstTIMs(),
  // getRotationInliersMask()) on many problems: one batched solve (tzr_solve_batch) and one batched certification of
  // its retained results (tzr_certify_last_solve) on this thread's context, one device.  Problem b is certified with
  // noise bound cert_params.noise_bound / scale_b; 2 * this solver's noise_bound certifies what the rotation solver
  // solved.  The per-problem getters of this object are not touched.
  std::vector<SolveCertifyResult> solveAndCertifyBatch(const std::vector<Mat3X>& src, const std::vector<Mat3X>& dst,
                                                       const DRSCertifier::Params& cert_params);
  // The front end of solveCloudPairs: FPFHEstimation::computeFPFHFeatures' radii and Matcher::calculateCorrespondences'
  // flags (same defaults).  Pair p uses tuple seed tuple_seed + p * 0x9E3779B97F4A7C15, the seed
  // Matcher::calculateCorrespondencesBatch gives its p-th pair (tuple_seed: a fresh Matcher's).
  struct CloudPairParams {
    double normal_search_radius = 0.03;
    double fpfh_search_radius = 0.05;
    bool use_absolute_scale = true;
    bool use_crosscheck = true;
    bool use_tuple_test = true;
    float tuple_scale = 0;
    uint64_t tuple_seed = 0x7ea5e2ull;
  };
  // One pair of solveCloudPairs.  status: 0 (TZR_OK) solved; TZR_ERR_TOO_LARGE (-6) a cloud with a point of more than
  // 4096 neighbours (no correspondences), or more correspondences than one solve takes (65536, or 46340 with
  // estimate_scaling; correspondences given, not solved); TZR_ERR_INVALID_ARG (-1) no correspondence.  An unsolved
  // pair has an invalid solution and an empty clique.
  struct CloudPairResult {
    int status = 0;
    std::vector<std::pair<int, int>> correspondences;  // sorted, unique (source index, target index)
    RegistrationSolution solution;
    std::vector<int> max_clique;  // sorted rows of correspondences
    float global_scale = 1;       // Matcher::getGlobalScale()
  };
  // FPFHEstimation::computeFPFHFeaturesBatch(clouds), Matcher::calculateCorrespondencesBatch over the pairs (source
  // cloud, target cloud) and solve(clouds[src], clouds[dst], correspondences) per pair with this solver's Params, in
  // one device call (tzr_register_cloud_pairs) on this thread's context: each cloud's descriptors are computed once,
  // however many pairs name it.  Every cloud must be non-empty.  The per-problem getters of this object are not
  // touched.
  std::vector<CloudPairResult> solveCloudPairs(const std::vector<PointCloud>& clouds,
                                               const std::vector<std::pair<int, int>>& pairs,
                                               const CloudPairParams& params);
  // solveCloudPairs, then point-to-point ICP of every pair whose solution is valid, on its two clouds, seeded with that
  // solution, in the same device call (tzr_register_cloud_pairs_icp).  refined = false (and icp zeroed) for a pair
  // that was not refined.  The pair results are those of the overload above.
  struct CloudPairICPResult : CloudPairResult {
    bool refined = false;
    PointToPointICPResult icp;
  };
  std::vector<CloudPairICPResult> solveCloudPairs(const std::vector<PointCloud>& clouds,
                                                  const std::vector<std::pair<int, int>>& pairs,
                                                  const CloudPairParams& params, const PointToPointICPParams& icp);
  // The overload above with point-to-plane ICP (tzr_register_cloud_pairs_icp_point_to_plane): each target cloud's
  // normals are the ones the call's FPFH stage computed at params.normal_search_radius (PointToPlaneICP's parameters
  // are PointToPointICP's).
  std::vector<CloudPairICPResult> solveCloudPairsPointToPlane(const std::vector<PointCloud>& clouds,
                                                              const std::vector<std::pair<int, int>>& pairs,
                                                              const CloudPairParams& params,
                                                              const PointToPointICPParams& icp);
  // The overload above with generalized ICP (tzr_register_cloud_pairs_icp_generalized): both clouds' normals are the
  // ones the call's FPFH stage computed at params.normal_search_radius.
  std::vector<CloudPairICPResult> solveCloudPairsGeneralizedICP(const std::vector<PointCloud>& clouds,
                                                                const std::vector<std::pair<int, int>>& pairs,
                                                                const CloudPairParams& params,
                                                                const GeneralizedICPParams& icp);
  // The two overloads above with a robust kernel (tzr_register_cloud_pairs_icp_robust); each refined record equals
  // PointToPlaneICP / GeneralizedICP with that kernel on the pair, seeded with its solution.
  std::vector<CloudPairICPResult> solveCloudPairsPointToPlane(const std::vector<PointCloud>& clouds,
                                                              const std::vector<std::pair<int, int>>& pairs,
                                                              const CloudPairParams& params,
                                                              const PointToPointICPParams& icp,
                                                              const RobustKernel& kernel);
  std::vector<CloudPairICPResult> solveCloudPairsGeneralizedICP(const std::vector<PointCloud>& clouds,
                                                                const std::vector<std::pair<int, int>>& pairs,
                                                                const CloudPairParams& params,
                                                                const GeneralizedICPParams& icp,
                                                                const RobustKernel& kernel);
  // The overloads above with coloured ICP (tzr_register_cloud_pairs_icp_colored): colors holds one ColorCloud per
  // cloud, aligned with it.  Each target's normals are the ones the call's FPFH stage computed at
  // params.normal_search_radius, and each cloud's colour gradients are computed once per call, at 2
  // max_correspondence_distance.  Each refined record equals ColoredICP with the same parameters and kernel (L2 by
  // default) on the pair, seeded with its solution, with those normals.
  std::vector<CloudPairICPResult> solveCloudPairsColoredICP(const std::vector<PointCloud>& clouds,
                                                            const std::vector<ColorCloud>& colors,
                                                            const std::vector<std::pair<int, int>>& pairs,
                                                            const CloudPairParams& params, const ColoredICPParams& icp,
                                                            const RobustKernel& kernel = RobustKernel());
  // Multiway registration (tzr_register_cloud_pairs_multiway): solveCloudPairsPointToPlane, then the information
  // matrix of every refined pair at its ICP transform and distance, then the GNC-TLS pose graph over the clouds with one
  // edge per refined pair, in one device call.  uncertain: one flag per pair; the overload without it takes Open3D's
  // tutorial rule, pair (k, k + 1) certain and every other pair uncertain.  estimate_scaling must be off (the pose
  // graph is rigid).  information and weights are zero, inliers false, for a pair that is not an edge; poses (one per
  // cloud, cloud into the world frame) are zero when pose_graph_status is not 0 (e.g. TZR_ERR_INVALID_ARG for a
  // disconnected graph).
  struct MultiwayResult {
    std::vector<CloudPairICPResult> pairs;
    std::vector<Eigen::Matrix<double, 6, 6>> information;
    std::vector<int> information_counts;
    std::vector<double> edge_weights;
    std::vector<bool> edge_inliers;
    std::vector<Eigen::Matrix4d> poses;
    int pose_graph_status = 0;
    int iterations = 0;
    int inner_iterations = 0;
    double cost = 0;
  };
  MultiwayResult solveMultiway(const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs,
                               const CloudPairParams& params, const PointToPointICPParams& icp,
                               const PoseGraphParams& pose_graph);
  MultiwayResult solveMultiway(const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs,
                               const CloudPairParams& params, const PointToPointICPParams& icp,
                               const PoseGraphParams& pose_graph, const std::vector<bool>& uncertain);
  // The two overloads above with coloured ICP (tzr_register_cloud_pairs_multiway_colored): solveCloudPairsColoredICP
  // in place of solveCloudPairsPointToPlane.  The information matrices are geometric, as without colours.
  MultiwayResult solveMultiway(const std::vector<PointCloud>& clouds, const std::vector<ColorCloud>& colors,
                               const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& params,
                               const ColoredICPParams& icp, const PoseGraphParams& pose_graph,
                               const RobustKernel& kernel = RobustKernel());
  MultiwayResult solveMultiway(const std::vector<PointCloud>& clouds, const std::vector<ColorCloud>& colors,
                               const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& params,
                               const ColoredICPParams& icp, const PoseGraphParams& pose_graph,
                               const std::vector<bool>& uncertain, const RobustKernel& kernel = RobustKernel());
  bool isMaxCliqueProvenOptimal() const { return clique_proven_; }
  long long getNumInlierGraphEdges() const { return n_edges_; }
  int getGNCRotationIterations() const { return gnc_iterations_; }

 private:
  void materialise_graph();
  void materialise_tims();
  RegistrationSolution solve_decoupled(const Mat3X& src, const Mat3X& dst);

  Params params_;
  RegistrationSolution solution_;
  BoolRow scale_inliers_mask_, rotation_inliers_mask_, translation_inliers_mask_;
  Mat3X src_tims_, dst_tims_, pruned_src_tims_, pruned_dst_tims_;
  Map2X src_tims_map_, dst_tims_map_, src_tims_map_rotation_, dst_tims_map_rotation_;
  std::vector<int> max_clique_, rotation_inliers_, translation_inliers_;
  teaser::Graph inlier_graph_;
  std::unique_ptr<AbstractScaleSolver> scale_solver_;
  std::unique_ptr<GNCRotationSolver> rotation_solver_;
  std::unique_ptr<AbstractTranslationSolver> translation_solver_;
  bool custom_estimators_ = false;
  // lazily materialised state
  Mat3X last_src_, last_dst_;
  bool have_graph_ = false, have_tims_ = false, solved_ = false;
  double gnc_cost_ = 0;
  int gnc_iterations_ = 0;
  bool clique_proven_ = false;
  long long n_edges_ = 0;
  unsigned long long graph_generation_ = 0;  // tzr_last_graph_info generation right after this solver's solve()
};

// Context shared by all façade objects of the calling thread (a tzr_ctx is not thread-safe).
tzr_ctx* b200_context();

}  // namespace teaser
