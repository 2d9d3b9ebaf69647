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
