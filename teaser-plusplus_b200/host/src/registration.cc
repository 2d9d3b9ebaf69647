// Implementation of the drop-in C++ façade (teaser/registration.h) on top of the C-ABI (teaser_b200.h).
// Host logic only: parameter marshalling, state for the getters, lazy materialisation.  All arithmetic of
// the hot path runs in libteaser_b200.so on the GPU.
#include "teaser/registration.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "teaser_b200.h"

namespace teaser {

namespace {

[[noreturn]] void fail(const char* what, int rc, tzr_ctx* ctx) {
  std::string msg = std::string(what) + ": " + tzr_status_string(rc);
  if (ctx) msg += std::string(" (") + tzr_last_error(ctx) + ")";
  throw std::runtime_error(msg);
}

tzr_params to_c(const RobustRegistrationSolver::Params& p) {
  tzr_params c;
  tzr_params_default(&c);
  c.noise_bound = p.noise_bound;
  c.cbar2 = p.cbar2;
  c.estimate_scaling = p.estimate_scaling ? 1 : 0;
  c.rotation_estimation_algorithm = static_cast<int>(p.rotation_estimation_algorithm);
  c.rotation_gnc_factor = p.rotation_gnc_factor;
  c.rotation_max_iterations = p.rotation_max_iterations;
  c.rotation_cost_threshold = p.rotation_cost_threshold;
  c.rotation_tim_graph = static_cast<int>(p.rotation_tim_graph);
  c.inlier_selection_mode = static_cast<int>(p.inlier_selection_mode);
  c.kcore_heuristic_threshold = p.kcore_heuristic_threshold;
  c.use_max_clique = p.use_max_clique ? 1 : 0;
  c.max_clique_exact_solution = p.max_clique_exact_solution ? 1 : 0;
  c.max_clique_time_limit = p.max_clique_time_limit;
  c.max_clique_num_threads = p.max_clique_num_threads;
  return c;
}

void mask_from_bytes(const std::vector<uint8_t>& b, size_t m, BoolRow* out) {
  out->resize(1, static_cast<Eigen::Index>(m));
  for (size_t i = 0; i < m; ++i) (*out)(static_cast<Eigen::Index>(i)) = b[i] != 0;
}

}  // namespace

tzr_ctx* b200_context() {
  struct Holder {
    tzr_ctx* c = nullptr;
    ~Holder() {
      if (c) tzr_ctx_destroy(c);
    }
  };
  thread_local Holder h;
  if (!h.c) {
    int rc = tzr_ctx_create(-1, &h.c);
    if (rc != TZR_OK) fail("teaser (GPU): cannot create a CUDA context", rc, nullptr);
    // the reference has no size limit: take the device's largest (65536 correspondences, large clique route)
    rc = tzr_ctx_set_max_n(h.c, 65536);
    if (rc != TZR_OK) fail("teaser (GPU): tzr_ctx_set_max_n", rc, h.c);
  }
  return h.c;
}

// ------------------------------------------------------------------------------------------------ sub-solvers
void ScalarTLSEstimator::estimate(const Eigen::RowVectorXd& X, const Eigen::RowVectorXd& ranges, double* estimate,
                                  BoolRow* inliers) {
  const size_t m = static_cast<size_t>(X.cols());
  std::vector<uint8_t> mask(m);
  double est = 0;
  tzr_ctx* ctx = b200_context();
  int rc = tzr_scalar_tls(ctx, X.data(), ranges.data(), static_cast<int64_t>(m), &est, mask.data());
  if (rc != TZR_OK) fail("ScalarTLSEstimator::estimate", rc, ctx);
  if (estimate) *estimate = est;
  if (inliers) mask_from_bytes(mask, m, inliers);
}

// registration.cc:410-425 (host side: the two norm rows; the K-element TLS runs on the device)
void TLSScaleSolver::solveForScale(const Mat3X& src, const Mat3X& dst, double* scale, BoolRow* inliers) {
  const Eigen::Index K = src.cols();
  Eigen::RowVectorXd raw(1, K), alphas(1, K);
  const double beta = 2 * noise_bound_ * std::sqrt(cbar2_);
  std::vector<std::pair<Eigen::Index, double>> d2_at_zero;  // (k, d2) of the TIMs with d1 = 0 (a repeated source point)
  for (Eigen::Index k = 0; k < K; ++k) {
    const double d1 = std::sqrt((src(0, k) * src(0, k) + src(1, k) * src(1, k)) + src(2, k) * src(2, k));
    const double d2 = std::sqrt((dst(0, k) * dst(0, k) + dst(1, k) * dst(1, k)) + dst(2, k) * dst(2, k));
    raw(k) = d2 / d1;
    alphas(k) = beta * (1.0 / d1);
    if (d1 == 0) d2_at_zero.emplace_back(k, d2);
  }
  tls_estimator_.estimate(raw, alphas, scale, inliers);
  // such a TIM is excluded from the estimate; it is an inlier iff d2 <= beta, the fixed-scale rule (DESIGN.md §3.4)
  if (inliers)
    for (const auto& z : d2_at_zero) (*inliers)(z.first) = z.second <= beta;
}

// registration.cc:427-443
void ScaleInliersSelector::solveForScale(const Mat3X& src, const Mat3X& dst, double* scale, BoolRow* inliers) {
  *scale = 1;
  const Eigen::Index K = src.cols();
  const double beta = 2 * noise_bound_ * std::sqrt(cbar2_);
  if (inliers) inliers->resize(1, K);
  for (Eigen::Index k = 0; k < K; ++k) {
    const double d1 = std::sqrt((src(0, k) * src(0, k) + src(1, k) * src(1, k)) + src(2, k) * src(2, k));
    const double d2 = std::sqrt((dst(0, k) * dst(0, k) + dst(1, k) * dst(1, k)) + dst(2, k) * dst(2, k));
    if (inliers) (*inliers)(k) = std::fabs(d1 - d2) <= beta;
  }
}

void TLSTranslationSolver::solveForTranslation(const Mat3X& src, const Mat3X& dst, Eigen::Vector3d* translation,
                                               BoolRow* inliers) {
  const size_t m = static_cast<size_t>(src.cols());
  std::vector<uint8_t> mask(m);
  double t[3];
  tzr_ctx* ctx = b200_context();
  int rc = tzr_tls_translation(ctx, src.data(), dst.data(), static_cast<int>(m), noise_bound_, cbar2_, t, mask.data());
  if (rc != TZR_OK) fail("TLSTranslationSolver::solveForTranslation", rc, ctx);
  if (translation) {
    (*translation)(0) = t[0];
    (*translation)(1) = t[1];
    (*translation)(2) = t[2];
  }
  if (inliers) mask_from_bytes(mask, m, inliers);
}

namespace {
void rotation_via_abi(int alg, const char* who, const GNCRotationSolver::Params& prm, const Mat3X& src, const Mat3X& dst,
                      Eigen::Matrix3d* rotation, BoolRow* inliers, double* cost_out) {
  const size_t m = static_cast<size_t>(src.cols());
  std::vector<uint8_t> mask(m);
  double R[9], cost = 0;
  int32_t iters = 0;
  tzr_ctx* ctx = b200_context();
  int rc = tzr_rotation_solve(ctx, alg, src.data(), dst.data(), static_cast<int>(m), prm.noise_bound, prm.gnc_factor,
                              prm.max_iterations, prm.cost_threshold, R, mask.data(), &cost, &iters);
  if (rc != TZR_OK) fail(who, rc, ctx);
  *cost_out = cost;
  if (rotation) std::memcpy(rotation->data(), R, sizeof(R));  // both column-major
  if (inliers) mask_from_bytes(mask, m, inliers);
}
}  // namespace

void GNCTLSRotationSolver::solveForRotation(const Mat3X& src, const Mat3X& dst, Eigen::Matrix3d* rotation,
                                            BoolRow* inliers) {
  rotation_via_abi(0, "GNCTLSRotationSolver::solveForRotation", params_, src, dst, rotation, inliers, &cost_);
}
void FastGlobalRegistrationSolver::solveForRotation(const Mat3X& src, const Mat3X& dst, Eigen::Matrix3d* rotation,
                                                    BoolRow* inliers) {
  rotation_via_abi(1, "FastGlobalRegistrationSolver::solveForRotation", params_, src, dst, rotation, inliers, &cost_);
}
void QuatroSolver::solveForRotation(const Mat3X& src, const Mat3X& dst, Eigen::Matrix3d* rotation, BoolRow* inliers) {
  rotation_via_abi(2, "QuatroSolver::solveForRotation", params_, src, dst, rotation, inliers, &cost_);
}

// ------------------------------------------------------------------------------------------------ max clique
std::vector<int> MaxCliqueSolver::findMaxClique(Graph graph) {
  const int n = graph.numVertices();
  if (n == 0) return {};
  int mode = static_cast<int>(params_.solver_mode);
  if (!params_.solve_exactly) mode = 1;  // graph.cc:15-17
  tzr_ctx* ctx = b200_context();
  const int W = tzr_words_per_row(n);
  std::vector<uint64_t> bits(static_cast<size_t>(n) * W, 0);
  for (int v = 0; v < n; ++v)
    for (int u : graph.getEdges(v)) bits[static_cast<size_t>(v) * W + (u >> 6)] |= 1ull << (u & 63);
  std::vector<int32_t> clique(n);
  int32_t m = 0, proven = 0;
  int rc = tzr_max_clique(ctx, bits.data(), n, mode, params_.kcore_heuristic_threshold, params_.time_limit,
                          clique.data(), &m, &proven);
  if (rc != TZR_OK) fail("MaxCliqueSolver::findMaxClique", rc, ctx);
  return std::vector<int>(clique.begin(), clique.begin() + m);
}

// ------------------------------------------------------------------------------------------------ solver
RobustRegistrationSolver::RobustRegistrationSolver() { reset(Params()); }

RobustRegistrationSolver::RobustRegistrationSolver(
    double noise_bound, double cbar2, bool estimate_scaling, ROTATION_ESTIMATION_ALGORITHM rotation_estimation_algorithm,
    double rotation_gnc_factor, size_t rotation_max_iterations, double rotation_cost_threshold,
    INLIER_GRAPH_FORMULATION rotation_tim_graph, INLIER_SELECTION_MODE inlier_selection_mode,
    double kcore_heuristic_threshold, bool use_max_clique, bool max_clique_exact_solution, double max_clique_time_limit,
    int max_clique_num_threads) {
  reset(noise_bound, cbar2, estimate_scaling, rotation_estimation_algorithm, rotation_gnc_factor,
        rotation_max_iterations, rotation_cost_threshold, rotation_tim_graph, inlier_selection_mode,
        kcore_heuristic_threshold, use_max_clique, max_clique_exact_solution, max_clique_time_limit,
        max_clique_num_threads);
}

RobustRegistrationSolver::RobustRegistrationSolver(const Params& params) { reset(params); }
RobustRegistrationSolver::~RobustRegistrationSolver() = default;

void RobustRegistrationSolver::reset(const Params& p) {
  reset(p.noise_bound, p.cbar2, p.estimate_scaling, p.rotation_estimation_algorithm, p.rotation_gnc_factor,
        p.rotation_max_iterations, p.rotation_cost_threshold, p.rotation_tim_graph, p.inlier_selection_mode,
        p.kcore_heuristic_threshold, p.use_max_clique, p.max_clique_exact_solution, p.max_clique_time_limit,
        p.max_clique_num_threads);
}

// registration.h:830-885 — installs the three sub-solvers; unlike the reference it also stores params_ (Q1)
void RobustRegistrationSolver::reset(const double noise_bound, const double cbar2, const bool estimate_scaling,
                                     const ROTATION_ESTIMATION_ALGORITHM rotation_estimation_algorithm,
                                     const double rotation_gnc_factor, const size_t rotation_max_iterations,
                                     const double rotation_cost_threshold,
                                     const INLIER_GRAPH_FORMULATION rotation_tim_graph,
                                     const INLIER_SELECTION_MODE inlier_selection_mode,
                                     const double kcore_heuristic_threshold, const bool use_max_clique,
                                     const bool max_clique_exact_solution, const double max_clique_time_limit,
                                     const int max_clique_num_threads) {
  params_.noise_bound = noise_bound;
  params_.cbar2 = cbar2;
  params_.estimate_scaling = estimate_scaling;
  params_.rotation_estimation_algorithm = rotation_estimation_algorithm;
  params_.rotation_gnc_factor = rotation_gnc_factor;
  params_.rotation_max_iterations = rotation_max_iterations;
  params_.rotation_cost_threshold = rotation_cost_threshold;
  params_.rotation_tim_graph = rotation_tim_graph;
  params_.inlier_selection_mode = inlier_selection_mode;
  params_.kcore_heuristic_threshold = kcore_heuristic_threshold;
  params_.use_max_clique = use_max_clique;
  params_.max_clique_exact_solution = max_clique_exact_solution;
  params_.max_clique_time_limit = max_clique_time_limit;
  params_.max_clique_num_threads = max_clique_num_threads;

  if (estimate_scaling)
    scale_solver_ = std::make_unique<TLSScaleSolver>(noise_bound, cbar2);
  else
    scale_solver_ = std::make_unique<ScaleInliersSelector>(noise_bound, cbar2);
  GNCRotationSolver::Params rp{rotation_max_iterations, rotation_cost_threshold, rotation_gnc_factor, noise_bound};
  switch (rotation_estimation_algorithm) {
    case ROTATION_ESTIMATION_ALGORITHM::GNC_TLS:
      rotation_solver_ = std::make_unique<GNCTLSRotationSolver>(rp);
      break;
    case ROTATION_ESTIMATION_ALGORITHM::FGR:
      rotation_solver_ = std::make_unique<FastGlobalRegistrationSolver>(rp);
      break;
    case ROTATION_ESTIMATION_ALGORITHM::QUATRO:
      rotation_solver_ = std::make_unique<QuatroSolver>(rp);
      break;
  }
  translation_solver_ = std::make_unique<TLSTranslationSolver>(noise_bound, cbar2);
  custom_estimators_ = false;
  max_clique_.clear();
  rotation_inliers_.clear();
  translation_inliers_.clear();
  inlier_graph_.clear();
  have_graph_ = have_tims_ = solved_ = false;
}

// registration.cc:512-551 (host-side materialisation; solve() itself never builds the O(N^2) TIMs)
Mat3X RobustRegistrationSolver::computeTIMs(const Mat3X& v, Map2X* map) {
  const Eigen::Index N = v.cols();
  const Eigen::Index K = N * (N - 1) / 2;
  Mat3X vt(3, K);
  if (map) map->resize(2, K);
  Eigen::Index k = 0;
  for (Eigen::Index i = 0; i + 1 < N; ++i)
    for (Eigen::Index j = i + 1; j < N; ++j, ++k) {
      vt(0, k) = v(0, j) - v(0, i);
      vt(1, k) = v(1, j) - v(1, i);
      vt(2, k) = v(2, j) - v(2, i);
      if (map) {
        (*map)(0, k) = static_cast<int>(i);
        (*map)(1, k) = static_cast<int>(j);
      }
    }
  return vt;
}

// registration.cc:553-566
RegistrationSolution RobustRegistrationSolver::solve(const teaser::PointCloud& src_cloud,
                                                     const teaser::PointCloud& dst_cloud,
                                                     const std::vector<std::pair<int, int>> correspondences) {
  const Eigen::Index n = static_cast<Eigen::Index>(correspondences.size());
  Mat3X src(3, n), dst(3, n);
  for (Eigen::Index i = 0; i < n; ++i) {
    const auto& s = src_cloud[correspondences[i].first];
    const auto& d = dst_cloud[correspondences[i].second];
    src(0, i) = s.x; src(1, i) = s.y; src(2, i) = s.z;
    dst(0, i) = d.x; dst(1, i) = d.y; dst(2, i) = d.z;
  }
  return solve(src, dst);
}

// registration.cc:568-737 — one C-ABI call
RegistrationSolution RobustRegistrationSolver::solve(const Mat3X& src, const Mat3X& dst) {
  if (src.cols() != dst.cols()) throw std::invalid_argument("teaser: src and dst must have the same number of columns");
  if (custom_estimators_) return solve_decoupled(src, dst);
  const int n = static_cast<int>(src.cols());
  tzr_ctx* ctx = b200_context();
  tzr_params p = to_c(params_);
  tzr_solution s;
  std::vector<int32_t> clique(n);
  const bool complete = params_.rotation_tim_graph == INLIER_GRAPH_FORMULATION::COMPLETE;
  std::vector<uint8_t> rot(complete ? static_cast<size_t>(n) * (n - 1) / 2 + 1 : static_cast<size_t>(n)), trans(n);
  int rc = tzr_solve(ctx, &p, src.data(), dst.data(), n, &s, clique.data(), rot.data(), trans.data());
  if (rc != TZR_OK) fail("RobustRegistrationSolver::solve", rc, ctx);

  last_src_ = src;
  last_dst_ = dst;
  have_graph_ = have_tims_ = false;
  solved_ = true;
  {
    uint64_t gen = 0;
    tzr_last_graph_info(ctx, nullptr, nullptr, nullptr, &gen);
    graph_generation_ = gen;
  }
  solution_.valid = s.valid != 0;
  solution_.scale = s.scale;
  for (int k = 0; k < 3; ++k) solution_.translation(k) = s.translation[k];
  std::memcpy(solution_.rotation.data(), s.rotation, sizeof(s.rotation));
  gnc_cost_ = s.gnc_cost;
  gnc_iterations_ = s.gnc_iterations;
  clique_proven_ = s.clique_proven_optimal != 0;
  if (!clique_proven_ && s.valid && to_c(params_).inlier_selection_mode == 0 && params_.use_max_clique &&
      params_.max_clique_exact_solution)
    // the exact search ran into max_clique_time_limit or its stack budget: the clique is the best one found, not
    // proven maximum (the reference's PMC prints its own time-limit notice in that situation)
    std::fprintf(stderr, "[teaser-b200] warning: maximum clique search incomplete (time/stack budget); returning the "
                         "best clique found (%d vertices)\n", s.clique_size);
  n_edges_ = s.n_edges;
  const size_t m = static_cast<size_t>(std::max(0, s.clique_size));
  max_clique_.assign(clique.begin(), clique.begin() + m);
  rotation_inliers_.clear();
  translation_inliers_.clear();
  if (!solution_.valid) return solution_;  // registration.cc:643-647

  const size_t n_rot = complete ? m * (m - 1) / 2 : m;
  mask_from_bytes(rot, n_rot, &rotation_inliers_mask_);
  mask_from_bytes(trans, m, &translation_inliers_mask_);
  for (size_t i = 0; i < n_rot; ++i)
    if (rot[i]) rotation_inliers_.push_back(static_cast<int>(i));
  for (size_t i = 0; i < m; ++i)
    if (trans[i]) translation_inliers_.push_back(static_cast<int>(i));
  if (complete) {  // registration.cc:681-694
    Mat3X si(3, m), di(3, m);
    for (size_t i = 0; i < m; ++i)
      for (int r = 0; r < 3; ++r) {
        si(r, i) = src(r, max_clique_[i]);
        di(r, i) = dst(r, max_clique_[i]);
      }
    pruned_dst_tims_ = computeTIMs(di, &dst_tims_map_rotation_);
    pruned_src_tims_ = computeTIMs(si, &src_tims_map_rotation_);
    pruned_dst_tims_ *= (1 / solution_.scale);
    return solution_;
  }
  // chain TIMs and their maps for the getters (registration.cc:657-680,697)
  pruned_src_tims_.resize(3, m);
  pruned_dst_tims_.resize(3, m);
  src_tims_map_rotation_.resize(2, m);
  dst_tims_map_rotation_.resize(2, m);
  const double inv_scale = 1 / solution_.scale;
  for (size_t i = 0; i < m; ++i) {
    const int root = max_clique_[i];
    const int leaf = (i + 1 != m) ? max_clique_[i + 1] : max_clique_[0];
    for (int r = 0; r < 3; ++r) {
      pruned_src_tims_(r, i) = src(r, leaf) - src(r, root);
      pruned_dst_tims_(r, i) = (dst(r, leaf) - dst(r, root)) * inv_scale;
    }
    src_tims_map_rotation_(0, i) = dst_tims_map_rotation_(0, i) = leaf;
    src_tims_map_rotation_(1, i) = dst_tims_map_rotation_(1, i) = root;
  }
  return solution_;
}

// Decoupled flow for callers that installed their own estimators (registration.h:623-644): the reference's
// orchestration (registration.cc:599-736) with each stage going through the installed strategy object.
RegistrationSolution RobustRegistrationSolver::solve_decoupled(const Mat3X& src, const Mat3X& dst) {
  last_src_ = src;
  last_dst_ = dst;
  solved_ = true;
  src_tims_ = computeTIMs(src, &src_tims_map_);
  dst_tims_ = computeTIMs(dst, &dst_tims_map_);
  have_tims_ = true;
  solveForScale(src_tims_, dst_tims_);
  int mode = static_cast<int>(params_.inlier_selection_mode);
  if (!params_.use_max_clique) mode = 3;
  if (!params_.max_clique_exact_solution) mode = 1;
  max_clique_.clear();
  inlier_graph_.clear();
  if (mode != 3) {
    inlier_graph_.populateVertices(static_cast<int>(src.cols()));
    for (Eigen::Index k = 0; k < scale_inliers_mask_.cols(); ++k)
      if (scale_inliers_mask_(k)) inlier_graph_.addEdge(src_tims_map_(0, k), src_tims_map_(1, k));
    have_graph_ = true;
    n_edges_ = inlier_graph_.numEdges();
    MaxCliqueSolver::Params cp;
    cp.solver_mode = static_cast<MaxCliqueSolver::CLIQUE_SOLVER_MODE>(mode);
    cp.time_limit = params_.max_clique_time_limit;
    cp.kcore_heuristic_threshold = params_.kcore_heuristic_threshold;
    MaxCliqueSolver cs(cp);
    max_clique_ = cs.findMaxClique(inlier_graph_);
    std::sort(max_clique_.begin(), max_clique_.end());
    if (max_clique_.size() <= 1) {
      solution_.valid = false;
      return solution_;
    }
  } else {
    for (Eigen::Index i = 0; i < src.cols(); ++i) max_clique_.push_back(static_cast<int>(i));
  }
  const size_t m = max_clique_.size();
  if (params_.rotation_tim_graph == INLIER_GRAPH_FORMULATION::COMPLETE) {  // registration.cc:681-694
    Mat3X si(3, m), di(3, m);
    for (size_t i = 0; i < m; ++i)
      for (int r = 0; r < 3; ++r) {
        si(r, i) = src(r, max_clique_[i]);
        di(r, i) = dst(r, max_clique_[i]);
      }
    pruned_dst_tims_ = computeTIMs(di, &dst_tims_map_rotation_);
    pruned_src_tims_ = computeTIMs(si, &src_tims_map_rotation_);
    pruned_dst_tims_ *= (1 / solution_.scale);
  } else {
    pruned_src_tims_.resize(3, m);
    pruned_dst_tims_.resize(3, m);
    src_tims_map_rotation_.resize(2, m);
    dst_tims_map_rotation_.resize(2, m);
    for (size_t i = 0; i < m; ++i) {
      const int root = max_clique_[i];
      const int leaf = (i + 1 != m) ? max_clique_[i + 1] : max_clique_[0];
      for (int r = 0; r < 3; ++r) {
        pruned_src_tims_(r, i) = src(r, leaf) - src(r, root);
        pruned_dst_tims_(r, i) = (dst(r, leaf) - dst(r, root)) * (1 / solution_.scale);
      }
      src_tims_map_rotation_(0, i) = dst_tims_map_rotation_(0, i) = leaf;
      src_tims_map_rotation_(1, i) = dst_tims_map_rotation_(1, i) = root;
    }
  }
  // fresh noise bound every call (the reference mutates it in place, SURVEY Q2)
  auto rp = rotation_solver_->getParams();
  const double saved_nb = rp.noise_bound;
  rp.noise_bound *= (2 / solution_.scale);
  rotation_solver_->setParams(rp);
  solveForRotation(pruned_src_tims_, pruned_dst_tims_);
  rp.noise_bound = saved_nb;
  rotation_solver_->setParams(rp);
  rotation_inliers_.clear();
  for (Eigen::Index i = 0; i < rotation_inliers_mask_.cols(); ++i)
    if (rotation_inliers_mask_(i)) rotation_inliers_.push_back(static_cast<int>(i));
  Mat3X rs(3, m), rd(3, m);
  for (size_t i = 0; i < m; ++i) {
    const int c = max_clique_[i];
    for (int r = 0; r < 3; ++r) {
      rs(r, i) = (solution_.scale * solution_.rotation(r, 0)) * src(0, c) +
                 (solution_.scale * solution_.rotation(r, 1)) * src(1, c) +
                 (solution_.scale * solution_.rotation(r, 2)) * src(2, c);
      rd(r, i) = dst(r, c);
    }
  }
  solveForTranslation(rs, rd);
  translation_inliers_.clear();
  for (Eigen::Index i = 0; i < translation_inliers_mask_.cols(); ++i)
    if (translation_inliers_mask_(i)) translation_inliers_.push_back(static_cast<int>(i));
  solution_.valid = true;
  return solution_;
}

double RobustRegistrationSolver::solveForScale(const Mat3X& v1, const Mat3X& v2) {
  scale_inliers_mask_.resize(1, v1.cols());
  scale_solver_->solveForScale(v1, v2, &solution_.scale, &scale_inliers_mask_);
  return solution_.scale;
}
Eigen::Vector3d RobustRegistrationSolver::solveForTranslation(const Mat3X& v1, const Mat3X& v2) {
  translation_inliers_mask_.resize(1, v1.cols());
  translation_solver_->solveForTranslation(v1, v2, &solution_.translation, &translation_inliers_mask_);
  return solution_.translation;
}
Eigen::Matrix3d RobustRegistrationSolver::solveForRotation(const Mat3X& v1, const Mat3X& v2) {
  rotation_inliers_mask_.resize(1, v1.cols());
  rotation_solver_->solveForRotation(v1, v2, &solution_.rotation, &rotation_inliers_mask_);
  gnc_cost_ = rotation_solver_->getCostAtTermination();
  return solution_.rotation;
}

// ------------------------------------------------------------------------------------------------ lazy getters
void RobustRegistrationSolver::materialise_graph() {
  if (have_graph_ || !solved_) return;
  const int n = static_cast<int>(last_src_.cols());
  tzr_ctx* ctx = b200_context();
  // The graph lives in the per-thread context until someone asks for it.  If another solver (or a stage call such as
  // MaxCliqueSolver::findMaxClique) has used the context since this object's solve(), the retained graph is not ours
  // any more: rebuild it by solving the stored inputs again.
  int32_t gB = 0, gn = 0, has = 0;
  uint64_t gen = 0;
  tzr_last_graph_info(ctx, &gB, &gn, &has, &gen);
  if (gen != graph_generation_ || gn != n || gB != 1) {
    tzr_params p = to_c(params_);
    tzr_solution s;
    int rc = tzr_solve(ctx, &p, last_src_.data(), last_dst_.data(), n, &s, nullptr, nullptr, nullptr);
    if (rc != TZR_OK) fail("getInlierGraph (re-solve)", rc, ctx);
    tzr_last_graph_info(ctx, &gB, &gn, &has, &gen);
    graph_generation_ = gen;
  }
  if (!has) {  // inlier selection NONE: populateVertices is never called, the reference's graph stays empty
    inlier_graph_.clear();
    have_graph_ = true;
    return;
  }
  const int W = tzr_words_per_row(n);
  std::vector<uint64_t> bits(static_cast<size_t>(n) * W);
  std::vector<int32_t> deg(n);
  int rc = tzr_last_graph(ctx, 0, bits.data(), deg.data());
  if (rc != TZR_OK) fail("getInlierGraph", rc, ctx);
  std::vector<std::vector<int>> adj(n);
  size_t twice = 0;
  for (int v = 0; v < n; ++v) {
    adj[v].reserve(deg[v]);
    for (int w = 0; w < W; ++w) {
      uint64_t m = bits[static_cast<size_t>(v) * W + w];
      while (m) {
        const int b = __builtin_ctzll(m);
        m &= m - 1;
        adj[v].push_back(w * 64 + b);  // ascending, like the reference's insertion order (graph.h:96-104)
      }
    }
    twice += adj[v].size();
  }
  inlier_graph_.setAdjList(std::move(adj), twice / 2);
  have_graph_ = true;
}

std::vector<RegistrationSolution> RobustRegistrationSolver::solveBatch(
    const std::vector<Mat3X>& src, const std::vector<Mat3X>& dst, std::vector<std::vector<int>>* cliques,
    const std::vector<int>& devices) {
  if (src.size() != dst.size()) throw std::invalid_argument("teaser: solveBatch needs as many src as dst clouds");
  const int B = static_cast<int>(src.size());
  std::vector<RegistrationSolution> out(B);
  if (B == 0) return out;
  std::vector<int32_t> n(B), dev(devices.begin(), devices.end());
  std::vector<const double*> sp(B), dp(B);
  int max_n = 0;
  for (int b = 0; b < B; ++b) {
    if (src[b].cols() != dst[b].cols()) throw std::invalid_argument("teaser: src and dst must have the same number of columns");
    n[b] = static_cast<int32_t>(src[b].cols());
    sp[b] = src[b].data();
    dp[b] = dst[b].data();
    max_n = std::max(max_n, static_cast<int>(n[b]));
  }
  std::vector<tzr_solution> sols(B);
  std::vector<int32_t> clq(cliques ? static_cast<size_t>(B) * max_n : 0);
  tzr_params p = to_c(params_);
  int rc = tzr_solve_batch_multi(dev.empty() ? nullptr : dev.data(), static_cast<int>(dev.size()), &p, B, n.data(),
                                 sp.data(), dp.data(), sols.data(), cliques ? clq.data() : nullptr, max_n);
  if (rc != TZR_OK) fail("RobustRegistrationSolver::solveBatch", rc, nullptr);
  if (cliques) cliques->assign(B, {});
  for (int b = 0; b < B; ++b) {
    out[b].valid = sols[b].valid != 0;
    out[b].scale = sols[b].scale;
    for (int k = 0; k < 3; ++k) out[b].translation(k) = sols[b].translation[k];
    std::memcpy(out[b].rotation.data(), sols[b].rotation, sizeof(sols[b].rotation));
    if (cliques) {
      const int m = std::max(0, sols[b].clique_size);
      (*cliques)[b].assign(clq.begin() + static_cast<size_t>(b) * max_n, clq.begin() + static_cast<size_t>(b) * max_n + m);
    }
  }
  return out;
}

std::vector<RobustRegistrationSolver::SolveCertifyResult> RobustRegistrationSolver::solveAndCertifyBatch(
    const std::vector<Mat3X>& src, const std::vector<Mat3X>& dst, const DRSCertifier::Params& cert_params) {
  if (src.size() != dst.size())
    throw std::invalid_argument("teaser: solveAndCertifyBatch needs as many src as dst clouds");
  const int B = static_cast<int>(src.size());
  std::vector<SolveCertifyResult> out(B);
  if (B == 0) return out;
  std::vector<int32_t> n(B);
  std::vector<const double*> sp(B), dp(B);
  int max_n = 0;
  for (int b = 0; b < B; ++b) {
    if (src[b].cols() != dst[b].cols()) throw std::invalid_argument("teaser: src and dst must have the same number of columns");
    n[b] = static_cast<int32_t>(src[b].cols());
    sp[b] = src[b].data();
    dp[b] = dst[b].data();
    max_n = std::max(max_n, static_cast<int>(n[b]));
  }
  tzr_ctx* ctx = b200_context();
  std::vector<tzr_solution> sols(B);
  std::vector<int32_t> clq(static_cast<size_t>(B) * max_n);
  const tzr_params p = to_c(params_);
  int rc = tzr_solve_batch(ctx, &p, B, n.data(), sp.data(), dp.data(), sols.data(), clq.data(), max_n);
  if (rc != TZR_OK) fail("RobustRegistrationSolver::solveAndCertifyBatch (solve)", rc, ctx);
  const bool complete = params_.rotation_tim_graph == INLIER_GRAPH_FORMULATION::COMPLETE;
  for (int b = 0; b < B; ++b) {
    SolveCertifyResult& r = out[b];
    r.solution.valid = sols[b].valid != 0;
    r.solution.scale = sols[b].scale;
    for (int k = 0; k < 3; ++k) r.solution.translation(k) = sols[b].translation[k];
    std::memcpy(r.solution.rotation.data(), sols[b].rotation, sizeof(sols[b].rotation));
    const size_t m = static_cast<size_t>(std::max(0, sols[b].clique_size));
    r.max_clique.assign(clq.begin() + static_cast<size_t>(b) * max_n, clq.begin() + static_cast<size_t>(b) * max_n + m);
    const size_t rot_cap = complete ? (m > 0 ? m * (m - 1) / 2 : 0) : m;
    std::vector<uint8_t> rm(std::max<size_t>(1, rot_cap)), tm(std::max<size_t>(1, m));
    int64_t n_rot = 0;
    int32_t n_trans = 0;
    rc = tzr_last_inliers(ctx, b, rm.data(), tm.data(), &n_rot, &n_trans);
    if (rc != TZR_OK) fail("RobustRegistrationSolver::solveAndCertifyBatch (inlier masks)", rc, ctx);
    mask_from_bytes(rm, static_cast<size_t>(n_rot), &r.rotation_inliers_mask);
    mask_from_bytes(tm, static_cast<size_t>(n_trans), &r.translation_inliers_mask);
  }
  tzr_certifier_params c;
  tzr_certifier_params_default(&c);
  c.noise_bound = cert_params.noise_bound;
  c.cbar2 = cert_params.cbar2;
  c.sub_optimality = cert_params.sub_optimality;
  c.max_iterations = cert_params.max_iterations;
  c.gamma_tau = cert_params.gamma_tau;
  c.eig_decomposition_solver = static_cast<int>(cert_params.eig_decomposition_solver);
  const int cap = static_cast<int>(std::max(1.0, std::ceil(cert_params.max_iterations)));
  std::vector<std::vector<double>> traj(B, std::vector<double>(cap));
  std::vector<double*> tp(B);
  for (int b = 0; b < B; ++b) tp[b] = traj[b].data();
  std::vector<int32_t> caps(B, cap), status(B);
  std::vector<tzr_certification_result> res(B);
  rc = tzr_certify_last_solve(ctx, &c, B, nullptr, res.data(), status.data(), tp.data(), caps.data());
  if (rc != TZR_OK && rc != TZR_ERR_TOO_LARGE) fail("RobustRegistrationSolver::solveAndCertifyBatch (certify)", rc, ctx);
  for (int b = 0; b < B; ++b) {
    SolveCertifyResult& r = out[b];
    r.certified = status[b] == TZR_OK;
    r.certification.is_optimal = res[b].is_optimal != 0;
    r.certification.best_suboptimality = res[b].best_suboptimality;
    r.certification.suboptimality_traj.assign(traj[b].begin(), traj[b].begin() + std::min(res[b].n_iterations, cap));
  }
  return out;
}

void icp_result_from_c(const tzr_icp_result& r, const int32_t* corr, PointToPointICPResult* out);  // icp.cc
tzr_line_process_params line_process_c(const LineProcessParams& p);                                  // pose_graph.cc
tzr_pose_graph_params pose_graph_c(const PoseGraphParams& p);                                        // pose_graph.cc

namespace {

// solveCloudPairs' body: tzr_register_cloud_pairs, or tzr_register_cloud_pairs_icp(_point_to_plane, _generalized,
// _robust, _colored) when icp is given (icp_res then receives P records)
enum class IcpMethod { kPointToPoint, kPointToPlane, kGeneralized, kColored };
// the multiway step's inputs and outputs (solveMultiway: tzr_register_cloud_pairs_multiway(_colored))
struct MultiwayCall {
  const int32_t* uncertain;
  const tzr_pose_graph_params* pg;
  double* information;
  int32_t* info_counts;
  double* edge_weights;
  uint8_t* edge_mask;
  tzr_similarity* poses;
  tzr_pose_graph_summary* summary;
  int32_t* pg_status;
  const tzr_line_process_params* lp = nullptr;  // the line process in place of GNC-TLS (pg unused)
  tzr_line_process_summary* lp_summary = nullptr;
  // solveMultiwayBatch (tzr_register_cloud_pairs_multiway(_line_process)_batch): G > 0 graphs at graph_offsets, the
  // summaries and pg_status G entries each, and the fused maps
  int G = 0;
  const int32_t* graph_offsets = nullptr;
  double map_voxel_size = 0;
  float* const* map_points = nullptr;
  int32_t* map_counts = nullptr;
  float* const* map_colors = nullptr;
};
std::vector<RobustRegistrationSolver::CloudPairResult> run_cloud_pairs(
    const tzr_params& p, const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs,
    const RobustRegistrationSolver::CloudPairParams& cp, const tzr_icp_params* icp,
    std::vector<tzr_icp_result>* icp_res, IcpMethod method = IcpMethod::kPointToPoint, double epsilon = 0,
    const RobustKernel* kernel = nullptr, const MultiwayCall* mw = nullptr,
    const std::vector<ColorCloud>* colors = nullptr, double lambda_geometric = 0,
    const std::vector<uint64_t>* tuple_seeds = nullptr) {
  using CloudPairResult = RobustRegistrationSolver::CloudPairResult;
  const int K = static_cast<int>(clouds.size()), P = static_cast<int>(pairs.size());
  std::vector<CloudPairResult> out(P);
  if (P == 0) return out;
  static_assert(sizeof(ColorRGB) == 3 * sizeof(float), "ColorRGB must be three packed floats");
  std::vector<const float*> col;
  if (method == IcpMethod::kColored) {
    if (colors->size() != clouds.size()) throw std::invalid_argument("teaser: solveCloudPairs: one ColorCloud per cloud");
    for (int c = 0; c < K; ++c) {
      if ((*colors)[c].size() != clouds[c].size())
        throw std::invalid_argument("teaser: solveCloudPairs: a ColorCloud's size differs from its cloud's");
      col.push_back(clouds[c].empty() ? nullptr : &(*colors)[c][0].r);
    }
  }
  static_assert(sizeof(PointXYZ) == 3 * sizeof(float), "PointXYZ must be three packed floats");
  std::vector<int32_t> n(K), pc(2 * static_cast<size_t>(P)), status(P), index(P);
  std::vector<const float*> pts(K);
  for (int c = 0; c < K; ++c) {
    if (clouds[c].empty()) throw std::invalid_argument("teaser: solveCloudPairs needs non-empty clouds");
    n[c] = static_cast<int32_t>(clouds[c].size());
    pts[c] = &clouds[c][0].x;
  }
  std::vector<uint64_t> seeds(P);
  std::vector<std::vector<int32_t>> corr(P), clq(P);
  std::vector<int32_t*> corr_p(P), clq_p(P);
  for (int p = 0; p < P; ++p) {
    const int a = pairs[p].first, b = pairs[p].second;
    if (a < 0 || a >= K || b < 0 || b >= K) throw std::invalid_argument("teaser: solveCloudPairs: no such cloud");
    pc[2 * p] = a;
    pc[2 * p + 1] = b;
    seeds[p] = tuple_seeds ? (*tuple_seeds)[p] : cp.tuple_seed + 0x9E3779B97F4A7C15ull * static_cast<uint64_t>(p);
    const size_t cap = static_cast<size_t>(n[a]) + n[b];
    corr[p].resize(2 * cap);
    clq[p].resize(cap);
    corr_p[p] = corr[p].data();
    clq_p[p] = clq[p].data();
  }
  tzr_frontend_params f;
  tzr_frontend_params_default(&f);
  f.normal_search_radius = cp.normal_search_radius;
  f.fpfh_search_radius = cp.fpfh_search_radius;
  f.use_absolute_scale = cp.use_absolute_scale ? 1 : 0;
  f.use_crosscheck = cp.use_crosscheck ? 1 : 0;
  f.use_tuple_test = cp.use_tuple_test ? 1 : 0;
  f.tuple_scale = cp.tuple_scale;
  std::vector<tzr_solution> sols(P);
  std::vector<int64_t> n_corr(P);
  std::vector<float> scales(P);
  tzr_ctx* ctx = b200_context();
  int rc;
  if (!icp) {
    rc = tzr_register_cloud_pairs(ctx, &f, &p, K, n.data(), pts.data(), P, pc.data(), seeds.data(), sols.data(),
                                  status.data(), index.data(), n_corr.data(), corr_p.data(), clq_p.data(),
                                  scales.data());
  } else {
    icp_res->assign(P, tzr_icp_result{});
    tzr_robust_kernel k;
    std::memset(&k, 0, sizeof(k));
    if (kernel) {
      k.type = static_cast<int32_t>(kernel->type);
      k.k = kernel->k;
    }
    if (mw && mw->G > 0) {
      const bool colored = method == IcpMethod::kColored;
      const float* const* cl = colored ? col.data() : nullptr;
      const double lam = colored ? lambda_geometric : 0.0;
      const tzr_robust_kernel* kp = colored && kernel ? &k : nullptr;
      rc = mw->lp ? tzr_register_cloud_pairs_multiway_line_process_batch(
                        ctx, &f, &p, K, n.data(), pts.data(), P, pc.data(), seeds.data(), sols.data(), status.data(),
                        index.data(), n_corr.data(), corr_p.data(), clq_p.data(), scales.data(), icp, cl, lam, kp,
                        icp_res->data(), mw->uncertain, mw->lp, mw->information, mw->info_counts, mw->edge_weights,
                        mw->edge_mask, mw->poses, mw->lp_summary, mw->pg_status, mw->G, mw->graph_offsets,
                        mw->map_voxel_size, mw->map_points, mw->map_counts, mw->map_colors)
                  : tzr_register_cloud_pairs_multiway_batch(
                        ctx, &f, &p, K, n.data(), pts.data(), P, pc.data(), seeds.data(), sols.data(), status.data(),
                        index.data(), n_corr.data(), corr_p.data(), clq_p.data(), scales.data(), icp, cl, lam, kp,
                        icp_res->data(), mw->uncertain, mw->pg, mw->information, mw->info_counts, mw->edge_weights,
                        mw->edge_mask, mw->poses, mw->summary, mw->pg_status, mw->G, mw->graph_offsets,
                        mw->map_voxel_size, mw->map_points, mw->map_counts, mw->map_colors);
    } else if (mw && mw->lp) {
      const bool colored = method == IcpMethod::kColored;
      rc = tzr_register_cloud_pairs_multiway_line_process(
          ctx, &f, &p, K, n.data(), pts.data(), P, pc.data(), seeds.data(), sols.data(), status.data(), index.data(),
          n_corr.data(), corr_p.data(), clq_p.data(), scales.data(), icp, colored ? col.data() : nullptr,
          colored ? lambda_geometric : 0.0, colored && kernel ? &k : nullptr, icp_res->data(), mw->uncertain, mw->lp,
          mw->information, mw->info_counts, mw->edge_weights, mw->edge_mask, mw->poses, mw->lp_summary,
          mw->pg_status);
    } else if (mw && method == IcpMethod::kColored) {
      rc = tzr_register_cloud_pairs_multiway_colored(
          ctx, &f, &p, K, n.data(), pts.data(), P, pc.data(), seeds.data(), sols.data(), status.data(), index.data(),
          n_corr.data(), corr_p.data(), clq_p.data(), scales.data(), icp, col.data(), lambda_geometric,
          kernel ? &k : nullptr, icp_res->data(), mw->uncertain, mw->pg, mw->information, mw->info_counts,
          mw->edge_weights, mw->edge_mask, mw->poses, mw->summary, mw->pg_status);
    } else if (mw) {
      rc = tzr_register_cloud_pairs_multiway(ctx, &f, &p, K, n.data(), pts.data(), P, pc.data(), seeds.data(),
                                             sols.data(), status.data(), index.data(), n_corr.data(), corr_p.data(),
                                             clq_p.data(), scales.data(), icp, icp_res->data(), mw->uncertain, mw->pg,
                                             mw->information, mw->info_counts, mw->edge_weights, mw->edge_mask,
                                             mw->poses, mw->summary, mw->pg_status);
    } else if (method == IcpMethod::kColored) {
      rc = tzr_register_cloud_pairs_icp_colored(ctx, &f, &p, K, n.data(), pts.data(), P, pc.data(), seeds.data(),
                                                sols.data(), status.data(), index.data(), n_corr.data(), corr_p.data(),
                                                clq_p.data(), scales.data(), icp, col.data(), lambda_geometric,
                                                kernel ? &k : nullptr, icp_res->data());
    } else if (kernel) {
      rc = tzr_register_cloud_pairs_icp_robust(ctx, &f, &p, K, n.data(), pts.data(), P, pc.data(), seeds.data(),
                                               sols.data(), status.data(), index.data(), n_corr.data(), corr_p.data(),
                                               clq_p.data(), scales.data(), icp,
                                               method == IcpMethod::kGeneralized ? 2 : 1, epsilon, &k,
                                               icp_res->data());
    } else if (method == IcpMethod::kGeneralized)
      rc = tzr_register_cloud_pairs_icp_generalized(ctx, &f, &p, K, n.data(), pts.data(), P, pc.data(), seeds.data(),
                                                    sols.data(), status.data(), index.data(), n_corr.data(),
                                                    corr_p.data(), clq_p.data(), scales.data(), icp, epsilon,
                                                    icp_res->data());
    else
      rc = (method == IcpMethod::kPointToPlane ? tzr_register_cloud_pairs_icp_point_to_plane
                                               : tzr_register_cloud_pairs_icp)(
          ctx, &f, &p, K, n.data(), pts.data(), P, pc.data(), seeds.data(), sols.data(), status.data(), index.data(),
          n_corr.data(), corr_p.data(), clq_p.data(), scales.data(), icp, icp_res->data());
  }
  if (rc != TZR_OK && rc != TZR_ERR_TOO_LARGE) fail("RobustRegistrationSolver::solveCloudPairs", rc, ctx);
  for (int q = 0; q < P; ++q) {
    CloudPairResult& r = out[q];
    r.status = status[q];
    r.global_scale = scales[q];
    r.correspondences.reserve(static_cast<size_t>(n_corr[q]));
    for (int64_t c = 0; c < n_corr[q]; ++c) r.correspondences.emplace_back(corr[q][2 * c], corr[q][2 * c + 1]);
    r.solution.valid = sols[q].valid != 0;
    r.solution.scale = sols[q].scale;
    for (int k = 0; k < 3; ++k) r.solution.translation(k) = sols[q].translation[k];
    std::memcpy(r.solution.rotation.data(), sols[q].rotation, sizeof(sols[q].rotation));
    if (index[q] >= 0) r.max_clique.assign(clq[q].begin(), clq[q].begin() + std::max(0, sols[q].clique_size));
  }
  return out;
}

}  // namespace

std::vector<RobustRegistrationSolver::CloudPairResult> RobustRegistrationSolver::solveCloudPairs(
    const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& cp) {
  return run_cloud_pairs(to_c(params_), clouds, pairs, cp, nullptr, nullptr);
}

// every ICP overload of solveCloudPairs
static std::vector<RobustRegistrationSolver::CloudPairICPResult> run_cloud_pairs_icp(
    const tzr_params& p, const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs,
    const RobustRegistrationSolver::CloudPairParams& cp, const PointToPointICPParams& icp, IcpMethod method,
    double epsilon = 0, const RobustKernel* kernel = nullptr, const std::vector<ColorCloud>* colors = nullptr,
    double lambda_geometric = 0) {
  using CloudPairResult = RobustRegistrationSolver::CloudPairResult;
  using CloudPairICPResult = RobustRegistrationSolver::CloudPairICPResult;
  tzr_icp_params ip;
  tzr_icp_params_default(&ip);
  ip.max_correspondence_distance = icp.max_correspondence_distance;
  ip.max_iteration = icp.max_iteration;
  ip.relative_fitness = icp.relative_fitness;
  ip.relative_rmse = icp.relative_rmse;
  std::vector<tzr_icp_result> res;
  std::vector<CloudPairResult> base =
      run_cloud_pairs(p, clouds, pairs, cp, &ip, &res, method, epsilon, kernel, nullptr, colors, lambda_geometric);
  std::vector<CloudPairICPResult> out(base.size());
  for (size_t q = 0; q < base.size(); ++q) {
    static_cast<CloudPairResult&>(out[q]) = std::move(base[q]);
    // a refined pair: solved with a valid solution (the library zeroes every other pair's record)
    out[q].refined = out[q].status == TZR_OK && out[q].solution.valid && res[q].transform.scale > 0;
    if (out[q].refined) icp_result_from_c(res[q], nullptr, &out[q].icp);
  }
  return out;
}

// Open3D's tutorial rule: pair (k, k + 1) certain, every other pair uncertain
static std::vector<bool> tutorial_uncertain(const std::vector<std::pair<int, int>>& pairs) {
  std::vector<bool> uncertain(pairs.size());
  for (size_t q = 0; q < pairs.size(); ++q) uncertain[q] = pairs[q].second != pairs[q].first + 1;
  return uncertain;
}

// One sequence's MultiwayResult from the multiway outputs: its P pairs from pair q0 of base, res and the per-pair
// arrays, its K poses from poses, its status and summaries
static RobustRegistrationSolver::MultiwayResult multiway_result(
    std::vector<RobustRegistrationSolver::CloudPairResult>& base, const std::vector<tzr_icp_result>& res,
    const double* info, const int32_t* counts, const double* w, const uint8_t* mask, size_t q0, size_t P,
    const tzr_similarity* poses, size_t K, int32_t pg_status, const tzr_pose_graph_summary& summary,
    const tzr_line_process_summary& lp_summary) {
  using CloudPairResult = RobustRegistrationSolver::CloudPairResult;
  RobustRegistrationSolver::MultiwayResult out;
  out.pairs.resize(P);
  out.information.resize(P);
  out.information_counts.assign(counts + q0, counts + q0 + P);
  out.edge_weights.assign(w + q0, w + q0 + P);
  out.edge_inliers.resize(P);
  for (size_t j = 0; j < P; ++j) {
    const size_t q = q0 + j;
    static_cast<CloudPairResult&>(out.pairs[j]) = std::move(base[q]);
    out.pairs[j].refined = out.pairs[j].status == TZR_OK && out.pairs[j].solution.valid && res[q].transform.scale > 0;
    if (out.pairs[j].refined) icp_result_from_c(res[q], nullptr, &out.pairs[j].icp);
    for (int r = 0; r < 6; ++r)
      for (int c = 0; c < 6; ++c) out.information[j](r, c) = info[36 * q + 6 * r + c];
    out.edge_inliers[j] = mask[q] != 0;
  }
  out.poses.resize(K);
  for (size_t k = 0; k < K; ++k) {
    Eigen::Matrix4d T = Eigen::Matrix4d::Zero();
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) T(r, c) = poses[k].rotation[3 * c + r];
      T(r, 3) = poses[k].translation[r];
    }
    T(3, 3) = 1.0;
    out.poses[k] = T;
  }
  out.pose_graph_status = pg_status;
  out.iterations = summary.iterations;
  out.inner_iterations = summary.inner_iterations;
  out.cost = summary.cost;
  for (int q = 0; q < 2; ++q) {
    out.line_process.iterations[q] = lp_summary.iterations[q];
    out.line_process.trials[q] = lp_summary.trials[q];
    out.line_process.stop_reason[q] = lp_summary.stop_reason[q];
    out.line_process.mu[q] = lp_summary.mu[q];
  }
  out.line_process.pruned = lp_summary.pruned;
  out.line_process.residual = lp_summary.residual;
  return out;
}

// every solveMultiway overload: point-to-plane without colours, coloured ICP with them
static RobustRegistrationSolver::MultiwayResult run_multiway(
    const tzr_params& p, const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs,
    const RobustRegistrationSolver::CloudPairParams& cp, const PointToPointICPParams& icp,
    const PoseGraphParams& pose_graph, const std::vector<bool>& uncertain,
    const std::vector<ColorCloud>* colors = nullptr, double lambda_geometric = 0,
    const RobustKernel* kernel = nullptr, const LineProcessParams* line_process = nullptr) {
  using CloudPairResult = RobustRegistrationSolver::CloudPairResult;
  const size_t P = pairs.size(), K = clouds.size();
  if (uncertain.size() != P) throw std::invalid_argument("teaser: solveMultiway: one uncertain flag per pair");
  tzr_icp_params ip;
  tzr_icp_params_default(&ip);
  ip.max_correspondence_distance = icp.max_correspondence_distance;
  ip.max_iteration = icp.max_iteration;
  ip.relative_fitness = icp.relative_fitness;
  ip.relative_rmse = icp.relative_rmse;
  tzr_pose_graph_params pg = pose_graph_c(pose_graph);
  std::vector<int32_t> unc(P), counts(P);
  for (size_t q = 0; q < P; ++q) unc[q] = uncertain[q] ? 1 : 0;
  std::vector<double> info(P * 36), w(P);
  std::vector<uint8_t> mask(P);
  std::vector<tzr_similarity> poses(K);
  tzr_pose_graph_summary summary{};
  int32_t pg_status = 0;
  MultiwayCall mw{unc.data(), &pg, info.data(), counts.data(), w.data(), mask.data(), poses.data(), &summary,
                  &pg_status};
  tzr_line_process_params lp;
  tzr_line_process_summary lp_summary{};
  if (line_process) {
    lp = line_process_c(*line_process);
    mw.lp = &lp;
    mw.lp_summary = &lp_summary;
  }
  std::vector<tzr_icp_result> res;
  std::vector<CloudPairResult> base =
      run_cloud_pairs(p, clouds, pairs, cp, &ip, &res, colors ? IcpMethod::kColored : IcpMethod::kPointToPlane, 0,
                      kernel, &mw, colors, lambda_geometric);
  return multiway_result(base, res, info.data(), counts.data(), w.data(), mask.data(), 0, P, poses.data(), K, pg_status,
                         summary, lp_summary);
}

// both solveMultiwayBatch overloads: the sequences flattened into one table (pair j of a sequence keeps its solo tuple
// seed), one call, the outputs split back per sequence
static std::vector<RobustRegistrationSolver::MultiwayResult> run_multiway_batch(
    const tzr_params& p, const std::vector<RobustRegistrationSolver::MultiwaySequence>& seqs,
    const RobustRegistrationSolver::CloudPairParams& cp, const ColoredICPParams& icp, const PoseGraphParams& pose_graph,
    const LineProcessParams* line_process, double map_voxel_size, const RobustKernel& kernel) {
  using CloudPairResult = RobustRegistrationSolver::CloudPairResult;
  const size_t G = seqs.size();
  if (G == 0) throw std::invalid_argument("teaser: solveMultiwayBatch: at least one sequence is required");
  const bool colored = !seqs[0].colors.empty();
  if (!colored && kernel.type != RobustKernel::kL2)
    throw std::invalid_argument("teaser: solveMultiwayBatch: a robust kernel needs colours (coloured ICP)");
  std::vector<PointCloud> clouds;
  std::vector<ColorCloud> colors;
  std::vector<std::pair<int, int>> pairs;
  std::vector<int32_t> unc, off{0};
  std::vector<uint64_t> seeds;
  std::vector<size_t> pair_off{0}, points(G, 0);
  for (size_t g = 0; g < G; ++g) {
    const auto& s = seqs[g];
    if (s.colors.empty() == colored)
      throw std::invalid_argument("teaser: solveMultiwayBatch: every sequence has colours, or none has");
    if (!s.uncertain.empty() && s.uncertain.size() != s.pairs.size())
      throw std::invalid_argument("teaser: solveMultiwayBatch: one uncertain flag per pair");
    const int K = static_cast<int>(s.clouds.size());
    for (size_t j = 0; j < s.pairs.size(); ++j) {
      const auto& q = s.pairs[j];
      if (q.first < 0 || q.first >= K || q.second < 0 || q.second >= K)
        throw std::invalid_argument("teaser: solveMultiwayBatch: a pair names a cloud outside its sequence");
      pairs.emplace_back(off.back() + q.first, off.back() + q.second);
      unc.push_back(s.uncertain.empty() ? (q.second != q.first + 1) : s.uncertain[j]);
      seeds.push_back(cp.tuple_seed + 0x9E3779B97F4A7C15ull * static_cast<uint64_t>(j));
    }
    for (const auto& c : s.clouds) points[g] += c.size();
    clouds.insert(clouds.end(), s.clouds.begin(), s.clouds.end());
    colors.insert(colors.end(), s.colors.begin(), s.colors.end());
    off.push_back(off.back() + K);
    pair_off.push_back(pairs.size());
  }
  const size_t P = pairs.size(), K = clouds.size();
  tzr_icp_params ip;
  tzr_icp_params_default(&ip);
  ip.max_correspondence_distance = icp.max_correspondence_distance;
  ip.max_iteration = icp.max_iteration;
  ip.relative_fitness = icp.relative_fitness;
  ip.relative_rmse = icp.relative_rmse;
  tzr_pose_graph_params pg = pose_graph_c(pose_graph);
  std::vector<int32_t> counts(P), status(G), map_counts(G);
  std::vector<double> info(P * 36), w(P);
  std::vector<uint8_t> mask(P);
  std::vector<tzr_similarity> poses(K);
  std::vector<tzr_pose_graph_summary> summary(G);
  std::vector<tzr_line_process_summary> lp_summary(G);
  std::vector<std::vector<float>> maps(G), map_cols(G);
  std::vector<float*> map_p(G), map_c(G);
  const bool with_map = map_voxel_size > 0;
  for (size_t g = 0; g < G && with_map; ++g) {
    maps[g].resize(3 * std::max<size_t>(points[g], 1));
    map_p[g] = maps[g].data();
    if (colored) {
      map_cols[g].resize(maps[g].size());
      map_c[g] = map_cols[g].data();
    }
  }
  MultiwayCall mw{unc.data(), &pg, info.data(), counts.data(), w.data(), mask.data(), poses.data(), summary.data(),
                  status.data()};
  tzr_line_process_params lp;
  if (line_process) {
    lp = line_process_c(*line_process);
    mw.lp = &lp;
    mw.lp_summary = lp_summary.data();
  }
  mw.G = static_cast<int>(G);
  mw.graph_offsets = off.data();
  mw.map_voxel_size = map_voxel_size;
  mw.map_points = with_map ? map_p.data() : nullptr;
  mw.map_counts = with_map ? map_counts.data() : nullptr;
  mw.map_colors = with_map && colored ? map_c.data() : nullptr;
  std::vector<tzr_icp_result> res;
  std::vector<CloudPairResult> base =
      run_cloud_pairs(p, clouds, pairs, cp, &ip, &res, colored ? IcpMethod::kColored : IcpMethod::kPointToPlane, 0,
                      colored ? &kernel : nullptr, &mw, colored ? &colors : nullptr, icp.lambda_geometric, &seeds);
  std::vector<RobustRegistrationSolver::MultiwayResult> out;
  for (size_t g = 0; g < G; ++g) {
    out.push_back(multiway_result(base, res, info.data(), counts.data(), w.data(), mask.data(), pair_off[g],
                                  pair_off[g + 1] - pair_off[g], poses.data() + off[g], off[g + 1] - off[g], status[g],
                                  summary[g], lp_summary[g]));
    for (int32_t r = 0; with_map && r < map_counts[g]; ++r) {
      out.back().map.push_back(PointXYZ{maps[g][3 * r], maps[g][3 * r + 1], maps[g][3 * r + 2]});
      if (colored) out.back().map_colors.push_back(ColorRGB{map_cols[g][3 * r], map_cols[g][3 * r + 1],
                                                            map_cols[g][3 * r + 2]});
    }
  }
  return out;
}

std::vector<RobustRegistrationSolver::MultiwayResult> RobustRegistrationSolver::solveMultiwayBatch(
    const std::vector<MultiwaySequence>& sequences, const CloudPairParams& cp, const ColoredICPParams& icp,
    const PoseGraphParams& pose_graph, double map_voxel_size, const RobustKernel& kernel) {
  return run_multiway_batch(to_c(params_), sequences, cp, icp, pose_graph, nullptr, map_voxel_size, kernel);
}

std::vector<RobustRegistrationSolver::MultiwayResult> RobustRegistrationSolver::solveMultiwayBatch(
    const std::vector<MultiwaySequence>& sequences, const CloudPairParams& cp, const ColoredICPParams& icp,
    const LineProcessParams& global_optimization, double map_voxel_size, const RobustKernel& kernel) {
  return run_multiway_batch(to_c(params_), sequences, cp, icp, PoseGraphParams(), &global_optimization,
                            map_voxel_size, kernel);
}

RobustRegistrationSolver::MultiwayResult RobustRegistrationSolver::solveMultiway(
    const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& cp,
    const PointToPointICPParams& icp, const LineProcessParams& global_optimization) {
  return solveMultiway(clouds, pairs, cp, icp, global_optimization, tutorial_uncertain(pairs));
}

RobustRegistrationSolver::MultiwayResult RobustRegistrationSolver::solveMultiway(
    const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& cp,
    const PointToPointICPParams& icp, const LineProcessParams& global_optimization,
    const std::vector<bool>& uncertain) {
  return run_multiway(to_c(params_), clouds, pairs, cp, icp, PoseGraphParams(), uncertain, nullptr, 0, nullptr,
                      &global_optimization);
}

RobustRegistrationSolver::MultiwayResult RobustRegistrationSolver::solveMultiway(
    const std::vector<PointCloud>& clouds, const std::vector<ColorCloud>& colors,
    const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& cp, const ColoredICPParams& icp,
    const LineProcessParams& global_optimization, const RobustKernel& kernel) {
  return solveMultiway(clouds, colors, pairs, cp, icp, global_optimization, tutorial_uncertain(pairs), kernel);
}

RobustRegistrationSolver::MultiwayResult RobustRegistrationSolver::solveMultiway(
    const std::vector<PointCloud>& clouds, const std::vector<ColorCloud>& colors,
    const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& cp, const ColoredICPParams& icp,
    const LineProcessParams& global_optimization, const std::vector<bool>& uncertain, const RobustKernel& kernel) {
  return run_multiway(to_c(params_), clouds, pairs, cp, icp, PoseGraphParams(), uncertain, &colors,
                      icp.lambda_geometric, &kernel, &global_optimization);
}

RobustRegistrationSolver::MultiwayResult RobustRegistrationSolver::solveMultiway(
    const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& cp,
    const PointToPointICPParams& icp, const PoseGraphParams& pose_graph) {
  return run_multiway(to_c(params_), clouds, pairs, cp, icp, pose_graph, tutorial_uncertain(pairs));
}

RobustRegistrationSolver::MultiwayResult RobustRegistrationSolver::solveMultiway(
    const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& cp,
    const PointToPointICPParams& icp, const PoseGraphParams& pose_graph, const std::vector<bool>& uncertain) {
  return run_multiway(to_c(params_), clouds, pairs, cp, icp, pose_graph, uncertain);
}

RobustRegistrationSolver::MultiwayResult RobustRegistrationSolver::solveMultiway(
    const std::vector<PointCloud>& clouds, const std::vector<ColorCloud>& colors,
    const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& cp, const ColoredICPParams& icp,
    const PoseGraphParams& pose_graph, const RobustKernel& kernel) {
  return solveMultiway(clouds, colors, pairs, cp, icp, pose_graph, tutorial_uncertain(pairs), kernel);
}

RobustRegistrationSolver::MultiwayResult RobustRegistrationSolver::solveMultiway(
    const std::vector<PointCloud>& clouds, const std::vector<ColorCloud>& colors,
    const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& cp, const ColoredICPParams& icp,
    const PoseGraphParams& pose_graph, const std::vector<bool>& uncertain, const RobustKernel& kernel) {
  return run_multiway(to_c(params_), clouds, pairs, cp, icp, pose_graph, uncertain, &colors, icp.lambda_geometric,
                      &kernel);
}

std::vector<RobustRegistrationSolver::CloudPairICPResult> RobustRegistrationSolver::solveCloudPairs(
    const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& cp,
    const PointToPointICPParams& icp) {
  return run_cloud_pairs_icp(to_c(params_), clouds, pairs, cp, icp, IcpMethod::kPointToPoint);
}

std::vector<RobustRegistrationSolver::CloudPairICPResult> RobustRegistrationSolver::solveCloudPairsPointToPlane(
    const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& cp,
    const PointToPointICPParams& icp) {
  return run_cloud_pairs_icp(to_c(params_), clouds, pairs, cp, icp, IcpMethod::kPointToPlane);
}

std::vector<RobustRegistrationSolver::CloudPairICPResult> RobustRegistrationSolver::solveCloudPairsGeneralizedICP(
    const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& cp,
    const GeneralizedICPParams& icp) {
  return run_cloud_pairs_icp(to_c(params_), clouds, pairs, cp, icp, IcpMethod::kGeneralized, icp.epsilon);
}

std::vector<RobustRegistrationSolver::CloudPairICPResult> RobustRegistrationSolver::solveCloudPairsPointToPlane(
    const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& cp,
    const PointToPointICPParams& icp, const RobustKernel& kernel) {
  return run_cloud_pairs_icp(to_c(params_), clouds, pairs, cp, icp, IcpMethod::kPointToPlane, 0, &kernel);
}

std::vector<RobustRegistrationSolver::CloudPairICPResult> RobustRegistrationSolver::solveCloudPairsGeneralizedICP(
    const std::vector<PointCloud>& clouds, const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& cp,
    const GeneralizedICPParams& icp, const RobustKernel& kernel) {
  return run_cloud_pairs_icp(to_c(params_), clouds, pairs, cp, icp, IcpMethod::kGeneralized, icp.epsilon, &kernel);
}

std::vector<RobustRegistrationSolver::CloudPairICPResult> RobustRegistrationSolver::solveCloudPairsColoredICP(
    const std::vector<PointCloud>& clouds, const std::vector<ColorCloud>& colors,
    const std::vector<std::pair<int, int>>& pairs, const CloudPairParams& cp, const ColoredICPParams& icp,
    const RobustKernel& kernel) {
  return run_cloud_pairs_icp(to_c(params_), clouds, pairs, cp, icp, IcpMethod::kColored, 0, &kernel, &colors,
                             icp.lambda_geometric);
}

void RobustRegistrationSolver::materialise_tims() {
  if (have_tims_ || !solved_) return;
  src_tims_ = computeTIMs(last_src_, &src_tims_map_);
  dst_tims_ = computeTIMs(last_dst_, &dst_tims_map_);
  materialise_graph();
  const Eigen::Index K = src_tims_.cols();
  scale_inliers_mask_.resize(1, K);
  for (Eigen::Index k = 0; k < K; ++k)
    scale_inliers_mask_(k) = inlier_graph_.numVertices() ? inlier_graph_.hasEdge(src_tims_map_(0, k), src_tims_map_(1, k))
                                                         : false;
  have_tims_ = true;
}

BoolRow RobustRegistrationSolver::getScaleInliersMask() {
  materialise_tims();
  return scale_inliers_mask_;
}
Map2X RobustRegistrationSolver::getScaleInliersMap() {
  materialise_tims();
  return src_tims_map_;
}
std::vector<std::tuple<int, int>> RobustRegistrationSolver::getScaleInliers() {
  materialise_graph();
  std::vector<std::tuple<int, int>> out;
  for (int v = 0; v < inlier_graph_.numVertices(); ++v)
    for (int u : inlier_graph_.getEdges(v))
      if (u > v) out.emplace_back(v, u);
  return out;
}
Eigen::Matrix<int, 1, Eigen::Dynamic> RobustRegistrationSolver::getRotationInliersMap() {
  Eigen::Matrix<int, 1, Eigen::Dynamic> m(1, static_cast<Eigen::Index>(max_clique_.size()));
  for (size_t i = 0; i < max_clique_.size(); ++i) m(static_cast<Eigen::Index>(i)) = max_clique_[i];
  return m;
}
Eigen::Matrix<int, 1, Eigen::Dynamic> RobustRegistrationSolver::getTranslationInliersMap() {
  return getRotationInliersMap();
}
std::vector<int> RobustRegistrationSolver::getInputOrderedTranslationInliers() {
  if (params_.rotation_estimation_algorithm == ROTATION_ESTIMATION_ALGORITHM::FGR)
    throw std::runtime_error("This function is not supported when using FGR since FGR does not use max clique.");
  std::vector<int> out;
  out.reserve(translation_inliers_.size());
  for (int i : translation_inliers_) out.push_back(max_clique_[i]);
  return out;
}
std::vector<std::vector<int>> RobustRegistrationSolver::getInlierGraph() {
  materialise_graph();
  return inlier_graph_.getAdjList();
}
Mat3X RobustRegistrationSolver::getSrcTIMs() {
  materialise_tims();
  return src_tims_;
}
Mat3X RobustRegistrationSolver::getDstTIMs() {
  materialise_tims();
  return dst_tims_;
}
Map2X RobustRegistrationSolver::getSrcTIMsMap() {
  materialise_tims();
  return src_tims_map_;
}
Map2X RobustRegistrationSolver::getDstTIMsMap() {
  materialise_tims();
  return dst_tims_map_;
}

}  // namespace teaser
