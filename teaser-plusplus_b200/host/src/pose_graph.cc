// teaser::informationMatrix(Batch) and teaser::PoseGraph (teaser/pose_graph.h) on top of the C-ABI: marshalling only,
// the sums and the solve run in libteaser_b200.so.
#include "teaser/pose_graph.h"

#include <cstring>
#include <stdexcept>
#include <string>

#include "teaser_b200.h"

namespace teaser {

tzr_ctx* b200_context();  // registration.cc: one context per host thread

namespace {

[[noreturn]] void fail(const char* who, int rc, tzr_ctx* ctx) {
  throw std::runtime_error(std::string(who) + ": " + tzr_status_string(rc) + ": " + tzr_last_error(ctx));
}

tzr_similarity sim_of(const RegistrationSolution& s) {
  tzr_similarity c;
  c.scale = s.scale;
  std::memcpy(c.rotation, s.rotation.data(), sizeof(c.rotation));
  for (int k = 0; k < 3; ++k) c.translation[k] = s.translation(k);
  return c;
}

tzr_similarity sim_of(const Eigen::Matrix4d& T) {
  tzr_similarity c;
  c.scale = 1.0;
  for (int r = 0; r < 3; ++r) {
    for (int col = 0; col < 3; ++col) c.rotation[3 * col + r] = T(r, col);
    c.translation[r] = T(r, 3);
  }
  return c;
}

Eigen::Matrix4d matrix_of(const tzr_similarity& s) {
  Eigen::Matrix4d T = Eigen::Matrix4d::Zero();
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) T(r, c) = s.rotation[3 * c + r];
    T(r, 3) = s.translation[r];
  }
  T(3, 3) = 1.0;
  return T;
}

Matrix6d matrix6_of(const double* L) {
  Matrix6d M;
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c) M(r, c) = L[6 * r + c];
  return M;
}

// The pointer-per-graph arrays of both optimisers' C calls (a single call's graph is a batch of one), and per graph the
// outputs: poses (K), a double (E), a byte (E) and a double (E) array
struct GraphArrays {
  std::vector<int32_t> K, E, status;
  std::vector<std::vector<int32_t>> ends, unc;
  std::vector<std::vector<tzr_similarity>> tr, init, poses;
  std::vector<std::vector<double>> L, d1, d2;
  std::vector<std::vector<uint8_t>> u8;
  std::vector<const int32_t*> ep, up;
  std::vector<const tzr_similarity*> tp, ip;
  std::vector<const double*> Lp;
  std::vector<tzr_similarity*> pp;
  std::vector<double*> d1p, d2p;
  std::vector<uint8_t*> u8p;

  GraphArrays(const std::vector<PoseGraph::Graph>& graphs, const char* who) {
    const size_t G = graphs.size(), P = G ? G : 1;
    K.resize(P);
    E.resize(P);
    status.resize(P);
    ends.resize(G);
    unc.resize(G);
    tr.resize(G);
    init.resize(G);
    poses.resize(G);
    L.resize(G);
    d1.resize(G);
    d2.resize(G);
    u8.resize(G);
    ep.resize(P);
    up.resize(P);
    tp.resize(P);
    ip.resize(P);
    Lp.resize(P);
    pp.resize(P);
    d1p.resize(P);
    d2p.resize(P);
    u8p.resize(P);
    for (size_t g = 0; g < G; ++g) {
      const PoseGraph::Graph& gr = graphs[g];
      const size_t Eg = gr.edges.size();
      if (!gr.initial_poses.empty() && gr.initial_poses.size() != static_cast<size_t>(gr.num_nodes))
        throw std::invalid_argument(std::string(who) + ": one initial pose per node");
      for (const PoseGraph::Edge& e : gr.edges) {
        ends[g].push_back(e.source);
        ends[g].push_back(e.target);
        unc[g].push_back(e.uncertain ? 1 : 0);
        tr[g].push_back(sim_of(e.transform));
        for (int r = 0; r < 6; ++r)
          for (int c = 0; c < 6; ++c) L[g].push_back(e.information(r, c));
      }
      for (const Eigen::Matrix4d& T : gr.initial_poses) init[g].push_back(sim_of(T));
      K[g] = gr.num_nodes;
      E[g] = static_cast<int32_t>(Eg);
      poses[g].resize(gr.num_nodes > 0 ? gr.num_nodes : 1);
      d1[g].resize(Eg ? Eg : 1);
      d2[g].resize(Eg ? Eg : 1);
      u8[g].resize(Eg ? Eg : 1);
      ep[g] = ends[g].data();
      up[g] = unc[g].data();
      tp[g] = tr[g].data();
      Lp[g] = L[g].data();
      ip[g] = gr.initial_poses.empty() ? nullptr : init[g].data();
      pp[g] = poses[g].data();
      d1p[g] = d1[g].data();
      d2p[g] = d2[g].data();
      u8p[g] = u8[g].data();
    }
  }
};

// The single calls' graph as a batch of one.  A non-null initial_poses must hold num_nodes poses, even none:
// GraphArrays reads an empty list as the breadth-first start.
std::vector<PoseGraph::Graph> one_graph(int num_nodes, const std::vector<PoseGraph::Edge>& edges,
                                        const std::vector<Eigen::Matrix4d>* initial_poses, const char* who) {
  if (initial_poses && initial_poses->size() != static_cast<size_t>(num_nodes))
    throw std::invalid_argument(std::string(who) + ": one initial pose per node");
  std::vector<PoseGraph::Graph> gs(1);
  gs[0].num_nodes = num_nodes;
  gs[0].edges = edges;
  if (initial_poses) gs[0].initial_poses = *initial_poses;
  return gs;
}

// Graph g's results, of either call of each optimiser
PoseGraph::Result pose_graph_result(const GraphArrays& a, size_t g, const tzr_pose_graph_summary& s) {
  PoseGraph::Result r;
  const size_t E = a.E[g];
  for (int k = 0; k < a.K[g]; ++k) r.poses.push_back(matrix_of(a.poses[g][k]));
  r.weights.assign(a.d1[g].begin(), a.d1[g].begin() + E);
  for (size_t e = 0; e < E; ++e) r.inliers.push_back(a.u8[g][e] != 0);
  r.residuals.assign(a.d2[g].begin(), a.d2[g].begin() + E);
  r.iterations = s.iterations;
  r.inner_iterations = s.inner_iterations;
  r.cost = s.cost;
  return r;
}

GlobalOptimization::Result line_process_result(const GraphArrays& a, size_t g, const tzr_line_process_summary& s) {
  GlobalOptimization::Result r;
  const size_t E = a.E[g];
  for (int k = 0; k < a.K[g]; ++k) r.poses.push_back(matrix_of(a.poses[g][k]));
  r.confidence.assign(a.d1[g].begin(), a.d1[g].begin() + E);
  for (size_t e = 0; e < E; ++e) r.kept.push_back(a.u8[g][e] != 0);
  r.residuals.assign(a.d2[g].begin(), a.d2[g].begin() + E);
  for (int q = 0; q < 2; ++q) {
    r.summary.iterations[q] = s.iterations[q];
    r.summary.trials[q] = s.trials[q];
    r.summary.stop_reason[q] = s.stop_reason[q];
    r.summary.mu[q] = s.mu[q];
  }
  r.summary.pruned = s.pruned;
  r.summary.residual = s.residual;
  return r;
}

}  // namespace

tzr_pose_graph_params pose_graph_c(const PoseGraphParams& q) {
  tzr_pose_graph_params p;
  tzr_pose_graph_params_default(&p);
  p.max_correspondence_distance = q.max_correspondence_distance;
  p.gnc_factor = q.gnc_factor;
  p.cost_threshold = q.cost_threshold;
  p.max_iterations = q.max_iterations;
  p.max_inner_iterations = q.max_inner_iterations;
  p.reference_node = q.reference_node;
  return p;
}

tzr_line_process_params line_process_c(const LineProcessParams& q) {
  tzr_line_process_params p;
  tzr_line_process_params_default(&p);
  p.max_correspondence_distance = q.max_correspondence_distance;
  p.edge_prune_threshold = q.edge_prune_threshold;
  p.preference_loop_closure = q.preference_loop_closure;
  p.reference_node = q.reference_node;
  p.max_iteration = q.max_iteration;
  p.min_relative_increment = q.min_relative_increment;
  p.min_relative_residual_increment = q.min_relative_residual_increment;
  p.min_right_term = q.min_right_term;
  p.min_residual = q.min_residual;
  p.max_iteration_lm = q.max_iteration_lm;
  p.upper_scale_factor = q.upper_scale_factor;
  p.lower_scale_factor = q.lower_scale_factor;
  return p;
}

std::vector<Matrix6d> informationMatrixBatch(const std::vector<PointCloud>& src, const std::vector<PointCloud>& dst,
                                             const std::vector<RegistrationSolution>& T,
                                             double max_correspondence_distance, std::vector<int>* counts) {
  const size_t B = src.size();
  if (dst.size() != B || T.size() != B)
    throw std::invalid_argument("teaser::informationMatrixBatch: one target and one transform per source");
  std::vector<Matrix6d> out(B);
  if (counts) counts->assign(B, 0);
  if (B == 0) return out;
  static_assert(sizeof(PointXYZ) == 3 * sizeof(float), "PointXYZ must be three packed floats");
  std::vector<int32_t> ns(B), nd(B), cnt(B);
  std::vector<const float*> sp(B), dp(B);
  std::vector<tzr_similarity> tr(B);
  for (size_t b = 0; b < B; ++b) {
    if (src[b].empty() || dst[b].empty())
      throw std::invalid_argument("teaser::informationMatrixBatch: clouds must be non-empty");
    ns[b] = static_cast<int32_t>(src[b].size());
    nd[b] = static_cast<int32_t>(dst[b].size());
    sp[b] = &src[b][0].x;
    dp[b] = &dst[b][0].x;
    tr[b] = sim_of(T[b]);
  }
  std::vector<double> L(36 * B);
  tzr_ctx* ctx = b200_context();
  const int rc = tzr_information_matrix_batch(ctx, static_cast<int>(B), ns.data(), sp.data(), nd.data(), dp.data(),
                                              tr.data(), max_correspondence_distance, L.data(), cnt.data());
  if (rc != TZR_OK) fail("teaser::informationMatrixBatch", rc, ctx);
  for (size_t b = 0; b < B; ++b) {
    out[b] = matrix6_of(&L[36 * b]);
    if (counts) (*counts)[b] = cnt[b];
  }
  return out;
}

Matrix6d informationMatrix(const PointCloud& src, const PointCloud& dst, const RegistrationSolution& T,
                           double max_correspondence_distance, int* count) {
  if (src.empty() || dst.empty()) throw std::invalid_argument("teaser::informationMatrix: clouds must be non-empty");
  const tzr_similarity tr = sim_of(T);
  double L[36];
  int32_t cnt = 0;
  tzr_ctx* ctx = b200_context();
  const int rc = tzr_information_matrix(ctx, &src[0].x, static_cast<int>(src.size()), &dst[0].x,
                                        static_cast<int>(dst.size()), &tr, max_correspondence_distance, L, &cnt);
  if (rc != TZR_OK) fail("teaser::informationMatrix", rc, ctx);
  if (count) *count = cnt;
  return matrix6_of(L);
}

PoseGraph::Result PoseGraph::optimize(int num_nodes, const std::vector<Edge>& edges,
                                      const std::vector<Eigen::Matrix4d>* initial_poses) const {
  const tzr_pose_graph_params p = pose_graph_c(params_);
  const char* who = "teaser::PoseGraph::optimize";
  const GraphArrays a(one_graph(num_nodes, edges, initial_poses, who), who);
  tzr_pose_graph_summary s{};
  tzr_ctx* ctx = b200_context();
  const int rc = tzr_pose_graph_optimize(ctx, &p, a.K[0], a.E[0], a.ep[0], a.tp[0], a.Lp[0], a.up[0], a.ip[0],
                                         a.pp[0], a.d1p[0], a.u8p[0], a.d2p[0], &s);
  if (rc != TZR_OK) fail(who, rc, ctx);
  return pose_graph_result(a, 0, s);
}

GlobalOptimization::Result GlobalOptimization::optimize(int num_nodes, const std::vector<Edge>& edges,
                                                        const std::vector<Eigen::Matrix4d>* initial_poses) const {
  const tzr_line_process_params p = line_process_c(params_);
  const char* who = "teaser::GlobalOptimization::optimize";
  const GraphArrays a(one_graph(num_nodes, edges, initial_poses, who), who);
  tzr_line_process_summary s{};
  tzr_ctx* ctx = b200_context();
  const int rc = tzr_pose_graph_optimize_line_process(ctx, &p, a.K[0], a.E[0], a.ep[0], a.tp[0], a.Lp[0], a.up[0],
                                                      a.ip[0], a.pp[0], a.d1p[0], a.u8p[0], a.d2p[0], &s);
  if (rc != TZR_OK) fail(who, rc, ctx);
  return line_process_result(a, 0, s);
}

std::vector<PoseGraph::Result> PoseGraph::optimizeBatch(const std::vector<Graph>& graphs,
                                                        std::vector<int>* status) const {
  const size_t G = graphs.size();
  const tzr_pose_graph_params p = pose_graph_c(params_);
  GraphArrays a(graphs, "teaser::PoseGraph::optimizeBatch");
  std::vector<tzr_pose_graph_summary> s(G ? G : 1);
  tzr_ctx* ctx = b200_context();
  const int rc = tzr_pose_graph_optimize_batch(ctx, &p, static_cast<int>(G), a.K.data(), a.E.data(), a.ep.data(),
                                               a.tp.data(), a.Lp.data(), a.up.data(), a.ip.data(), a.pp.data(),
                                               a.d1p.data(), a.u8p.data(), a.d2p.data(), s.data(), a.status.data());
  if (rc != TZR_OK) fail("teaser::PoseGraph::optimizeBatch", rc, ctx);
  std::vector<Result> out(G);
  if (status) status->assign(a.status.begin(), a.status.begin() + G);
  for (size_t g = 0; g < G; ++g)
    if (a.status[g] == TZR_OK) out[g] = pose_graph_result(a, g, s[g]);
  return out;
}

std::vector<GlobalOptimization::Result> GlobalOptimization::optimizeBatch(const std::vector<Graph>& graphs,
                                                                          std::vector<int>* status) const {
  const size_t G = graphs.size();
  const tzr_line_process_params p = line_process_c(params_);
  GraphArrays a(graphs, "teaser::GlobalOptimization::optimizeBatch");
  std::vector<tzr_line_process_summary> s(G ? G : 1);
  tzr_ctx* ctx = b200_context();
  const int rc = tzr_pose_graph_optimize_line_process_batch(ctx, &p, static_cast<int>(G), a.K.data(), a.E.data(),
                                                            a.ep.data(), a.tp.data(), a.Lp.data(), a.up.data(),
                                                            a.ip.data(), a.pp.data(), a.d1p.data(), a.u8p.data(),
                                                            a.d2p.data(), s.data(), a.status.data());
  if (rc != TZR_OK) fail("teaser::GlobalOptimization::optimizeBatch", rc, ctx);
  std::vector<Result> out(G);
  if (status) status->assign(a.status.begin(), a.status.begin() + G);
  for (size_t g = 0; g < G; ++g)
    if (a.status[g] == TZR_OK) out[g] = line_process_result(a, g, s[g]);
  return out;
}

}  // namespace teaser
