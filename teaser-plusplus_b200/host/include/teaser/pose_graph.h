// Multiway registration on the GPU through the C-ABI (include/teaser_b200.h, DESIGN.md §3.16): Open3D's
// get_information_matrix_from_point_clouds (teaser::informationMatrix, informationMatrixBatch: tzr_information_matrix,
// tzr_information_matrix_batch) and a pose graph with GNC-TLS on its uncertain edges (teaser::PoseGraph:
// tzr_pose_graph_optimize; PoseGraph::optimizeBatch: tzr_pose_graph_optimize_batch, DESIGN.md §3.24).
// RobustRegistrationSolver::solveMultiway (teaser/registration.h) chains both after the
// cloud-pair call.  teaser::GlobalOptimization is Open3D's global_optimization with the line process
// (tzr_pose_graph_optimize_line_process, DESIGN.md §3.22), and solveMultiway has overloads that take its Params.  No CPU
// implementation: without a CUDA device the first call throws std::runtime_error.
#pragma once

#include <vector>

#include "teaser/geometry.h"
#include "teaser/registration.h"

namespace teaser {

using Matrix6d = Eigen::Matrix<double, 6, 6>;

// Lambda (6 x 6, ordering (omega, tau)) of the correspondences of src moved by T against dst, ICP's search at distance
// max_correspondence_distance; *count (may be null) receives the correspondence count, Lambda(5,5).
Matrix6d informationMatrix(const PointCloud& src, const PointCloud& dst, const RegistrationSolution& T,
                           double max_correspondence_distance, int* count = nullptr);
// Many pairs in one device call; entry b is informationMatrix(src[b], dst[b], T[b]) bit for bit.
std::vector<Matrix6d> informationMatrixBatch(const std::vector<PointCloud>& src, const std::vector<PointCloud>& dst,
                                             const std::vector<RegistrationSolution>& T,
                                             double max_correspondence_distance, std::vector<int>* counts = nullptr);

class PoseGraph {
 public:
  using Params = PoseGraphParams;
  // An edge in the cloud-pair orientation: p_target ~ transform p_source (a rigid 4 x 4 matrix).
  struct Edge {
    int source = 0, target = 0;
    Eigen::Matrix4d transform;
    Matrix6d information;
    bool uncertain = false;
  };
  struct Result {
    std::vector<Eigen::Matrix4d> poses;  // node k into the world frame
    std::vector<double> weights;         // per edge
    std::vector<bool> inliers;           // weight >= 0.5
    std::vector<double> residuals;       // the normalised residual r-bar at the returned poses
    int iterations = 0;                  // GNC-TLS iterations
    int inner_iterations = 0;            // Levenberg-Marquardt iterations, summed
    double cost = 0;
  };
  // One graph of a batch (both optimisers' optimizeBatch): initial_poses empty means the breadth-first start from the
  // reference node.
  struct Graph {
    int num_nodes = 0;
    std::vector<Edge> edges;
    std::vector<Eigen::Matrix4d> initial_poses;
  };

  PoseGraph() = default;
  explicit PoseGraph(const Params& params) : params_(params) {}

  // tzr_pose_graph_optimize over num_nodes nodes on this thread's context.  initial_poses (null: breadth-first from
  // the reference node) holds num_nodes rigid matrices.  Throws std::runtime_error with the library's message on an
  // invalid graph (disconnected, more than 1024 nodes, a non-rigid edge).
  Result optimize(int num_nodes, const std::vector<Edge>& edges,
                  const std::vector<Eigen::Matrix4d>* initial_poses = nullptr) const;

  // tzr_pose_graph_optimize_batch: every graph in one call.  Entry g equals optimize() on graphs[g] for a graph of
  // more than 128 nodes, and has its decisions for a smaller one (DESIGN.md §3.24).  A graph the single call would
  // refuse gets an empty Result (no poses) and its status in *status (may be null; TZR_OK = 0 otherwise).  Throws
  // std::runtime_error only on call-level errors (invalid parameters, an empty batch, the workspace).
  std::vector<Result> optimizeBatch(const std::vector<Graph>& graphs, std::vector<int>* status = nullptr) const;

  const Params& getParams() const { return params_; }
  void setParams(const Params& params) { params_ = params; }

 private:
  Params params_;
};

// Open3D's global_optimization with GlobalOptimizationLevenbergMarquardt: the line process, pruning of the uncertain
// edges whose confidence is at most edge_prune_threshold, a second pass on the kept edges, then the compensation that
// returns the reference node to its starting pose.
class GlobalOptimization {
 public:
  using Params = LineProcessParams;
  using Edge = PoseGraph::Edge;
  using Graph = PoseGraph::Graph;
  struct Result {
    std::vector<Eigen::Matrix4d> poses;  // node k into the world frame
    std::vector<double> confidence;      // per edge: pass 2's for a kept edge, pass 1's for a pruned one
    std::vector<bool> kept;
    std::vector<double> residuals;       // zeta^T Lambda zeta at the returned poses
    LineProcessSummary summary;
  };

  GlobalOptimization() = default;
  explicit GlobalOptimization(const Params& params) : params_(params) {}

  // tzr_pose_graph_optimize_line_process over num_nodes nodes on this thread's context; initial_poses as
  // PoseGraph::optimize's.  Throws std::runtime_error with the library's message on an invalid graph or parameters.
  Result optimize(int num_nodes, const std::vector<Edge>& edges,
                  const std::vector<Eigen::Matrix4d>* initial_poses = nullptr) const;

  // tzr_pose_graph_optimize_line_process_batch: every graph in one call.  Entry g equals optimize() on graphs[g] for
  // a graph of more than 128 nodes, and has its decisions for a smaller one (DESIGN.md §3.23).  A graph the single
  // call would refuse gets an empty Result (no poses) and its status in *status (may be null; TZR_OK = 0 otherwise).
  // Throws std::runtime_error only on call-level errors (invalid parameters, an empty batch, the workspace).
  std::vector<Result> optimizeBatch(const std::vector<Graph>& graphs, std::vector<int>* status = nullptr) const;

  const Params& getParams() const { return params_; }
  void setParams(const Params& params) { params_ = params; }

 private:
  Params params_;
};

}  // namespace teaser
