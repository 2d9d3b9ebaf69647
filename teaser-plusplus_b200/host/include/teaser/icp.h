// teaser::PointToPointICP — the refinement step of the reference's FPFH + TEASER++ + ICP tutorial
// (examples/teaser_python_fpfh_icp: Open3D's registration_icp with TransformationEstimationPointToPoint), on the GPU
// through the C-ABI (tzr_icp, tzr_icp_batch; include/teaser_b200.h defines the loop).  teaser::PointToPlaneICP is the
// same with TransformationEstimationPointToPlane (tzr_icp_point_to_plane, tzr_icp_point_to_plane_batch), given the
// target normals (teaser::estimateNormals, teaser/normals.h).  teaser::GeneralizedICP is the same with Open3D's
// registration_generalized_icp (tzr_icp_generalized, tzr_icp_generalized_batch), given both clouds' normals.  Both of
// the last two take a teaser::RobustKernel (teaser/registration.h; L2 by default), Open3D's robust losses
// (tzr_icp_point_to_plane_robust_batch, tzr_icp_generalized_robust_batch).  teaser::ColoredICP is Open3D's
// registration_colored_icp (tzr_icp_colored, tzr_icp_colored_batch), given the target normals and both clouds'
// colours.  teaser::MultiScaleICP runs Open3D's coarse-to-fine schedule over a cloud table (tzr_icp_multiscale_batch):
// at each scale voxel downsampling, normals and one of the four methods above.  No CPU implementation: without a CUDA
// device the first call throws std::runtime_error.
#pragma once

#include <vector>

#include "teaser/fpfh.h"
#include "teaser/geometry.h"
#include "teaser/pose_graph.h"
#include "teaser/registration.h"

namespace teaser {

class PointToPointICP {
 public:
  using Params = PointToPointICPParams;
  using Result = PointToPointICPResult;

  PointToPointICP() = default;
  explicit PointToPointICP(const Params& params) : params_(params) {}

  // ICP of src onto dst seeded with init (its scale held fixed), on this thread's context.  Both clouds non-empty.
  Result refine(const PointCloud& src, const PointCloud& dst, const RegistrationSolution& init) const;
  // Many problems in one device call (tzr_icp_batch); result b is refine(src[b], dst[b], init[b]) bit for bit.
  std::vector<Result> refineBatch(const std::vector<PointCloud>& src, const std::vector<PointCloud>& dst,
                                  const std::vector<RegistrationSolution>& init) const;

  const Params& getParams() const { return params_; }
  void setParams(const Params& params) { params_ = params; }

 private:
  Params params_;
};

class PointToPlaneICP {
 public:
  using Params = PointToPointICPParams;
  using Result = PointToPointICPResult;

  PointToPlaneICP() = default;
  explicit PointToPlaneICP(const Params& params) : params_(params) {}
  PointToPlaneICP(const Params& params, const RobustKernel& kernel) : params_(params), kernel_(kernel) {}

  // Point-to-plane ICP of src onto dst seeded with init (its scale held fixed), on this thread's context.  dst_normals:
  // one normal per target point (curvature ignored; used as given, their signs do not matter).  Both clouds non-empty.
  Result refine(const PointCloud& src, const PointCloud& dst, const NormalCloud& dst_normals,
                const RegistrationSolution& init) const;
  // Many problems in one device call (tzr_icp_point_to_plane_batch); result b is refine(src[b], dst[b],
  // dst_normals[b], init[b]) bit for bit.
  std::vector<Result> refineBatch(const std::vector<PointCloud>& src, const std::vector<PointCloud>& dst,
                                  const std::vector<NormalCloud>& dst_normals,
                                  const std::vector<RegistrationSolution>& init) const;

  const Params& getParams() const { return params_; }
  void setParams(const Params& params) { params_ = params; }
  // The robust kernel: L2 (the default) runs tzr_icp_point_to_plane(_batch), any other tzr_icp_point_to_plane_robust_batch
  const RobustKernel& getKernel() const { return kernel_; }
  void setKernel(const RobustKernel& kernel) { kernel_ = kernel; }

 private:
  Params params_;
  RobustKernel kernel_;
};

class GeneralizedICP {
 public:
  using Params = GeneralizedICPParams;
  using Result = PointToPointICPResult;

  GeneralizedICP() = default;
  explicit GeneralizedICP(const Params& params) : params_(params) {}
  GeneralizedICP(const Params& params, const RobustKernel& kernel) : params_(params), kernel_(kernel) {}

  // Generalized ICP of src onto dst seeded with init (its scale held fixed), on this thread's context.  src_normals /
  // dst_normals: one normal per source / target point (curvature ignored; used up to length and sign).  Both clouds
  // non-empty.
  Result refine(const PointCloud& src, const PointCloud& dst, const NormalCloud& src_normals,
                const NormalCloud& dst_normals, const RegistrationSolution& init) const;
  // Many problems in one device call (tzr_icp_generalized_batch); result b is refine(src[b], dst[b], src_normals[b],
  // dst_normals[b], init[b]) bit for bit.
  std::vector<Result> refineBatch(const std::vector<PointCloud>& src, const std::vector<PointCloud>& dst,
                                  const std::vector<NormalCloud>& src_normals,
                                  const std::vector<NormalCloud>& dst_normals,
                                  const std::vector<RegistrationSolution>& init) const;

  const Params& getParams() const { return params_; }
  void setParams(const Params& params) { params_ = params; }
  // The robust kernel: L2 (the default) runs tzr_icp_generalized(_batch), any other tzr_icp_generalized_robust_batch
  const RobustKernel& getKernel() const { return kernel_; }
  void setKernel(const RobustKernel& kernel) { kernel_ = kernel; }

 private:
  Params params_;
  RobustKernel kernel_;
};

// Open3D's registration_colored_icp (tzr_icp_colored, tzr_icp_colored_batch): point-to-plane's geometric row plus a
// photometric row from both clouds' colours and the target's colour gradients (computed inside the call at 2
// max_correspondence_distance, as teaser::estimateColorGradients gives them).  With lambda_geometric = 1 the results
// are PointToPlaneICP's bit for bit.
class ColoredICP {
 public:
  using Params = ColoredICPParams;
  using Result = PointToPointICPResult;

  ColoredICP() = default;
  explicit ColoredICP(const Params& params) : params_(params) {}
  ColoredICP(const Params& params, const RobustKernel& kernel) : params_(params), kernel_(kernel) {}

  // Coloured ICP of src onto dst seeded with init (its scale held fixed), on this thread's context.  dst_normals: one
  // normal per target point; src_colors / dst_colors: one colour per source / target point.  Both clouds non-empty.
  Result refine(const PointCloud& src, const PointCloud& dst, const NormalCloud& dst_normals,
                const ColorCloud& src_colors, const ColorCloud& dst_colors, const RegistrationSolution& init) const;
  // Many problems in one device call (tzr_icp_colored_batch); result b is refine(src[b], dst[b], dst_normals[b],
  // src_colors[b], dst_colors[b], init[b]) bit for bit.
  std::vector<Result> refineBatch(const std::vector<PointCloud>& src, const std::vector<PointCloud>& dst,
                                  const std::vector<NormalCloud>& dst_normals,
                                  const std::vector<ColorCloud>& src_colors, const std::vector<ColorCloud>& dst_colors,
                                  const std::vector<RegistrationSolution>& init) const;

  const Params& getParams() const { return params_; }
  void setParams(const Params& params) { params_ = params; }
  // The robust kernel: L2 (the default) passes no kernel, any other is weighted per row
  const RobustKernel& getKernel() const { return kernel_; }
  void setKernel(const RobustKernel& kernel) { kernel_ = kernel; }

 private:
  Params params_;
  RobustKernel kernel_;
};

// One scale of MultiScaleICP's schedule (tzr_icp_scale): voxel_size > 0 downsamples every cloud, 0 keeps the clouds as
// given; normal_search_radius is read by the methods with normals (Open3D's tutorials: 2 voxel_size, which the
// three-argument constructor sets).
struct ICPScale {
  double voxel_size = 0;
  double max_correspondence_distance = 0;  // no default: must be set (> 0)
  double normal_search_radius = 0;
  int max_iteration = 30;
  double relative_fitness = 1e-6;
  double relative_rmse = 1e-6;
  ICPScale() = default;
  ICPScale(double voxel, double distance, int iterations)
      : voxel_size(voxel), max_correspondence_distance(distance), normal_search_radius(2 * voxel),
        max_iteration(iterations) {}
};

// Open3D's multi-scale refinement (the coloured-ICP tutorial's schedule, the reconstruction system's multiscale_icp) for
// many pairs of one cloud table in one device call (tzr_icp_multiscale_batch; include/teaser_b200.h states the
// contract).  Scale s's record of each pair equals voxelDownSampleBatch, estimateNormalsBatch and the method's
// refineBatch at that scale, seeded by the pair's record at s - 1, bit for bit.
class MultiScaleICP {
 public:
  enum Method { kPointToPoint = 0, kPointToPlane = 1, kGeneralized = 2, kColored = 3 };  // TZR_ICP_*
  struct Params {
    std::vector<ICPScale> scales;
    Method method = kPointToPlane;
    double lambda_geometric = 0.968;  // kColored
    double epsilon = 1e-3;            // kGeneralized
    RobustKernel kernel;              // L2 (the default) passes no kernel; point-to-point takes none
  };
  struct Result {
    // records[p][s]: pair p's refinement at scale s (no correspondences).  A pair whose cloud has no point at a scale
    // carries its pose (iterations 0); a zeroed record (normals that overflowed) has solution.valid = false.
    std::vector<std::vector<PointToPointICPResult>> records;
    std::vector<std::vector<int>> n_down;  // [cloud][scale]: each cloud's points at each scale
    std::vector<std::vector<int>> status;  // [cloud][scale]: 0, or TZR_ERR_TOO_LARGE
    bool too_large = false;                // some status is TZR_ERR_TOO_LARGE (the records are still what the call wrote)
    std::vector<Matrix6d> information;     // with information: per pair, at the last scale (zero where not refined)
    std::vector<int> info_counts;
  };

  MultiScaleICP() = default;
  explicit MultiScaleICP(const Params& params) : params_(params) {}

  // pairs (source cloud, target cloud) index clouds; colors (one per cloud) for kColored only, may be empty otherwise;
  // init: one seed per pair (its scale held fixed).  Throws std::invalid_argument for malformed inputs and
  // std::runtime_error for any error other than TZR_ERR_TOO_LARGE, which sets too_large instead.
  Result refineBatch(const std::vector<PointCloud>& clouds, const std::vector<ColorCloud>& colors,
                     const std::vector<std::pair<int, int>>& pairs, const std::vector<RegistrationSolution>& init,
                     bool information = false) const;

  const Params& getParams() const { return params_; }
  void setParams(const Params& params) { params_ = params; }

 private:
  Params params_;
};

}  // namespace teaser
