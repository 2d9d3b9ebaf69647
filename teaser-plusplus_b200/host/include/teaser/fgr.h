// GPU extra: teaser::FastGlobalRegistration is Zhou, Park and Koltun's Fast Global Registration as Open3D runs it
// (registration_fgr_based_on_correspondence: tzr_fgr, tzr_fgr_batch; registration_fgr_based_on_feature_matching over a
// table of clouds: tzr_register_cloud_pairs_fgr).  Not teaser::FastGlobalRegistrationSolver, the rotation estimator of
// the robust solve.  No CPU implementation: without a CUDA device the first call throws std::runtime_error.
#pragma once

#include <utility>
#include <vector>

#include "teaser/geometry.h"
#include "teaser/registration.h"

namespace teaser {

// Open3D's FastGlobalRegistrationOption (tzr_fgr_params); the library refuses division_factor or
// maximum_correspondence_distance <= 0 or non-finite, and iteration_number < 0.
struct FastGlobalRegistrationParams {
  double division_factor = 1.4;
  bool use_absolute_scale = false;
  bool decrease_mu = true;
  double maximum_correspondence_distance = 0.025;
  int iteration_number = 64;
};

class FastGlobalRegistration {
 public:
  using Params = FastGlobalRegistrationParams;
  // solution: the source onto the target (scale 1); fitness, inlier_rmse and correspondences: the evaluation
  // (tzr_icp_batch with max_iteration = 0 at maximum_correspondence_distance); iterations: iteration_number, or 0
  // for the fallback (fewer than 10 usable correspondences), when converged is false
  using Result = PointToPointICPResult;
  using CloudPairParams = RobustRegistrationSolver::CloudPairParams;
  // One pair of registerCloudPairs.  status: 0 (TZR_OK) registered; TZR_ERR_TOO_LARGE (-6) a cloud with a point of
  // more than 4096 neighbours (no correspondences); TZR_ERR_INVALID_ARG (-1) no correspondence.  registered = false
  // (and fgr zeroed) for a pair that was not registered.
  struct CloudPairResult {
    int status = 0;
    std::vector<std::pair<int, int>> correspondences;  // the matcher's sorted, unique (source index, target index)
    float global_scale = 1;                            // Matcher::getGlobalScale()
    bool registered = false;
    Result fgr;
  };

  FastGlobalRegistration() = default;
  explicit FastGlobalRegistration(const Params& params) : params_(params) {}

  // FGR of src onto dst on the (source index, target index) correspondences corr, on this thread's context (tzr_fgr).
  // Both clouds non-empty; every index inside its cloud.
  Result registerPair(const PointCloud& src, const PointCloud& dst,
                      const std::vector<std::pair<int, int>>& corr) const;
  // Many problems in one device call (tzr_fgr_batch); result b is registerPair(src[b], dst[b], corr[b]) bit for bit.
  std::vector<Result> registerBatch(const std::vector<PointCloud>& src, const std::vector<PointCloud>& dst,
                                    const std::vector<std::vector<std::pair<int, int>>>& corr) const;
  // FPFH of every cloud, matching of every pair (source cloud, target cloud) and FGR of every pair with
  // correspondences, in one device call (tzr_register_cloud_pairs_fgr), with no robust solve.  The pairs' tuple
  // seeds are RobustRegistrationSolver::solveCloudPairs' (params.tuple_seed + 0x9E3779B97F4A7C15 p), so the
  // correspondences are that call's.  Every cloud must be non-empty.  TZR_ERR_TOO_LARGE is reported per pair; other
  // errors throw.
  std::vector<CloudPairResult> registerCloudPairs(const std::vector<PointCloud>& clouds,
                                                  const std::vector<std::pair<int, int>>& pairs,
                                                  const CloudPairParams& params) const;

  const Params& getParams() const { return params_; }
  void setParams(const Params& params) { params_ = params; }

 private:
  Params params_;
};

}  // namespace teaser
