// teaser::PointToPointICP — the refinement step of the reference's FPFH + TEASER++ + ICP tutorial
// (examples/teaser_python_fpfh_icp: Open3D's registration_icp with TransformationEstimationPointToPoint), on the GPU
// through the C-ABI (tzr_icp, tzr_icp_batch; include/teaser_b200.h defines the loop).  No CPU implementation: without a
// CUDA device the first call throws std::runtime_error.
#pragma once

#include <vector>

#include "teaser/geometry.h"
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

}  // namespace teaser
