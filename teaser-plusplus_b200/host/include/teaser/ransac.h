// GPU extra: teaser::RANSACRegistration is correspondence RANSAC in the shape of Open3D's
// registration_ransac_based_on_correspondence (tzr_ransac, tzr_ransac_batch) and, over a table of clouds,
// registration_ransac_based_on_feature_matching (tzr_register_cloud_pairs_ransac), as include/teaser_b200.h defines it.
// No CPU implementation: without a CUDA device the first call throws std::runtime_error.
#pragma once

#include <cstdint>
#include <utility>
#include <vector>

#include "teaser/fpfh.h"
#include "teaser/geometry.h"
#include "teaser/registration.h"

namespace teaser {

// tzr_ransac_params: Open3D's ransac_n, RANSACConvergenceCriteria and its three correspondence checkers, each off unless
// enabled.  max_correspondence_distance has no default: the library refuses <= 0 or non-finite, ransac_n outside
// [3, 16], max_iteration < 0, confidence outside [0, 1] and a non-finite threshold of an enabled checker.
struct RANSACRegistrationParams {
  double max_correspondence_distance = 0;
  int ransac_n = 3;
  int max_iteration = 100000;
  double confidence = 0.999;
  bool check_edge_length = false;
  double edge_length_similarity = 0.9;
  bool check_distance = false;
  double distance_threshold = 0;
  bool check_normal = false;                          // needs both clouds' normals
  double normal_angle_threshold = 0.52359877559829882;  // radians
};

// tzr_ransac_info: one problem's loop summary
struct RANSACInfo {
  int drawn = 0;    // hypotheses drawn (the record's iterations)
  int passed = 0;   // of them, those that passed every enabled checker
  int winner = -1;  // the winning hypothesis's index, -1: none (the identity)
  int inliers = 0;  // its inliers among the usable rows
  int usable = 0;   // rows with both ends finite
  double rmse = 0;  // its score's rmse
};

class RANSACRegistration {
 public:
  using Params = RANSACRegistrationParams;
  // solution: the winner, the source onto the target (scale 1); fitness, inlier_rmse and correspondences: the
  // evaluation (tzr_icp_batch with max_iteration = 0 at max_correspondence_distance); iterations: the hypotheses
  // drawn; converged: the confidence bound stopped the loop before max_iteration
  using Result = PointToPointICPResult;
  using CloudPairParams = RobustRegistrationSolver::CloudPairParams;
  // One pair of registerCloudPairs.  status: 0 (TZR_OK) registered; TZR_ERR_TOO_LARGE (-6) a cloud with a point of
  // more than 4096 neighbours (no correspondences); TZR_ERR_INVALID_ARG (-1) no correspondence.  registered = false
  // (and ransac, info zeroed) for a pair that was not registered.
  struct CloudPairResult {
    int status = 0;
    std::vector<std::pair<int, int>> correspondences;  // the matcher's sorted, unique (source index, target index)
    float global_scale = 1;                            // Matcher::getGlobalScale()
    bool registered = false;
    Result ransac;
    RANSACInfo info;
  };

  RANSACRegistration() = default;
  explicit RANSACRegistration(const Params& params) : params_(params) {}

  // RANSAC of src onto dst on the (source index, target index) correspondences corr with a 64-bit seed, on this
  // thread's context (tzr_ransac).  Both clouds non-empty; every index inside its cloud.  The normals (one per point)
  // are read by the normal checker only and may be null without it.  info (may be null): the loop's summary.
  Result registerPair(const PointCloud& src, const PointCloud& dst, const std::vector<std::pair<int, int>>& corr,
                      uint64_t seed = 0, const NormalCloud* src_normals = nullptr,
                      const NormalCloud* dst_normals = nullptr, RANSACInfo* info = nullptr) const;
  // Many problems in one device call (tzr_ransac_batch); result b is registerPair(src[b], dst[b], corr[b], seeds[b],
  // ...) bit for bit.  seeds: empty (0 for every problem) or one per problem; normals: empty, or one cloud per problem
  // (required with the normal checker).  info (may be null): resized to one summary per problem.
  std::vector<Result> registerBatch(const std::vector<PointCloud>& src, const std::vector<PointCloud>& dst,
                                    const std::vector<std::vector<std::pair<int, int>>>& corr,
                                    const std::vector<uint64_t>& seeds = {},
                                    const std::vector<NormalCloud>& src_normals = {},
                                    const std::vector<NormalCloud>& dst_normals = {},
                                    std::vector<RANSACInfo>* info = nullptr) const;
  // FPFH of every cloud, matching of every pair (source cloud, target cloud) and RANSAC of every pair with
  // correspondences, in one device call (tzr_register_cloud_pairs_ransac), with no robust solve.  The pairs' tuple
  // seeds are RobustRegistrationSolver::solveCloudPairs' (params.tuple_seed + 0x9E3779B97F4A7C15 p), so the
  // correspondences are that call's; ransac_seeds: empty (0 for every pair) or one per pair.  The normal checker reads
  // the FPFH stage's normals.  Every cloud must be non-empty.  TZR_ERR_TOO_LARGE is reported per pair; other errors
  // throw.
  std::vector<CloudPairResult> registerCloudPairs(const std::vector<PointCloud>& clouds,
                                                  const std::vector<std::pair<int, int>>& pairs,
                                                  const CloudPairParams& params,
                                                  const std::vector<uint64_t>& ransac_seeds = {}) const;

  const Params& getParams() const { return params_; }
  void setParams(const Params& params) { params_ = params; }

 private:
  Params params_;
};

}  // namespace teaser
