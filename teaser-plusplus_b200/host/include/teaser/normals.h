// teaser::estimateNormals — the normals FPFHEstimation computes (PCL's NormalEstimationOMP with a radius search,
// viewpoint at the origin), without the descriptors: the target normals of teaser::PointToPlaneICP.  On the GPU through
// the C-ABI (tzr_estimate_normals, tzr_estimate_normals_batch); bit-identical to FPFHEstimation::getNormals() after
// computeFPFHFeatures at the same normal radius.  No CPU implementation: without a CUDA device the first call throws
// std::runtime_error.
#pragma once

#include <vector>

#include "teaser/fpfh.h"
#include "teaser/geometry.h"

namespace teaser {

// One cloud (may be empty: the result is empty), on this thread's context.  A point with fewer than 3 neighbours gets a
// NaN normal.  Throws std::runtime_error when a point has more than 4096 neighbours inside the radius.
NormalCloud estimateNormals(const PointCloud& cloud, double normal_search_radius = 0.03);

// Many clouds in one device call; result b is estimateNormals(clouds[b], normal_search_radius) bit for bit.
std::vector<NormalCloud> estimateNormalsBatch(const std::vector<PointCloud>& clouds,
                                              double normal_search_radius = 0.03);

}  // namespace teaser
