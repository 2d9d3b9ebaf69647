// teaser::estimateNormals — the normals FPFHEstimation computes (PCL's NormalEstimationOMP with a radius search,
// viewpoint at the origin), without the descriptors: the target normals of teaser::PointToPlaneICP.  On the GPU through
// the C-ABI (tzr_estimate_normals, tzr_estimate_normals_batch); bit-identical to FPFHEstimation::getNormals() after
// computeFPFHFeatures at the same normal radius.  No CPU implementation: without a CUDA device the first call throws
// std::runtime_error.
#pragma once

#include <array>
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

// Open3D's colour gradients of coloured ICP (InitializePointCloudForColoredICP; tzr_estimate_color_gradients(_batch)):
// one gradient per point from its 30 nearest neighbours inside radius, given its normals and colours (one per point).
// ColoredICP computes them itself at 2 max_correspondence_distance; these calls give the same bits.  An empty cloud
// gives an empty result.
std::vector<std::array<double, 3>> estimateColorGradients(const PointCloud& cloud, const NormalCloud& normals,
                                                          const ColorCloud& colors, double radius);
// Many clouds in one device call; result b is estimateColorGradients(clouds[b], normals[b], colors[b], radius) bit for
// bit.
std::vector<std::vector<std::array<double, 3>>> estimateColorGradientsBatch(const std::vector<PointCloud>& clouds,
                                                                          const std::vector<NormalCloud>& normals,
                                                                          const std::vector<ColorCloud>& colors,
                                                                          double radius);

}  // namespace teaser
