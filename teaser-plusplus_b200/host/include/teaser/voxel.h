// teaser::voxelDownSample — the first step of the reference's FPFH + TEASER++ + ICP tutorial (Open3D's
// voxel_down_sample on both raw scans), on the GPU through the C-ABI (tzr_voxel_downsample, tzr_voxel_downsample_batch;
// include/teaser_b200.h defines the result: voxel means of the finite points, ordered by each voxel's first member).
// No CPU implementation: without a CUDA device the first call throws std::runtime_error.
#pragma once

#include <vector>

#include "teaser/geometry.h"

namespace teaser {

// One cloud (may be empty: the result is empty), on this thread's context.  voxel_of (may be null) receives the
// output index of every input point, or -1 for a point with a non-finite coordinate.  Throws std::invalid_argument for
// a voxel size that is not finite and > 0, std::runtime_error when the cloud's grid is too large for the voxel size.
PointCloud voxelDownSample(const PointCloud& cloud, double voxel_size, std::vector<int>* voxel_of = nullptr);

// Many clouds in one device call; result b is voxelDownSample(clouds[b], voxel_size) bit for bit.  voxel_of (may be
// null) receives one trace per cloud.
std::vector<PointCloud> voxelDownSampleBatch(const std::vector<PointCloud>& clouds, double voxel_size,
                                             std::vector<std::vector<int>>* voxel_of = nullptr);

// With colours (tzr_voxel_downsample_colors(_batch)): the same points, and in colors_out each voxel's colour mean, summed
// in ascending input index like its point.  colors: one per point.
PointCloud voxelDownSample(const PointCloud& cloud, const ColorCloud& colors, double voxel_size, ColorCloud* colors_out,
                           std::vector<int>* voxel_of = nullptr);
std::vector<PointCloud> voxelDownSampleBatch(const std::vector<PointCloud>& clouds,
                                             const std::vector<ColorCloud>& colors, double voxel_size,
                                             std::vector<ColorCloud>* colors_out,
                                             std::vector<std::vector<int>>* voxel_of = nullptr);

}  // namespace teaser
