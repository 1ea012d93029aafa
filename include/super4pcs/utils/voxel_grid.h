// super4pcs-b200: voxel-grid downsampling to centroids on the GPU (s4g_voxel_grid, include/s4g.h).
//
// Raw scans hold 10^6 - 10^8 points whose density varies by orders of magnitude with range, and every later step (the
// neighbour queries of the outlier filters, clustering, normals, the sampler of ComputeTransformation) pays for that
// density and has parameters whose meaning depends on it.  The usual chain therefore downsamples first:
//
//   std::vector<Point3D> P, Q;  ... ReadObject ...
//   Utils::VoxelGridFilter(P, 0.005f);
//   Utils::RemoveStatisticalOutliers(P, 16, 2.0);
//   ... segment the support plane, cluster ...
//   Utils::EstimateNormals(P, 16);
//
// A centroid averages out sensor noise, where the sampler's kept raw point does not.  ComputeTransformation itself
// downsamples nothing beyond its own sampling; the caller decides.
#ifndef SUPER4PCS_UTILS_VOXEL_GRID_H_
#define SUPER4PCS_UTILS_VOXEL_GRID_H_

#include <vector>

#include "super4pcs/shared4pcs.h"

namespace GlobalRegistration {
namespace Utils {

/// Replaces `cloud` by one point per voxel of edge `leaf` that holds at least min_points points (PCL's VoxelGrid with
/// setMinimumPointsNumberPerVoxel), computed on the GPU by s4g_voxel_grid, and returns the new size.  The voxel of a
/// point is (floor(x / leaf), ...) with s4g_voxel_sample's arithmetic.  Each new point is its voxel's centroid, with the
/// normal of the summed normals (zero when they cancel or the cloud has none; stored through set_normal), in the order
/// of each voxel's first point.  Colours are averaged only when every point has one, i.e. an rgb other than Point3D's
/// default (-1, -1, -1) (hasColor() cannot tell: the default's squared norm is 3); otherwise the new points keep the
/// default "no colour", because averaging the sentinel with real colours would give a wrong colour.  Averaged normals
/// assume consistently oriented input normals: downsample first and estimate normals afterwards.
///
/// The call uses a short-lived context on the device S4PCS_DEVICE names (default 0).  Throws std::runtime_error when
/// leaf is not finite and > 0, min_points < 1, a coordinate is not finite, the cloud spans 2^21 or more voxels along an
/// axis, or the device fails; the cloud is then unchanged.
int VoxelGridFilter(std::vector<Point3D>& cloud, Point3D::Scalar leaf, int min_points = 1);

}  // namespace Utils
}  // namespace GlobalRegistration

#endif  // SUPER4PCS_UTILS_VOXEL_GRID_H_
