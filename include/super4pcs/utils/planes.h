// super4pcs-b200: RANSAC plane segmentation on the GPU (s4g_segment_planes, include/s4g.h).
//
// Objects in a scan stand on a floor or a table, and that support plane touches every one of them: clustered as it is,
// the scene is one cluster.  Remove the plane first, then cluster the rest and register the model against each cluster
// that is big enough:
//
//   std::vector<Point3D> model, scene;  ... ReadObject ...
//   Utils::RemoveStatisticalOutliers(scene, 16, 2.0);
//   std::vector<Utils::PlaneModel> support = Utils::SegmentPlanes(scene, 0.005f);
//   ... keep the points of scene not in support[0].inliers ...
//   for (const std::vector<int>& c : Utils::ExtractEuclideanClusters(rest, 0.01f, 500)) { ... }
//
// ComputeTransformation itself segments nothing; the caller decides.
#ifndef SUPER4PCS_UTILS_PLANES_H_
#define SUPER4PCS_UTILS_PLANES_H_

#include <array>
#include <cstdint>
#include <vector>

#include "super4pcs/shared4pcs.h"

namespace GlobalRegistration {
namespace Utils {

/// One plane a x + b y + c z + d = 0 (|(a, b, c)| = 1) and its inliers: ascending indices into the cloud.
struct PlaneModel {
  std::array<float, 4> coefficients;
  std::vector<int> inliers;
};

/// The planes of `cloud` (PCL's SACSegmentation with a plane model and optimize_coefficients, made exact), computed on
/// the GPU by s4g_segment_planes: each round scores `iterations` RANSAC hypotheses drawn from a SplitMix64 stream of
/// `seed` (all of them, no early termination), takes the one with the most points at |a x + b y + c z + d| < threshold
/// (fp32), refits it by least squares over its inliers when `refine`, and keeps the points within `threshold` of the
/// result -- if there are at least `min_inliers`; the next round runs on the points no plane claimed.  At most
/// `max_planes` planes, in the order found.  The result is a pure function of the arguments.
/// threshold >= 0 (not NaN), 1 <= iterations <= 2^20, max_planes >= 1, min_inliers >= 1.
///
/// The call uses a short-lived context on the device S4PCS_DEVICE names (default 0); its grid, which the planes do not
/// use, follows the rule of Utils::EstimateNormals with k = 16.  Throws std::runtime_error when an argument is out of
/// range or the device fails.
std::vector<PlaneModel> SegmentPlanes(const std::vector<Point3D>& cloud, Point3D::Scalar threshold, int max_planes = 1,
                                      int min_inliers = 1, int iterations = 1000, std::uint64_t seed = 0,
                                      bool refine = true);

}  // namespace Utils
}  // namespace GlobalRegistration

#endif  // SUPER4PCS_UTILS_PLANES_H_
