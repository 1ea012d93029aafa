// super4pcs-b200: Euclidean cluster extraction on the GPU (s4g_euclidean_clusters, include/s4g.h).
//
// Two uses before a registration: dropping detached blobs of stray points that a radius filter keeps (each of them has
// enough neighbours, the blob as a whole is small), and finding an object in a scene -- cut the scene into clusters,
// then register the model against each cluster that is big enough:
//
//   std::vector<Point3D> model, scene;  ... ReadObject ...
//   Utils::RemoveStatisticalOutliers(scene, 16, 2.0);
//   for (const std::vector<int>& c : Utils::ExtractEuclideanClusters(scene, 0.01f, 500)) {
//     std::vector<Point3D> part;
//     for (int j : c) part.push_back(scene[j]);
//     Utils::EstimateNormals(part, 16);
//     matcher.ComputeTransformation(part, &model, mat);   // ... keep the best LCP
//   }
//
// ComputeTransformation itself clusters nothing; the caller decides.
#ifndef SUPER4PCS_UTILS_CLUSTERS_H_
#define SUPER4PCS_UTILS_CLUSTERS_H_

#include <climits>
#include <vector>

#include "super4pcs/shared4pcs.h"

namespace GlobalRegistration {
namespace Utils {

/// The Euclidean clusters of `cloud` (PCL's EuclideanClusterExtraction, made exact), computed on the GPU by
/// s4g_euclidean_clusters: the connected components of the graph joining two points at a distance below `tolerance`
/// (squared in fp32, the strict test of the kd-tree's range query), kept when min_size <= size <= max_size.  Each cluster
/// is the list of its points' indices in `cloud`, ascending; the clusters are ordered by size, largest first, ties by
/// their smallest index.  tolerance >= 0 (0: every point alone; +inf: one component), 1 <= min_size <= max_size.
///
/// The call uses a short-lived context on the device S4PCS_DEVICE names (default 0) whose grid's delta is
/// tolerance / 2.02 (cells of edge about `tolerance`, as Utils::RemoveRadiusOutliers); when that is not a positive finite
/// number (tolerance 0 or +inf), the rule of Utils::EstimateNormals with k = 16.  Either sets only the time the call
/// takes.  Throws std::runtime_error when an argument is out of range or the device fails.
std::vector<std::vector<int>> ExtractEuclideanClusters(const std::vector<Point3D>& cloud, Point3D::Scalar tolerance,
                                                       int min_size = 1, int max_size = INT_MAX);

}  // namespace Utils
}  // namespace GlobalRegistration

#endif  // SUPER4PCS_UTILS_CLUSTERS_H_
