// super4pcs-b200: outlier removal on the GPU (s4g_statistical_outliers, s4g_radius_outliers, include/s4g.h).
//
// Raw scans carry stray points that every later stage pays for: the sampler keeps them, the pair lists grow with them,
// they dilute the LCP, and an isolated point gets a meaningless PCA normal.  The usual pre-processing chain removes them
// first, between IOManager::ReadObject and ComputeTransformation:
//
//   std::vector<Point3D> P, Q;  ... ReadObject ...
//   Utils::RemoveStatisticalOutliers(P, 16, 2.0);
//   Utils::RemoveStatisticalOutliers(Q, 16, 2.0);
//   Utils::EstimateNormals(P, 16);
//   Utils::EstimateNormals(Q, 16);
//   matcher.ComputeTransformation(P, &Q, mat);
//
// ComputeTransformation itself filters nothing; the caller decides.
#ifndef SUPER4PCS_UTILS_OUTLIERS_H_
#define SUPER4PCS_UTILS_OUTLIERS_H_

#include <vector>

#include "super4pcs/shared4pcs.h"

namespace GlobalRegistration {
namespace Utils {

/// Removes from `cloud` every point whose mean distance to its k nearest other points is above mu + std_ratio * sigma,
/// mu and sigma the mean and sample standard deviation of that mean distance over the cloud (PCL's
/// StatisticalOutlierRemoval), computed on the GPU by s4g_statistical_outliers, and returns how many points were removed.
/// The survivors keep their order, normals and colours.  1 <= k <= 64, std_ratio finite (it may be negative or zero).
///
/// The call uses a short-lived context on the device S4PCS_DEVICE names (default 0), its grid's delta set by the rule of
/// EstimateNormals (0.5 * E * sqrt(k / n)); the rule sets only the time the query takes, never its result.
/// Throws std::runtime_error when k or std_ratio is out of range or the device fails; the cloud is then unchanged.
int RemoveStatisticalOutliers(std::vector<Point3D>& cloud, int k, double std_ratio);

/// Removes from `cloud` every point with fewer than min_neighbors other points at a distance below `radius` (squared in
/// fp32, the strict test of the kd-tree's range query; PCL's RadiusOutlierRemoval), computed on the GPU by
/// s4g_radius_outliers, and returns how many points were removed.  The survivors keep their order, normals and colours.
/// radius >= 0 (0 removes every point; +inf counts every other point), min_neighbors >= 1.
///
/// The call uses a short-lived context on S4PCS_DEVICE (default 0) whose grid's delta is radius / 2.02, i.e. cells of edge
/// about `radius`, so the ball around a point reaches at most one cell beyond its own per axis; when that is not a
/// positive finite number (radius 0 or +inf), the rule of EstimateNormals with k = min_neighbors.  Either sets only the
/// time the count takes.  Throws std::runtime_error when radius or min_neighbors is out of range or the device fails; the
/// cloud is then unchanged.
int RemoveRadiusOutliers(std::vector<Point3D>& cloud, Point3D::Scalar radius, int min_neighbors);

}  // namespace Utils
}  // namespace GlobalRegistration

#endif  // SUPER4PCS_UTILS_OUTLIERS_H_
