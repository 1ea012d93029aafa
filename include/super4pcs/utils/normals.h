// super4pcs-b200: point normals estimated on the GPU (s4g_normals, include/s4g.h).
//
// Clouds read from files without normals (raw scans, PTX, XYZ) load with zero normals, and the pair query's normal filter
// (Match4PCSOptions::max_normal_difference) then passes every pair.  EstimateNormals gives such a cloud PCA normals
// between IOManager::ReadObject and ComputeTransformation:
//
//   std::vector<Point3D> P, Q;  ... ReadObject ...
//   Utils::EstimateNormals(P, 16);
//   Utils::EstimateNormals(Q, 16);
//   options.max_normal_difference = 40;
//   matcher.ComputeTransformation(P, &Q, mat);
#ifndef SUPER4PCS_UTILS_NORMALS_H_
#define SUPER4PCS_UTILS_NORMALS_H_

#include <limits>
#include <vector>

#include "super4pcs/shared4pcs.h"

namespace GlobalRegistration {
namespace Utils {

/// Sets the normal of every point of `cloud` to the PCA normal of its k nearest points (itself included) within
/// max_distance (squared in fp32; +inf: unbounded), computed on the GPU by s4g_normals, and returns how many points got
/// a non-zero normal.  The normal goes through Point3D::set_normal.  A point whose neighbourhood holds fewer than 3
/// points, or only coincident ones, gets (0, 0, 0), which the normal filter skips.  Without a viewpoint the normals are
/// unoriented (the component of largest magnitude is positive), which is all the normal filter needs: it compares
/// normals up to sign.  With one, each normal faces it.  3 <= k <= 64.
///
/// The call uses a short-lived context on the device S4PCS_DEVICE names (default 0).  Its grid's delta is
///   delta = 0.5 * E * sqrt(k / n)   (E: the largest edge of the cloud's bounding box, n: the number of points),
/// or 1 when E is 0: cells of edge ~2 delta then hold about k points of a surface sampled evenly over an E x E square.
/// The rule sets only the time the query takes, never its result.
/// Throws std::runtime_error when k or max_distance is out of range or the device fails; the cloud is then unchanged.
int EstimateNormals(std::vector<Point3D>& cloud, int k,
                    Point3D::Scalar max_distance = std::numeric_limits<Point3D::Scalar>::infinity(),
                    const Point3D::VectorType* viewpoint = nullptr);

/// Orients the normals of `cloud` consistently, on the GPU by s4g_orient_normals (Hoppe et al. 1992; Open3D's
/// orient_normals_consistent_tangent_plane), and returns the number of components.  The k-nearest graph of the points
/// (each point's k nearest other points within max_distance, squared in fp32; +inf: unbounded), made symmetric and
/// restricted to the points with a non-zero normal, is weighted by |n_i . n_j|; signs propagate along its minimum
/// spanning forest (largest |n_i . n_j| first, ties by index), flipping where n_i . n_j < 0.  Each component keeps the
/// sign of one anchor: its smallest index, or with a viewpoint the point nearest to it, turned to face it (the rule of
/// EstimateNormals).  So with a viewpoint outside a closed surface sampled densely enough, every normal points outward,
/// which the per-point viewpoint rule cannot give for points that face away from it.  Points with a zero normal keep it.
///
///   Utils::EstimateNormals(P, 16);                 // on the dense cloud, where the PCA has the most support
///   Utils::OrientNormals(P, 16, inf, &viewpoint);  // consistent signs
///   Utils::VoxelGridFilter(P, 0.005f);             // the averaged normals no longer cancel
///
/// A flipped normal is stored as set_normal(-normal()), which renormalises in float: its last bit may move.  Normals
/// that keep their sign are not touched.  The short-lived context and its grid's delta are EstimateNormals'.
/// 1 <= k <= 64.  Throws std::runtime_error when k or max_distance is out of range, a normal is not finite or the device
/// fails; the cloud is then unchanged.
int OrientNormals(std::vector<Point3D>& cloud, int k,
                  Point3D::Scalar max_distance = std::numeric_limits<Point3D::Scalar>::infinity(),
                  const Point3D::VectorType* viewpoint = nullptr);

}  // namespace Utils
}  // namespace GlobalRegistration

#endif  // SUPER4PCS_UTILS_NORMALS_H_
