// super4pcs-b200: FPFH point descriptors and their nearest-descriptor correspondences, on the GPU (s4g_fpfh and
// s4g_fpfh_match, include/s4g.h).
//
// The descriptors of a feature-based estimator (RANSAC on correspondences, FGR, TEASER), a cross-check of a Super4PCS
// result, or a way to pick which cluster of a scene to register a model against.  The chain of Open3D's global
// registration preprocessing:
//
//   Utils::EstimateNormals(P, 16);                   // on the dense cloud
//   Utils::OrientNormals(P, 16, inf, &viewpoint);    // FPFH needs consistently oriented normals
//   Utils::VoxelGridFilter(P, 0.005f);               // the averaged normals no longer cancel
//   auto fp = Utils::ComputeFPFH(P, 32, 0.025f);     // likewise for Q
//   std::vector<int> corr = Utils::MatchFPFH(fp, fq);  // one Q index per P point, or -1
#ifndef SUPER4PCS_UTILS_FEATURES_H_
#define SUPER4PCS_UTILS_FEATURES_H_

#include <array>
#include <limits>
#include <vector>

#include "super4pcs/shared4pcs.h"

namespace GlobalRegistration {
namespace Utils {

/// 33 bins: 0-10 f1 (the angle of the neighbour's normal about the pair's axis), 11-21 f2, 22-32 f3
using FPFHSignature = std::array<float, 33>;

/// The FPFH descriptor of every point of `cloud` (Rusu et al. 2009; Open3D's compute_fpfh_feature) from its k nearest
/// other points within max_distance (squared in fp32; +inf: unbounded) and Point3D::normal(), computed on the GPU by
/// s4g_fpfh.  A zero or non-finite normal is no normal: such a point gets an all-zero descriptor and is left out of its
/// neighbours'.  The signs of the normals matter (negating them mirrors the f1 and f3 blocks), so orient them
/// consistently first (OrientNormals).  The short-lived context and its grid's delta are EstimateNormals'.
/// 1 <= k <= 64.  Throws std::runtime_error when k or max_distance is out of range or the device fails.
std::vector<FPFHSignature> ComputeFPFH(const std::vector<Point3D>& cloud, int k,
                                       Point3D::Scalar max_distance = std::numeric_limits<Point3D::Scalar>::infinity());

/// For every source descriptor, the index of the target descriptor with the smallest squared distance (summed in fp32
/// over the 33 bins; ties to the smaller index), or -1 when no distance is finite, by brute force on the GPU
/// (s4g_fpfh_match).  mutual: -1 also unless the source descriptor is in turn the nearest to that target, Open3D's
/// mutual filter.  Throws std::runtime_error when the device fails.
std::vector<int> MatchFPFH(const std::vector<FPFHSignature>& source, const std::vector<FPFHSignature>& target,
                           bool mutual = true);

}  // namespace Utils
}  // namespace GlobalRegistration

#endif  // SUPER4PCS_UTILS_FEATURES_H_
