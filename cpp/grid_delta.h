// super4pcs-b200 (private): the grid delta of the short-lived contexts of the point-cloud utilities (Utils::EstimateNormals,
// Utils::RemoveStatisticalOutliers).  It sets only the time their queries take, never their results.
#ifndef SUPER4PCS_B200_CPP_GRID_DELTA_H_
#define SUPER4PCS_B200_CPP_GRID_DELTA_H_

#include <algorithm>
#include <cmath>
#include <cstddef>
#include <vector>

namespace GlobalRegistration {
namespace Utils {
namespace internal {

// the grid's delta of a cloud (xyz: n x 3): 0.5 * E * sqrt(k / n), E the largest edge of its bounding box; 1 when E is 0
inline float GridDelta(const std::vector<float>& xyz, std::size_t n, int k) {
  float lo[3] = {xyz[0], xyz[1], xyz[2]}, hi[3] = {xyz[0], xyz[1], xyz[2]};
  for (std::size_t i = 0; i < n; ++i)
    for (int c = 0; c < 3; ++c) {
      lo[c] = std::min(lo[c], xyz[3 * i + c]);
      hi[c] = std::max(hi[c], xyz[3 * i + c]);
    }
  const double E = std::max({double(hi[0]) - lo[0], double(hi[1]) - lo[1], double(hi[2]) - lo[2]});
  const float delta = float(0.5 * E * std::sqrt(double(k) / double(n)));
  return delta > 0.f ? delta : 1.f;
}

}  // namespace internal
}  // namespace Utils
}  // namespace GlobalRegistration

#endif  // SUPER4PCS_B200_CPP_GRID_DELTA_H_
