// super4pcs-b200 (private): the short-lived context of the point-cloud utilities (Utils::EstimateNormals,
// Utils::RemoveStatisticalOutliers, ...): the xyz they hand to it, its grid delta, and the context itself.
#ifndef SUPER4PCS_B200_CPP_UTILS_CONTEXT_H_
#define SUPER4PCS_B200_CPP_UTILS_CONTEXT_H_

#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <vector>

#include "s4g.h"
#include "super4pcs/shared4pcs.h"

namespace GlobalRegistration {
namespace Utils {
namespace internal {

// the positions of a cloud, n x 3
inline std::vector<float> Positions(const std::vector<Point3D>& cloud) {
  std::vector<float> xyz(3 * cloud.size());
  for (std::size_t i = 0; i < cloud.size(); ++i)
    for (int c = 0; c < 3; ++c) xyz[3 * i + c] = cloud[i].pos()[c];
  return xyz;
}

// the grid's delta of a cloud (xyz: n x 3): 0.5 * E * sqrt(k / n), E the largest edge of its bounding box; 1 when E is
// 0.  It sets only the time the queries take, never their results.
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

// runs body(ctx) -> s4g status on a context of its own on device S4PCS_DEVICE (default 0), then destroys the context.
// Throws "super4pcs-b200: <who>: ..." when there is no device or the body fails.
template <class Body>
void WithContext(const char* who, Body body) {
  int device = 0;
  if (const char* e = std::getenv("S4PCS_DEVICE")) device = std::atoi(e);
  s4g_ctx* ctx = nullptr;
  if (s4g_create(device, &ctx) != S4G_OK)
    throw std::runtime_error(std::string("super4pcs-b200: ") + who + ": no CUDA device (there is no CPU fallback)");
  const int rc = body(ctx);
  const std::string msg = rc == S4G_OK ? std::string() : std::string(s4g_error_string(ctx));
  s4g_destroy(ctx);
  if (rc != S4G_OK) throw std::runtime_error(std::string("super4pcs-b200: ") + who + ": " + msg);
}

}  // namespace internal
}  // namespace Utils
}  // namespace GlobalRegistration

#endif  // SUPER4PCS_B200_CPP_UTILS_CONTEXT_H_
