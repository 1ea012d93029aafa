// super4pcs-b200: Utils::RemoveStatisticalOutliers and Utils::RemoveRadiusOutliers on top of s4g_statistical_outliers and
// s4g_radius_outliers (include/s4g.h).
#include "super4pcs/utils/outliers.h"

#include <cmath>
#include <cstdint>
#include <stdexcept>

#include "s4g.h"
#include "utils_context.h"

namespace GlobalRegistration {
namespace Utils {

namespace {

// runs filter(ctx, keep, &n_kept) on a short-lived context holding the cloud with grid delta `delta`, then keeps the
// points keep[0 .. n_kept) (ascending) in place; returns how many were removed
template <class Filter>
int Apply(std::vector<Point3D>& cloud, const std::vector<float>& xyz, float delta, const char* who, Filter filter) {
  const std::size_t n = cloud.size();
  std::vector<int32_t> keep(n);
  int64_t n_kept = 0;
  internal::WithContext(who, [&](s4g_ctx* ctx) {
    const int rc = s4g_set_cloud_p(ctx, xyz.data(), int(n), delta);
    return rc == S4G_OK ? filter(ctx, keep.data(), &n_kept) : rc;
  });
  for (int64_t s = 0; s < n_kept; ++s)
    if (keep[s] != s) cloud[s] = cloud[keep[s]];   // keep[s] >= s: ascending, so no survivor is overwritten first
  cloud.resize(std::size_t(n_kept));
  return int(n - std::size_t(n_kept));
}

}  // namespace

int RemoveStatisticalOutliers(std::vector<Point3D>& cloud, int k, double std_ratio) {
  if (cloud.empty()) return 0;
  const std::vector<float> xyz = internal::Positions(cloud);
  return Apply(cloud, xyz, internal::GridDelta(xyz, cloud.size(), k), "RemoveStatisticalOutliers",
               [&](s4g_ctx* ctx, int32_t* keep, int64_t* n_kept) {
                 return s4g_statistical_outliers(ctx, k, std_ratio, keep, n_kept, nullptr, nullptr);
               });
}

int RemoveRadiusOutliers(std::vector<Point3D>& cloud, Point3D::Scalar radius, int min_neighbors) {
  if (std::isnan(radius) || radius < 0)
    throw std::runtime_error("super4pcs-b200: RemoveRadiusOutliers: radius is negative or NaN");
  if (cloud.empty()) return 0;
  const std::vector<float> xyz = internal::Positions(cloud);
  float delta = radius / 2.02f;
  if (!(delta > 0.f) || !std::isfinite(delta)) delta = internal::GridDelta(xyz, cloud.size(), min_neighbors);
  return Apply(cloud, xyz, delta, "RemoveRadiusOutliers", [&](s4g_ctx* ctx, int32_t* keep, int64_t* n_kept) {
    return s4g_radius_outliers(ctx, radius * radius, min_neighbors, keep, n_kept, nullptr);
  });
}

}  // namespace Utils
}  // namespace GlobalRegistration
