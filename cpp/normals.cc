// super4pcs-b200: Utils::EstimateNormals on top of s4g_normals (include/s4g.h).
#include "super4pcs/utils/normals.h"

#include <cmath>
#include <stdexcept>

#include "s4g.h"
#include "utils_context.h"

namespace GlobalRegistration {
namespace Utils {

int EstimateNormals(std::vector<Point3D>& cloud, int k, Point3D::Scalar max_distance,
                    const Point3D::VectorType* viewpoint) {
  if (std::isnan(max_distance) || max_distance < 0)
    throw std::runtime_error("super4pcs-b200: EstimateNormals: max_distance is negative or NaN");
  if (cloud.empty()) return 0;
  const std::size_t n = cloud.size();
  const std::vector<float> xyz = internal::Positions(cloud);
  std::vector<float> normals(3 * n);
  const float vp[3] = {viewpoint ? (*viewpoint)[0] : 0.f, viewpoint ? (*viewpoint)[1] : 0.f,
                       viewpoint ? (*viewpoint)[2] : 0.f};
  internal::WithContext("EstimateNormals", [&](s4g_ctx* ctx) {
    const int rc = s4g_set_cloud_p(ctx, xyz.data(), int(n), internal::GridDelta(xyz, n, k));
    return rc == S4G_OK
               ? s4g_normals(ctx, k, max_distance * max_distance, viewpoint ? vp : nullptr, normals.data(), nullptr)
               : rc;
  });
  int nonzero = 0;
  for (std::size_t i = 0; i < n; ++i) {
    const Point3D::VectorType v(normals[3 * i], normals[3 * i + 1], normals[3 * i + 2]);
    cloud[i].set_normal(v);
    nonzero += v.squaredNorm() > 0.f ? 1 : 0;
  }
  return nonzero;
}

}  // namespace Utils
}  // namespace GlobalRegistration
