// super4pcs-b200: Utils::OrientNormals on top of s4g_orient_normals (include/s4g.h).
#include "super4pcs/utils/normals.h"

#include <cmath>
#include <cstdint>
#include <cstring>
#include <stdexcept>

#include "s4g.h"
#include "utils_context.h"

namespace GlobalRegistration {
namespace Utils {

int OrientNormals(std::vector<Point3D>& cloud, int k, Point3D::Scalar max_distance, const Point3D::VectorType* viewpoint) {
  if (std::isnan(max_distance) || max_distance < 0)
    throw std::runtime_error("super4pcs-b200: OrientNormals: max_distance is negative or NaN");
  if (cloud.empty()) return 0;
  const std::size_t n = cloud.size();
  const std::vector<float> xyz = internal::Positions(cloud);
  std::vector<float> nrm(3 * n);
  for (std::size_t i = 0; i < n; ++i)
    for (int c = 0; c < 3; ++c) nrm[3 * i + c] = cloud[i].normal()[c];
  std::vector<float> out(3 * n);
  int64_t out2[2] = {0, 0};
  const float vp[3] = {viewpoint ? (*viewpoint)[0] : 0.f, viewpoint ? (*viewpoint)[1] : 0.f,
                       viewpoint ? (*viewpoint)[2] : 0.f};
  internal::WithContext("OrientNormals", [&](s4g_ctx* ctx) {
    const int rc = s4g_set_cloud_p(ctx, xyz.data(), int(n), internal::GridDelta(xyz, n, k));
    return rc == S4G_OK ? s4g_orient_normals(ctx, nrm.data(), k, max_distance * max_distance, viewpoint ? vp : nullptr,
                                             out.data(), nullptr, out2, nullptr)
                        : rc;
  });
  for (std::size_t i = 0; i < n; ++i)
    if (std::memcmp(&out[3 * i], &nrm[3 * i], 3 * sizeof(float)) != 0) cloud[i].set_normal(-cloud[i].normal());
  return int(out2[0]);
}

}  // namespace Utils
}  // namespace GlobalRegistration
