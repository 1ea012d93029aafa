// super4pcs-b200: Utils::ExtractEuclideanClusters on top of s4g_euclidean_clusters (include/s4g.h).
#include "super4pcs/utils/clusters.h"

#include <cmath>
#include <cstdint>
#include <stdexcept>

#include "s4g.h"
#include "utils_context.h"

namespace GlobalRegistration {
namespace Utils {

std::vector<std::vector<int>> ExtractEuclideanClusters(const std::vector<Point3D>& cloud, Point3D::Scalar tolerance,
                                                       int min_size, int max_size) {
  if (std::isnan(tolerance) || tolerance < 0 || min_size < 1 || max_size < min_size)
    throw std::runtime_error("super4pcs-b200: ExtractEuclideanClusters: bad arguments (tolerance >= 0, "
                             "1 <= min_size <= max_size)");
  std::vector<std::vector<int>> out;
  const std::size_t n = cloud.size();
  if (n == 0) return out;
  const std::vector<float> xyz = internal::Positions(cloud);
  float delta = tolerance / 2.02f;
  if (!(delta > 0.f) || !std::isfinite(delta)) delta = internal::GridDelta(xyz, n, 16);
  std::vector<int32_t> labels(n), members(n);
  std::vector<int64_t> offsets(n + 1);
  int64_t n_clusters = 0;
  internal::WithContext("ExtractEuclideanClusters", [&](s4g_ctx* ctx) {
    const int rc = s4g_set_cloud_p(ctx, xyz.data(), int(n), delta);
    return rc == S4G_OK ? s4g_euclidean_clusters(ctx, tolerance * tolerance, min_size, max_size, labels.data(), nullptr,
                                                 &n_clusters, offsets.data(), members.data())
                        : rc;
  });
  out.resize(std::size_t(n_clusters));
  for (int64_t c = 0; c < n_clusters; ++c)
    out[std::size_t(c)].assign(members.begin() + offsets[c], members.begin() + offsets[c + 1]);
  return out;
}

}  // namespace Utils
}  // namespace GlobalRegistration
