// super4pcs-b200: Utils::SegmentPlanes on top of s4g_segment_planes (include/s4g.h).
#include "super4pcs/utils/planes.h"

#include <algorithm>
#include <cmath>
#include <stdexcept>

#include "s4g.h"
#include "utils_context.h"

namespace GlobalRegistration {
namespace Utils {

std::vector<PlaneModel> SegmentPlanes(const std::vector<Point3D>& cloud, Point3D::Scalar threshold, int max_planes,
                                      int min_inliers, int iterations, std::uint64_t seed, bool refine) {
  if (std::isnan(threshold) || threshold < 0 || max_planes < 1 || min_inliers < 1 || iterations < 1 ||
      iterations > (1 << 20))
    throw std::runtime_error("super4pcs-b200: SegmentPlanes: bad arguments (threshold >= 0, max_planes >= 1, "
                             "min_inliers >= 1, 1 <= iterations <= 2^20)");
  std::vector<PlaneModel> out;
  const std::size_t n = cloud.size();
  if (n == 0) return out;
  const std::vector<float> xyz = internal::Positions(cloud);
  // at most n planes are accepted (each claims a point), so the outputs never need more rows than that
  const int rows = int(std::min<std::size_t>(std::size_t(max_planes), n));
  std::vector<int32_t> labels(n), members(n);
  std::vector<int64_t> offsets(std::size_t(rows) + 1);
  std::vector<s4g_plane> planes{std::size_t(rows)};
  int n_planes = 0;
  internal::WithContext("SegmentPlanes", [&](s4g_ctx* ctx) {
    const int rc = s4g_set_cloud_p(ctx, xyz.data(), int(n), internal::GridDelta(xyz, n, 16));
    return rc == S4G_OK ? s4g_segment_planes(ctx, threshold, iterations, seed, refine ? 1 : 0, rows, min_inliers,
                                             labels.data(), planes.data(), &n_planes, offsets.data(), members.data(),
                                             nullptr)
                        : rc;
  });
  out.resize(std::size_t(n_planes));
  for (int r = 0; r < n_planes; ++r) {
    for (int c = 0; c < 4; ++c) out[std::size_t(r)].coefficients[std::size_t(c)] = planes[std::size_t(r)].coefficients[c];
    out[std::size_t(r)].inliers.assign(members.begin() + offsets[std::size_t(r)], members.begin() + offsets[std::size_t(r) + 1]);
  }
  return out;
}

}  // namespace Utils
}  // namespace GlobalRegistration
