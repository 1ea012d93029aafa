// super4pcs-b200: Utils::VoxelGridFilter on top of s4g_voxel_grid (include/s4g.h).
#include "super4pcs/utils/voxel_grid.h"

#include <cmath>
#include <cstdint>
#include <stdexcept>

#include "s4g.h"
#include "utils_context.h"

namespace GlobalRegistration {
namespace Utils {

int VoxelGridFilter(std::vector<Point3D>& cloud, Point3D::Scalar leaf, int min_points) {
  if (!std::isfinite(leaf) || !(leaf > 0) || min_points < 1)
    throw std::runtime_error("super4pcs-b200: VoxelGridFilter: bad arguments (leaf finite and > 0, min_points >= 1)");
  const std::size_t n = cloud.size();
  if (n == 0) return 0;
  // a point without a colour holds Point3D's default (-1, -1, -1), which hasColor() does not tell apart (its squared
  // norm is 3); averaging it with real colours would give a wrong colour
  const Point3D::VectorType none = Point3D().rgb();
  bool colour = true;
  for (const Point3D& p : cloud) colour = colour && p.rgb() != none;
  std::vector<float> xyz(3 * n), nrm(3 * n), rgb(colour ? 3 * n : 0);
  for (std::size_t i = 0; i < n; ++i)
    for (int c = 0; c < 3; ++c) {
      xyz[3 * i + c] = cloud[i].pos()[c];
      nrm[3 * i + c] = cloud[i].normal()[c];
      if (colour) rgb[3 * i + c] = cloud[i].rgb()[c];
    }
  std::vector<float> xyz_out(3 * n), nrm_out(3 * n), rgb_out(colour ? 3 * n : 0);
  int64_t m = 0;
  internal::WithContext("VoxelGridFilter", [&](s4g_ctx* ctx) {
    return s4g_voxel_grid(ctx, xyz.data(), nrm.data(), colour ? rgb.data() : nullptr, int64_t(n), leaf, min_points,
                          xyz_out.data(), nrm_out.data(), colour ? rgb_out.data() : nullptr, nullptr, nullptr, nullptr,
                          &m);
  });
  std::vector<Point3D> out(static_cast<std::size_t>(m));
  for (std::size_t v = 0; v < out.size(); ++v) {
    out[v] = Point3D(xyz_out[3 * v], xyz_out[3 * v + 1], xyz_out[3 * v + 2]);
    out[v].set_normal(Point3D::VectorType(nrm_out[3 * v], nrm_out[3 * v + 1], nrm_out[3 * v + 2]));
    if (colour) out[v].set_rgb(Point3D::VectorType(rgb_out[3 * v], rgb_out[3 * v + 1], rgb_out[3 * v + 2]));
  }
  cloud.swap(out);
  return int(cloud.size());
}

}  // namespace Utils
}  // namespace GlobalRegistration
