// super4pcs-b200: Utils::ComputeFPFH and Utils::MatchFPFH on top of s4g_fpfh and s4g_fpfh_match (include/s4g.h).
#include "super4pcs/utils/features.h"

#include <cmath>
#include <cstdint>
#include <stdexcept>

#include "s4g.h"
#include "utils_context.h"

namespace GlobalRegistration {
namespace Utils {

std::vector<FPFHSignature> ComputeFPFH(const std::vector<Point3D>& cloud, int k, Point3D::Scalar max_distance) {
  if (std::isnan(max_distance) || max_distance < 0)
    throw std::runtime_error("super4pcs-b200: ComputeFPFH: max_distance is negative or NaN");
  if (k < 1 || k > 64) throw std::runtime_error("super4pcs-b200: ComputeFPFH: k is outside 1 .. 64");
  std::vector<FPFHSignature> out(cloud.size());
  if (cloud.empty()) return out;
  const std::size_t n = cloud.size();
  const std::vector<float> xyz = internal::Positions(cloud);
  std::vector<float> nrm(3 * n);
  for (std::size_t i = 0; i < n; ++i)
    for (int c = 0; c < 3; ++c) nrm[3 * i + c] = cloud[i].normal()[c];
  internal::WithContext("ComputeFPFH", [&](s4g_ctx* ctx) {
    const int rc = s4g_set_cloud_p(ctx, xyz.data(), int(n), internal::GridDelta(xyz, n, k));
    return rc == S4G_OK ? s4g_fpfh(ctx, nrm.data(), k, max_distance * max_distance, out.data()->data()) : rc;
  });
  return out;
}

std::vector<int> MatchFPFH(const std::vector<FPFHSignature>& source, const std::vector<FPFHSignature>& target,
                           bool mutual) {
  std::vector<int> index(source.size(), -1);
  if (source.empty()) return index;
  static_assert(sizeof(FPFHSignature) == 33 * sizeof(float), "FPFHSignature rows must be contiguous");
  static_assert(sizeof(int) == sizeof(int32_t), "int is 32 bits");
  internal::WithContext("MatchFPFH", [&](s4g_ctx* ctx) {
    return s4g_fpfh_match(ctx, source.data()->data(), int64_t(source.size()),
                          target.empty() ? nullptr : target.data()->data(), int64_t(target.size()), mutual ? 1 : 0,
                          reinterpret_cast<int32_t*>(index.data()), nullptr);
  });
  return index;
}

}  // namespace Utils
}  // namespace GlobalRegistration
