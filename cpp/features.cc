// super4pcs-b200: Utils::ComputeFPFH and Utils::MatchFPFH on top of s4g_fpfh and s4g_fpfh_match (include/s4g.h).
#include "super4pcs/utils/features.h"

#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <stdexcept>
#include <string>

#include "grid_delta.h"
#include "s4g.h"

namespace GlobalRegistration {
namespace Utils {

namespace {

s4g_ctx* create(const char* who) {
  int device = 0;
  if (const char* e = std::getenv("S4PCS_DEVICE")) device = std::atoi(e);
  s4g_ctx* ctx = nullptr;
  if (s4g_create(device, &ctx) != S4G_OK)
    throw std::runtime_error(std::string("super4pcs-b200: ") + who + ": no CUDA device (there is no CPU fallback)");
  return ctx;
}

void finish(s4g_ctx* ctx, int rc, const char* who) {
  const std::string msg = rc == S4G_OK ? std::string() : std::string(s4g_error_string(ctx));
  s4g_destroy(ctx);
  if (rc != S4G_OK) throw std::runtime_error(std::string("super4pcs-b200: ") + who + ": " + msg);
}

}  // namespace

std::vector<FPFHSignature> ComputeFPFH(const std::vector<Point3D>& cloud, int k, Point3D::Scalar max_distance) {
  if (std::isnan(max_distance) || max_distance < 0)
    throw std::runtime_error("super4pcs-b200: ComputeFPFH: max_distance is negative or NaN");
  if (k < 1 || k > 64) throw std::runtime_error("super4pcs-b200: ComputeFPFH: k is outside 1 .. 64");
  std::vector<FPFHSignature> out(cloud.size());
  if (cloud.empty()) return out;
  const std::size_t n = cloud.size();
  std::vector<float> xyz(3 * n), nrm(3 * n);
  for (std::size_t i = 0; i < n; ++i)
    for (int c = 0; c < 3; ++c) {
      xyz[3 * i + c] = cloud[i].pos()[c];
      nrm[3 * i + c] = cloud[i].normal()[c];
    }
  s4g_ctx* ctx = create("ComputeFPFH");
  int rc = s4g_set_cloud_p(ctx, xyz.data(), int(n), internal::GridDelta(xyz, n, k));
  if (rc == S4G_OK) rc = s4g_fpfh(ctx, nrm.data(), k, max_distance * max_distance, out.data()->data());
  finish(ctx, rc, "ComputeFPFH");
  return out;
}

std::vector<int> MatchFPFH(const std::vector<FPFHSignature>& source, const std::vector<FPFHSignature>& target,
                           bool mutual) {
  std::vector<int> index(source.size(), -1);
  if (source.empty()) return index;
  static_assert(sizeof(FPFHSignature) == 33 * sizeof(float), "FPFHSignature rows must be contiguous");
  static_assert(sizeof(int) == sizeof(int32_t), "int is 32 bits");
  s4g_ctx* ctx = create("MatchFPFH");
  const int rc = s4g_fpfh_match(ctx, source.data()->data(), int64_t(source.size()),
                                target.empty() ? nullptr : target.data()->data(), int64_t(target.size()), mutual ? 1 : 0,
                                reinterpret_cast<int32_t*>(index.data()), nullptr);
  finish(ctx, rc, "MatchFPFH");
  return index;
}

}  // namespace Utils
}  // namespace GlobalRegistration
