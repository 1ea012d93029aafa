// TEST INFRASTRUCTURE ONLY: answers s4g_fpfh and s4g_fpfh_match on the CPU for the C++ layer's tests of
// Utils::ComputeFPFH and Utils::MatchFPFH (tests/test_fpfh_cpu.py), next to the oracle stand-in of libs4g
// (tests/stubs/s4g_oracle_shim.cc), which has no such entry points.  Preloaded AHEAD of that stand-in (LD_PRELOAD="<this>
// <stand-in>"), it keeps a copy of the P cloud every context receives, passes the cloud and life-cycle calls on to the
// next definition (RTLD_NEXT), and answers the two calls with the restatement of oracle/fpfh_port.cc (and the brute
// force of oracle/knn_port.cc), compiled into the same library.
#include <dlfcn.h>

#include <cstdint>
#include <map>
#include <mutex>
#include <vector>

#include "s4g.h"

extern "C" int fpfh_port(const float* P, long n, const float* normals, int k, float sq_radius, const int32_t* rows_in,
                         const float* sq_in, float* fpfh, double* spfh_out);
extern "C" void fpfh_match_port(const float* a, long na, const float* b, long nb, int mutual, int32_t* index,
                                float* sq_dist);

namespace {

std::mutex g_mu;
std::map<const s4g_ctx*, std::vector<float>> g_P;

template <class F>
F next(const char* name) {
  return reinterpret_cast<F>(dlsym(RTLD_NEXT, name));
}

}  // namespace

extern "C" {

int s4g_set_cloud_p(s4g_ctx* c, const float* xyz, int n, float delta) {
  static const auto fwd = next<int (*)(s4g_ctx*, const float*, int, float)>("s4g_set_cloud_p");
  const int rc = fwd(c, xyz, n, delta);
  if (rc == S4G_OK) {
    std::lock_guard<std::mutex> lock(g_mu);
    g_P[c].assign(xyz, xyz + 3 * (size_t)n);
  }
  return rc;
}

void s4g_destroy(s4g_ctx* c) {
  static const auto fwd = next<void (*)(s4g_ctx*)>("s4g_destroy");
  {
    std::lock_guard<std::mutex> lock(g_mu);
    g_P.erase(c);
  }
  fwd(c);
}

int s4g_fpfh(s4g_ctx* c, const float* normals, int k, float sq_radius, float* fpfh) {
  if (!c) return S4G_ERR_ARG;
  std::lock_guard<std::mutex> lock(g_mu);
  auto it = g_P.find(c);
  if (it == g_P.end() || it->second.empty()) return S4G_ERR_STATE;
  const long n = (long)(it->second.size() / 3);
  return fpfh_port(it->second.data(), n, normals, k, sq_radius, nullptr, nullptr, fpfh, nullptr) == 0 ? S4G_OK
                                                                                                       : S4G_ERR_ARG;
}

int s4g_fpfh_match(s4g_ctx* c, const float* a, int64_t n_a, const float* b, int64_t n_b, int mutual, int32_t* index,
                   float* sq_dist) {
  if (!c || n_a < 0 || n_b < 0 || (n_a > 0 && (!a || !index)) || (n_a > 0 && n_b > 0 && !b)) return S4G_ERR_ARG;
  if (n_a > 0) fpfh_match_port(a, (long)n_a, b, (long)n_b, mutual, index, sq_dist);
  return S4G_OK;
}

}  // extern "C"
