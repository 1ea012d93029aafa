// TEST INFRASTRUCTURE ONLY: answers s4g_statistical_outliers and s4g_radius_outliers on the CPU for the C++ layer's tests
// of Utils::RemoveStatisticalOutliers and Utils::RemoveRadiusOutliers (tests/test_outliers_cpu.py), next to the oracle
// stand-in of libs4g (tests/stubs/s4g_oracle_shim.cc), which has no such entry points.  Preloaded AHEAD of that stand-in
// (LD_PRELOAD="<this> <stand-in>"), it keeps a copy of the P cloud every context receives, passes the cloud and life-cycle
// calls on to the next definition (RTLD_NEXT), and answers the two filters with the restatement of
// oracle/outliers_port.cc (and the brute force of oracle/knn_port.cc), compiled into the same library.
#include <dlfcn.h>

#include <cmath>
#include <cstdint>
#include <map>
#include <mutex>
#include <vector>

#include "s4g.h"

extern "C" void statistical_port(const float* P, long nP, int k, double std_ratio, uint8_t* flags, double* mean_dist,
                                 double* out2);
extern "C" void radius_port(const float* P, long nP, float sq_radius, int min_neighbors, int64_t* raw, int32_t* counts,
                            uint8_t* flags);

namespace {

std::mutex g_mu;
std::map<const s4g_ctx*, std::vector<float>> g_P;

template <class F>
F next(const char* name) {
  return reinterpret_cast<F>(dlsym(RTLD_NEXT, name));
}

// the flagged j, ascending
void compact(const std::vector<uint8_t>& flags, int32_t* keep, int64_t* n_kept) {
  int64_t m = 0;
  for (std::size_t j = 0; j < flags.size(); ++j)
    if (flags[j]) keep[m++] = (int32_t)j;
  *n_kept = m;
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

int s4g_statistical_outliers(s4g_ctx* c, int k, double std_ratio, int32_t* keep, int64_t* n_kept, double* mean_dist,
                             double* out2) {
  if (!c) return S4G_ERR_ARG;
  if (k < 1 || k > 64 || !std::isfinite(std_ratio) || !keep || !n_kept) return S4G_ERR_ARG;
  std::lock_guard<std::mutex> lock(g_mu);
  auto it = g_P.find(c);
  if (it == g_P.end() || it->second.empty()) return S4G_ERR_STATE;
  const long n = (long)(it->second.size() / 3);
  std::vector<uint8_t> flags(n);
  std::vector<double> mean(n);
  double o2[2];
  statistical_port(it->second.data(), n, k, std_ratio, flags.data(), mean.data(), o2);
  compact(flags, keep, n_kept);
  if (mean_dist)
    for (long j = 0; j < n; ++j) mean_dist[j] = mean[j];
  if (out2) out2[0] = o2[0], out2[1] = o2[1];
  return S4G_OK;
}

int s4g_radius_outliers(s4g_ctx* c, float sq_radius, int min_neighbors, int32_t* keep, int64_t* n_kept, int32_t* counts) {
  if (!c) return S4G_ERR_ARG;
  if (std::isnan(sq_radius) || min_neighbors < 1 || !keep || !n_kept) return S4G_ERR_ARG;
  std::lock_guard<std::mutex> lock(g_mu);
  auto it = g_P.find(c);
  if (it == g_P.end() || it->second.empty()) return S4G_ERR_STATE;
  const long n = (long)(it->second.size() / 3);
  std::vector<uint8_t> flags(n);
  std::vector<int32_t> cnt(n);
  radius_port(it->second.data(), n, sq_radius, min_neighbors, nullptr, cnt.data(), flags.data());
  compact(flags, keep, n_kept);
  if (counts)
    for (long j = 0; j < n; ++j) counts[j] = cnt[j];
  return S4G_OK;
}

}  // extern "C"
