// TEST INFRASTRUCTURE ONLY: answers s4g_knn on the CPU for the C++ layer's host-logic tests (tests/test_knn_cpu.py), next
// to the oracle stand-in of libs4g (tests/stubs/s4g_oracle_shim.cc), which has no such entry point.  Preloaded AHEAD of
// that stand-in (LD_PRELOAD="<this> <stand-in>"), it keeps a copy of the P cloud every context receives, passes the
// cloud and life-cycle calls on to the next definition (RTLD_NEXT), and answers s4g_knn with the brute force of
// oracle/knn_port.cc, which is compiled into the same library.
#include <dlfcn.h>

#include <cmath>
#include <cstdint>
#include <map>
#include <mutex>
#include <vector>

#include "s4g.h"

extern "C" void knn_bruteforce(const float* P, long nP, const float* X, long n, const float* T, int k, float sq_radius,
                               const int32_t* exclude, int32_t* out_index, float* out_sq);

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

int s4g_knn(s4g_ctx* c, const float* xyz, int n, const float* T, int k, float sq_radius, const int32_t* exclude,
            int32_t* index, float* sq_dist) {
  if (!c) return S4G_ERR_ARG;
  if (n < 0 || (n > 0 && (!xyz || !index)) || k < 1 || k > 64 || std::isnan(sq_radius)) return S4G_ERR_ARG;
  std::lock_guard<std::mutex> lock(g_mu);
  auto it = g_P.find(c);
  if (it == g_P.end() || it->second.empty()) return S4G_ERR_STATE;
  knn_bruteforce(it->second.data(), (long)(it->second.size() / 3), xyz, n, T, k, sq_radius, exclude, index, sq_dist);
  return S4G_OK;
}

}  // extern "C"
