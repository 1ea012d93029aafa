// TEST INFRASTRUCTURE ONLY: answers s4g_verify_nearest on the CPU for the C++ layer's host-logic tests
// (tests/test_verify_nearest_cpu.py), next to the oracle stand-in of libs4g (tests/stubs/s4g_oracle_shim.cc), which has no
// such entry point.  Preloaded AHEAD of that stand-in (LD_PRELOAD="<this> <stand-in>"), it keeps a copy of the clouds every
// context receives, passes the cloud and life-cycle calls on to the next definition (RTLD_NEXT), and answers
// s4g_verify_nearest with the brute force of oracle/nearest_port.cc, which is compiled into the same library.
#include <dlfcn.h>

#include <cstdint>
#include <map>
#include <mutex>
#include <vector>

#include "s4g.h"

extern "C" void nearest_bruteforce(const float* P, long nP, const float* Q, long nQ, float delta, const float* T16k, long K,
                                   int32_t* out_index, float* out_sq, uint32_t* out_counts);

namespace {

struct Clouds {
  std::vector<float> P, Q;
  float delta = 0.f;
};
std::mutex g_mu;
std::map<const s4g_ctx*, Clouds> g_clouds;

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
    Clouds& k = g_clouds[c];
    k.P.assign(xyz, xyz + 3 * (size_t)n);
    k.delta = delta;
  }
  return rc;
}

int s4g_set_cloud_q(s4g_ctx* c, const float* xyz, const float* normals, const float* rgb, int n) {
  static const auto fwd = next<int (*)(s4g_ctx*, const float*, const float*, const float*, int)>("s4g_set_cloud_q");
  const int rc = fwd(c, xyz, normals, rgb, n);
  if (rc == S4G_OK) {
    std::lock_guard<std::mutex> lock(g_mu);
    g_clouds[c].Q.assign(xyz, xyz + 3 * (size_t)n);
  }
  return rc;
}

void s4g_destroy(s4g_ctx* c) {
  static const auto fwd = next<void (*)(s4g_ctx*)>("s4g_destroy");
  {
    std::lock_guard<std::mutex> lock(g_mu);
    g_clouds.erase(c);
  }
  fwd(c);
}

int s4g_verify_nearest(s4g_ctx* c, const float* T, int K, int32_t* index, float* sq_dist, uint32_t* counts) {
  if (!c) return S4G_ERR_ARG;
  if (K < 0 || (K > 0 && (!T || !index))) return S4G_ERR_ARG;
  Clouds k;
  {
    std::lock_guard<std::mutex> lock(g_mu);
    auto it = g_clouds.find(c);
    if (it == g_clouds.end() || it->second.P.empty() || it->second.Q.empty()) return S4G_ERR_STATE;
    k = it->second;
  }
  if (K > 0)
    nearest_bruteforce(k.P.data(), (long)(k.P.size() / 3), k.Q.data(), (long)(k.Q.size() / 3), k.delta, T, K, index,
                       sq_dist, counts);
  return S4G_OK;
}

}  // extern "C"
