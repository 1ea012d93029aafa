// TEST INFRASTRUCTURE ONLY: answers s4g_range / s4g_get_range on the CPU for the C++ layer's host-logic tests
// (tests/test_range_cpu.py), next to the oracle stand-in of libs4g (tests/stubs/s4g_oracle_shim.cc), which has no such
// entry points.  Preloaded AHEAD of that stand-in (LD_PRELOAD="<this> <stand-in>"), it keeps a copy of the P cloud every
// context receives, passes the cloud and life-cycle calls on to the next definition (RTLD_NEXT), and answers s4g_range
// with the brute force of oracle/range_port.cc, which is compiled into the same library.
#include <dlfcn.h>

#include <cmath>
#include <cstdint>
#include <cstring>
#include <map>
#include <mutex>
#include <vector>

#include "s4g.h"

extern "C" void range_bruteforce_count(const float* P, long nP, const float* X, long n, const float* T, float sq_radius,
                                       int64_t* offsets);
extern "C" void range_bruteforce_fill(const float* P, long nP, const float* X, long n, const float* T, float sq_radius,
                                      const int64_t* offsets, int32_t* out_index, float* out_sq);

namespace {

struct State {
  std::vector<float> P;
  bool has_result = false;
  std::vector<int32_t> index;
  std::vector<float> sq;
};

std::mutex g_mu;
std::map<const s4g_ctx*, State> g_s;

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
    g_s[c].P.assign(xyz, xyz + 3 * (size_t)n);
  }
  return rc;
}

void s4g_destroy(s4g_ctx* c) {
  static const auto fwd = next<void (*)(s4g_ctx*)>("s4g_destroy");
  {
    std::lock_guard<std::mutex> lock(g_mu);
    g_s.erase(c);
  }
  fwd(c);
}

int s4g_range(s4g_ctx* c, const float* xyz, int n, const float* T, float sq_radius, int64_t* offsets, int64_t* total) {
  if (!c) return S4G_ERR_ARG;
  if (n < 0 || (n > 0 && !xyz) || !offsets || !total || std::isnan(sq_radius)) return S4G_ERR_ARG;
  std::lock_guard<std::mutex> lock(g_mu);
  auto it = g_s.find(c);
  if (it == g_s.end() || it->second.P.empty()) return S4G_ERR_STATE;
  State& s = it->second;
  const long nP = (long)(s.P.size() / 3);
  range_bruteforce_count(s.P.data(), nP, xyz, n, T, sq_radius, offsets);
  s.index.resize((size_t)offsets[n]);
  s.sq.resize((size_t)offsets[n]);
  range_bruteforce_fill(s.P.data(), nP, xyz, n, T, sq_radius, offsets, s.index.data(), s.sq.data());
  s.has_result = true;
  *total = offsets[n];
  return S4G_OK;
}

int s4g_get_range(s4g_ctx* c, int32_t* indices, float* sq_dist) {
  if (!c) return S4G_ERR_ARG;
  std::lock_guard<std::mutex> lock(g_mu);
  auto it = g_s.find(c);
  if (it == g_s.end() || !it->second.has_result) return S4G_ERR_STATE;
  const State& s = it->second;
  if (s.index.empty()) return S4G_OK;
  if (!indices) return S4G_ERR_ARG;
  std::memcpy(indices, s.index.data(), s.index.size() * sizeof(int32_t));
  if (sq_dist) std::memcpy(sq_dist, s.sq.data(), s.sq.size() * sizeof(float));
  return S4G_OK;
}

}  // extern "C"
