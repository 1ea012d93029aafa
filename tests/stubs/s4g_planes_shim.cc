// TEST INFRASTRUCTURE ONLY: answers s4g_segment_planes on the CPU for the C++ layer's tests of Utils::SegmentPlanes
// (tests/test_planes_cpu.py), next to the oracle stand-in of libs4g (tests/stubs/s4g_oracle_shim.cc), which has no such
// entry point.  Preloaded AHEAD of that stand-in (LD_PRELOAD="<this> <stand-in>"), it keeps a copy of the P cloud every
// context receives, passes the cloud and life-cycle calls on to the next definition (RTLD_NEXT), and answers the
// segmentation with the restatement of oracle/planes_port.cc, compiled into the same library.
#include <dlfcn.h>

#include <cmath>
#include <cstdint>
#include <map>
#include <mutex>
#include <vector>

#include "s4g.h"

extern "C" void planes_port(const float* P, long n, float threshold, int H, uint64_t seed, int refine, int max_planes,
                            int64_t min_inliers, int32_t* labels, void* planes, int* n_planes, int64_t* offsets,
                            int32_t* members, uint32_t* hyp_counts);

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

int s4g_segment_planes(s4g_ctx* c, float threshold, int n_hypotheses, uint64_t seed, int refine, int max_planes,
                       int64_t min_inliers, int32_t* labels, s4g_plane* planes, int* n_planes, int64_t* offsets,
                       int32_t* members, uint32_t* hyp_counts) {
  if (!c) return S4G_ERR_ARG;
  if (std::isnan(threshold) || threshold < 0.f || n_hypotheses < 1 || n_hypotheses > (1 << 20) || max_planes < 1 ||
      min_inliers < 1 || !labels || !planes || !n_planes)
    return S4G_ERR_ARG;
  std::lock_guard<std::mutex> lock(g_mu);
  auto it = g_P.find(c);
  if (it == g_P.end() || it->second.empty()) return S4G_ERR_STATE;
  const long n = (long)(it->second.size() / 3);
  std::vector<int64_t> off((size_t)max_planes + 1);
  std::vector<int32_t> mem((size_t)n);
  planes_port(it->second.data(), n, threshold, n_hypotheses, seed, refine, max_planes, min_inliers, labels, planes,
              n_planes, off.data(), mem.data(), hyp_counts);
  if (offsets)
    for (int k = 0; k <= *n_planes; ++k) offsets[k] = off[(size_t)k];
  if (members)
    for (int64_t k = 0; k < off[(size_t)*n_planes]; ++k) members[k] = mem[(size_t)k];
  return S4G_OK;
}

}  // extern "C"
