// TEST INFRASTRUCTURE ONLY: answers s4g_orient_normals on the CPU for the C++ layer's tests of Utils::OrientNormals
// (tests/test_orient_normals_cpu.py), next to the oracle stand-in of libs4g (tests/stubs/s4g_oracle_shim.cc), which has
// no such entry point.  Preloaded AHEAD of that stand-in (LD_PRELOAD="<this> <stand-in>"), it keeps a copy of the P
// cloud every context receives, passes the cloud and life-cycle calls on to the next definition (RTLD_NEXT), and answers
// s4g_orient_normals with the restatement of oracle/orient_normals_port.cc (and the brute force of oracle/knn_port.cc),
// compiled into the same library.
#include <dlfcn.h>

#include <cstdint>
#include <map>
#include <mutex>
#include <vector>

#include "s4g.h"

extern "C" int orient_normals_port(const float* P, long n, const float* normals, int k, float sq_radius,
                                   const float* viewpoint, const int32_t* rows_in, float* normals_out, int32_t* root,
                                   int64_t* out2, int32_t* tree_edges);

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

int s4g_orient_normals(s4g_ctx* c, const float* normals, int k, float sq_radius, const float* viewpoint,
                       float* normals_out, int32_t* root, int64_t* out2, int32_t* tree_edges) {
  if (!c) return S4G_ERR_ARG;
  std::lock_guard<std::mutex> lock(g_mu);
  auto it = g_P.find(c);
  if (it == g_P.end() || it->second.empty()) return S4G_ERR_STATE;
  const long n = (long)(it->second.size() / 3);
  return orient_normals_port(it->second.data(), n, normals, k, sq_radius, viewpoint, nullptr, normals_out, root, out2,
                             tree_edges) == 0 ? S4G_OK : S4G_ERR_ARG;
}

}  // extern "C"
