// TEST INFRASTRUCTURE ONLY: answers s4g_voxel_grid on the CPU for the C++ layer's tests of Utils::VoxelGridFilter
// (tests/test_voxel_grid_cpu.py), next to the oracle stand-in of libs4g (tests/stubs/s4g_oracle_shim.cc), which has no
// such entry point and provides the context's life cycle.  Preloaded AHEAD of that stand-in (LD_PRELOAD="<this>
// <stand-in>"), it answers the call with the restatement of oracle/voxel_grid_port.cc, compiled into the same library.
#include <cstdint>

#include "s4g.h"

extern "C" int voxel_grid_port(const float* xyz, const float* normals, const float* rgb, long n, float leaf,
                               int min_points, float* xyz_out, float* normals_out, float* rgb_out, int32_t* counts,
                               int32_t* first, int32_t* voxel_of, int64_t* n_out);

extern "C" int s4g_voxel_grid(s4g_ctx* ctx, const float* xyz, const float* normals, const float* rgb, int64_t n,
                              float leaf, int min_points, float* xyz_out, float* normals_out, float* rgb_out,
                              int32_t* counts, int32_t* first, int32_t* voxel_of, int64_t* n_out) {
  if (!ctx || !xyz || !xyz_out || !n_out) return S4G_ERR_ARG;
  return voxel_grid_port(xyz, normals, rgb, (long)n, leaf, min_points, xyz_out, normals_out, rgb_out, counts, first,
                         voxel_of, n_out);
}
