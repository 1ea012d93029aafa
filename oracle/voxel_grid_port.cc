// TEST INFRASTRUCTURE ONLY (oracle/_build.py and tests/build_shim.py build it; never linked into the product).
//
// Plain restatement of s4g_voxel_grid (include/s4g.h), operation for operation:
//   s = 1.0f / leaf; the voxel of point i is (floor(fl(x s)), floor(fl(y s)), floor(fl(z s))); a floor that is NaN or
//   outside [-2^31, 2^31) (every non-finite coordinate among them) or a span of 2^21 or more voxels per axis -> error 2;
//   members of a voxel in ascending i; each sum in double: runs of 1024 members summed left to right from 0.0, then the
//   run sums left to right from 0.0; centroid and rgb = sum / m, normal = S / sqrt((Sx Sx + Sy Sy) + Sz Sz) or 0 when
//   that is 0, each rounded to float; voxels with m < min_points dropped; output in ascending order of the first member.
// Compiled -ffp-contract=off: no FMA, as the device.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

extern "C" {

// 0, or 2 (S4G_ERR_ARG) for bad arguments, an invalid coordinate or too wide a span.  Outputs of capacity n; normals /
// normals_out, rgb / rgb_out, counts, first and voxel_of may be null.
int voxel_grid_port(const float* xyz, const float* normals, const float* rgb, long n, float leaf, int min_points,
                    float* xyz_out, float* normals_out, float* rgb_out, int32_t* counts, int32_t* first,
                    int32_t* voxel_of, int64_t* n_out) {
  if (!std::isfinite(leaf) || !(leaf > 0.f) || min_points < 1 || n < 0 || n >= (1l << 31)) return 2;
  if ((normals == nullptr) != (normals_out == nullptr) || (rgb == nullptr) != (rgb_out == nullptr)) return 2;
  *n_out = 0;
  if (n == 0) return 0;
  const float s = 1.0f / leaf;
  std::vector<int64_t> cell(3 * (size_t)n);
  int64_t lo[3] = {INT64_MAX, INT64_MAX, INT64_MAX}, hi[3] = {INT64_MIN, INT64_MIN, INT64_MIN};
  for (long i = 0; i < n; ++i)
    for (int a = 0; a < 3; ++a) {
      const float c = std::floor(xyz[3 * i + a] * s);
      if (!(c >= -2147483648.f && c < 2147483648.f)) return 2;
      cell[3 * i + a] = (int64_t)c;
      lo[a] = std::min(lo[a], cell[3 * i + a]);
      hi[a] = std::max(hi[a], cell[3 * i + a]);
    }
  for (int a = 0; a < 3; ++a)
    if (hi[a] - lo[a] >= (1ll << 21)) return 2;
  std::vector<std::pair<uint64_t, int32_t>> key((size_t)n);
  for (long i = 0; i < n; ++i) {
    const uint64_t k = ((uint64_t)(cell[3 * i] - lo[0]) << 42) | ((uint64_t)(cell[3 * i + 1] - lo[1]) << 21) |
                       (uint64_t)(cell[3 * i + 2] - lo[2]);
    key[i] = {k, (int32_t)i};
  }
  std::sort(key.begin(), key.end());   // (key, i): members in ascending i
  // voxels as [b, e) of the sorted list; the survivors in ascending order of their first member
  std::vector<std::pair<int32_t, long>> order;   // (first member, b)
  std::vector<long> end_of;
  for (long b = 0; b < n;) {
    long e = b + 1;
    while (e < n && key[e].first == key[b].first) ++e;
    if (e - b >= min_points) order.push_back({key[b].second, b});
    end_of.push_back(e);
    b = e;
  }
  std::sort(order.begin(), order.end());
  if (voxel_of)
    for (long i = 0; i < n; ++i) voxel_of[i] = -1;
  const float* src[3] = {xyz, normals, rgb};
  for (size_t o = 0; o < order.size(); ++o) {
    const long b = order[o].second;
    long e = b + 1;
    while (e < n && key[e].first == key[b].first) ++e;
    const long m = e - b;
    double S[9];
    for (int c = 0; c < 9; ++c) {
      const float* x = src[c / 3];
      double total = 0.0;
      if (x)
        for (long r = b; r < e; r += 1024) {
          double run = 0.0;
          for (long t = r; t < e && t < r + 1024; ++t) run = run + (double)x[3 * (long)key[t].second + c % 3];
          total = total + run;
        }
      S[c] = total;
    }
    for (int a = 0; a < 3; ++a) xyz_out[3 * o + a] = (float)(S[a] / (double)m);
    if (normals) {
      const double len = std::sqrt((S[3] * S[3] + S[4] * S[4]) + S[5] * S[5]);
      for (int a = 0; a < 3; ++a) normals_out[3 * o + a] = len == 0.0 ? 0.f : (float)(S[3 + a] / len);
    }
    if (rgb)
      for (int a = 0; a < 3; ++a) rgb_out[3 * o + a] = (float)(S[6 + a] / (double)m);
    if (counts) counts[o] = (int32_t)m;
    if (first) first[o] = key[b].second;
    if (voxel_of)
      for (long t = b; t < e; ++t) voxel_of[key[t].second] = (int32_t)o;
  }
  *n_out = (int64_t)order.size();
  return 0;
}

}  // extern "C"
