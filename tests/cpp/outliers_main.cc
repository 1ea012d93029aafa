// Test program of Utils::RemoveStatisticalOutliers and Utils::RemoveRadiusOutliers (tests/test_outliers_cpu.py,
// tests/test_outliers_gpu.py).  Linked against the C++ layer; with LD_PRELOAD of the oracle stand-in it runs on
// the CPU.
//   outliers_main IN OUT statistical k std_ratio
//   outliers_main IN OUT radius radius min_neighbors
// IN : int32 n, float32 xyz[n][3], float32 normals[n][3], float32 rgb[n][3]
// OUT: int32 threw (1: the call threw; nothing else follows), int32 returned count, int32 m (points left),
//      float32 [m][9] (position, normal, rgb of each point left, as Point3D holds them)
#include "super4pcs/utils/outliers.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <vector>

using namespace GlobalRegistration;

int main(int argc, char** argv) {
  if (argc != 6) return 2;
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 2;
  int n = 0;
  if (std::fread(&n, sizeof(int), 1, in) != 1) return 2;
  std::vector<float> raw(9 * size_t(n));
  if (std::fread(raw.data(), sizeof(float), raw.size(), in) != raw.size()) return 2;
  std::fclose(in);
  const float* xyz = raw.data();
  const float* nrm = xyz + 3 * size_t(n);
  const float* rgb = nrm + 3 * size_t(n);
  std::vector<Point3D> cloud;
  for (int i = 0; i < n; ++i) {
    cloud.emplace_back(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
    cloud.back().set_normal(Point3D::VectorType(nrm[3 * i], nrm[3 * i + 1], nrm[3 * i + 2]));
    cloud.back().set_rgb(Point3D::VectorType(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]));
  }
  int threw = 0, count = 0;
  try {
    if (std::strcmp(argv[3], "statistical") == 0)
      count = Utils::RemoveStatisticalOutliers(cloud, std::atoi(argv[4]), std::atof(argv[5]));
    else
      count = Utils::RemoveRadiusOutliers(cloud, float(std::atof(argv[4])), std::atoi(argv[5]));
  } catch (const std::runtime_error&) {
    threw = 1;
  }
  FILE* out = std::fopen(argv[2], "wb");
  if (!out) return 2;
  std::fwrite(&threw, sizeof(int), 1, out);
  if (!threw) {
    const int m = int(cloud.size());
    std::fwrite(&count, sizeof(int), 1, out);
    std::fwrite(&m, sizeof(int), 1, out);
    for (const Point3D& p : cloud) {
      const float v[9] = {p.pos()[0],    p.pos()[1],    p.pos()[2], p.normal()[0], p.normal()[1],
                          p.normal()[2], p.rgb()[0], p.rgb()[1], p.rgb()[2]};
      std::fwrite(v, sizeof(float), 9, out);
    }
  }
  std::fclose(out);
  return 0;
}
