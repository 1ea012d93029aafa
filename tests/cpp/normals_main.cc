// Test program of Utils::EstimateNormals (tests/test_normals_cpu.py, tests/test_normals_gpu.py).  Linked against the C++
// layer; with LD_PRELOAD of the oracle stand-in it runs on the CPU.
//   normals_main IN OUT k max_distance [vx vy vz]
// IN : int32 n, float32 xyz[n][3]
// OUT: int32 threw (1: EstimateNormals threw; nothing else follows), int32 returned count, float32 normals[n][3] (what
//      Point3D::normal() holds afterwards)
#include "super4pcs/utils/normals.h"

#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <vector>

using namespace GlobalRegistration;

int main(int argc, char** argv) {
  if (argc != 5 && argc != 8) return 2;
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 2;
  int n = 0;
  if (std::fread(&n, sizeof(int), 1, in) != 1) return 2;
  std::vector<float> raw(3 * size_t(n));
  if (std::fread(raw.data(), sizeof(float), raw.size(), in) != raw.size()) return 2;
  std::fclose(in);
  std::vector<Point3D> cloud;
  for (int i = 0; i < n; ++i) cloud.emplace_back(raw[3 * i], raw[3 * i + 1], raw[3 * i + 2]);
  Point3D::VectorType vp;
  if (argc == 8) vp = Point3D::VectorType(float(std::atof(argv[5])), float(std::atof(argv[6])), float(std::atof(argv[7])));
  int threw = 0, count = 0;
  try {
    count = Utils::EstimateNormals(cloud, std::atoi(argv[3]), float(std::atof(argv[4])), argc == 8 ? &vp : nullptr);
  } catch (const std::runtime_error&) {
    threw = 1;
  }
  FILE* out = std::fopen(argv[2], "wb");
  if (!out) return 2;
  std::fwrite(&threw, sizeof(int), 1, out);
  if (!threw) {
    std::fwrite(&count, sizeof(int), 1, out);
    for (const Point3D& p : cloud) {
      const float v[3] = {p.normal()[0], p.normal()[1], p.normal()[2]};
      std::fwrite(v, sizeof(float), 3, out);
    }
  }
  std::fclose(out);
  return 0;
}
