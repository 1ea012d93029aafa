// Test program of Utils::SegmentPlanes (tests/test_planes_cpu.py, tests/test_planes_gpu.py).  Linked against the C++
// layer; with LD_PRELOAD of the oracle stand-in it runs on the CPU.
//   planes_main IN OUT threshold max_planes min_inliers iterations seed refine
// IN : int32 n, float32 xyz[n][3]
// OUT: int32 threw (1: the call threw; nothing else follows), int32 n_planes, then per plane float32 coefficients[4],
//      int32 size and its int32 inliers
#include "super4pcs/utils/planes.h"

#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <vector>

using namespace GlobalRegistration;

int main(int argc, char** argv) {
  if (argc != 9) return 2;
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 2;
  int n = 0;
  if (std::fread(&n, sizeof(int), 1, in) != 1) return 2;
  std::vector<float> xyz(3 * size_t(n));
  if (std::fread(xyz.data(), sizeof(float), xyz.size(), in) != xyz.size()) return 2;
  std::fclose(in);
  std::vector<Point3D> cloud;
  for (int i = 0; i < n; ++i) cloud.emplace_back(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
  int threw = 0;
  std::vector<Utils::PlaneModel> planes;
  try {
    planes = Utils::SegmentPlanes(cloud, float(std::atof(argv[3])), std::atoi(argv[4]), std::atoi(argv[5]),
                                  std::atoi(argv[6]), std::strtoull(argv[7], nullptr, 10), std::atoi(argv[8]) != 0);
  } catch (const std::runtime_error&) {
    threw = 1;
  }
  FILE* out = std::fopen(argv[2], "wb");
  if (!out) return 2;
  std::fwrite(&threw, sizeof(int), 1, out);
  if (!threw) {
    const int m = int(planes.size());
    std::fwrite(&m, sizeof(int), 1, out);
    for (const Utils::PlaneModel& p : planes) {
      std::fwrite(p.coefficients.data(), sizeof(float), 4, out);
      const int s = int(p.inliers.size());
      std::fwrite(&s, sizeof(int), 1, out);
      std::fwrite(p.inliers.data(), sizeof(int), p.inliers.size(), out);
    }
  }
  std::fclose(out);
  return 0;
}
