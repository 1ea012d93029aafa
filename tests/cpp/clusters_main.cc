// Test program of Utils::ExtractEuclideanClusters (tests/test_clusters_cpu.py, tests/test_clusters_gpu.py).  Linked
// against the C++ layer; with LD_PRELOAD of the oracle stand-in it runs on the CPU.
//   clusters_main IN OUT tolerance min_size max_size
// IN : int32 n, float32 xyz[n][3]
// OUT: int32 threw (1: the call threw; nothing else follows), int32 n_clusters, then per cluster int32 size and its
//      int32 indices
#include "super4pcs/utils/clusters.h"

#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <vector>

using namespace GlobalRegistration;

int main(int argc, char** argv) {
  if (argc != 6) return 2;
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
  std::vector<std::vector<int>> clusters;
  try {
    clusters = Utils::ExtractEuclideanClusters(cloud, float(std::atof(argv[3])), std::atoi(argv[4]), std::atoi(argv[5]));
  } catch (const std::runtime_error&) {
    threw = 1;
  }
  FILE* out = std::fopen(argv[2], "wb");
  if (!out) return 2;
  std::fwrite(&threw, sizeof(int), 1, out);
  if (!threw) {
    const int m = int(clusters.size());
    std::fwrite(&m, sizeof(int), 1, out);
    for (const std::vector<int>& c : clusters) {
      const int s = int(c.size());
      std::fwrite(&s, sizeof(int), 1, out);
      std::fwrite(c.data(), sizeof(int), c.size(), out);
    }
  }
  std::fclose(out);
  return 0;
}
