// Test program of Utils::ComputeFPFH and Utils::MatchFPFH (tests/test_fpfh_cpu.py, tests/test_fpfh_gpu.py).  Linked
// against the C++ layer; with LD_PRELOAD of the oracle stand-in it runs on the CPU.
//   fpfh_main IN OUT compute k max_distance
//     IN : int32 n, float32 xyz[n][3], float32 normals[n][3] (stored through Point3D::set_normal)
//     OUT: int32 threw (1: ComputeFPFH threw), float32 fpfh[n][33] (when it did not throw)
//   fpfh_main IN OUT match mutual
//     IN : int32 n_source, int32 n_target, float32 source[n_source][33], float32 target[n_target][33]
//     OUT: int32 threw (1: MatchFPFH threw), int32 index[n_source] (when it did not throw)
#include "super4pcs/utils/features.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <vector>

using namespace GlobalRegistration;

int main(int argc, char** argv) {
  if (argc < 4) return 2;
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 2;
  int threw = 0;
  std::vector<float> outf;
  std::vector<int> outi;
  if (std::strcmp(argv[3], "compute") == 0 && argc == 6) {
    int n = 0;
    if (std::fread(&n, sizeof(int), 1, in) != 1) return 2;
    std::vector<float> raw(6 * size_t(n));
    if (std::fread(raw.data(), sizeof(float), raw.size(), in) != raw.size()) return 2;
    std::vector<Point3D> cloud;
    for (int i = 0; i < n; ++i) {
      cloud.emplace_back(raw[3 * i], raw[3 * i + 1], raw[3 * i + 2]);
      const size_t o = 3 * (size_t(n) + i);
      cloud.back().set_normal(Point3D::VectorType(raw[o], raw[o + 1], raw[o + 2]));
    }
    try {
      for (const Utils::FPFHSignature& f : Utils::ComputeFPFH(cloud, std::atoi(argv[4]), float(std::atof(argv[5]))))
        outf.insert(outf.end(), f.begin(), f.end());
    } catch (const std::runtime_error&) {
      threw = 1;
    }
  } else if (std::strcmp(argv[3], "match") == 0 && argc == 5) {
    int ns = 0, nt = 0;
    if (std::fread(&ns, sizeof(int), 1, in) != 1 || std::fread(&nt, sizeof(int), 1, in) != 1) return 2;
    std::vector<Utils::FPFHSignature> s(ns), t(nt);
    for (auto& f : s)
      if (std::fread(f.data(), sizeof(float), 33, in) != 33) return 2;
    for (auto& f : t)
      if (std::fread(f.data(), sizeof(float), 33, in) != 33) return 2;
    try {
      outi = Utils::MatchFPFH(s, t, std::atoi(argv[4]) != 0);
    } catch (const std::runtime_error&) {
      threw = 1;
    }
  } else {
    return 2;
  }
  std::fclose(in);
  FILE* out = std::fopen(argv[2], "wb");
  if (!out) return 2;
  std::fwrite(&threw, sizeof(int), 1, out);
  if (!outf.empty()) std::fwrite(outf.data(), sizeof(float), outf.size(), out);
  if (!outi.empty()) std::fwrite(outi.data(), sizeof(int), outi.size(), out);
  std::fclose(out);
  return 0;
}
