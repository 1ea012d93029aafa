// Test program of Match4PCSBase::getKNearest (tests/test_knn_cpu.py, tests/test_knn_gpu.py): runs
// MatchSuper4PCS::ComputeTransformation on two clouds, then the k nearest neighbours under the found transform for a few
// (k, max_distance).  Linked against the C++ layer; with LD_PRELOAD of the oracle stand-in it runs on the CPU.
//   knn_main IN OUT delta overlap sample_size
// IN : int32 nP, int32 nQ, float32 P[nP][3], float32 Q[nQ][3]
// OUT: int32 threw_before (1: getKNearest threw before any registration), float32 score, float32 C[16] (the centred
//      transform behind the score, column-major), int32 nSP, float32 sampled P[nSP][3], int32 nSQ, float32 sampled
//      Q[nSQ][3], int32 K, K x (int32 k, float32 max_distance), K x (int32 indices[nSQ][k], float32 sq[nSQ][k])
#include "super4pcs/algorithms/super4pcs.h"

#include <cstdio>
#include <cstdlib>
#include <limits>
#include <stdexcept>
#include <vector>

using namespace GlobalRegistration;

namespace {
struct Probe : MatchSuper4PCS {
  Probe(const Match4PCSOptions& o, const Utils::Logger& l) : MatchSuper4PCS(o, l) {}
  const MatrixType& centred() const { return transform_; }
};

template <class T> void put(FILE* f, const T* p, size_t n) { std::fwrite(p, sizeof(T), n, f); }

void put_cloud(FILE* f, const std::vector<Point3D>& c) {
  const int n = (int)c.size();
  put(f, &n, 1);
  for (const Point3D& p : c) {
    const float xyz[3] = {p.pos()[0], p.pos()[1], p.pos()[2]};
    put(f, xyz, 3);
  }
}
}  // namespace

int main(int argc, char** argv) {
  if (argc != 6) return 2;
  FILE* in = std::fopen(argv[1], "rb");
  if (!in) return 2;
  int n[2] = {0, 0};
  if (std::fread(n, sizeof(int), 2, in) != 2) return 2;
  std::vector<float> raw(3 * size_t(n[0] + n[1]));
  if (std::fread(raw.data(), sizeof(float), raw.size(), in) != raw.size()) return 2;
  std::fclose(in);
  std::vector<Point3D> P, Q;
  for (int i = 0; i < n[0] + n[1]; ++i) (i < n[0] ? P : Q).emplace_back(raw[3 * i], raw[3 * i + 1], raw[3 * i + 2]);

  Match4PCSOptions opt;
  opt.delta = (float)std::atof(argv[3]);
  opt.sample_size = (size_t)std::atol(argv[5]);
  opt.max_time_seconds = 1000;
  opt.configureOverlap((float)std::atof(argv[4]));
  Utils::Logger logger(Utils::NoLog);
  Probe m(opt, logger);

  int threw_before = 0;
  std::vector<int> indices;
  std::vector<float> sq;
  try {
    m.getKNearest(&indices, &sq, 4);
  } catch (const std::runtime_error&) {
    threw_before = 1;
  }
  Match4PCSBase::MatrixType T = Match4PCSBase::MatrixType::Identity();
  const float score = m.ComputeTransformation(P, &Q, T);

  FILE* out = std::fopen(argv[2], "wb");
  if (!out) return 2;
  put(out, &threw_before, 1);
  put(out, &score, 1);
  const Match4PCSBase::MatrixType C = m.centred();
  put(out, C.data(), 16);
  put_cloud(out, m.getFirstSampled());
  put_cloud(out, m.getSecondSampled());
  const float inf = std::numeric_limits<float>::infinity();
  const std::vector<std::pair<int, float>> runs = {{1, opt.delta}, {8, 3 * opt.delta}, {16, inf}, {64, inf}};
  const int K = (int)runs.size();
  put(out, &K, 1);
  for (const auto& r : runs) {
    put(out, &r.first, 1);
    put(out, &r.second, 1);
  }
  for (const auto& r : runs) {
    if (r.second == inf) m.getKNearest(&indices, &sq, r.first);   // the default max_distance
    else m.getKNearest(&indices, &sq, r.first, r.second);
    put(out, indices.data(), indices.size());
    put(out, sq.data(), sq.size());
  }
  std::fclose(out);
  return 0;
}
