// Test program of Match4PCSBase::getCorrespondences (tests/test_verify_nearest_cpu.py, tests/test_verify_nearest_gpu.py):
// runs MatchSuper4PCS::ComputeTransformation on two clouds and writes what the registration found together with the
// correspondences of its transform.  Linked against the C++ layer; with LD_PRELOAD of the oracle stand-in it runs on the
// CPU.
//   correspondences_main IN OUT delta overlap sample_size
// IN : int32 nP, int32 nQ, float32 P[nP][3], float32 Q[nQ][3]
// OUT: int32 threw_before (1: getCorrespondences threw before any registration), float32 score, float32 T[16]
//      (the returned global transform, column-major), float32 C[16] (the centred transform behind the score),
//      int32 nSP, int32 nSQ, float32 sampled P[nSP][3], float32 sampled Q[nSQ][3], int32 nearest[nSQ], float32 sq[nSQ],
//      int32 nearest2[nSQ] (the call without sq_dist)
#include "super4pcs/algorithms/super4pcs.h"

#include <cstdio>
#include <cstdlib>
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
  std::vector<int> nearest, nearest2;
  std::vector<float> sq;
  try {
    m.getCorrespondences(&nearest);
  } catch (const std::runtime_error&) {
    threw_before = 1;
  }
  Match4PCSBase::MatrixType T = Match4PCSBase::MatrixType::Identity();
  const float score = m.ComputeTransformation(P, &Q, T);
  m.getCorrespondences(&nearest, &sq);
  m.getCorrespondences(&nearest2);

  FILE* out = std::fopen(argv[2], "wb");
  if (!out) return 2;
  put(out, &threw_before, 1);
  put(out, &score, 1);
  put(out, T.data(), 16);
  const Match4PCSBase::MatrixType C = m.centred();
  put(out, C.data(), 16);
  put_cloud(out, m.getFirstSampled());
  put_cloud(out, m.getSecondSampled());
  put(out, nearest.data(), nearest.size());
  put(out, sq.data(), sq.size());
  put(out, nearest2.data(), nearest2.size());
  std::fclose(out);
  return 0;
}
