// Test program of Match4PCSBase::getNeighbors (tests/test_range_cpu.py, tests/test_range_gpu.py): runs
// MatchSuper4PCS::ComputeTransformation on two clouds, then the neighbours of the found transform at max_distance =
// delta and 3 delta.  Linked against the C++ layer; with LD_PRELOAD of the oracle stand-in it runs on the
// CPU.
//   range_main IN OUT delta overlap sample_size
// IN : int32 nP, int32 nQ, float32 P[nP][3], float32 Q[nQ][3]
// OUT: int32 threw_before (1: getNeighbors threw before any registration), float32 score, float32 C[16] (the centred
//      transform behind the score, column-major), int32 nSP, float32 sampled P[nSP][3], int32 nSQ, float32 sampled
//      Q[nSQ][3], int32 K, float32 max_distance[K], K x (int64 offsets[nSQ + 1], int32 indices[total],
//      float32 sq[total]) with total = offsets[nSQ]
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
  std::vector<int64_t> offsets;
  std::vector<int> indices;
  std::vector<float> sq;
  try {
    m.getNeighbors(&offsets, &indices, opt.delta, &sq);
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
  const std::vector<float> dists = {opt.delta, 3 * opt.delta};
  const int K = (int)dists.size();
  put(out, &K, 1);
  put(out, dists.data(), dists.size());
  for (float d : dists) {
    m.getNeighbors(&offsets, &indices, d, &sq);
    put(out, offsets.data(), offsets.size());
    put(out, indices.data(), indices.size());
    put(out, sq.data(), sq.size());
  }
  std::fclose(out);
  return 0;
}
