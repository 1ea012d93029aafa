// TEST INFRASTRUCTURE ONLY (oracle/planes.py builds it; never linked into the product).
//
// Plain restatement of s4g_segment_planes (include/s4g.h), operation for operation: per round the ascending active list
// A_r, the SplitMix64 draws, the hypothesis planes in double rounded to float, every hypothesis tested on every active
// point in fp32 (((a x + b y) + c z) + d, |r| < threshold), the winner by (count, -h), the refit's two passes over the
// inliers in runs of 1024 (each run from 0.0 left to right, then the run sums), the cyclic Jacobi of s4g_normals with its
// stable sort and column rule, the sign rule, the final test, accept or stop.  Compiled -ffp-contract=off: no FMA, as the
// device.  OpenMP over the hypotheses; the counts are integers, so the threads change nothing.
#include <cmath>
#include <cstdint>
#include <vector>

namespace {

struct Plane {   // s4g_plane
  float coefficients[4];
  float hypothesis[4];
  int32_t hypothesis_index;
  int32_t sample[3];
  int64_t hypothesis_inliers;
  int64_t n_inliers;
};
static_assert(sizeof(Plane) == 64, "s4g_plane is 64 bytes");

const long kRun = 1024;

uint64_t SplitMix64(uint64_t s, uint64_t k) {
  uint64_t z = s + k * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

bool Inlier(const float* pl, const float* p, float threshold) {
  const float ax = pl[0] * p[0], by = pl[1] * p[1], cz = pl[2] * p[2];
  const float r = ((ax + by) + cz) + pl[3];
  return std::fabs(r) < threshold;
}

// n / len, the component of largest magnitude made positive (ties to the lowest axis), d = -n.p, rounded
void RoundPlane(double n[3], double len, const double p[3], float* out) {
  for (int c = 0; c < 3; ++c) n[c] = n[c] / len;
  int a = 0;
  for (int c = 1; c < 3; ++c)
    if (std::fabs(n[c]) > std::fabs(n[a])) a = c;
  if (n[a] < 0.0)
    for (int c = 0; c < 3; ++c) n[c] = -n[c];
  const double d = -((n[0] * p[0] + n[1] * p[1]) + n[2] * p[2]);
  for (int c = 0; c < 3; ++c) out[c] = (float)n[c];
  out[3] = (float)d;
}

// hypothesis h of a round: its three positions j and its plane; false when invalid
bool Hypothesis(const float* P, const int32_t* act, long m, uint64_t seed_r, long h, int32_t* sample, float* plane) {
  double p[3][3];
  for (int t = 0; t < 3; ++t) {
    const uint64_t z = SplitMix64(seed_r, 3ull * (uint64_t)h + (uint64_t)t + 1ull);
    const long pos = (long)(((z >> 32) * (uint64_t)m) >> 32);
    sample[t] = act[pos];
    for (int c = 0; c < 3; ++c) p[t][c] = (double)P[3 * (long)act[pos] + c];
  }
  const double ux = p[1][0] - p[0][0], uy = p[1][1] - p[0][1], uz = p[1][2] - p[0][2];
  const double vx = p[2][0] - p[0][0], vy = p[2][1] - p[0][1], vz = p[2][2] - p[0][2];
  double n[3] = {uy * vz - uz * vy, uz * vx - ux * vz, ux * vy - uy * vx};
  const double len = std::sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]);
  if (len == 0.0) {
    for (int c = 0; c < 4; ++c) plane[c] = NAN;
    return false;
  }
  RoundPlane(n, len, p[0], plane);
  return true;
}

void Rotate(double& x, double& y, double s, double tau) {
  const double g = x, h = y;
  x = g - s * (h + g * tau);
  y = h + s * (g - h * tau);
}

struct Sym3 {
  double a[3][3];
  double& at(int p, int q) { return p <= q ? a[p][q] : a[q][p]; }
};

void JacobiPair(Sym3& A, double V[3][3], int p, int q) {
  const int r = 3 - p - q;
  double& apq = A.at(p, q);
  if (apq == 0.0) return;
  double& app = A.at(p, p);
  double& aqq = A.at(q, q);
  const double g = 100.0 * std::fabs(apq);
  if (std::fabs(app) + g == std::fabs(app) && std::fabs(aqq) + g == std::fabs(aqq)) {
    apq = 0.0;
    return;
  }
  const double h = aqq - app;
  double t;
  if (std::fabs(h) + g == std::fabs(h)) {
    t = apq / h;
  } else {
    const double theta = (0.5 * h) / apq;
    t = 1.0 / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
    if (theta < 0.0) t = -t;
  }
  const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c, tau = s / (1.0 + c), d = t * apq;
  app = app - d;
  aqq = aqq + d;
  apq = 0.0;
  Rotate(A.at(r, p), A.at(r, q), s, tau);
  for (int i = 0; i < 3; ++i) Rotate(V[i][p], V[i][q], s, tau);
}

// the refit of the inliers I (positions j, ascending); false when |I| < 3 or C is exactly zero
bool Refit(const float* P, const std::vector<int32_t>& I, float* out) {
  const long n = (long)I.size();
  if (n < 3) return false;
  double cen[3], tot[3] = {0.0, 0.0, 0.0};
  for (long b = 0; b < n; b += kRun) {
    double run[3] = {0.0, 0.0, 0.0};
    for (long i = b; i < n && i < b + kRun; ++i)
      for (int c = 0; c < 3; ++c) run[c] = run[c] + (double)P[3 * (long)I[i] + c];
    for (int c = 0; c < 3; ++c) tot[c] = tot[c] + run[c];
  }
  for (int c = 0; c < 3; ++c) cen[c] = tot[c] / (double)n;
  const int pp[6] = {0, 0, 0, 1, 1, 2}, qq[6] = {0, 1, 2, 1, 2, 2};
  double mom[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (long b = 0; b < n; b += kRun) {
    double run[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (long i = b; i < n && i < b + kRun; ++i)
      for (int t = 0; t < 6; ++t) {
        const double dp = (double)P[3 * (long)I[i] + pp[t]] - cen[pp[t]], dq = (double)P[3 * (long)I[i] + qq[t]] - cen[qq[t]];
        run[t] = run[t] + dp * dq;
      }
    for (int t = 0; t < 6; ++t) mom[t] = mom[t] + run[t];
  }
  Sym3 A = {};
  bool zero = true;
  for (int t = 0; t < 6; ++t) {
    A.a[pp[t]][qq[t]] = mom[t] / (double)n;
    zero = zero && A.a[pp[t]][qq[t]] == 0.0;
  }
  if (zero) return false;
  double V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int sweep = 0; sweep < 50; ++sweep) {
    if (A.a[0][1] == 0.0 && A.a[0][2] == 0.0 && A.a[1][2] == 0.0) break;
    JacobiPair(A, V, 0, 1);
    JacobiPair(A, V, 0, 2);
    JacobiPair(A, V, 1, 2);
  }
  int o[3] = {0, 1, 2};   // insertion sort, strict <: equal eigenvalues keep the column order
  for (int i = 1; i < 3; ++i)
    for (int x = i; x > 0 && A.a[o[x]][o[x]] < A.a[o[x - 1]][o[x - 1]]; --x) {
      const int s = o[x];
      o[x] = o[x - 1];
      o[x - 1] = s;
    }
  double nv[3] = {V[0][o[0]], V[1][o[0]], V[2][o[0]]};
  const double len = std::sqrt((nv[0] * nv[0] + nv[1] * nv[1]) + nv[2] * nv[2]);
  RoundPlane(nv, len, cen, out);
  return true;
}

}  // namespace

extern "C" {

// the draws and planes of round seed_r over the active positions act [m]: sample [H x 3], plane [H x 4] (NaN when
// invalid), valid [H]
void planes_hypotheses(const float* P, const int32_t* act, long m, long H, uint64_t seed_r, int32_t* sample, float* plane,
                       uint8_t* valid) {
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
  for (long h = 0; h < H; ++h) valid[h] = Hypothesis(P, act, m, seed_r, h, sample + 3 * h, plane + 4 * h) ? 1 : 0;
}

// counts [H] of the planes [H x 4] over the active positions act [m]
void planes_counts(const float* P, const int32_t* act, long m, long H, const float* plane, float threshold,
                   uint32_t* counts) {
  std::vector<float> X(3 * (size_t)m);
  for (long i = 0; i < m; ++i)
    for (int c = 0; c < 3; ++c) X[3 * i + c] = P[3 * (long)act[i] + c];
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 4)
#endif
  for (long h = 0; h < H; ++h) {
    uint32_t cnt = 0;
    const float* pl = plane + 4 * h;
    for (long i = 0; i < m; ++i) cnt += Inlier(pl, &X[3 * i], threshold) ? 1u : 0u;
    counts[h] = cnt;
  }
}

// the whole contract: labels [n], planes [max_planes], *n_planes, offsets [max_planes + 1], members [n], hyp_counts
// [max_planes x H] (may be null)
void planes_port(const float* P, long n, float threshold, int H, uint64_t seed, int refine, int max_planes,
                 int64_t min_inliers, int32_t* labels, void* planes_out, int* n_planes, int64_t* offsets, int32_t* members,
                 uint32_t* hyp_counts) {
  Plane* planes = static_cast<Plane*>(planes_out);
  for (long j = 0; j < n; ++j) labels[j] = -1;
  if (hyp_counts)
    for (long e = 0; e < (long)max_planes * H; ++e) hyp_counts[e] = 0u;
  *n_planes = 0;
  offsets[0] = 0;
  std::vector<int32_t> sample(3 * (size_t)H);
  std::vector<float> plane(4 * (size_t)H);
  std::vector<uint8_t> valid((size_t)H);
  std::vector<uint32_t> counts((size_t)H);
  for (int r = 0; r < max_planes; ++r) {
    std::vector<int32_t> act;
    for (long j = 0; j < n; ++j)
      if (labels[j] < 0) act.push_back((int32_t)j);
    const long m = (long)act.size();
    if (m < 3) break;
    const uint64_t seed_r = seed + (uint64_t)r;
    planes_hypotheses(P, act.data(), m, H, seed_r, sample.data(), plane.data(), valid.data());
    planes_counts(P, act.data(), m, H, plane.data(), threshold, counts.data());
    if (hyp_counts)
      for (long h = 0; h < H; ++h) hyp_counts[(long)r * H + h] = counts[h];
    long best = -1;
    for (long h = 0; h < H; ++h)
      if (valid[h] && (best < 0 || counts[h] > counts[best])) best = h;
    if (best < 0) break;
    const float* hp = &plane[4 * best];
    float fin[4] = {hp[0], hp[1], hp[2], hp[3]};
    if (refine) {
      std::vector<int32_t> I;
      for (long i = 0; i < m; ++i)
        if (Inlier(hp, P + 3 * (long)act[i], threshold)) I.push_back(act[i]);
      Refit(P, I, fin);
    }
    std::vector<int32_t> fin_in;
    for (long i = 0; i < m; ++i)
      if (Inlier(fin, P + 3 * (long)act[i], threshold)) fin_in.push_back(act[i]);
    if ((int64_t)fin_in.size() < min_inliers) break;
    Plane& rec = planes[r];
    for (int c = 0; c < 4; ++c) {
      rec.coefficients[c] = fin[c];
      rec.hypothesis[c] = hp[c];
    }
    rec.hypothesis_index = (int32_t)best;
    for (int t = 0; t < 3; ++t) rec.sample[t] = sample[3 * best + t];
    rec.hypothesis_inliers = counts[best];
    rec.n_inliers = (int64_t)fin_in.size();
    for (size_t e = 0; e < fin_in.size(); ++e) {
      labels[fin_in[e]] = r;
      members[offsets[r] + (int64_t)e] = fin_in[e];
    }
    offsets[r + 1] = offsets[r] + (int64_t)fin_in.size();
    *n_planes = r + 1;
  }
}

}  // extern "C"
