// TEST INFRASTRUCTURE ONLY (oracle/fpfh.py builds it together with oracle/knn_port.cc; never linked into the product).
//
// Plain restatement of s4g_fpfh and s4g_fpfh_match (include/s4g.h): the brute-force s4g_knn row of every p_j with
// exclude = j and its d^2 (knn_bruteforce), or rows given by the caller; Open3D's pair feature in double with the exact
// swap and f1 face tests; the SPFH counts; the FPFH sums in row order and the per-block S_h; and the nearest descriptor
// by a plain double loop over every pair in ascending j.  Compiled with -ffp-contract=off: no FMA.  Shares no code with
// the device.
#include <cmath>
#include <cstdint>
#include <limits>
#include <vector>

extern "C" void knn_bruteforce(const float* P, long nP, const float* X, long n, const float* T, int k, float sq_radius,
                               const int32_t* exclude, int32_t* out_index, float* out_sq);

namespace {

const double kC[11] = {0.0, -0x1.aeb8c8764f0bap-1, -0x1.a9628d9c712b6p-2, 0x1.2375f640f44dbp-3, 0x1.4f49e7f775887p-1,
                       0x1.eb42a9bcd5057p-1, 0x1.eb42a9bcd5057p-1, 0x1.4f49e7f775887p-1, 0x1.2375f640f44dbp-3,
                       -0x1.a9628d9c712b6p-2, -0x1.aeb8c8764f0bap-1};
const double kS[11] = {0.0, -0x1.14cedf8bb580bp-1, -0x1.d1bb48eee2c13p-1, -0x1.fac9e043842efp-1, -0x1.82f19bb3a28a1p-1,
                       -0x1.207e7fd768dbfp-2, 0x1.207e7fd768dbfp-2, 0x1.82f19bb3a28a1p-1, 0x1.fac9e043842efp-1,
                       0x1.d1bb48eee2c13p-1, 0x1.14cedf8bb580bp-1};

struct V {
  double x, y, z;
};
double dot(const V& a, const V& b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
V cross(const V& a, const V& b) { return V{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }

bool normal_of(const float* N, long j, V& n) {
  const float x = N[3 * j], y = N[3 * j + 1], z = N[3 * j + 2];
  if (!std::isfinite(x) || !std::isfinite(y) || !std::isfinite(z)) return false;
  if (x == 0.f && y == 0.f && z == 0.f) return false;
  n = V{x, y, z};
  const double l = std::sqrt(dot(n, n));
  n = V{n.x / l, n.y / l, n.z / l};
  return true;
}

int bin_of(double f) {
  const double h = std::floor(11 * (f + 1.0) * 0.5);
  if (h < 0.0) return 0;
  if (h > 10.0) return 10;
  return (int)h;
}

int f1_bin(double x, double y) {
  if (y == 0.0) return x < 0.0 ? 10 : 5;
  int lo = y > 0.0 ? 6 : 1, b = y > 0.0 ? 5 : 0;
  for (int i = lo; i < lo + 5; ++i)
    if (kC[i] * y - kS[i] * x >= 0.0) ++b;
  return b;
}

void pair_feature_bins(const V& p1, const V& n1, const V& p2, const V& n2, int bins[3]) {
  bins[0] = 5;
  bins[1] = 16;
  bins[2] = 27;
  V dp{p2.x - p1.x, p2.y - p1.y, p2.z - p1.z};
  const double d = std::sqrt(dot(dp, dp));
  if (d == 0.0) return;
  const double a1 = dot(n1, dp) / d;
  const double a2 = dot(n2, dp) / d;
  V u = n1, m = n2;
  double f3 = a1;
  if (std::fabs(a1) < std::fabs(a2)) {
    u = n2;
    m = n1;
    dp = V{-dp.x, -dp.y, -dp.z};
    f3 = -a2;
  }
  V v = cross(dp, u);
  const double vn = std::sqrt(dot(v, v));
  if (vn == 0.0) return;
  v = V{v.x / vn, v.y / vn, v.z / vn};
  const V w = cross(u, v);
  bins[0] = f1_bin(dot(u, m), dot(w, m));
  bins[1] = 11 + bin_of(dot(v, m));
  bins[2] = 22 + bin_of(f3);
}

}  // namespace

extern "C" {

// 0 on success; 2 (S4G_ERR_ARG) for bad arguments.  rows_in / sq_in: n x k (index, -1 padding at the end; d^2) or null
// for the brute force.  fpfh: n x 33.  spfh_out (n x 33 doubles) may be null.
int fpfh_port(const float* P, long n, const float* normals, int k, float sq_radius, const int32_t* rows_in,
              const float* sq_in, float* fpfh, double* spfh_out) {
  if (k < 1 || k > 64 || std::isnan(sq_radius) || sq_radius < 0.f || !normals || !fpfh || n < 1) return 2;
  std::vector<int32_t> rows;
  std::vector<float> sq;
  if (!rows_in) {
    rows.resize((size_t)n * k);
    sq.resize((size_t)n * k);
    std::vector<int32_t> excl(n);
    for (long j = 0; j < n; ++j) excl[j] = (int32_t)j;
    knn_bruteforce(P, n, P, n, nullptr, k, sq_radius, excl.data(), rows.data(), sq.data());
    rows_in = rows.data();
    sq_in = sq.data();
  }
  std::vector<double> spfh((size_t)n * 33, 0.0);
  std::vector<char> has(n, 0);
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 256)
#endif
  for (long j = 0; j < n; ++j) {
    V nj;
    if (!normal_of(normals, j, nj)) continue;
    has[j] = 1;
    const V pj{P[3 * j], P[3 * j + 1], P[3 * j + 2]};
    int cnt[33] = {0};
    int m = 0;
    for (int e = 0; e < k; ++e) {
      const long i = rows_in[j * k + e];
      if (i < 0) break;
      V ni;
      if (!normal_of(normals, i, ni)) continue;
      const V pi{P[3 * i], P[3 * i + 1], P[3 * i + 2]};
      int bins[3];
      pair_feature_bins(pj, nj, pi, ni, bins);
      for (int c = 0; c < 3; ++c) ++cnt[bins[c]];
      ++m;
    }
    if (m > 0)
      for (int b = 0; b < 33; ++b) spfh[j * 33 + b] = (100.0 * cnt[b]) / m;
  }
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 256)
#endif
  for (long j = 0; j < n; ++j) {
    if (!has[j]) {
      for (int b = 0; b < 33; ++b) fpfh[j * 33 + b] = 0.f;
      continue;
    }
    double acc[33];
    for (int b = 0; b < 33; ++b) acc[b] = 0.0;
    for (int e = 0; e < k; ++e) {
      const long i = rows_in[j * k + e];
      if (i < 0) break;
      const double d2 = sq_in[j * k + e];
      if (!has[i] || !(d2 > 0.0)) continue;
      for (int b = 0; b < 33; ++b) acc[b] = acc[b] + spfh[i * 33 + b] / d2;
    }
    for (int h = 0; h < 3; ++h) {
      double S = 0.0;
      for (int b = 11 * h; b < 11 * h + 11; ++b) S = S + acc[b];
      for (int b = 11 * h; b < 11 * h + 11; ++b)
        fpfh[j * 33 + b] = S != 0.0 ? (float)(acc[b] * (100.0 / S) + spfh[j * 33 + b]) : (float)spfh[j * 33 + b];
    }
  }
  if (spfh_out)
    for (size_t i = 0; i < spfh.size(); ++i) spfh_out[i] = spfh[i];
  return 0;
}

// the nearest b-row of every a-row (s4g_fpfh_match): index [n_a], sq_dist [n_a] (or null)
void fpfh_match_port(const float* a, long na, const float* b, long nb, int mutual, int32_t* index, float* sq_dist) {
  auto nearest = [](const float* X, long nx, const float* Y, long ny, std::vector<int32_t>& idx, std::vector<float>& d) {
    idx.assign(nx, -1);
    d.assign(nx, std::numeric_limits<float>::infinity());
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 64)
#endif
    for (long i = 0; i < nx; ++i)
      for (long j = 0; j < ny; ++j) {
        float s = 0.0f;
        for (int c = 0; c < 33; ++c) {
          const float t = X[i * 33 + c] - Y[j * 33 + c];
          s = s + t * t;
        }
        if (s < d[i]) {
          d[i] = s;
          idx[i] = (int32_t)j;
        }
      }
  };
  std::vector<int32_t> ab, ba;
  std::vector<float> dab, dba;
  nearest(a, na, b, nb, ab, dab);
  if (mutual) nearest(b, nb, a, na, ba, dba);
  for (long i = 0; i < na; ++i) {
    int32_t j = ab[i];
    if (mutual && j >= 0 && ba[j] != i) j = -1;
    index[i] = j;
    if (sq_dist) sq_dist[i] = dab[i];
  }
}

}  // extern "C"
