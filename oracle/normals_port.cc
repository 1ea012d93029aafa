// TEST INFRASTRUCTURE ONLY (oracle/normals.py builds it together with oracle/knn_port.cc; never linked into the product).
//
// Plain restatement of s4g_normals (include/s4g.h), operation for operation: the neighbourhood of P point j is the
// brute-force s4g_knn row of the query p_j (knn_bruteforce: no T, no exclusion); in double, summed from 0 in row order,
// c = sum p / m and C = sum (p - c)(p - c)^T / m; cyclic Jacobi on C with the pairs (0,1), (0,2), (1,2), a pair's entry
// zeroed when 100 |a_pq| is lost against |a_pp| and |a_qq|, at most 50 sweeps; the diagonal sorted stably; the normal the
// column of the smallest, normalised, its sign from the viewpoint (double) or from the largest component of the rounded
// normal (ties to the lowest axis); (0, 0, 0) when m < 3 or C == 0.  Compiled -ffp-contract=off: no FMA, as the device.
#include <cmath>
#include <cstdint>
#include <vector>

extern "C" void knn_bruteforce(const float* P, long nP, const float* X, long n, const float* T, int k, float sq_radius,
                               const int32_t* exclude, int32_t* out_index, float* out_sq);

namespace {

struct Sym3 {
  double a[3][3];   // symmetric: only a[p][q] with p <= q is read and written
  double& at(int p, int q) { return p <= q ? a[p][q] : a[q][p]; }
};

void Rotate(double& x, double& y, double s, double tau) {
  const double g = x, h = y;
  x = g - s * (h + g * tau);
  y = h + s * (g - h * tau);
}

// one Jacobi step on the pair (p, q), r the third index; V's columns p and q rotate with it
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

void Normal(const float* P, const int32_t* row, int k, const float* self, const float* viewpoint, float* normal, float* eig) {
  int m = 0;
  double sum[3] = {0.0, 0.0, 0.0};
  for (; m < k && row[m] >= 0; ++m)
    for (int c = 0; c < 3; ++c) sum[c] = sum[c] + (double)P[3 * (long)row[m] + c];
  const double dm = (double)m;
  double cen[3];
  for (int c = 0; c < 3; ++c) cen[c] = sum[c] / dm;
  Sym3 A = {};
  for (int e = 0; e < m; ++e) {
    double d[3];
    for (int c = 0; c < 3; ++c) d[c] = (double)P[3 * (long)row[e] + c] - cen[c];
    for (int p = 0; p < 3; ++p)
      for (int q = p; q < 3; ++q) A.a[p][q] = A.a[p][q] + d[p] * d[q];
  }
  bool zero = true;
  for (int p = 0; p < 3; ++p)
    for (int q = p; q < 3; ++q) {
      A.a[p][q] = A.a[p][q] / dm;
      zero = zero && A.a[p][q] == 0.0;
    }
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
  if (eig)
    for (int i = 0; i < 3; ++i) eig[i] = (float)A.a[o[i]][o[i]];
  normal[0] = normal[1] = normal[2] = 0.f;
  if (m < 3 || zero) return;
  double n[3] = {V[0][o[0]], V[1][o[0]], V[2][o[0]]};
  const double len = std::sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
  for (int c = 0; c < 3; ++c) n[c] = n[c] / len;
  if (viewpoint) {
    double dot = 0.0;
    for (int c = 0; c < 3; ++c) {
      const double term = ((double)viewpoint[c] - (double)self[c]) * n[c];
      dot = c == 0 ? term : dot + term;
    }
    if (dot < 0.0)
      for (int c = 0; c < 3; ++c) n[c] = -n[c];
  }
  for (int c = 0; c < 3; ++c) normal[c] = (float)n[c];
  if (!viewpoint) {
    int a = 0;
    for (int c = 1; c < 3; ++c)
      if (std::fabs(normal[c]) > std::fabs(normal[a])) a = c;
    if (normal[a] < 0.f)
      for (int c = 0; c < 3; ++c) normal[c] = -normal[c];
  }
}

}  // namespace

extern "C" {

// P: nP x 3; which: the n P points to answer (null: all, n = nP); viewpoint: 3 floats or null; out: n x 3 each (eig may
// be null); rows_out: n x k rows of knn_bruteforce, or null
void normals_port(const float* P, long nP, const int64_t* which, long n, int k, float sq_radius, const float* viewpoint,
                  float* normals, float* eig, int32_t* rows_out) {
  std::vector<float> X(3 * (size_t)n);
  for (long i = 0; i < n; ++i)
    for (int c = 0; c < 3; ++c) X[3 * i + c] = P[3 * (which ? which[i] : i) + c];
  std::vector<int32_t> rows((size_t)n * (size_t)k);
  knn_bruteforce(P, nP, X.data(), n, nullptr, k, sq_radius, nullptr, rows.data(), nullptr);
#ifdef _OPENMP
#pragma omp parallel for schedule(static)
#endif
  for (long i = 0; i < n; ++i)
    Normal(P, rows.data() + (size_t)i * (size_t)k, k, X.data() + 3 * i, viewpoint, normals + 3 * i, eig ? eig + 3 * i : nullptr);
  if (rows_out)
    for (size_t e = 0; e < rows.size(); ++e) rows_out[e] = rows[e];
}

}  // extern "C"
