// TEST INFRASTRUCTURE ONLY (oracle/outliers.py builds it together with oracle/knn_port.cc; never linked into the product).
//
// Plain restatement of the two outlier filters of include/s4g.h, operation for operation.
//   s4g_statistical_outliers: the row of P point j is the brute-force s4g_knn row of the query p_j (knn_bruteforce: no T,
//   exclude = j, unbounded); mean_dist[j] = (sum over the row's real entries in row order, from 0.0, of
//   sqrt((double) d^2)) / m, 0 when m = 0; mu = S1 / nP and sigma = sqrt(S2 / (nP - 1)) (0 when nP = 1), each S the sum
//   of runs of 1024 consecutive j summed left to right from 0.0, then of the run sums left to right from 0.0; j kept iff
//   mean_dist[j] <= mu + std_ratio * sigma.
//   s4g_radius_outliers: c_j = #{i != j : d^2(p_i, p_j) < sq_radius} over all of P, d^2 = dx^2 + (dy^2 + dz^2) of
//   p_j - p_i in fp32 (kdtree.h:417); counts[j] = min(c_j, min_neighbors); j kept iff c_j >= min_neighbors.
// Compiled -ffp-contract=off: no FMA, as the device.
#include <cmath>
#include <cstdint>
#include <limits>
#include <vector>

extern "C" void knn_bruteforce(const float* P, long nP, const float* X, long n, const float* T, int k, float sq_radius,
                               const int32_t* exclude, int32_t* out_index, float* out_sq);

extern "C" {

// mean_dist of the P points `which` (n of them; null: all, n = nP) -> out [n]
void outlier_mean_rows(const float* P, long nP, const int64_t* which, long n, int k, double* out) {
  std::vector<float> X(3 * (size_t)n);
  std::vector<int32_t> excl((size_t)n);
  for (long i = 0; i < n; ++i) {
    const long j = which ? (long)which[i] : i;
    excl[i] = (int32_t)j;
    for (int c = 0; c < 3; ++c) X[3 * i + c] = P[3 * j + c];
  }
  std::vector<int32_t> index((size_t)n * (size_t)k);
  std::vector<float> sq((size_t)n * (size_t)k);
  knn_bruteforce(P, nP, X.data(), n, nullptr, k, std::numeric_limits<float>::infinity(), excl.data(), index.data(),
                 sq.data());
  for (long i = 0; i < n; ++i) {
    double s = 0.0;
    int m = 0;
    for (; m < k && index[(size_t)i * k + m] >= 0; ++m) s = s + std::sqrt((double)sq[(size_t)i * k + m]);
    out[i] = m > 0 ? s / (double)m : 0.0;
  }
}

// out2 = {mu, sigma} of mean_dist [n], in the fixed order of the contract
void outlier_moments(const double* mean_dist, long n, double* out2) {
  const long kRun = 1024;
  double S[2] = {0.0, 0.0};
  for (int pass = 0; pass < 2; ++pass) {
    const double mu = pass == 0 ? 0.0 : S[0] / (double)n;
    double total = 0.0;
    for (long b = 0; b < n; b += kRun) {
      double run = 0.0;
      for (long j = b; j < n && j < b + kRun; ++j) {
        double x = mean_dist[j];
        if (pass == 1) {
          x = x - mu;
          x = x * x;
        }
        run = run + x;
      }
      total = total + run;
    }
    S[pass] = total;
  }
  out2[0] = S[0] / (double)n;
  out2[1] = n > 1 ? std::sqrt(S[1] / (double)(n - 1)) : 0.0;
}

// keep flags [n] of mean_dist against mu + std_ratio * sigma
void outlier_flags(const double* mean_dist, long n, const double* out2, double std_ratio, uint8_t* flags) {
  const double threshold = out2[0] + std_ratio * out2[1];
  for (long j = 0; j < n; ++j) flags[j] = mean_dist[j] <= threshold ? 1 : 0;
}

// the whole statistical filter: flags [nP], mean_dist [nP], out2 [2]
void statistical_port(const float* P, long nP, int k, double std_ratio, uint8_t* flags, double* mean_dist, double* out2) {
  outlier_mean_rows(P, nP, nullptr, nP, k, mean_dist);
  outlier_moments(mean_dist, nP, out2);
  outlier_flags(mean_dist, nP, out2, std_ratio, flags);
}

// the radius filter: raw [nP] = c_j (uncapped, may be null), counts [nP] = min(c_j, min_neighbors), flags [nP]
void radius_port(const float* P, long nP, float sq_radius, int min_neighbors, int64_t* raw, int32_t* counts,
                 uint8_t* flags) {
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 64)
#endif
  for (long j = 0; j < nP; ++j) {
    const float x = P[3 * j], y = P[3 * j + 1], z = P[3 * j + 2];
    int64_t c = 0;
    for (long i = 0; i < nP; ++i) {
      if (i == j) continue;
      const float dx = x - P[3 * i], dy = y - P[3 * i + 1], dz = z - P[3 * i + 2];
      const float d2 = dx * dx + (dy * dy + dz * dz);
      if (d2 < sq_radius) ++c;
    }
    if (raw) raw[j] = c;
    counts[j] = c < (int64_t)min_neighbors ? (int32_t)c : min_neighbors;
    flags[j] = c >= (int64_t)min_neighbors ? 1 : 0;
  }
}

}  // extern "C"
