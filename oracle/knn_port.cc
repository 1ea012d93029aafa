// TEST INFRASTRUCTURE ONLY (oracle/knn.py builds it; never linked into the product).
//
// Brute-force restatement of s4g_knn (include/s4g.h): for every query x_i, the k smallest (d^2, index) over ALL P points
// (no accelerator) with d^2 <= sq_radius and index != exclude[i], in ascending (d^2, index); the row is padded at its end
// with -1 / +inf.  y = T x in the reference's operation order (match4pcsBase.cc:532) or x when T is null;
// d^2 = dx^2 + (dy^2 + dz^2) (kdtree.h:417); fp32, no contraction (-ffp-contract=off).
#include <cstddef>
#include <cstdint>
#include <limits>
#include <vector>

extern "C" {

// P: nP x 3, X: n x 3, T16: column-major 4x4 or null, exclude: n entries or null; out_index: n x k, out_sq: n x k or null
void knn_bruteforce(const float* P, long nP, const float* X, long n, const float* T, int k, float sq_radius,
                    const int32_t* exclude, int32_t* out_index, float* out_sq) {
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 16)
#endif
  for (long i = 0; i < n; ++i) {
    const float x = X[3 * i], y = X[3 * i + 1], z = X[3 * i + 2];
    float tx = x, ty = y, tz = z;
    if (T) {
      tx = ((T[0] * x + T[4] * y) + T[8] * z) + T[12];
      ty = ((T[1] * x + T[5] * y) + T[9] * z) + T[13];
      tz = ((T[2] * x + T[6] * y) + T[10] * z) + T[14];
    }
    const long excl = exclude ? (long)exclude[i] : -1;
    std::vector<float> bd;                                 // the row so far, ascending (d^2, j)
    std::vector<int32_t> bj;
    for (long j = 0; j < nP; ++j) {                        // ascending j: a later j goes after an equal d^2
      if (j == excl) continue;
      const float dx = tx - P[3 * j], dy = ty - P[3 * j + 1], dz = tz - P[3 * j + 2];
      const float d2 = dx * dx + (dy * dy + dz * dz);
      if (!(d2 <= sq_radius)) continue;                    // beyond the radius, or NaN
      if ((long)bd.size() == k && !(d2 < bd.back())) continue;
      std::size_t at = bd.size();
      while (at > 0 && bd[at - 1] > d2) --at;
      bd.insert(bd.begin() + at, d2);
      bj.insert(bj.begin() + at, (int32_t)j);
      if ((long)bd.size() > k) {
        bd.pop_back();
        bj.pop_back();
      }
    }
    for (int e = 0; e < k; ++e) {
      const bool held = e < (int)bd.size();
      out_index[i * k + e] = held ? bj[e] : -1;
      if (out_sq) out_sq[i * k + e] = held ? bd[e] : std::numeric_limits<float>::infinity();
    }
  }
}

}  // extern "C"
