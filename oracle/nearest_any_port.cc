// TEST INFRASTRUCTURE ONLY (oracle/nearest_any.py builds it; never linked into the product).
//
// Brute-force restatement of s4g_nearest (include/s4g.h): for every query x_i, the P point with the smallest
// d^2 <= sq_radius and index != exclude[i] over ALL P points (no accelerator), equal d^2 -> the smallest index; -1 / +inf
// when there is none.  y = T x in the reference's operation order (match4pcsBase.cc:532) or x when T is null;
// d^2 = dx^2 + (dy^2 + dz^2) (kdtree.h:417); fp32, no contraction (-ffp-contract=off).
#include <cstdint>
#include <limits>

extern "C" {

// P: nP x 3, X: n x 3, T16: column-major 4x4 or null, exclude: n entries or null; out_index: n, out_sq: n or null
void nearest_any_bruteforce(const float* P, long nP, const float* X, long n, const float* T, float sq_radius,
                            const int32_t* exclude, int32_t* out_index, float* out_sq) {
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 64)
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
    float best = sq_radius;
    int32_t bj = -1;
    for (long j = 0; j < nP; ++j) {                       // ascending j: the first of equal d^2 is kept
      if (j == excl) continue;
      const float dx = tx - P[3 * j], dy = ty - P[3 * j + 1], dz = tz - P[3 * j + 2];
      const float d2 = dx * dx + (dy * dy + dz * dz);
      if (d2 < best || (d2 == best && bj < 0)) { best = d2; bj = (int32_t)j; }
    }
    out_index[i] = bj;
    if (out_sq) out_sq[i] = bj >= 0 ? best : std::numeric_limits<float>::infinity();
  }
}

}  // extern "C"
