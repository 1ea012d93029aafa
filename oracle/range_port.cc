// TEST INFRASTRUCTURE ONLY (oracle/range.py builds it; never linked into the product).
//
// Brute-force restatement of s4g_range (include/s4g.h): for every query x_i, every P index j with d^2 < sq_radius
// (strict) over ALL P points (no accelerator), in ascending j.  y = T x in the reference's operation order
// (match4pcsBase.cc:532) or x when T is null; d^2 = dx^2 + (dy^2 + dz^2) (kdtree.h:485 via squaredNorm); fp32, no
// contraction (-ffp-contract=off).  Two calls, as the CSR output needs: the lengths and their prefix, then the lists.
#include <cstdint>

namespace {

inline void transform(const float* X, long i, const float* T, float& tx, float& ty, float& tz) {
  const float x = X[3 * i], y = X[3 * i + 1], z = X[3 * i + 2];
  tx = x, ty = y, tz = z;
  if (T) {
    tx = ((T[0] * x + T[4] * y) + T[8] * z) + T[12];
    ty = ((T[1] * x + T[5] * y) + T[9] * z) + T[13];
    tz = ((T[2] * x + T[6] * y) + T[10] * z) + T[14];
  }
}

inline float sq(const float* P, long j, float tx, float ty, float tz) {
  const float dx = tx - P[3 * j], dy = ty - P[3 * j + 1], dz = tz - P[3 * j + 2];
  return dx * dx + (dy * dy + dz * dz);
}

}  // namespace

extern "C" {

// P: nP x 3, X: n x 3, T16: column-major 4x4 or null; offsets: n + 1 entries, written as the CSR offsets of the lists
void range_bruteforce_count(const float* P, long nP, const float* X, long n, const float* T, float sq_radius,
                            int64_t* offsets) {
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 16)
#endif
  for (long i = 0; i < n; ++i) {
    float tx, ty, tz;
    transform(X, i, T, tx, ty, tz);
    int64_t c = 0;
    for (long j = 0; j < nP; ++j) c += sq(P, j, tx, ty, tz) < sq_radius;
    offsets[i + 1] = c;
  }
  offsets[0] = 0;
  for (long i = 0; i < n; ++i) offsets[i + 1] += offsets[i];
}

// the lists themselves, at the offsets range_bruteforce_count wrote; out_sq may be null
void range_bruteforce_fill(const float* P, long nP, const float* X, long n, const float* T, float sq_radius,
                           const int64_t* offsets, int32_t* out_index, float* out_sq) {
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 16)
#endif
  for (long i = 0; i < n; ++i) {
    float tx, ty, tz;
    transform(X, i, T, tx, ty, tz);
    int64_t at = offsets[i];
    for (long j = 0; j < nP; ++j) {                       // ascending j
      const float d2 = sq(P, j, tx, ty, tz);
      if (d2 < sq_radius) {
        out_index[at] = (int32_t)j;
        if (out_sq) out_sq[at] = d2;
        ++at;
      }
    }
  }
}

}  // extern "C"
