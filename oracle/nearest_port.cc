// TEST INFRASTRUCTURE ONLY (oracle/nearest.py builds it; never linked into the product).
//
// Brute-force restatement of s4g_verify_nearest (include/s4g.h): for every query q_i and transform T_k, the P point with
// the smallest d^2 <= delta^2 over ALL P points (no accelerator), equal d^2 -> the smallest index; -1 / +inf when there
// is none.  Arithmetic of the reference's Verify (match4pcsBase.cc:531-536) and kd-tree leaf test (kdtree.h:417-418):
//   T q = ((m0 x + m1 y) + m2 z) + m3 per row,  d^2 = dx^2 + (dy^2 + dz^2),  fp32, no contraction (-ffp-contract=off).
#include <cstdint>
#include <cstddef>
#include <limits>

extern "C" {

// P: nP x 3, Q: nQ x 3 (the centred sampled clouds), T16k: K column-major 4x4.  out_index, out_sq: K x nQ (out_sq may be
// null); out_counts (nullable): K = the number of entries >= 0 per transform.
void nearest_bruteforce(const float* P, long nP, const float* Q, long nQ, float delta, const float* T16k, long K,
                        int32_t* out_index, float* out_sq, uint32_t* out_counts) {
  const float sq_eps = delta * delta;                     // match4pcsBase.cc:522
  for (long c = 0; c < K; ++c) {
    const float* T = T16k + 16 * c;
    uint32_t good = 0;
#ifdef _OPENMP
#pragma omp parallel for schedule(static) reduction(+ : good)
#endif
    for (long i = 0; i < nQ; ++i) {
      const float x = Q[3 * i], y = Q[3 * i + 1], z = Q[3 * i + 2];
      const float tx = ((T[0] * x + T[4] * y) + T[8] * z) + T[12];
      const float ty = ((T[1] * x + T[5] * y) + T[9] * z) + T[13];
      const float tz = ((T[2] * x + T[6] * y) + T[10] * z) + T[14];
      float best = sq_eps;
      int32_t bj = -1;
      for (long j = 0; j < nP; ++j) {                     // ascending j: the first of equal d^2 is kept
        const float dx = tx - P[3 * j], dy = ty - P[3 * j + 1], dz = tz - P[3 * j + 2];
        const float d2 = dx * dx + (dy * dy + dz * dz);
        if (d2 < best || (d2 == best && bj < 0)) { best = d2; bj = (int32_t)j; }
      }
      out_index[c * nQ + i] = bj;
      if (out_sq) out_sq[c * nQ + i] = bj >= 0 ? best : std::numeric_limits<float>::infinity();
      good += bj >= 0 ? 1u : 0u;
    }
    if (out_counts) out_counts[c] = good;
  }
}

}  // extern "C"
