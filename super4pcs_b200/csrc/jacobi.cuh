// The symmetric 3x3 eigen-solver of the PCA fits (k_normals in normals.cu, the plane refit in planes.cu): cyclic Jacobi
// rotations in the classic threshold form, then a stable ascending sort of the diagonal.  Every value is made of IEEE
// basic operations in double (the library is compiled with -fmad=false), so a CPU restatement compiled without
// contraction gives the same bits.
#pragma once

constexpr int kJacobiSweeps = 50;

// one Givens rotation (x, y) <- (x - s (y + x tau), y + s (x - y tau))
__device__ __forceinline__ void rotate(double& x, double& y, double s, double tau) {
  const double g = x, h = y;
  x = g - s * (h + g * tau);
  y = h + s * (g - h * tau);
}

// the Jacobi step of the pair (p, q) of a symmetric 3x3: app, aqq, apq its entries, arp / arq those of the third row r;
// vp / vq the columns p and q of V.  A negligible apq (100 |apq| lost against both |app| and |aqq|) is set to zero.
__device__ __forceinline__ void jacobi_pair(double& app, double& aqq, double& apq, double& arp, double& arq, double (&vp)[3],
                                            double (&vq)[3]) {
  if (apq == 0.0) return;
  const double g = 100.0 * fabs(apq);
  if (fabs(app) + g == fabs(app) && fabs(aqq) + g == fabs(aqq)) {
    apq = 0.0;
    return;
  }
  const double h = aqq - app;
  double t;
  if (fabs(h) + g == fabs(h)) {
    t = apq / h;
  } else {
    const double theta = (0.5 * h) / apq;
    t = 1.0 / (fabs(theta) + sqrt(theta * theta + 1.0));
    if (theta < 0.0) t = -t;
  }
  const double c = 1.0 / sqrt(t * t + 1.0), s = t * c, tau = s / (1.0 + c), d = t * apq;
  app = app - d;
  aqq = aqq + d;
  apq = 0.0;
  rotate(arp, arq, s, tau);
#pragma unroll
  for (int r = 0; r < 3; ++r) rotate(vp[r], vq[r], s, tau);
}

__device__ __forceinline__ double pick3(double a, double b, double c, int i) { return i == 0 ? a : i == 1 ? b : c; }

// C = [[a00 a01 a02] [. a11 a12] [. . a22]] -> its eigenvalues on the diagonal and the eigenvectors in the columns v0, v1,
// v2 (which start as the identity): the pairs (0,1), (0,2), (1,2) per sweep until the off-diagonal entries are exactly
// zero or kJacobiSweeps sweeps have run
__device__ __forceinline__ void jacobi_sweeps(double& a00, double& a01, double& a02, double& a11, double& a12, double& a22,
                                              double (&v0)[3], double (&v1)[3], double (&v2)[3]) {
#pragma unroll 1
  for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
    if (a01 == 0.0 && a02 == 0.0 && a12 == 0.0) break;
    jacobi_pair(a00, a11, a01, a02, a12, v0, v1);
    jacobi_pair(a00, a22, a02, a01, a12, v0, v2);
    jacobi_pair(a11, a22, a12, a01, a02, v1, v2);
  }
}

// the stable ascending order of the diagonal: o0 <= o1 <= o2 (int variables the statement declares), equal values in
// column order; the normal of the fit is the column o0 (the smallest eigenvalue).  A statement macro rather than a
// function: the same statements written through an inlined function compiled k_normals into different (if equivalent)
// instructions.
#define S4G_EIGEN_ORDER(a00, a11, a22, o0, o1, o2)                                                  \
  int o0 = 0, o1 = 1, o2 = 2;                                                                       \
  if (pick3(a00, a11, a22, o1) < pick3(a00, a11, a22, o0)) { const int s = o0; o0 = o1; o1 = s; }   \
  if (pick3(a00, a11, a22, o2) < pick3(a00, a11, a22, o1)) {                                        \
    const int s = o1; o1 = o2; o2 = s;                                                              \
    if (pick3(a00, a11, a22, o1) < pick3(a00, a11, a22, o0)) { const int s2 = o0; o0 = o1; o1 = s2; } \
  }
