// Point normals of the resident P from k-nearest neighbourhoods (s4g_normals, include/s4g.h).
//
// Rows.  The neighbourhood of P point j is exactly the s4g_knn row of the query p_j: no transform, no exclusion, the
// caller's k and sq_radius.  It holds p_j itself unless more than k points coincide with it.  The rows come from the
// existing k_knn instances (query.cu), fed the P points in the grid's sorted order (GridDev::pts, w = original index)
// so that neighbouring threads descend neighbouring boxes; row t belongs to sorted point t.
//
// k_normals, one thread per sorted point t of original index j.  In double, over the m real entries of the row in row
// order (ascending (d^2, index); the padding at its end is skipped):
//   c = sum p / m;  C = sum (p - c)(p - c)^T / m   (each sum from 0.0, left to right)
// then cyclic Jacobi rotations on C (jacobi_pair, the classic threshold form) until the off-diagonal entries are exactly
// zero or kJacobiSweeps sweeps have run; the diagonal holds the eigenvalues and the accumulated rotation V the
// eigenvectors (columns).  The eigenvalues are ordered ascending by a stable sort of the columns, so equal eigenvalues
// keep the column order of V; the normal is the column of the first, normalised in double, its sign set (below) and
// rounded to float.  Sign: with a viewpoint v, the normal n is negated when (v - p_j) . n < 0 (double); without one, the
// component of largest magnitude of the rounded normal is made positive, ties to the lowest axis.  m < 3 or C exactly
// zero (coincident points): the normal is (0, 0, 0).  The eigenvalues are written in every case.
//
// Determinism.  The rows are fixed (k_knn's lexicographic k-minimum does not depend on the search order), the sums run in
// row order, and every value is made of IEEE basic operations (+ - * /, sqrt, fabs, compares) in double, compiled with
// -fmad=false so that no product is contracted into an FMA.  So a CPU restatement of the same operations, compiled
// without contraction (-ffp-contract=off), gives the same bits.
#include "s4g_internal.cuh"
#include <cmath>

namespace {

constexpr int kNormalsThreads = 128;
constexpr int kJacobiSweeps = 50;
constexpr int kNormalsMinK = 3, kNormalsMaxK = 64;   // k = 64: k_knn's widest instance

// sorted P (float4, w = original index) -> the n x 3 query array of k_knn
__global__ void k_normals_queries(const float4* __restrict__ pts, int n, float* __restrict__ xyz) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const float4 p = pts[t];
  xyz[3 * t] = p.x;
  xyz[3 * t + 1] = p.y;
  xyz[3 * t + 2] = p.z;
}

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

__global__ void __launch_bounds__(kNormalsThreads)
k_normals(const float4* __restrict__ sorted, const float4* __restrict__ P, const int32_t* __restrict__ rows, int n, int k,
          bool has_vp, float vx, float vy, float vz, float* __restrict__ normals, float* __restrict__ eigenvalues) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const float4 self = __ldg(&sorted[t]);
  const long long j = __float_as_int(self.w);
  const int32_t* __restrict__ row = rows + t * (long long)k;
  int m = 0;
  double sx = 0.0, sy = 0.0, sz = 0.0;
#pragma unroll 1
  for (; m < k; ++m) {
    const int32_t e = __ldg(&row[m]);
    if (e < 0) break;
    const float4 p = __ldg(&P[e]);
    sx = sx + (double)p.x;
    sy = sy + (double)p.y;
    sz = sz + (double)p.z;
  }
  const double dm = (double)m, cx = sx / dm, cy = sy / dm, cz = sz / dm;
  double a00 = 0.0, a01 = 0.0, a02 = 0.0, a11 = 0.0, a12 = 0.0, a22 = 0.0;
#pragma unroll 1
  for (int i = 0; i < m; ++i) {
    const float4 p = __ldg(&P[__ldg(&row[i])]);
    const double dx = (double)p.x - cx, dy = (double)p.y - cy, dz = (double)p.z - cz;
    a00 = a00 + dx * dx;
    a01 = a01 + dx * dy;
    a02 = a02 + dx * dz;
    a11 = a11 + dy * dy;
    a12 = a12 + dy * dz;
    a22 = a22 + dz * dz;
  }
  a00 = a00 / dm;
  a01 = a01 / dm;
  a02 = a02 / dm;
  a11 = a11 / dm;
  a12 = a12 / dm;
  a22 = a22 / dm;
  const bool none = m < 3 || (a00 == 0.0 && a01 == 0.0 && a02 == 0.0 && a11 == 0.0 && a12 == 0.0 && a22 == 0.0);
  double v0[3] = {1.0, 0.0, 0.0}, v1[3] = {0.0, 1.0, 0.0}, v2[3] = {0.0, 0.0, 1.0};   // the columns of V
#pragma unroll 1
  for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
    if (a01 == 0.0 && a02 == 0.0 && a12 == 0.0) break;
    jacobi_pair(a00, a11, a01, a02, a12, v0, v1);
    jacobi_pair(a00, a22, a02, a01, a12, v0, v2);
    jacobi_pair(a11, a22, a12, a01, a02, v1, v2);
  }
  // stable ascending order of the diagonal: o0 <= o1 <= o2, equal values in column order
  int o0 = 0, o1 = 1, o2 = 2;
  if (pick3(a00, a11, a22, o1) < pick3(a00, a11, a22, o0)) { const int s = o0; o0 = o1; o1 = s; }
  if (pick3(a00, a11, a22, o2) < pick3(a00, a11, a22, o1)) {
    const int s = o1; o1 = o2; o2 = s;
    if (pick3(a00, a11, a22, o1) < pick3(a00, a11, a22, o0)) { const int s2 = o0; o0 = o1; o1 = s2; }
  }
  if (eigenvalues != nullptr) {
    eigenvalues[3 * j] = (float)pick3(a00, a11, a22, o0);
    eigenvalues[3 * j + 1] = (float)pick3(a00, a11, a22, o1);
    eigenvalues[3 * j + 2] = (float)pick3(a00, a11, a22, o2);
  }
  float fx = 0.f, fy = 0.f, fz = 0.f;
  if (!none) {
    double nx = pick3(v0[0], v1[0], v2[0], o0), ny = pick3(v0[1], v1[1], v2[1], o0), nz = pick3(v0[2], v1[2], v2[2], o0);
    const double len = sqrt(nx * nx + ny * ny + nz * nz);
    nx = nx / len;
    ny = ny / len;
    nz = nz / len;
    if (has_vp && ((double)vx - (double)self.x) * nx + ((double)vy - (double)self.y) * ny + ((double)vz - (double)self.z) * nz < 0.0) {
      nx = -nx;
      ny = -ny;
      nz = -nz;
    }
    fx = (float)nx;
    fy = (float)ny;
    fz = (float)nz;
    if (!has_vp) {
      float big = fx;                                    // the component of largest magnitude, the lowest axis on a tie
      if (fabsf(fy) > fabsf(big)) big = fy;
      if (fabsf(fz) > fabsf(big)) big = fz;
      if (big < 0.f) {
        fx = -fx;
        fy = -fy;
        fz = -fz;
      }
    }
  }
  normals[3 * j] = fx;
  normals[3 * j + 1] = fy;
  normals[3 * j + 2] = fz;
}

unsigned nblk(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

int normals_args(s4g_ctx* ctx, const char* who, int k, float sq_radius, const void* normals) {
  if (k < kNormalsMinK || k > kNormalsMaxK || std::isnan(sq_radius) || sq_radius < 0.f || normals == nullptr) {
    ctx->err = std::string(who) + ": bad arguments (3 <= k <= 64, sq_radius >= 0 and not NaN, normals != NULL)";
    return S4G_ERR_ARG;
  }
  if (ctx->nP <= 0) {
    ctx->err = std::string(who) + ": call s4g_set_cloud_p first";
    return S4G_ERR_STATE;
  }
  return S4G_OK;
}

// enqueue the three launches on the context's stream: the sorted queries (scratch A), their k_knn rows (scratch B), and
// k_normals into the device outputs
int launch_normals(s4g_ctx* ctx, int k, float sq_radius, const float* viewpoint, float* d_normals, float* d_eigenvalues) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  const int n = ctx->nP;
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, (size_t)n * 3 * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, (size_t)n * (size_t)k * sizeof(int32_t)));
  float* d_xyz = ctx->dScratchA.as<float>();
  int32_t* d_rows = ctx->dScratchB.as<int32_t>();
  S4G_TRY(s4g_launch_sorted_queries(ctx, d_xyz));
  S4G_TRY(s4g_launch_knn(ctx, d_xyz, n, nullptr, k, sq_radius, nullptr, d_rows, nullptr, nullptr));
  const bool has_vp = viewpoint != nullptr;
  k_normals<<<nblk(n, kNormalsThreads), kNormalsThreads, 0, ctx->stream>>>(
      ctx->grid.pts, ctx->dP.as<float4>(), d_rows, n, k, has_vp, has_vp ? viewpoint[0] : 0.f, has_vp ? viewpoint[1] : 0.f,
      has_vp ? viewpoint[2] : 0.f, d_normals, d_eigenvalues);
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;
}

}  // namespace

int s4g_launch_sorted_queries(s4g_ctx* ctx, float* d_xyz) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  k_normals_queries<<<nblk(ctx->nP, 256), 256, 0, ctx->stream>>>(ctx->grid.pts, ctx->nP, d_xyz);
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;
}

extern "C" int s4g_normals_dev(s4g_ctx* ctx, int k, float sq_radius, const float* viewpoint, float* d_normals,
                               float* d_eigenvalues) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(normals_args(ctx, "s4g_normals_dev", k, sq_radius, d_normals));
  return launch_normals(ctx, k, sq_radius, viewpoint, d_normals, d_eigenvalues);
}

extern "C" int s4g_normals(s4g_ctx* ctx, int k, float sq_radius, const float* viewpoint, float* normals,
                           float* eigenvalues) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(normals_args(ctx, "s4g_normals", k, sq_radius, normals));
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t bytes = (size_t)ctx->nP * 3 * sizeof(float);
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchC, bytes));
  if (eigenvalues != nullptr) S4G_TRY(s4g_reserve(ctx, ctx->dScratchD, bytes));
  float* d_eig = eigenvalues != nullptr ? ctx->dScratchD.as<float>() : nullptr;
  S4G_TRY(launch_normals(ctx, k, sq_radius, viewpoint, ctx->dScratchC.as<float>(), d_eig));
  S4G_CUDA(cudaMemcpyAsync(normals, ctx->dScratchC.p, bytes, cudaMemcpyDeviceToHost, st));
  if (eigenvalues != nullptr) S4G_CUDA(cudaMemcpyAsync(eigenvalues, d_eig, bytes, cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  return S4G_OK;
}
