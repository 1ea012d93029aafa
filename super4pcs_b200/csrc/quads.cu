// a4 -- IndexedNormalSet<Point,3,7,float> (reference accelerators/normalset.h:71-153,
//       accelerators/normalset.hpp:57-210; index helpers accelerators/utils.h:139-148)
// a5 -- MatchSuper4PCS::FindCongruentQuadrilaterals (reference algorithms/super4pcs.cc:80-177)
//
// The reference allocates a dense egSize^3 table of pointers to 343-bin angular grids on every
// call (infeasible for fine epsilon, SURVEY.md 8(a) row a4).  Here every P-pair k gets the 64-bit
// key  cell(k) * 343 + bin(k)  (cell = Euclidean cell of its invariant point, bin = direction bin
// of its segment), the (key, k) list is radix-sorted, and each Q-pair (one thread) binary-searches
// its single cell, renders the reference's cone of sample directions into a 343-bit mask and walks
// the cell's sorted entries.  All index arithmetic reproduces the reference's truncating casts; the
// cone constants that need libm (acosf, atanf, sinf, cosf) are evaluated on the HOST with the same
// glibc the reference uses and handed to the kernel as a table, the per-query quaternion
// (Eigen setFromTwoVectors incl. its nearly-opposite SVD branch), rotation and normalisation are
// plain IEEE float operations reproduced operation by operation.
// Output order = the reference's std::set<(id,i)> order (super4pcs.cc:127,166-174): quads are
// radix-sorted by (index in P_pairs, index in Q_pairs).
#include "s4g_internal.cuh"
#include <cub/cub.cuh>
#include <cmath>
#include <cstring>
#include <algorithm>
#include <vector>

int s4g_sort_pairs(s4g_ctx* ctx, int slot);

namespace {

struct NSet {
  float nepsilon;   // 1/7 + 1e-5 as float (normalset.h:115)
  float epsilon;    // 1 / egSize (normalset.h:121)
  long long egSize;
};

struct QuadArgs {
  NSet g;
  float inv1, inv2, thr2, alpha_cos;
  int nbSample;
  float3 ring[56];  // (sin a cos t, sin a sin t, cos a), normalset.hpp:186-190
};

__device__ __forceinline__ long long index_pos(const NSet& g, float3 p) {
  // UnrollIndexLoop over p / _epsilon with truncating casts (utils.h:139-148)
  float3 c = s4_div(p, g.epsilon);
  return ((long long)(int)c.z * g.egSize + (long long)(int)c.y) * g.egSize + (long long)(int)c.x;
}
__device__ __forceinline__ int index_normal(const NSet& g, float3 n) {
  float cx = __fdiv_rn(__fadd_rn(__fdiv_rn(n.x, 2.f), 0.5f), g.nepsilon);
  float cy = __fdiv_rn(__fadd_rn(__fdiv_rn(n.y, 2.f), 0.5f), g.nepsilon);
  float cz = __fdiv_rn(__fadd_rn(__fdiv_rn(n.z, 2.f), 0.5f), g.nepsilon);
  return ((int)cz * 7 + (int)cy) * 7 + (int)cx;
}

// ---- Eigen's nearly-opposite branch of setFromTwoVectors: third column of the Householder Q of
// ColPivHouseholderQR([v0 | v1]) (JacobiSVD<2x3> with ComputeFullV; the Jacobi sweeps and the
// sort only touch columns 0 and 1 of V).
__device__ void make_householder(const float* v, int n, float* ess, float* tau, float* beta) {
  float tailSq = 0.f;
  for (int i = 1; i < n; ++i) tailSq = (i == 1) ? __fmul_rn(v[i], v[i]) : __fadd_rn(tailSq, __fmul_rn(v[i], v[i]));
  float c0 = v[0];
  const float tol = 1.17549435e-38f;
  if (tailSq <= tol) {
    *tau = 0.f;
    *beta = c0;
    for (int i = 0; i < n - 1; ++i) ess[i] = 0.f;
  } else {
    float b = __fsqrt_rn(__fadd_rn(__fmul_rn(c0, c0), tailSq));
    if (c0 >= 0.f) b = -b;
    for (int i = 0; i < n - 1; ++i) ess[i] = __fdiv_rn(v[i + 1], __fsub_rn(c0, b));
    *tau = __fdiv_rn(__fsub_rn(b, c0), b);
    *beta = b;
  }
}
__device__ void apply_householder_left(float* M, int ld, int rows, int cols, const float* ess, float tau) {
  if (rows == 1) {
    for (int j = 0; j < cols; ++j) M[j] = __fmul_rn(M[j], __fsub_rn(1.f, tau));
    return;
  }
  if (tau == 0.f) return;
  float tmp[3];
  for (int j = 0; j < cols; ++j) {
    float acc = 0.f;
    for (int i = 0; i < rows - 1; ++i) {
      float t = __fmul_rn(ess[i], M[(i + 1) * ld + j]);
      acc = (i == 0) ? t : __fadd_rn(acc, t);
    }
    tmp[j] = __fadd_rn(acc, M[j]);
  }
  for (int j = 0; j < cols; ++j) M[j] = __fsub_rn(M[j], __fmul_rn(tau, tmp[j]));
  for (int i = 0; i < rows - 1; ++i)
    for (int j = 0; j < cols; ++j)
      M[(i + 1) * ld + j] = __fsub_rn(M[(i + 1) * ld + j], __fmul_rn(__fmul_rn(tau, ess[i]), tmp[j]));
}
__device__ float3 svd_null_axis(float3 v0, float3 v1) {
  float sc = fmaxf(fmaxf(fmaxf(fabsf(v0.x), fabsf(v0.y)), fmaxf(fabsf(v0.z), fabsf(v1.x))), fmaxf(fabsf(v1.y), fabsf(v1.z)));
  if (sc == 0.f) sc = 1.f;
  float A[3][2] = {{__fdiv_rn(v0.x, sc), __fdiv_rn(v1.x, sc)},
                   {__fdiv_rn(v0.y, sc), __fdiv_rn(v1.y, sc)},
                   {__fdiv_rn(v0.z, sc), __fdiv_rn(v1.z, sc)}};
  float nrm[2];
  for (int k = 0; k < 2; ++k)
    nrm[k] = __fsqrt_rn(s4_sum3(__fmul_rn(A[0][k], A[0][k]), __fmul_rn(A[1][k], A[1][k]), __fmul_rn(A[2][k], A[2][k])));
  float hc[2] = {0.f, 0.f};
  float ess[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
  for (int k = 0; k < 2; ++k) {
    if (k == 0 && nrm[1] > nrm[0]) {
      for (int r = 0; r < 3; ++r) { float t = A[r][0]; A[r][0] = A[r][1]; A[r][1] = t; }
      float t = nrm[0]; nrm[0] = nrm[1]; nrm[1] = t;
    }
    float col[3];
    for (int r = k; r < 3; ++r) col[r - k] = A[r][k];
    float beta;
    make_householder(col, 3 - k, ess[k], &hc[k], &beta);
    A[k][k] = beta;
    if (k == 0) {
      float M[3] = {A[0][1], A[1][1], A[2][1]};
      apply_householder_left(M, 1, 3, 1, ess[0], hc[0]);
      A[0][1] = M[0]; A[1][1] = M[1]; A[2][1] = M[2];
    }
  }
  float Qm[9] = {1.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 1.f};
  apply_householder_left(&Qm[4], 3, 2, 2, ess[1], hc[1]);
  apply_householder_left(&Qm[0], 3, 3, 3, ess[0], hc[0]);
  return make_float3(Qm[2], Qm[5], Qm[8]);
}

// QuaternionBase::setFromTwoVectors((0,0,1), n) + _transformVector (Geometry/Quaternion.h:472-481,578-612)
struct Quat { float x, y, z, w; };
__device__ Quat quat_from_z_to(float3 n) {
  float3 v0 = s4_normalized(make_float3(0.f, 0.f, 1.f)), v1 = s4_normalized(n);
  float c = s4_dot(v1, v0);
  Quat q;
  if (c < __fadd_rn(-1.f, 1e-5f)) {
    c = fmaxf(c, -1.f);
    float3 axis = svd_null_axis(v0, v1);
    float w2 = __fmul_rn(__fadd_rn(1.f, c), 0.5f);
    q.w = __fsqrt_rn(w2);
    float k = __fsqrt_rn(__fsub_rn(1.f, w2));
    q.x = __fmul_rn(axis.x, k); q.y = __fmul_rn(axis.y, k); q.z = __fmul_rn(axis.z, k);
    return q;
  }
  float3 axis = s4_cross(v0, v1);
  float sq = __fsqrt_rn(__fmul_rn(__fadd_rn(1.f, c), 2.f));
  float invs = __fdiv_rn(1.f, sq);
  q.x = __fmul_rn(axis.x, invs); q.y = __fmul_rn(axis.y, invs); q.z = __fmul_rn(axis.z, invs);
  q.w = __fmul_rn(sq, 0.5f);
  return q;
}
__device__ __forceinline__ float3 quat_rotate(const Quat& q, float3 v) {
  float3 qv = make_float3(q.x, q.y, q.z);
  float3 uv = s4_cross(qv, v);
  uv = s4_add(uv, uv);
  return s4_add(s4_add(v, s4_scale(q.w, uv)), s4_cross(qv, uv));
}

// ---- the stages shared by the per-base kernels and the batched ones (s4g_try_bases)

// first key of the cell that holds p: the keys of the cell's 343 direction bins are [k, k + 343)
__device__ __forceinline__ unsigned long long cell_key(const NSet& g, float3 p) {
  return (unsigned long long)index_pos(g, p) * 343ull;
}

// key cell * 343 + bin of the P-pair (p1, p2) (unit-cube coordinates)
__device__ __forceinline__ unsigned long long ppair_key(const QuadArgs& A, float3 p1, float3 p2) {
  float3 d = s4_sub(p2, p1);
  float3 n = s4_normalized(d);                                  // super4pcs.cc:121
  float3 pos = s4_add(p1, s4_scale(A.inv1, d));                 // super4pcs.cc:123
  return cell_key(A.g, pos) + (unsigned long long)index_normal(A.g, n);
}

// invariant point p1 + invariant2 * (p2 - p1) of a Q-pair: `query` in unit-cube coordinates (super4pcs.cc:141),
// `queryQ` in sampled-Q coordinates (super4pcs.cc:142)
__device__ __forceinline__ float3 query_point(const QuadArgs& A, float3 p1, float3 p2) {
  return s4_add(p1, s4_scale(A.inv2, s4_sub(p2, p1)));
}

// first position in keys[0, n) whose key is >= k
__device__ __forceinline__ long long lower_bound(const unsigned long long* __restrict__ keys, long long n,
                                                 unsigned long long k) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    long long mid = (lo + hi) >> 1;
    if (keys[mid] < k) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// the direction bins of the cone around the Q-pair direction d, as a 343-bit mask (normalset.hpp:186-190)
__device__ __forceinline__ void cone_mask(const QuadArgs& A, float3 d, uint32_t (&mask)[11]) {
  float3 queryn = s4_normalized(d);
  Quat qt = quat_from_z_to(queryn);
#pragma unroll
  for (int w = 0; w < 11; ++w) mask[w] = 0u;
  for (int a = 0; a < A.nbSample; ++a) {
    float3 dir = s4_normalized(quat_rotate(qt, A.ring[a]));
    int id = index_normal(A.g, dir);
    if ((unsigned)id < 343u) mask[id >> 5] |= 1u << (id & 31);
  }
}

// does the P-pair pp (sampled-Q indices) form a quad with the Q-pair of invariant point queryQ
__device__ __forceinline__ bool ppair_matches(const QuadArgs& A, const float4* __restrict__ q, int2 pp, float3 queryQ) {
  float3 pp1 = s4_xyz(q[pp.x]), pp2 = s4_xyz(q[pp.y]);
  float3 dd = s4_sub(pp2, pp1);
  float3 invPoint = s4_add(pp1, make_float3(__fmul_rn(dd.x, A.inv1), __fmul_rn(dd.y, A.inv1), __fmul_rn(dd.z, A.inv1)));
  // squared norm vs the UN-squared threshold, as the reference does (super4pcs.cc:160)
  return s4_sqnorm(s4_sub(queryQ, invPoint)) <= A.thr2;
}

// ---- build: key of every P-pair
__global__ void k_quad_keys(QuadArgs A, const float4* __restrict__ qunit, const int2* __restrict__ pairs1,
                            long long n1, unsigned long long* __restrict__ keys, uint32_t* __restrict__ vals) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n1) return;
  int2 pr = pairs1[i];
  keys[i] = ppair_key(A, s4_xyz(qunit[pr.x]), s4_xyz(qunit[pr.y]));
  vals[i] = (uint32_t)i;
}

// ---- query: one thread per Q-pair.  kFill == false counts, kFill == true writes (id, i) keys.
template <bool kFill>
__global__ void __launch_bounds__(128)
k_quad_query(QuadArgs A, const float4* __restrict__ qunit, const float4* __restrict__ q,
             const int2* __restrict__ pairs1, const int2* __restrict__ pairs2, long long n1, long long n2,
             const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ vals,
             unsigned long long* __restrict__ counts, const unsigned long long* __restrict__ offsets,
             unsigned long long* __restrict__ out) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n2) return;
  int2 pr = pairs2[i];
  float3 p1 = s4_xyz(qunit[pr.x]), p2 = s4_xyz(qunit[pr.y]);
  unsigned long long kbeg = cell_key(A.g, query_point(A, p1, p2)), kend = kbeg + 343ull;
  long long lo = lower_bound(keys, n1, kbeg);
  unsigned long long cnt = 0;
  if (lo < n1 && keys[lo] < kend) {                             // angularGrid(p) != NULL
    uint32_t mask[11];
    cone_mask(A, s4_sub(p2, p1), mask);
    float3 queryQ = query_point(A, s4_xyz(q[pr.x]), s4_xyz(q[pr.y]));
    unsigned long long wr = kFill ? offsets[i] : 0ull;
    for (long long e = lo; e < n1; ++e) {
      unsigned long long k = keys[e];
      if (k >= kend) break;
      int bin = (int)(k - kbeg);
      if (!((mask[bin >> 5] >> (bin & 31)) & 1u)) continue;
      uint32_t id = vals[e];
      if (ppair_matches(A, q, pairs1[id], queryQ)) {
        if (kFill) out[wr] = ((unsigned long long)id << 32) | (unsigned long long)(uint32_t)i;
        ++wr;
        ++cnt;
      }
    }
  }
  if (!kFill) counts[i] = cnt;
}

__global__ void k_emit_quads(const unsigned long long* __restrict__ keys, long long n,
                             const int2* __restrict__ pairs1, const int2* __restrict__ pairs2,
                             int4* __restrict__ quads) {
  long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  unsigned long long k = keys[t];
  int2 a = pairs1[(uint32_t)(k >> 32)], b = pairs2[(uint32_t)(k & 0xffffffffull)];
  quads[t] = make_int4(a.x, a.y, b.x, b.y);
}

// host: Eigen normalized()/dot in float (x86-64 baseline: no FMA contraction)
inline void h_normalized(const float* a, float* o) {
  volatile float xx = a[0] * a[0], yy = a[1] * a[1], zz = a[2] * a[2];
  volatile float yz = yy + zz;
  volatile float z = xx + yz;
  if (z > 0.f) {
    float s = std::sqrt((float)z);
    o[0] = a[0] / s; o[1] = a[1] / s; o[2] = a[2] / s;
  } else {
    o[0] = a[0]; o[1] = a[1]; o[2] = a[2];
  }
}

int bits_for(long long n) {
  int b = 1;
  while ((1ll << b) < n && b < 62) ++b;
  return b;
}

}  // namespace

// QuadArgs of one FindCongruentQuadrilaterals call (cone constants through the host's libm, like the reference)
static int make_quad_args(s4g_ctx* ctx, float invariant1, float invariant2, float distance_threshold2, const float* base_xyz,
                          QuadArgs& A, int& gridDepth_out) {
  std::memset(&A, 0, sizeof A);
  A.inv1 = invariant1;
  A.inv2 = invariant2;
  A.thr2 = distance_threshold2;
  {
    // alpha = (b1-b0).normalized().dot((b3-b2).normalized()), super4pcs.cc:109-111
    float u[3] = {base_xyz[3] - base_xyz[0], base_xyz[4] - base_xyz[1], base_xyz[5] - base_xyz[2]};
    float v[3] = {base_xyz[9] - base_xyz[6], base_xyz[10] - base_xyz[7], base_xyz[11] - base_xyz[8]};
    float un[3], vn[3];
    h_normalized(u, un);
    h_normalized(v, vn);
    volatile float a0 = un[0] * vn[0], a1 = un[1] * vn[1], a2 = un[2] * vn[2];
    volatile float a12 = a1 + a2;
    A.alpha_cos = a0 + a12;
  }
  const float eps = distance_threshold2 / ctx->ratio;           // getNormalizedEpsilon, super4pcs.cc:114
  A.g.nepsilon = (float)(1.f / 7.f + 0.00001);                  // normalset.h:115
  const int gridDepth = -std::log2(eps);
  gridDepth_out = gridDepth;                        // normalset.h:119
  if (!(eps > 0.f) || gridDepth < 0 || gridDepth > 18) {
    ctx->err = "s4g_find_quads: distance_threshold2 / ratio out of the supported range (2^-18 .. 1)";
    return S4G_ERR_ARG;
  }
  A.g.egSize = (long long)std::pow(2, gridDepth);               // normalset.h:120
  A.g.epsilon = 1.f / (float)A.g.egSize;                        // normalset.h:121
  {
    // getNeighbors constants, normalset.hpp:174-181 (host libm == the reference's libm)
    const float alpha = std::acos(A.alpha_cos);
    const float perimeter = (float)(2.f * M_PI * std::atan(alpha));
    const float nbf = 2 * std::ceil(perimeter * 7.f / 2.f);
    unsigned int nbSample = (nbf == nbf && nbf > 0.f) ? (unsigned int)nbf : 0u;
    if (nbSample > 56u) nbSample = 56u;                          // 2*ceil(2*pi*atan(pi)*3.5) = 56 is the maximum
    const float angleStep = (float)(2.f * M_PI / float(nbSample));
    const float sinAlpha = std::sin(alpha);
    A.nbSample = (int)nbSample;
    for (unsigned int a = 0; a < nbSample; ++a) {
      float theta = float(a) * angleStep;
      A.ring[a] = make_float3(sinAlpha * std::cos(theta), sinAlpha * std::sin(theta), A.alpha_cos);
    }
  }
  return S4G_OK;
}

extern "C" int s4g_find_quads(s4g_ctx* ctx, float invariant1, float invariant2, float distance_threshold2,
                              const float* base_xyz, int64_t* n_quads) {
  if (!ctx) return S4G_ERR_ARG;
  if (!base_xyz) { ctx->err = "s4g_find_quads: null base"; return S4G_ERR_ARG; }
  if (ctx->nQ <= 0) { ctx->err = "s4g_find_quads: call s4g_set_cloud_q first"; return S4G_ERR_STATE; }
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  ctx->nQuads = 0;
  if (n_quads) *n_quads = 0;
  const long long n1 = ctx->nPairs[0], n2 = ctx->nPairs[1];
  if (n1 == 0 || n2 == 0) return S4G_OK;
  if (n1 >= (1ll << 32) || n2 >= (1ll << 32)) { ctx->err = "s4g_find_quads: pair lists must be < 2^32"; return S4G_ERR_ARG; }

  QuadArgs A;
  int gridDepth = 0;
  S4G_TRY(make_quad_args(ctx, invariant1, invariant2, distance_threshold2, base_xyz, A, gridDepth));
  if (A.nbSample == 0) return S4G_OK;

  // extracted lists are put in canonical (sorted) order first; uploaded lists keep the caller's order
  S4G_TRY(s4g_sort_pairs(ctx, 0));
  S4G_TRY(s4g_sort_pairs(ctx, 1));
  const int2* pairs1 = ctx->dPairs[0].as<int2>();
  const int2* pairs2 = ctx->dPairs[1].as<int2>();

  // build the sorted (key, id) list of the P-pairs
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, (size_t)n1 * 2 * sizeof(unsigned long long)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, (size_t)n1 * 2 * sizeof(uint32_t)));
  unsigned long long* keys_in = ctx->dScratchA.as<unsigned long long>();
  unsigned long long* keys = keys_in + n1;
  uint32_t* vals_in = ctx->dScratchB.as<uint32_t>();
  uint32_t* vals = vals_in + n1;
  S4G_EV_START(ctx, S4G_EV_QUADS);
  k_quad_keys<<<(unsigned)((n1 + 255) / 256), 256, 0, st>>>(A, ctx->dQunit.as<float4>(), pairs1, n1, keys_in, vals_in);
  int kbits = std::min(64, 3 * gridDepth + 9 + 1);
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, keys_in, keys, vals_in, vals, (long long)n1, 0, kbits, st);
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, cub_bytes));
  cub::DeviceRadixSort::SortPairs(ctx->dCub.p, cub_bytes, keys_in, keys, vals_in, vals, (long long)n1, 0, kbits, st);

  // count -> scan -> fill
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchC, (size_t)(2 * (n2 + 1)) * sizeof(unsigned long long)));
  unsigned long long* counts = ctx->dScratchC.as<unsigned long long>();
  unsigned long long* offsets = counts + (n2 + 1);
  S4G_CUDA(cudaMemsetAsync(counts, 0, (size_t)(n2 + 1) * sizeof(unsigned long long), st));
  k_quad_query<false><<<(unsigned)((n2 + 127) / 128), 128, 0, st>>>(A, ctx->dQunit.as<float4>(), ctx->dQ.as<float4>(),
                                                                  pairs1, pairs2, n1, n2, keys, vals, counts, nullptr, nullptr);
  size_t scan_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, counts, offsets, (long long)(n2 + 1), st);
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, scan_bytes));
  cub::DeviceScan::ExclusiveSum(ctx->dCub.p, scan_bytes, counts, offsets, (long long)(n2 + 1), st);
  ctx->launches += 5;
  unsigned long long total = 0;
  S4G_CUDA(cudaMemcpyAsync(&total, offsets + n2, sizeof total, cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  if (total == 0) {
    S4G_EV_STOP(ctx, S4G_EV_QUADS);
    return S4G_OK;
  }
  if (total >= (1ull << 32) - 1) { ctx->err = "s4g_find_quads: more than 2^32-2 quads"; return S4G_ERR_NOMEM; }
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchD, (size_t)total * 2 * sizeof(unsigned long long)));
  unsigned long long* qk_in = ctx->dScratchD.as<unsigned long long>();
  unsigned long long* qk = qk_in + total;
  k_quad_query<true><<<(unsigned)((n2 + 127) / 128), 128, 0, st>>>(A, ctx->dQunit.as<float4>(), ctx->dQ.as<float4>(),
                                                                 pairs1, pairs2, n1, n2, keys, vals, nullptr, offsets, qk_in);
  // std::set<(id,i)> order
  cub_bytes = 0;
  int b2 = bits_for(n2), b1 = bits_for(n1);
  cub::DeviceRadixSort::SortKeys(nullptr, cub_bytes, qk_in, qk, (long long)total, 0, 32 + b1, st);
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, cub_bytes));
  (void)b2;
  cub::DeviceRadixSort::SortKeys(ctx->dCub.p, cub_bytes, qk_in, qk, (long long)total, 0, 32 + b1, st);
  S4G_TRY(s4g_reserve(ctx, ctx->dQuads, (size_t)total * sizeof(int4)));
  k_emit_quads<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(qk, (long long)total, pairs1, pairs2, ctx->dQuads.as<int4>());
  S4G_EV_STOP(ctx, S4G_EV_QUADS);
  ctx->launches += 4;
  S4G_CUDA(cudaGetLastError());
  S4G_CUDA(cudaStreamSynchronize(st));
  ctx->nQuads = (long long)total;
  if (n_quads) *n_quads = (int64_t)total;
  return S4G_OK;
}

// ============================================================================================
// f1: the quad stage of B bases at once (s4g_try_bases).  Input: the batch's sorted pair keys
// (segment << 52 | first << 26 | second; segment 2b = P-pairs of base b, 2b + 1 = its Q-pairs).  Every kernel
// runs over ALL entries; the base comes from the key's prefix, its QuadArgs from an array.
// ============================================================================================
namespace {

__device__ __forceinline__ int2 key_pair(unsigned long long k) {
  return make_int2((int)((k >> kBatchIdBits) & ((1ull << kBatchIdBits) - 1ull)), (int)(k & ((1ull << kBatchIdBits) - 1ull)));
}

// P-pair entries -> (base << 52 | cell * 343 + bin, id local to the base's P list); Q-pair entries -> padding key
__global__ void k_bquad_keys(const QuadArgs* __restrict__ args, const float4* __restrict__ qunit,
                             const unsigned long long* __restrict__ pkeys, long long n, const uint32_t* __restrict__ segOff,
                             unsigned long long* __restrict__ keys, uint32_t* __restrict__ vals, uint32_t* __restrict__ err) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long pk = pkeys[i];
  const uint32_t seg = (uint32_t)(pk >> kBatchSegShift);
  if (seg & 1u) { keys[i] = ~0ull; vals[i] = 0u; return; }
  const int2 pr = key_pair(pk);
  const unsigned long long ck = ppair_key(args[seg >> 1], s4_xyz(qunit[pr.x]), s4_xyz(qunit[pr.y]));
  if (ck >> kBatchSegShift) atomicAdd(err, 1u);                 // cannot happen for grid depths <= 14 (checked by the host)
  keys[i] = ((unsigned long long)(seg >> 1) << kBatchSegShift) | ck;
  vals[i] = (uint32_t)(i - segOff[seg]);
}

// one thread per entry; Q-pair entries look up their base's sorted P keys (prefix base << 52)
template <bool kFill>
__global__ void __launch_bounds__(128)
k_bquad_query(const QuadArgs* __restrict__ args, const float4* __restrict__ qunit, const float4* __restrict__ q,
              const unsigned long long* __restrict__ pkeys, long long n, const uint32_t* __restrict__ segOff,
              const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ vals, long long nP,
              uint32_t* __restrict__ counts, const uint32_t* __restrict__ offsets, unsigned long long* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long pk = pkeys[i];
  const uint32_t seg = (uint32_t)(pk >> kBatchSegShift);
  uint32_t cnt = 0;
  if (seg & 1u) {
    const uint32_t base = seg >> 1;
    const QuadArgs& A = args[base];
    const int2 pr = key_pair(pk);
    float3 p1 = s4_xyz(qunit[pr.x]), p2 = s4_xyz(qunit[pr.y]);
    const unsigned long long pre = (unsigned long long)base << kBatchSegShift;
    const unsigned long long kbeg = pre | cell_key(A.g, query_point(A, p1, p2)), kend = kbeg + 343ull;
    const long long lo = lower_bound(keys, nP, kbeg);
    if (A.nbSample > 0 && lo < nP && keys[lo] < kend) {          // angularGrid(p) != NULL
      uint32_t mask[11];
      cone_mask(A, s4_sub(p2, p1), mask);
      float3 queryQ = query_point(A, s4_xyz(q[pr.x]), s4_xyz(q[pr.y]));
      const uint32_t pOff = segOff[seg - 1u];                   // the base's P-pair segment
      const uint32_t iLocal = (uint32_t)(i - segOff[seg]);
      uint32_t wr = kFill ? offsets[i] : 0u;
      for (long long e = lo; e < nP; ++e) {
        unsigned long long k = keys[e];
        if (k >= kend) break;
        int bin = (int)(k - kbeg);
        if (!((mask[bin >> 5] >> (bin & 31)) & 1u)) continue;
        const uint32_t id = vals[e];
        if (ppair_matches(A, q, key_pair(pkeys[pOff + id]), queryQ)) {
          if (kFill) out[wr] = pre | ((unsigned long long)id << kBatchIdBits) | (unsigned long long)iLocal;
          ++wr;
          ++cnt;
        }
      }
    }
  }
  if (!kFill) counts[i] = cnt;
}

// (base, id, i) keys -> quads; also the first quad of every base
__global__ void k_bquad_emit(const unsigned long long* __restrict__ qk, long long n, const unsigned long long* __restrict__ pkeys,
                             const uint32_t* __restrict__ segOff, int4* __restrict__ quads) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const unsigned long long k = qk[t];
  const uint32_t base = (uint32_t)(k >> kBatchSegShift);
  const uint32_t id = (uint32_t)((k >> kBatchIdBits) & ((1ull << kBatchIdBits) - 1ull)), i2 = (uint32_t)(k & ((1ull << kBatchIdBits) - 1ull));
  const int2 a = key_pair(pkeys[segOff[2 * base] + id]), b = key_pair(pkeys[segOff[2 * base + 1] + i2]);
  quads[t] = make_int4(a.x, a.y, b.x, b.y);
}

__global__ void k_bquad_offsets(const uint32_t* __restrict__ offsets, const uint32_t* __restrict__ segOff, int B, long long n,
                                uint32_t* __restrict__ quadOff) {
  const int b = threadIdx.x;
  if (b < B) quadOff[b] = offsets[segOff[2 * b + 1]];
  if (b == B) quadOff[B] = offsets[n];
}

}  // namespace

int s4g_batch_quads(s4g_ctx* ctx, const s4g_base_desc* bases, float thr2, BatchHost& bh) {
  cudaStream_t st = ctx->stream;
  const int B = bh.B;
  const long long n = (long long)bh.nPairs, nP = (long long)bh.nPPairs;
  bh.nQuads = 0;
  for (int b = 0; b <= B; ++b) bh.quadOff[b] = 0;
  if (n == 0 || nP == 0 || nP == n) return S4G_OK;
  std::vector<QuadArgs> args((size_t)B);
  int maxDepth = 0;
  for (int b = 0; b < B; ++b) {
    int depth = 0;
    float bx[12];
    for (int k = 0; k < 4; ++k)
      for (int c = 0; c < 3; ++c) bx[3 * k + c] = bases[b].base_p[k][c];
    S4G_TRY(make_quad_args(ctx, bases[b].invariant1, bases[b].invariant2, thr2, bx, args[(size_t)b], depth));
    maxDepth = std::max(maxDepth, depth);
  }
  if (3 * maxDepth + 9 + 1 > kBatchSegShift) { ctx->err = "s4g_try_bases: distance_threshold2 / ratio too small for the batched quad keys"; return S4G_ERR_ARG; }
  const unsigned long long* pkeys = ctx->bPairKeys[1].as<unsigned long long>();
  S4G_TRY(s4g_reserve(ctx, ctx->bArgs, std::max<size_t>(args.size() * sizeof(QuadArgs), 64 * 1024)));
  S4G_TRY(s4g_reserve(ctx, ctx->bMisc, 4096));
  uint32_t* d_segOff = ctx->bMisc.as<uint32_t>();                 // [0 .. 2B]: segment offsets, [256 ..]: quad offsets, [512]: error flag,
                                                                   // [520, 522): 64-bit quad total
  uint32_t* d_quadOff = d_segOff + 256;
  uint32_t* d_err = d_segOff + 512;
  S4G_CUDA(cudaMemcpyAsync(ctx->bArgs.p, args.data(), args.size() * sizeof(QuadArgs), cudaMemcpyHostToDevice, st));
  S4G_CUDA(cudaMemcpyAsync(d_segOff, bh.segOff, (size_t)(2 * B + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  S4G_CUDA(cudaMemsetAsync(d_err, 0, 4, st));
  for (int k = 0; k < 2; ++k) {
    S4G_TRY(s4g_reserve(ctx, ctx->bQKeys[k], (size_t)n * sizeof(unsigned long long)));
    S4G_TRY(s4g_reserve(ctx, ctx->bQVals[k], (size_t)n * sizeof(uint32_t)));
  }
  S4G_TRY(s4g_reserve(ctx, ctx->bQCnt, (size_t)(2 * (n + 1)) * sizeof(uint32_t)));
  const QuadArgs* d_args = ctx->bArgs.as<QuadArgs>();
  unsigned long long* keys_in = ctx->bQKeys[0].as<unsigned long long>();
  unsigned long long* keys = ctx->bQKeys[1].as<unsigned long long>();
  uint32_t* vals_in = ctx->bQVals[0].as<uint32_t>();
  uint32_t* vals = ctx->bQVals[1].as<uint32_t>();
  uint32_t* counts = ctx->bQCnt.as<uint32_t>();
  uint32_t* offsets = counts + (n + 1);
  S4G_EV_START(ctx, S4G_EV_QUADS);
  k_bquad_keys<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_args, ctx->dQunit.as<float4>(), pkeys, n, d_segOff, keys_in, vals_in, d_err);
  int baseBits = 1;
  while ((1 << baseBits) < B) ++baseBits;
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, keys_in, keys, vals_in, vals, n, 0, 64, st);
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, cub_bytes));
  cub::DeviceRadixSort::SortPairs(ctx->dCub.p, cub_bytes, keys_in, keys, vals_in, vals, n, 0, 64, st);   // (padding keys = ~0 sort last)
  S4G_CUDA(cudaMemsetAsync(counts, 0, (size_t)(n + 1) * sizeof(uint32_t), st));
  k_bquad_query<false><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(d_args, ctx->dQunit.as<float4>(), ctx->dQ.as<float4>(), pkeys, n,
                                                                  d_segOff, keys, vals, nP, counts, nullptr, nullptr);
  size_t scan_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, counts, offsets, (long long)(n + 1), st);
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, scan_bytes));
  cub::DeviceScan::ExclusiveSum(ctx->dCub.p, scan_bytes, counts, offsets, (long long)(n + 1), st);
  k_bquad_offsets<<<1, 128, 0, st>>>(offsets, d_segOff, B, n, d_quadOff);
  // the 32-bit offsets wrap once the batch has 2^32 quads: their total is summed again in 64 bits
  unsigned long long* d_total = reinterpret_cast<unsigned long long*>(d_segOff + 520);
  size_t sum_bytes = 0;
  cub::DeviceReduce::Sum(nullptr, sum_bytes, counts, d_total, n, st);
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, sum_bytes));
  cub::DeviceReduce::Sum(ctx->dCub.p, sum_bytes, counts, d_total, n, st);
  ctx->launches += 7;
  S4G_CUDA(cudaGetLastError());
  uint32_t herr = 0;
  unsigned long long total = 0;
  S4G_CUDA(cudaMemcpyAsync(bh.quadOff, d_quadOff, (size_t)(B + 1) * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaMemcpyAsync(&herr, d_err, 4, cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaMemcpyAsync(&total, d_total, sizeof total, cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));                              // read-back 2 of 3
  if (herr) { ctx->err = "s4g_try_bases: internal error (quad cell key exceeds 52 bits)"; return S4G_ERR_CUDA; }
  if (total >= (1ull << 31)) { ctx->err = "s4g_try_bases: more than 2^31-1 quads in one batch"; return S4G_ERR_NOMEM; }
  bh.nQuads = total;
  if (total == 0) {
    S4G_EV_STOP(ctx, S4G_EV_QUADS);
    return S4G_OK;
  }
  for (int k = 0; k < 2; ++k) S4G_TRY(s4g_reserve(ctx, ctx->bQuadKeys[k], (size_t)total * sizeof(unsigned long long)));
  S4G_TRY(s4g_reserve(ctx, ctx->bQuads, (size_t)total * sizeof(int4)));
  unsigned long long* qk_in = ctx->bQuadKeys[0].as<unsigned long long>();
  unsigned long long* qk = ctx->bQuadKeys[1].as<unsigned long long>();
  k_bquad_query<true><<<(unsigned)((n + 127) / 128), 128, 0, st>>>(d_args, ctx->dQunit.as<float4>(), ctx->dQ.as<float4>(), pkeys, n,
                                                                 d_segOff, keys, vals, nP, nullptr, offsets, qk_in);
  cub_bytes = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, cub_bytes, qk_in, qk, (long long)total, 0, kBatchSegShift + baseBits, st);
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, cub_bytes));
  cub::DeviceRadixSort::SortKeys(ctx->dCub.p, cub_bytes, qk_in, qk, (long long)total, 0, kBatchSegShift + baseBits, st);
  k_bquad_emit<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(qk, (long long)total, pkeys, d_segOff, ctx->bQuads.as<int4>());
  S4G_EV_STOP(ctx, S4G_EV_QUADS);
  ctx->launches += 3;
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;                      // quads: ctx->bQuads, their (base, id, i) keys: ctx->bQuadKeys[1]
}

extern "C" int s4g_get_quads(s4g_ctx* ctx, int32_t* out_quads) {
  if (!ctx) return S4G_ERR_ARG;
  if (ctx->nQuads == 0) return S4G_OK;
  if (!out_quads) { ctx->err = "s4g_get_quads: null output"; return S4G_ERR_ARG; }
  S4G_CUDA(cudaSetDevice(ctx->device));
  S4G_CUDA(cudaMemcpyAsync(out_quads, ctx->dQuads.p, (size_t)ctx->nQuads * sizeof(int4), cudaMemcpyDeviceToHost, ctx->stream));
  S4G_CUDA(cudaStreamSynchronize(ctx->stream));
  return S4G_OK;
}
