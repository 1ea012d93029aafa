// FPFH point descriptors on the resident P (s4g_fpfh, include/s4g.h; Rusu et al. 2009, Open3D's compute_fpfh_feature)
// and the nearest-descriptor search between two descriptor arrays (s4g_fpfh_match).
//
// Rows.  The P points go to the existing k_knn instances (query.cu) in the grid's sorted order
// (s4g_launch_sorted_queries, as outliers.cu), each excluding its own original index (s4g_launch_exclude_self), no T,
// the caller's k and sq_radius, with d^2.  Row t belongs to sorted point t of original index j = GridDev::pts[t].w: it is
// the s4g_knn row of p_j with exclude = j, in ascending (d^2, index), padded at its end.
//
// k_fpfh_spfh, one thread per sorted point t: the entries of j's row that have a normal, in row order; for each the
// pair feature of (p_j, n_j) and (p_e, n_e) in double, its three bins, and the counts cnt_j[33] (at most 64 each, k <= 64)
// with m_j, the number of such entries, stored as 36 bytes per original index j (byte 33 = m_j).  The counts are integers
// and each thread writes only its own j, so they do not depend on the order in which threads run.
//
// k_fpfh_gather, one thread per sorted point t with 33 double accumulators in registers (the bins fully unrolled): over
// the row's entries e with a normal and d^2_e > 0, in row order from 0.0, acc[b] = acc[b] + ((100.0 cnt_e[b]) / m_e) /
// d^2_e; then S_h per block of 11 bins left to right and fpfh[j][b] = (float)(acc[b] (100.0 / S_h) + spfh_j[b]).  The
// sums run in the row's order, which k_knn fixes (its lexicographic k-minimum does not depend on the search order).  A
// neighbour whose SPFH is zero (m_e = 0, or no normal) adds +0.0 to each acc, which changes no bit, so leaving it out and
// taking it in agree.
//
// Determinism.  Every value is made of IEEE basic operations (+ - * /, sqrt, floor, compares) in double, each written in
// a fixed order, compiled with -fmad=false so that no product is contracted into an FMA; the f1 bin is decided by exact
// half-plane tests against tabulated directions instead of a rounded atan2.  A CPU restatement of the same operations
// compiled without contraction (-ffp-contract=off) gives the same bits.
//
// Match.  k_fpfh_nearest: a CTA holds kMatchRows rows of X per thread in registers and walks a range of Y in tiles of
// kMatchTile rows staged in shared memory, ascending; the squared distance is summed in fp32 over c = 0..32 left to right
// from 0.0f, s = s + (x_c - y_c) (x_c - y_c), and a strictly smaller finite s replaces the thread's best, so a NaN never
// wins and ties keep the smaller index.  Each CTA posts its best (bits(d^2) << 32 | index) by a 64-bit atomicMin: the
// bits of a finite non-negative float order as its value, so the minimum is the lexicographically smallest (d^2, index)
// whatever the order of the posts.  k_fpfh_match_out turns the keys into index / sq_dist, and with `mutual` keeps
// index[i] only when the B -> A key of index[i] names i.
#include "s4g_internal.cuh"
#include <algorithm>
#include <cmath>

namespace {

constexpr int kThreads = 128;
constexpr int kMaxK = 64;                // k_knn's widest instance
constexpr int kBins = 33;
constexpr int kCountWords = 9;           // 33 one-byte counts and m_j (byte 33) per point
constexpr int kMatchThreads = 128;
constexpr int kMatchRows = 4;            // X rows per thread
constexpr int kMatchTile = 64;           // Y rows per shared-memory tile
constexpr int kMatchStride = 36;         // floats per staged Y row (33 and zero padding, 16-byte aligned)
constexpr unsigned long long kNoMatch = ~0ull;

unsigned nblk(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }
size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// cos and sin of beta_i = -pi + 2 pi i / 11, i = 1..5, correctly rounded; c_{11-i} = c_i, s_{11-i} = -s_i
__device__ __constant__ double kFaceC[5] = {-0x1.aeb8c8764f0bap-1, -0x1.a9628d9c712b6p-2, 0x1.2375f640f44dbp-3,
                                            0x1.4f49e7f775887p-1, 0x1.eb42a9bcd5057p-1};
__device__ __constant__ double kFaceS[5] = {-0x1.14cedf8bb580bp-1, -0x1.d1bb48eee2c13p-1, -0x1.fac9e043842efp-1,
                                            -0x1.82f19bb3a28a1p-1, -0x1.207e7fd768dbfp-2};

struct D3 {
  double x, y, z;
};
__device__ __forceinline__ double dot3(D3 a, D3 b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a.x, b.x), __dmul_rn(a.y, b.y)), __dmul_rn(a.z, b.z));
}
__device__ __forceinline__ D3 cross3(D3 a, D3 b) {
  return D3{__dsub_rn(__dmul_rn(a.y, b.z), __dmul_rn(a.z, b.y)), __dsub_rn(__dmul_rn(a.z, b.x), __dmul_rn(a.x, b.z)),
            __dsub_rn(__dmul_rn(a.x, b.y), __dmul_rn(a.y, b.x))};
}

// the normal of point j in double, divided by its length; false: no normal ((0, 0, 0) or a non-finite component)
__device__ __forceinline__ bool unit_normal(const float* __restrict__ nrm, long long j, D3& n) {
  const float x = __ldg(&nrm[3 * j]), y = __ldg(&nrm[3 * j + 1]), z = __ldg(&nrm[3 * j + 2]);
  if (!isfinite(x) || !isfinite(y) || !isfinite(z) || (x == 0.f && y == 0.f && z == 0.f)) return false;
  n = D3{(double)x, (double)y, (double)z};
  const double l = __dsqrt_rn(dot3(n, n));
  n = D3{__ddiv_rn(n.x, l), __ddiv_rn(n.y, l), __ddiv_rn(n.z, l)};
  return true;
}

// floor(11 (f + 1.0) 0.5) clamped to [0, 10]
__device__ __forceinline__ int bin_of(double f) {
  const double h = floor(__dmul_rn(__dmul_rn(11.0, __dadd_rn(f, 1.0)), 0.5));
  return h < 0.0 ? 0 : h > 10.0 ? 10 : (int)h;
}

// the bin of floor(11 (atan2(y, x) + pi) / 2 pi) by exact half-plane tests: c_i y - s_i x >= 0
__device__ __forceinline__ int angle_bin(double x, double y) {
  if (y == 0.0) return x < 0.0 ? 10 : 5;
  int b = 0;
  if (y > 0.0) {
#pragma unroll
    for (int i = 6; i <= 10; ++i) b += __dsub_rn(__dmul_rn(kFaceC[10 - i], y), __dmul_rn(-kFaceS[10 - i], x)) >= 0.0;
    return 5 + b;
  }
#pragma unroll
  for (int i = 1; i <= 5; ++i) b += __dsub_rn(__dmul_rn(kFaceC[i - 1], y), __dmul_rn(kFaceS[i - 1], x)) >= 0.0;
  return b;
}

// the three bins (f1, 11 + f2, 22 + f3) of the pair (p1, n1), (p2, n2): Open3D's ComputePairFeatures with exact decisions
__device__ __forceinline__ void pair_bins(D3 p1, D3 n1, D3 p2, D3 n2, int& b1, int& b2, int& b3) {
  D3 dp{__dsub_rn(p2.x, p1.x), __dsub_rn(p2.y, p1.y), __dsub_rn(p2.z, p1.z)};
  b1 = 5;
  b2 = 16;
  b3 = 27;
  const double d = __dsqrt_rn(dot3(dp, dp));
  if (d == 0.0) return;
  const double a1 = __ddiv_rn(dot3(n1, dp), d), a2 = __ddiv_rn(dot3(n2, dp), d);
  D3 u = n1, np = n2;
  double f3 = a1;
  if (fabs(a1) < fabs(a2)) {
    u = n2;
    np = n1;
    dp = D3{-dp.x, -dp.y, -dp.z};
    f3 = -a2;
  }
  D3 v = cross3(dp, u);
  const double vn = __dsqrt_rn(dot3(v, v));
  if (vn == 0.0) return;
  v = D3{__ddiv_rn(v.x, vn), __ddiv_rn(v.y, vn), __ddiv_rn(v.z, vn)};
  const D3 w = cross3(u, v);
  b1 = angle_bin(dot3(u, np), dot3(w, np));
  b2 = 11 + bin_of(dot3(v, np));
  b3 = 22 + bin_of(f3);
}

__device__ __forceinline__ D3 point_of(const float4* __restrict__ P, long long j) {
  const float4 p = __ldg(&P[j]);
  return D3{(double)p.x, (double)p.y, (double)p.z};
}

// counts[j]: the SPFH bin counts and m_j of original index j (bytes; byte 33 = m_j)
__global__ void __launch_bounds__(kThreads)
k_fpfh_spfh(const float4* __restrict__ sorted, const float4* __restrict__ P, const int32_t* __restrict__ index, int n,
            int k, const float* __restrict__ nrm, uint32_t* __restrict__ counts) {
  __shared__ uint8_t cnt[kCountWords * 4][kThreads];
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
#pragma unroll
  for (int b = 0; b < kCountWords * 4; ++b) cnt[b][threadIdx.x] = 0;
  const long long j = __float_as_int(__ldg(&sorted[t]).w);
  D3 n1;
  int m = 0;
  if (unit_normal(nrm, j, n1)) {
    const D3 p1 = point_of(P, j);
    const long long row = t * (long long)k;
#pragma unroll 1
    for (int e = 0; e < k; ++e) {
      const int i = __ldg(&index[row + e]);
      if (i < 0) break;
      D3 n2;
      if (!unit_normal(nrm, i, n2)) continue;
      int b1, b2, b3;
      pair_bins(p1, n1, point_of(P, i), n2, b1, b2, b3);
      cnt[b1][threadIdx.x]++;
      cnt[b2][threadIdx.x]++;
      cnt[b3][threadIdx.x]++;
      ++m;
    }
  }
  cnt[kBins][threadIdx.x] = (uint8_t)m;
  uint32_t* out = counts + j * kCountWords;
#pragma unroll
  for (int w = 0; w < kCountWords; ++w)
    out[w] = (uint32_t)cnt[4 * w][threadIdx.x] | ((uint32_t)cnt[4 * w + 1][threadIdx.x] << 8) |
             ((uint32_t)cnt[4 * w + 2][threadIdx.x] << 16) | ((uint32_t)cnt[4 * w + 3][threadIdx.x] << 24);
}

__device__ __forceinline__ void load_counts(const uint32_t* __restrict__ counts, long long j, uint32_t (&c)[kCountWords]) {
#pragma unroll
  for (int w = 0; w < kCountWords; ++w) c[w] = __ldg(&counts[j * kCountWords + w]);
}
__device__ __forceinline__ uint32_t count_of(const uint32_t (&c)[kCountWords], int b) { return (c[b >> 2] >> (8 * (b & 3))) & 0xFFu; }

__global__ void __launch_bounds__(kThreads)
k_fpfh_gather(const float4* __restrict__ sorted, const int32_t* __restrict__ index, const float* __restrict__ sq, int n,
              int k, const float* __restrict__ nrm, const uint32_t* __restrict__ counts, float* __restrict__ fpfh) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const long long j = __float_as_int(__ldg(&sorted[t]).w);
  float* out = fpfh + j * kBins;
  D3 nj;
  if (!unit_normal(nrm, j, nj)) {
#pragma unroll
    for (int b = 0; b < kBins; ++b) out[b] = 0.f;
    return;
  }
  double acc[kBins];
#pragma unroll
  for (int b = 0; b < kBins; ++b) acc[b] = 0.0;
  const long long row = t * (long long)k;
#pragma unroll 1
  for (int e = 0; e < k; ++e) {
    const int i = __ldg(&index[row + e]);
    if (i < 0) break;
    const double d2 = (double)__ldg(&sq[row + e]);
    if (!(d2 > 0.0)) continue;
    uint32_t c[kCountWords];
    load_counts(counts, i, c);
    const uint32_t m = count_of(c, kBins);
    if (m == 0) continue;                 // no normal, or no neighbour with one: the SPFH is zero
    const double dm = (double)m;
#pragma unroll
    for (int b = 0; b < kBins; ++b) {
      const uint32_t cb = count_of(c, b);
      if (cb != 0) acc[b] = __dadd_rn(acc[b], __ddiv_rn(__ddiv_rn(__dmul_rn(100.0, (double)cb), dm), d2));
    }
  }
  uint32_t c[kCountWords];
  load_counts(counts, j, c);
  const uint32_t m = count_of(c, kBins);
#pragma unroll
  for (int h = 0; h < 3; ++h) {
    double s = acc[11 * h];
#pragma unroll
    for (int b = 1; b < 11; ++b) s = __dadd_rn(s, acc[11 * h + b]);
    const double scale = s != 0.0 ? __ddiv_rn(100.0, s) : 0.0;
#pragma unroll
    for (int b = 11 * h; b < 11 * h + 11; ++b) {
      const double own = m != 0 ? __ddiv_rn(__dmul_rn(100.0, (double)count_of(c, b)), (double)m) : 0.0;
      out[b] = (float)(s != 0.0 ? __dadd_rn(__dmul_rn(acc[b], scale), own) : own);
    }
  }
}

// keys[i] = min over the Y rows of this CTA's range of (bits(d^2) << 32 | index), finite d^2 only (atomicMin)
__global__ void __launch_bounds__(kMatchThreads)
k_fpfh_nearest(const float* __restrict__ X, int nx, const float* __restrict__ Y, int ny, int tiles_per_cta,
               unsigned long long* __restrict__ keys) {
  __shared__ __align__(16) float ys[kMatchTile * kMatchStride];
  float x[kMatchRows][kBins];
  const long long base = ((long long)blockIdx.x * kMatchThreads + threadIdx.x) * kMatchRows;
#pragma unroll
  for (int r = 0; r < kMatchRows; ++r) {
    const long long i = min(base + r, (long long)nx - 1);
#pragma unroll
    for (int c = 0; c < kBins; ++c) x[r][c] = __ldg(&X[i * kBins + c]);
  }
  float best[kMatchRows];
  int bj[kMatchRows];
#pragma unroll
  for (int r = 0; r < kMatchRows; ++r) {
    best[r] = INFINITY;
    bj[r] = -1;
  }
  const long long tile0 = (long long)blockIdx.y * tiles_per_cta;
#pragma unroll 1
  for (long long tile = tile0; tile < tile0 + tiles_per_cta; ++tile) {
    const long long y0 = tile * kMatchTile;
    if (y0 >= ny) break;
    const int rows = (int)min((long long)kMatchTile, (long long)ny - y0);
    __syncthreads();
    for (int f = threadIdx.x; f < kMatchTile * kMatchStride; f += kMatchThreads) {
      const int r = f / kMatchStride, c = f - r * kMatchStride;
      ys[f] = (r < rows && c < kBins) ? __ldg(&Y[(y0 + r) * kBins + c]) : 0.f;
    }
    __syncthreads();
#pragma unroll 1
    for (int r = 0; r < rows; ++r) {
      const float4* yr = reinterpret_cast<const float4*>(ys + r * kMatchStride);
      float s[kMatchRows];
#pragma unroll
      for (int q = 0; q < kMatchRows; ++q) s[q] = 0.f;
#pragma unroll
      for (int w = 0; w < kMatchStride / 4; ++w) {
        const float4 v = yr[w];
        const float yv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int l = 0; l < 4; ++l) {
          const int c = 4 * w + l;
          if (c < kBins) {
#pragma unroll
            for (int q = 0; q < kMatchRows; ++q) {
              const float d = __fsub_rn(x[q][c], yv[l]);
              s[q] = __fadd_rn(s[q], __fmul_rn(d, d));
            }
          }
        }
      }
#pragma unroll
      for (int q = 0; q < kMatchRows; ++q)
        if (s[q] < best[q]) {
          best[q] = s[q];
          bj[q] = (int)(y0 + r);
        }
    }
  }
#pragma unroll
  for (int r = 0; r < kMatchRows; ++r)
    if (base + r < nx && bj[r] >= 0)
      atomicMin(&keys[base + r], ((unsigned long long)__float_as_uint(best[r]) << 32) | (uint32_t)bj[r]);
}

__device__ __forceinline__ int key_index(unsigned long long key) { return key == kNoMatch ? -1 : (int)(uint32_t)key; }

__global__ void __launch_bounds__(kThreads)
k_fpfh_match_out(const unsigned long long* __restrict__ ab, int na, const unsigned long long* __restrict__ ba,
                 int32_t* __restrict__ index, float* __restrict__ sq_dist) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= na) return;
  const unsigned long long key = ab[i];
  int j = key_index(key);
  if (ba != nullptr && j >= 0 && key_index(ba[j]) != (int)i) j = -1;
  index[i] = j;
  if (sq_dist != nullptr) sq_dist[i] = key == kNoMatch ? INFINITY : __uint_as_float((uint32_t)(key >> 32));
}

int fpfh_args(s4g_ctx* ctx, const char* who, const void* normals, int k, float sq_radius, const void* fpfh) {
  if (k < 1 || k > kMaxK || std::isnan(sq_radius) || sq_radius < 0.f || normals == nullptr || fpfh == nullptr) {
    ctx->err = std::string(who) + ": bad arguments (1 <= k <= 64, sq_radius >= 0 and not NaN, normals and fpfh != NULL)";
    return S4G_ERR_ARG;
  }
  if (ctx->nP <= 0) {
    ctx->err = std::string(who) + ": call s4g_set_cloud_p first";
    return S4G_ERR_STATE;
  }
  return S4G_OK;
}

// enqueue the descriptors on the context's stream.  Scratch A: the sorted queries (12 bytes per point); B / C: the rows
// (index, d^2; 4k bytes each); D: the exclusion list, then the counts (36 bytes per point)
int launch_fpfh(s4g_ctx* ctx, const float* d_normals, int k, float sq_radius, float* d_fpfh) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  const int n = ctx->nP;
  const size_t N = (size_t)n;
  cudaStream_t st = ctx->stream;
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, N * 3 * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, N * (size_t)k * sizeof(int32_t)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchC, N * (size_t)k * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchD, N * kCountWords * sizeof(uint32_t)));
  int32_t* rows = ctx->dScratchB.as<int32_t>();
  float* sq = ctx->dScratchC.as<float>();
  uint32_t* counts = ctx->dScratchD.as<uint32_t>();   // written once the rows (and so the exclusion list) are consumed
  S4G_TRY(s4g_launch_sorted_queries(ctx, ctx->dScratchA.as<float>()));
  S4G_TRY(s4g_launch_exclude_self(ctx, ctx->dScratchD.as<int32_t>()));
  S4G_TRY(s4g_launch_knn(ctx, ctx->dScratchA.as<float>(), n, nullptr, k, sq_radius, ctx->dScratchD.as<int32_t>(), rows,
                         sq, nullptr));
  k_fpfh_spfh<<<nblk(n, kThreads), kThreads, 0, st>>>(ctx->grid.pts, ctx->dP.as<float4>(), rows, n, k, d_normals, counts);
  k_fpfh_gather<<<nblk(n, kThreads), kThreads, 0, st>>>(ctx->grid.pts, rows, sq, n, k, d_normals, counts, d_fpfh);
  ctx->launches += 2;
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;
}

int match_args(s4g_ctx* ctx, const char* who, const void* a, int64_t na, const void* b, int64_t nb, const void* index) {
  if (na < 0 || nb < 0 || na > INT32_MAX || nb > INT32_MAX || (na > 0 && (a == nullptr || index == nullptr)) ||
      (nb > 0 && na > 0 && b == nullptr)) {
    ctx->err = std::string(who) + ": bad arguments (0 <= n_a, n_b < 2^31, a, b and index != NULL)";
    return S4G_ERR_ARG;
  }
  return S4G_OK;
}

// keys[i] for every X row: the nearest Y row (X, Y device arrays; nx > 0)
int launch_nearest(s4g_ctx* ctx, const float* X, int nx, const float* Y, int ny, unsigned long long* keys) {
  cudaStream_t st = ctx->stream;
  S4G_CUDA(cudaMemsetAsync(keys, 0xFF, (size_t)nx * sizeof(unsigned long long), st));
  if (ny == 0) return S4G_OK;
  const unsigned gx = nblk(nx, kMatchThreads * kMatchRows);
  const long long tiles = (ny + kMatchTile - 1) / kMatchTile;
  // split Y so that about 8 CTAs per SM run; each CTA walks a contiguous range of tiles
  const long long want = std::max(1ll, (8ll * ctx->sm_count + gx - 1) / gx);
  const long long split = std::min(tiles, std::min(want, 65535ll));
  const int per = (int)((tiles + split - 1) / split);
  const unsigned gy = (unsigned)((tiles + per - 1) / per);
  k_fpfh_nearest<<<dim3(gx, gy), kMatchThreads, 0, st>>>(X, nx, Y, ny, per, keys);
  ctx->launches += 2;
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;
}

// enqueue the match on the context's stream.  Scratch A: the A -> B keys (8 bytes per A row), then the B -> A keys
// (8 bytes per B row) when mutual
int launch_match(s4g_ctx* ctx, const float* d_a, int na, const float* d_b, int nb, int mutual, int32_t* d_index,
                 float* d_sq_dist) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  const bool mut = mutual != 0 && nb > 0;
  const size_t ka = align256((size_t)na * 8);
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, ka + (mut ? (size_t)nb * 8 : 0)));
  unsigned long long* ab = ctx->dScratchA.as<unsigned long long>();
  unsigned long long* ba = mut ? reinterpret_cast<unsigned long long*>(ctx->dScratchA.as<char>() + ka) : nullptr;
  S4G_TRY(launch_nearest(ctx, d_a, na, d_b, nb, ab));
  if (mut) S4G_TRY(launch_nearest(ctx, d_b, nb, d_a, na, ba));
  k_fpfh_match_out<<<nblk(na, kThreads), kThreads, 0, ctx->stream>>>(ab, na, ba, d_index, d_sq_dist);
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;
}

}  // namespace

extern "C" int s4g_fpfh_dev(s4g_ctx* ctx, const float* d_normals, int k, float sq_radius, float* d_fpfh) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(fpfh_args(ctx, "s4g_fpfh_dev", d_normals, k, sq_radius, d_fpfh));
  return launch_fpfh(ctx, d_normals, k, sq_radius, d_fpfh);
}

// the device copies in ctx->dFilter: normals, then the descriptors
extern "C" int s4g_fpfh(s4g_ctx* ctx, const float* normals, int k, float sq_radius, float* fpfh) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(fpfh_args(ctx, "s4g_fpfh", normals, k, sq_radius, fpfh));
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t N = (size_t)ctx->nP, a3 = align256(12 * N);
  S4G_TRY(s4g_reserve(ctx, ctx->dFilter, a3 + 4 * kBins * N));
  float* d_n = ctx->dFilter.as<float>();
  float* d_f = reinterpret_cast<float*>(ctx->dFilter.as<char>() + a3);
  S4G_CUDA(cudaMemcpyAsync(d_n, normals, 12 * N, cudaMemcpyHostToDevice, st));
  S4G_TRY(launch_fpfh(ctx, d_n, k, sq_radius, d_f));
  S4G_CUDA(cudaMemcpyAsync(fpfh, d_f, 4 * kBins * N, cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  return S4G_OK;
}

extern "C" int s4g_fpfh_match_dev(s4g_ctx* ctx, const float* d_a, int64_t n_a, const float* d_b, int64_t n_b, int mutual,
                                  int32_t* d_index, float* d_sq_dist) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(match_args(ctx, "s4g_fpfh_match_dev", d_a, n_a, d_b, n_b, d_index));
  if (n_a == 0) return S4G_OK;
  return launch_match(ctx, d_a, (int)n_a, d_b, (int)n_b, mutual, d_index, d_sq_dist);
}

// the device copies in ctx->dFilter: a, b, index, sq_dist
extern "C" int s4g_fpfh_match(s4g_ctx* ctx, const float* a, int64_t n_a, const float* b, int64_t n_b, int mutual,
                              int32_t* index, float* sq_dist) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(match_args(ctx, "s4g_fpfh_match", a, n_a, b, n_b, index));
  if (n_a == 0) return S4G_OK;
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t NA = (size_t)n_a, NB = (size_t)n_b;
  const size_t fa = align256(4 * kBins * NA), fb = align256(4 * kBins * NB), fi = align256(4 * NA);
  S4G_TRY(s4g_reserve(ctx, ctx->dFilter, fa + fb + fi + 4 * NA));
  char* p = ctx->dFilter.as<char>();
  float* d_a = reinterpret_cast<float*>(p);
  float* d_b = reinterpret_cast<float*>(p + fa);
  int32_t* d_i = reinterpret_cast<int32_t*>(p + fa + fb);
  float* d_s = reinterpret_cast<float*>(p + fa + fb + fi);
  S4G_CUDA(cudaMemcpyAsync(d_a, a, 4 * kBins * NA, cudaMemcpyHostToDevice, st));
  if (NB > 0) S4G_CUDA(cudaMemcpyAsync(d_b, b, 4 * kBins * NB, cudaMemcpyHostToDevice, st));
  S4G_TRY(launch_match(ctx, d_a, (int)n_a, d_b, (int)n_b, mutual, d_i, d_s));
  S4G_CUDA(cudaMemcpyAsync(index, d_i, 4 * NA, cudaMemcpyDeviceToHost, st));
  if (sq_dist != nullptr) S4G_CUDA(cudaMemcpyAsync(sq_dist, d_s, 4 * NA, cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  return S4G_OK;
}
