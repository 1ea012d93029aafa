// Plane segmentation of the resident P (s4g_segment_planes, include/s4g.h): RANSAC with every hypothesis counted
// exactly, the winner refitted by least squares, several planes in turn.
//
// Each round r is one fixed chain of launches on the context's stream, and the host never waits for the device between
// them: whether a round runs is a flag in PlaneState that the device sets when a round stops, and every later kernel
// reads it first.  A round:
//   k_plane_active       flags[j] = labels[j] < 0 (no plane claimed j);
//   select + gather      cub::DeviceSelect::Flagged of the j in ascending order, then A[i] = P[j] as float4 (w = j): A_r
//                        in ascending j, contiguous for the draws and the scan; m = |A_r| on the device;
//   k_plane_hypotheses   one thread per h: the three SplitMix64 draws and the plane in double, rounded to float; an
//                        invalid plane is stored as NaN, whose test is false for every point, so it counts 0 with no
//                        branch in the count;
//   k_plane_count        the hot path: H x m tests.  A CTA of kCountThreads threads holds kHypPerThread planes per thread
//                        in registers and walks a slice of A_r through shared memory, kPointTile points at a time, every
//                        lane reading the same point (a broadcast); counters in registers, one integer atomicAdd per
//                        (CTA, hypothesis) at the end.  The grid is hypothesis tiles x point slices, the slices cut from
//                        the device's m;
//   k_plane_argmax       the largest packed key (count << 32) | (0xFFFFFFFF - h) over the valid h: the largest count, ties
//                        to the smallest h (Verify's key); key 0: no valid hypothesis, stop;
//   k_plane_inliers      flags[i] = A_r[i] passes the winner's test; cub::DeviceSelect::Flagged gives I in ascending j;
//   k_plane_runs / k_plane_centroid / k_plane_runs / k_plane_refit
//                        the refit's two fixed-order passes (runs of kRun, one thread per component, then the run sums)
//                        and a single-thread finish: Jacobi (jacobi.cuh, shared with k_normals), the column rule, the sign
//                        rule, d.  Without refine only k_plane_refit runs, and keeps the hypothesis;
//   k_plane_final        the final test over A_r, counted by __syncthreads_count and one atomicAdd per CTA;
//   k_plane_accept       one thread: the plane's record, offsets[r + 1], *n_planes -- or stop;
//   k_plane_label        labels[j] = r for the final inliers of an accepted plane.
// After the rounds, the members are a stable radix sort of (label, j) with j entering in ascending order.
//
// Determinism.  The draws are integer arithmetic; the hypothesis planes and the refit are IEEE basic operations in double
// (+ - * /, sqrt, fabs, compares) in a stated order, compiled with -fmad=false; the test is fp32 with explicit _rn
// operations; the counts are integer sums; every sum of the refit runs in a fixed order; the selects and the sort are
// stable.  Nothing depends on the schedule, so a CPU restatement compiled without contraction (-ffp-contract=off) gives
// the same bits.
#include "s4g_internal.cuh"
#include "jacobi.cuh"
#include <cub/cub.cuh>
#include <algorithm>
#include <cmath>

namespace {

constexpr int kMaxHypotheses = 1 << 20;
constexpr int kThreads = 256;
constexpr int kCountThreads = 128;                                 // threads of a k_plane_count CTA
constexpr int kHypPerThread = 4;                                   // planes held per thread
constexpr int kHypTile = kCountThreads * kHypPerThread;            // hypotheses per CTA
constexpr int kPointTile = 1024;                                   // points staged per step (16 KiB)
constexpr int kCountCtasPerSm = 8;                                 // the grid's target, in CTAs per SM
constexpr int kRun = 1024;                                         // points per run of the refit's fixed-order sums
constexpr int kRunThreads = 128;                                   // threads staging one run
constexpr int kMoments = 6;                                        // C00 C01 C02 C11 C12 C22

// the device state of one call
struct PlaneState {
  long long m;                // |A_r| (the select's count)
  long long n_inl;            // |I|
  unsigned long long key;     // the winner's packed key
  unsigned long long final_count;
  long long total;            // the members of the accepted planes so far
  double c[3];                // the refit's centroid
  float4 plane;               // the round's final coefficients
  int stop;                   // 1: a round stopped; every later kernel returns at once
  int n_planes;
};

unsigned nblk(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

int key_bits(long long n) {
  int b = 1;
  while (b < 31 && ((long long)1 << b) <= n) ++b;
  return b;
}

// r = ((a x + b y) + c z) + d in fp32, each operation rounded on its own
__device__ __forceinline__ float plane_residual(float4 pl, float4 p) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(pl.x, p.x), __fmul_rn(pl.y, p.y)), __fmul_rn(pl.z, p.z)), pl.w);
}

__device__ __forceinline__ bool plane_inlier(float4 pl, float4 p, float threshold) {
  return fabsf(plane_residual(pl, p)) < threshold;
}

// the SplitMix64 output of index k of a stream seeded with s
__device__ __forceinline__ unsigned long long splitmix64(unsigned long long s, unsigned long long k) {
  unsigned long long z = s + k * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// n normalised in double, the component of largest magnitude made positive (ties to the lowest axis), d = -n.p, rounded
__device__ __forceinline__ float4 plane_round(double nx, double ny, double nz, double len, double px, double py, double pz) {
  nx = nx / len;
  ny = ny / len;
  nz = nz / len;
  double big = nx;
  if (fabs(ny) > fabs(big)) big = ny;
  if (fabs(nz) > fabs(big)) big = nz;
  if (big < 0.0) {
    nx = -nx;
    ny = -ny;
    nz = -nz;
  }
  const double d = -((nx * px + ny * py) + nz * pz);
  return make_float4((float)nx, (float)ny, (float)nz, (float)d);
}

__global__ void k_plane_active(const int32_t* __restrict__ labels, int n, const PlaneState* __restrict__ st,
                               uint8_t* __restrict__ flags) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  flags[j] = (!st->stop && labels[j] < 0) ? 1 : 0;
}

__global__ void k_plane_gather(const float4* __restrict__ P, const int32_t* __restrict__ act, int n,
                               const PlaneState* __restrict__ st, float4* __restrict__ A) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || i >= st->m) return;
  A[i] = P[act[i]];
}

// planes[h] (NaN when invalid) and samples[h] = (j0, j1, j2, valid)
__global__ void k_plane_hypotheses(const float4* __restrict__ A, const PlaneState* __restrict__ st, int H,
                                   unsigned long long seed_r, float4* __restrict__ planes, int4* __restrict__ samples) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= H || st->stop) return;
  const long long m = st->m;
  float4 p[3];
  int j[3] = {-1, -1, -1};
  if (m >= 3) {
#pragma unroll
    for (int t = 0; t < 3; ++t) {
      const unsigned long long z = splitmix64(seed_r, 3ull * (unsigned long long)h + (unsigned long long)t + 1ull);
      const long long pos = (long long)(((z >> 32) * (unsigned long long)m) >> 32);
      p[t] = A[pos];
      j[t] = __float_as_int(p[t].w);
    }
  }
  float4 pl = make_float4(NAN, NAN, NAN, NAN);
  bool valid = false;
  if (m >= 3) {
    const double ux = (double)p[1].x - (double)p[0].x, uy = (double)p[1].y - (double)p[0].y, uz = (double)p[1].z - (double)p[0].z;
    const double vx = (double)p[2].x - (double)p[0].x, vy = (double)p[2].y - (double)p[0].y, vz = (double)p[2].z - (double)p[0].z;
    const double nx = uy * vz - uz * vy, ny = uz * vx - ux * vz, nz = ux * vy - uy * vx;
    const double len = sqrt((nx * nx + ny * ny) + nz * nz);
    if (len != 0.0) {
      pl = plane_round(nx, ny, nz, len, (double)p[0].x, (double)p[0].y, (double)p[0].z);
      valid = true;
    }
  }
  planes[h] = pl;
  samples[h] = make_int4(j[0], j[1], j[2], valid ? 1 : 0);
}

// counts[h] += the inliers of hypothesis h among the CTA's slice of A_r (blockIdx.x: the slice, blockIdx.y: the
// hypothesis tile)
__global__ void __launch_bounds__(kCountThreads)
k_plane_count(const float4* __restrict__ A, const PlaneState* __restrict__ st, const float4* __restrict__ planes, int H,
              float threshold, uint32_t* __restrict__ counts) {
  __shared__ float4 tile[kPointTile];
  if (st->stop) return;
  const long long m = st->m;
  const long long slices = gridDim.x;
  const long long per = ((m + slices - 1) / slices + kPointTile - 1) / kPointTile * kPointTile;
  const long long lo = (long long)blockIdx.x * per, hi = min(m, lo + per);
  if (lo >= hi) return;
  const int h0 = blockIdx.y * kHypTile + threadIdx.x;
  float4 pl[kHypPerThread];
  uint32_t cnt[kHypPerThread];
#pragma unroll
  for (int i = 0; i < kHypPerThread; ++i) {
    const int h = h0 + i * kCountThreads;
    pl[i] = h < H ? planes[h] : make_float4(NAN, NAN, NAN, NAN);
    cnt[i] = 0u;
  }
#pragma unroll 1
  for (long long base = lo; base < hi; base += kPointTile) {
    const int len = (int)min((long long)kPointTile, hi - base);
    __syncthreads();
    for (int t = threadIdx.x; t < len; t += kCountThreads) tile[t] = A[base + t];
    __syncthreads();
#pragma unroll 4
    for (int q = 0; q < len; ++q) {
      const float4 p = tile[q];
#pragma unroll
      for (int i = 0; i < kHypPerThread; ++i) cnt[i] += plane_inlier(pl[i], p, threshold) ? 1u : 0u;
    }
  }
#pragma unroll
  for (int i = 0; i < kHypPerThread; ++i) {
    const int h = h0 + i * kCountThreads;
    if (h < H && cnt[i] != 0u) atomicAdd(&counts[h], cnt[i]);
  }
}

// one CTA of 1024 threads: st->key = the largest packed key of the valid hypotheses; 0 -> stop
__global__ void __launch_bounds__(1024)
k_plane_argmax(const uint32_t* __restrict__ counts, const int4* __restrict__ samples, int H, PlaneState* __restrict__ st) {
  __shared__ unsigned long long warp_best[32];
  if (st->stop) return;
  unsigned long long best = 0ull;
  for (int h = threadIdx.x; h < H; h += blockDim.x)
    if (samples[h].w) best = max(best, ((unsigned long long)counts[h] << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)h));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0) warp_best[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) best = max(best, warp_best[w]);
  st->key = best;
  st->final_count = 0ull;
  if (best == 0ull) st->stop = 1;
}

__device__ __forceinline__ int winner(const PlaneState* st) { return (int)(0xFFFFFFFFu - (uint32_t)(st->key & 0xFFFFFFFFull)); }

// flags[i] = A_r[i] is an inlier of the winner, i < n (0 past m)
__global__ void k_plane_inliers(const float4* __restrict__ A, int n, const PlaneState* __restrict__ st,
                                const float4* __restrict__ planes, float threshold, uint8_t* __restrict__ flags) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  flags[i] = (!st->stop && i < st->m && plane_inlier(planes[winner(st)], A[i], threshold)) ? 1 : 0;
}

// one block per run of kRun inliers (ascending j): thread t sums component t of the run left to right from 0.0 -- the
// coordinates (first pass) or the moments (p - c)_p (p - c)_q of C (second pass, c = st->c)
__global__ void __launch_bounds__(kRunThreads)
k_plane_runs(const float4* __restrict__ I, const PlaneState* __restrict__ st, bool second, double* __restrict__ runs) {
  __shared__ float4 v[kRun];
  if (st->stop) return;
  const long long begin = (long long)blockIdx.x * kRun;
  const long long n = st->n_inl;
  if (begin >= n) return;
  const int len = (int)min((long long)kRun, n - begin);
  for (int i = threadIdx.x; i < len; i += blockDim.x) v[i] = I[begin + i];
  __syncthreads();
  const int t = threadIdx.x;
  if (t >= (second ? kMoments : 3)) return;
  double s = 0.0;
  if (!second) {
#pragma unroll 1
    for (int i = 0; i < len; ++i) s = s + (double)reinterpret_cast<const float*>(&v[i])[t];
  } else {
    const int p = t < 3 ? 0 : t < 5 ? 1 : 2;              // (0,0) (0,1) (0,2) (1,1) (1,2) (2,2)
    const int q = t < 3 ? t : t < 5 ? t - 2 : 2;
    const double cp = st->c[p], cq = st->c[q];
#pragma unroll 1
    for (int i = 0; i < len; ++i) {
      const float* x = reinterpret_cast<const float*>(&v[i]);
      const double dp = (double)x[p] - cp, dq = (double)x[q] - cq;
      s = s + dp * dq;
    }
  }
  runs[(long long)blockIdx.x * kMoments + t] = s;
}

// one thread: the run sums of the first pass left to right from 0.0 -> c = sum p / |I|
__global__ void k_plane_centroid(const double* __restrict__ runs, PlaneState* __restrict__ st) {
  if (st->stop || st->n_inl < 3) return;
  const long long n = st->n_inl;
  const int n_runs = (int)((n + kRun - 1) / kRun);
  double s[3] = {0.0, 0.0, 0.0};
#pragma unroll 1
  for (int r = 0; r < n_runs; ++r)
    for (int c = 0; c < 3; ++c) s[c] = s[c] + runs[(long long)r * kMoments + c];
  for (int c = 0; c < 3; ++c) st->c[c] = s[c] / (double)n;
}

// one thread: st->plane = the refitted plane, or the winner's hypothesis (no refine, |I| < 3 or C exactly zero)
__global__ void k_plane_refit(const double* __restrict__ runs, const float4* __restrict__ planes, bool refine,
                              PlaneState* __restrict__ st) {
  if (st->stop) return;
  float4 pl = planes[winner(st)];
  const long long n = st->n_inl;
  if (refine && n >= 3) {
    const int n_runs = (int)((n + kRun - 1) / kRun);
    double a[kMoments] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll 1
    for (int r = 0; r < n_runs; ++r)
      for (int t = 0; t < kMoments; ++t) a[t] = a[t] + runs[(long long)r * kMoments + t];
    const double dn = (double)n;
    double a00 = a[0] / dn, a01 = a[1] / dn, a02 = a[2] / dn, a11 = a[3] / dn, a12 = a[4] / dn, a22 = a[5] / dn;
    if (!(a00 == 0.0 && a01 == 0.0 && a02 == 0.0 && a11 == 0.0 && a12 == 0.0 && a22 == 0.0)) {
      double v0[3] = {1.0, 0.0, 0.0}, v1[3] = {0.0, 1.0, 0.0}, v2[3] = {0.0, 0.0, 1.0};
      jacobi_sweeps(a00, a01, a02, a11, a12, a22, v0, v1, v2);
      S4G_EIGEN_ORDER(a00, a11, a22, o0, o1, o2);
      const double nx = pick3(v0[0], v1[0], v2[0], o0), ny = pick3(v0[1], v1[1], v2[1], o0),
                   nz = pick3(v0[2], v1[2], v2[2], o0);
      const double len = sqrt((nx * nx + ny * ny) + nz * nz);
      pl = plane_round(nx, ny, nz, len, st->c[0], st->c[1], st->c[2]);
    }
  }
  st->plane = pl;
}

// st->final_count = the inliers of the final plane among A_r
__global__ void k_plane_final(const float4* __restrict__ A, int n, PlaneState* __restrict__ st, float threshold) {
  if (st->stop) return;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = i < n && i < st->m && plane_inlier(st->plane, A[i], threshold);
  const int c = __syncthreads_count(in);
  if (threadIdx.x == 0 && c > 0) atomicAdd(&st->final_count, (unsigned long long)c);
}

// one thread: accept round r (its record, offsets[r + 1], *n_planes) or stop
__global__ void k_plane_accept(int r, long long min_inliers, const float4* __restrict__ planes, const int4* __restrict__ samples,
                               PlaneState* __restrict__ st, s4g_plane* __restrict__ out, int* __restrict__ n_planes,
                               int64_t* __restrict__ offsets) {
  if (st->stop) return;
  const long long count = (long long)st->final_count;
  if (count < min_inliers) {
    st->stop = 1;
    return;
  }
  const int h = winner(st);
  const float4 hp = planes[h];
  const int4 s = samples[h];
  s4g_plane rec;
  rec.coefficients[0] = st->plane.x;
  rec.coefficients[1] = st->plane.y;
  rec.coefficients[2] = st->plane.z;
  rec.coefficients[3] = st->plane.w;
  rec.hypothesis[0] = hp.x;
  rec.hypothesis[1] = hp.y;
  rec.hypothesis[2] = hp.z;
  rec.hypothesis[3] = hp.w;
  rec.hypothesis_index = h;
  rec.sample[0] = s.x;
  rec.sample[1] = s.y;
  rec.sample[2] = s.z;
  rec.hypothesis_inliers = (int64_t)(st->key >> 32);
  rec.n_inliers = count;
  out[r] = rec;
  st->total += count;
  if (offsets != nullptr) offsets[r + 1] = st->total;
  st->n_planes = r + 1;
  *n_planes = r + 1;
}

__global__ void k_plane_label(const float4* __restrict__ A, int n, const PlaneState* __restrict__ st, float threshold, int r,
                              int32_t* __restrict__ labels) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || st->stop || i >= st->m) return;
  const float4 p = A[i];
  if (plane_inlier(st->plane, p, threshold)) labels[__float_as_int(p.w)] = r;
}

// member sort keys: the label, `none` for -1; vals[j] = j
__global__ void k_plane_member_keys(const int32_t* __restrict__ labels, int n, uint32_t none, uint32_t* __restrict__ keys,
                                    int* __restrict__ vals) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int32_t l = labels[j];
  keys[j] = l >= 0 ? (uint32_t)l : none;
  vals[j] = (int)j;
}

int plane_args(s4g_ctx* ctx, const char* who, float threshold, int H, int max_planes, long long min_inliers,
               const void* labels, const void* planes, const void* n_planes) {
  if (std::isnan(threshold) || threshold < 0.f || H < 1 || H > kMaxHypotheses || max_planes < 1 || min_inliers < 1 ||
      labels == nullptr || planes == nullptr || n_planes == nullptr) {
    ctx->err = std::string(who) + ": bad arguments (threshold >= 0 and not NaN, 1 <= n_hypotheses <= 2^20, max_planes "
                                  ">= 1, min_inliers >= 1, labels, planes and n_planes != NULL)";
    return S4G_ERR_ARG;
  }
  if (ctx->nP <= 0) {
    ctx->err = std::string(who) + ": call s4g_set_cloud_p first";
    return S4G_ERR_STATE;
  }
  return S4G_OK;
}

// the rounds that can draw: round r starts with at most nP - r points, and needs 3
int plane_rounds(int nP, int max_planes) { return nP < 3 ? 0 : (int)std::min<long long>(max_planes, (long long)nP - 2); }

// the ascending j with flags[j] != 0, or the A_r[i] with flags[i] != 0: cub::DeviceSelect::Flagged over n items
template <class In, class Out>
int select_flagged(s4g_ctx* ctx, In in, const uint8_t* flags, Out out, long long* count, int n) {
  size_t bytes = 0;
  S4G_CUDA(cub::DeviceSelect::Flagged(nullptr, bytes, in, flags, out, count, n, ctx->stream));
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, bytes));
  S4G_CUDA(cub::DeviceSelect::Flagged(ctx->dCub.p, bytes, in, flags, out, count, n, ctx->stream));
  ctx->launches++;
  return S4G_OK;
}

// enqueue the whole call.  Scratch A: A_r and I (float4 each, 32 bytes per point; the member sort's keys and values
// afterwards); B: the active positions (int32) and the flags (uint8); dMisc: the state, the hypotheses' planes, samples
// and counts (36 bytes per hypothesis), the runs' sums.
int launch_planes(s4g_ctx* ctx, float threshold, int H, unsigned long long seed, bool refine, int max_planes,
                  long long min_inliers, int32_t* d_labels, s4g_plane* d_planes, int* d_n_planes, int64_t* d_offsets,
                  int32_t* d_members, uint32_t* d_hyp_counts) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  const int n = ctx->nP;
  const size_t nn = (size_t)n;
  const int rounds = plane_rounds(n, max_planes);
  const int n_runs = (int)nblk(n, kRun);
  cudaStream_t st = ctx->stream;
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, 2 * nn * sizeof(float4)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, nn * (sizeof(int32_t) + 1)));
  const size_t state_bytes = (sizeof(PlaneState) + 15) / 16 * 16;
  const size_t hyp_bytes = (size_t)H * (sizeof(float4) + sizeof(int4));
  const size_t count_bytes = (size_t)H * sizeof(uint32_t);
  const size_t misc = state_bytes + hyp_bytes + (count_bytes + 15) / 16 * 16 + (size_t)n_runs * kMoments * sizeof(double);
  S4G_TRY(s4g_reserve(ctx, ctx->dMisc, misc));
  float4* A = ctx->dScratchA.as<float4>();
  float4* I = A + nn;
  int32_t* act = ctx->dScratchB.as<int32_t>();
  uint8_t* flags = reinterpret_cast<uint8_t*>(act + nn);
  char* base = ctx->dMisc.as<char>();
  PlaneState* d_st = reinterpret_cast<PlaneState*>(base);
  float4* hyp = reinterpret_cast<float4*>(base + state_bytes);
  int4* samples = reinterpret_cast<int4*>(hyp + H);
  uint32_t* scratch_counts = reinterpret_cast<uint32_t*>(samples + H);
  double* runs = reinterpret_cast<double*>(base + state_bytes + hyp_bytes + (count_bytes + 15) / 16 * 16);

  S4G_CUDA(cudaMemsetAsync(d_st, 0, sizeof(PlaneState), st));
  S4G_CUDA(cudaMemsetAsync(d_labels, 0xff, nn * sizeof(int32_t), st));
  S4G_CUDA(cudaMemsetAsync(d_n_planes, 0, sizeof(int), st));
  if (d_offsets != nullptr) S4G_CUDA(cudaMemsetAsync(d_offsets, 0, sizeof(int64_t), st));
  if (d_hyp_counts != nullptr)
    S4G_CUDA(cudaMemsetAsync(d_hyp_counts, 0, (size_t)max_planes * (size_t)H * sizeof(uint32_t), st));

  // k_plane_count's grid: hypothesis tiles x point slices, about kCountCtasPerSm CTAs per SM in all, slices of at least
  // one point tile
  const int hyp_tiles = (int)nblk(H, kHypTile);
  const long long want = std::max(1ll, (long long)ctx->sm_count * kCountCtasPerSm / hyp_tiles);
  const int slices = (int)std::min<long long>(want, std::max(1ll, (long long)nblk(n, kPointTile)));
  const dim3 count_grid((unsigned)slices, (unsigned)hyp_tiles);

  for (int r = 0; r < rounds; ++r) {
    uint32_t* counts = d_hyp_counts != nullptr ? d_hyp_counts + (size_t)r * (size_t)H : scratch_counts;
    if (d_hyp_counts == nullptr) S4G_CUDA(cudaMemsetAsync(counts, 0, count_bytes, st));
    k_plane_active<<<nblk(n, kThreads), kThreads, 0, st>>>(d_labels, n, d_st, flags);
    ctx->launches++;
    S4G_CUDA(cudaGetLastError());
    S4G_TRY(select_flagged(ctx, cub::CountingInputIterator<int32_t>(0), flags, act, &d_st->m, n));
    k_plane_gather<<<nblk(n, kThreads), kThreads, 0, st>>>(ctx->dP.as<float4>(), act, n, d_st, A);
    k_plane_hypotheses<<<nblk(H, kThreads), kThreads, 0, st>>>(A, d_st, H, seed + (unsigned long long)r, hyp, samples);
    k_plane_count<<<count_grid, kCountThreads, 0, st>>>(A, d_st, hyp, H, threshold, counts);
    k_plane_argmax<<<1, 1024, 0, st>>>(counts, samples, H, d_st);
    ctx->launches += 4;
    S4G_CUDA(cudaGetLastError());
    if (refine) {
      k_plane_inliers<<<nblk(n, kThreads), kThreads, 0, st>>>(A, n, d_st, hyp, threshold, flags);
      ctx->launches++;
      S4G_CUDA(cudaGetLastError());
      S4G_TRY(select_flagged(ctx, A, flags, I, &d_st->n_inl, n));
      k_plane_runs<<<n_runs, kRunThreads, 0, st>>>(I, d_st, false, runs);
      k_plane_centroid<<<1, 1, 0, st>>>(runs, d_st);
      k_plane_runs<<<n_runs, kRunThreads, 0, st>>>(I, d_st, true, runs);
      ctx->launches += 3;
    }
    k_plane_refit<<<1, 1, 0, st>>>(runs, hyp, refine, d_st);
    k_plane_final<<<nblk(n, kThreads), kThreads, 0, st>>>(A, n, d_st, threshold);
    k_plane_accept<<<1, 1, 0, st>>>(r, min_inliers, hyp, samples, d_st, d_planes, d_n_planes, d_offsets);
    k_plane_label<<<nblk(n, kThreads), kThreads, 0, st>>>(A, n, d_st, threshold, r, d_labels);
    ctx->launches += 4;
    S4G_CUDA(cudaGetLastError());
  }

  if (d_members != nullptr) {
    uint32_t* key0 = reinterpret_cast<uint32_t*>(A);   // A_r and I are consumed
    uint32_t* key1 = key0 + nn;
    int* val0 = reinterpret_cast<int*>(key1 + nn);
    int* val1 = val0 + nn;
    k_plane_member_keys<<<nblk(n, kThreads), kThreads, 0, st>>>(d_labels, n, (uint32_t)rounds, key0, val0);
    ctx->launches++;
    S4G_CUDA(cudaGetLastError());
    cub::DoubleBuffer<uint32_t> keys(key0, key1);
    cub::DoubleBuffer<int> vals(val0, val1);
    const int bits = key_bits(rounds);
    size_t bytes = 0;
    S4G_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, keys, vals, n, 0, bits, st));
    S4G_TRY(s4g_reserve(ctx, ctx->dCub, bytes));
    S4G_CUDA(cub::DeviceRadixSort::SortPairs(ctx->dCub.p, bytes, keys, vals, n, 0, bits, st));
    ctx->launches++;
    S4G_CUDA(cudaMemcpyAsync(d_members, vals.Current(), nn * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  }
  return S4G_OK;
}

}  // namespace

extern "C" int s4g_segment_planes_dev(s4g_ctx* ctx, float threshold, int n_hypotheses, uint64_t seed, int refine,
                                      int max_planes, int64_t min_inliers, int32_t* d_labels, s4g_plane* d_planes,
                                      int* d_n_planes, int64_t* d_offsets, int32_t* d_members, uint32_t* d_hyp_counts) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(plane_args(ctx, "s4g_segment_planes_dev", threshold, n_hypotheses, max_planes, min_inliers, d_labels, d_planes,
                     d_n_planes));
  return launch_planes(ctx, threshold, n_hypotheses, seed, refine != 0, max_planes, min_inliers, d_labels, d_planes,
                       d_n_planes, d_offsets, d_members, d_hyp_counts);
}

// the device outputs staged in ctx->dFilter: planes [rounds], offsets [rounds + 1], n_planes, labels and members [nP],
// hyp_counts [rounds x H]; then n_planes back first, and only the defined parts of the rest
extern "C" int s4g_segment_planes(s4g_ctx* ctx, float threshold, int n_hypotheses, uint64_t seed, int refine,
                                  int max_planes, int64_t min_inliers, int32_t* labels, s4g_plane* planes, int* n_planes,
                                  int64_t* offsets, int32_t* members, uint32_t* hyp_counts) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(plane_args(ctx, "s4g_segment_planes", threshold, n_hypotheses, max_planes, min_inliers, labels, planes,
                     n_planes));
  S4G_CUDA(cudaSetDevice(ctx->device));
  const size_t n = (size_t)ctx->nP;
  const int rounds = plane_rounds(ctx->nP, max_planes);
  const size_t R = (size_t)rounds, H = (size_t)n_hypotheses;
  const bool need_off = offsets != nullptr || members != nullptr;   // the members' total is offsets[n_planes]
  S4G_TRY(s4g_reserve(ctx, ctx->dFilter, std::max<size_t>(R, 1) * sizeof(s4g_plane) + (R + 1) * sizeof(int64_t) + 16 +
                                             2 * n * sizeof(int32_t) + (hyp_counts != nullptr ? R * H * sizeof(uint32_t) : 0)));
  s4g_plane* d_planes = ctx->dFilter.as<s4g_plane>();
  int64_t* d_off = reinterpret_cast<int64_t*>(d_planes + std::max<size_t>(R, 1));
  int* d_np = reinterpret_cast<int*>(d_off + R + 1);
  int32_t* d_labels = d_np + 4;
  int32_t* d_members = d_labels + n;
  uint32_t* d_hc = reinterpret_cast<uint32_t*>(d_members + n);
  cudaStream_t st = ctx->stream;
  // the device form's max_planes is the rounds that can draw: the rows past them are zeroed here on the host
  S4G_TRY(launch_planes(ctx, threshold, n_hypotheses, seed, refine != 0, std::max(rounds, 1), min_inliers, d_labels, d_planes,
                        d_np, need_off ? d_off : nullptr, members != nullptr ? d_members : nullptr,
                        hyp_counts != nullptr && rounds > 0 ? d_hc : nullptr));
  int np = 0;
  S4G_CUDA(cudaMemcpyAsync(&np, d_np, sizeof np, cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaMemcpyAsync(labels, d_labels, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (hyp_counts != nullptr && rounds > 0)
    S4G_CUDA(cudaMemcpyAsync(hyp_counts, d_hc, R * H * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  if (hyp_counts != nullptr)
    std::fill(hyp_counts + R * H, hyp_counts + (size_t)max_planes * H, 0u);
  *n_planes = np;
  int64_t total = 0;
  if (np > 0) {
    S4G_CUDA(cudaMemcpyAsync(planes, d_planes, (size_t)np * sizeof(s4g_plane), cudaMemcpyDeviceToHost, st));
    if (need_off) S4G_CUDA(cudaMemcpyAsync(&total, d_off + np, sizeof total, cudaMemcpyDeviceToHost, st));
    S4G_CUDA(cudaStreamSynchronize(st));
  }
  if (offsets != nullptr) {
    offsets[0] = 0;
    if (np > 0) S4G_CUDA(cudaMemcpyAsync(offsets, d_off, ((size_t)np + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  }
  if (members != nullptr && total > 0)
    S4G_CUDA(cudaMemcpyAsync(members, d_members, (size_t)total * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  return S4G_OK;
}
