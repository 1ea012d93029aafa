// Outlier removal on the resident P (s4g_statistical_outliers, s4g_radius_outliers, include/s4g.h).  Both filters write
// the kept original indices j in ascending order and their number, compacted by cub::DeviceSelect::Flagged from a flag
// per j (the output form of s4g_voxel_sample).
//
// Statistical filter.  Rows: the P points go to the existing k_knn instances (query.cu) in the grid's sorted order
// (s4g_launch_sorted_queries, as normals.cu), each excluding itself (exclude[t] = the original index of sorted point t),
// no T, sq_radius = +inf.  So row t is the s4g_knn row of p_j with exclude = j: min(k, nP - 1) real entries.
// k_outlier_mean, one thread per sorted point t of original index j: over the row's real entries in row order,
//   s = 0.0;  s = s + sqrt((double) d2_e);  mean_dist[j] = s / m   (m = 0, i.e. nP = 1: 0.0).
// Moments, in double, in one fixed order: the points in ascending j are cut into runs of kRun = 1024 (the last may be
// shorter); each run is summed left to right from 0.0 (k_outlier_runs), then the run sums left to right from 0.0
// (k_outlier_moments).
//   pass 1: mu = S1 / nP, S1 the sum of mean_dist;
//   pass 2: sigma = sqrt(S2 / (nP - 1)), S2 the sum of (mean_dist - mu)^2 (nP = 1: sigma = 0).
// k_outlier_flags: j is kept iff mean_dist[j] <= mu + std_ratio * sigma (double).
//
// Determinism.  The rows are fixed (k_knn's lexicographic k-minimum does not depend on the search order), every sum runs in
// a fixed order, and every value is made of IEEE basic operations (+ - * /, sqrt, compares) in double, compiled with
// -fmad=false so that no product is contracted into an FMA.  A CPU restatement of the same operations compiled without
// contraction (-ffp-contract=off) gives the same bits: mean_dist, mu, sigma and the kept set.
//
// Radius filter.  k_radius_count (query.cu: the same descent, drop rule and point test as k_range) writes the capped
// count and the flag of every j; its exactness argument is in its header.
#include "s4g_internal.cuh"
#include <cub/cub.cuh>
#include <cmath>

namespace {

constexpr int kRun = 1024;              // points per run of the fixed-order sums
constexpr int kRunThreads = 128;        // threads staging one run
constexpr int kOutlierThreads = 128;
constexpr int kOutlierMaxK = 64;        // k_knn's widest instance

unsigned nblk(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// sorted P (float4, w = original index) -> the exclusion list of the rows: exclude[t] = the original index of point t
__global__ void k_outlier_exclude(const float4* __restrict__ pts, int n, int32_t* __restrict__ exclude) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  exclude[t] = __float_as_int(pts[t].w);
}

__global__ void __launch_bounds__(kOutlierThreads)
k_outlier_mean(const float4* __restrict__ sorted, const int32_t* __restrict__ index, const float* __restrict__ sq, int n,
               int k, double* __restrict__ mean_dist) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const long long j = __float_as_int(__ldg(&sorted[t]).w);
  const long long row = t * (long long)k;
  double s = 0.0;
  int m = 0;
#pragma unroll 1
  for (; m < k; ++m) {
    if (__ldg(&index[row + m]) < 0) break;
    s = s + sqrt((double)__ldg(&sq[row + m]));
  }
  mean_dist[j] = m > 0 ? s / (double)m : 0.0;
}

// one block per run r of kRun points (ascending j): runs[r] = the run's values summed left to right from 0.0, the values
// being mean_dist (second = false) or (mean_dist - mu)^2 with mu = moments[0] (second = true).  The block stages the
// run's values in shared memory; one thread adds them in order.
__global__ void __launch_bounds__(kRunThreads)
k_outlier_runs(const double* __restrict__ mean_dist, int n, const double* __restrict__ moments, bool second,
               double* __restrict__ runs) {
  __shared__ double v[kRun];
  const long long begin = (long long)blockIdx.x * kRun;
  const int len = (int)min((long long)kRun, (long long)n - begin);
  const double mu = second ? moments[0] : 0.0;
  for (int i = threadIdx.x; i < len; i += blockDim.x) {
    double x = mean_dist[begin + i];
    if (second) {
      x = x - mu;
      x = x * x;
    }
    v[i] = x;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double s = 0.0;
#pragma unroll 1
  for (int i = 0; i < len; ++i) s = s + v[i];
  runs[blockIdx.x] = s;
}

// one thread: the run sums left to right from 0.0 -> moments[0] = mu (first pass) or moments[1] = sigma (second)
__global__ void k_outlier_moments(const double* __restrict__ runs, int n_runs, int n, bool second, double* __restrict__ moments) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double s = 0.0;
#pragma unroll 1
  for (int r = 0; r < n_runs; ++r) s = s + runs[r];
  if (!second)
    moments[0] = s / (double)n;
  else
    moments[1] = n > 1 ? sqrt(s / (double)(n - 1)) : 0.0;
}

__global__ void k_outlier_flags(const double* __restrict__ mean_dist, int n, const double* __restrict__ moments,
                                double std_ratio, uint8_t* __restrict__ keep) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const double threshold = moments[0] + std_ratio * moments[1];
  keep[j] = mean_dist[j] <= threshold ? 1 : 0;
}

// the kept j in ascending order and their number, from the flags: d_keep [nP], d_n_kept [1]
int compact(s4g_ctx* ctx, const uint8_t* d_flags, int32_t* d_keep, int64_t* d_n_kept) {
  cub::CountingInputIterator<int32_t> counting(0);
  size_t bytes = 0;
  S4G_CUDA(cub::DeviceSelect::Flagged(nullptr, bytes, counting, d_flags, d_keep, d_n_kept, ctx->nP, ctx->stream));
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, bytes));
  S4G_CUDA(cub::DeviceSelect::Flagged(ctx->dCub.p, bytes, counting, d_flags, d_keep, d_n_kept, ctx->nP, ctx->stream));
  ctx->launches++;
  return S4G_OK;
}

int need_p(s4g_ctx* ctx, const char* who) {
  if (ctx->nP <= 0) {
    ctx->err = std::string(who) + ": call s4g_set_cloud_p first";
    return S4G_ERR_STATE;
  }
  return S4G_OK;
}

int statistical_args(s4g_ctx* ctx, const char* who, int k, double std_ratio, const void* keep, const void* n_kept) {
  if (k < 1 || k > kOutlierMaxK || !std::isfinite(std_ratio) || keep == nullptr || n_kept == nullptr) {
    ctx->err = std::string(who) + ": bad arguments (1 <= k <= 64, std_ratio finite, keep and n_kept != NULL)";
    return S4G_ERR_ARG;
  }
  return need_p(ctx, who);
}

int radius_args(s4g_ctx* ctx, const char* who, float sq_radius, int min_neighbors, const void* keep, const void* n_kept) {
  if (std::isnan(sq_radius) || min_neighbors < 1 || keep == nullptr || n_kept == nullptr) {
    ctx->err = std::string(who) + ": bad arguments (sq_radius not NaN, min_neighbors >= 1, keep and n_kept != NULL)";
    return S4G_ERR_ARG;
  }
  return need_p(ctx, who);
}

// enqueue the statistical filter on the context's stream.  Scratch: A the sorted queries, B / C the rows (index, d^2),
// D the exclusion list then the flags, dMisc the run sums, the moments when d_out2 is NULL and mean_dist when
// d_mean_dist is NULL.
int launch_statistical(s4g_ctx* ctx, int k, double std_ratio, int32_t* d_keep, int64_t* d_n_kept, double* d_mean_dist,
                       double* d_out2) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  const int n = ctx->nP;
  const int n_runs = (int)nblk(n, kRun);
  cudaStream_t st = ctx->stream;
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, (size_t)n * 3 * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, (size_t)n * (size_t)k * sizeof(int32_t)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchC, (size_t)n * (size_t)k * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchD, (size_t)n * sizeof(int32_t)));
  const size_t misc = (size_t)n_runs + 2 + (d_mean_dist == nullptr ? (size_t)n : 0);
  S4G_TRY(s4g_reserve(ctx, ctx->dMisc, misc * sizeof(double)));
  float* d_xyz = ctx->dScratchA.as<float>();
  int32_t* d_excl = ctx->dScratchD.as<int32_t>();
  uint8_t* d_flags = ctx->dScratchD.as<uint8_t>();   // written once the rows (and so the exclusion list) are consumed
  double* d_runs = ctx->dMisc.as<double>();
  double* d_mom = d_out2 != nullptr ? d_out2 : d_runs + n_runs;
  double* d_mean = d_mean_dist != nullptr ? d_mean_dist : d_runs + n_runs + 2;
  S4G_TRY(s4g_launch_sorted_queries(ctx, d_xyz));
  k_outlier_exclude<<<nblk(n, 256), 256, 0, st>>>(ctx->grid.pts, n, d_excl);
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  S4G_TRY(s4g_launch_knn(ctx, d_xyz, n, nullptr, k, INFINITY, d_excl, ctx->dScratchB.as<int32_t>(),
                         ctx->dScratchC.as<float>(), nullptr));
  k_outlier_mean<<<nblk(n, kOutlierThreads), kOutlierThreads, 0, st>>>(ctx->grid.pts, ctx->dScratchB.as<int32_t>(),
                                                                      ctx->dScratchC.as<float>(), n, k, d_mean);
  for (int pass = 0; pass < 2; ++pass) {
    k_outlier_runs<<<n_runs, kRunThreads, 0, st>>>(d_mean, n, d_mom, pass == 1, d_runs);
    k_outlier_moments<<<1, 32, 0, st>>>(d_runs, n_runs, n, pass == 1, d_mom);
  }
  k_outlier_flags<<<nblk(n, 256), 256, 0, st>>>(d_mean, n, d_mom, std_ratio, d_flags);
  ctx->launches += 6;
  S4G_CUDA(cudaGetLastError());
  return compact(ctx, d_flags, d_keep, d_n_kept);
}

int launch_radius(s4g_ctx* ctx, float sq_radius, int min_neighbors, int32_t* d_keep, int64_t* d_n_kept, int32_t* d_counts) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchD, (size_t)ctx->nP));
  uint8_t* d_flags = ctx->dScratchD.as<uint8_t>();
  S4G_TRY(s4g_launch_radius_count(ctx, sq_radius, min_neighbors, d_counts, d_flags));
  return compact(ctx, d_flags, d_keep, d_n_kept);
}

// the host forms' device outputs in ctx->dFilter: doubles [mean_dist n | out2 2], then n_kept (int64), then keep (n int32)
// or counts (n int32) after keep
struct FilterOut {
  double* mean;
  double* out2;
  int64_t* n_kept;
  int32_t* keep;
  int32_t* counts;
};

int filter_out(s4g_ctx* ctx, bool mean, bool counts, FilterOut& o) {
  const size_t n = (size_t)ctx->nP;
  const size_t doubles = (mean ? n : 0) + 2;
  S4G_TRY(s4g_reserve(ctx, ctx->dFilter, doubles * sizeof(double) + sizeof(int64_t) + (counts ? 2 : 1) * n * sizeof(int32_t)));
  double* d = ctx->dFilter.as<double>();
  o.mean = mean ? d : nullptr;
  o.out2 = d + (mean ? n : 0);
  o.n_kept = reinterpret_cast<int64_t*>(d + doubles);
  o.keep = reinterpret_cast<int32_t*>(o.n_kept + 1);
  o.counts = counts ? o.keep + n : nullptr;
  return S4G_OK;
}

// n_kept back first, then only the kept part of the list
int copy_keep(s4g_ctx* ctx, const FilterOut& o, int32_t* keep, int64_t* n_kept) {
  cudaStream_t st = ctx->stream;
  int64_t nk = 0;
  S4G_CUDA(cudaMemcpyAsync(&nk, o.n_kept, sizeof nk, cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  if (nk > 0) S4G_CUDA(cudaMemcpyAsync(keep, o.keep, (size_t)nk * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  *n_kept = nk;
  return S4G_OK;
}

}  // namespace

int s4g_launch_exclude_self(s4g_ctx* ctx, int32_t* d_exclude) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  k_outlier_exclude<<<nblk(ctx->nP, 256), 256, 0, ctx->stream>>>(ctx->grid.pts, ctx->nP, d_exclude);
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;
}

extern "C" int s4g_statistical_outliers_dev(s4g_ctx* ctx, int k, double std_ratio, int32_t* d_keep, int64_t* d_n_kept,
                                            double* d_mean_dist, double* d_out2) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(statistical_args(ctx, "s4g_statistical_outliers_dev", k, std_ratio, d_keep, d_n_kept));
  return launch_statistical(ctx, k, std_ratio, d_keep, d_n_kept, d_mean_dist, d_out2);
}

extern "C" int s4g_statistical_outliers(s4g_ctx* ctx, int k, double std_ratio, int32_t* keep, int64_t* n_kept,
                                        double* mean_dist, double* out2) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(statistical_args(ctx, "s4g_statistical_outliers", k, std_ratio, keep, n_kept));
  S4G_CUDA(cudaSetDevice(ctx->device));
  FilterOut o;
  S4G_TRY(filter_out(ctx, mean_dist != nullptr, false, o));
  S4G_TRY(launch_statistical(ctx, k, std_ratio, o.keep, o.n_kept, o.mean, o.out2));
  cudaStream_t st = ctx->stream;
  if (mean_dist != nullptr)
    S4G_CUDA(cudaMemcpyAsync(mean_dist, o.mean, (size_t)ctx->nP * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (out2 != nullptr) S4G_CUDA(cudaMemcpyAsync(out2, o.out2, 2 * sizeof(double), cudaMemcpyDeviceToHost, st));
  S4G_TRY(copy_keep(ctx, o, keep, n_kept));
  S4G_CUDA(cudaStreamSynchronize(ctx->stream));
  return S4G_OK;
}

extern "C" int s4g_radius_outliers_dev(s4g_ctx* ctx, float sq_radius, int min_neighbors, int32_t* d_keep, int64_t* d_n_kept,
                                       int32_t* d_counts) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(radius_args(ctx, "s4g_radius_outliers_dev", sq_radius, min_neighbors, d_keep, d_n_kept));
  return launch_radius(ctx, sq_radius, min_neighbors, d_keep, d_n_kept, d_counts);
}

extern "C" int s4g_radius_outliers(s4g_ctx* ctx, float sq_radius, int min_neighbors, int32_t* keep, int64_t* n_kept,
                                   int32_t* counts) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(radius_args(ctx, "s4g_radius_outliers", sq_radius, min_neighbors, keep, n_kept));
  S4G_CUDA(cudaSetDevice(ctx->device));
  FilterOut o;
  S4G_TRY(filter_out(ctx, false, counts != nullptr, o));
  S4G_TRY(launch_radius(ctx, sq_radius, min_neighbors, o.keep, o.n_kept, o.counts));
  if (counts != nullptr)
    S4G_CUDA(cudaMemcpyAsync(counts, o.counts, (size_t)ctx->nP * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
  S4G_TRY(copy_keep(ctx, o, keep, n_kept));
  S4G_CUDA(cudaStreamSynchronize(ctx->stream));
  return S4G_OK;
}
