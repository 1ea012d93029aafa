// Voxel-grid downsampling to centroids (s4g_voxel_grid, include/s4g.h): PCL's VoxelGrid / Open3D's voxel_down_sample,
// made exact.  Every point goes to the voxel (floor(x s), floor(y s), floor(z s)), s = 1.0f / leaf, the arithmetic of
// s4g_voxel_sample (sampler.cu); a voxel's members are its points in ascending input index, and every output value is a
// fixed-order double sum of them.
//
// Launch chain (all on the context's stream, no host synchronisation until the host form reads the result back):
//   k_vg_bounds   the smallest and largest voxel coordinate per axis (integer atomics) and a flag for a coordinate whose
//                 scaled floor is NaN or outside the int32 range (non-finite inputs included)
//   k_vg_keys     key = (cx - min x) << 42 | (cy - min y) << 21 | (cz - min z), value = the input index
//   cub::DeviceRadixSort::SortPairs over 63 bits: stable, so each voxel's members come out in ascending index
//   k_vg_heads + cub::DeviceScan::InclusiveSum: the voxel (1-based) of every sorted position
//   k_vg_starts   start[v] = the first sorted position of voxel v, start[n_voxels] = n
//   k_vg_gather   xyz, normals and rgb into sorted order, so that the sums below read consecutive addresses
//   k_vg_runs     the sum of every full run of 1024 members of a voxel that has more than one run, one thread per run
//                 (the run holding sorted position 1024 q goes to thread q: a full run holds exactly one multiple of 1024)
//   k_vg_flags + cub::DeviceScan::ExclusiveSum: a flag at the input position of the first member of every voxel with
//                 m >= min_points, scanned in input order, gives each surviving voxel its output index (the compaction
//                 of sampler.cu)
//   k_vg_count    *n_out, or -1 when a coordinate or the span was invalid
//   k_vg_order    order[o] = the voxel of output o (and ov[v] = o for voxel_of)
//   k_vg_final    one thread per output o, so that the outputs are written coalesced: the sum of the voxel's last (or
//                 only) run, the run sums left to right, the centroid, normal, rgb, count and first member
//   k_vg_voxel_of voxel_of[i] for every input point
// The hot path is streaming: keys, the sort, the gather and the sums each read or write every point a fixed number of
// times.  Every value is made of IEEE basic operations in double in the contract's order, compiled with -fmad=false, so
// that a CPU restatement of the contract, compiled without contraction, gives the same bits.
#include "s4g_internal.cuh"
#include <cub/cub.cuh>
#include <climits>
#include <cmath>

namespace {

constexpr int kRun = 1024;               // members per run of the fixed-order sums
constexpr int kRunShift = 10;
constexpr int kThreads = 256;
constexpr long long kSpan = 1ll << 21;   // voxels per axis a 21-bit key field holds

// device state of one call: bounds, flags and counts (int32 words)
struct VgMeta {
  int mn[3], mx[3];
  int bad;          // some scaled coordinate was NaN or its floor outside the int32 range
  int n_voxels;     // occupied voxels
  int last_first;   // 1 when input point n - 1 is the first member of a surviving voxel
  int kept;         // surviving voxels
  int pad[6];
};

unsigned nblk(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// floor(fl(x s)) as a float; a coordinate is valid iff this lies in [-2^31, 2^31) (NaN fails both tests)
__device__ __forceinline__ float vg_cell(float x, float s) { return floorf(__fmul_rn(x, s)); }
__device__ __forceinline__ bool vg_valid(float c) { return c >= -2147483648.f && c < 2147483648.f; }

__global__ void k_vg_init(VgMeta* __restrict__ meta) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  for (int a = 0; a < 3; ++a) meta->mn[a] = INT_MAX, meta->mx[a] = INT_MIN;
  meta->bad = 0;
  meta->n_voxels = 0;
  meta->last_first = 0;
  meta->kept = 0;
}

__global__ void __launch_bounds__(kThreads)
k_vg_bounds(const float* __restrict__ xyz, long long n, float s, VgMeta* __restrict__ meta) {
  int mn[3] = {INT_MAX, INT_MAX, INT_MAX}, mx[3] = {INT_MIN, INT_MIN, INT_MIN};
  int bad = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float c = vg_cell(xyz[3 * i + a], s);
      if (!vg_valid(c)) {
        bad = 1;
        continue;
      }
      mn[a] = min(mn[a], (int)c);
      mx[a] = max(mx[a], (int)c);
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    mn[a] = __reduce_min_sync(0xffffffffu, mn[a]);
    mx[a] = __reduce_max_sync(0xffffffffu, mx[a]);
  }
  bad = __reduce_or_sync(0xffffffffu, (unsigned)bad);
  if ((threadIdx.x & 31) != 0) return;
  for (int a = 0; a < 3; ++a) {
    if (mn[a] != INT_MAX) atomicMin(&meta->mn[a], mn[a]);
    if (mx[a] != INT_MIN) atomicMax(&meta->mx[a], mx[a]);
  }
  if (bad) atomicOr(&meta->bad, 1);
}

__global__ void __launch_bounds__(kThreads)
k_vg_keys(const float* __restrict__ xyz, long long n, float s, const VgMeta* __restrict__ meta,
          unsigned long long* __restrict__ keys, int32_t* __restrict__ vals) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned long long key = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float c = vg_cell(xyz[3 * i + a], s);
    // an invalid coordinate makes the call fail (k_vg_count); its key only has to stay within 21 bits per field
    const long long d = vg_valid(c) ? (long long)(int)c - (long long)meta->mn[a] : 0;
    key = (key << 21) | ((unsigned long long)d & (unsigned long long)(kSpan - 1));
  }
  keys[i] = key;
  vals[i] = (int32_t)i;
}

__global__ void __launch_bounds__(kThreads)
k_vg_heads(const unsigned long long* __restrict__ keys, long long n, int32_t* __restrict__ head) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  head[t] = (t == 0 || keys[t] != keys[t - 1]) ? 1 : 0;
}

// seg[t] = 1 + the voxel of sorted position t
__global__ void __launch_bounds__(kThreads)
k_vg_starts(const int32_t* __restrict__ seg, long long n, int32_t* __restrict__ start, VgMeta* __restrict__ meta) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const int v = seg[t];
  if (t == 0 || seg[t - 1] != v) start[v - 1] = (int32_t)t;
  if (t == n - 1) {
    start[v] = (int32_t)n;
    meta->n_voxels = v;
  }
}

__global__ void __launch_bounds__(kThreads)
k_vg_gather(const int32_t* __restrict__ idx, long long n, const float* __restrict__ xyz, const float* __restrict__ nrm,
            const float* __restrict__ rgb, float* __restrict__ gx, float* __restrict__ gn, float* __restrict__ gc) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const long long i = idx[t];
#pragma unroll
  for (int a = 0; a < 3; ++a) gx[3 * t + a] = __ldg(&xyz[3 * i + a]);
  if (gn != nullptr) {
#pragma unroll
    for (int a = 0; a < 3; ++a) gn[3 * t + a] = __ldg(&nrm[3 * i + a]);
  }
  if (gc != nullptr) {
#pragma unroll
    for (int a = 0; a < 3; ++a) gc[3 * t + a] = __ldg(&rgb[3 * i + a]);
  }
}

// the 9 sums (xyz, normal, rgb) of sorted positions [b, b + len), each left to right from 0.0
struct Sums {
  double v[9];
};
__device__ __forceinline__ void run_sums(const float* __restrict__ gx, const float* __restrict__ gn,
                                         const float* __restrict__ gc, long long b, int len, Sums& r) {
#pragma unroll
  for (int c = 0; c < 9; ++c) r.v[c] = 0.0;
#pragma unroll 4
  for (int k = 0; k < len; ++k) {
    const long long t = b + k;
#pragma unroll
    for (int a = 0; a < 3; ++a) r.v[a] = r.v[a] + (double)__ldg(&gx[3 * t + a]);
    if (gn != nullptr) {
#pragma unroll
      for (int a = 0; a < 3; ++a) r.v[3 + a] = r.v[3 + a] + (double)__ldg(&gn[3 * t + a]);
    }
    if (gc != nullptr) {
#pragma unroll
      for (int a = 0; a < 3; ++a) r.v[6 + a] = r.v[6 + a] + (double)__ldg(&gc[3 * t + a]);
    }
  }
}

// thread q: the full run that holds sorted position 1024 q, when it is not its voxel's last run -> runsum[q]
__global__ void __launch_bounds__(kThreads)
k_vg_runs(const int32_t* __restrict__ seg, const int32_t* __restrict__ start, long long n, const float* __restrict__ gx,
          const float* __restrict__ gn, const float* __restrict__ gc, Sums* __restrict__ runsum) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long p = q << kRunShift;
  if (p >= n) return;
  const int v = seg[p] - 1;
  const long long s = start[v], m = (long long)start[v + 1] - s;
  const long long k = (p - s) >> kRunShift;
  if (k >= (m - 1) >> kRunShift) return;   // the last run: k_vg_final sums it
  Sums r;
  run_sums(gx, gn, gc, s + (k << kRunShift), kRun, r);
  runsum[q] = r;
}

// thread v: the survival flag of voxel v at the input position of its first member, and v itself there
__global__ void __launch_bounds__(kThreads)
k_vg_flags(const int32_t* __restrict__ start, const int32_t* __restrict__ idx, long long n, int min_points,
           int32_t* __restrict__ flags, int32_t* __restrict__ vat, VgMeta* __restrict__ meta) {
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= meta->n_voxels) return;
  const int s = start[v];
  const int first = idx[s];
  const int keep = start[v + 1] - s >= min_points ? 1 : 0;
  flags[first] = keep;
  vat[first] = (int32_t)v;
  if (first == n - 1) meta->last_first = keep;
}

// thread i (input order): the surviving voxel whose first member is i gets output index o = pos[i]: order[o] = v,
// ov[v] = o (ov of the dropped voxels stays -1)
__global__ void __launch_bounds__(kThreads)
k_vg_order(const int32_t* __restrict__ flags, const int32_t* __restrict__ pos, const int32_t* __restrict__ vat,
           long long n, int32_t* __restrict__ order, int32_t* __restrict__ ov) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !flags[i]) return;
  const int o = pos[i], v = vat[i];
  order[o] = v;
  if (ov != nullptr) ov[v] = o;
}

// thread o (output order, so that the outputs are written coalesced): voxel v = order[o]
__global__ void __launch_bounds__(kThreads)
k_vg_final(const int32_t* __restrict__ order, const int32_t* __restrict__ start, const int32_t* __restrict__ idx,
           const VgMeta* __restrict__ meta, const float* __restrict__ gx, const float* __restrict__ gn,
           const float* __restrict__ gc, const Sums* __restrict__ runsum, float* __restrict__ xyz_out,
           float* __restrict__ normals_out, float* __restrict__ rgb_out, int32_t* __restrict__ counts,
           int32_t* __restrict__ first_out) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= meta->kept) return;
  const int v = order[o];
  const long long s = start[v];
  const int m = (int)(start[v + 1] - s);
  double S[9];
#pragma unroll
  for (int c = 0; c < 9; ++c) S[c] = 0.0;
  const long long full = (long long)(m - 1) >> kRunShift;   // runs before the last
  const long long q0 = (s + kRun - 1) >> kRunShift;        // runsum slot of the first of them
#pragma unroll 1
  for (long long k = 0; k < full; ++k) {
    const Sums& r = runsum[q0 + k];
#pragma unroll
    for (int c = 0; c < 9; ++c) S[c] = S[c] + r.v[c];
  }
  Sums last;
  run_sums(gx, gn, gc, s + (full << kRunShift), (int)(m - (full << kRunShift)), last);
#pragma unroll
  for (int c = 0; c < 9; ++c) S[c] = S[c] + last.v[c];
  const double dm = (double)m;
#pragma unroll
  for (int a = 0; a < 3; ++a) xyz_out[3 * o + a] = (float)(S[a] / dm);
  if (normals_out != nullptr) {
    const double len = sqrt((S[3] * S[3] + S[4] * S[4]) + S[5] * S[5]);
#pragma unroll
    for (int a = 0; a < 3; ++a) normals_out[3 * o + a] = len == 0.0 ? 0.f : (float)(S[3 + a] / len);
  }
  if (rgb_out != nullptr) {
#pragma unroll
    for (int a = 0; a < 3; ++a) rgb_out[3 * o + a] = (float)(S[6 + a] / dm);
  }
  if (counts != nullptr) counts[o] = m;
  if (first_out != nullptr) first_out[o] = idx[s];
}

__global__ void k_vg_count(const int32_t* __restrict__ pos, long long n, VgMeta* __restrict__ meta,
                           int64_t* __restrict__ n_out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  bool bad = meta->bad != 0;
  for (int a = 0; a < 3; ++a) bad = bad || (long long)meta->mx[a] - (long long)meta->mn[a] >= kSpan;
  meta->kept = pos[n - 1] + meta->last_first;
  *n_out = bad ? -1 : (int64_t)meta->kept;
}

__global__ void __launch_bounds__(kThreads)
k_vg_voxel_of(const int32_t* __restrict__ seg, const int32_t* __restrict__ idx, const int32_t* __restrict__ ov,
              long long n, int32_t* __restrict__ voxel_of) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  voxel_of[idx[t]] = ov[seg[t] - 1];
}

size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

// scratch bytes of n points: keys 2 x 8, indices 2 x 4, heads / flags 4, voxel of each sorted position 4, starts 4
// (+1), the gathered attributes 12 each; the output-order arrays (pos, ov, order, vat) reuse the key buffers once the
// keys are consumed
struct Scratch {
  unsigned long long* keys[2];
  int32_t* vals[2];
  int32_t* flags;   // head flags, then the survival flags
  int32_t* seg;
  int32_t* start;
  float *gx, *gn, *gc;
  Sums* runsum;
  VgMeta* meta;
};

int reserve_scratch(s4g_ctx* ctx, long long n, bool normals, bool rgb, Scratch& S) {
  const size_t N = (size_t)n;
  const size_t n_runs = (N + kRun - 1) / kRun;
  const size_t sizes[] = {8 * N, 8 * N, 4 * N, 4 * N, 4 * N, 4 * N, 4 * (N + 1), 12 * N, normals ? 12 * N : 0,
                          rgb ? 12 * N : 0, sizeof(Sums) * n_runs, sizeof(VgMeta)};
  size_t total = 0;
  for (size_t b : sizes) total += align256(b);
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, total));
  char* p = ctx->dScratchA.as<char>();
  char* part[12];
  for (int k = 0; k < 12; ++k) {
    part[k] = sizes[k] ? p : nullptr;
    p += align256(sizes[k]);
  }
  S.keys[0] = reinterpret_cast<unsigned long long*>(part[0]);
  S.keys[1] = reinterpret_cast<unsigned long long*>(part[1]);
  S.vals[0] = reinterpret_cast<int32_t*>(part[2]);
  S.vals[1] = reinterpret_cast<int32_t*>(part[3]);
  S.flags = reinterpret_cast<int32_t*>(part[4]);
  S.seg = reinterpret_cast<int32_t*>(part[5]);
  S.start = reinterpret_cast<int32_t*>(part[6]);
  S.gx = reinterpret_cast<float*>(part[7]);
  S.gn = reinterpret_cast<float*>(part[8]);
  S.gc = reinterpret_cast<float*>(part[9]);
  S.runsum = reinterpret_cast<Sums*>(part[10]);
  S.meta = reinterpret_cast<VgMeta*>(part[11]);
  return S4G_OK;
}

int check_args(s4g_ctx* ctx, const char* who, const void* xyz, const void* normals, const void* rgb, int64_t n, float leaf,
               int min_points, const void* xyz_out, const void* normals_out, const void* rgb_out, const void* n_out) {
  if (!xyz || !xyz_out || !n_out || (normals == nullptr) != (normals_out == nullptr) ||
      (rgb == nullptr) != (rgb_out == nullptr) || !std::isfinite(leaf) || !(leaf > 0.f) || min_points < 1 || n < 0 ||
      n >= (1ll << 31)) {
    ctx->err = std::string(who) +
               ": bad arguments (xyz, xyz_out and n_out != NULL, normals / normals_out and rgb / rgb_out both NULL or "
               "both given, leaf finite and > 0, min_points >= 1, 0 <= n < 2^31)";
    return S4G_ERR_ARG;
  }
  return S4G_OK;
}

// enqueue the whole call for n >= 1 points on the context's stream; every array a device pointer
int launch(s4g_ctx* ctx, const float* xyz, const float* nrm, const float* rgb, long long n, float leaf, int min_points,
           float* xyz_out, float* normals_out, float* rgb_out, int32_t* counts, int32_t* first, int32_t* voxel_of,
           int64_t* n_out, VgMeta** meta_out) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  Scratch S;
  S4G_TRY(reserve_scratch(ctx, n, nrm != nullptr, rgb != nullptr, S));
  const float s = 1.0f / leaf;   // sampling.h:75, as s4g_voxel_sample
  const unsigned nb = nblk(n, kThreads);
  k_vg_init<<<1, 32, 0, st>>>(S.meta);
  k_vg_bounds<<<std::min(nb, (unsigned)(ctx->sm_count * 8)), kThreads, 0, st>>>(xyz, n, s, S.meta);
  k_vg_keys<<<nb, kThreads, 0, st>>>(xyz, n, s, S.meta, S.keys[0], S.vals[0]);
  ctx->launches += 3;
  S4G_CUDA(cudaGetLastError());

  cub::DoubleBuffer<unsigned long long> dk(S.keys[0], S.keys[1]);
  cub::DoubleBuffer<int32_t> dv(S.vals[0], S.vals[1]);
  size_t sort_bytes = 0, incl_bytes = 0, excl_bytes = 0;
  S4G_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, dk, dv, (int)n, 0, 63, st));
  S4G_CUDA(cub::DeviceScan::InclusiveSum(nullptr, incl_bytes, S.flags, S.seg, (int)n, st));
  S4G_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, excl_bytes, S.flags, S.flags, (int)n, st));
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, std::max(sort_bytes, std::max(incl_bytes, excl_bytes))));
  S4G_CUDA(cub::DeviceRadixSort::SortPairs(ctx->dCub.p, sort_bytes, dk, dv, (int)n, 0, 63, st));
  const unsigned long long* keys = dk.Current();
  const int32_t* idx = dv.Current();
  // the key buffers are free once the heads are flagged: pos, ov, order and vat [n each] go there
  int32_t* pos = reinterpret_cast<int32_t*>(S.keys[0]);
  int32_t* ov = pos + n;
  int32_t* order = reinterpret_cast<int32_t*>(S.keys[1]);
  int32_t* vat = order + n;

  k_vg_heads<<<nb, kThreads, 0, st>>>(keys, n, S.flags);
  S4G_CUDA(cub::DeviceScan::InclusiveSum(ctx->dCub.p, incl_bytes, S.flags, S.seg, (int)n, st));
  k_vg_starts<<<nb, kThreads, 0, st>>>(S.seg, n, S.start, S.meta);
  k_vg_gather<<<nb, kThreads, 0, st>>>(idx, n, xyz, nrm, rgb, S.gx, S.gn, S.gc);
  k_vg_runs<<<nblk(nblk(n, kRun), kThreads), kThreads, 0, st>>>(S.seg, S.start, n, S.gx, S.gn, S.gc, S.runsum);
  S4G_CUDA(cudaMemsetAsync(S.flags, 0, (size_t)n * sizeof(int32_t), st));
  if (voxel_of != nullptr) S4G_CUDA(cudaMemsetAsync(ov, 0xFF, (size_t)n * sizeof(int32_t), st));
  k_vg_flags<<<nb, kThreads, 0, st>>>(S.start, idx, n, min_points, S.flags, vat, S.meta);
  S4G_CUDA(cub::DeviceScan::ExclusiveSum(ctx->dCub.p, excl_bytes, S.flags, pos, (int)n, st));
  k_vg_count<<<1, 32, 0, st>>>(pos, n, S.meta, n_out);
  k_vg_order<<<nb, kThreads, 0, st>>>(S.flags, pos, vat, n, order, voxel_of != nullptr ? ov : nullptr);
  k_vg_final<<<nb, kThreads, 0, st>>>(order, S.start, idx, S.meta, S.gx, S.gn, S.gc, S.runsum, xyz_out, normals_out,
                                      rgb_out, counts, first);
  ctx->launches += 12;
  if (voxel_of != nullptr) {
    k_vg_voxel_of<<<nb, kThreads, 0, st>>>(S.seg, idx, ov, n, voxel_of);
    ctx->launches++;
  }
  S4G_CUDA(cudaGetLastError());
  if (meta_out) *meta_out = S.meta;
  return S4G_OK;
}

}  // namespace

extern "C" int s4g_voxel_grid_dev(s4g_ctx* ctx, const float* d_xyz, const float* d_normals, const float* d_rgb, int64_t n,
                                  float leaf, int min_points, float* d_xyz_out, float* d_normals_out, float* d_rgb_out,
                                  int32_t* d_counts, int32_t* d_first, int32_t* d_voxel_of, int64_t* d_n_out) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(check_args(ctx, "s4g_voxel_grid_dev", d_xyz, d_normals, d_rgb, n, leaf, min_points, d_xyz_out, d_normals_out,
                     d_rgb_out, d_n_out));
  if (n == 0) {
    S4G_CUDA(cudaSetDevice(ctx->device));
    S4G_CUDA(cudaMemsetAsync(d_n_out, 0, sizeof(int64_t), ctx->stream));
    return S4G_OK;
  }
  return launch(ctx, d_xyz, d_normals, d_rgb, n, leaf, min_points, d_xyz_out, d_normals_out, d_rgb_out, d_counts, d_first,
                d_voxel_of, d_n_out, nullptr);
}

extern "C" int s4g_voxel_grid(s4g_ctx* ctx, const float* xyz, const float* normals, const float* rgb, int64_t n, float leaf,
                              int min_points, float* xyz_out, float* normals_out, float* rgb_out, int32_t* counts,
                              int32_t* first, int32_t* voxel_of, int64_t* n_out) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(check_args(ctx, "s4g_voxel_grid", xyz, normals, rgb, n, leaf, min_points, xyz_out, normals_out, rgb_out, n_out));
  if (n == 0) {
    *n_out = 0;
    return S4G_OK;
  }
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  // device copies: the inputs (12 bytes per point per array), then the outputs (12 per array, 4 per index array) and n_out
  const size_t N = (size_t)n, a3 = align256(12 * N), a1 = align256(4 * N);
  const int k = 1 + (normals != nullptr) + (rgb != nullptr);
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, 2 * k * a3 + 3 * a1 + 256));
  char* p = ctx->dScratchB.as<char>();
  auto take = [&](size_t b) { char* r = p; p += b; return r; };
  float* d_xyz = reinterpret_cast<float*>(take(a3));
  float* d_nrm = normals ? reinterpret_cast<float*>(take(a3)) : nullptr;
  float* d_rgb = rgb ? reinterpret_cast<float*>(take(a3)) : nullptr;
  float* o_xyz = reinterpret_cast<float*>(take(a3));
  float* o_nrm = normals ? reinterpret_cast<float*>(take(a3)) : nullptr;
  float* o_rgb = rgb ? reinterpret_cast<float*>(take(a3)) : nullptr;
  int32_t* o_counts = counts ? reinterpret_cast<int32_t*>(take(a1)) : nullptr;
  int32_t* o_first = first ? reinterpret_cast<int32_t*>(take(a1)) : nullptr;
  int32_t* o_voxel_of = voxel_of ? reinterpret_cast<int32_t*>(take(a1)) : nullptr;
  int64_t* o_n = reinterpret_cast<int64_t*>(take(256));
  S4G_CUDA(cudaMemcpyAsync(d_xyz, xyz, 12 * N, cudaMemcpyHostToDevice, st));
  if (normals) S4G_CUDA(cudaMemcpyAsync(d_nrm, normals, 12 * N, cudaMemcpyHostToDevice, st));
  if (rgb) S4G_CUDA(cudaMemcpyAsync(d_rgb, rgb, 12 * N, cudaMemcpyHostToDevice, st));
  VgMeta* d_meta = nullptr;
  S4G_TRY(launch(ctx, d_xyz, d_nrm, d_rgb, n, leaf, min_points, o_xyz, o_nrm, o_rgb, o_counts, o_first, o_voxel_of, o_n,
                 &d_meta));
  int64_t m = 0;
  VgMeta meta;
  S4G_CUDA(cudaMemcpyAsync(&m, o_n, sizeof m, cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaMemcpyAsync(&meta, d_meta, sizeof meta, cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  if (m < 0) {
    ctx->err = meta.bad ? "s4g_voxel_grid: a coordinate is not finite or its scaled floor is outside the int32 range"
                        : "s4g_voxel_grid: the cloud spans 2^21 or more voxels along an axis";
    return S4G_ERR_ARG;
  }
  const size_t M = (size_t)m;
  S4G_CUDA(cudaMemcpyAsync(xyz_out, o_xyz, 12 * M, cudaMemcpyDeviceToHost, st));
  if (normals) S4G_CUDA(cudaMemcpyAsync(normals_out, o_nrm, 12 * M, cudaMemcpyDeviceToHost, st));
  if (rgb) S4G_CUDA(cudaMemcpyAsync(rgb_out, o_rgb, 12 * M, cudaMemcpyDeviceToHost, st));
  if (counts) S4G_CUDA(cudaMemcpyAsync(counts, o_counts, 4 * M, cudaMemcpyDeviceToHost, st));
  if (first) S4G_CUDA(cudaMemcpyAsync(first, o_first, 4 * M, cudaMemcpyDeviceToHost, st));
  if (voxel_of) S4G_CUDA(cudaMemcpyAsync(voxel_of, o_voxel_of, 4 * N, cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  *n_out = m;
  return S4G_OK;
}
