// Context, cloud upload and grid construction of libs4g.so.
//
// s4g_set_cloud_p  replaces Match4PCSBase::initKdTree (reference algorithms/match4pcsBase.cc:
//                  353-363; accelerators/kdtree.h:349-364,554-635): instead of a kd-tree the
//                  device holds a bricked uniform grid (cell edge ~2*delta) over the centred
//                  sampled P, a summed-area table of its coarse occupancy (tile cull) and the
//                  "delta-field" (2 bits per voxel of edge h/4, 2 x 8 bits per boundary voxel for its
//                  sub-voxels: is any / is certainly some P point within delta of this location?)
//                  that lets Verify decide most (query, candidate) pairs without a point test.
// s4g_set_cloud_q  replaces PairCreationFunctor::synch3DContent (reference
//                  algorithms/pairCreationFunctor.h:90-122).
#include "s4g_internal.cuh"
#include <cub/cub.cuh>
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <vector>

// Scratch buffers grow through the device's stream-ordered memory pool (cudaMallocAsync / cudaFreeAsync on the context's
// stream): unlike cudaFree + cudaMalloc -- which synchronise the WHOLE device, i.e. every other context on it: the lanes
// of row f1, the peers of S4PCS_DEVICES -- a re-allocation only orders against this context's own stream, and the pool
// keeps freed blocks (release threshold = max) so that growth is a sub-allocation after the first few bases.
int s4g_reserve(s4g_ctx* ctx, DevBuf& b, size_t bytes) {
  if (bytes <= b.cap) return S4G_OK;
  if (b.p) S4G_CUDA(cudaFreeAsync(b.p, ctx->stream));
  b.p = nullptr;
  b.cap = 0;
  // geometric growth from a 1 MiB floor so that a context settles after a few bases; large buffers (>= 256 MiB) keep
  // 25 % head-room.  Falls back to the exact size.
  size_t want = bytes < (size_t(256) << 20) ? (2 * bytes > (size_t(1) << 20) ? 2 * bytes : (size_t(1) << 20))
                                            : bytes + bytes / 4 + 256;
  cudaError_t e = cudaMallocAsync(&b.p, want, ctx->stream);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    e = cudaMallocAsync(&b.p, bytes, ctx->stream);
    want = bytes;
  }
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    char m[160];
    snprintf(m, sizeof m, "device allocation of %zu bytes failed: %s", bytes, cudaGetErrorString(e));
    ctx->err = m;
    b.p = nullptr;
    return S4G_ERR_NOMEM;
  }
  b.cap = want;
  return S4G_OK;
}

static void free_buf(s4g_ctx* ctx, DevBuf& b) {
  if (b.p) cudaFreeAsync(b.p, ctx->stream);
  b.p = nullptr;
  b.cap = 0;
}

extern "C" int s4g_abi_version(void) { return S4G_ABI_VERSION; }

extern "C" int s4g_device_count(int* out_count) {
  if (!out_count) return S4G_ERR_ARG;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
    (void)cudaGetLastError();
    *out_count = 0;
    return S4G_ERR_CUDA;
  }
  *out_count = ndev;
  return S4G_OK;
}

extern "C" int s4g_create(int device, s4g_ctx** out_ctx) {
  if (!out_ctx) return S4G_ERR_ARG;
  *out_ctx = nullptr;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
    (void)cudaGetLastError();
    return S4G_ERR_CUDA;  // no CUDA device: there is deliberately no CPU fallback
  }
  s4g_ctx* ctx = new s4g_ctx;
  ctx->device = device;
  if (cudaSetDevice(device) != cudaSuccess ||
      cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking) != cudaSuccess) {
    (void)cudaGetLastError();
    delete ctx;
    return S4G_ERR_CUDA;
  }
  ctx->stream = ctx->own_stream;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 2; ++j)
      if (cudaEventCreate(&ctx->ev[i][j]) != cudaSuccess) {
        (void)cudaGetLastError();
        delete ctx;
        return S4G_ERR_CUDA;
      }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) {
    ctx->sm_count = prop.multiProcessorCount;
    if (prop.l2CacheSize > 0) ctx->l2_bytes = prop.l2CacheSize;
  }
  // A/B knob: a fixed number of query patches for Verify instead of the one derived from the L2 size (verify.cu)
  if (const char* e = std::getenv("S4G_VERIFY_PATCHES")) ctx->verify_patches = std::max(0, std::min(kVerifyMaxPatches, std::atoi(e)));
  // test knob: a smaller window of the per-list sort of s4g_range, so that small results take its multi-chunk path
  if (const char* e = std::getenv("S4G_RANGE_SORT_WINDOW")) ctx->range_window = std::max(0ll, std::atoll(e));
  {
    // keep freed scratch in the pool instead of returning it to the driver at every synchronisation
    cudaMemPool_t pool = nullptr;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
      unsigned long long keep = ~0ull;
      (void)cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    (void)cudaGetLastError();
  }
  ctx->hPinnedBytes = 1 << 16;
  if (cudaMallocHost(&ctx->hPinned, ctx->hPinnedBytes) != cudaSuccess) {
    (void)cudaGetLastError();
    ctx->hPinned = nullptr;
  }
  *out_ctx = ctx;
  return S4G_OK;
}

extern "C" void s4g_destroy(s4g_ctx* ctx) {
  if (!ctx) return;
  if (ctx->stuck) return;  // (comm.cu: the stream holds a collective that can never finish; nothing to wait for or to free)
  if (ctx->comm) (void)s4g_comm_destroy(ctx);
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  DevBuf* all[] = {&ctx->dP, &ctx->dPsorted, &ctx->dTop, &ctx->dCellStart, &ctx->dCsat, &ctx->dVtop, &ctx->dVox, &ctx->dVocc, &ctx->dVbase, &ctx->dVfine, &ctx->dQtiles, &ctx->dQmside, &ctx->dQ, &ctx->dQmorton,
                   &ctx->dQn, &ctx->dQrgb, &ctx->dQunit, &ctx->dQgroups, &ctx->dPairs[0], &ctx->dPairs[1], &ctx->dQuads,
                   &ctx->dScratchA, &ctx->dScratchB, &ctx->dScratchC, &ctx->dScratchD, &ctx->dCub,
                   &ctx->dRms, &ctx->dOk, &ctx->dCandIdx, &ctx->dCounts, &ctx->dResult,
                   &ctx->dMisc, &ctx->bArgs, &ctx->bCounts, &ctx->bPairKeys[0], &ctx->bPairKeys[1], &ctx->bQKeys[0], &ctx->bQKeys[1],
                   &ctx->bQVals[0], &ctx->bQVals[1], &ctx->bQCnt, &ctx->bQuadKeys[0], &ctx->bQuadKeys[1], &ctx->bQuads, &ctx->bMisc,
                   &ctx->bResults, &ctx->dQpatch, &ctx->dVrec, &ctx->dVsort, &ctx->dRangeOff, &ctx->dRangeIdx,
                   &ctx->dRangeSq, &ctx->dFilter};
  for (DevBuf* b : all) free_buf(ctx, *b);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->hPinned) cudaFreeHost(ctx->hPinned);
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 2; ++j)
      if (ctx->ev[i][j]) cudaEventDestroy(ctx->ev[i][j]);
  if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
  delete ctx;
}

extern "C" const char* s4g_error_string(const s4g_ctx* ctx) {
  return ctx ? ctx->err.c_str() : "null context";
}

extern "C" int s4g_set_stream(s4g_ctx* ctx, void* cuda_stream) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_CUDA(cudaSetDevice(ctx->device));
  S4G_CUDA(cudaStreamSynchronize(ctx->stream));
  ctx->stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : ctx->own_stream;
  return S4G_OK;
}

extern "C" int s4g_synchronize(s4g_ctx* ctx) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_CUDA(cudaSetDevice(ctx->device));
  S4G_CUDA(cudaStreamSynchronize(ctx->stream));
  return S4G_OK;
}

extern "C" int s4g_get_timings(s4g_ctx* ctx, double* out5) {
  if (!ctx || !out5) return S4G_ERR_ARG;
  S4G_CUDA(cudaSetDevice(ctx->device));
  for (int i = 0; i < 4; ++i) {
    if (ctx->ev_pending[i]) {
      float ms = 0.f;
      S4G_CUDA(cudaEventSynchronize(ctx->ev[i][1]));
      if (cudaEventElapsedTime(&ms, ctx->ev[i][0], ctx->ev[i][1]) == cudaSuccess) ctx->ms[i] = ms;
      else (void)cudaGetLastError();
      ctx->ev_pending[i] = false;
    }
    out5[i] = ctx->ms[i];
  }
  out5[4] = (double)ctx->launches;
  return S4G_OK;
}

// =============================================================================================
// grid over P
// =============================================================================================
__global__ void k_pack_xyz(const float* __restrict__ xyz, int n, float4* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = make_float4(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], __int_as_float(i));
}

__device__ __forceinline__ int3 cell_of(const GridDev& g, float x, float y, float z) {
  int cx = (int)floorf((x - g.ox) * g.inv_h);
  int cy = (int)floorf((y - g.oy) * g.inv_h);
  int cz = (int)floorf((z - g.oz) * g.inv_h);
  cx = min(max(cx, 0), g.nx - 1);
  cy = min(max(cy, 0), g.ny - 1);
  cz = min(max(cz, 0), g.nz - 1);
  return make_int3(cx, cy, cz);
}

__global__ void k_mark_bricks(GridDev g, const float4* __restrict__ P, int n, int* __restrict__ top) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 p = P[i];
  int3 c = cell_of(g, p.x, p.y, p.z);
  top[brick_index(g, c.x, c.y, c.z)] = 1;
}

__global__ void k_rank_bricks(int* __restrict__ top, const int* __restrict__ excl, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  top[i] = top[i] ? excl[i] : -1;
}

__global__ void k_cell_keys(GridDev g, const float4* __restrict__ P, int n, uint32_t* __restrict__ keys,
                            uint32_t* __restrict__ vals, uint32_t* __restrict__ cellCount) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 p = P[i];
  int3 c = cell_of(g, p.x, p.y, p.z);
  uint32_t key = cell_slot(g, g.top[brick_index(g, c.x, c.y, c.z)], c.x, c.y, c.z);
  keys[i] = key;
  vals[i] = (uint32_t)i;
  atomicAdd(&cellCount[key], 1u);
}

// coarse occupancy flags (turned into a summed-area table by k_sat_scan) for the tile cull of Verify
__global__ void k_mark_coarse(GridDev g, const float4* __restrict__ P, int n, uint32_t* __restrict__ csat) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 p = P[i];
  int3 c = cell_of(g, p.x, p.y, p.z);
  const uint32_t X = (uint32_t)(c.x >> g.cshift) + 1u, Y = (uint32_t)(c.y >> g.cshift) + 1u, Z = (uint32_t)(c.z >> g.cshift) + 1u;
  csat[csat_slot(g, X, Y, Z)] = 1u;
}

// occupancy nibbles of the 2x2x2-cell blocks the exact test of Verify probes (GridDev::vocc): a point in cell c marks
// row (dy, dz) of the 8 blocks with origin c - (dx, dy, dz).  Origins are >= 0: the grid has a 1.5-cell margin.
__global__ void k_mark_vocc(GridDev g, const float4* __restrict__ P, int n, uint32_t* __restrict__ vocc, unsigned int* __restrict__ err) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 p = P[i];
  int3 c = cell_of(g, p.x, p.y, p.z);
#pragma unroll
  for (int d = 0; d < 8; ++d) {
    const int dx = d & 1, dy = (d >> 1) & 1, dz = d >> 2;
    const int ox = c.x - dx, oy = c.y - dy, oz = c.z - dz;
    if (ox < 0 || oy < 0 || oz < 0) { atomicAdd(err, 1u); continue; }
    const int rank = g.vtop[brick_index(g, ox, oy, oz)];
    if (rank < 0) { atomicAdd(err, 1u); continue; }              // cannot happen: k_mark_vbricks marks every origin's brick
    const uint32_t cell = cell_slot(g, rank, ox, oy, oz);
    const uint32_t bit = 1u << (vocc_shift(cell) + (uint32_t)(dz * 2 + dy));
    if (!(vocc[vocc_word(cell)] & bit)) atomicOr(&vocc[vocc_word(cell)], bit);
  }
}

// in-place inclusive prefix sum of the (nx1 x ny1 x nz1) table along one axis; one thread per line
__global__ void k_sat_scan(uint32_t* __restrict__ t, int nx1, int ny1, int nz1, int axis) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int len, lines, stride;
  size_t base;
  if (axis == 0) { len = nx1; lines = ny1 * nz1; stride = 1; base = (size_t)i * nx1; }
  else if (axis == 1) { len = ny1; lines = nx1 * nz1; stride = nx1; base = (size_t)(i / nx1) * nx1 * ny1 + (i % nx1); }
  else { len = nz1; lines = nx1 * ny1; stride = nx1 * ny1; base = (size_t)i; }
  if (i >= lines) return;
  uint32_t acc = 0;
  for (int k = 0; k < len; ++k) {
    acc += t[base + (size_t)k * stride];
    t[base + (size_t)k * stride] = acc;
  }
}

__global__ void k_gather_f4(const float4* __restrict__ src, const uint32_t* __restrict__ idx, int n,
                            float4* __restrict__ dst) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  dst[i] = src[idx[i]];
}

// ---- delta-field (see GridDev::vox): v-bricks = bricks within `reach` of a P point: every brick the box p +- reach
// touches.  For centred clouds reach is below one cell and these are the bricks of the box's 8 corners; far from the
// origin the field's slack grows with the coordinates and the box can span several bricks per axis.
__global__ void k_mark_vbricks(GridDev g, const float4* __restrict__ P, int n, float reach, int* __restrict__ vtop) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float4 p = P[i];
  const int3 a = cell_of(g, p.x - reach, p.y - reach, p.z - reach), b = cell_of(g, p.x + reach, p.y + reach, p.z + reach);
  const int bs = g.bshift;
  for (int z = a.z >> bs; z <= b.z >> bs; ++z)
    for (int y = a.y >> bs; y <= b.y >> bs; ++y)
      for (int x = a.x >> bs; x <= b.x >> bs; ++x) vtop[brick_index(g, x << bs, y << bs, z << bs)] = 1;
  // ... and the origin cells c - (dx, dy, dz) of the 2x2x2 blocks that contain the point's cell (GridDev::vocc lives there)
  const int3 c = cell_of(g, p.x, p.y, p.z);
#pragma unroll
  for (int d = 0; d < 8; ++d) {
    const int ox = max(c.x - (d & 1), 0), oy = max(c.y - ((d >> 1) & 1), 0), oz = max(c.z - (d >> 2), 0);
    vtop[brick_index(g, ox, oy, oz)] = 1;
  }
}

// The delta-field builders: one warp per P point visits each of the (2R+1)^3 voxels around it inside the lattice; voxel k
// spans [ox + k v, ox + (k+1) v) per axis, v = 1 / inv_v.  Double: conservative, not bit-compatible with anything.
struct FieldPoint { double px, py, pz, ox, oy, oz, v, r_maybe, r_cert; };
template <class Visit>
__device__ __forceinline__ void for_voxels_near(const GridDev& g, const float4* __restrict__ P, int n, int R, double delta,
                                                double md, Visit visit) {
  const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= n) return;
  const float4 pf = P[gw];
  const double v = 1.0 / (double)g.inv_v;
  const double px = pf.x, py = pf.y, pz = pf.z, ox = g.ox, oy = g.oy, oz = g.oz;
  const long long kx = (long long)floor((px - ox) / v), ky = (long long)floor((py - oy) / v),
                  kz = (long long)floor((pz - oz) / v);
  const int side = 2 * R + 1, total = side * side * side;
  const FieldPoint f{px, py, pz, ox, oy, oz, v, (delta + md) * (delta + md), delta > md ? (delta - md) * (delta - md) : -1.0};
  for (int o = lane; o < total; o += 32) {
    const int dz = o / (side * side) - R, dy = (o / side) % side - R, dx = o % side - R;
    const long long X = kx + dx, Y = ky + dy, Z = kz + dz;
    if (X < 0 || Y < 0 || Z < 0 || X >= 4ll * g.nx || Y >= 4ll * g.ny || Z >= 4ll * g.nz) continue;
    visit((int)X, (int)Y, (int)Z, f);
  }
}
// squared distances from the point of f to the nearest (x) and the farthest (y) location of the box [lo, hi]
__device__ __forceinline__ double2 box_dist2(const FieldPoint& f, double lx, double ly, double lz, double hx, double hy,
                                             double hz) {
  const double nx_ = fmax(0.0, fmax(lx - f.px, f.px - hx)), ny_ = fmax(0.0, fmax(ly - f.py, f.py - hy)),
               nz_ = fmax(0.0, fmax(lz - f.pz, f.pz - hz));
  const double fx = fmax(f.px - lx, hx - f.px), fy = fmax(f.py - ly, hy - f.py), fz = fmax(f.pz - lz, hz - f.pz);
  return make_double2(nx_ * nx_ + ny_ * ny_ + nz_ * nz_, fx * fx + fy * fy + fz * fz);
}

// Classify the voxels around every P point.  The box is inflated by `slack` (position uncertainty of the query's voxel)
// and the radius by +-md (rounding of the fp32 decision d^2 <= delta^2), so that
//   MAYBE clear   =>  no location of the voxel is within delta of this point  (for every point: no inlier possible)
//   CERTAIN set   =>  every location of the voxel is within delta of this point (inlier, whatever the exact position)
__global__ void k_mark_voxels(GridDev g, const float4* __restrict__ P, int n, int R, double delta, double slack,
                              double md, uint32_t* __restrict__ vox, unsigned int* __restrict__ err) {
  for_voxels_near(g, P, n, R, delta, md, [&](int X, int Y, int Z, const FieldPoint& f) {
    const double2 d = box_dist2(f, f.ox + (double)X * f.v - slack, f.oy + (double)Y * f.v - slack, f.oz + (double)Z * f.v - slack,
                                f.ox + (double)(X + 1) * f.v + slack, f.oy + (double)(Y + 1) * f.v + slack,
                                f.oz + (double)(Z + 1) * f.v + slack);
    if (!(d.x <= f.r_maybe)) return;
    const int rank = g.vtop[brick_index<0, 2>(g, X, Y, Z)];
    if (rank < 0) { atomicAdd(err, 1u); return; }   // cannot happen (k_mark_vbricks is a superset); checked by the host
    const uint32_t word = vox_word(vox_cell(g, rank, X, Y, Z), Z);
    const uint32_t bits = (d.y <= f.r_cert ? 3u : 1u) << vox_shift(X, Y);
    if ((vox[word] & bits) != bits) atomicOr(&vox[word], bits);
  });
}

// per cell of the v-bricks: number of boundary voxels (-> exclusive scan = GridDev::vbase)
__global__ void k_count_boundary(const uint32_t* __restrict__ vox, long long nCells, uint32_t* __restrict__ counts) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nCells) return;
  const uint4 w = vox_cells(vox)[i];
  counts[i] = (uint32_t)(__popc(boundary_bits(w.x)) + __popc(boundary_bits(w.y)) + __popc(boundary_bits(w.z)) +
                         __popc(boundary_bits(w.w)));
}

// Second level of the delta-field: for every boundary voxel within reach of a point, classify its 2x2x2 sub-voxels
// against that point exactly like k_mark_voxels classifies voxels (same margins).
__global__ void k_mark_subvoxels(GridDev g, const float4* __restrict__ P, int n, int R, double delta, double slack,
                                 double md, uint32_t* __restrict__ fine32) {
  for_voxels_near(g, P, n, R, delta, md, [&](int X, int Y, int Z, const FieldPoint& f) {
    const double v = f.v, hv = 0.5 * v;
    const double lx = f.ox + (double)X * v, ly = f.oy + (double)Y * v, lz = f.oz + (double)Z * v;   // voxel's low corner
    if (!(box_dist2(f, lx - slack, ly - slack, lz - slack, lx + v + slack, ly + v + slack, lz + v + slack).x <= f.r_maybe))
      return;                                                                   // no child can be MAYBE for this point
    const int rank = g.vtop[brick_index<0, 2>(g, X, Y, Z)];
    if (rank < 0) return;
    const uint32_t cell = vox_cell(g, rank, X, Y, Z);
    const uint4 cw = vox_cells(g.vox)[cell];
    const uint32_t ws[4] = {cw.x, cw.y, cw.z, cw.w}, w = ws[Z & 3];
    const uint32_t sh = vox_shift(X, Y);
    if (((boundary_bits(w) >> sh) & 1u) == 0u) return;                        // voxel decided at the first level
    const uint32_t slot = boundary_slot(g.vbase[cell], cw, w, Z & 3, sh);
    uint32_t bits = 0u;
#pragma unroll
    for (int ch = 0; ch < 8; ++ch) {
      const double ax = lx + ((ch & 1) ? hv : 0.0) - slack, bx = ax + hv + 2.0 * slack;
      const double ay = ly + ((ch & 2) ? hv : 0.0) - slack, by = ay + hv + 2.0 * slack;
      const double az = lz + ((ch & 4) ? hv : 0.0) - slack, bz = az + hv + 2.0 * slack;
      const double2 d = box_dist2(f, ax, ay, az, bx, by, bz);
      if (d.x <= f.r_maybe) bits |= fine_maybe(ch);
      if (d.y <= f.r_cert) bits |= fine_certain(ch);
    }
    if (bits) {
      const uint32_t word = fine_word(slot), s16 = fine_half(slot);
      if (((fine32[word] >> s16) & bits) != bits) atomicOr(&fine32[word], bits << s16);
    }
  });
}

static inline int nblk(long long n, int t) { return (int)((n + t - 1) / t); }

// brick flags (1 = marked) -> ranks (exclusive prefix, -1 where unmarked), count = marked bricks; count >= limit fails first
static int rank_flags(s4g_ctx* ctx, int* flags, long long ntop, long long limit, const char* too_many, long long& count) {
  cudaStream_t st = ctx->stream;
  size_t cub_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, cub_bytes, flags, ctx->dScratchB.as<int>(), (int)ntop, st);
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, cub_bytes));
  cub::DeviceScan::ExclusiveSum(ctx->dCub.p, cub_bytes, flags, ctx->dScratchB.as<int>(), (int)ntop, st);
  int last_flag = 0, last_excl = 0;
  S4G_CUDA(cudaMemcpyAsync(&last_flag, flags + (ntop - 1), sizeof(int), cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaMemcpyAsync(&last_excl, ctx->dScratchB.as<int>() + (ntop - 1), sizeof(int), cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  count = (long long)last_flag + last_excl;
  if (count >= limit) { ctx->err = too_many; return S4G_ERR_NOMEM; }
  k_rank_bricks<<<nblk(ntop, 256), 256, 0, st>>>(flags, ctx->dScratchB.as<int>(), (int)ntop);
  return S4G_OK;
}

// zero the error word dMisc[0], enqueue launch(word), then fail with `msg` if a thread counted an error in it
template <class Launch>
static int launch_checked(s4g_ctx* ctx, const char* msg, Launch launch) {
  S4G_CUDA(cudaMemsetAsync(ctx->dMisc.p, 0, 4, ctx->stream));
  launch(ctx->dMisc.as<unsigned int>());
  S4G_CUDA(cudaGetLastError());
  unsigned int err = 0;
  S4G_CUDA(cudaMemcpyAsync(&err, ctx->dMisc.p, 4, cudaMemcpyDeviceToHost, ctx->stream));
  S4G_CUDA(cudaStreamSynchronize(ctx->stream));
  if (err) { ctx->err = msg; return S4G_ERR_CUDA; }
  return S4G_OK;
}

extern "C" int s4g_set_cloud_p(s4g_ctx* ctx, const float* xyz, int n, float delta) {
  if (!ctx) return S4G_ERR_ARG;
  if (!xyz || n <= 0 || !(delta > 0.f)) {
    ctx->err = "s4g_set_cloud_p: need xyz != NULL, n > 0, delta > 0";
    return S4G_ERR_ARG;
  }
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  ctx->nP = 0;

  // bounding box on the host while the upload is in flight
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, (size_t)n * 3 * sizeof(float)));
  S4G_CUDA(cudaMemcpyAsync(ctx->dScratchA.p, xyz, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, st));
  float mn[3] = {xyz[0], xyz[1], xyz[2]}, mx[3] = {xyz[0], xyz[1], xyz[2]};
  for (int i = 0; i < n; ++i)
    for (int k = 0; k < 3; ++k) {
      float v = xyz[3 * i + k];
      if (!std::isfinite(v)) { ctx->err = "s4g_set_cloud_p: NaN or infinite coordinate"; return S4G_ERR_ARG; }
      mn[k] = std::min(mn[k], v);
      mx[k] = std::max(mx[k], v);
    }

  // cell edge: >= 2*delta*(1+1%) so that the 2x2x2 octant probe of Verify provably covers the
  // delta-ball whatever the float rounding of the cell coordinates (see verify.cu).
  double h = 2.0 * (double)delta * 1.01;
  const double kMaxCellsPerAxis = 2000.0;  // keeps the cell-coordinate rounding far below the probe margin
  double ext = std::max({(double)mx[0] - mn[0], (double)mx[1] - mn[1], (double)mx[2] - mn[2]});
  if (ext / h > kMaxCellsPerAxis) h = ext / kMaxCellsPerAxis;
  GridDev g{};
  int bs = 2;
  long long ntop = 0;
  for (;;) {
    g.ox = (float)(mn[0] - 1.5 * h);
    g.oy = (float)(mn[1] - 1.5 * h);
    g.oz = (float)(mn[2] - 1.5 * h);
    g.inv_h = (float)(1.0 / h);
    g.nx = (int)std::ceil((mx[0] - g.ox) / h) + 2;
    g.ny = (int)std::ceil((mx[1] - g.oy) / h) + 2;
    g.nz = (int)std::ceil((mx[2] - g.oz) / h) + 2;
    for (bs = 2; bs <= 6; ++bs) {
      int B = 1 << bs;
      g.tbx = (g.nx + B - 1) / B;
      g.tby = (g.ny + B - 1) / B;
      g.tbz = (g.nz + B - 1) / B;
      ntop = (long long)g.tbx * g.tby * g.tbz;
      if (ntop <= (1ll << 24)) break;
    }
    if (ntop <= (1ll << 24)) break;
    h *= 1.5;
  }
  g.bshift = bs;

  S4G_TRY(s4g_reserve(ctx, ctx->dP, (size_t)n * sizeof(float4)));
  S4G_TRY(s4g_reserve(ctx, ctx->dPsorted, (size_t)n * sizeof(float4)));
  S4G_TRY(s4g_reserve(ctx, ctx->dTop, (size_t)ntop * sizeof(int)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, (size_t)ntop * sizeof(int)));
  k_pack_xyz<<<nblk(n, 256), 256, 0, st>>>(ctx->dScratchA.as<float>(), n, ctx->dP.as<float4>());
  S4G_CUDA(cudaMemsetAsync(ctx->dTop.p, 0, (size_t)ntop * sizeof(int), st));
  g.top = ctx->dTop.as<int>();
  k_mark_bricks<<<nblk(n, 256), 256, 0, st>>>(g, ctx->dP.as<float4>(), n, ctx->dTop.as<int>());
  long long nBricks = 0;
  S4G_TRY(rank_flags(ctx, ctx->dTop.as<int>(), ntop, 1ll << (31 - 3 * bs),   // i.e. nBricks << 3*bs cells >= 2^31
                     "s4g_set_cloud_p: grid too large (cells >= 2^31); delta too small for this cloud", nBricks));
  long long nCells = nBricks << (3 * bs);

  S4G_TRY(s4g_reserve(ctx, ctx->dCellStart, (size_t)(nCells + 1) * sizeof(uint32_t)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchC, (size_t)(nCells + 1) * sizeof(uint32_t)));  // counts
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, (size_t)n * 4 * sizeof(uint32_t)));         // keys/vals in+out
  uint32_t* keys_in = ctx->dScratchB.as<uint32_t>();
  uint32_t* vals_in = keys_in + n;
  uint32_t* keys_out = vals_in + n;
  uint32_t* vals_out = keys_out + n;
  S4G_CUDA(cudaMemsetAsync(ctx->dScratchC.p, 0, (size_t)(nCells + 1) * sizeof(uint32_t), st));
  k_cell_keys<<<nblk(n, 256), 256, 0, st>>>(g, ctx->dP.as<float4>(), n, keys_in, vals_in,
                                            ctx->dScratchC.as<uint32_t>());
  int key_bits = 1;
  while ((1ll << key_bits) < nCells && key_bits < 32) ++key_bits;
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, keys_in, keys_out, vals_in, vals_out, n, 0, key_bits, st);
  size_t scan_bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, ctx->dScratchC.as<uint32_t>(),
                                ctx->dCellStart.as<uint32_t>(), (int)(nCells + 1), st);
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, std::max(cub_bytes, scan_bytes)));
  cub::DeviceRadixSort::SortPairs(ctx->dCub.p, cub_bytes, keys_in, keys_out, vals_in, vals_out, n, 0, key_bits, st);
  cub::DeviceScan::ExclusiveSum(ctx->dCub.p, scan_bytes, ctx->dScratchC.as<uint32_t>(),
                                ctx->dCellStart.as<uint32_t>(), (int)(nCells + 1), st);
  k_gather_f4<<<nblk(n, 256), 256, 0, st>>>(ctx->dP.as<float4>(), vals_out, n, ctx->dPsorted.as<float4>());
  ctx->launches += 6 + 8;
  S4G_CUDA(cudaGetLastError());
  S4G_CUDA(cudaStreamSynchronize(st));

  g.cellStart = ctx->dCellStart.as<uint32_t>();
  g.pts = ctx->dPsorted.as<float4>();
  g.csat = nullptr;
  g.vocc = nullptr;
  // coarse blocks for the tile cull: as fine as a 1M-entry (4 MB) summed-area table allows -- 4x4x4 cells at 1M points.
  // (2x2x2-cell blocks cull a few more (warp, candidate) pairs, but their table is 8x larger and competes with the rest
  // of the working set for L2; S4G_CSHIFT_MIN selects coarser blocks for an A/B.)
  int cshift_min = 1;
  if (const char* e = std::getenv("S4G_CSHIFT_MIN")) cshift_min = std::max(1, std::min(11, std::atoi(e)));   // A/B knob: coarser cull blocks
  for (g.cshift = cshift_min; g.cshift < 12; ++g.cshift) {
    g.cnx = (g.nx >> g.cshift) + 1;
    g.cny = (g.ny >> g.cshift) + 1;
    g.cnz = (g.nz >> g.cshift) + 1;
    if ((unsigned long long)(g.cnx + 1) * (g.cny + 1) * (g.cnz + 1) <= (1ull << 20)) break;
  }
  {
    const size_t sat = (size_t)(g.cnx + 1) * (g.cny + 1) * (g.cnz + 1);
    S4G_TRY(s4g_reserve(ctx, ctx->dCsat, sat * sizeof(uint32_t)));
    S4G_CUDA(cudaMemsetAsync(ctx->dCsat.p, 0, sat * sizeof(uint32_t), st));
    k_mark_coarse<<<nblk(n, 256), 256, 0, st>>>(g, ctx->dP.as<float4>(), n, ctx->dCsat.as<uint32_t>());
    const int nx1 = g.cnx + 1, ny1 = g.cny + 1, nz1 = g.cnz + 1;
    k_sat_scan<<<nblk((long long)ny1 * nz1, 128), 128, 0, st>>>(ctx->dCsat.as<uint32_t>(), nx1, ny1, nz1, 0);
    k_sat_scan<<<nblk((long long)nx1 * nz1, 128), 128, 0, st>>>(ctx->dCsat.as<uint32_t>(), nx1, ny1, nz1, 1);
    k_sat_scan<<<nblk((long long)nx1 * ny1, 128), 128, 0, st>>>(ctx->dCsat.as<uint32_t>(), nx1, ny1, nz1, 2);
    ctx->launches += 4;
    S4G_CUDA(cudaGetLastError());
    g.csat = ctx->dCsat.as<uint32_t>();
  }
  {
    // delta-field: v-brick table, then 2 bits per voxel (edge h/4)
    g.inv_v = 4.f * g.inv_h;
    const double v = 1.0 / (double)g.inv_v;
    double pabs = 0.0;
    for (int k = 0; k < 3; ++k) pabs = std::max({pabs, std::fabs((double)mn[k]), std::fabs((double)mx[k])});
    // position uncertainty the field tolerates: 2 % of a voxel, or the fp32 rounding of a rigid motion of clouds of this
    // extent if that is larger (k_verify checks every candidate against it and otherwise derives the voxel from the exact T q)
    const double slack = std::max(0.02 * v, std::ldexp(8.0 * (1.0 + pabs), -20));
    const double md = 1e-5 * (double)delta + std::ldexp(1.0 + pabs, -40);
    g.vslack = (float)(slack * 0.999);
    const double reach = (double)delta + md + slack;
    const int R = (int)std::ceil(1.0 + reach / v);   // voxels further than (|d| - 1) v - slack > delta + md can hold no bit
    S4G_TRY(s4g_reserve(ctx, ctx->dVtop, (size_t)ntop * sizeof(int)));
    S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, (size_t)ntop * sizeof(int)));
    S4G_CUDA(cudaMemsetAsync(ctx->dVtop.p, 0, (size_t)ntop * sizeof(int), st));
    k_mark_vbricks<<<nblk(n, 256), 256, 0, st>>>(g, ctx->dP.as<float4>(), n, (float)(reach * 1.05 + 1e-3 * h),
                                                 ctx->dVtop.as<int>());
    long long nVB = 0;
    S4G_TRY(rank_flags(ctx, ctx->dVtop.as<int>(), ntop, LLONG_MAX, nullptr, nVB));
    const size_t vwords = ((size_t)nVB << (3 * bs)) * 4;
    if (vwords >= (size_t(1) << 32)) {
      ctx->err = "s4g_set_cloud_p: delta-field too large (>= 16 GiB); delta too small for this cloud";
      return S4G_ERR_NOMEM;
    }
    S4G_TRY(s4g_reserve(ctx, ctx->dVox, std::max<size_t>(vwords, 4) * sizeof(uint32_t)));
    S4G_TRY(s4g_reserve(ctx, ctx->dMisc, 256));
    S4G_CUDA(cudaMemsetAsync(ctx->dVox.p, 0, std::max<size_t>(vwords, 4) * sizeof(uint32_t), st));
    g.vtop = ctx->dVtop.as<int>();
    g.vox = ctx->dVox.as<uint32_t>();
    ctx->launches += 5;
    S4G_TRY(launch_checked(ctx, "s4g_set_cloud_p: internal error (delta-field voxel outside its v-bricks)", [&](unsigned int* err) {
      k_mark_voxels<<<nblk((long long)n * 32, 256), 256, 0, st>>>(g, ctx->dP.as<float4>(), n, R, (double)delta, slack, md,
                                                                  ctx->dVox.as<uint32_t>(), err);
    }));
    ctx->nVBricks = nVB;
    {
      // occupancy nibbles of the blocks the exact test probes, per origin cell of the v-bricks
      const size_t owords = (size_t)((nVB << (3 * bs)) + 7) / 8 + 1;
      S4G_TRY(s4g_reserve(ctx, ctx->dVocc, owords * sizeof(uint32_t)));
      S4G_CUDA(cudaMemsetAsync(ctx->dVocc.p, 0, owords * sizeof(uint32_t), st));
      ctx->launches++;
      S4G_TRY(launch_checked(ctx, "s4g_set_cloud_p: internal error (block origin outside the v-bricks)", [&](unsigned int* err) {
        k_mark_vocc<<<nblk(n, 256), 256, 0, st>>>(g, ctx->dP.as<float4>(), n, ctx->dVocc.as<uint32_t>(), err);
      }));
      g.vocc = ctx->dVocc.as<uint32_t>();
    }
    // second level: sub-voxel bits of the boundary voxels
    const long long nVCells = nVB << (3 * bs);
    g.vbase = nullptr;
    g.vfine = nullptr;
    ctx->nVBoundary = 0;
    if (nVCells > 0) {
      S4G_TRY(s4g_reserve(ctx, ctx->dVbase, (size_t)(nVCells + 1) * sizeof(uint32_t)));
      S4G_TRY(s4g_reserve(ctx, ctx->dScratchC, (size_t)(nVCells + 1) * sizeof(uint32_t)));
      S4G_CUDA(cudaMemsetAsync(ctx->dScratchC.p, 0, (size_t)(nVCells + 1) * sizeof(uint32_t), st));
      k_count_boundary<<<nblk(nVCells, 256), 256, 0, st>>>(ctx->dVox.as<uint32_t>(), nVCells, ctx->dScratchC.as<uint32_t>());
      size_t sb = 0;
      cub::DeviceScan::ExclusiveSum(nullptr, sb, ctx->dScratchC.as<uint32_t>(), ctx->dVbase.as<uint32_t>(), (long long)(nVCells + 1), st);
      S4G_TRY(s4g_reserve(ctx, ctx->dCub, sb));
      cub::DeviceScan::ExclusiveSum(ctx->dCub.p, sb, ctx->dScratchC.as<uint32_t>(), ctx->dVbase.as<uint32_t>(), (long long)(nVCells + 1), st);
      uint32_t nBnd = 0;
      S4G_CUDA(cudaMemcpyAsync(&nBnd, ctx->dVbase.as<uint32_t>() + nVCells, sizeof nBnd, cudaMemcpyDeviceToHost, st));
      S4G_CUDA(cudaStreamSynchronize(st));
      const size_t fwords = ((size_t)nBnd + 1) / 2 + 1;
      S4G_TRY(s4g_reserve(ctx, ctx->dVfine, fwords * sizeof(uint32_t)));
      S4G_CUDA(cudaMemsetAsync(ctx->dVfine.p, 0, fwords * sizeof(uint32_t), st));
      g.vbase = ctx->dVbase.as<uint32_t>();
      g.vfine = ctx->dVfine.as<uint16_t>();
      k_mark_subvoxels<<<nblk((long long)n * 32, 256), 256, 0, st>>>(g, ctx->dP.as<float4>(), n, R, (double)delta, slack, md,
                                                                     ctx->dVfine.as<uint32_t>());
      ctx->launches += 4;
      S4G_CUDA(cudaGetLastError());
      S4G_CUDA(cudaStreamSynchronize(st));
      ctx->nVBoundary = nBnd;
    }
  }
  ctx->grid = g;
  ctx->nBricks = nBricks;
  ctx->nCells = nCells;
  ctx->cell_h = (float)h;
  ctx->delta = delta;
  ctx->nP = n;
  return S4G_OK;
}

__global__ void k_count_nonempty(const uint32_t* __restrict__ cellStart, long long nCells,
                                 unsigned long long* out) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  int ne = (i < nCells) && (cellStart[i + 1] != cellStart[i]);
  unsigned b = __ballot_sync(0xffffffffu, ne);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(out, (unsigned long long)__popc(b));
}

extern "C" int s4g_get_grid_stats(s4g_ctx* ctx, double* out6) {
  if (!ctx || !out6) return S4G_ERR_ARG;
  if (ctx->nP <= 0) { ctx->err = "s4g_get_grid_stats: no P cloud"; return S4G_ERR_STATE; }
  S4G_CUDA(cudaSetDevice(ctx->device));
  S4G_TRY(s4g_reserve(ctx, ctx->dMisc, 256));
  S4G_CUDA(cudaMemsetAsync(ctx->dMisc.p, 0, 8, ctx->stream));
  k_count_nonempty<<<nblk(ctx->nCells, 256), 256, 0, ctx->stream>>>(ctx->grid.cellStart, ctx->nCells,
                                                                   ctx->dMisc.as<unsigned long long>());
  ctx->launches++;
  unsigned long long ne = 0;
  S4G_CUDA(cudaMemcpyAsync(&ne, ctx->dMisc.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
  S4G_CUDA(cudaStreamSynchronize(ctx->stream));
  out6[0] = ctx->cell_h;
  out6[1] = (double)ctx->nBricks;
  out6[2] = (double)(1 << ctx->grid.bshift);
  out6[3] = (double)ctx->nCells;
  out6[4] = ne ? (double)ctx->nP / (double)ne : 0.0;
  out6[5] = s4g_grid_bytes(ctx);
  return S4G_OK;
}

// Every term is a whole number of bytes (vocc: half a byte per cell) far below 2^53, so the sum is exact in any order.
double s4g_grid_bytes(const s4g_ctx* ctx) {
  const double ntop = (double)ctx->grid.tbx * ctx->grid.tby * ctx->grid.tbz;
  const double vcells = (double)(ctx->nVBricks << (3 * ctx->grid.bshift));
  const double pts = 16.0 * ctx->nP, cellStart = 4.0 * (ctx->nCells + 1), top = 4.0 * ntop, vtop = 4.0 * ntop;
  const double vocc = 0.5 * vcells, vox = 16.0 * vcells, vbase = 4.0 * vcells, vfine = 2.0 * ctx->nVBoundary;
  return pts + cellStart + top + vtop + vocc + vox + vbase + vfine;
}

// =============================================================================================
// Q side
// =============================================================================================
__global__ void k_pack_q(const float* __restrict__ xyz, const float* __restrict__ nrm,
                         const float* __restrict__ rgb, int n, float gx, float gy, float gz, float ratio,
                         float bx, float by, float bz, float mscale, float4* __restrict__ q,
                         float4* __restrict__ qn, float4* __restrict__ qrgb, float4* __restrict__ qunit,
                         uint32_t* __restrict__ mkeys, uint32_t* __restrict__ mvals) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
  q[i] = make_float4(x, y, z, __int_as_float(i));
  qn[i] = nrm ? make_float4(nrm[3 * i], nrm[3 * i + 1], nrm[3 * i + 2], 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
  qrgb[i] = rgb ? make_float4(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2], 0.f) : make_float4(-1.f, -1.f, -1.f, 0.f);
  // worldToUnit, pairCreationFunctor.h:66-70: (p - _gcenter) / _ratio + 0.5
  qunit[i] = make_float4(__fadd_rn(__fdiv_rn(__fsub_rn(x, gx), ratio), 0.5f),
                         __fadd_rn(__fdiv_rn(__fsub_rn(y, gy), ratio), 0.5f),
                         __fadd_rn(__fdiv_rn(__fsub_rn(z, gz), ratio), 0.5f), __int_as_float(i));
  // 30-bit Morton code of the position inside the bounding box (ordering only)
  uint32_t ux = min(1023u, (uint32_t)max(0.f, (x - bx) * mscale));
  uint32_t uy = min(1023u, (uint32_t)max(0.f, (y - by) * mscale));
  uint32_t uz = min(1023u, (uint32_t)max(0.f, (z - bz) * mscale));
  mkeys[i] = morton_spread10(ux) | (morton_spread10(uy) << 1) | (morton_spread10(uz) << 2);
  mvals[i] = (uint32_t)i;
}

// bounding sphere of every run of `tile` Morton-consecutive points (one warp per run): centre of
// the AABB, radius = largest distance to it (rounded up)
__global__ void k_tile_spheres(const float4* __restrict__ qm, int n, int nTiles, int tile, float4* __restrict__ out) {
  int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (t >= nTiles) return;
  float3 lo = make_float3(3.0e38f, 3.0e38f, 3.0e38f), hi = make_float3(-3.0e38f, -3.0e38f, -3.0e38f);
  for (int k = lane; k < tile; k += 32) {
    int i = t * tile + k;
    if (i < n) {
      float4 a = qm[i];
      lo.x = fminf(lo.x, a.x); lo.y = fminf(lo.y, a.y); lo.z = fminf(lo.z, a.z);
      hi.x = fmaxf(hi.x, a.x); hi.y = fmaxf(hi.y, a.y); hi.z = fmaxf(hi.z, a.z);
    }
  }
  warp_aabb(lo, hi);
  float3 c = make_float3(0.5f * (lo.x + hi.x), 0.5f * (lo.y + hi.y), 0.5f * (lo.z + hi.z));
  float r2 = 0.f;
  for (int k = lane; k < tile; k += 32) {
    int i = t * tile + k;
    if (i < n) {
      float4 a = qm[i];
      float dx = a.x - c.x, dy = a.y - c.y, dz = a.z - c.z;
      r2 = fmaxf(r2, dx * dx + dy * dy + dz * dz);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) r2 = fmaxf(r2, __shfl_xor_sync(0xffffffffu, r2, o));
  if (lane == 0) out[t] = make_float4(c.x, c.y, c.z, sqrtf(r2) * 1.0001f + 1e-7f);
}

extern "C" int s4g_set_cloud_q(s4g_ctx* ctx, const float* xyz, const float* normals, const float* rgb, int n) {
  if (!ctx) return S4G_ERR_ARG;
  if (!xyz || n <= 0) { ctx->err = "s4g_set_cloud_q: need xyz != NULL, n > 0"; return S4G_ERR_ARG; }
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  ctx->nQ = 0;
  ctx->patch_np = 0;
  ctx->pair_index_ready = false;
  ctx->nPairs[0] = ctx->nPairs[1] = 0;
  ctx->nQuads = 0;
  size_t b3 = (size_t)n * 3 * sizeof(float);
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, b3 * 3));
  float* d_xyz = ctx->dScratchA.as<float>();
  float* d_nrm = normals ? d_xyz + (size_t)n * 3 : nullptr;
  float* d_rgb = rgb ? d_xyz + (size_t)n * 6 : nullptr;
  S4G_CUDA(cudaMemcpyAsync(d_xyz, xyz, b3, cudaMemcpyHostToDevice, st));
  if (normals) S4G_CUDA(cudaMemcpyAsync(d_nrm, normals, b3, cudaMemcpyHostToDevice, st));
  if (rgb) S4G_CUDA(cudaMemcpyAsync(d_rgb, rgb, b3, cudaMemcpyHostToDevice, st));

  // AABB (Eigen::AlignedBox::extend), centre = (min+max)/2, _ratio = max extent + 0.001 (the
  // literal is a double: float + double -> double -> float), pairCreationFunctor.h:101-111
  float mn[3] = {xyz[0], xyz[1], xyz[2]}, mx[3] = {xyz[0], xyz[1], xyz[2]};
  for (int i = 0; i < n; ++i)
    for (int k = 0; k < 3; ++k) {
      float v = xyz[3 * i + k];
      if (!std::isfinite(v)) { ctx->err = "s4g_set_cloud_q: NaN or infinite coordinate"; return S4G_ERR_ARG; }
      mn[k] = std::min(mn[k], v);
      mx[k] = std::max(mx[k], v);
    }
  for (int k = 0; k < 3; ++k) ctx->gcenter[k] = (mn[k] + mx[k]) / 2.f;
  for (int k = 0; k < 3; ++k) ctx->qabs[k] = std::max(std::fabs(mn[k]), std::fabs(mx[k]));
  float dg[3] = {mx[0] - mn[0], mx[1] - mn[1], mx[2] - mn[2]};
  float mc = std::max(dg[0], std::max(dg[1], dg[2]));
  ctx->ratio = (float)((double)mc + 0.001);
  float mscale = mc > 0 ? 1024.f / mc : 0.f;

  size_t b4 = (size_t)n * sizeof(float4);
  S4G_TRY(s4g_reserve(ctx, ctx->dQ, b4));
  S4G_TRY(s4g_reserve(ctx, ctx->dQn, b4));
  S4G_TRY(s4g_reserve(ctx, ctx->dQrgb, b4));
  S4G_TRY(s4g_reserve(ctx, ctx->dQunit, b4));
  S4G_TRY(s4g_reserve(ctx, ctx->dQmorton, b4));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, (size_t)n * 4 * sizeof(uint32_t)));
  uint32_t* keys_in = ctx->dScratchB.as<uint32_t>();
  uint32_t* vals_in = keys_in + n;
  uint32_t* keys_out = vals_in + n;
  uint32_t* vals_out = keys_out + n;
  k_pack_q<<<nblk(n, 256), 256, 0, st>>>(d_xyz, d_nrm, d_rgb, n, ctx->gcenter[0], ctx->gcenter[1],
                                         ctx->gcenter[2], ctx->ratio, mn[0], mn[1], mn[2], mscale,
                                         ctx->dQ.as<float4>(), ctx->dQn.as<float4>(), ctx->dQrgb.as<float4>(),
                                         ctx->dQunit.as<float4>(), keys_in, vals_in);
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, keys_in, keys_out, vals_in, vals_out, n, 0, 30, st);
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, cub_bytes));
  cub::DeviceRadixSort::SortPairs(ctx->dCub.p, cub_bytes, keys_in, keys_out, vals_in, vals_out, n, 0, 30, st);
  k_gather_f4<<<nblk(n, 256), 256, 0, st>>>(ctx->dQ.as<float4>(), vals_out, n, ctx->dQmorton.as<float4>());
  {
    // Morton-ordered side arrays for the pair predicate (unit coordinates | normals | rgb)
    S4G_TRY(s4g_reserve(ctx, ctx->dQmside, (size_t)n * 3 * sizeof(float4)));
    float4* side = ctx->dQmside.as<float4>();
    k_gather_f4<<<nblk(n, 256), 256, 0, st>>>(ctx->dQunit.as<float4>(), vals_out, n, side);
    k_gather_f4<<<nblk(n, 256), 256, 0, st>>>(ctx->dQn.as<float4>(), vals_out, n, side + n);
    k_gather_f4<<<nblk(n, 256), 256, 0, st>>>(ctx->dQrgb.as<float4>(), vals_out, n, side + 2 * (size_t)n);
    ctx->launches += 3;
  }
  {
    // tile cull of k_verify, two levels: one sphere per kVerifyTile (128) consecutive Morton points and one per kVerifySub
    // (32) = the queries of one warp
    const int nTiles = (n + kVerifyTile - 1) / kVerifyTile, nSubs = (n + kVerifySub - 1) / kVerifySub;
    S4G_TRY(s4g_reserve(ctx, ctx->dQtiles, (size_t)(nTiles + nSubs) * sizeof(float4)));
    float4* t128 = ctx->dQtiles.as<float4>();
    k_tile_spheres<<<(nTiles + 3) / 4, 128, 0, st>>>(ctx->dQmorton.as<float4>(), n, nTiles, kVerifyTile, t128);
    k_tile_spheres<<<(nSubs + 3) / 4, 128, 0, st>>>(ctx->dQmorton.as<float4>(), n, nSubs, kVerifySub, t128 + nTiles);
    ctx->launches++;
  }
  ctx->launches += 3 + 4;
  S4G_CUDA(cudaGetLastError());
  S4G_CUDA(cudaStreamSynchronize(st));
  ctx->q_has_normals = normals != nullptr;
  ctx->q_has_rgb = rgb != nullptr;
  ctx->nQ = n;
  return S4G_OK;
}

extern "C" int s4g_get_q_normalization(s4g_ctx* ctx, float* out5) {
  if (!ctx || !out5) return S4G_ERR_ARG;
  if (ctx->nQ <= 0) { ctx->err = "s4g_get_q_normalization: no Q cloud"; return S4G_ERR_STATE; }
  out5[0] = ctx->gcenter[0];
  out5[1] = ctx->gcenter[1];
  out5[2] = ctx->gcenter[2];
  out5[3] = ctx->ratio;
  out5[4] = 0.f;
  return S4G_OK;
}
