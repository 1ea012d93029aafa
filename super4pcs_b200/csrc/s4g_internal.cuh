// Internal declarations shared by the .cu files of libs4g.so (not part of the ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include "s4g.h"

#define S4G_CUDA(call)                                                                   \
  do {                                                                                   \
    cudaError_t e__ = (call);                                                            \
    if (e__ != cudaSuccess) {                                                            \
      char b__[512];                                                                     \
      snprintf(b__, sizeof b__, "%s:%d: %s -> %s", __FILE__, __LINE__, #call,            \
               cudaGetErrorString(e__));                                                 \
      ctx->err = b__;                                                                    \
      return S4G_ERR_CUDA;                                                               \
    }                                                                                    \
  } while (0)

#define S4G_TRY(expr)                 \
  do {                                \
    int rc__ = (expr);                \
    if (rc__ != S4G_OK) return rc__;  \
  } while (0)

// grow-only device buffer
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  template <class T> T* as() const { return static_cast<T*>(p); }
};

// Uniform grid over the centred sampled P, bricked: a dense top-level table of bricks
// (edge 2^bshift cells) holds the rank of each occupied brick; occupied bricks own a dense
// block of cellStart entries; P is sorted by (brick rank, local cell) so every cell -- and
// every x-adjacent cell pair inside a brick -- is one contiguous run of float4 points.
// The address arithmetic of every table is defined once, by the helpers below the struct.
struct GridDev {
  float ox, oy, oz;     // world coordinate of cell (0,0,0)'s low corner
  float inv_h;          // 1 / cell edge
  int nx, ny, nz;       // extent in cells
  int bshift;           // log2(brick edge in cells)
  int tbx, tby, tbz;    // extent in bricks
  const int* top;       // [tbx*tby*tbz] brick rank or -1 (brick_index)
  const uint32_t* cellStart;  // [(nBricks << 3*bshift) + 1] (cell_slot)
  const float4* pts;    // sorted points, w = original index (bit pattern)
  const uint32_t* csat; // summed-area table of the coarse occupancy ((2^cshift)^3-cell blocks):
                        // csat[(Z*(cny+1)+Y)*(cnx+1)+X] = #occupied blocks with x<X, y<Y, z<Z; or nullptr
  int cnx, cny, cnz, cshift;
  // ---- delta-field (verify.cu phase 1): 2 bits per voxel of edge h/4 (4x4x4 voxels per cell), stored per "v-brick"
  // (the bricks of `top`'s lattice that hold at least one voxel within delta of a P point): bit 0 = MAYBE (some P
  // point may lie within delta of some location of the voxel), bit 1 = CERTAIN (one P point lies within delta of
  // EVERY location of the voxel).  Neither bit: no P point within delta of any location of the voxel.
  const int* vtop;      // [tbx*tby*tbz] v-brick rank or -1 (brick_index<0, 2>)
  const uint32_t* vox;  // [nVBricks << (3*bshift + 2)] words (vox_cell, vox_word, vox_shift)
  // vbase, vfine: for the BOUNDARY voxels (MAYBE, not CERTAIN) the same bits of their 2x2x2 sub-voxels (boundary_slot, fine_*);
  // vocc: which x-rows of each 2x2x2-cell block the exact test probes hold points, per v-brick cell (vocc_word, vocc_shift)
  const uint32_t* vocc;
  const uint32_t* vbase;
  const uint16_t* vfine;
  float inv_v;          // 4 * inv_h (voxels per world unit)
  float vslack;         // world-unit uncertainty of a query's voxel position the field was built to tolerate
};

// ---- table layouts of GridDev: written by s4g_set_cloud_p (context.cu), read by k_verify (verify.cu).  kBS > 0: the
// brick shift known at compile time (2 = the common 4x4x4-cell bricks), 0: read from the grid.  bs = log2(brick edge),
// m = brick edge - 1; kSub = 2 addresses the bricks by voxel of the delta-field (4 per cell edge) instead of by cell.
struct BrickShape { int bs, m; };
template <int kBS = 0>
__device__ __forceinline__ BrickShape brick_shape(const GridDev& g, int sub = 0) {
  const int bs = kBS > 0 ? kBS : g.bshift; return BrickShape{bs + sub, (1 << bs) - 1};
}
// top / vtop: index of the brick that holds cell (x, y, z) = the first brick of its row (y, z) + x >> bs
__device__ __forceinline__ int brick_row(const GridDev& g, BrickShape b, int y, int z) { return ((z >> b.bs) * g.tby + (y >> b.bs)) * g.tbx; }
__device__ __forceinline__ int brick_in_row(BrickShape b, int row, int x) { return row + (x >> b.bs); }
template <int kBS = 0, int kSub = 0>
__device__ __forceinline__ int brick_index(const GridDev& g, int x, int y, int z) {
  const BrickShape b = brick_shape<kBS>(g, kSub);
  return brick_in_row(b, brick_row(g, b, y, z), x);
}
// cellStart, vocc, vbase (and vox, 4 words per slot): slot of cell (x, y, z) in the brick of rank `rank` = rank << 3*bs |
// local cell (z, y, x bits), so that a brick's cells, and an x-row's cells, are consecutive; cell_row = the row's bits
__device__ __forceinline__ uint32_t cell_row(BrickShape b, int y, int z) { return (uint32_t)((((z & b.m) << b.bs) | (y & b.m)) << b.bs); }
__device__ __forceinline__ uint32_t cell_in_row(BrickShape b, int rank, uint32_t row, int x) { return ((uint32_t)rank << (3 * b.bs)) | row | (uint32_t)(x & b.m); }
template <int kBS = 0>
__device__ __forceinline__ uint32_t cell_slot(const GridDev& g, int rank, int x, int y, int z) {
  const BrickShape b = brick_shape<kBS>(g);
  return cell_in_row(b, rank, cell_row(b, y, z), x);
}
template <int kBS = 0>  // the cell of voxel (X, Y, Z) of the delta-field
__device__ __forceinline__ uint32_t vox_cell(const GridDev& g, int rank, int X, int Y, int Z) { return cell_slot<kBS>(g, rank, X >> 2, Y >> 2, Z >> 2); }
__device__ __forceinline__ const uint4* vox_cells(const uint32_t* vox) { return reinterpret_cast<const uint4*>(vox); }  // per slot
// vox: word of voxel (X, Y, Z) in cell slot `cell` (one word per z-slab of the cell's 4x4x4 voxels) and the position of
// the voxel's 2 bits in it (bit 0 MAYBE, bit 1 CERTAIN)
__device__ __forceinline__ uint32_t vox_word(uint32_t cell, int Z) { return (cell << 2) | (uint32_t)(Z & 3); }
__device__ __forceinline__ uint32_t vox_shift(int X, int Y) { return 2u * (uint32_t)(((Y & 3) << 2) | (X & 3)); }
// boundary voxels (MAYBE, not CERTAIN) of a vox word: bit 2k set <=> voxel k is one
__device__ __forceinline__ uint32_t boundary_bits(uint32_t w) { return w & ~(w >> 1) & 0x55555555u; }
// vfine slot of the boundary voxel at shift `sh` of word `vz` (= w) of a cell whose 4 words are `cw`: vbase[cell]
// (`base`, the boundary voxels of the cells before it in slot order) + the boundary voxels before it in bit order
__device__ __forceinline__ uint32_t boundary_slot(uint32_t base, uint4 cw, uint32_t w, int vz, uint32_t sh) {
  uint32_t slot = base + (uint32_t)__popc(boundary_bits(w) & ((1u << sh) - 1u));
  slot += vz > 0 ? (uint32_t)__popc(boundary_bits(cw.x)) : 0u;
  slot += vz > 1 ? (uint32_t)__popc(boundary_bits(cw.y)) : 0u;
  slot += vz > 2 ? (uint32_t)__popc(boundary_bits(cw.z)) : 0u;
  return slot;
}
// vfine[slot]: 16 bits per boundary voxel, MAYBE of child ch at bit ch, CERTAIN at bit 8 + ch; the child of the upper
// half along x, y, z is bit 0, 1, 2 of ch (fine_child: of the position (fx, fy, fz) voxels above the low corner).  The
// builder ORs into the 32-bit word fine_word(slot), at bit fine_half(slot).
__device__ __forceinline__ uint32_t fine_child(float fx, float fy, float fz) { return (fx >= 0.5f ? 1u : 0u) | (fy >= 0.5f ? 2u : 0u) | (fz >= 0.5f ? 4u : 0u); }
__device__ __forceinline__ uint32_t fine_maybe(int ch) { return 1u << ch; }
__device__ __forceinline__ uint32_t fine_certain(int ch) { return 0x101u << ch; }   // CERTAIN implies MAYBE
// bit 0 MAYBE, bit 1 CERTAIN, as in vox
__device__ __forceinline__ uint32_t fine_state(uint32_t f, uint32_t ch) { return ((f >> ch) & 1u) | (((f >> (8u + ch)) & 1u) << 1); }
__device__ __forceinline__ uint32_t fine_word(uint32_t slot) { return slot >> 1; }
__device__ __forceinline__ uint32_t fine_half(uint32_t slot) { return (slot & 1u) * 16u; }
// vocc: nibble of block origin cell slot `cell`; bit r: row (y0 + (r & 1), z0 + (r >> 1)) of the 2x2x2-cell block has points
__device__ __forceinline__ uint32_t vocc_word(uint32_t cell) { return cell >> 3; }
__device__ __forceinline__ uint32_t vocc_shift(uint32_t cell) { return (cell & 7u) * 4u; }
// csat: entry of corner (X, Y, Z) = #occupied coarse blocks with x < X, y < Y, z < Z
__device__ __forceinline__ uint32_t csat_slot(const GridDev& g, uint32_t X, uint32_t Y, uint32_t Z) {
  return (Z * (uint32_t)(g.cny + 1) + Y) * (uint32_t)(g.cnx + 1) + X;
}
// number of occupied coarse blocks in the inclusive box [x0, x1] x [y0, y1] x [z0, z1] of block coordinates (8 look-ups)
__device__ __forceinline__ uint32_t csat_count(const GridDev& g, int x0, int x1, int y0, int y1, int z0, int z1) {
  const uint32_t* __restrict__ S = g.csat;
  const uint32_t X0 = (uint32_t)x0, X1 = (uint32_t)x1 + 1u, Y0 = (uint32_t)y0, Y1 = (uint32_t)y1 + 1u;
  const uint32_t Z0 = (uint32_t)z0, Z1 = (uint32_t)z1 + 1u;
  return (__ldg(&S[csat_slot(g, X1, Y1, Z1)]) - __ldg(&S[csat_slot(g, X0, Y1, Z1)]) - __ldg(&S[csat_slot(g, X1, Y0, Z1)]) +
          __ldg(&S[csat_slot(g, X0, Y0, Z1)])) -
         (__ldg(&S[csat_slot(g, X1, Y1, Z0)]) - __ldg(&S[csat_slot(g, X0, Y1, Z0)]) - __ldg(&S[csat_slot(g, X1, Y0, Z0)]) +
          __ldg(&S[csat_slot(g, X0, Y0, Z0)]));
}

// ---- warp helpers of the Morton-ordered query side
// AABB of the warp's boxes: every lane ends with the union
__device__ __forceinline__ void warp_aabb(float3& lo, float3& hi) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo.x = fminf(lo.x, __shfl_xor_sync(0xffffffffu, lo.x, o));
    lo.y = fminf(lo.y, __shfl_xor_sync(0xffffffffu, lo.y, o));
    lo.z = fminf(lo.z, __shfl_xor_sync(0xffffffffu, lo.z, o));
    hi.x = fmaxf(hi.x, __shfl_xor_sync(0xffffffffu, hi.x, o));
    hi.y = fmaxf(hi.y, __shfl_xor_sync(0xffffffffu, hi.y, o));
    hi.z = fmaxf(hi.z, __shfl_xor_sync(0xffffffffu, hi.z, o));
  }
}
// the 10 low bits of v spread to every third bit (one axis of a 30-bit Morton code)
__device__ __forceinline__ uint32_t morton_spread10(uint32_t v) {
  v = (v | (v << 16)) & 0x030000FFu;
  v = (v | (v << 8)) & 0x0300F00Fu;
  v = (v | (v << 4)) & 0x030C30C3u;
  v = (v | (v << 2)) & 0x09249249u;
  return v;
}

struct s4g_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t own_stream = nullptr;
  std::string err;
  int sm_count = 132;
  long long l2_bytes = 50ll << 20;   // the device's L2 (sizes the query patches of Verify)

  // ---- P side
  int nP = 0;
  float delta = 0.f;
  float cell_h = 0.f;
  GridDev grid{};
  long long nBricks = 0, nCells = 0;
  DevBuf dP, dPsorted, dTop, dCellStart, dCsat, dVtop, dVox, dVocc, dVbase, dVfine;
  long long nVBricks = 0, nVBoundary = 0;

  // ---- Q side
  int nQ = 0;
  DevBuf dQ;        // float4 original order (w = index bits)
  DevBuf dQmorton;  // float4 Morton order (w = original index bits)
  DevBuf dQn;       // float4 normals (w = 0)
  DevBuf dQrgb;     // float4 rgb (w = 0)
  DevBuf dQunit;    // float4 unit-cube coordinates (pairCreationFunctor.h:66-70)
  DevBuf dQmside;   // Morton-ordered copies of unit coordinates | normals | rgb (3 x n float4) for the pair predicate
  DevBuf dQtiles;   // bounding spheres (centre, radius): [nTiles] of every kVerifyTile consecutive Morton points, then [nSubs] of every kVerifySub
  DevBuf dQgroups;  // AABBs of the 64-point groups / 64-group supergroups of the Morton order
  DevBuf dQpatch;   // centres (float4) of Verify's query patches: runs of patch_tiles consecutive super-tiles (verify.cu)
  int patch_np = 0, patch_tiles = 0;   // patch count and length the centres were computed for (0: none yet)
  int verify_patches = 0;   // requested patch count (S4G_VERIFY_PATCHES when the context was created); 0: from the L2 size
  bool pair_index_ready = false;
  bool q_has_normals = false, q_has_rgb = false;
  float qabs[3] = {0, 0, 0};   // largest |coordinate| of sampled Q per axis (rounding bound of the cell-space transform)
  float gcenter[3] = {0, 0, 0};
  float ratio = 1.f;

  // ---- pairs / quads
  DevBuf dPairs[2];
  long long nPairs[2] = {0, 0};
  bool pairs_sorted[2] = {false, false};
  DevBuf dQuads;
  long long nQuads = 0;

  // ---- the last s4g_range result (s4g_get_range): offsets [range_n + 1], indices and d^2 [range_total]
  DevBuf dRangeOff, dRangeIdx, dRangeSq;
  int range_n = -1;   // -1: none
  long long range_total = 0;
  long long range_window = 0;   // largest sort window of s4g_range (S4G_RANGE_SORT_WINDOW when the context was created); 0: none

  // ---- several bases per launch chain (s4g_try_bases): shared lists keyed by the base index
  DevBuf bArgs, bCounts, bPairKeys[2], bQKeys[2], bQVals[2], bQCnt, bQuadKeys[2], bQuads, bMisc, bResults;

  // ---- scratch
  DevBuf dScratchA, dScratchB, dScratchC, dScratchD, dCub;
  DevBuf dRms, dOk, dCandIdx, dCounts, dResult, dMisc;
  DevBuf dVrec, dVsort;   // Verify: per-candidate records; per-patch candidate order (sort keys, values, CUB temp)
  DevBuf dFilter;         // the outlier filters' host forms: their device outputs before the copy back (outliers.cu)
  void* hPinned = nullptr;  // small pinned staging block
  size_t hPinnedBytes = 0;

  // ---- timing
  // event pairs: 0 = Verify, 1 = rigid fit, 2 = pair extraction, 3 = quad extraction
  cudaEvent_t ev[4][2] = {{nullptr, nullptr}, {nullptr, nullptr}, {nullptr, nullptr}, {nullptr, nullptr}};
  bool ev_pending[4] = {false, false, false, false};
  double ms[4] = {0, 0, 0, 0};
  unsigned long long launches = 0;

  // ---- communicator of the sharded candidate set (comm.cu; null = the caller merges the shards)
  void* comm = nullptr;  // ncclComm_t
  int comm_ranks = 1, comm_rank = 0;
  int comm_timeout_s = 60;
  bool stuck = false;    // a timed-out collective whose stream never drained: s4g_destroy does not wait for it
  unsigned long long collectives = 0;
};

// queries per Verify tile (= threads per Verify CTA)
constexpr int kVerifyTile = 128;
// queries per cull unit (= one warp of a Verify CTA); s4g_set_cloud_q pre-computes one bounding sphere per unit
constexpr int kVerifySub = 32;
// most query patches of one Verify launch (verify.cu, choose_patches): the sort's scratch is 24 bytes per (patch, candidate)
constexpr int kVerifyMaxPatches = 16;

int s4g_reserve(s4g_ctx* ctx, DevBuf& b, size_t bytes);
// device bytes of the sorted P, its grid and the delta-field (what Verify looks up besides Q)
double s4g_grid_bytes(const s4g_ctx* ctx);

// comm.cu: the reduction of the shards' winners on the device (active when a communicator is attached and shard_world > 1)
bool s4g_comm_active(const s4g_ctx* ctx, int shard_world);
int s4g_comm_check_shard(s4g_ctx* ctx, int shard_rank, int shard_world);
int s4g_comm_max_u64(s4g_ctx* ctx, const unsigned long long* d_in, unsigned long long* d_out, cudaStream_t st);
int s4g_comm_reduce_result(s4g_ctx* ctx, const unsigned long long* d_local, unsigned long long* d_global,
                           s4g_tcs_result* rec, cudaStream_t st);
int s4g_comm_wait(s4g_ctx* ctx, cudaStream_t st);  // stream synchronize, with the communicator's deadline when one is attached

// host-side state of one s4g_try_bases call (the three stages live next to the kernels they share code with)
constexpr int kBatchMaxBases = 64;
constexpr int kBatchIdBits = 26;                 // point / list indices inside the packed 64-bit keys
constexpr int kBatchSegShift = 2 * kBatchIdBits; // (segment or base) << 52 | first << 26 | second
struct BatchHost {
  int B = 0;
  unsigned long long nPairs = 0;                 // ordered pairs of all 2B extractions
  uint32_t segCount[2 * kBatchMaxBases] = {};    // ... per extraction (segment 2b + slot)
  uint32_t segOff[2 * kBatchMaxBases + 1] = {};  // exclusive prefix
  unsigned long long nPPairs = 0;                // pairs of the even (P-pair) segments
  unsigned long long nQuads = 0;
  uint32_t quadOff[kBatchMaxBases + 1] = {};     // first quad of every base in the shared quad list
};
int s4g_batch_pairs(s4g_ctx* ctx, const s4g_base_desc* bases, int B, float eps, const s4g_pair_filters* f, BatchHost& bh);
int s4g_batch_quads(s4g_ctx* ctx, const s4g_base_desc* bases, float thr2, BatchHost& bh);
int s4g_batch_tcs(s4g_ctx* ctx, const s4g_base_desc* bases, float max_angle_deg, float rms_threshold, BatchHost& bh,
                  s4g_base_result* out);
enum { S4G_EV_VERIFY = 0, S4G_EV_RIGID = 1, S4G_EV_PAIRS = 2, S4G_EV_QUADS = 3 };
// record the start / stop event of a timed kernel group on the context's stream
#define S4G_EV_START(ctx, which) S4G_CUDA(cudaEventRecord((ctx)->ev[which][0], (ctx)->stream))
#define S4G_EV_STOP(ctx, which)                                          \
  do {                                                                   \
    S4G_CUDA(cudaEventRecord((ctx)->ev[which][1], (ctx)->stream));       \
    (ctx)->ev_pending[which] = true;                                     \
  } while (0)

// ---- device helpers: the reference's float arithmetic, operation by operation -------------
// The whole library is compiled with -fmad=false; the _rn intrinsics below additionally
// make the association order explicit where parity with the reference depends on it.
__device__ __forceinline__ float s4_sum3(float a, float b, float c) {
  // Eigen's redux of a fixed 3-vector: a0 + (a1 + a2)
  return __fadd_rn(a, __fadd_rn(b, c));
}
__device__ __forceinline__ float s4_dot(float3 a, float3 b) {
  return s4_sum3(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y), __fmul_rn(a.z, b.z));
}
__device__ __forceinline__ float s4_sqnorm(float3 a) { return s4_dot(a, a); }
__device__ __forceinline__ float3 s4_sub(float3 a, float3 b) {
  return make_float3(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z));
}
__device__ __forceinline__ float3 s4_add(float3 a, float3 b) {
  return make_float3(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y), __fadd_rn(a.z, b.z));
}
__device__ __forceinline__ float3 s4_scale(float s, float3 a) {
  return make_float3(__fmul_rn(s, a.x), __fmul_rn(s, a.y), __fmul_rn(s, a.z));
}
__device__ __forceinline__ float3 s4_div(float3 a, float s) {
  return make_float3(__fdiv_rn(a.x, s), __fdiv_rn(a.y, s), __fdiv_rn(a.z, s));
}
__device__ __forceinline__ float3 s4_cross(float3 a, float3 b) {
  return make_float3(__fsub_rn(__fmul_rn(a.y, b.z), __fmul_rn(a.z, b.y)),
                     __fsub_rn(__fmul_rn(a.z, b.x), __fmul_rn(a.x, b.z)),
                     __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x)));
}
// MatrixBase::normalized(): n / sqrt(squaredNorm) when squaredNorm > 0
__device__ __forceinline__ float3 s4_normalized(float3 a) {
  float z = s4_sqnorm(a);
  if (z > 0.f) return s4_div(a, __fsqrt_rn(z));
  return a;
}
__device__ __forceinline__ float3 s4_xyz(float4 v) { return make_float3(v.x, v.y, v.z); }
// T q in the reference's operation order: ((m0 x + m1 y) + m2 z) + m3 per row (Verify's exact test and the point queries)
__device__ __forceinline__ void exact_tq(const float* __restrict__ m, float4 q, float& tx, float& ty, float& tz) {
  tx = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[0], q.x), __fmul_rn(m[1], q.y)), __fmul_rn(m[2], q.z)), m[3]);
  ty = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[4], q.x), __fmul_rn(m[5], q.y)), __fmul_rn(m[6], q.z)), m[7]);
  tz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[8], q.x), __fmul_rn(m[9], q.y)), __fmul_rn(m[10], q.z)), m[11]);
}

// ---- Verify's candidate records (verify.cu), written by whatever produces the candidates (k_pack_rec for the API
// entry points, the rigid fits of rigid.cu), so that Verify needs no launch of its own to derive them
struct __align__(16) VerifyCand {
  float T[12];     // exact 3x4, row-major (r00 r01 r02 t0 | r10 ...): the top three rows of T (decision arithmetic)
  float V[12];     // voxel-space 3x4 V = S T (selection only)
  float scale;     // tile-cull radius scale (>= the operator norm of T's 3x3 part); < 0: robust path, no cull
  float pad[3];
};
// what a record depends on besides T: the grid's origin and voxel scale, the delta-field's margin, max |q| per axis of Q
struct VerifyRecArgs {
  float ox, oy, oz, inv_v, vslack, qax, qay, qaz;
};
inline VerifyRecArgs s4g_verify_rec_args(const s4g_ctx* ctx) {
  return VerifyRecArgs{ctx->grid.ox, ctx->grid.oy, ctx->grid.oz, ctx->grid.inv_v, ctx->grid.vslack,
                       ctx->qabs[0], ctx->qabs[1], ctx->qabs[2]};
}
__device__ __forceinline__ void s4g_verify_record(const float (&m)[12], const VerifyRecArgs& a, VerifyCand* __restrict__ out) {
  VerifyCand r;
#pragma unroll
  for (int i = 0; i < 12; ++i) {
    const int col = i & 3, row = i >> 2;
    const float o = row == 0 ? a.ox : row == 1 ? a.oy : a.oz;
    r.T[i] = m[i];
    r.V[i] = col < 3 ? m[i] * a.inv_v : (m[i] - o) * a.inv_v;
  }
  // rounding bound of this candidate's voxel position (fast path) against the margin the field was built with:
  // |x~ - fl(T q)| <= 2^-20 max_r (sum_j |T_rj| |q_j| + |T_r3| + |o_r|)   (16 roundings of relative size 2^-24)
  const float w0 = fabsf(m[0]) * a.qax + fabsf(m[1]) * a.qay + fabsf(m[2]) * a.qaz + fabsf(m[3]) + fabsf(a.ox);
  const float w1 = fabsf(m[4]) * a.qax + fabsf(m[5]) * a.qay + fabsf(m[6]) * a.qaz + fabsf(m[7]) + fabsf(a.oy);
  const float w2 = fabsf(m[8]) * a.qax + fabsf(m[9]) * a.qay + fabsf(m[10]) * a.qaz + fabsf(m[11]) + fabsf(a.oz);
  const float E = fmaxf(w0, fmaxf(w1, w2)) * 9.5367431640625e-7f;   // 2^-20
  // operator norm of the 3x3 part: ||A||_2^2 = lambda_max(A^T A) <= max row sum of |A^T A| (= 1 for a rotation)
  const float g00 = m[0] * m[0] + m[4] * m[4] + m[8] * m[8], g11 = m[1] * m[1] + m[5] * m[5] + m[9] * m[9],
              g22 = m[2] * m[2] + m[6] * m[6] + m[10] * m[10];
  const float g01 = fabsf(m[0] * m[1] + m[4] * m[5] + m[8] * m[9]), g02 = fabsf(m[0] * m[2] + m[4] * m[6] + m[8] * m[10]),
              g12 = fabsf(m[1] * m[2] + m[5] * m[6] + m[9] * m[10]);
  const float n2 = fmaxf(g00 + g01 + g02, fmaxf(g01 + g11 + g12, g02 + g12 + g22));
  const float s = sqrtf(n2) * 1.00001f;
  const bool precise = (E <= a.vslack) && (s <= 1.0e6f);     // false for NaN / Inf
  r.scale = precise ? s : -1.f;
  r.pad[0] = r.pad[1] = r.pad[2] = 0.f;
  *out = r;
}
// Enqueue Verify of K candidate records (device); zeroes d_counts first.  d_K: the candidate count when only the device
// knows it (K is then its upper bound)
int s4g_launch_verify(s4g_ctx* ctx, const VerifyCand* d_recs, int K, uint32_t* d_counts, bool timed, const uint32_t* d_K);
// Enqueue the k_knn instance of k (1 <= k <= 64) on the context's stream: the rows of s4g_knn_dev for n device queries
// (query.cu).  The arguments are checked by the caller, and n > 0.  stats: nullptr or the two counters of the statistics
// variant.
int s4g_launch_knn(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T, int k, float sq_radius,
                   const int32_t* d_exclude, int32_t* d_index, float* d_sq_dist, unsigned long long* stats);
// Enqueue the resident P points in the grid's sorted order as n x 3 queries (normals.cu): query t is GridDev::pts[t]
int s4g_launch_sorted_queries(s4g_ctx* ctx, float* d_xyz);
// Enqueue k_radius_count over the resident P (query.cu): d_counts[j] = min(c_j, min_neighbors) (d_counts may be
// nullptr), d_keep[j] = c_j >= min_neighbors, c_j the number of other P points with d^2 < sq_radius.  min_neighbors >= 1.
int s4g_launch_radius_count(s4g_ctx* ctx, float sq_radius, int min_neighbors, int32_t* d_counts, uint8_t* d_keep);
