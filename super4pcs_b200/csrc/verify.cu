// a8 -- Match4PCSBase::Verify (reference algorithms/match4pcsBase.cc:508-567) for a batch of
// candidate transforms, on the bricked uniform grid + delta-field built by s4g_set_cloud_p.
//
//   counts[k] = #{ q in sampled_Q : exists p in sampled_P, ||T_k q - p||^2 <= delta^2 }
//
// Arithmetic of the DECISION follows the reference's binary operation by operation (SURVEY.md
// A.3 / B.3):
//   T q  = ((m0 x + m1 y) + m2 z) + m3   per row, fp32, no FMA      (match4pcsBase.cc:532)
//   d^2  = dx^2 + (dy^2 + dz^2)                                     (kdtree.h:417)
//   hit  = d^2 <= delta*delta                                       (kdtree.h:418, cc:522)
//
// Schedule.  The working set (Q 16 MB, delta-field 27 + 35 MB, sorted P 16 MB, cellStart, brick
// tables, a 4 MB summed-area table: ~110 MB at 1M points) is about twice the 50 MB L2 of an H100, but the
// Morton order of the queries keeps the look-ups of a warp local; the design minimises instructions and look-ups
// per (query, candidate) pair -- by deciding as many pairs as possible from pre-computed bits instead of point tests:
//  * sampled_Q is streamed in Morton order, one coalesced float4 per thread per tile; a CTA stages a
//    chunk of 16 candidate transforms and owns 8 tiles of 128 queries.  What a CTA stages of a candidate (exact and
//    voxel-space matrix, cull scale or robust path) is a record (VerifyCand) written by whatever produced the
//    candidate (k_pack_rec, the rigid fits), not derived by every CTA.
//  * grid order: the queries are cut into patches sized from the L2 and the CTAs of one patch run together, each
//    patch with the candidates ordered by where they map its centre (k_verify, choose_patches).  A count is a sum of
//    per-pair decisions that do not depend on which CTA makes them, so the order cannot change it.
//  * phase 0 (two levels, one thread per (tile, candidate), then one per (surviving pair, warp)): the bounding sphere of
//    the 128 queries of a tile -- then of the 32 Morton-consecutive queries one WARP owns -- transformed and grown by
//    delta, is tested against the summed-area table of the coarse occupancy (8 look-ups); a warp only visits the
//    candidates that survive for its own queries.
//  * phase 1 (every surviving pair, ~40 instructions): the VOXEL-space image V q (V = the transform
//    pre-multiplied by the world->voxel map, voxel edge = h/4 ~ delta/2; 9 FMAs) addresses the
//    delta-field (GridDev::vox): v-brick table entry, then 2 bits:
//        neither  -> no P point within delta of any location of that voxel: not an inlier, done;
//        CERTAIN  -> some P point is within delta of every location of the voxel: inlier, done;
//        MAYBE    -> refined by the same two bits of the 2x2x2 sub-voxel (edge h/8) that holds the position
//                    (GridDev::vfine); only a pair that is MAYBE again is queued for the exact test.
//    The field is built with a margin (GridDev::vslack) that covers the rounding difference between
//    V q (FMA chain) and the reference-order T q for rigid motions of clouds of this size; every
//    candidate's rounding bound is checked against it when the CTA stages it, and a candidate that
//    exceeds it (huge coefficients, non-rigid 4x4, NaN) takes the robust path: the voxel is derived
//    from the reference-order T q itself, whose voxel coordinate is accurate to 1e-3 voxel whatever T.
//    Either way the bits only replace point tests whose outcome they imply, so counts stay exact.
//  * phase 2 (dense, one queued pair per lane; every WARP has its own queue across its tiles and flushes it on
//    its own -- no CTA barrier inside the tile loop): exact T q in the reference's operation order, the 2x2x2
//    cell block that contains every P point within delta, its occupancy nibble (GridDev::vocc), the non-empty
//    rows' contiguous point runs, d^2 <= delta^2, first hit wins.
//
// Probe (phase 2): cell edge h >= 2.02*delta, so the delta-ball around t = T q touches at most 2 cells per
// axis: x0 = floor(u - 0.5), u = (t - o)/h, cells {x0, x0+1}.  For a point p with |t - p|_x <= delta(1+1e-6):
// |u - v| <= 0.4951, u in [x0+0.5, x0+1.5) => v in (x0+0.0049, x0+1.9951); the 0.0049-cell margin
// dominates the rounding of u and v (< 4e-4 cell for grids <= 2048 cells per axis), so the block is
// conservative and the count exact.
#include "s4g_internal.cuh"
#include <cub/cub.cuh>
#include <algorithm>
#include <cmath>

namespace {

constexpr int kThreads = kVerifyTile;   // 128: one query per thread per tile
constexpr int kCandPerBlock = 16;   // transforms staged per CTA
constexpr int kTilesPerBlock = kThreads / 16;  // (tile, candidate) pairs of a CTA = one per thread in the cull phase
// Compile-time knobs for A/B runs on the GPU (scripts/verify_ab.sh rebuilds libs4g with S4G_NVCC_DEFINES and re-runs
// parity + bench).
#ifndef S4G_QUEUE_CAP
#define S4G_QUEUE_CAP 2048
#endif
#ifndef S4G_VERIFY_MIN_BLOCKS
#define S4G_VERIFY_MIN_BLOCKS 12
#endif
#ifndef S4G_SUBVOXEL
#define S4G_SUBVOXEL 1             // 0: ignore the second level of the delta-field (A/B)
#endif
#ifndef S4G_FLUSH_MIN
#define S4G_FLUSH_MIN (S4G_QUEUE_CAP / 2)
#endif
constexpr int kQueueCap = S4G_QUEUE_CAP;   // queued pairs of a CTA (uint16 entries: candidate << 10 | tile << 7 | thread)
constexpr int kWarpQueue = kQueueCap / (kThreads / 32);   // ... of one warp
constexpr int kWarpFlush = S4G_FLUSH_MIN / (kThreads / 32);   // a warp runs phase 2 once this many of its pairs wait (or at its last tile)
static_assert(kQueueCap >= kThreads && kQueueCap <= 16384, "queue capacity (uint16 entries in shared memory)");
static_assert(kTilesPerBlock == 8 && kCandPerBlock == 16, "entry layout: 4 + 3 + 7 bits; 4-bit certain counters hold <= 8");

struct ProbeStats {
  unsigned long long tested = 0, ranges = 0, bricks = 0, bitmap = 0, culled = 0;
};

// Scan one contiguous run of P points; single exit, flag based.  Two points are in flight per
// iteration (the loads of a run are independent; the kernel is latency-bound here).
template <bool kStats>
__device__ __forceinline__ bool probe_run(const GridDev& g, uint32_t s, uint32_t e, float tx, float ty,
                                          float tz, float sq_eps, ProbeStats& st) {
  bool found = false;
  for (uint32_t k = s; k < e && !found; k += 2) {
    const bool two = k + 1 < e;
    const float4 p = __ldg(&g.pts[k]);
    const float4 r = __ldg(&g.pts[two ? k + 1 : k]);
    const float dx = __fsub_rn(tx, p.x), dy = __fsub_rn(ty, p.y), dz = __fsub_rn(tz, p.z);
    const float ex = __fsub_rn(tx, r.x), ey = __fsub_rn(ty, r.y), ez = __fsub_rn(tz, r.z);
    const float d2 = __fadd_rn(__fmul_rn(dx, dx), __fadd_rn(__fmul_rn(dy, dy), __fmul_rn(dz, dz)));
    const float e2 = __fadd_rn(__fmul_rn(ex, ex), __fadd_rn(__fmul_rn(ey, ey), __fmul_rn(ez, ez)));
    if (kStats) st.tested += two ? 2 : 1;
    found = d2 <= sq_eps || e2 <= sq_eps;
  }
  return found;
}

// Does any P point of row r (cells (x0..x0+1, y0 + (r&1), z0 + (r>>1))) of the block with origin
// (x0,y0,z0) lie within delta of t?  The caller guarantees -1 <= x0 <= nx-1 (same for y, z).
template <bool kStats>
__device__ __forceinline__ bool walk_row(const GridDev& g, int x0, int y0, int z0, int r, float tx, float ty,
                                         float tz, float sq_eps, ProbeStats& st) {
  const BrickShape b = brick_shape(g);
  const int xa = max(x0, 0), xb = min(x0 + 1, g.nx - 1);
  const bool same_brick = brick_in_row(b, 0, xa) == brick_in_row(b, 0, xb);
  const int cz = z0 + (r >> 1), cy = y0 + (r & 1);
  bool found = false;
  if (cz >= 0 && cz < g.nz && cy >= 0 && cy < g.ny) {
    const int rowb = brick_row(g, b, cy, cz);
    const uint32_t rowl = cell_row(b, cy, cz);
    const int ra = __ldg(&g.top[brick_in_row(b, rowb, xa)]);
    if (kStats) st.bricks++;
    if (ra >= 0) {
      const uint32_t idx = cell_in_row(b, ra, rowl, xa);
      const uint32_t s = __ldg(&g.cellStart[idx]);
      const uint32_t e = __ldg(&g.cellStart[idx + (same_brick ? (uint32_t)(xb - xa) : 0u) + 1u]);
      if (kStats) st.ranges++;
      found = probe_run<kStats>(g, s, e, tx, ty, tz, sq_eps, st);
    }
    if (!same_brick && !found) {
      const int rb = __ldg(&g.top[brick_in_row(b, rowb, xb)]);
      if (kStats) st.bricks++;
      if (rb >= 0) {
        const uint32_t idx = cell_in_row(b, rb, rowl, xb);
        const uint32_t s = __ldg(&g.cellStart[idx]);
        const uint32_t e = __ldg(&g.cellStart[idx + 1u]);
        if (kStats) st.ranges++;
        found = probe_run<kStats>(g, s, e, tx, ty, tz, sq_eps, st);
      }
    }
  }
  return found;
}

// Occupancy nibble of the 2x2x2 block with origin cell (x0,y0,z0) (GridDev::vocc): bit r = row r holds points.  Origins
// outside the lattice or outside the v-bricks have no points in their block.
__device__ __forceinline__ uint32_t block_rows(const GridDev& g, int x0, int y0, int z0) {
  uint32_t nib = 0xFu;
  if (g.vocc != nullptr) {
    nib = 0u;
    if (x0 >= 0 && y0 >= 0 && z0 >= 0) {
      const int rank = __ldg(&g.vtop[brick_index(g, x0, y0, z0)]);
      if (rank >= 0) {
        const uint32_t cell = cell_slot(g, rank, x0, y0, z0);
        nib = (__ldg(&g.vocc[vocc_word(cell)]) >> vocc_shift(cell)) & 0xFu;
      }
    }
  }
  return nib;
}

// T q in the reference's operation order: ((m0 x + m1 y) + m2 z) + m3 per row
__device__ __forceinline__ void exact_tq(const float* __restrict__ m, float4 q, float& tx, float& ty, float& tz) {
  tx = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[0], q.x), __fmul_rn(m[1], q.y)), __fmul_rn(m[2], q.z)), m[3]);
  ty = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[4], q.x), __fmul_rn(m[5], q.y)), __fmul_rn(m[6], q.z)), m[7]);
  tz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[8], q.x), __fmul_rn(m[9], q.y)), __fmul_rn(m[10], q.z)), m[11]);
}

// Origin (x0,y0,z0) of the 2x2x2 cell block around t = T q that holds every P point within delta of t (conservative, see
// the header).  false: t is so far outside the grid that no P point is within delta (x0.. are then left unset).
__device__ __forceinline__ bool block_origin(const GridDev& g, float tx, float ty, float tz, int& x0, int& y0, int& z0) {
  const float ux = __fsub_rn(__fmul_rn(__fsub_rn(tx, g.ox), g.inv_h), 0.5f);
  const float uy = __fsub_rn(__fmul_rn(__fsub_rn(ty, g.oy), g.inv_h), 0.5f);
  const float uz = __fsub_rn(__fmul_rn(__fsub_rn(tz, g.oz), g.inv_h), 0.5f);
  const bool in = ux >= -1.f && uy >= -1.f && uz >= -1.f && ux < (float)g.nx && uy < (float)g.ny && uz < (float)g.nz;
  if (in) {
    x0 = __float2int_rd(ux);
    y0 = __float2int_rd(uy);
    z0 = __float2int_rd(uz);
  }
  return in;
}

// voxel coordinates of the query under one candidate.  Fast path: FMA chain of the voxel-space matrix (selection only,
// its rounding is covered by the field's margin for candidates that passed the bound check).  Robust path: from the
// reference-order T q (accurate to 1e-3 voxel for any T).
template <bool kRobust>
__device__ __forceinline__ void voxel_of(const GridDev& g, const float* __restrict__ v, const float* __restrict__ m,
                                         float4 q, float& ux, float& uy, float& uz) {
  if (!kRobust) {
    ux = __fmaf_rn(v[0], q.x, __fmaf_rn(v[1], q.y, __fmaf_rn(v[2], q.z, v[3])));
    uy = __fmaf_rn(v[4], q.x, __fmaf_rn(v[5], q.y, __fmaf_rn(v[6], q.z, v[7])));
    uz = __fmaf_rn(v[8], q.x, __fmaf_rn(v[9], q.y, __fmaf_rn(v[10], q.z, v[11])));
  } else {
    float tx, ty, tz;
    exact_tq(m, q, tx, ty, tz);
    ux = __fmul_rn(__fsub_rn(tx, g.ox), g.inv_v);
    uy = __fmul_rn(__fsub_rn(ty, g.oy), g.inv_v);
    uz = __fmul_rn(__fsub_rn(tz, g.oz), g.inv_v);
  }
}

// Tile-level cull: can ANY point of a query tile (bounding sphere `sph`, world units) come within
// delta of a P point under the candidate whose voxel-space matrix is `v`?  Conservative test on the
// summed-area table of the coarse occupancy ((2^cshift)^3-cell blocks): the transformed sphere (radius scaled by
// `scale` >= the operator norm of the candidate's 3x3 part), grown by delta, is boxed and the number of occupied blocks
// the box touches follows from 8 table look-ups.  Run by ONE thread per (tile, candidate).
__device__ bool tile_live(const GridDev& g, const float* __restrict__ v, float4 sph, float scale) {
  // single exit, flag based (see DESIGN.md section 7 on early returns + warp votes)
  bool live = true;
  if (g.csat != nullptr) {
    // centre in cell coordinates, radius in cells: r/h + delta/h (< 0.4951) + the rounding of the centre.  The centre comes
    // from the same FMA chain as a fast-path voxel, so its error is within the candidate's bound E <= vslack (world units,
    // s4g_verify_record): 0.52 cells cover it for centred clouds, and vslack / h, which grows with |coordinates|, beyond
    const float cx = 0.25f * __fmaf_rn(v[0], sph.x, __fmaf_rn(v[1], sph.y, __fmaf_rn(v[2], sph.z, v[3])));
    const float cy = 0.25f * __fmaf_rn(v[4], sph.x, __fmaf_rn(v[5], sph.y, __fmaf_rn(v[6], sph.z, v[7])));
    const float cz = 0.25f * __fmaf_rn(v[8], sph.x, __fmaf_rn(v[9], sph.y, __fmaf_rn(v[10], sph.z, v[11])));
    const float R = sph.w * g.inv_h * scale * 1.0001f + fmaxf(0.52f, 0.5f + g.vslack * g.inv_h * 1.0001f);
    const float fx0 = cx - R, fx1 = cx + R, fy0 = cy - R, fy1 = cy + R, fz0 = cz - R, fz1 = cz + R;
    // boxes entirely outside the grid cannot match anything
    const bool inside = fx1 >= 0.f && fy1 >= 0.f && fz1 >= 0.f && fx0 < (float)g.nx && fy0 < (float)g.ny &&
                        fz0 < (float)g.nz;
    live = false;
    if (inside) {
      // number of occupied coarse blocks the box touches, from the summed-area table: 8 look-ups
      const int cs = g.cshift;
      const int x0 = max(0, __float2int_rd(fx0)) >> cs, x1 = (min(g.nx - 1, __float2int_rd(fx1)) >> cs) + 1;
      const int y0 = max(0, __float2int_rd(fy0)) >> cs, y1 = (min(g.ny - 1, __float2int_rd(fy1)) >> cs) + 1;
      const int z0 = max(0, __float2int_rd(fz0)) >> cs, z1 = (min(g.nz - 1, __float2int_rd(fz1)) >> cs) + 1;
      const uint32_t sx = (uint32_t)(g.cnx + 1), sxy = sx * (uint32_t)(g.cny + 1);
      const uint32_t* __restrict__ S = g.csat;
      const uint32_t a = (uint32_t)z1 * sxy, b = (uint32_t)z0 * sxy, c = (uint32_t)y1 * sx, d = (uint32_t)y0 * sx;
      const uint32_t cnt = (__ldg(&S[a + c + x1]) - __ldg(&S[a + c + x0]) - __ldg(&S[a + d + x1]) + __ldg(&S[a + d + x0])) -
                           (__ldg(&S[b + c + x1]) - __ldg(&S[b + c + x0]) - __ldg(&S[b + d + x1]) + __ldg(&S[b + d + x0]));
      live = cnt != 0u;
    }
  }
  return live;
}

// second level: state of the sub-voxel (edge h/8) of boundary voxel (X,Y,Z) that holds the position (ux,uy,uz); w = the
// voxel's slab word, sh = its bit position
__device__ __forceinline__ uint32_t vox_refine(const GridDev& g, uint32_t cell, uint32_t w, uint32_t sh, int X, int Y, int Z, float ux,
                                               float uy, float uz) {
  const uint4 cw = __ldg(vox_cells(g.vox) + cell);
  const uint32_t f = __ldg(&g.vfine[boundary_slot(__ldg(&g.vbase[cell]), cw, w, Z & 3, sh)]);
  return fine_state(f, fine_child(ux - (float)X, uy - (float)Y, uz - (float)Z));
}

// state of the voxel (X,Y,Z) = floor of the voxel-space position (ux,uy,uz): bit 0 MAYBE, bit 1 CERTAIN; a BOUNDARY voxel
// (MAYBE, not CERTAIN) is refined to the state of its sub-voxel.
template <int kBS>
__device__ __forceinline__ uint32_t vox_state(const GridDev& g, int rank, int X, int Y, int Z, float ux, float uy, float uz) {
  const uint32_t cell = vox_cell<kBS>(g, rank, X, Y, Z), sh = vox_shift(X, Y);
  const uint32_t w = __ldg(&g.vox[vox_word(cell, Z)]);
  uint32_t s = (w >> sh) & 3u;
  if (S4G_SUBVOXEL && s == 1u && g.vfine != nullptr) s = vox_refine(g, cell, w, sh, X, Y, Z, ux, uy, uz);
  return s;
}

constexpr int kCandFloats = 25;   // staged floats of a VerifyCand (s4g_internal.cuh): T, V, scale

// The schedule (see DESIGN.md section 3.1): the Morton-ordered queries are split into NP patches of `ptiles` consecutive
// super-tiles (kThreads * kTilesPerBlock queries each), and every patch has its own order of the candidates, `perm`
// ([NP][Kall]: similar transforms next to each other; nullptr = the identity).  CTA b of a launch over `nchunks` chunks
// of 16 candidates starting at chunk `chunk0` takes super-tile b % ptiles of patch b / (ptiles * nchunks), chunk
// (b / ptiles) % nchunks of that patch's order, so the CTAs resident at one time share one patch and a run of similar
// candidates.  Every (query, candidate) pair is still decided by exactly one CTA, as before: only the order changes.
template <bool kStats, int kBS>
__global__ void __launch_bounds__(kThreads, kStats ? 1 : S4G_VERIFY_MIN_BLOCKS)
k_verify(GridDev g, const float4* __restrict__ Q, const float4* __restrict__ tiles, const float4* __restrict__ subs, int nQ,
         const VerifyCand* __restrict__ recs, const uint32_t* __restrict__ perm, int Kall, int chunk0, int nchunks, int ptiles,
         float sq_eps, uint32_t* __restrict__ counts, unsigned long long* __restrict__ stats, const uint32_t* __restrict__ dK) {
  const unsigned pt = blockIdx.x / (unsigned)ptiles;
  const int patch = (int)(pt / (unsigned)nchunks);
  const long long qbase = ((long long)patch * ptiles + (blockIdx.x - pt * (unsigned)ptiles)) * (kThreads * kTilesPerBlock);
  const int c0 = (chunk0 + (int)(pt - (unsigned)patch * (unsigned)nchunks)) * kCandPerBlock;
  // candidate count known only on the device (s4g_try_bases): Kall is its upper bound
  const int K = dK != nullptr ? min(Kall, (int)__ldg(dK)) : Kall;
  if (qbase >= nQ || c0 >= K) return;             // CTA-uniform (the last patch may be short)
  const uint32_t* __restrict__ pp = perm != nullptr ? perm + (size_t)patch * Kall : nullptr;
  __shared__ __align__(16) float sT[kCandPerBlock * 12];     // exact transforms (decision arithmetic)
  __shared__ __align__(16) float sV[kCandPerBlock * 12];     // voxel-space transforms (selection only)
  __shared__ float sScale[kCandPerBlock];                    // tile-cull radius scale; < 0: robust path, no cull
  __shared__ uint32_t sLive[kTilesPerBlock * (kThreads / 32)];   // [tile * 4 + warp] bit c: candidate c may hit that warp's 32 queries
  __shared__ uint32_t sCnt[kCandPerBlock];
  __shared__ uint16_t sQueue[kQueueCap];                     // (candidate, tile, query) pairs waiting for the exact test, one quarter per warp
  __shared__ uint8_t sPair[kThreads];                        // phase 0: surviving (tile << 4 | candidate) pairs
  __shared__ uint32_t sPairN[kThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31;
  const int nc = min(kCandPerBlock, K - c0);
  for (int i = tid; i < nc * kCandFloats; i += kThreads) {
    const int c = i / kCandFloats, e = i - c * kCandFloats;
    const int k = pp != nullptr ? (int)__ldg(&pp[c0 + c]) : c0 + c;
    const float v = __ldg(reinterpret_cast<const float*>(&recs[k]) + e);
    if (e < 12) sT[c * 12 + e] = v;
    else if (e < 24) sV[c * 12 + e - 12] = v;
    else sScale[c] = v;
  }
  if (tid < kCandPerBlock) {
    sCnt[tid] = 0;
    if (tid >= nc) sScale[tid] = -1.f;
  }
  __syncthreads();
  uint32_t imprec = 0;                            // bit c: candidate c takes the robust path (CTA-uniform)
#pragma unroll
  for (int c = 0; c < kCandPerBlock; ++c) imprec |= (sScale[c] < 0.f ? 1u : 0u) << c;

  ProbeStats st;
  uint16_t* const wq = &sQueue[(tid >> 5) * kWarpQueue];   // this warp's queue
  uint32_t qn = 0u;                               // entries waiting in it (warp-uniform)
  // ---- phase 0, two levels.  (a) one thread per (128-query tile, candidate): the tile's bounding sphere against the
  // summed-area table; survivors (~1 in 4) are compacted into a list.  (b) one thread per (surviving pair, warp of the
  // tile): the bounding sphere of that warp's 32 queries -- half the radius, an eighth of the box -- against the table
  // again.  sLive[tile * 4 + warp] = candidates that warp has to visit for that tile.
  static_assert(kCandPerBlock == 16 && kThreads == 128 && kVerifySub == 32 && kTilesPerBlock * kCandPerBlock == kThreads, "cull mapping");
  {
    const int t = tid >> 4, c = tid & 15;
    const long long tile0 = qbase + (long long)t * kThreads;
    bool live = false;
    if (tile0 < nQ && c < nc)
      live = ((imprec >> c) & 1u) ? true : tile_live(g, &sV[c * 12], __ldg(&tiles[tile0 / kThreads]), sScale[c]);
    const unsigned b = __ballot_sync(0xffffffffu, live);
    if (lane == 0) sPairN[tid >> 5] = (uint32_t)__popc(b);
    if (tid < kTilesPerBlock * (kThreads / 32)) sLive[tid] = 0u;
    __syncthreads();
    uint32_t before = 0, nLive = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) {
      const uint32_t k = sPairN[w];
      before += w < (tid >> 5) ? k : 0u;
      nLive += k;
    }
    if (live) sPair[before + __popc(b & ((1u << lane) - 1u))] = (uint8_t)tid;     // tid == tile << 4 | candidate
    __syncthreads();
#pragma unroll 1
    for (uint32_t j = (uint32_t)tid; j < 4u * nLive; j += kThreads) {
      const uint32_t code = sPair[j >> 2], sub = (code >> 4) * 4u + (j & 3u), cc = code & 15u;
      const long long q0 = qbase + (long long)sub * kVerifySub;
      if (q0 < nQ) {
        const bool l2 = ((imprec >> cc) & 1u) ? true : tile_live(g, &sV[cc * 12], __ldg(&subs[q0 / kVerifySub]), sScale[cc]);
        if (l2) atomicOr(&sLive[sub], 1u << cc);
      }
    }
  }
  __syncthreads();
  int last_tile = 0;                              // last tile of this CTA that exists (CTA-uniform)
  for (int t = kTilesPerBlock - 1; t > 0; --t)
    if (qbase + (long long)t * kThreads < nQ) { last_tile = t; break; }
  unsigned long long cert = 0ull;                 // 4-bit counters: CERTAIN inliers of this thread's queries per candidate
#pragma unroll 1
  for (int t = 0; t <= last_tile; ++t) {
    const long long tile0 = qbase + (long long)t * kThreads;
    uint32_t live_mask = sLive[t * 4 + (tid >> 5)];                 // this warp's candidates (warp-uniform)
    if (kStats) st.culled += (lane == 0 && tile0 + (tid & ~31) < nQ) ? (unsigned long long)(nc - __popc(live_mask)) : 0ull;
    const bool last = t == last_tile;
    if (live_mask == 0u && !last) continue;       // warp-uniform: nothing to do for this warp's 32 queries (no CTA barrier below)
    const long long qi = tile0 + tid;
    const bool valid = qi < nQ;
    float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
    if (valid && live_mask) q = __ldg(&Q[qi]);

    // ---- phase 1: delta-field state per (query, candidate), live candidates only; two candidates per
    // iteration so that two table loads are in flight.  Fast loop: every live candidate passed the rounding bound
    // (finite, bounded coefficients), so the voxel comes from the FMA chain and the range test is an unsigned compare.
    uint32_t pend = 0u;                           // bit c: pair (this query, candidate c) needs the exact test
    const uint32_t limX = (uint32_t)g.nx << 2, limY = (uint32_t)g.ny << 2, limZ = (uint32_t)g.nz << 2;
    if ((live_mask & imprec) == 0u) {
      const uint32_t lx = valid ? limX : 0u;        // a lane without a query fails the range test of every candidate
#pragma unroll 1
      while (live_mask) {
        const int ca = __ffs(live_mask) - 1;
        live_mask &= live_mask - 1;
        const bool two = live_mask != 0u;
        const int cb = two ? __ffs(live_mask) - 1 : ca;
        live_mask &= live_mask - 1;                  // (0 stays 0)
        float ax, ay, az, bx, by, bz;
        voxel_of<false>(g, &sV[ca * 12], nullptr, q, ax, ay, az);
        voxel_of<false>(g, &sV[cb * 12], nullptr, q, bx, by, bz);
        const int aX = __float2int_rd(ax), aY = __float2int_rd(ay), aZ = __float2int_rd(az);
        const int bX = __float2int_rd(bx), bY = __float2int_rd(by), bZ = __float2int_rd(bz);
        const bool ina = (uint32_t)aX < lx && (uint32_t)aY < limY && (uint32_t)aZ < limZ;
        const bool inb = two && (uint32_t)bX < lx && (uint32_t)bY < limY && (uint32_t)bZ < limZ;
        const int ra = ina ? __ldg(&g.vtop[brick_index<kBS, 2>(g, aX, aY, aZ)]) : -1;
        const int rb = inb ? __ldg(&g.vtop[brick_index<kBS, 2>(g, bX, bY, bZ)]) : -1;
        if (kStats) st.bitmap += (ina ? 1 : 0) + (inb ? 1 : 0);
        if ((ra & rb) >= 0) {                        // some lane of the warp landed in a v-brick (for a or for b): both words in flight
          const uint32_t cella = vox_cell<kBS>(g, ra, aX, aY, aZ), cellb = vox_cell<kBS>(g, rb, bX, bY, bZ);
          const uint32_t sha = vox_shift(aX, aY), shb = vox_shift(bX, bY);
          const uint32_t wa = ra >= 0 ? __ldg(&g.vox[vox_word(cella, aZ)]) : 0u;
          const uint32_t wb = rb >= 0 ? __ldg(&g.vox[vox_word(cellb, bZ)]) : 0u;
          uint32_t sa = (wa >> sha) & 3u, sb = (wb >> shb) & 3u;
          if (kStats) st.bitmap += (ra >= 0 ? 1 : 0) + (rb >= 0 ? 1 : 0);
          if (S4G_SUBVOXEL && g.vfine != nullptr) {
            if (sa == 1u) sa = vox_refine(g, cella, wa, sha, aX, aY, aZ, ax, ay, az);
            if (sb == 1u) sb = vox_refine(g, cellb, wb, shb, bX, bY, bZ, bx, by, bz);
          }
          if (sa & 2u) cert += 1ull << (4 * ca);
          else if (sa & 1u) pend |= 1u << ca;
          if (sb & 2u) cert += 1ull << (4 * cb);
          else if (sb & 1u) pend |= 1u << cb;
        }
      }
    } else {
      // robust loop (a live candidate failed the bound: huge / non-rigid / NaN coefficients): voxel from the reference-order
      // T q, float range test (NaN and out-of-range coordinates fail it before any int conversion is used).  The other
      // candidates keep the voxel of the fast loop (for finite coordinates its range test is the same), so the path of a
      // (query, candidate) pair -- and with it the probe statistics -- does not depend on which candidates share its chunk.
#pragma unroll 1
      while (live_mask) {
        const int c = __ffs(live_mask) - 1;
        live_mask &= live_mask - 1;
        float ux, uy, uz;
        if ((imprec >> c) & 1u) voxel_of<true>(g, &sV[c * 12], &sT[c * 12], q, ux, uy, uz);
        else voxel_of<false>(g, &sV[c * 12], nullptr, q, ux, uy, uz);
        const bool in = valid && ux >= 0.f && uy >= 0.f && uz >= 0.f && ux < (float)limX && uy < (float)limY && uz < (float)limZ;
        const int X = in ? __float2int_rd(ux) : 0, Y = in ? __float2int_rd(uy) : 0, Z = in ? __float2int_rd(uz) : 0;
        const int r = in ? __ldg(&g.vtop[brick_index<kBS, 2>(g, X, Y, Z)]) : -1;
        if (kStats) st.bitmap += in ? 1 : 0;
        if (r >= 0) {
          const uint32_t sa = vox_state<kBS>(g, r, X, Y, Z, ux, uy, uz);
          if (kStats) st.bitmap++;
          if (sa & 2u) cert += 1ull << (4 * c);
          else if (sa & 1u) pend |= 1u << c;
        }
      }
    }
    // ---- per-WARP queue: rounds of { compaction of pending pairs -> this warp's queue ; flush = phase 2 when enough
    // pairs wait, the queue is full, or this is the last tile }.  Warp-synchronous: no CTA barrier in the tile loop, the
    // four warps of the CTA drift apart freely (their live candidates differ).
    bool again;
    do {
      if (__any_sync(0xffffffffu, pend != 0u)) {
        const uint32_t cnt = (uint32_t)__popc(pend);
        uint32_t incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += v;
        }
        const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
        uint32_t base = qn + incl - cnt;
        while (pend && base < (uint32_t)kWarpQueue) {
          const int c = __ffs(pend) - 1;
          pend &= pend - 1u;
          wq[base++] = (uint16_t)((c << 10) | (t << 7) | tid);
        }
        qn = min(qn + total, (uint32_t)kWarpQueue);
      }
      again = __any_sync(0xffffffffu, pend != 0u);                  // leftovers: the queue is full
      if (again || last || qn >= (uint32_t)kWarpFlush) {
        __syncwarp();                                               // the queue entries of all lanes are visible
        // ---- phase 2: one queued pair per lane, densely packed
#pragma unroll 1
        for (uint32_t i = (uint32_t)lane; i < qn; i += 32u) {
          const uint32_t e = wq[i];
          const int c = (int)(e >> 10);
          const float4 qq = __ldg(&Q[qbase + (long long)(e & 1023u)]);
          float tx, ty, tz;
          exact_tq(&sT[c * 12], qq, tx, ty, tz);
          bool found = false;
          int x0, y0, z0;
          if (block_origin(g, tx, ty, tz, x0, y0, z0)) {
            uint32_t nib = block_rows(g, x0, y0, z0);
            if (kStats) st.bitmap += 2;
#pragma unroll 1
            while (nib && !found) {
              const int r = __ffs(nib) - 1;
              nib &= nib - 1u;
              found = walk_row<kStats>(g, x0, y0, z0, r, tx, ty, tz, sq_eps, st);
            }
          }
          if (found) atomicAdd(&sCnt[c], 1u);
        }
        __syncwarp();                                               // every lane is done with the queue
        qn = 0u;
      }
    } while (again);
  }
  // CERTAIN inliers: 16 packed 4-bit counters per thread -> one warp reduction per candidate
#pragma unroll
  for (int c = 0; c < kCandPerBlock; ++c) {
    const uint32_t v = __reduce_add_sync(0xffffffffu, (uint32_t)(cert >> (4 * c)) & 15u);
    if (lane == 0 && v) atomicAdd(&sCnt[c], v);
  }
  __syncthreads();
  if (tid < nc) {
    const uint32_t v = sCnt[tid];
    if (v) atomicAdd(&counts[pp != nullptr ? __ldg(&pp[c0 + tid]) : (uint32_t)(c0 + tid)], v);
  }
  if (kStats) {
    atomicAdd(&stats[0], st.tested);
    atomicAdd(&stats[1], st.ranges);
    atomicAdd(&stats[2], st.bricks);
    atomicAdd(&stats[3], st.bitmap);
    atomicAdd(&stats[4], st.culled);   // (32-query sub-tile, candidate) pairs culled (lane 0 of every warp counted them)
  }
}

// ---- nearest P point within delta of every query (s4g_verify_nearest).  Same decision arithmetic as the exact test of
// k_verify -- exact T q, block_origin, block_rows -- but every point of the block's non-empty rows is scanned (no first
// hit) and the lexicographic minimum of (d^2, original P index) is kept, so the winner does not depend on the sort order
// of the grid.  best_d2 starts at delta^2 and best_j at INT_MAX: a point is taken iff d^2 <= delta^2 and it beats the best
// so far, exactly the hit test of k_verify; NaN distances compare false and are never taken.
__device__ __forceinline__ void nearest_run(const GridDev& g, uint32_t s, uint32_t e, float tx, float ty, float tz,
                                            float& best_d2, int& best_j) {
  for (uint32_t k = s; k < e; ++k) {
    const float4 p = __ldg(&g.pts[k]);
    const float dx = __fsub_rn(tx, p.x), dy = __fsub_rn(ty, p.y), dz = __fsub_rn(tz, p.z);
    const float d2 = __fadd_rn(__fmul_rn(dx, dx), __fadd_rn(__fmul_rn(dy, dy), __fmul_rn(dz, dz)));
    const int j = __float_as_int(p.w);
    if (d2 < best_d2 || (d2 == best_d2 && j < best_j)) {
      best_d2 = d2;
      best_j = j;
    }
  }
}

// every P point of row r (cells (x0..x0+1, y0 + (r&1), z0 + (r>>1))) of the block with origin (x0,y0,z0); the caller
// guarantees -1 <= x0 <= nx-1 (same for y, z).  The two cells are one run when they share a brick, else one run each.
__device__ __forceinline__ void nearest_row(const GridDev& g, int x0, int y0, int z0, int r, float tx, float ty, float tz,
                                            float& best_d2, int& best_j) {
  const BrickShape b = brick_shape(g);
  const int cz = z0 + (r >> 1), cy = y0 + (r & 1);
  if (cz < 0 || cz >= g.nz || cy < 0 || cy >= g.ny) return;
  const int xa = max(x0, 0), xb = min(x0 + 1, g.nx - 1);
  const bool same_brick = brick_in_row(b, 0, xa) == brick_in_row(b, 0, xb);
  const int rowb = brick_row(g, b, cy, cz);
  const uint32_t rowl = cell_row(b, cy, cz);
  const int ra = __ldg(&g.top[brick_in_row(b, rowb, xa)]);
  if (ra >= 0) {
    const uint32_t idx = cell_in_row(b, ra, rowl, xa);
    const uint32_t e = __ldg(&g.cellStart[idx + (same_brick ? (uint32_t)(xb - xa) : 0u) + 1u]);
    nearest_run(g, __ldg(&g.cellStart[idx]), e, tx, ty, tz, best_d2, best_j);
  }
  if (!same_brick) {
    const int rb = __ldg(&g.top[brick_in_row(b, rowb, xb)]);
    if (rb >= 0) {
      const uint32_t idx = cell_in_row(b, rb, rowl, xb);
      nearest_run(g, __ldg(&g.cellStart[idx]), __ldg(&g.cellStart[idx + 1u]), tx, ty, tz, best_d2, best_j);
    }
  }
}

// One thread per query (Morton order, so that the block look-ups of a warp stay local), blockIdx.y = transform k0 + y.
// index / sq_dist rows are written at the query's original position; counts[k] gets one atomic per CTA.
__global__ void __launch_bounds__(kThreads)
k_verify_nearest(GridDev g, const float4* __restrict__ Q, int nQ, const VerifyCand* __restrict__ recs, int k0, float sq_eps,
                 int32_t* __restrict__ index, float* __restrict__ sq_dist, uint32_t* __restrict__ counts) {
  const int k = k0 + (int)blockIdx.y;
  const long long qi = (long long)blockIdx.x * kThreads + threadIdx.x;
  bool found = false;
  if (qi < nQ) {
    const float4 q = __ldg(&Q[qi]);
    float tx, ty, tz;
    exact_tq(recs[k].T, q, tx, ty, tz);
    float best_d2 = sq_eps;
    int best_j = 0x7fffffff;
    int x0, y0, z0;
    if (block_origin(g, tx, ty, tz, x0, y0, z0)) {
      uint32_t nib = block_rows(g, x0, y0, z0);
      while (nib) {
        const int r = __ffs(nib) - 1;
        nib &= nib - 1u;
        nearest_row(g, x0, y0, z0, r, tx, ty, tz, best_d2, best_j);
      }
    }
    found = best_j != 0x7fffffff;
    const size_t at = (size_t)k * (size_t)nQ + (size_t)__float_as_int(q.w);
    index[at] = found ? best_j : -1;
    if (sq_dist != nullptr) sq_dist[at] = found ? best_d2 : __int_as_float(0x7f800000);
  }
  const int n = __syncthreads_count(found);
  if (counts != nullptr && threadIdx.x == 0 && n > 0) atomicAdd(&counts[k], (uint32_t)n);
}

// ---- nearest P point at any radius, for arbitrary query points (s4g_nearest): the restricted closest-point query of the
// reference's kd-tree (KdTree::doQueryRestrictedClosestIndex, kdtree.h:388-453).  One thread per query: y = T x
// (exact_tq) or x; the answer is the lexicographic minimum of (d^2, original P index) over the P points with
// d^2 <= sq_radius and index != exclude, d^2 = dx^2 + (dy^2 + dz^2) in fp32 as in nearest_run (nearest_run_excl).
//
// Search.  The cell coordinates of y, u = (y - o) * inv_h, are taken in double.  The coarse blocks of GridDev::csat
// ((2^cshift)^3 cells) form an implicit tree of boxes: the root is the whole coarse lattice, and a box splits into two
// halves of its longest axis down to single blocks.  The thread descends it depth first with an explicit stack, nearer
// half first: a box is dropped when its lower bound (below) exceeds the best d^2 so far or when csat says it holds no
// point (8 look-ups); a single block left is scanned row by row -- rows whose bound exceeds the best are skipped, the
// others are contiguous runs of the sorted points, one per brick they cross.  best_d2 starts at sq_radius, so nothing
// beyond the radius is ever opened.  A dropped point has a d^2 strictly above the best at that time, so it could neither
// win nor tie: the answer is the lexicographic minimum whatever the order of the search.
// Work: every box opened either is a block that is scanned or has a child that is not empty and within the bound, so a
// query opens at most (1 + 2 x depth) boxes per block it scans (depth <= log2 of the lattice's extents, ~30); empty
// space costs one look-up of csat per box, whatever its size.  The blocks scanned are those within the best distance
// found along the way: for a query near the cloud a handful; for one far outside, those near the first hit.
//
// Lower bound.  A point stored in cell c (on one axis) was binned by floorf(fl(fl(p - o) * inv_h)) (context.cu, cell_of;
// never clamped, the grid has a 1.5-cell margin): two roundings of relative size 2^-24 of a value below n + 1 cells, so
// its exact coordinate v = (p - o) * inv_h lies in (c - eps, c + 1 + eps) with eps = (max(nx, ny, nz) + 2) * 2^-21,
// twice the rounding (1e-3 cell for 2048 cells).  For every point binned in a box of cells, |y - p| on that axis is at least
// gap / inv_h, gap = the distance from u to [c0 - eps, c1 + 1 + eps], so L = sum gap^2 / inv_h^2 bounds the exact d^2.  The
// d^2 the kernel computes takes five roundings of relative size 2^-24 (plus 2^-148 when it is subnormal), so it is at
// least L (1 - 2^-20) - 2^-140; that value, from double arithmetic (relative error ~2^-50) rounded down to fp32, is the
// bound.  A bound that is too low only costs time; this one is never above a d^2 the kernel computes.
struct NearestQuery {
  float tx, ty, tz;   // y
  int excl;           // original P index never taken (-1: none)
  double ux, uy, uz;  // cell coordinates of y
  double eps, h2;     // binning margin of the points (cells); squared cell edge
};

struct NearestStats {
  unsigned long long tested = 0, blocks = 0;
};

// nearest_run (same d^2, same rule) without the point of original index q.excl.  A separate copy, so that the code of
// k_verify_nearest stays as it is.
__device__ __forceinline__ void nearest_run_excl(const GridDev& g, uint32_t s, uint32_t e, const NearestQuery& q,
                                                 float& best_d2, int& best_j) {
  for (uint32_t k = s; k < e; ++k) {
    const float4 p = __ldg(&g.pts[k]);
    const float dx = __fsub_rn(q.tx, p.x), dy = __fsub_rn(q.ty, p.y), dz = __fsub_rn(q.tz, p.z);
    const float d2 = __fadd_rn(__fmul_rn(dx, dx), __fadd_rn(__fmul_rn(dy, dy), __fmul_rn(dz, dz)));
    const int j = __float_as_int(p.w);
    if ((d2 < best_d2 || (d2 == best_d2 && j < best_j)) && j != q.excl) {
      best_d2 = d2;
      best_j = j;
    }
  }
}

// lower bound of the d^2 k_nearest computes between y and any point binned in the cells [x0, x1] x [y0, y1] x [z0, z1]
__device__ __forceinline__ float cells_bound(const NearestQuery& q, int x0, int x1, int y0, int y1, int z0, int z1) {
  const double gx = fmax(0.0, fmax(((double)x0 - q.eps) - q.ux, q.ux - ((double)x1 + 1.0 + q.eps)));
  const double gy = fmax(0.0, fmax(((double)y0 - q.eps) - q.uy, q.uy - ((double)y1 + 1.0 + q.eps)));
  const double gz = fmax(0.0, fmax(((double)z0 - q.eps) - q.uz, q.uz - ((double)z1 + 1.0 + q.eps)));
  const double b = (gx * gx + gy * gy + gz * gz) * q.h2 * (1.0 - 0x1p-20) - 0x1p-140;
  return b > 0.0 ? __double2float_rd(b) : 0.f;
}

// every cell row of the cell box [x0, x1] x [y0, y1] x [z0, z1] that may hold a better point: one run per brick it crosses
template <bool kStats>
__device__ __forceinline__ void nearest_cells(const GridDev& g, const NearestQuery& q, int x0, int x1, int y0, int y1,
                                              int z0, int z1, float& best_d2, int& best_j, NearestStats& st) {
  const BrickShape b = brick_shape(g);
#pragma unroll 1
  for (int cz = z0; cz <= z1; ++cz)
#pragma unroll 1
    for (int cy = y0; cy <= y1; ++cy) {
      if (cells_bound(q, x0, x1, cy, cy, cz, cz) > best_d2) continue;
      const int rowb = brick_row(g, b, cy, cz);
      const uint32_t rowl = cell_row(b, cy, cz);
#pragma unroll 1
      for (int x = x0; x <= x1;) {
        const int xe = min(x1, x | b.m);   // the last cell of the row inside x's brick
        const int rank = __ldg(&g.top[brick_in_row(b, rowb, x)]);
        if (rank >= 0) {
          const uint32_t s = __ldg(&g.cellStart[cell_in_row(b, rank, rowl, x)]);
          const uint32_t e = __ldg(&g.cellStart[cell_in_row(b, rank, rowl, xe) + 1u]);
          if (kStats) st.tested += e - s;
          nearest_run_excl(g, s, e, q, best_d2, best_j);
        }
        x = xe + 1;
      }
    }
}

// a box of coarse blocks [x0, x1] x [y0, y1] x [z0, z1], packed lo | hi << 16 per axis (the coarse lattice has < 2^16
// blocks per axis: its table has <= 2^20 entries)
struct BlockBox {
  uint32_t x, y, z;
};
__device__ __forceinline__ int box_lo(uint32_t a) { return (int)(a & 0xFFFFu); }
__device__ __forceinline__ int box_hi(uint32_t a) { return (int)(a >> 16); }
__device__ __forceinline__ uint32_t box_axis(int lo, int hi) { return (uint32_t)lo | ((uint32_t)hi << 16); }
constexpr int kNearestStack = 3 * 16 + 1;   // depth of the box tree (<= 16 halvings per axis) + 1: the stack's most entries

// One thread per query, written at its own position.  T16: column-major 4x4 or nullptr; exclude: n entries or nullptr.
// stats (kStats): [0] += P points tested, [1] += coarse blocks scanned.
template <bool kStats>
__global__ void __launch_bounds__(kThreads)
k_nearest(GridDev g, const float* __restrict__ xyz, int n, const float* __restrict__ T16, float sq_radius,
          const int32_t* __restrict__ exclude, int32_t* __restrict__ index, float* __restrict__ sq_dist,
          unsigned long long* __restrict__ stats) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  NearestStats st;
  if (i < n) {
    const float4 x = make_float4(__ldg(&xyz[3 * i]), __ldg(&xyz[3 * i + 1]), __ldg(&xyz[3 * i + 2]), 0.f);
    NearestQuery q;
    if (T16 != nullptr) {
      float m[12];
#pragma unroll
      for (int e = 0; e < 12; ++e) m[e] = __ldg(&T16[(e & 3) * 4 + (e >> 2)]);
      exact_tq(m, x, q.tx, q.ty, q.tz);
    } else {
      q.tx = x.x;
      q.ty = x.y;
      q.tz = x.z;
    }
    q.excl = exclude != nullptr ? __ldg(&exclude[i]) : -1;
    float best_d2 = sq_radius;
    int best_j = 0x7fffffff;
    if (!isnan(q.tx) && !isnan(q.ty) && !isnan(q.tz)) {   // (a NaN coordinate makes every d^2 NaN: nothing is taken)
      const double ih = (double)g.inv_h;
      q.ux = ((double)q.tx - (double)g.ox) * ih;
      q.uy = ((double)q.ty - (double)g.oy) * ih;
      q.uz = ((double)q.tz - (double)g.oz) * ih;
      q.eps = (double)(max(g.nx, max(g.ny, g.nz)) + 2) * 0x1p-21;
      q.h2 = 1.0 / (ih * ih);
      const int cs = g.cshift, mx = g.nx - 1, my = g.ny - 1, mz = g.nz - 1;
      BlockBox stack[kNearestStack];
      int top = 0;
      stack[top++] = BlockBox{box_axis(0, g.cnx - 1), box_axis(0, g.cny - 1), box_axis(0, g.cnz - 1)};
#pragma unroll 1
      while (top > 0) {
        const BlockBox b = stack[--top];
        const int x0 = box_lo(b.x), x1 = box_hi(b.x), y0 = box_lo(b.y), y1 = box_hi(b.y), z0 = box_lo(b.z), z1 = box_hi(b.z);
        // its cells (the last block of an axis may reach past the grid: clipped; a block wholly past it holds nothing)
        const int cx0 = x0 << cs, cy0 = y0 << cs, cz0 = z0 << cs;
        const int cx1 = min(((x1 + 1) << cs) - 1, mx), cy1 = min(((y1 + 1) << cs) - 1, my), cz1 = min(((z1 + 1) << cs) - 1, mz);
        if (cx0 > cx1 || cy0 > cy1 || cz0 > cz1) continue;
        if (cells_bound(q, cx0, cx1, cy0, cy1, cz0, cz1) > best_d2) continue;
        if (csat_count(g, x0, x1, y0, y1, z0, z1) == 0u) continue;
        const int ex = x1 - x0, ey = y1 - y0, ez = z1 - z0;
        if ((ex | ey | ez) == 0) {                       // one block: its cell rows
          if (kStats) st.blocks++;
          nearest_cells<kStats>(g, q, cx0, cx1, cy0, cy1, cz0, cz1, best_d2, best_j, st);
          continue;
        }
        // halve the longest axis; the half nearer to u is pushed last, so it is searched first
        BlockBox lo = b, hi = b;
        bool lo_near;
        if (ex >= ey && ex >= ez) {
          const int mid = (x0 + x1) >> 1;
          lo.x = box_axis(x0, mid);
          hi.x = box_axis(mid + 1, x1);
          lo_near = q.ux < (double)((mid + 1) << cs);
        } else if (ey >= ez) {
          const int mid = (y0 + y1) >> 1;
          lo.y = box_axis(y0, mid);
          hi.y = box_axis(mid + 1, y1);
          lo_near = q.uy < (double)((mid + 1) << cs);
        } else {
          const int mid = (z0 + z1) >> 1;
          lo.z = box_axis(z0, mid);
          hi.z = box_axis(mid + 1, z1);
          lo_near = q.uz < (double)((mid + 1) << cs);
        }
        stack[top++] = lo_near ? hi : lo;
        stack[top++] = lo_near ? lo : hi;
      }
    }
    const bool found = best_j != 0x7fffffff;
    index[i] = found ? best_j : -1;
    if (sq_dist != nullptr) sq_dist[i] = found ? best_d2 : __int_as_float(0x7f800000);
  }
  if (kStats) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      st.tested += __shfl_down_sync(0xffffffffu, st.tested, o);
      st.blocks += __shfl_down_sync(0xffffffffu, st.blocks, o);
    }
    if ((threadIdx.x & 31) == 0) {
      atomicAdd(&stats[0], st.tested);
      atomicAdd(&stats[1], st.blocks);
    }
  }
}

// ---- every P point within a radius, for arbitrary query points (s4g_range): the range query of the reference's kd-tree
// (KdTree::doQueryDistProcessIndices, kdtree.h:462-514).  One thread per query: y = T x (exact_tq) or x; its list is every
// original P index j with d^2 < sq_radius (strict: the kd-tree's point test, kdtree.h:485), d^2 computed as in
// nearest_run_excl.  The lists come out in the order of the search; s4g_range sorts each by j afterwards.
//
// Search.  The box descent of k_nearest (NearestQuery, cells_bound, BlockBox) with the fixed bound sq_radius in place of
// the shrinking best: a box, or a cell row of a block, is dropped when csat says it is empty or when
// cells_bound(...) >= sq_radius.  The comparison is >=, not the > of k_nearest: cells_bound never exceeds a d^2 the kernel
// computes (the argument above), so every point of a dropped box or row has d^2 >= sq_radius and is not in the list --
// a d^2 equal to the radius is excluded here, where k_nearest has to keep it.  Nothing is dropped for any other reason,
// so the list is exact whatever the order of the descent (children are pushed low half first).  sq_radius <= 0 drops the
// root (the bound is >= 0); +inf drops nothing that is occupied, and takes every point whose d^2 is finite.
// Two passes run the identical traversal: kFill = false writes the list's length to offsets[i]; kFill = true writes the
// list from offsets[i] (their exclusive scan).
template <bool kFill>
__global__ void __launch_bounds__(kThreads)
k_range(GridDev g, const float* __restrict__ xyz, int n, const float* __restrict__ T16, float sq_radius,
        int64_t* __restrict__ offsets, int32_t* __restrict__ indices, float* __restrict__ sq_dist) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const float4 x = make_float4(__ldg(&xyz[3 * i]), __ldg(&xyz[3 * i + 1]), __ldg(&xyz[3 * i + 2]), 0.f);
  NearestQuery q;
  if (T16 != nullptr) {
    float m[12];
#pragma unroll
    for (int e = 0; e < 12; ++e) m[e] = __ldg(&T16[(e & 3) * 4 + (e >> 2)]);
    exact_tq(m, x, q.tx, q.ty, q.tz);
  } else {
    q.tx = x.x;
    q.ty = x.y;
    q.tz = x.z;
  }
  q.excl = -1;
  int64_t out = kFill ? offsets[i] : 0;   // fill: the next entry of this list; count: its length so far
  if (!isnan(q.tx) && !isnan(q.ty) && !isnan(q.tz)) {   // (a NaN coordinate makes every d^2 NaN: the list is empty)
    const double ih = (double)g.inv_h;
    q.ux = ((double)q.tx - (double)g.ox) * ih;
    q.uy = ((double)q.ty - (double)g.oy) * ih;
    q.uz = ((double)q.tz - (double)g.oz) * ih;
    q.eps = (double)(max(g.nx, max(g.ny, g.nz)) + 2) * 0x1p-21;
    q.h2 = 1.0 / (ih * ih);
    const int cs = g.cshift, mx = g.nx - 1, my = g.ny - 1, mz = g.nz - 1;
    const BrickShape bs = brick_shape(g);
    BlockBox stack[kNearestStack];
    int top = 0;
    stack[top++] = BlockBox{box_axis(0, g.cnx - 1), box_axis(0, g.cny - 1), box_axis(0, g.cnz - 1)};
#pragma unroll 1
    while (top > 0) {
      const BlockBox b = stack[--top];
      const int x0 = box_lo(b.x), x1 = box_hi(b.x), y0 = box_lo(b.y), y1 = box_hi(b.y), z0 = box_lo(b.z), z1 = box_hi(b.z);
      const int cx0 = x0 << cs, cy0 = y0 << cs, cz0 = z0 << cs;
      const int cx1 = min(((x1 + 1) << cs) - 1, mx), cy1 = min(((y1 + 1) << cs) - 1, my), cz1 = min(((z1 + 1) << cs) - 1, mz);
      if (cx0 > cx1 || cy0 > cy1 || cz0 > cz1) continue;
      if (cells_bound(q, cx0, cx1, cy0, cy1, cz0, cz1) >= sq_radius) continue;
      if (csat_count(g, x0, x1, y0, y1, z0, z1) == 0u) continue;
      const int ex = x1 - x0, ey = y1 - y0, ez = z1 - z0;
      if ((ex | ey | ez) != 0) {                       // halve the longest axis
        BlockBox lo = b, hi = b;
        if (ex >= ey && ex >= ez) {
          const int mid = (x0 + x1) >> 1;
          lo.x = box_axis(x0, mid);
          hi.x = box_axis(mid + 1, x1);
        } else if (ey >= ez) {
          const int mid = (y0 + y1) >> 1;
          lo.y = box_axis(y0, mid);
          hi.y = box_axis(mid + 1, y1);
        } else {
          const int mid = (z0 + z1) >> 1;
          lo.z = box_axis(z0, mid);
          hi.z = box_axis(mid + 1, z1);
        }
        stack[top++] = hi;
        stack[top++] = lo;
        continue;
      }
      // one block: its cell rows within the bound, one contiguous run of sorted points per brick a row crosses
#pragma unroll 1
      for (int cz = cz0; cz <= cz1; ++cz)
#pragma unroll 1
        for (int cy = cy0; cy <= cy1; ++cy) {
          if (cells_bound(q, cx0, cx1, cy, cy, cz, cz) >= sq_radius) continue;
          const int rowb = brick_row(g, bs, cy, cz);
          const uint32_t rowl = cell_row(bs, cy, cz);
#pragma unroll 1
          for (int cx = cx0; cx <= cx1;) {
            const int xe = min(cx1, cx | bs.m);
            const int rank = __ldg(&g.top[brick_in_row(bs, rowb, cx)]);
            if (rank >= 0) {
              const uint32_t s = __ldg(&g.cellStart[cell_in_row(bs, rank, rowl, cx)]);
              const uint32_t e = __ldg(&g.cellStart[cell_in_row(bs, rank, rowl, xe) + 1u]);
#pragma unroll 1
              for (uint32_t k = s; k < e; ++k) {
                const float4 p = __ldg(&g.pts[k]);
                const float dx = __fsub_rn(q.tx, p.x), dy = __fsub_rn(q.ty, p.y), dz = __fsub_rn(q.tz, p.z);
                const float d2 = __fadd_rn(__fmul_rn(dx, dx), __fadd_rn(__fmul_rn(dy, dy), __fmul_rn(dz, dz)));
                if (d2 < sq_radius) {
                  if (kFill) {
                    indices[out] = __float_as_int(p.w);
                    if (sq_dist != nullptr) sq_dist[out] = d2;
                  }
                  ++out;
                }
              }
            }
            cx = xe + 1;
          }
        }
    }
  }
  if (!kFill) offsets[i] = out;
}

// ---- the neighbour counts of the radius outlier filter (s4g_radius_outliers): for every resident P point j,
// c_j = #{i != j : d^2(p_i, p_j) < sq_radius}, counted up to min_neighbors.  One thread per sorted point t (GridDev::pts,
// w = original index j); the query is p_j as stored, d^2 as in k_range.
//
// Search.  k_range's descent and point test with the bound sq_radius: a box, or a cell row of a block, is dropped when csat
// says it is empty or when cells_bound(...) >= sq_radius, and a point is counted when d^2 < sq_radius and its index is not
// j.  Run to the end, that count is k_range's list of p_j without j's own entry (its d^2 to itself is exactly 0, in the list
// whenever sq_radius > 0) -- exact by k_range's argument, whatever the order of the descent.  The thread stops as soon as
// the count reaches min_neighbors: every point adds at most 1, so it stops at min(c_j, min_neighbors) in any search
// order, and that capped value is all the filter needs.  In a dense region a thread opens a few cells however loose the
// radius; without the cap it would cost what k_range's count pass costs.  sq_radius <= 0 drops the root (c_j = 0).
// counts[j] = the capped count (counts may be nullptr); keep[j] = 1 when it reached min_neighbors, else 0.
__global__ void __launch_bounds__(kThreads)
k_radius_count(GridDev g, int n, float sq_radius, int min_neighbors, int32_t* __restrict__ counts,
               uint8_t* __restrict__ keep) {
  const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (t >= n) return;
  const float4 self = __ldg(&g.pts[t]);
  NearestQuery q;
  q.tx = self.x;
  q.ty = self.y;
  q.tz = self.z;
  q.excl = __float_as_int(self.w);
  int c = 0;
  const double ih = (double)g.inv_h;
  q.ux = ((double)q.tx - (double)g.ox) * ih;
  q.uy = ((double)q.ty - (double)g.oy) * ih;
  q.uz = ((double)q.tz - (double)g.oz) * ih;
  q.eps = (double)(max(g.nx, max(g.ny, g.nz)) + 2) * 0x1p-21;
  q.h2 = 1.0 / (ih * ih);
  const int cs = g.cshift, mx = g.nx - 1, my = g.ny - 1, mz = g.nz - 1;
  const BrickShape bs = brick_shape(g);
  BlockBox stack[kNearestStack];
  int top = 0;
  stack[top++] = BlockBox{box_axis(0, g.cnx - 1), box_axis(0, g.cny - 1), box_axis(0, g.cnz - 1)};
#pragma unroll 1
  while (top > 0 && c < min_neighbors) {
    const BlockBox b = stack[--top];
    const int x0 = box_lo(b.x), x1 = box_hi(b.x), y0 = box_lo(b.y), y1 = box_hi(b.y), z0 = box_lo(b.z), z1 = box_hi(b.z);
    const int cx0 = x0 << cs, cy0 = y0 << cs, cz0 = z0 << cs;
    const int cx1 = min(((x1 + 1) << cs) - 1, mx), cy1 = min(((y1 + 1) << cs) - 1, my), cz1 = min(((z1 + 1) << cs) - 1, mz);
    if (cx0 > cx1 || cy0 > cy1 || cz0 > cz1) continue;
    if (cells_bound(q, cx0, cx1, cy0, cy1, cz0, cz1) >= sq_radius) continue;
    if (csat_count(g, x0, x1, y0, y1, z0, z1) == 0u) continue;
    const int ex = x1 - x0, ey = y1 - y0, ez = z1 - z0;
    if ((ex | ey | ez) != 0) {                       // halve the longest axis, the nearer half searched first
      BlockBox lo = b, hi = b;
      bool lo_near;
      if (ex >= ey && ex >= ez) {
        const int mid = (x0 + x1) >> 1;
        lo.x = box_axis(x0, mid);
        hi.x = box_axis(mid + 1, x1);
        lo_near = q.ux < (double)((mid + 1) << cs);
      } else if (ey >= ez) {
        const int mid = (y0 + y1) >> 1;
        lo.y = box_axis(y0, mid);
        hi.y = box_axis(mid + 1, y1);
        lo_near = q.uy < (double)((mid + 1) << cs);
      } else {
        const int mid = (z0 + z1) >> 1;
        lo.z = box_axis(z0, mid);
        hi.z = box_axis(mid + 1, z1);
        lo_near = q.uz < (double)((mid + 1) << cs);
      }
      stack[top++] = lo_near ? hi : lo;
      stack[top++] = lo_near ? lo : hi;
      continue;
    }
    // one block: its cell rows within the bound, one contiguous run of sorted points per brick a row crosses
#pragma unroll 1
    for (int cz = cz0; cz <= cz1; ++cz)
#pragma unroll 1
      for (int cy = cy0; cy <= cy1; ++cy) {
        if (cells_bound(q, cx0, cx1, cy, cy, cz, cz) >= sq_radius) continue;
        const int rowb = brick_row(g, bs, cy, cz);
        const uint32_t rowl = cell_row(bs, cy, cz);
#pragma unroll 1
        for (int cx = cx0; cx <= cx1;) {
          const int xe = min(cx1, cx | bs.m);
          const int rank = __ldg(&g.top[brick_in_row(bs, rowb, cx)]);
          if (rank >= 0) {
            const uint32_t s = __ldg(&g.cellStart[cell_in_row(bs, rank, rowl, cx)]);
            const uint32_t e = __ldg(&g.cellStart[cell_in_row(bs, rank, rowl, xe) + 1u]);
#pragma unroll 1
            for (uint32_t k = s; k < e; ++k) {
              const float4 p = __ldg(&g.pts[k]);
              const float dx = __fsub_rn(q.tx, p.x), dy = __fsub_rn(q.ty, p.y), dz = __fsub_rn(q.tz, p.z);
              const float d2 = __fadd_rn(__fmul_rn(dx, dx), __fadd_rn(__fmul_rn(dy, dy), __fmul_rn(dz, dz)));
              if (d2 < sq_radius && __float_as_int(p.w) != q.excl && ++c == min_neighbors) goto done;
            }
          }
          cx = xe + 1;
        }
      }
  }
done:
  if (counts != nullptr) counts[q.excl] = c;
  keep[q.excl] = c >= min_neighbors ? 1 : 0;
}

// the segments of one sort chunk (s4g_range): query i's list is [offsets[i], offsets[i + 1]); the chunk takes the lists
// that start in [base, base + window), relative to base, and gives every other query an empty segment
__global__ void k_range_chunk(const int64_t* __restrict__ offsets, int n, int64_t base, int64_t window,
                              int* __restrict__ begin, int* __restrict__ end) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t b = offsets[i], e = offsets[i + 1];
  const bool in = b >= base && b < base + window;
  begin[i] = in ? (int)(b - base) : 0;
  end[i] = in ? (int)(e - base) : 0;
}

// ---- the k nearest P points within a radius, for arbitrary query points (s4g_knn).  One thread per query: y = T x
// (exact_tq) or x; its row is the k lexicographically smallest (d^2, original P index j) over the P points with
// d^2 <= sq_radius and j != exclude, ascending, d^2 computed as in nearest_run_excl; a row with fewer such points is
// padded with (-1, +inf).  k = 1 is k_nearest's answer.
//
// Search.  The box descent of k_nearest (NearestQuery, cells_bound, BlockBox, csat) with one change: the bound is
// sq_radius while fewer than k points are held, and the d^2 of the k-th held entry once k are.  A box or cell row is
// dropped when its cells_bound is strictly above the bound, as in k_nearest.  A point is inserted when d^2 <= sq_radius,
// j != exclude and (d^2, j) is below the k-th held entry (a NaN d^2 fails the first test and is never taken).
// Determinism.  cells_bound never exceeds a d^2 the kernel computes (the argument above k_nearest), so every point of a
// dropped box or row has d^2 > bound: beyond the radius while the row is not full, and after that above the k-th held
// d^2, which only decreases -- such a point is above the final k-th entry too, so it could be neither in the row nor tie
// with its last entry.  A point at exactly the k-th distance with a smaller j is never dropped (the test is strict) and
// displaces the entry with the larger j.  Every other point is compared with the held list, and every P point is binned
// in one cell, so it is seen once: the row is the lexicographic k-minimum whatever the order of the search.
// Storage.  The held entries are 64-bit keys (d^2 bits << 32 | j), which order as (d^2, j) because d^2 is never negative
// nor NaN; kEmpty, above every key, marks a free slot.  They sit in a per-thread array of kCap slots, sorted ascending
// (local memory: it is indexed by the run-time k), and an insertion shifts the larger keys up by one.  kCap is k rounded
// up to 8, 16, 32 or 64, so that a small k does not carry the stack frame of the largest.  The descent loop and the row
// walk are written out here as in k_range: folding k_nearest's into a shared template moves one instruction of its SASS.
constexpr unsigned long long kEmpty = ~0ull;

template <int kCap, bool kStats>
__global__ void __launch_bounds__(kThreads)
k_knn(GridDev g, const float* __restrict__ xyz, int n, const float* __restrict__ T16, int k, float sq_radius,
      const int32_t* __restrict__ exclude, int32_t* __restrict__ index, float* __restrict__ sq_dist,
      unsigned long long* __restrict__ stats) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  NearestStats st;
  if (i < n) {
    const float4 x = make_float4(__ldg(&xyz[3 * i]), __ldg(&xyz[3 * i + 1]), __ldg(&xyz[3 * i + 2]), 0.f);
    NearestQuery q;
    if (T16 != nullptr) {
      float m[12];
#pragma unroll
      for (int e = 0; e < 12; ++e) m[e] = __ldg(&T16[(e & 3) * 4 + (e >> 2)]);
      exact_tq(m, x, q.tx, q.ty, q.tz);
    } else {
      q.tx = x.x;
      q.ty = x.y;
      q.tz = x.z;
    }
    q.excl = exclude != nullptr ? __ldg(&exclude[i]) : -1;
    unsigned long long held[kCap];
#pragma unroll 1
    for (int e = 0; e < k; ++e) held[e] = kEmpty;
    unsigned long long kth = kEmpty;   // held[k - 1]
    float bound = sq_radius;
    if (!isnan(q.tx) && !isnan(q.ty) && !isnan(q.tz)) {   // (a NaN coordinate makes every d^2 NaN: nothing is taken)
      const double ih = (double)g.inv_h;
      q.ux = ((double)q.tx - (double)g.ox) * ih;
      q.uy = ((double)q.ty - (double)g.oy) * ih;
      q.uz = ((double)q.tz - (double)g.oz) * ih;
      q.eps = (double)(max(g.nx, max(g.ny, g.nz)) + 2) * 0x1p-21;
      q.h2 = 1.0 / (ih * ih);
      const int cs = g.cshift, mx = g.nx - 1, my = g.ny - 1, mz = g.nz - 1;
      const BrickShape bs = brick_shape(g);
      BlockBox stack[kNearestStack];
      int top = 0;
      stack[top++] = BlockBox{box_axis(0, g.cnx - 1), box_axis(0, g.cny - 1), box_axis(0, g.cnz - 1)};
#pragma unroll 1
      while (top > 0) {
        const BlockBox b = stack[--top];
        const int x0 = box_lo(b.x), x1 = box_hi(b.x), y0 = box_lo(b.y), y1 = box_hi(b.y), z0 = box_lo(b.z), z1 = box_hi(b.z);
        const int cx0 = x0 << cs, cy0 = y0 << cs, cz0 = z0 << cs;
        const int cx1 = min(((x1 + 1) << cs) - 1, mx), cy1 = min(((y1 + 1) << cs) - 1, my), cz1 = min(((z1 + 1) << cs) - 1, mz);
        if (cx0 > cx1 || cy0 > cy1 || cz0 > cz1) continue;
        if (cells_bound(q, cx0, cx1, cy0, cy1, cz0, cz1) > bound) continue;
        if (csat_count(g, x0, x1, y0, y1, z0, z1) == 0u) continue;
        const int ex = x1 - x0, ey = y1 - y0, ez = z1 - z0;
        if ((ex | ey | ez) != 0) {                       // halve the longest axis, the nearer half searched first
          BlockBox lo = b, hi = b;
          bool lo_near;
          if (ex >= ey && ex >= ez) {
            const int mid = (x0 + x1) >> 1;
            lo.x = box_axis(x0, mid);
            hi.x = box_axis(mid + 1, x1);
            lo_near = q.ux < (double)((mid + 1) << cs);
          } else if (ey >= ez) {
            const int mid = (y0 + y1) >> 1;
            lo.y = box_axis(y0, mid);
            hi.y = box_axis(mid + 1, y1);
            lo_near = q.uy < (double)((mid + 1) << cs);
          } else {
            const int mid = (z0 + z1) >> 1;
            lo.z = box_axis(z0, mid);
            hi.z = box_axis(mid + 1, z1);
            lo_near = q.uz < (double)((mid + 1) << cs);
          }
          stack[top++] = lo_near ? hi : lo;
          stack[top++] = lo_near ? lo : hi;
          continue;
        }
        // one block: its cell rows within the bound, one contiguous run of sorted points per brick a row crosses
        if (kStats) st.blocks++;
#pragma unroll 1
        for (int cz = cz0; cz <= cz1; ++cz)
#pragma unroll 1
          for (int cy = cy0; cy <= cy1; ++cy) {
            if (cells_bound(q, cx0, cx1, cy, cy, cz, cz) > bound) continue;
            const int rowb = brick_row(g, bs, cy, cz);
            const uint32_t rowl = cell_row(bs, cy, cz);
#pragma unroll 1
            for (int cx = cx0; cx <= cx1;) {
              const int xe = min(cx1, cx | bs.m);
              const int rank = __ldg(&g.top[brick_in_row(bs, rowb, cx)]);
              if (rank >= 0) {
                const uint32_t s = __ldg(&g.cellStart[cell_in_row(bs, rank, rowl, cx)]);
                const uint32_t e = __ldg(&g.cellStart[cell_in_row(bs, rank, rowl, xe) + 1u]);
                if (kStats) st.tested += e - s;
#pragma unroll 1
                for (uint32_t t = s; t < e; ++t) {
                  const float4 p = __ldg(&g.pts[t]);
                  const float dx = __fsub_rn(q.tx, p.x), dy = __fsub_rn(q.ty, p.y), dz = __fsub_rn(q.tz, p.z);
                  const float d2 = __fadd_rn(__fmul_rn(dx, dx), __fadd_rn(__fmul_rn(dy, dy), __fmul_rn(dz, dz)));
                  const int j = __float_as_int(p.w);
                  if (!(d2 <= sq_radius) || j == q.excl) continue;
                  const unsigned long long key = ((unsigned long long)__float_as_uint(d2) << 32) | (uint32_t)j;
                  if (key >= kth) continue;
                  int at = k - 1;
#pragma unroll 1
                  for (; at > 0 && held[at - 1] > key; --at) held[at] = held[at - 1];
                  held[at] = key;
                  kth = held[k - 1];
                  if (kth != kEmpty) bound = __uint_as_float((uint32_t)(kth >> 32));
                }
              }
              cx = xe + 1;
            }
          }
      }
    }
    const long long row = i * (long long)k;
#pragma unroll 1
    for (int e = 0; e < k; ++e) {
      const unsigned long long key = held[e];
      index[row + e] = key != kEmpty ? (int32_t)(uint32_t)key : -1;
      if (sq_dist != nullptr)
        sq_dist[row + e] = key != kEmpty ? __uint_as_float((uint32_t)(key >> 32)) : __int_as_float(0x7f800000);
    }
  }
  if (kStats) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      st.tested += __shfl_down_sync(0xffffffffu, st.tested, o);
      st.blocks += __shfl_down_sync(0xffffffffu, st.blocks, o);
    }
    if ((threadIdx.x & 31) == 0) {
      atomicAdd(&stats[0], st.tested);
      atomicAdd(&stats[1], st.blocks);
    }
  }
}

// column-major 4x4 (16 floats) -> the candidate's record (one thread per candidate)
__global__ void k_pack_rec(const float* __restrict__ T16, int K, VerifyRecArgs ra, VerifyCand* __restrict__ recs) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  float m[12];
#pragma unroll
  for (int e = 0; e < 12; ++e) m[e] = T16[(size_t)k * 16 + (e & 3) * 4 + (e >> 2)];
  s4g_verify_record(m, ra, &recs[k]);
}

// One thread per candidate, when the candidates are ordered per query patch: the sort key of every (patch, candidate)
// pair: patch << 32 | beyond the device-side count << 31 | robust path << 30 | 30-bit Morton code of T c_patch in cell
// coordinates (scaled by `mscale` to 10 bits per axis).  Candidates beyond the count sort last in every patch, so the
// CTA-uniform early return of k_verify still skips exactly their chunks.
__global__ void k_verify_keys(const VerifyCand* __restrict__ recs, int K, const uint32_t* __restrict__ dK,
                              const float4* __restrict__ centres, int NP, float mscale, unsigned long long* __restrict__ keys,
                              uint32_t* __restrict__ vals) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  const bool live = dK == nullptr || k < (int)__ldg(dK);
  const float* __restrict__ V = recs[k].V;
  const bool fast = live && recs[k].scale >= 0.f;   // finite, bounded coefficients: the image of the centre is finite
  for (int p = 0; p < NP; ++p) {
    uint32_t code = live ? 0x40000000u : 0x80000000u;
    if (fast) {
      const float4 c = __ldg(&centres[p]);
      const float x = (V[0] * c.x + V[1] * c.y + V[2] * c.z + V[3]) * mscale;
      const float y = (V[4] * c.x + V[5] * c.y + V[6] * c.z + V[7]) * mscale;
      const float z = (V[8] * c.x + V[9] * c.y + V[10] * c.z + V[11]) * mscale;
      const uint32_t ux = (uint32_t)min(1023, max(0, __float2int_rd(x)));
      const uint32_t uy = (uint32_t)min(1023, max(0, __float2int_rd(y)));
      const uint32_t uz = (uint32_t)min(1023, max(0, __float2int_rd(z)));
      code = morton_spread10(ux) | (morton_spread10(uy) << 1) | (morton_spread10(uz) << 2);
    }
    keys[(size_t)p * K + k] = (unsigned long long)p << 32 | code;
    vals[(size_t)p * K + k] = (uint32_t)k;
  }
}

// centre of the bounding box of the tile spheres of every patch (one warp per patch)
__global__ void k_patch_centres(const float4* __restrict__ tiles, int nTiles, int tiles_per_patch, float4* __restrict__ out) {
  const int p = blockIdx.x, lane = threadIdx.x;
  float3 lo = make_float3(3.0e38f, 3.0e38f, 3.0e38f), hi = make_float3(-3.0e38f, -3.0e38f, -3.0e38f);
  const int end = min(nTiles, (p + 1) * tiles_per_patch);
  for (int t = p * tiles_per_patch + lane; t < end; t += 32) {
    const float4 s = tiles[t];
    lo.x = fminf(lo.x, s.x - s.w); lo.y = fminf(lo.y, s.y - s.w); lo.z = fminf(lo.z, s.z - s.w);
    hi.x = fmaxf(hi.x, s.x + s.w); hi.y = fmaxf(hi.y, s.y + s.w); hi.z = fmaxf(hi.z, s.z + s.w);
  }
  warp_aabb(lo, hi);
  if (lane == 0) out[p] = make_float4(0.5f * (lo.x + hi.x), 0.5f * (lo.y + hi.y), 0.5f * (lo.z + hi.z), 0.f);
}

// Query patches (see k_verify): as many as it takes for one patch's queries and the part of the grid and delta-field its
// images touch to fit in half of the L2 (that part is taken to be the patch's share of the whole grid); one patch when
// everything fits.  On the H100 at 1M points this gives 5 patches; 8 and 16 measured the same within noise, 2 and 1 slower
// (DESIGN.md section 9).  At most kVerifyMaxPatches: the sort's scratch is 24 bytes per (patch, candidate) pair.
// ctx->verify_patches > 0 (the environment variable S4G_VERIFY_PATCHES when the context was created) requests the count
// instead, for A/B runs and tests; it is capped the same way.
constexpr int kMaxPatches = kVerifyMaxPatches;
void choose_patches(const s4g_ctx* ctx, int nST, int& NP, int& ptiles) {
  long long np = ctx->verify_patches;
  if (np <= 0) {
    const double ws = (double)ctx->nQ * sizeof(float4) + s4g_grid_bytes(ctx);
    np = (long long)std::ceil(2.0 * ws / (double)ctx->l2_bytes);
  }
  np = std::max(1ll, std::min<long long>(std::min<long long>(np, kMaxPatches), nST));
  ptiles = (int)((nST + np - 1) / np);
  NP = (nST + ptiles - 1) / ptiles;
}

// Enqueue Verify of K candidate records (device), zeroing `counts` first.  stats != nullptr: the statistics variant.
int run_verify(s4g_ctx* ctx, const VerifyCand* recs, int K, uint32_t* d_counts, bool timed, const uint32_t* d_K,
               unsigned long long* stats) {
  if (K <= 0) return S4G_OK;
  cudaStream_t st = ctx->stream;
  S4G_CUDA(cudaMemsetAsync(d_counts, 0, (size_t)K * sizeof(uint32_t), st));
  const float sq_eps = ctx->delta * ctx->delta;  // epsilon*epsilon, match4pcsBase.cc:522
  const int per_block = kThreads * kTilesPerBlock;
  const int nST = (ctx->nQ + per_block - 1) / per_block;
  const int nTiles = (ctx->nQ + kVerifyTile - 1) / kVerifyTile;
  const int nChunks = (K + kCandPerBlock - 1) / kCandPerBlock;
  int NP = 1, ptiles = nST;
  choose_patches(ctx, nST, NP, ptiles);
  if ((long long)NP * K > 0x7fffffffll) { NP = 1; ptiles = nST; }   // (CUB sorts at most 2^31 - 1 keys)
  const bool order = NP > 1 && nChunks > 1;     // a single chunk has nothing to order
  if (timed) S4G_EV_START(ctx, S4G_EV_VERIFY);
  unsigned long long* keys = nullptr;
  uint32_t* vals = nullptr;
  const uint32_t* perm = nullptr;
  size_t cub_bytes = 0;
  const size_t n = (size_t)NP * K;
  const int end_bit = 32 + (NP > 1 ? 32 - __builtin_clz((unsigned)(NP - 1)) : 0);
  if (order) {
    if (ctx->patch_np != NP || ctx->patch_tiles != ptiles) {
      S4G_TRY(s4g_reserve(ctx, ctx->dQpatch, (size_t)NP * sizeof(float4)));
      k_patch_centres<<<NP, 32, 0, st>>>(ctx->dQtiles.as<float4>(), nTiles, ptiles * kTilesPerBlock, ctx->dQpatch.as<float4>());
      ctx->launches++;
      ctx->patch_np = NP;
      ctx->patch_tiles = ptiles;
    }
    cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                    (uint32_t*)nullptr, (uint32_t*)nullptr, (int)n, 0, end_bit, st);
    S4G_TRY(s4g_reserve(ctx, ctx->dVsort, n * 24 + cub_bytes + 256));
    keys = ctx->dVsort.as<unsigned long long>();
    vals = reinterpret_cast<uint32_t*>(keys + 2 * n);
  }
  const int gx = ctx->grid.nx, gy = ctx->grid.ny, gz = ctx->grid.nz;
  const float mscale = 0.25f * 1024.f / (float)std::max(gx, std::max(gy, gz));   // voxel -> cell -> 10 bits
  if (order) {
    k_verify_keys<<<(K + 127) / 128, 128, 0, st>>>(recs, K, d_K, ctx->dQpatch.as<float4>(), NP, mscale, keys, vals);
    void* tmp = reinterpret_cast<void*>(((uintptr_t)(vals + 2 * n) + 255) & ~(uintptr_t)255);
    S4G_CUDA(cub::DeviceRadixSort::SortPairs(tmp, cub_bytes, keys, keys + n, vals, vals + n, (int)n, 0, end_bit, st));
    perm = vals + n;
    ctx->launches += 5;
  }
  // 1-D grid (at most 2^31 - 1 CTAs per launch): slabs of candidate chunks only beyond that
  const long long per_chunk = (long long)NP * ptiles;
  const int max_chunks = (int)std::min<long long>(nChunks, 0x7fffffffll / per_chunk);
  const float4* tiles = ctx->dQtiles.as<float4>();
  for (int ch = 0; ch < nChunks; ch += max_chunks) {
    const int nch = std::min(max_chunks, nChunks - ch);
    const unsigned grid = (unsigned)(per_chunk * nch);
    if (stats != nullptr)
      k_verify<true, 0><<<grid, kThreads, 0, st>>>(ctx->grid, ctx->dQmorton.as<float4>(), tiles, tiles + nTiles, ctx->nQ,
                                                   recs, perm, K, ch, nch, ptiles, sq_eps, d_counts,
                                                   stats, d_K);
    else if (ctx->grid.bshift == 2)
      k_verify<false, 2><<<grid, kThreads, 0, st>>>(ctx->grid, ctx->dQmorton.as<float4>(), tiles, tiles + nTiles, ctx->nQ,
                                                    recs, perm, K, ch, nch, ptiles, sq_eps, d_counts,
                                                    nullptr, d_K);
    else
      k_verify<false, 0><<<grid, kThreads, 0, st>>>(ctx->grid, ctx->dQmorton.as<float4>(), tiles, tiles + nTiles, ctx->nQ,
                                                    recs, perm, K, ch, nch, ptiles, sq_eps, d_counts,
                                                    nullptr, d_K);
    ctx->launches++;
  }
  if (timed) S4G_EV_STOP(ctx, S4G_EV_VERIFY);
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;
}

}  // namespace

int s4g_launch_verify(s4g_ctx* ctx, const VerifyCand* d_recs, int K, uint32_t* d_counts, bool timed, const uint32_t* d_K) {
  return run_verify(ctx, d_recs, K, d_counts, timed, d_K, nullptr);
}

static int check_ready(s4g_ctx* ctx, const char* who) {
  if (ctx->nP <= 0 || ctx->nQ <= 0) {
    ctx->err = std::string(who) + ": call s4g_set_cloud_p and s4g_set_cloud_q first";
    return S4G_ERR_STATE;
  }
  return S4G_OK;
}

extern "C" int s4g_verify_dev(s4g_ctx* ctx, const float* d_T, int K, uint32_t* d_counts) {
  if (!ctx) return S4G_ERR_ARG;
  if (K < 0 || (K > 0 && (!d_T || !d_counts))) { ctx->err = "s4g_verify_dev: bad arguments"; return S4G_ERR_ARG; }
  S4G_TRY(check_ready(ctx, "s4g_verify_dev"));
  if (K == 0) return S4G_OK;
  S4G_CUDA(cudaSetDevice(ctx->device));
  S4G_TRY(s4g_reserve(ctx, ctx->dVrec, (size_t)K * sizeof(VerifyCand)));
  k_pack_rec<<<(K + 127) / 128, 128, 0, ctx->stream>>>(d_T, K, s4g_verify_rec_args(ctx), ctx->dVrec.as<VerifyCand>());
  ctx->launches++;
  return s4g_launch_verify(ctx, ctx->dVrec.as<VerifyCand>(), K, d_counts, true, nullptr);
}

extern "C" int s4g_verify(s4g_ctx* ctx, const float* T, int K, uint32_t* counts) {
  if (!ctx) return S4G_ERR_ARG;
  if (K < 0 || (K > 0 && (!T || !counts))) { ctx->err = "s4g_verify: bad arguments"; return S4G_ERR_ARG; }
  S4G_TRY(check_ready(ctx, "s4g_verify"));
  if (K == 0) return S4G_OK;
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, (size_t)K * 16 * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dCounts, (size_t)K * sizeof(uint32_t)));
  S4G_CUDA(cudaMemcpyAsync(ctx->dScratchA.p, T, (size_t)K * 16 * sizeof(float), cudaMemcpyHostToDevice, st));
  S4G_TRY(s4g_verify_dev(ctx, ctx->dScratchA.as<float>(), K, ctx->dCounts.as<uint32_t>()));
  S4G_CUDA(cudaMemcpyAsync(counts, ctx->dCounts.p, (size_t)K * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  return S4G_OK;
}

extern "C" int s4g_verify_probe_stats(s4g_ctx* ctx, const float* T, int K, uint64_t* out5) {
  if (!ctx) return S4G_ERR_ARG;
  if (K <= 0 || !T || !out5) { ctx->err = "s4g_verify_probe_stats: bad arguments"; return S4G_ERR_ARG; }
  S4G_TRY(check_ready(ctx, "s4g_verify_probe_stats"));
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, (size_t)K * 16 * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dCounts, (size_t)K * sizeof(uint32_t)));
  S4G_TRY(s4g_reserve(ctx, ctx->dVrec, (size_t)K * sizeof(VerifyCand)));
  S4G_TRY(s4g_reserve(ctx, ctx->dMisc, 256));
  S4G_CUDA(cudaMemcpyAsync(ctx->dScratchA.p, T, (size_t)K * 16 * sizeof(float), cudaMemcpyHostToDevice, st));
  S4G_CUDA(cudaMemsetAsync(ctx->dMisc.p, 0, 40, st));
  k_pack_rec<<<(K + 127) / 128, 128, 0, st>>>(ctx->dScratchA.as<float>(), K, s4g_verify_rec_args(ctx), ctx->dVrec.as<VerifyCand>());
  ctx->launches++;
  S4G_TRY(run_verify(ctx, ctx->dVrec.as<VerifyCand>(), K, ctx->dCounts.as<uint32_t>(), false, nullptr,
                     ctx->dMisc.as<unsigned long long>()));
  unsigned long long h[5] = {0, 0, 0, 0, 0};
  S4G_CUDA(cudaMemcpyAsync(h, ctx->dMisc.p, 40, cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < 5; ++i) out5[i] = h[i];
  return S4G_OK;
}

extern "C" int s4g_verify_nearest_dev(s4g_ctx* ctx, const float* d_T, int K, int32_t* d_index, float* d_sq_dist,
                                      uint32_t* d_counts) {
  if (!ctx) return S4G_ERR_ARG;
  if (K < 0 || (K > 0 && (!d_T || !d_index))) { ctx->err = "s4g_verify_nearest_dev: bad arguments"; return S4G_ERR_ARG; }
  S4G_TRY(check_ready(ctx, "s4g_verify_nearest_dev"));
  if (K == 0) return S4G_OK;
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  S4G_TRY(s4g_reserve(ctx, ctx->dVrec, (size_t)K * sizeof(VerifyCand)));
  k_pack_rec<<<(K + 127) / 128, 128, 0, st>>>(d_T, K, s4g_verify_rec_args(ctx), ctx->dVrec.as<VerifyCand>());
  ctx->launches++;
  if (d_counts != nullptr) S4G_CUDA(cudaMemsetAsync(d_counts, 0, (size_t)K * sizeof(uint32_t), st));
  const unsigned nblk = (unsigned)((ctx->nQ + kThreads - 1) / kThreads);
  constexpr int kMaxY = 65535;   // gridDim.y limit: slabs of transforms beyond it
  for (int k0 = 0; k0 < K; k0 += kMaxY) {
    const dim3 grid(nblk, (unsigned)std::min(kMaxY, K - k0));
    k_verify_nearest<<<grid, kThreads, 0, st>>>(ctx->grid, ctx->dQmorton.as<float4>(), ctx->nQ, ctx->dVrec.as<VerifyCand>(),
                                                k0, ctx->delta * ctx->delta, d_index, d_sq_dist, d_counts);
    ctx->launches++;
  }
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;
}

extern "C" int s4g_verify_nearest(s4g_ctx* ctx, const float* T, int K, int32_t* index, float* sq_dist, uint32_t* counts) {
  if (!ctx) return S4G_ERR_ARG;
  if (K < 0 || (K > 0 && (!T || !index))) { ctx->err = "s4g_verify_nearest: bad arguments"; return S4G_ERR_ARG; }
  S4G_TRY(check_ready(ctx, "s4g_verify_nearest"));
  if (K == 0) return S4G_OK;
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t n = (size_t)K * (size_t)ctx->nQ;
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, (size_t)K * 16 * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, n * sizeof(int32_t)));
  if (sq_dist != nullptr) S4G_TRY(s4g_reserve(ctx, ctx->dScratchC, n * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dCounts, (size_t)K * sizeof(uint32_t)));
  S4G_CUDA(cudaMemcpyAsync(ctx->dScratchA.p, T, (size_t)K * 16 * sizeof(float), cudaMemcpyHostToDevice, st));
  S4G_TRY(s4g_verify_nearest_dev(ctx, ctx->dScratchA.as<float>(), K, ctx->dScratchB.as<int32_t>(),
                                 sq_dist != nullptr ? ctx->dScratchC.as<float>() : nullptr, ctx->dCounts.as<uint32_t>()));
  S4G_CUDA(cudaMemcpyAsync(index, ctx->dScratchB.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (sq_dist != nullptr) S4G_CUDA(cudaMemcpyAsync(sq_dist, ctx->dScratchC.p, n * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (counts != nullptr)
    S4G_CUDA(cudaMemcpyAsync(counts, ctx->dCounts.p, (size_t)K * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  return S4G_OK;
}

static int nearest_args(s4g_ctx* ctx, const char* who, int n, const void* xyz, float sq_radius, const void* index) {
  if (n < 0 || (n > 0 && (!xyz || !index)) || std::isnan(sq_radius)) {
    ctx->err = std::string(who) + ": bad arguments (n >= 0, xyz and index when n > 0, sq_radius not NaN)";
    return S4G_ERR_ARG;
  }
  if (ctx->nP <= 0) {
    ctx->err = std::string(who) + ": call s4g_set_cloud_p first";
    return S4G_ERR_STATE;
  }
  return S4G_OK;
}

// enqueue k_nearest on the context's stream (stats != nullptr: the statistics variant)
static int launch_nearest(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T, float sq_radius,
                          const int32_t* d_exclude, int32_t* d_index, float* d_sq_dist, unsigned long long* stats) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  const unsigned nblk = (unsigned)((n + kThreads - 1) / kThreads);
  if (stats != nullptr)
    k_nearest<true><<<nblk, kThreads, 0, ctx->stream>>>(ctx->grid, d_xyz, n, d_T, sq_radius, d_exclude, d_index, d_sq_dist,
                                                        stats);
  else
    k_nearest<false><<<nblk, kThreads, 0, ctx->stream>>>(ctx->grid, d_xyz, n, d_T, sq_radius, d_exclude, d_index, d_sq_dist,
                                                         nullptr);
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;
}

extern "C" int s4g_nearest_dev(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T, float sq_radius,
                               const int32_t* d_exclude, int32_t* d_index, float* d_sq_dist) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(nearest_args(ctx, "s4g_nearest_dev", n, d_xyz, sq_radius, d_index));
  if (n == 0) return S4G_OK;
  return launch_nearest(ctx, d_xyz, n, d_T, sq_radius, d_exclude, d_index, d_sq_dist, nullptr);
}

// host buffers -> the context's scratch, launch(d_xyz, d_T, d_exclude, d_index, d_sq_dist, d_stats), back: the staging of
// s4g_nearest and s4g_knn, whose outputs have `width` entries per query.  stats: nullptr or the two counters of the
// statistics variant.  The arguments are checked by the caller, and n > 0.
template <class Launch>
static int query_host(s4g_ctx* ctx, const float* xyz, int n, const float* T, int width, const int32_t* exclude,
                      int32_t* index, float* sq_dist, uint64_t* stats, Launch launch) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t nn = (size_t)n, nw = nn * (size_t)width;
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, nn * 3 * sizeof(float) + 16 * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, nw * sizeof(int32_t)));
  if (sq_dist != nullptr) S4G_TRY(s4g_reserve(ctx, ctx->dScratchC, nw * sizeof(float)));
  if (exclude != nullptr) S4G_TRY(s4g_reserve(ctx, ctx->dScratchD, nn * sizeof(int32_t)));
  if (stats != nullptr) S4G_TRY(s4g_reserve(ctx, ctx->dMisc, 256));
  float* d_xyz = ctx->dScratchA.as<float>();
  float* d_T = T != nullptr ? d_xyz + nn * 3 : nullptr;
  S4G_CUDA(cudaMemcpyAsync(d_xyz, xyz, nn * 3 * sizeof(float), cudaMemcpyHostToDevice, st));
  if (T != nullptr) S4G_CUDA(cudaMemcpyAsync(d_T, T, 16 * sizeof(float), cudaMemcpyHostToDevice, st));
  if (exclude != nullptr)
    S4G_CUDA(cudaMemcpyAsync(ctx->dScratchD.p, exclude, nn * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (stats != nullptr) S4G_CUDA(cudaMemsetAsync(ctx->dMisc.p, 0, 2 * sizeof(unsigned long long), st));
  S4G_TRY(launch(d_xyz, d_T, exclude != nullptr ? ctx->dScratchD.as<int32_t>() : nullptr, ctx->dScratchB.as<int32_t>(),
                 sq_dist != nullptr ? ctx->dScratchC.as<float>() : nullptr,
                 stats != nullptr ? ctx->dMisc.as<unsigned long long>() : nullptr));
  S4G_CUDA(cudaMemcpyAsync(index, ctx->dScratchB.p, nw * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (sq_dist != nullptr) S4G_CUDA(cudaMemcpyAsync(sq_dist, ctx->dScratchC.p, nw * sizeof(float), cudaMemcpyDeviceToHost, st));
  unsigned long long h[2] = {0, 0};
  if (stats != nullptr) S4G_CUDA(cudaMemcpyAsync(h, ctx->dMisc.p, sizeof h, cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  if (stats != nullptr) {
    stats[0] = h[0];
    stats[1] = h[1];
  }
  return S4G_OK;
}

// host buffers -> the context's scratch, k_nearest, back; stats: nullptr or the two counters of the statistics variant
static int nearest_host(s4g_ctx* ctx, const char* who, const float* xyz, int n, const float* T, float sq_radius,
                        const int32_t* exclude, int32_t* index, float* sq_dist, uint64_t* stats) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(nearest_args(ctx, who, n, xyz, sq_radius, index));
  if (n == 0) return S4G_OK;
  return query_host(ctx, xyz, n, T, 1, exclude, index, sq_dist, stats,
                    [&](const float* d_xyz, const float* d_T, const int32_t* d_excl, int32_t* d_index, float* d_sq,
                        unsigned long long* d_stats) {
                      return launch_nearest(ctx, d_xyz, n, d_T, sq_radius, d_excl, d_index, d_sq, d_stats);
                    });
}

extern "C" int s4g_nearest(s4g_ctx* ctx, const float* xyz, int n, const float* T, float sq_radius, const int32_t* exclude,
                           int32_t* index, float* sq_dist) {
  return nearest_host(ctx, "s4g_nearest", xyz, n, T, sq_radius, exclude, index, sq_dist, nullptr);
}

extern "C" int s4g_nearest_probe_stats(s4g_ctx* ctx, const float* xyz, int n, const float* T, float sq_radius,
                                       const int32_t* exclude, int32_t* index, float* sq_dist, uint64_t* out2) {
  if (ctx && !out2) { ctx->err = "s4g_nearest_probe_stats: bad arguments"; return S4G_ERR_ARG; }
  if (out2) out2[0] = out2[1] = 0;
  return nearest_host(ctx, "s4g_nearest_probe_stats", xyz, n, T, sq_radius, exclude, index, sq_dist, out2);
}

constexpr int kKnnMax = 64;   // the largest k of s4g_knn (the slots of k_knn's widest instance)

static int knn_args(s4g_ctx* ctx, const char* who, int n, const void* xyz, int k, float sq_radius, const void* index) {
  if (k < 1 || k > kKnnMax) {
    ctx->err = std::string(who) + ": bad arguments (1 <= k <= 64)";
    return S4G_ERR_ARG;
  }
  return nearest_args(ctx, who, n, xyz, sq_radius, index);
}

// enqueue k_knn on the context's stream: the instance whose slots are k rounded up to 8, 16, 32 or 64 (stats != nullptr:
// the statistics variant)
template <int kCap>
static void launch_knn_cap(s4g_ctx* ctx, unsigned nblk, const float* d_xyz, int n, const float* d_T, int k, float sq_radius,
                           const int32_t* d_exclude, int32_t* d_index, float* d_sq_dist, unsigned long long* stats) {
  if (stats != nullptr)
    k_knn<kCap, true><<<nblk, kThreads, 0, ctx->stream>>>(ctx->grid, d_xyz, n, d_T, k, sq_radius, d_exclude, d_index,
                                                          d_sq_dist, stats);
  else
    k_knn<kCap, false><<<nblk, kThreads, 0, ctx->stream>>>(ctx->grid, d_xyz, n, d_T, k, sq_radius, d_exclude, d_index,
                                                           d_sq_dist, nullptr);
}

int s4g_launch_knn(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T, int k, float sq_radius,
                   const int32_t* d_exclude, int32_t* d_index, float* d_sq_dist, unsigned long long* stats) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  const unsigned nblk = (unsigned)((n + kThreads - 1) / kThreads);
  if (k <= 8)
    launch_knn_cap<8>(ctx, nblk, d_xyz, n, d_T, k, sq_radius, d_exclude, d_index, d_sq_dist, stats);
  else if (k <= 16)
    launch_knn_cap<16>(ctx, nblk, d_xyz, n, d_T, k, sq_radius, d_exclude, d_index, d_sq_dist, stats);
  else if (k <= 32)
    launch_knn_cap<32>(ctx, nblk, d_xyz, n, d_T, k, sq_radius, d_exclude, d_index, d_sq_dist, stats);
  else
    launch_knn_cap<kKnnMax>(ctx, nblk, d_xyz, n, d_T, k, sq_radius, d_exclude, d_index, d_sq_dist, stats);
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;
}

extern "C" int s4g_knn_dev(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T, int k, float sq_radius,
                           const int32_t* d_exclude, int32_t* d_index, float* d_sq_dist) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(knn_args(ctx, "s4g_knn_dev", n, d_xyz, k, sq_radius, d_index));
  if (n == 0) return S4G_OK;
  return s4g_launch_knn(ctx, d_xyz, n, d_T, k, sq_radius, d_exclude, d_index, d_sq_dist, nullptr);
}

static int knn_host(s4g_ctx* ctx, const char* who, const float* xyz, int n, const float* T, int k, float sq_radius,
                    const int32_t* exclude, int32_t* index, float* sq_dist, uint64_t* stats) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(knn_args(ctx, who, n, xyz, k, sq_radius, index));
  if (n == 0) return S4G_OK;
  return query_host(ctx, xyz, n, T, k, exclude, index, sq_dist, stats,
                    [&](const float* d_xyz, const float* d_T, const int32_t* d_excl, int32_t* d_index, float* d_sq,
                        unsigned long long* d_stats) {
                      return s4g_launch_knn(ctx, d_xyz, n, d_T, k, sq_radius, d_excl, d_index, d_sq, d_stats);
                    });
}

extern "C" int s4g_knn(s4g_ctx* ctx, const float* xyz, int n, const float* T, int k, float sq_radius,
                       const int32_t* exclude, int32_t* index, float* sq_dist) {
  return knn_host(ctx, "s4g_knn", xyz, n, T, k, sq_radius, exclude, index, sq_dist, nullptr);
}

extern "C" int s4g_knn_probe_stats(s4g_ctx* ctx, const float* xyz, int n, const float* T, int k, float sq_radius,
                                   const int32_t* exclude, int32_t* index, float* sq_dist, uint64_t* out2) {
  if (ctx && !out2) { ctx->err = "s4g_knn_probe_stats: bad arguments"; return S4G_ERR_ARG; }
  if (out2) out2[0] = out2[1] = 0;
  return knn_host(ctx, "s4g_knn_probe_stats", xyz, n, T, k, sq_radius, exclude, index, sq_dist, out2);
}

int s4g_launch_radius_count(s4g_ctx* ctx, float sq_radius, int min_neighbors, int32_t* d_counts, uint8_t* d_keep) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  const int n = ctx->nP;
  k_radius_count<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, ctx->stream>>>(ctx->grid, n, sq_radius,
                                                                                          min_neighbors, d_counts, d_keep);
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;
}

static int range_args(s4g_ctx* ctx, const char* who, int n, const void* xyz, float sq_radius, const void* offsets) {
  if (n < 0 || (n > 0 && (!xyz || !offsets)) || std::isnan(sq_radius)) {
    ctx->err = std::string(who) + ": bad arguments (n >= 0, xyz and offsets when n > 0, sq_radius not NaN)";
    return S4G_ERR_ARG;
  }
  if (ctx->nP <= 0) {
    ctx->err = std::string(who) + ": call s4g_set_cloud_p first";
    return S4G_ERR_STATE;
  }
  return S4G_OK;
}

// enqueue the count pass of k_range and the scan of the lengths: d_offsets [n + 1] = 0, ..., total
static int range_count(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T, float sq_radius, int64_t* d_offsets) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  S4G_CUDA(cudaMemsetAsync(d_offsets + n, 0, sizeof(int64_t), st));
  k_range<false><<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, st>>>(ctx->grid, d_xyz, n, d_T, sq_radius,
                                                                                 d_offsets, nullptr, nullptr);
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  size_t bytes = 0;
  S4G_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, d_offsets, d_offsets, (long long)n + 1, st));
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, bytes));
  S4G_CUDA(cub::DeviceScan::ExclusiveSum(ctx->dCub.p, bytes, d_offsets, d_offsets, (long long)n + 1, st));
  return S4G_OK;
}

// enqueue the fill pass of k_range into d_indices / d_sq_dist (nullptr: not written) from d_offsets (total = its last
// entry), then sort every list by index, its d^2 carried along.  CUB's segmented sort addresses the items with int, so the
// lists are sorted in chunks: chunk c takes the lists that start in the window [c w, (c + 1) w) of the output, and a list
// that starts there ends before c w + w + |P| <= c w + INT_MAX.  One chunk when total <= INT_MAX.  The sort ping-pongs
// with a buffer of the chunk's size; when there is more than one chunk, that buffer starts as a copy of the output, so
// the entries of the neighbouring chunks are copied back unchanged.
static int range_fill(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T, float sq_radius, const int64_t* d_offsets,
                      int64_t total, int32_t* d_indices, float* d_sq_dist) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  k_range<true><<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, st>>>(
      ctx->grid, d_xyz, n, d_T, sq_radius, const_cast<int64_t*>(d_offsets), d_indices, d_sq_dist);
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  if (total == 0) return S4G_OK;
  const int64_t kMaxItems = 0x7fffffff;
  int64_t window = total <= kMaxItems ? total : std::max<int64_t>(1, kMaxItems - ctx->nP);
  if (ctx->range_window > 0) window = std::min<int64_t>(window, ctx->range_window);
  const bool chunked = window < total;
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchD, 2 * (size_t)n * sizeof(int)));
  int* seg_begin = ctx->dScratchD.as<int>();
  int* seg_end = seg_begin + n;
  for (int64_t base = 0; base < total; base += window) {
    const int len = (int)std::min<int64_t>(total - base, kMaxItems);
    S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, (size_t)len * sizeof(int32_t)));
    if (d_sq_dist != nullptr) S4G_TRY(s4g_reserve(ctx, ctx->dScratchC, (size_t)len * sizeof(float)));
    int32_t* keys = d_indices + base;
    float* vals = d_sq_dist != nullptr ? d_sq_dist + base : nullptr;
    if (chunked) {
      S4G_CUDA(cudaMemcpyAsync(ctx->dScratchB.p, keys, (size_t)len * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
      if (vals != nullptr)
        S4G_CUDA(cudaMemcpyAsync(ctx->dScratchC.p, vals, (size_t)len * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    k_range_chunk<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_offsets, n, base, window, seg_begin, seg_end);
    ctx->launches++;
    S4G_CUDA(cudaGetLastError());
    cub::DoubleBuffer<int32_t> dk(keys, ctx->dScratchB.as<int32_t>());
    cub::DoubleBuffer<float> dv(vals, ctx->dScratchC.as<float>());
    size_t bytes = 0;
    if (vals != nullptr) {
      S4G_CUDA(cub::DeviceSegmentedSort::SortPairs(nullptr, bytes, dk, dv, len, n, seg_begin, seg_end, st));
      S4G_TRY(s4g_reserve(ctx, ctx->dCub, bytes));
      S4G_CUDA(cub::DeviceSegmentedSort::SortPairs(ctx->dCub.p, bytes, dk, dv, len, n, seg_begin, seg_end, st));
    } else {
      S4G_CUDA(cub::DeviceSegmentedSort::SortKeys(nullptr, bytes, dk, len, n, seg_begin, seg_end, st));
      S4G_TRY(s4g_reserve(ctx, ctx->dCub, bytes));
      S4G_CUDA(cub::DeviceSegmentedSort::SortKeys(ctx->dCub.p, bytes, dk, len, n, seg_begin, seg_end, st));
    }
    if (dk.Current() != keys)
      S4G_CUDA(cudaMemcpyAsync(keys, dk.Current(), (size_t)len * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    if (vals != nullptr && dv.Current() != vals)
      S4G_CUDA(cudaMemcpyAsync(vals, dv.Current(), (size_t)len * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  return S4G_OK;
}

extern "C" int s4g_range_count_dev(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T, float sq_radius,
                                   int64_t* d_offsets) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(range_args(ctx, "s4g_range_count_dev", n, d_xyz, sq_radius, d_offsets));
  if (n == 0) {
    if (d_offsets != nullptr) {
      S4G_CUDA(cudaSetDevice(ctx->device));
      S4G_CUDA(cudaMemsetAsync(d_offsets, 0, sizeof(int64_t), ctx->stream));
    }
    return S4G_OK;
  }
  return range_count(ctx, d_xyz, n, d_T, sq_radius, d_offsets);
}

extern "C" int s4g_range_fill_dev(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T, float sq_radius,
                                  const int64_t* d_offsets, int64_t total, int32_t* d_indices, float* d_sq_dist) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(range_args(ctx, "s4g_range_fill_dev", n, d_xyz, sq_radius, d_offsets));
  if (total < 0 || (n == 0 && total != 0) || (total > 0 && !d_indices)) {
    ctx->err = "s4g_range_fill_dev: bad arguments (total = d_offsets[n] >= 0, indices when total > 0)";
    return S4G_ERR_ARG;
  }
  if (n == 0) return S4G_OK;
  return range_fill(ctx, d_xyz, n, d_T, sq_radius, d_offsets, total, d_indices, d_sq_dist);
}

extern "C" int s4g_range(s4g_ctx* ctx, const float* xyz, int n, const float* T, float sq_radius, int64_t* offsets,
                         int64_t* total) {
  if (!ctx) return S4G_ERR_ARG;
  ctx->range_n = -1;   // a failed call leaves no result
  ctx->range_total = 0;
  S4G_TRY(range_args(ctx, "s4g_range", n, xyz, sq_radius, offsets));
  if (!offsets || !total) {
    ctx->err = "s4g_range: bad arguments (offsets and total)";
    return S4G_ERR_ARG;
  }
  if (n == 0) {
    offsets[0] = 0;
    *total = 0;
    ctx->range_n = 0;
    return S4G_OK;
  }
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t nn = (size_t)n;
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, nn * 3 * sizeof(float) + 16 * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dRangeOff, (nn + 1) * sizeof(int64_t)));
  float* d_xyz = ctx->dScratchA.as<float>();
  float* d_T = T != nullptr ? d_xyz + nn * 3 : nullptr;
  S4G_CUDA(cudaMemcpyAsync(d_xyz, xyz, nn * 3 * sizeof(float), cudaMemcpyHostToDevice, st));
  if (T != nullptr) S4G_CUDA(cudaMemcpyAsync(d_T, T, 16 * sizeof(float), cudaMemcpyHostToDevice, st));
  int64_t* d_off = ctx->dRangeOff.as<int64_t>();
  S4G_TRY(range_count(ctx, d_xyz, n, d_T, sq_radius, d_off));
  S4G_CUDA(cudaMemcpyAsync(offsets, d_off, (nn + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  const int64_t tot = offsets[n];
  S4G_TRY(s4g_reserve(ctx, ctx->dRangeIdx, (size_t)std::max<int64_t>(tot, 1) * sizeof(int32_t)));
  S4G_TRY(s4g_reserve(ctx, ctx->dRangeSq, (size_t)std::max<int64_t>(tot, 1) * sizeof(float)));
  S4G_TRY(range_fill(ctx, d_xyz, n, d_T, sq_radius, d_off, tot, ctx->dRangeIdx.as<int32_t>(), ctx->dRangeSq.as<float>()));
  S4G_CUDA(cudaStreamSynchronize(st));
  ctx->range_n = n;
  ctx->range_total = tot;
  *total = tot;
  return S4G_OK;
}

extern "C" int s4g_get_range(s4g_ctx* ctx, int32_t* indices, float* sq_dist) {
  if (!ctx) return S4G_ERR_ARG;
  if (ctx->range_n < 0) {
    ctx->err = "s4g_get_range: no s4g_range result";
    return S4G_ERR_STATE;
  }
  const size_t tot = (size_t)ctx->range_total;
  if (tot == 0) return S4G_OK;
  if (!indices) {
    ctx->err = "s4g_get_range: null indices";
    return S4G_ERR_ARG;
  }
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  S4G_CUDA(cudaMemcpyAsync(indices, ctx->dRangeIdx.p, tot * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (sq_dist != nullptr) S4G_CUDA(cudaMemcpyAsync(sq_dist, ctx->dRangeSq.p, tot * sizeof(float), cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  return S4G_OK;
}
