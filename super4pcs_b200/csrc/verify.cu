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
#define S4G_VERIFY_MIN_BLOCKS 16           // 16 CTAs (64 warps) per SM: 32 registers (DESIGN.md section 9)
#endif
#ifndef S4G_SUBVOXEL
#define S4G_SUBVOXEL 1             // 0: ignore the second level of the delta-field (A/B)
#endif
#ifndef S4G_FLUSH_MIN
#define S4G_FLUSH_MIN (S4G_QUEUE_CAP / 2)
#endif
#ifndef S4G_VERIFY_CLOCKS
#define S4G_VERIFY_CLOCKS 0        // 1: k_verify<false, .> sums its SM cycles per phase (scripts/verify_phases.py)
#endif
constexpr int kQueueCap = S4G_QUEUE_CAP;   // queued pairs of a CTA (uint16 entries: candidate << 10 | tile << 7 | thread)
constexpr int kWarpQueue = kQueueCap / (kThreads / 32);   // ... of one warp
constexpr int kWarpFlush = S4G_FLUSH_MIN / (kThreads / 32);   // a warp runs phase 2 once this many of its pairs wait (or at its last tile)
static_assert(kQueueCap >= kThreads && kQueueCap <= 16384, "queue capacity (uint16 entries in shared memory)");
static_assert(kTilesPerBlock == 8 && kCandPerBlock == 16, "entry layout: 4 + 3 + 7 bits; 4-bit certain counters hold <= 8");

struct ProbeStats {
  unsigned long long tested = 0, ranges = 0, bricks = 0, bitmap = 0, culled = 0;
};

#if S4G_VERIFY_CLOCKS
// SM cycles summed over the warps of every k_verify<false, .> launch: [0] staging and both cull levels, [1] the
// delta-field look-ups of the tiles (the query load and the refinement included), [2] the queue and the exact test,
// [3] everything (the rest of the tile loop and the final reduction are [3] - [0] - [1] - [2]).
__device__ unsigned long long g_verify_clocks[4];
#endif

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
  constexpr bool kClk = S4G_VERIFY_CLOCKS && !kStats;
  uint32_t clk[4] = {0u, 0u, 0u, 0u};             // this warp's cycles per phase (g_verify_clocks; a CTA lasts << 2^32 cycles)
  const uint32_t clk0 = kClk ? (uint32_t)clock() : 0u;
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
  if (kClk) clk[0] = (uint32_t)clock() - clk0;
  unsigned long long cert = 0ull;                 // 4-bit counters: CERTAIN inliers of this thread's queries per candidate
#pragma unroll 1
  for (int t = 0; t <= last_tile; ++t) {
    const long long tile0 = qbase + (long long)t * kThreads;
    uint32_t live_mask = sLive[t * 4 + (tid >> 5)];                 // this warp's candidates (warp-uniform)
    if (kStats) st.culled += (lane == 0 && tile0 + (tid & ~31) < nQ) ? (unsigned long long)(nc - __popc(live_mask)) : 0ull;
    const bool last = t == last_tile;
    if (live_mask == 0u && !last) continue;       // warp-uniform: nothing to do for this warp's 32 queries (no CTA barrier below)
    uint32_t clk_t = kClk ? (uint32_t)clock() : 0u;
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
    if (kClk) {
      const uint32_t now = (uint32_t)clock();
      clk[1] += now - clk_t;
      clk_t = now;
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
    if (kClk) clk[2] += (uint32_t)clock() - clk_t;
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
#if S4G_VERIFY_CLOCKS
  if (kClk && lane == 0) {
    clk[3] = (uint32_t)clock() - clk0;
#pragma unroll
    for (int i = 0; i < 4; ++i) atomicAdd(&g_verify_clocks[i], (unsigned long long)clk[i]);
  }
#endif
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

#if S4G_VERIFY_CLOCKS
// Only in builds with -DS4G_VERIFY_CLOCKS=1 (not part of include/s4g.h): the phase cycles of g_verify_clocks summed since the
// last reset, after the context's stream has finished; reset != 0 zeroes them afterwards.
extern "C" int s4g_verify_clocks(s4g_ctx* ctx, uint64_t* out4, int reset) {
  if (!ctx || !out4) return S4G_ERR_ARG;
  S4G_CUDA(cudaSetDevice(ctx->device));
  S4G_CUDA(cudaStreamSynchronize(ctx->stream));
  unsigned long long h[4];
  S4G_CUDA(cudaMemcpyFromSymbol(h, g_verify_clocks, sizeof(h)));
  for (int i = 0; i < 4; ++i) out4[i] = h[i];
  if (reset) {
    const unsigned long long z[4] = {0, 0, 0, 0};
    S4G_CUDA(cudaMemcpyToSymbol(g_verify_clocks, z, sizeof(z)));
  }
  return S4G_OK;
}
#endif

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
