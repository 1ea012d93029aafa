// Point queries on the resident P grid, for arbitrary query points: the k nearest P points within a radius (s4g_knn;
// s4g_nearest is its k = 1), every P point within a radius (s4g_range), the capped neighbour counts of the radius
// outlier filter (s4g_radius_outliers) and the union-find of the Euclidean clusters (s4g_euclidean_clusters).  They are
// the reference kd-tree's queries: the restricted closest point
// (KdTree::doQueryRestrictedClosestIndex, kdtree.h:388-453) and the range query (KdTree::doQueryDistProcessIndices,
// kdtree.h:462-514).  One thread per query; y = T x (exact_tq) or x, and d^2 = dx^2 + (dy^2 + dz^2) in fp32 as in
// Verify's exact test.
//
// Search.  The cell coordinates of y, u = (y - o) * inv_h, are taken in double.  The coarse blocks of GridDev::csat
// ((2^cshift)^3 cells) form an implicit tree of boxes: the root is the whole coarse lattice, and a box splits into two
// halves of its longest axis down to single blocks.  The thread descends it depth first with an explicit stack: a box is
// dropped when csat says it holds no point (8 look-ups) or by its lower bound (below); a single block left is scanned row
// by row -- rows dropped by their bound are skipped, the others are contiguous runs of the sorted points, one per brick
// they cross.
// Work: every box opened either is a block that is scanned or has a child that is not empty and within the bound, so a
// query opens at most (1 + 2 x depth) boxes per block it scans (depth <= log2 of the lattice's extents, ~30); empty
// space costs one look-up of csat per box, whatever its size.
//
// Lower bound (cells_bound).  A point stored in cell c (on one axis) was binned by floorf(fl(fl(p - o) * inv_h))
// (context.cu, cell_of; never clamped, the grid has a 1.5-cell margin): two roundings of relative size 2^-24 of a value
// below n + 1 cells, so its exact coordinate v = (p - o) * inv_h lies in (c - eps, c + 1 + eps) with
// eps = (max(nx, ny, nz) + 2) * 2^-21, twice the rounding (1e-3 cell for 2048 cells).  For every point binned in a box of
// cells, |y - p| on that axis is at least gap / inv_h, gap = the distance from u to [c0 - eps, c1 + 1 + eps], so
// L = sum gap^2 / inv_h^2 bounds the exact d^2.  The d^2 the kernel computes takes five roundings of relative size 2^-24
// (plus 2^-148 when it is subnormal), so it is at least L (1 - 2^-20) - 2^-140; that value, from double arithmetic
// (relative error ~2^-50) rounded down to fp32, is the bound.  A bound that is too low only costs time; this one is never
// above a d^2 the kernel computes.
//
// Drop rule and search order.  Every point of a dropped box or row therefore has a d^2 at least its bound.  The k-nearest
// rows drop a bound strictly above theirs (>): a point at exactly the bound may still win a tie on its index.  The range
// lists and radius counts drop a bound at or above sq_radius (>=): their test is d^2 < sq_radius, strict, so such a point
// is not taken.  Each query's answer is fixed by this alone -- it does not depend on the order in which the boxes are
// opened (see each kernel).
//
// The descent is written out in each kernel; the query set-up (load_query, query_ready, query_cells) is shared.  One
// descent template with a per-query policy (scripts/shared_descent.patch) was measured slower: DESIGN.md, the k-nearest
// section.
#include "s4g_internal.cuh"
#include <cub/cub.cuh>
#include <algorithm>
#include <cmath>

namespace {

constexpr int kThreads = 128;   // queries per CTA of the query kernels

struct NearestQuery {
  float tx, ty, tz;   // y
  int excl;           // original P index never taken (-1: none)
  double ux, uy, uz;  // cell coordinates of y
  double eps, h2;     // binning margin of the points (cells); squared cell edge
};

struct NearestStats {
  unsigned long long tested = 0, blocks = 0;
};

// y = T x of query i (T16: column-major 4x4 or nullptr: y = x)
__device__ __forceinline__ void load_query(const float* __restrict__ xyz, long long i, const float* __restrict__ T16,
                                           NearestQuery& q) {
  const float4 x = make_float4(__ldg(&xyz[3 * i]), __ldg(&xyz[3 * i + 1]), __ldg(&xyz[3 * i + 2]), 0.f);
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
}

// the cell coordinates of y and the constants of its bound
__device__ __forceinline__ void query_cells(const GridDev& g, NearestQuery& q) {
  const double ih = (double)g.inv_h;
  q.ux = ((double)q.tx - (double)g.ox) * ih;
  q.uy = ((double)q.ty - (double)g.oy) * ih;
  q.uz = ((double)q.tz - (double)g.oz) * ih;
  q.eps = (double)(max(g.nx, max(g.ny, g.nz)) + 2) * 0x1p-21;
  q.h2 = 1.0 / (ih * ih);
}

// query_cells; false (nothing to search) when y has a NaN coordinate: every d^2 is then NaN and nothing is taken
__device__ __forceinline__ bool query_ready(const GridDev& g, NearestQuery& q) {
  if (isnan(q.tx) || isnan(q.ty) || isnan(q.tz)) return false;
  query_cells(g, q);
  return true;
}

// lower bound of the d^2 the kernels compute between y and any point binned in the cells [x0, x1] x [y0, y1] x [z0, z1]
__device__ __forceinline__ float cells_bound(const NearestQuery& q, int x0, int x1, int y0, int y1, int z0, int z1) {
  const double gx = fmax(0.0, fmax(((double)x0 - q.eps) - q.ux, q.ux - ((double)x1 + 1.0 + q.eps)));
  const double gy = fmax(0.0, fmax(((double)y0 - q.eps) - q.uy, q.uy - ((double)y1 + 1.0 + q.eps)));
  const double gz = fmax(0.0, fmax(((double)z0 - q.eps) - q.uz, q.uz - ((double)z1 + 1.0 + q.eps)));
  const double b = (gx * gx + gy * gy + gz * gz) * q.h2 * (1.0 - 0x1p-20) - 0x1p-140;
  return b > 0.0 ? __double2float_rd(b) : 0.f;
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

// ---- every P point within a radius, for arbitrary query points (s4g_range): the range query of the reference's kd-tree
// (KdTree::doQueryDistProcessIndices, kdtree.h:462-514).  One thread per query: y = T x (exact_tq) or x; its list is every
// original P index j with d^2 < sq_radius (strict: the kd-tree's point test, kdtree.h:485), d^2 computed as in the
// header.  The lists come out in the order of the search; s4g_range sorts each by j afterwards.
//
// Search.  The box descent of the header with the fixed bound sq_radius: a box, or a cell row of a block, is dropped when
// csat says it is empty or when cells_bound(...) >= sq_radius, so every point of a dropped box or row has
// d^2 >= sq_radius and is not in the list.  Nothing is dropped for any other reason,
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
  NearestQuery q;
  load_query(xyz, i, T16, q);
  q.excl = -1;
  int64_t out = kFill ? offsets[i] : 0;   // fill: the next entry of this list; count: its length so far
  if (query_ready(g, q)) {
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
  query_cells(g, q);
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

// ---- the union-find of the Euclidean clusters (s4g_euclidean_clusters, finished in clusters.cu): the graph on the
// resident P with an edge (i, j), i != j, iff d^2(p_i, p_j) < sq_radius.  parent[] is indexed by original index and starts
// as parent[x] = x; on return every edge's two endpoints are in one set, and sets were only ever joined along an edge.
// One thread per
// sorted point t (GridDev::pts, w = original index j); the query is p_j as stored, d^2 as in k_range.
//
// Search.  k_range's descent, drop rule and point test with the bound sq_radius: a box, or a cell row of a block, is
// dropped when csat says it is empty or when cells_bound(...) >= sq_radius, and a point i is a neighbour when
// d^2 < sq_radius.  Every neighbour i < j is merged with j (cluster_unite).  sq_radius <= 0 drops the root: no edges.
// Invariant parent[x] <= x.  A hook writes parent[hi] = lo only where hi is a root (atomicCAS from hi) and lo < hi; the
// path halving of cluster_find (s4g_internal.cuh) writes parent[x] = parent[parent[x]], an ancestor of x, so never above
// x.  So parents strictly decrease along a path (no cycle), and the root of a set is its smallest index: the contract's
// root, with no further reduction.  A node's ancestors only ever gain members of its own set, so a read that misses
// another thread's write still returns an ancestor: it costs steps (or a failed atomicCAS), never a wrong merge.
// Correctness.
//   - Every edge is seen from its larger endpoint.  The descent is exact (the argument of the header and of k_range): the
//     thread of j meets every i with d^2(p_j, p_i) < sq_radius.  The graph is symmetric bit for bit -- under round to
//     nearest fl(a - b) = -fl(b - a), so each squared difference, and d^2, is the same float from either end -- so the
//     edge (i, j), i < j, is met by j's thread, and taking only i < j loses none.
//   - Concurrent hooks only merge sets that share an edge.  cluster_unite hooks a root only under a member of the other
//     endpoint's set, found from that edge's two ends; a failed atomicCAS (the root was hooked meanwhile) retries from
//     the new parent, and agreeing finds (both ends in one set, which stays so) end the call without a write.
//   - So the final sets are the connected components: the result depends on the edge set only, not on thread order, and
//     each component's root is its smallest index.
// Registers.  __maxnreg__(64) stands in for __launch_bounds__ (the two exclude each other): left to itself, ptxas gives
// this kernel 32 registers and spills in the point loop; at 64 it takes 60 and spills nothing.
__device__ __forceinline__ void cluster_unite(int* parent, int a, int b) {
#pragma unroll 1
  while (true) {
    const int ra = cluster_find(parent, a), rb = cluster_find(parent, b);
    if (ra == rb) return;
    const int hi = max(ra, rb), lo = min(ra, rb);
    const int old = atomicCAS(&parent[hi], hi, lo);
    if (old == hi) return;
    a = old;   // hi was hooked meanwhile: retry from its new parent, in the same set
    b = lo;
  }
}

__global__ void __maxnreg__(64)
k_cluster_link(GridDev g, int n, float sq_radius, int* __restrict__ parent) {
  const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (t >= n) return;
  const float4 self = __ldg(&g.pts[t]);
  NearestQuery q;
  q.tx = self.x;
  q.ty = self.y;
  q.tz = self.z;
  q.excl = __float_as_int(self.w);
  query_cells(g, q);
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
              const int i = __float_as_int(p.w);
              if (d2 < sq_radius && i < q.excl) cluster_unite(parent, i, q.excl);
            }
          }
          cx = xe + 1;
        }
      }
  }
}

// the sort keys of one sort chunk (s4g_range): entry base + t of the output, in query i's list [offsets[i], offsets[i + 1]),
// gets the key (i << jbits) | j, so that one radix sort of the chunk orders every list by j and keeps the lists in place
__global__ void k_range_keys(const int64_t* __restrict__ offsets, int n, int64_t base, int len,
                             const int32_t* __restrict__ indices, int jbits, unsigned long long* __restrict__ keys) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= len) return;
  const int64_t p = base + t;
  int lo = 0, hi = n - 1;   // the last i with offsets[i] <= p (offsets[0] = 0): the non-empty list that holds p
  while (lo < hi) {
    const int mid = lo + (hi - lo + 1) / 2;
    if (offsets[mid] <= p) lo = mid; else hi = mid - 1;
  }
  keys[t] = ((unsigned long long)lo << jbits) | (unsigned)indices[p];
}

// the sorted keys of a chunk back to the indices they hold
__global__ void k_range_unkey(const unsigned long long* __restrict__ keys, int len, unsigned long long jmask,
                              int32_t* __restrict__ indices) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < len) indices[t] = (int32_t)(keys[t] & jmask);
}

// ---- the k nearest P points within a radius, for arbitrary query points (s4g_knn).  One thread per query: y = T x
// (exact_tq) or x; its row is the k lexicographically smallest (d^2, original P index j) over the P points with
// d^2 <= sq_radius and j != exclude, ascending; a row with fewer such points is padded with (-1, +inf).  k = 1 is
// s4g_nearest's answer: a single best (d^2, j) under the same test and drop rule.
//
// Search.  The box descent of the header, nearer half first; the bound is
// sq_radius while fewer than k points are held, and the d^2 of the k-th held entry once k are.  A box or cell row is
// dropped when its cells_bound is strictly above the bound.  A point is inserted when d^2 <= sq_radius,
// j != exclude and (d^2, j) is below the k-th held entry (a NaN d^2 fails the first test and is never taken).
// Determinism.  cells_bound never exceeds a d^2 the kernel computes (the argument of the header), so every point of a
// dropped box or row has d^2 > bound: beyond the radius while the row is not full, and after that above the k-th held
// d^2, which only decreases -- such a point is above the final k-th entry too, so it could be neither in the row nor tie
// with its last entry.  A point at exactly the k-th distance with a smaller j is never dropped (the test is strict) and
// displaces the entry with the larger j.  Every other point is compared with the held list, and every P point is binned
// in one cell, so it is seen once: the row is the lexicographic k-minimum whatever the order of the search.
// Storage.  The held entries are 64-bit keys (d^2 bits << 32 | j), which order as (d^2, j) because d^2 is never negative
// nor NaN; kEmpty, above every key, marks a free slot.  They sit in a per-thread array of kCap slots, sorted ascending
// (local memory: it is indexed by the run-time k), and an insertion shifts the larger keys up by one.  kCap is k rounded
// up to 8, 16, 32 or 64, so that a small k does not carry the stack frame of the largest.
constexpr unsigned long long kEmpty = ~0ull;

template <int kCap, bool kStats>
__global__ void __launch_bounds__(kThreads)
k_knn(GridDev g, const float* __restrict__ xyz, int n, const float* __restrict__ T16, int k, float sq_radius,
      const int32_t* __restrict__ exclude, int32_t* __restrict__ index, float* __restrict__ sq_dist,
      unsigned long long* __restrict__ stats) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  NearestStats st;
  if (i < n) {
    NearestQuery q;
    load_query(xyz, i, T16, q);
    q.excl = exclude != nullptr ? __ldg(&exclude[i]) : -1;
    unsigned long long held[kCap];
#pragma unroll 1
    for (int e = 0; e < k; ++e) held[e] = kEmpty;
    unsigned long long kth = kEmpty;   // held[k - 1]
    float bound = sq_radius;
    if (query_ready(g, q)) {
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

// the checks every query entry point shares; `out` names its output array
int query_args(s4g_ctx* ctx, const char* who, int n, const void* xyz, float sq_radius, const void* out, const char* out_name) {
  if (n < 0 || (n > 0 && (!xyz || !out)) || std::isnan(sq_radius)) {
    ctx->err = std::string(who) + ": bad arguments (n >= 0, xyz and " + out_name + " when n > 0, sq_radius not NaN)";
    return S4G_ERR_ARG;
  }
  if (ctx->nP <= 0) {
    ctx->err = std::string(who) + ": call s4g_set_cloud_p first";
    return S4G_ERR_STATE;
  }
  return S4G_OK;
}

constexpr int kKnnMax = 64;   // the largest k of s4g_knn (the slots of k_knn's widest instance)

int knn_args(s4g_ctx* ctx, const char* who, int n, const void* xyz, int k, float sq_radius, const void* index) {
  if (k < 1 || k > kKnnMax) {
    ctx->err = std::string(who) + ": bad arguments (1 <= k <= 64)";
    return S4G_ERR_ARG;
  }
  return query_args(ctx, who, n, xyz, sq_radius, index, "index");
}

// n host query points and T (nullptr: none) -> the start of the context's scratch A: d_xyz, then d_T (nullptr when T is)
int stage_queries(s4g_ctx* ctx, const float* xyz, int n, const float* T, float*& d_xyz, float*& d_T) {
  const size_t nn = (size_t)n;
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, nn * 3 * sizeof(float) + 16 * sizeof(float)));
  d_xyz = ctx->dScratchA.as<float>();
  d_T = T != nullptr ? d_xyz + nn * 3 : nullptr;
  S4G_CUDA(cudaMemcpyAsync(d_xyz, xyz, nn * 3 * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  if (T != nullptr) S4G_CUDA(cudaMemcpyAsync(d_T, T, 16 * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  return S4G_OK;
}

// enqueue k_knn on the context's stream: the instance whose slots are k rounded up to 8, 16, 32 or 64 (stats != nullptr:
// the statistics variant)
template <int kCap>
void launch_knn_cap(s4g_ctx* ctx, unsigned nblk, const float* d_xyz, int n, const float* d_T, int k, float sq_radius,
                    const int32_t* d_exclude, int32_t* d_index, float* d_sq_dist, unsigned long long* stats) {
  if (stats != nullptr)
    k_knn<kCap, true><<<nblk, kThreads, 0, ctx->stream>>>(ctx->grid, d_xyz, n, d_T, k, sq_radius, d_exclude, d_index,
                                                          d_sq_dist, stats);
  else
    k_knn<kCap, false><<<nblk, kThreads, 0, ctx->stream>>>(ctx->grid, d_xyz, n, d_T, k, sq_radius, d_exclude, d_index,
                                                           d_sq_dist, nullptr);
}

int knn_dev(s4g_ctx* ctx, const char* who, const float* d_xyz, int n, const float* d_T, int k, float sq_radius,
            const int32_t* d_exclude, int32_t* d_index, float* d_sq_dist) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(knn_args(ctx, who, n, d_xyz, k, sq_radius, d_index));
  if (n == 0) return S4G_OK;
  return s4g_launch_knn(ctx, d_xyz, n, d_T, k, sq_radius, d_exclude, d_index, d_sq_dist, nullptr);
}

// host buffers -> the context's scratch, k_knn, back; stats: nullptr or the two counters of the statistics variant
int knn_host(s4g_ctx* ctx, const char* who, const float* xyz, int n, const float* T, int k, float sq_radius,
             const int32_t* exclude, int32_t* index, float* sq_dist, uint64_t* stats) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(knn_args(ctx, who, n, xyz, k, sq_radius, index));
  if (n == 0) return S4G_OK;
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t nn = (size_t)n, nk = nn * (size_t)k;
  float *d_xyz, *d_T;
  S4G_TRY(stage_queries(ctx, xyz, n, T, d_xyz, d_T));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, nk * sizeof(int32_t)));
  if (sq_dist != nullptr) S4G_TRY(s4g_reserve(ctx, ctx->dScratchC, nk * sizeof(float)));
  if (exclude != nullptr) S4G_TRY(s4g_reserve(ctx, ctx->dScratchD, nn * sizeof(int32_t)));
  if (stats != nullptr) S4G_TRY(s4g_reserve(ctx, ctx->dMisc, 256));
  if (exclude != nullptr)
    S4G_CUDA(cudaMemcpyAsync(ctx->dScratchD.p, exclude, nn * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if (stats != nullptr) S4G_CUDA(cudaMemsetAsync(ctx->dMisc.p, 0, 2 * sizeof(unsigned long long), st));
  S4G_TRY(s4g_launch_knn(ctx, d_xyz, n, d_T, k, sq_radius, exclude != nullptr ? ctx->dScratchD.as<int32_t>() : nullptr,
                         ctx->dScratchB.as<int32_t>(), sq_dist != nullptr ? ctx->dScratchC.as<float>() : nullptr,
                         stats != nullptr ? ctx->dMisc.as<unsigned long long>() : nullptr));
  S4G_CUDA(cudaMemcpyAsync(index, ctx->dScratchB.p, nk * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (sq_dist != nullptr) S4G_CUDA(cudaMemcpyAsync(sq_dist, ctx->dScratchC.p, nk * sizeof(float), cudaMemcpyDeviceToHost, st));
  unsigned long long h[2] = {0, 0};
  if (stats != nullptr) S4G_CUDA(cudaMemcpyAsync(h, ctx->dMisc.p, sizeof h, cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  if (stats != nullptr) {
    stats[0] = h[0];
    stats[1] = h[1];
  }
  return S4G_OK;
}

// enqueue the count pass of k_range and the scan of the lengths: d_offsets [n + 1] = 0, ..., total
int range_count(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T, float sq_radius, int64_t* d_offsets) {
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
// entry), then sort every list by index, its d^2 carried along: one radix sort of the keys (list, index), which leaves
// every list where it is.  (Not CUB's segmented sort: with more than a few hundred segments it reads its partition sizes
// back to the host and synchronises the stream.)  The sort addresses the items with int, so the lists are sorted in
// chunks: chunk c sorts the w + |P| entries of the output from c w on (at most INT_MAX), which hold every list that starts
// in the window [c w, (c + 1) w), since a list has at most |P| entries.  A list cut off at the chunk's start is the
// suffix of a list an earlier chunk sorted whole, so it stays sorted; one cut off at its end starts in a later window,
// whose chunk sorts it whole.  One chunk when total <= INT_MAX.  The scratch is 20 bytes per entry of a chunk: the keys
// and their double buffer, and the double buffer of the d^2.
int range_fill(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T, float sq_radius, const int64_t* d_offsets,
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
  auto bits = [](unsigned v) { return v ? 32 - __builtin_clz(v) : 0; };
  const int jbits = bits((unsigned)(ctx->nP - 1)), end_bit = std::max(1, jbits + bits((unsigned)(n - 1)));
  const unsigned long long jmask = (1ull << jbits) - 1;
  for (int64_t base = 0; base < total; base += window) {
    const int len = (int)std::min<int64_t>({total - base, window + ctx->nP, kMaxItems});
    S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, 2 * (size_t)len * sizeof(unsigned long long)));
    if (d_sq_dist != nullptr) S4G_TRY(s4g_reserve(ctx, ctx->dScratchC, (size_t)len * sizeof(float)));
    unsigned long long* keys = ctx->dScratchB.as<unsigned long long>();
    float* vals = d_sq_dist != nullptr ? d_sq_dist + base : nullptr;
    const unsigned blocks = (unsigned)((len + 255) / 256);
    k_range_keys<<<blocks, 256, 0, st>>>(d_offsets, n, base, len, d_indices, jbits, keys);
    ctx->launches++;
    S4G_CUDA(cudaGetLastError());
    cub::DoubleBuffer<unsigned long long> dk(keys, keys + len);
    cub::DoubleBuffer<float> dv(vals, ctx->dScratchC.as<float>());
    size_t bytes = 0;
    if (vals != nullptr) {
      S4G_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, dk, dv, len, 0, end_bit, st));
      S4G_TRY(s4g_reserve(ctx, ctx->dCub, bytes));
      S4G_CUDA(cub::DeviceRadixSort::SortPairs(ctx->dCub.p, bytes, dk, dv, len, 0, end_bit, st));
    } else {
      S4G_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, bytes, dk, len, 0, end_bit, st));
      S4G_TRY(s4g_reserve(ctx, ctx->dCub, bytes));
      S4G_CUDA(cub::DeviceRadixSort::SortKeys(ctx->dCub.p, bytes, dk, len, 0, end_bit, st));
    }
    k_range_unkey<<<blocks, 256, 0, st>>>(dk.Current(), len, jmask, d_indices + base);
    ctx->launches++;
    S4G_CUDA(cudaGetLastError());
    if (vals != nullptr && dv.Current() != vals)
      S4G_CUDA(cudaMemcpyAsync(vals, dv.Current(), (size_t)len * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  return S4G_OK;
}

}  // namespace

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

int s4g_launch_radius_count(s4g_ctx* ctx, float sq_radius, int min_neighbors, int32_t* d_counts, uint8_t* d_keep) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  const int n = ctx->nP;
  k_radius_count<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, ctx->stream>>>(ctx->grid, n, sq_radius,
                                                                                          min_neighbors, d_counts, d_keep);
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;
}

int s4g_launch_cluster_link(s4g_ctx* ctx, float sq_radius, int* d_parent) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  const int n = ctx->nP;
  k_cluster_link<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, ctx->stream>>>(ctx->grid, n, sq_radius, d_parent);
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;
}

// s4g_nearest* is the k = 1 row of s4g_knn* (the same accept test and drop rule as a single best (d^2, j))
extern "C" int s4g_nearest_dev(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T, float sq_radius,
                               const int32_t* d_exclude, int32_t* d_index, float* d_sq_dist) {
  return knn_dev(ctx, "s4g_nearest_dev", d_xyz, n, d_T, 1, sq_radius, d_exclude, d_index, d_sq_dist);
}

extern "C" int s4g_nearest(s4g_ctx* ctx, const float* xyz, int n, const float* T, float sq_radius, const int32_t* exclude,
                           int32_t* index, float* sq_dist) {
  return knn_host(ctx, "s4g_nearest", xyz, n, T, 1, sq_radius, exclude, index, sq_dist, nullptr);
}

extern "C" int s4g_nearest_probe_stats(s4g_ctx* ctx, const float* xyz, int n, const float* T, float sq_radius,
                                       const int32_t* exclude, int32_t* index, float* sq_dist, uint64_t* out2) {
  if (ctx && !out2) { ctx->err = "s4g_nearest_probe_stats: bad arguments"; return S4G_ERR_ARG; }
  if (out2) out2[0] = out2[1] = 0;
  return knn_host(ctx, "s4g_nearest_probe_stats", xyz, n, T, 1, sq_radius, exclude, index, sq_dist, out2);
}

extern "C" int s4g_knn_dev(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T, int k, float sq_radius,
                           const int32_t* d_exclude, int32_t* d_index, float* d_sq_dist) {
  return knn_dev(ctx, "s4g_knn_dev", d_xyz, n, d_T, k, sq_radius, d_exclude, d_index, d_sq_dist);
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

extern "C" int s4g_range_count_dev(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T, float sq_radius,
                                   int64_t* d_offsets) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(query_args(ctx, "s4g_range_count_dev", n, d_xyz, sq_radius, d_offsets, "offsets"));
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
  S4G_TRY(query_args(ctx, "s4g_range_fill_dev", n, d_xyz, sq_radius, d_offsets, "offsets"));
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
  S4G_TRY(query_args(ctx, "s4g_range", n, xyz, sq_radius, offsets, "offsets"));
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
  float *d_xyz, *d_T;
  S4G_TRY(stage_queries(ctx, xyz, n, T, d_xyz, d_T));
  S4G_TRY(s4g_reserve(ctx, ctx->dRangeOff, (nn + 1) * sizeof(int64_t)));
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
