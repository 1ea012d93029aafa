// Consistent orientation of point normals on the resident P (s4g_orient_normals, include/s4g.h): Hoppe et al.'s
// propagation of signs along a minimum spanning tree of the k-nearest graph, with |n_i . n_j| as the weight, made exact.
//
// Graph.  A vertex is a point whose normal is not (0, 0, 0).  Rows: the P points go to the existing k_knn instances
// (query.cu) in the grid's sorted order (s4g_launch_sorted_queries, as outliers.cu), each excluding itself, no T, the
// caller's k and sq_radius; row t belongs to sorted point t of original index u = GridDev::pts[t].w.  Every real row
// entry v with both ends vertices is an arc (u, v) of the undirected edge {u, v}; an edge held by both rows is seen
// twice, which changes no minimum below.  Edge values, fp32, no FMA: dot = (xu xv + yu yv) + zu zv (the same float from
// either end), flip f = dot < 0, and the order key (~bits(|dot|), lo, hi): |dot| descending, then lo = min(u, v), then
// hi = max(u, v).  A NaN dot (products that overflow to opposite infinities) ranks as 0x7FC00000, above +inf.
//
// Borůvka rounds.  Every point x holds a link word L[x] = (y << 1) | p: y an ancestor of x in the forest being built and
// p the xor of f over the forest path from x to y.  A root r holds (r << 1).  Round r, all on the context's stream:
//   k_on_find     every x follows and halves its links to its root: cp[x] = (comp << 1) | par, the component's
//                 representative and x's parity relative to it (L[x] is left pointing there); the best-edge slots reset;
//   k_on_best<1>  per row, over the entries whose ends lie in different components: the smallest (~bits(|dot|), lo) as
//                 one 64-bit atomicMin at both components (the row's own end reduced in registers first);
//   k_on_best<2>  among those entries, the ones equal to their component's minimum: the smallest hi (32-bit atomicMin);
//   k_on_hook     every representative c with a best edge (u in c, v in d = comp[v]): unless the edge is also d's best
//                 edge and c < d, L[c] = (d << 1) | (par[u] ^ f(u, v) ^ par[v]) and the edge is recorded in the forest.
// A round that finds no edge between two components clears its `active` flag; the kernels of every later round read
// the flag and return, so the host enqueues the fixed chain of ceil(log2 nP) + 1 rounds (non-isolated components at
// least halve per round) with no synchronisation.
//
// Why the hooks form a forest, and the unique one.  The order is total, so every component has one smallest leaving
// edge, and by the cut property that edge lies in the (unique) minimum spanning forest.  The hooks c -> d have
// out-degree at most 1.  Along a chain c1 -> c2 -> c3 the edge c2 chose is at most the edge {c1, c2} c1 chose, and equal
// only when it is the same edge; so a cycle of three or more components would need a strictly decreasing cycle of edges,
// which cannot be.  The only cycles are mutual pairs, two components choosing the same edge, and the larger hooks under
// the smaller: a forest, each hook one forest edge, recorded once.  The recorded edges are therefore the minimum
// spanning forest whatever the order in which threads ran.
//
// Why par is the parity of the forest path.  Invariant: L[x] = (y, p) with y an ancestor of x and p the xor of f over
// the path x -> y.  It holds at the start (y = x, p = 0).  A hook sets L[c] = (d, par[u] ^ f(u, v) ^ par[v]) with par
// taken from the snapshot cp of this round: the path c -> d is c -> u inside c's tree, the edge (u, v), v -> d inside
// d's tree, so the xor is exactly that.  k_on_find composes (x -> y) and (y -> z) into (x -> z) by xor; each link word
// is one 32-bit load or store, so a thread reading a word another is rewriting sees the old or the new pair, both true.
// So par[x] after the last round is the parity of the forest path from x to its tree's root, and the parity of the
// path between a member x and the component's anchor a is par[x] ^ par[a]: a function of the forest alone.
//
// Finish.  k_on_roots: root = the smallest member (atomicMin on j), the anchor = the smallest (bits(d^2), j) with
// d = p - v in fp32 (viewpoint only), the component count.  k_on_anchor: per component, the anchor's sign relative to
// the representative, with s4g_normals' viewpoint rule ((v - p_a) . n_a < 0 in double).  k_on_output: each normal is
// its input, negated iff that sign xor par[x]: an exact sign flip.  The forest edges, recorded as lo << B | hi in
// arbitrary order, are put in ascending (lo, hi) by cub::DeviceRadixSort::SortKeys (the unused slots hold all ones and
// sort last) and written as int32 pairs.  Every output is integer work on the forest plus a comparison of a double dot
// product computed in a fixed order: the same bits on every run and on a CPU restatement compiled without contraction.
#include "s4g_internal.cuh"
#include <cub/cub.cuh>
#include <cmath>

namespace {

constexpr int kThreads = 256;
constexpr int kRowThreads = 128;
constexpr int kMaxK = 64;                      // k_knn's widest instance
constexpr int kMaxRounds = 32;                 // ceil(log2 nP) + 1 for nP < 2^31
constexpr unsigned long long kNoEdge = ~0ull;

// device state of one call (int32 words)
struct OnMeta {
  int bad;            // some normal component is not finite
  int n_tree;         // forest edges recorded
  int n_components;
  int pad;
  int active[kMaxRounds];   // active[r]: round r found an edge between two components
};

unsigned nblk(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

__device__ __forceinline__ float3 on_normal(const float* __restrict__ nrm, long long j) {
  return make_float3(__ldg(&nrm[3 * j]), __ldg(&nrm[3 * j + 1]), __ldg(&nrm[3 * j + 2]));
}
__device__ __forceinline__ bool on_vertex(float3 n) { return !(n.x == 0.f && n.y == 0.f && n.z == 0.f); }
// (xa xb + ya yb) + za zb, each operation one fp32 rounding
__device__ __forceinline__ float on_dot(float3 a, float3 b) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fmul_rn(a.z, b.z));
}
// (~bits(|dot|)) << 32 | lo: the first two fields of the edge order as one unsigned minimum
__device__ __forceinline__ unsigned long long on_key(float dot, uint32_t lo) {
  const float a = fabsf(dot);
  const uint32_t b = a != a ? 0x7FC00000u : __float_as_uint(a);
  return ((unsigned long long)(~b) << 32) | lo;
}

// i < n: exclude[i] = the original index of sorted point i, L[i] = (i << 1), the finiteness of normal i;
// i < n - 1: the forest key slot i holds the filler (all ones over 2B bits, after every real key)
__global__ void __launch_bounds__(kThreads)
k_on_init(const float4* __restrict__ pts, int n, const float* __restrict__ nrm, int32_t* __restrict__ exclude,
          uint32_t* __restrict__ L, unsigned long long* __restrict__ keys, unsigned long long filler,
          OnMeta* __restrict__ meta) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  exclude[i] = __float_as_int(pts[i].w);
  L[i] = (uint32_t)i << 1;
  if (i < n - 1) keys[i] = filler;
  const float3 v = on_normal(nrm, i);
  if (!isfinite(v.x) || !isfinite(v.y) || !isfinite(v.z)) atomicOr(&meta->bad, 1);
}

// cp[x] = (root << 1) | parity of x relative to it, following and halving x's links; the best-edge slots of x reset.
// gate >= 0: only when round `gate` hooked something
__global__ void __launch_bounds__(kThreads)
k_on_find(int n, uint32_t* L, uint32_t* __restrict__ cp, unsigned long long* __restrict__ best1,
          uint32_t* __restrict__ best2, const OnMeta* __restrict__ meta, int gate) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= n || (gate >= 0 && !meta->active[gate])) return;
  const uint32_t w = __ldcg(&L[x]);
  uint32_t h = w >> 1, p = w & 1u;
#pragma unroll 1
  while (true) {
    const uint32_t w2 = __ldcg(&L[h]);
    if ((w2 >> 1) == h) break;   // h is a root
    h = w2 >> 1;
    p ^= w2 & 1u;
    __stcg(&L[x], (h << 1) | p);
  }
  cp[x] = (h << 1) | p;
  best1[x] = kNoEdge;
  best2[x] = ~0u;
}

// one thread per row t (original index u): kPass 1, the smallest (~bits(|dot|), lo) of the edges leaving comp[u] /
// entering comp[v]; kPass 2, the smallest hi among the edges equal to those minima
template <int kPass>
__global__ void __launch_bounds__(kRowThreads)
k_on_best(const float4* __restrict__ sorted, const int32_t* __restrict__ rows, int n, int k, const float* __restrict__ nrm,
          const uint32_t* __restrict__ cp, unsigned long long* best1, uint32_t* best2, OnMeta* meta, int r) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  if (kPass == 1 ? (r > 0 && !meta->active[r - 1]) : !meta->active[r]) return;
  const uint32_t u = (uint32_t)__float_as_int(__ldg(&sorted[t]).w);
  const float3 nu = on_normal(nrm, u);
  if (!on_vertex(nu)) return;
  const uint32_t cu = __ldg(&cp[u]) >> 1;
  const unsigned long long target = kPass == 2 ? best1[cu] : 0ull;
  const int32_t* __restrict__ row = rows + t * (long long)k;
  unsigned long long m1 = kNoEdge;
  uint32_t mh = ~0u;
#pragma unroll 1
  for (int e = 0; e < k; ++e) {
    const int32_t v = __ldg(&row[e]);
    if (v < 0) break;                  // the padding sits at the row's end
    const float3 nv = on_normal(nrm, v);
    if (!on_vertex(nv)) continue;
    const uint32_t cv = __ldg(&cp[v]) >> 1;
    if (cv == cu) continue;
    const uint32_t lo = min(u, (uint32_t)v), hi = max(u, (uint32_t)v);
    const unsigned long long key = on_key(on_dot(nu, nv), lo);
    if (kPass == 1) {
      m1 = min(m1, key);
      atomicMin(&best1[cv], key);
    } else {
      if (key == target) mh = min(mh, hi);
      if (key == best1[cv]) atomicMin(&best2[cv], hi);
    }
  }
  if (kPass == 1 && m1 != kNoEdge) {
    atomicMin(&best1[cu], m1);
    if (!*(volatile int*)&meta->active[r]) meta->active[r] = 1;
  }
  if (kPass == 2 && mh != ~0u) atomicMin(&best2[cu], mh);
}

// one thread per representative c with a best edge: the hook of c under the component at its far end (see the header)
__global__ void __launch_bounds__(kThreads)
k_on_hook(int n, const float* __restrict__ nrm, const uint32_t* __restrict__ cp, const unsigned long long* __restrict__ best1,
          const uint32_t* __restrict__ best2, uint32_t* L, unsigned long long* __restrict__ keys, int key_shift,
          OnMeta* meta, int r) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= n || !meta->active[r]) return;
  const uint32_t c = (uint32_t)x;
  if (cp[c] != (c << 1)) return;       // not a representative
  const unsigned long long b1 = best1[c];
  if (b1 == kNoEdge) return;
  const uint32_t lo = (uint32_t)b1, hi = best2[c];
  const bool lo_in = (cp[lo] >> 1) == c;
  const uint32_t u = lo_in ? lo : hi, v = lo_in ? hi : lo;
  const uint32_t d = cp[v] >> 1;
  if (best1[d] == b1 && best2[d] == hi && c < d) return;   // a mutual pair: the larger representative hooks
  const uint32_t f = on_dot(on_normal(nrm, lo), on_normal(nrm, hi)) < 0.f ? 1u : 0u;
  __stcg(&L[c], (d << 1) | ((cp[u] ^ cp[v] ^ f) & 1u));
  const int slot = atomicAdd(&meta->n_tree, 1);
  keys[slot] = ((unsigned long long)lo << key_shift) | hi;
}

// per vertex x of component c: minj[c] = the smallest member, anchor[c] = the smallest (bits(d^2), x) (viewpoint only),
// and the number of components
__global__ void __launch_bounds__(kThreads)
k_on_roots(int n, const float* __restrict__ nrm, const float4* __restrict__ P, const uint32_t* __restrict__ cp, bool has_vp,
           float vx, float vy, float vz, unsigned long long* __restrict__ anchor, uint32_t* __restrict__ minj,
           OnMeta* __restrict__ meta) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = x < n && on_vertex(on_normal(nrm, x));
  const uint32_t c = live ? cp[x] >> 1 : 0u;
  if (live) {
    atomicMin(&minj[c], (uint32_t)x);
    if (has_vp) {
      const float4 p = __ldg(&P[x]);
      const float dx = __fsub_rn(p.x, vx), dy = __fsub_rn(p.y, vy), dz = __fsub_rn(p.z, vz);
      const float d2 = __fadd_rn(__fmul_rn(dx, dx), __fadd_rn(__fmul_rn(dy, dy), __fmul_rn(dz, dz)));
      atomicMin(&anchor[c], ((unsigned long long)__float_as_uint(d2) << 32) | (uint32_t)x);
    }
  }
  const unsigned roots = __ballot_sync(0xffffffffu, live && c == (uint32_t)x);
  if ((threadIdx.x & 31) == 0 && roots != 0u) atomicAdd(&meta->n_components, __popc(roots));
}

// per representative c of a component: anchor[c] = the anchor's sign relative to c (bit 0)
__global__ void __launch_bounds__(kThreads)
k_on_anchor(int n, const float* __restrict__ nrm, const float4* __restrict__ P, const uint32_t* __restrict__ cp, bool has_vp,
            float vx, float vy, float vz, unsigned long long* __restrict__ anchor, const uint32_t* __restrict__ minj) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= n) return;
  const uint32_t c = (uint32_t)x;
  if (cp[c] != (c << 1) || minj[c] == ~0u) return;   // not a representative, or not a vertex
  const uint32_t a = has_vp ? (uint32_t)anchor[c] : minj[c];
  uint32_t neg = 0u;
  if (has_vp) {
    const float4 p = __ldg(&P[a]);
    const float3 na = on_normal(nrm, a);
    neg = ((double)vx - (double)p.x) * (double)na.x + ((double)vy - (double)p.y) * (double)na.y +
                  ((double)vz - (double)p.z) * (double)na.z < 0.0 ? 1u : 0u;
  }
  anchor[c] = (unsigned long long)((neg ^ cp[a]) & 1u);
}

// the outputs of point x: its normal, negated iff its component's anchor sign xor par[x]; root (-1: no normal)
__global__ void __launch_bounds__(kThreads)
k_on_output(int n, const float* nrm, float* out, const uint32_t* __restrict__ cp, const unsigned long long* __restrict__ anchor,
            const uint32_t* __restrict__ minj, int32_t* __restrict__ root) {
  const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= n) return;
  float3 v = make_float3(nrm[3 * x], nrm[3 * x + 1], nrm[3 * x + 2]);
  int32_t rx = -1;
  if (on_vertex(v)) {
    const uint32_t c = cp[x] >> 1;
    if (((uint32_t)anchor[c] ^ cp[x]) & 1u) v = make_float3(-v.x, -v.y, -v.z);
    rx = (int32_t)minj[c];
  }
  out[3 * x] = v.x;
  out[3 * x + 1] = v.y;
  out[3 * x + 2] = v.z;
  if (root != nullptr) root[x] = rx;
}

// out2 = {n_components or -1 for a non-finite normal, n_tree_edges}; the sorted forest keys as (lo, hi) int32 pairs
__global__ void __launch_bounds__(kThreads)
k_on_edges(const unsigned long long* __restrict__ keys, int n_slots, int key_shift, const OnMeta* __restrict__ meta,
           int32_t* __restrict__ tree, int64_t* __restrict__ out2) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) {
    out2[0] = meta->bad ? -1 : (int64_t)meta->n_components;
    out2[1] = meta->n_tree;
  }
  if (tree == nullptr || i >= n_slots || i >= meta->n_tree) return;
  const unsigned long long key = keys[i];
  tree[2 * i] = (int32_t)(key >> key_shift);
  tree[2 * i + 1] = (int32_t)(key & ((1ull << key_shift) - 1ull));
}

size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

// bits of one index field of the forest keys: every index is below 2^B
int key_shift(int n) {
  int b = 1;
  while (b < 31 && ((int64_t)1 << b) < (int64_t)n) ++b;
  return b;
}

int rounds(int n) {
  int r = 1;
  while (((int64_t)1 << (r - 1)) < (int64_t)n) ++r;
  return r;   // ceil(log2 n) + 1
}

int check_args(s4g_ctx* ctx, const char* who, const void* normals, int k, float sq_radius, const float* viewpoint,
               const void* normals_out, const void* out2) {
  const bool vp_ok = viewpoint == nullptr ||
                     (std::isfinite(viewpoint[0]) && std::isfinite(viewpoint[1]) && std::isfinite(viewpoint[2]));
  if (k < 1 || k > kMaxK || std::isnan(sq_radius) || sq_radius < 0.f || normals == nullptr || normals_out == nullptr ||
      out2 == nullptr || !vp_ok) {
    ctx->err = std::string(who) + ": bad arguments (1 <= k <= 64, sq_radius >= 0 and not NaN, normals, normals_out and "
                                  "out2 != NULL, viewpoint NULL or finite)";
    return S4G_ERR_ARG;
  }
  if (ctx->nP <= 0) {
    ctx->err = std::string(who) + ": call s4g_set_cloud_p first";
    return S4G_ERR_STATE;
  }
  return S4G_OK;
}

// enqueue the whole call on the context's stream, every array a device pointer.  Scratch A: the sorted queries (12 bytes
// per point); B: the rows (4k); C: exclude, L, cp, best1 (also the anchors), best2 (also the smallest members), the two
// forest key buffers and the meta block (40 bytes per point); dCub: the sort's storage.
int launch(s4g_ctx* ctx, const float* d_normals, int k, float sq_radius, const float* viewpoint, float* d_normals_out,
           int32_t* d_root, int64_t* d_out2, int32_t* d_tree_edges) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  const int n = ctx->nP;
  const size_t N = (size_t)n;
  cudaStream_t st = ctx->stream;
  const size_t sizes[] = {4 * N, 4 * N, 4 * N, 8 * N, 4 * N, 8 * N, 8 * N, sizeof(OnMeta)};
  size_t total = 0;
  for (size_t b : sizes) total += align256(b);
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, N * 3 * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, N * (size_t)k * sizeof(int32_t)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchC, total));
  const int shift = key_shift(n);
  const int n_slots = n - 1;
  size_t sort_bytes = 0;
  cub::DoubleBuffer<unsigned long long> dk(nullptr, nullptr);
  if (n_slots > 0) S4G_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, sort_bytes, dk, n_slots, 0, 2 * shift, st));
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, sort_bytes));
  char* p = ctx->dScratchC.as<char>();
  char* part[8];
  for (int i = 0; i < 8; ++i) {
    part[i] = p;
    p += align256(sizes[i]);
  }
  float* d_xyz = ctx->dScratchA.as<float>();
  int32_t* rows = ctx->dScratchB.as<int32_t>();
  int32_t* excl = reinterpret_cast<int32_t*>(part[0]);
  uint32_t* L = reinterpret_cast<uint32_t*>(part[1]);
  uint32_t* cp = reinterpret_cast<uint32_t*>(part[2]);
  unsigned long long* best1 = reinterpret_cast<unsigned long long*>(part[3]);
  uint32_t* best2 = reinterpret_cast<uint32_t*>(part[4]);
  unsigned long long* keys0 = reinterpret_cast<unsigned long long*>(part[5]);
  unsigned long long* keys1 = reinterpret_cast<unsigned long long*>(part[6]);
  OnMeta* meta = reinterpret_cast<OnMeta*>(part[7]);
  const unsigned long long filler = (1ull << (2 * shift)) - 1ull;
  const unsigned nb = nblk(n, kThreads), nr = nblk(n, kRowThreads);

  S4G_CUDA(cudaMemsetAsync(meta, 0, sizeof(OnMeta), st));
  k_on_init<<<nb, kThreads, 0, st>>>(ctx->grid.pts, n, d_normals, excl, L, keys0, filler, meta);
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  S4G_TRY(s4g_launch_sorted_queries(ctx, d_xyz));
  S4G_TRY(s4g_launch_knn(ctx, d_xyz, n, nullptr, k, sq_radius, excl, rows, nullptr, nullptr));
  const int R = rounds(n);
  for (int r = 0; r < R; ++r) {
    k_on_find<<<nb, kThreads, 0, st>>>(n, L, cp, best1, best2, meta, r - 1);
    k_on_best<1><<<nr, kRowThreads, 0, st>>>(ctx->grid.pts, rows, n, k, d_normals, cp, best1, best2, meta, r);
    k_on_best<2><<<nr, kRowThreads, 0, st>>>(ctx->grid.pts, rows, n, k, d_normals, cp, best1, best2, meta, r);
    k_on_hook<<<nb, kThreads, 0, st>>>(n, d_normals, cp, best1, best2, L, keys0, shift, meta, r);
    ctx->launches += 4;
    S4G_CUDA(cudaGetLastError());
  }
  // every link resolved (ungated), the slots reset for the smallest members and the anchors
  k_on_find<<<nb, kThreads, 0, st>>>(n, L, cp, best1, best2, meta, -1);
  const bool has_vp = viewpoint != nullptr;
  const float vx = has_vp ? viewpoint[0] : 0.f, vy = has_vp ? viewpoint[1] : 0.f, vz = has_vp ? viewpoint[2] : 0.f;
  const float4* P = ctx->dP.as<float4>();
  k_on_roots<<<nb, kThreads, 0, st>>>(n, d_normals, P, cp, has_vp, vx, vy, vz, best1, best2, meta);
  k_on_anchor<<<nb, kThreads, 0, st>>>(n, d_normals, P, cp, has_vp, vx, vy, vz, best1, best2);
  k_on_output<<<nb, kThreads, 0, st>>>(n, d_normals, d_normals_out, cp, best1, best2, d_root);
  ctx->launches += 4;
  S4G_CUDA(cudaGetLastError());
  const unsigned long long* sorted = keys0;
  if (d_tree_edges != nullptr && n_slots > 0) {
    cub::DoubleBuffer<unsigned long long> keys(keys0, keys1);
    S4G_CUDA(cub::DeviceRadixSort::SortKeys(ctx->dCub.p, sort_bytes, keys, n_slots, 0, 2 * shift, st));
    ctx->launches++;
    sorted = keys.Current();
  }
  k_on_edges<<<std::max(1u, nblk(n_slots, kThreads)), kThreads, 0, st>>>(sorted, n_slots, shift, meta, d_tree_edges,
                                                                        d_out2);
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;
}

}  // namespace

extern "C" int s4g_orient_normals_dev(s4g_ctx* ctx, const float* d_normals, int k, float sq_radius, const float* viewpoint,
                                      float* d_normals_out, int32_t* d_root, int64_t* d_out2, int32_t* d_tree_edges) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(check_args(ctx, "s4g_orient_normals_dev", d_normals, k, sq_radius, viewpoint, d_normals_out, d_out2));
  return launch(ctx, d_normals, k, sq_radius, viewpoint, d_normals_out, d_root, d_out2, d_tree_edges);
}

// the device copies in ctx->dFilter: normals (worked on in place), root, the forest, out2; then out2 back first, and only
// the defined part of the forest
extern "C" int s4g_orient_normals(s4g_ctx* ctx, const float* normals, int k, float sq_radius, const float* viewpoint,
                                  float* normals_out, int32_t* root, int64_t* out2, int32_t* tree_edges) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(check_args(ctx, "s4g_orient_normals", normals, k, sq_radius, viewpoint, normals_out, out2));
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t N = (size_t)ctx->nP, a3 = align256(12 * N), a1 = align256(4 * N), a2 = align256(8 * N);
  S4G_TRY(s4g_reserve(ctx, ctx->dFilter, a3 + a1 + a2 + 256));
  char* p = ctx->dFilter.as<char>();
  float* d_n = reinterpret_cast<float*>(p);
  int32_t* d_root = reinterpret_cast<int32_t*>(p + a3);
  int32_t* d_tree = reinterpret_cast<int32_t*>(p + a3 + a1);
  int64_t* d_out2 = reinterpret_cast<int64_t*>(p + a3 + a1 + a2);
  S4G_CUDA(cudaMemcpyAsync(d_n, normals, 12 * N, cudaMemcpyHostToDevice, st));
  S4G_TRY(launch(ctx, d_n, k, sq_radius, viewpoint, d_n, root != nullptr ? d_root : nullptr, d_out2,
                 tree_edges != nullptr ? d_tree : nullptr));
  int64_t o2[2] = {0, 0};
  S4G_CUDA(cudaMemcpyAsync(o2, d_out2, sizeof o2, cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  if (o2[0] < 0) {
    ctx->err = "s4g_orient_normals: a normal component is not finite";
    return S4G_ERR_ARG;
  }
  S4G_CUDA(cudaMemcpyAsync(normals_out, d_n, 12 * N, cudaMemcpyDeviceToHost, st));
  if (root != nullptr) S4G_CUDA(cudaMemcpyAsync(root, d_root, 4 * N, cudaMemcpyDeviceToHost, st));
  if (tree_edges != nullptr && o2[1] > 0)
    S4G_CUDA(cudaMemcpyAsync(tree_edges, d_tree, 8 * (size_t)o2[1], cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  out2[0] = o2[0];
  out2[1] = o2[1];
  return S4G_OK;
}
