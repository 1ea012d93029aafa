// TEST INFRASTRUCTURE ONLY (oracle/orient_normals.py builds it together with oracle/knn_port.cc; never linked into the
// product).
//
// Plain restatement of s4g_orient_normals (include/s4g.h): the brute-force s4g_knn row of every p_j with exclude = j
// (knn_bruteforce), or rows given by the caller; the undirected edges {i, j} between vertices (non-zero normals) of the
// symmetrised rows; each edge's dot = (xi xj + yi yj) + zi zj and flip dot < 0 in fp32 (-ffp-contract=off: no FMA);
// Kruskal over the edges sorted by (|dot| descending, lo, hi) with a sequential union-find; root = the smallest member of
// each component; the anchor (the root, or the member nearest the viewpoint with s4g_normals' sign rule); and the parity
// of every member by a breadth-first walk of the forest from the anchor.  Shares no code with the device.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <deque>
#include <vector>

extern "C" void knn_bruteforce(const float* P, long nP, const float* X, long n, const float* T, int k, float sq_radius,
                               const int32_t* exclude, int32_t* out_index, float* out_sq);

namespace {

struct Edge {
  uint32_t abits;   // bits of |dot| (a NaN as 0x7FC00000)
  int32_t lo, hi;
  int flip;
};

bool vertex(const float* n) { return !(n[0] == 0.f && n[1] == 0.f && n[2] == 0.f); }

int find(std::vector<int>& parent, int x) {
  while (parent[x] != x) {
    parent[x] = parent[parent[x]];
    x = parent[x];
  }
  return x;
}

}  // namespace

extern "C" {

// 0 on success; 2 (S4G_ERR_ARG) for bad arguments or a non-finite normal component.  rows_in: n x k (index, -1 padding
// at the end) or null for the brute force.  root and tree_edges may be null.
int orient_normals_port(const float* P, long n, const float* normals, int k, float sq_radius, const float* viewpoint,
                        const int32_t* rows_in, float* normals_out, int32_t* root, int64_t* out2, int32_t* tree_edges) {
  if (k < 1 || k > 64 || std::isnan(sq_radius) || sq_radius < 0.f || !normals || !normals_out || !out2 || n < 1)
    return 2;
  if (viewpoint && !(std::isfinite(viewpoint[0]) && std::isfinite(viewpoint[1]) && std::isfinite(viewpoint[2]))) return 2;
  for (long i = 0; i < 3 * n; ++i)
    if (!std::isfinite(normals[i])) return 2;
  std::vector<int32_t> rows;
  if (!rows_in) {
    rows.resize((size_t)n * k);
    std::vector<int32_t> excl(n);
    for (long j = 0; j < n; ++j) excl[j] = (int32_t)j;
    knn_bruteforce(P, n, P, n, nullptr, k, sq_radius, excl.data(), rows.data(), nullptr);
    rows_in = rows.data();
  }
  std::vector<Edge> edges;
  for (long u = 0; u < n; ++u) {
    if (!vertex(normals + 3 * u)) continue;
    for (int e = 0; e < k; ++e) {
      const int32_t v = rows_in[u * k + e];
      if (v < 0) continue;
      if (!vertex(normals + 3 * (long)v)) continue;
      const float* a = normals + 3 * u;
      const float* b = normals + 3 * (long)v;
      const float dot = (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2];
      const float ad = std::fabs(dot);
      uint32_t bits;
      std::memcpy(&bits, &ad, 4);
      if (std::isnan(ad)) bits = 0x7FC00000u;
      edges.push_back(Edge{bits, (int32_t)std::min<long>(u, v), (int32_t)std::max<long>(u, v), dot < 0.f ? 1 : 0});
    }
  }
  std::sort(edges.begin(), edges.end(), [](const Edge& x, const Edge& y) {
    if (x.abits != y.abits) return x.abits > y.abits;
    if (x.lo != y.lo) return x.lo < y.lo;
    return x.hi < y.hi;
  });
  edges.erase(std::unique(edges.begin(), edges.end(), [](const Edge& x, const Edge& y) {
                return x.lo == y.lo && x.hi == y.hi;
              }), edges.end());
  // Kruskal
  std::vector<int> parent(n);
  for (long j = 0; j < n; ++j) parent[j] = (int)j;
  std::vector<std::vector<std::pair<int, int>>> adj(n);   // forest: (neighbour, flip)
  std::vector<std::pair<int32_t, int32_t>> tree;
  for (const Edge& e : edges) {
    const int a = find(parent, e.lo), b = find(parent, e.hi);
    if (a == b) continue;
    parent[std::max(a, b)] = std::min(a, b);
    tree.emplace_back(e.lo, e.hi);
    adj[e.lo].emplace_back(e.hi, e.flip);
    adj[e.hi].emplace_back(e.lo, e.flip);
  }
  // components, roots, anchors
  std::vector<int> comp(n, -1), minj(n, -1), anchor(n, -1);
  std::vector<float> ad2(n, 0.f);
  long n_comp = 0, n_vert = 0;
  for (long j = 0; j < n; ++j) {
    if (!vertex(normals + 3 * j)) continue;
    ++n_vert;
    const int c = find(parent, (int)j);
    comp[j] = c;
    if (minj[c] < 0) {
      minj[c] = (int)j;   // ascending j: the first member met is the smallest
      ++n_comp;
    }
    if (viewpoint) {
      const float dx = P[3 * j] - viewpoint[0], dy = P[3 * j + 1] - viewpoint[1], dz = P[3 * j + 2] - viewpoint[2];
      const float d2 = dx * dx + (dy * dy + dz * dz);
      if (anchor[c] < 0 || d2 < ad2[c]) {   // strict: a tie keeps the smaller j met first
        anchor[c] = (int)j;
        ad2[c] = d2;
      }
    }
  }
  // parity by a breadth-first walk from each component's anchor
  std::vector<int> flip(n, -1);
  for (long j = 0; j < n; ++j) {
    if (comp[j] < 0 || minj[comp[j]] != (int)j) continue;   // once per component, at its root
    const int c = comp[j];
    const int a = viewpoint ? anchor[c] : (int)j;
    int neg = 0;
    if (viewpoint) {
      const double s = ((double)viewpoint[0] - (double)P[3 * a]) * (double)normals[3 * a] +
                       ((double)viewpoint[1] - (double)P[3 * a + 1]) * (double)normals[3 * a + 1] +
                       ((double)viewpoint[2] - (double)P[3 * a + 2]) * (double)normals[3 * a + 2];
      neg = s < 0.0 ? 1 : 0;
    }
    std::deque<int> q{a};
    flip[a] = neg;
    while (!q.empty()) {
      const int x = q.front();
      q.pop_front();
      for (const auto& nb : adj[x])
        if (flip[nb.first] < 0) {
          flip[nb.first] = flip[x] ^ nb.second;
          q.push_back(nb.first);
        }
    }
  }
  for (long j = 0; j < n; ++j) {
    for (int c = 0; c < 3; ++c) {
      const float v = normals[3 * j + c];
      normals_out[3 * j + c] = flip[j] == 1 ? -v : v;
    }
    if (root) root[j] = comp[j] < 0 ? -1 : minj[comp[j]];
  }
  std::sort(tree.begin(), tree.end());
  if (tree_edges)
    for (size_t i = 0; i < tree.size(); ++i) {
      tree_edges[2 * i] = tree[i].first;
      tree_edges[2 * i + 1] = tree[i].second;
    }
  out2[0] = n_comp;
  out2[1] = (int64_t)tree.size();
  return n_vert - n_comp == (long)tree.size() ? 0 : 1;
}

}  // extern "C"
