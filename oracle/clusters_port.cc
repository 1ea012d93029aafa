// TEST INFRASTRUCTURE ONLY (oracle/clusters.py builds it; never linked into the product).
//
// Plain restatement of s4g_euclidean_clusters (include/s4g.h).
//   Edges: (i, j), i < j, iff d^2 < sq_radius, d^2 = dx^2 + (dy^2 + dz^2) of p_j - p_i in fp32 (the device's query is p_j,
//   the point p_i), tested for every pair: O(n^2), OpenMP over blocks of rows, compiled -ffp-contract=off (no FMA).
//   Components: a sequential union-find, the larger root hooked under the smaller, so a root is its set's smallest index.
//   Clusters: the roots with min_size <= size <= max_size, ordered by (size descending, root ascending); labels[j] = the
//   rank of j's cluster or -1; offsets the running sums of the ordered sizes; members in ascending j per cluster.
#include <algorithm>
#include <cstdint>
#include <vector>

namespace {

int find(std::vector<int32_t>& parent, int32_t x) {
  while (parent[x] != x) {
    parent[x] = parent[parent[x]];
    x = parent[x];
  }
  return x;
}

void unite(std::vector<int32_t>& parent, int32_t a, int32_t b) {
  const int32_t ra = find(parent, a), rb = find(parent, b);
  if (ra < rb)
    parent[rb] = ra;
  else if (rb < ra)
    parent[ra] = rb;
}

void roots(std::vector<int32_t>& parent, long n, int32_t* root) {
  for (long j = 0; j < n; ++j) root[j] = find(parent, (int32_t)j);
}

std::vector<int32_t> singletons(long n) {
  std::vector<int32_t> parent((size_t)n);
  for (long j = 0; j < n; ++j) parent[j] = (int32_t)j;
  return parent;
}

}  // namespace

extern "C" {

// root [n] of the graph d^2 < sq_radius over P [n x 3], every pair tested
void clusters_root_bruteforce(const float* P, long n, float sq_radius, int32_t* root) {
  std::vector<int32_t> parent = singletons(n);
  const long kRows = 256;
  std::vector<std::vector<int32_t>> nb((size_t)kRows);
  for (long j0 = 0; j0 < n; j0 += kRows) {
    const long j1 = std::min(n, j0 + kRows);
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 4)
#endif
    for (long j = j0; j < j1; ++j) {
      std::vector<int32_t>& row = nb[(size_t)(j - j0)];
      row.clear();
      const float x = P[3 * j], y = P[3 * j + 1], z = P[3 * j + 2];
      for (long i = 0; i < j; ++i) {
        const float dx = x - P[3 * i], dy = y - P[3 * i + 1], dz = z - P[3 * i + 2];
        const float d2 = dx * dx + (dy * dy + dz * dz);
        if (d2 < sq_radius) row.push_back((int32_t)i);
      }
    }
    for (long j = j0; j < j1; ++j)
      for (int32_t i : nb[(size_t)(j - j0)]) unite(parent, i, (int32_t)j);
  }
  roots(parent, n, root);
}

// root [n] of the graph whose edges are (j, indices[offsets[j] .. offsets[j + 1])) -- e.g. range lists
void clusters_root_from_lists(long n, const int64_t* offsets, const int32_t* indices, int32_t* root) {
  std::vector<int32_t> parent = singletons(n);
  for (long j = 0; j < n; ++j)
    for (int64_t e = offsets[j]; e < offsets[j + 1]; ++e) unite(parent, indices[e], (int32_t)j);
  roots(parent, n, root);
}

// the clusters of a component map root [n] (root[j] = the smallest index of j's component): labels [n], *n_clusters,
// offsets [n_clusters + 1], members [offsets[n_clusters]]
void clusters_finish(long n, const int32_t* root, int min_size, int max_size, int32_t* labels, int64_t* n_clusters,
                     int64_t* offsets, int32_t* members) {
  std::vector<int64_t> size((size_t)n, 0);
  for (long j = 0; j < n; ++j) ++size[root[j]];
  std::vector<int32_t> order;
  for (long r = 0; r < n; ++r)
    if (root[r] == r && size[r] >= min_size && size[r] <= max_size) order.push_back((int32_t)r);
  std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return size[a] > size[b]; });
  std::vector<int32_t> rank((size_t)n, -1);
  for (size_t c = 0; c < order.size(); ++c) rank[order[c]] = (int32_t)c;
  *n_clusters = (int64_t)order.size();
  std::vector<int64_t> cursor(order.size() + 1, 0);
  for (size_t c = 0; c < order.size(); ++c) cursor[c + 1] = cursor[c] + size[order[c]];
  for (size_t c = 0; c <= order.size(); ++c) offsets[c] = cursor[c];
  for (long j = 0; j < n; ++j) {
    const int32_t l = rank[root[j]];
    labels[j] = l;
    if (l >= 0) members[cursor[l]++] = (int32_t)j;
  }
}

// the whole contract on P: root [n] (may be null), labels [n], *n_clusters, offsets [n + 1], members [n]
void clusters_port(const float* P, long n, float sq_radius, int min_size, int max_size, int32_t* labels, int32_t* root,
                   int64_t* n_clusters, int64_t* offsets, int32_t* members) {
  std::vector<int32_t> r((size_t)n);
  clusters_root_bruteforce(P, n, sq_radius, r.data());
  if (root)
    for (long j = 0; j < n; ++j) root[j] = r[j];
  clusters_finish(n, r.data(), min_size, max_size, labels, n_clusters, offsets, members);
}

}  // extern "C"
