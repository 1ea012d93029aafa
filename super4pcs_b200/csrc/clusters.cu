// Euclidean clusters of the resident P (s4g_euclidean_clusters, include/s4g.h): the connected components of the graph
// d^2(p_i, p_j) < sq_radius, their sizes, the clusters among them ordered by (size descending, root ascending), labels
// and the members in CSR form.
//
// Stages, all on the context's stream:
//   k_cluster_init      parent[j] = j, size[j] = 0, val[j] = j;
//   k_cluster_link      (query.cu) the concurrent union-find driven by k_range's descent: on return each set of parent[]
//                       is a component and its root is its smallest index -- the correctness argument is in its header;
//   k_cluster_compress  root[j] = find(j) (the links are all in: find only follows and halves paths), and the component
//                       sizes by integer atomicAdd at the root;
//   k_cluster_flags     key[j] = size[j] when j is a root whose size is within [min_size, max_size], else 0, and the
//                       number of such roots;
//   sort by key         cub::DeviceRadixSort::SortPairsDescending of (key, j): stable, and the j enter in ascending
//                       order, so the clusters come first by size descending, ties by root ascending; the keys 0 last;
//   offsets             the exclusive scan of the sorted keys (k_cluster_sizes copies them into the offsets, widened);
//   k_cluster_rank      rank[root] = the position of the root in that order;
//   k_cluster_labels    labels[j] = rank[root[j]] (-1: not a cluster), and the sort key of j's membership;
//   members             cub::DeviceRadixSort::SortPairs of (label, j) with the no-cluster label last: stable, j in
//                       ascending order within each cluster.
// Determinism.  The partition depends on the edge set alone (k_cluster_link), so root, size and the flags do; the counts
// are integer sums; both sorts are stable radix sorts of integer keys with the values entering in a fixed order; the scan
// is of integers.  Nothing in the output depends on scheduling.
#include "s4g_internal.cuh"
#include <cub/cub.cuh>
#include <cmath>

namespace {

constexpr int kClusterThreads = 256;

unsigned nblk(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// bits of the sort keys: every key is at most n
int key_bits(int n) {
  int b = 1;
  while (b < 31 && ((int64_t)1 << b) <= (int64_t)n) ++b;
  return b;
}

__global__ void k_cluster_init(int n, int* __restrict__ parent, uint32_t* __restrict__ size, int* __restrict__ val) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  parent[j] = (int)j;
  size[j] = 0u;
  val[j] = (int)j;
}

// root[j] = the root of j's set (cluster_find: path halving, every write an ancestor of its node), size[root]++
__global__ void k_cluster_compress(int n, int* __restrict__ parent, int32_t* __restrict__ root, uint32_t* __restrict__ size) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int r = cluster_find(parent, (int)j);
  root[j] = r;
  atomicAdd(&size[r], 1u);
}

__global__ void k_cluster_flags(int n, const int32_t* __restrict__ root, int min_size, int max_size,
                                uint32_t* __restrict__ key, int64_t* __restrict__ n_clusters) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint32_t s = key[j];
  const bool cluster = root[j] == (int32_t)j && s >= (uint32_t)min_size && s <= (uint32_t)max_size;
  key[j] = cluster ? s : 0u;
  if (cluster) atomicAdd(reinterpret_cast<unsigned long long*>(n_clusters), 1ull);
}

// offsets[c] = the size of the c-th cluster in order (0 past the last), c in [0, n]: the input of the exclusive scan
__global__ void k_cluster_sizes(int n, const uint32_t* __restrict__ sorted_key, int64_t* __restrict__ offsets) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c > n) return;
  offsets[c] = c < n ? (int64_t)sorted_key[c] : 0;
}

__global__ void k_cluster_rank(int n, const uint32_t* __restrict__ sorted_key, const int* __restrict__ sorted_root,
                               int32_t* __restrict__ rank) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n || sorted_key[c] == 0u) return;
  rank[sorted_root[c]] = (int32_t)c;
}

// labels[j]; member_key[j] = the label, n when there is none (after every rank); val[j] = j again
__global__ void k_cluster_labels(int n, const int32_t* __restrict__ root, const int32_t* __restrict__ rank,
                                 int32_t* __restrict__ labels, uint32_t* __restrict__ member_key, int* __restrict__ val) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int32_t l = rank[root[j]];
  labels[j] = l;
  if (member_key != nullptr) {
    member_key[j] = l >= 0 ? (uint32_t)l : (uint32_t)n;
    val[j] = (int)j;
  }
}

int need_p(s4g_ctx* ctx, const char* who) {
  if (ctx->nP <= 0) {
    ctx->err = std::string(who) + ": call s4g_set_cloud_p first";
    return S4G_ERR_STATE;
  }
  return S4G_OK;
}

int cluster_args(s4g_ctx* ctx, const char* who, float sq_radius, int min_size, int max_size, const void* labels,
                 const void* n_clusters) {
  if (std::isnan(sq_radius) || min_size < 1 || max_size < min_size || labels == nullptr || n_clusters == nullptr) {
    ctx->err = std::string(who) + ": bad arguments (sq_radius not NaN, 1 <= min_size <= max_size, labels and n_clusters "
                                  "!= NULL)";
    return S4G_ERR_ARG;
  }
  return need_p(ctx, who);
}

// a stable radix sort of n (key, value) pairs over the low `bits` key bits; the result is in keys / vals .Current()
template <bool kDescending>
int sort_pairs(s4g_ctx* ctx, cub::DoubleBuffer<uint32_t>& keys, cub::DoubleBuffer<int>& vals, int n, int bits) {
  size_t bytes = 0;
  if (kDescending)
    S4G_CUDA(cub::DeviceRadixSort::SortPairsDescending(nullptr, bytes, keys, vals, n, 0, bits, ctx->stream));
  else
    S4G_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, bytes, keys, vals, n, 0, bits, ctx->stream));
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, bytes));
  if (kDescending)
    S4G_CUDA(cub::DeviceRadixSort::SortPairsDescending(ctx->dCub.p, bytes, keys, vals, n, 0, bits, ctx->stream));
  else
    S4G_CUDA(cub::DeviceRadixSort::SortPairs(ctx->dCub.p, bytes, keys, vals, n, 0, bits, ctx->stream));
  ctx->launches++;
  return S4G_OK;
}

// enqueue the whole chain.  Scratch A: parent (then rank), root when d_root is NULL, two key and two value buffers (24
// bytes per point); dCub the sorts' and the scan's temporary storage.
int launch_clusters(s4g_ctx* ctx, float sq_radius, int min_size, int max_size, int32_t* d_labels, int32_t* d_root,
                    int64_t* d_n_clusters, int64_t* d_offsets, int32_t* d_members) {
  S4G_CUDA(cudaSetDevice(ctx->device));
  const int n = ctx->nP;
  const size_t nn = (size_t)n;
  cudaStream_t st = ctx->stream;
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, 6 * nn * sizeof(int32_t)));
  int* parent = ctx->dScratchA.as<int>();
  int32_t* root = d_root != nullptr ? d_root : parent + nn;
  uint32_t* key0 = reinterpret_cast<uint32_t*>(parent + 2 * nn);
  uint32_t* key1 = key0 + nn;
  int* val0 = parent + 4 * nn;
  int* val1 = val0 + nn;
  const int bits = key_bits(n);
  S4G_CUDA(cudaMemsetAsync(d_n_clusters, 0, sizeof(int64_t), st));
  k_cluster_init<<<nblk(n, kClusterThreads), kClusterThreads, 0, st>>>(n, parent, key0, val0);
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  S4G_TRY(s4g_launch_cluster_link(ctx, sq_radius, parent));
  k_cluster_compress<<<nblk(n, kClusterThreads), kClusterThreads, 0, st>>>(n, parent, root, key0);
  k_cluster_flags<<<nblk(n, kClusterThreads), kClusterThreads, 0, st>>>(n, root, min_size, max_size, key0, d_n_clusters);
  ctx->launches += 2;
  S4G_CUDA(cudaGetLastError());
  cub::DoubleBuffer<uint32_t> keys(key0, key1);
  cub::DoubleBuffer<int> vals(val0, val1);
  S4G_TRY(sort_pairs<true>(ctx, keys, vals, n, bits));
  if (d_offsets != nullptr) {
    k_cluster_sizes<<<nblk(nn + 1, kClusterThreads), kClusterThreads, 0, st>>>(n, keys.Current(), d_offsets);
    ctx->launches++;
    S4G_CUDA(cudaGetLastError());
    size_t bytes = 0;
    S4G_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, bytes, d_offsets, d_offsets, (long long)n + 1, st));
    S4G_TRY(s4g_reserve(ctx, ctx->dCub, bytes));
    S4G_CUDA(cub::DeviceScan::ExclusiveSum(ctx->dCub.p, bytes, d_offsets, d_offsets, (long long)n + 1, st));
    ctx->launches++;
  }
  int32_t* rank = parent;   // the links are consumed: parent's storage holds the ranks
  S4G_CUDA(cudaMemsetAsync(rank, 0xff, nn * sizeof(int32_t), st));
  k_cluster_rank<<<nblk(n, kClusterThreads), kClusterThreads, 0, st>>>(n, keys.Current(), vals.Current(), rank);
  // the sorted keys and values are consumed by the rank: the member sort reuses both pairs of buffers
  k_cluster_labels<<<nblk(n, kClusterThreads), kClusterThreads, 0, st>>>(n, root, rank, d_labels,
                                                                        d_members != nullptr ? key0 : nullptr, val0);
  ctx->launches += 2;
  S4G_CUDA(cudaGetLastError());
  if (d_members != nullptr) {
    cub::DoubleBuffer<uint32_t> mkeys(key0, key1);
    cub::DoubleBuffer<int> mvals(val0, val1);
    S4G_TRY(sort_pairs<false>(ctx, mkeys, mvals, n, bits));
    S4G_CUDA(cudaMemcpyAsync(d_members, mvals.Current(), nn * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  }
  return S4G_OK;
}

}  // namespace

extern "C" int s4g_euclidean_clusters_dev(s4g_ctx* ctx, float sq_radius, int min_size, int max_size, int32_t* d_labels,
                                          int32_t* d_root, int64_t* d_n_clusters, int64_t* d_offsets, int32_t* d_members) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(cluster_args(ctx, "s4g_euclidean_clusters_dev", sq_radius, min_size, max_size, d_labels, d_n_clusters));
  return launch_clusters(ctx, sq_radius, min_size, max_size, d_labels, d_root, d_n_clusters, d_offsets, d_members);
}

// the device outputs staged in ctx->dFilter: int64 [n_clusters | offsets (n + 1)], then int32 [labels | root | members]
// (n each); then n_clusters back first, and only the defined part of offsets and members
extern "C" int s4g_euclidean_clusters(s4g_ctx* ctx, float sq_radius, int min_size, int max_size, int32_t* labels,
                                      int32_t* root, int64_t* n_clusters, int64_t* offsets, int32_t* members) {
  if (!ctx) return S4G_ERR_ARG;
  S4G_TRY(cluster_args(ctx, "s4g_euclidean_clusters", sq_radius, min_size, max_size, labels, n_clusters));
  S4G_CUDA(cudaSetDevice(ctx->device));
  const size_t n = (size_t)ctx->nP;
  S4G_TRY(s4g_reserve(ctx, ctx->dFilter, (n + 2) * sizeof(int64_t) + 3 * n * sizeof(int32_t)));
  int64_t* d_nc = ctx->dFilter.as<int64_t>();
  int64_t* d_off = d_nc + 1;
  int32_t* d_labels = reinterpret_cast<int32_t*>(d_off + n + 1);
  int32_t* d_root = d_labels + n;
  int32_t* d_members = d_root + n;
  const bool need_off = offsets != nullptr || members != nullptr;   // the members' total is offsets[n_clusters]
  S4G_TRY(launch_clusters(ctx, sq_radius, min_size, max_size, d_labels, root != nullptr ? d_root : nullptr, d_nc,
                          need_off ? d_off : nullptr, members != nullptr ? d_members : nullptr));
  cudaStream_t st = ctx->stream;
  int64_t nc = 0, total = 0;
  S4G_CUDA(cudaMemcpyAsync(&nc, d_nc, sizeof nc, cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaMemcpyAsync(labels, d_labels, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (root != nullptr) S4G_CUDA(cudaMemcpyAsync(root, d_root, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  *n_clusters = nc;
  if (need_off) {
    S4G_CUDA(cudaMemcpyAsync(&total, d_off + nc, sizeof total, cudaMemcpyDeviceToHost, st));
    if (offsets != nullptr)
      S4G_CUDA(cudaMemcpyAsync(offsets, d_off, ((size_t)nc + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    S4G_CUDA(cudaStreamSynchronize(st));
  }
  if (members != nullptr && total > 0) {
    S4G_CUDA(cudaMemcpyAsync(members, d_members, (size_t)total * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    S4G_CUDA(cudaStreamSynchronize(st));
  }
  return S4G_OK;
}
