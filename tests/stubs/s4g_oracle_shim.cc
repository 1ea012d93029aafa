// TEST INFRASTRUCTURE ONLY -- never built into, linked by or shipped with the product.
//
// A stand-in for libs4g.so whose stage entry points are answered by the CPU oracle
// (oracle/port.cc).  It exists so that the HOST logic of the header-compatible C++ layer
// (cpp/*.cc, include/super4pcs/**: sampling, centring, RNG order, base selection, the RANSAC
// loop, speculative multi-base execution, visitor protocol, global transform) can be exercised
// by the `-m "not gpu"` tests in a container without a GPU: tests/test_host_logic_cpu.py runs a
// subprocess with LD_PRELOAD=<this library>, so the s4g_* symbols of the C++ layer resolve here
// instead of to the CUDA library.  The point-cloud utilities (nearest, k-nearest and range queries,
// normals, outliers, clusters, planes, voxel grid, FPFH) are answered by their restatements
// (oracle/<name>_port.cc), compiled into this library, for the tests of the C++ layer's Utils.
// The product itself has no CPU path: libs4g.so fails with S4G_ERR_CUDA when there is no device
// (tests/test_abi.py::test_no_cpu_fallback).
#include <atomic>
#include <cmath>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "s4g.h"

extern "C" {
void* port_create(const float* Pxyz, int nP, const float* Qxyz, const float* Qnrm, const float* Qrgb, int nQ,
                  float delta);
void port_destroy(void* h);
void port_get_normalization(void* h, float* out5);
double port_verify_batch(void* h, const float* T16k, long K, float best_lcp, int nthreads, float* out_lcp,
                         uint32_t* out_good);
void port_rigid_batch(void* h, const int* base_ids4, const int* quads4k, long K, float max_angle_deg, float* out_T,
                      float* out_rms, int* out_ok);
long port_extract_pairs(void* h, float pair_distance, float pair_normals_angle, float eps, const float* base_p1,
                        const float* base_p2, const float* filters4);
long port_extract_pairs_ordered(void* h, float pair_distance, float pair_normals_angle, float eps, const float* base_p1,
                                const float* base_p2, const float* filters4);
void port_get_pairs(void* h, int32_t* out);
long port_find_quads(void* h, float invariant1, float invariant2, float distance_threshold2, const float* base_xyz,
                     const int32_t* pairs1, long n1, const int32_t* pairs2, long n2);
void port_get_quads(void* h, int32_t* out);

// the restatements of the point-cloud utilities, oracle/<name>_port.cc
void nearest_bruteforce(const float* P, long nP, const float* Q, long nQ, float delta, const float* T16k, long K,
                        int32_t* out_index, float* out_sq, uint32_t* out_counts);
void nearest_any_bruteforce(const float* P, long nP, const float* X, long n, const float* T, float sq_radius,
                            const int32_t* exclude, int32_t* out_index, float* out_sq);
void knn_bruteforce(const float* P, long nP, const float* X, long n, const float* T, int k, float sq_radius,
                    const int32_t* exclude, int32_t* out_index, float* out_sq);
void range_bruteforce_count(const float* P, long nP, const float* X, long n, const float* T, float sq_radius,
                            int64_t* offsets);
void range_bruteforce_fill(const float* P, long nP, const float* X, long n, const float* T, float sq_radius,
                           const int64_t* offsets, int32_t* out_index, float* out_sq);
void normals_port(const float* P, long nP, const int64_t* which, long n, int k, float sq_radius, const float* viewpoint,
                  float* normals, float* eig, int32_t* rows_out);
int orient_normals_port(const float* P, long n, const float* normals, int k, float sq_radius, const float* viewpoint,
                        const int32_t* rows_in, float* normals_out, int32_t* root, int64_t* out2, int32_t* tree_edges);
void statistical_port(const float* P, long nP, int k, double std_ratio, uint8_t* flags, double* mean_dist,
                      double* out2);
void radius_port(const float* P, long nP, float sq_radius, int min_neighbors, int64_t* raw, int32_t* counts,
                 uint8_t* flags);
void clusters_port(const float* P, long n, float sq_radius, int min_size, int max_size, int32_t* labels, int32_t* root,
                   int64_t* n_clusters, int64_t* offsets, int32_t* members);
void planes_port(const float* P, long n, float threshold, int H, uint64_t seed, int refine, int max_planes,
                 int64_t min_inliers, int32_t* labels, void* planes, int* n_planes, int64_t* offsets, int32_t* members,
                 uint32_t* hyp_counts);
int voxel_grid_port(const float* xyz, const float* normals, const float* rgb, long n, float leaf, int min_points,
                    float* xyz_out, float* normals_out, float* rgb_out, int32_t* counts, int32_t* first,
                    int32_t* voxel_of, int64_t* n_out);
int fpfh_port(const float* P, long n, const float* normals, int k, float sq_radius, const int32_t* rows_in,
              const float* sq_in, float* fpfh, double* spfh_out);
void fpfh_match_port(const float* a, long na, const float* b, long nb, int mutual, int32_t* index, float* sq_dist);
}

// stand-in for the communicator of csrc/comm.cu: the shard threads of one base meet here and leave with the global record
struct ShimComm {
  std::mutex m;
  std::condition_variable cv;
  int n = 0, arrived = 0;
  long generation = 0;
  std::vector<s4g_tcs_result> slot;
  s4g_tcs_result merged;
};

struct s4g_ctx {
  std::shared_ptr<ShimComm> comm;
  int comm_rank = 0;
  int ordinal = 0;  // n-th context of the process (S4G_SHIM_FAIL_QUADS_ON_CONTEXT)
  void* port = nullptr;
  std::vector<float> P, Q, Qn, Qrgb;
  bool has_n = false, has_rgb = false;
  float delta = 0;
  std::vector<int32_t> pairs[2], quads;
  bool has_range = false;  // the lists of the last s4g_range, for s4g_get_range
  std::vector<int32_t> range_index;
  std::vector<float> range_sq;
  std::string err;
};

namespace {

// S4G_SHIM_STATS=1: report at exit how many contexts were created and the largest number of stage
// calls that were in flight at once (proof that the lanes of row f1 really ran concurrently)
std::atomic<int> g_created{0}, g_inflight{0}, g_max_inflight{0};
std::atomic<int> g_max_device{0}, g_sharded_calls{0}, g_collectives{0};  // S4PCS_DEVICES: largest ordinal asked for, tcs calls with world > 1
struct InFlight {
  InFlight() {
    const int now = ++g_inflight;
    int seen = g_max_inflight.load();
    while (now > seen && !g_max_inflight.compare_exchange_weak(seen, now)) {}
  }
  ~InFlight() { --g_inflight; }
};
struct Report {
  ~Report() {
    if (std::getenv("S4G_SHIM_STATS"))
      std::fprintf(stderr, "SHIM contexts=%d max_inflight=%d max_device=%d sharded_calls=%d collectives=%d\n", g_created.load(),
                   g_max_inflight.load(), g_max_device.load(), g_sharded_calls.load(), g_collectives.load());
  }
} g_report;

int fail(s4g_ctx* c, int code, const char* msg) {
  c->err = msg;
  return code;
}

int ready(s4g_ctx* c) {
  if (c->P.empty() || c->Q.empty())
    return fail(c, S4G_ERR_STATE, "shim: call s4g_set_cloud_p and s4g_set_cloud_q first");
  if (c->port == nullptr)
    c->port = port_create(c->P.data(), int(c->P.size() / 3), c->Q.data(), c->has_n ? c->Qn.data() : nullptr,
                          c->has_rgb ? c->Qrgb.data() : nullptr, int(c->Q.size() / 3), c->delta);
  return S4G_OK;
}

// the point-cloud utilities need only the P cloud
int need_p(s4g_ctx* c) { return c->P.empty() ? fail(c, S4G_ERR_STATE, "shim: call s4g_set_cloud_p first") : S4G_OK; }

long n_p(const s4g_ctx* c) { return long(c->P.size() / 3); }

// the flagged j, ascending
void compact(const std::vector<uint8_t>& flags, int32_t* keep, int64_t* n_kept) {
  int64_t m = 0;
  for (std::size_t j = 0; j < flags.size(); ++j)
    if (flags[j]) keep[m++] = int32_t(j);
  *n_kept = m;
}

void drop_port(s4g_ctx* c) {
  if (c->port) port_destroy(c->port);
  c->port = nullptr;
}

// what csrc/comm.cu does with two allreduces: the record of the shard with the largest key (rank 0's when nothing was
// verified anywhere) and the sum of the gate counts, on every rank
int reduce_shards(s4g_ctx* c, int shard_rank, int shard_world, s4g_tcs_result* out) {
  ShimComm& k = *c->comm;
  if (shard_world != k.n || shard_rank != c->comm_rank) return fail(c, S4G_ERR_ARG, "shim: shard differs from the communicator");
  std::unique_lock<std::mutex> lock(k.m);
  k.slot[size_t(shard_rank)] = *out;
  const long my_generation = k.generation;
  if (++k.arrived == k.n) {
    size_t win = 0;
    uint32_t gate = 0;
    for (size_t r = 0; r < k.slot.size(); ++r) {
      gate += k.slot[r].n_gate_pass;
      if (k.slot[r].key > k.slot[win].key) win = r;
    }
    k.merged = k.slot[win];
    k.merged.n_gate_pass = gate;
    k.arrived = 0;
    ++k.generation;
    g_collectives += 2;
    k.cv.notify_all();
  } else {
    k.cv.wait(lock, [&] { return k.generation != my_generation; });
  }
  *out = k.merged;
  return S4G_OK;
}

int tcs_local(s4g_ctx* c, const float* base_xyz, const int32_t* quads, int64_t K, float max_angle_deg, int shard_rank,
              int shard_world, s4g_tcs_result* out);

int tcs(s4g_ctx* c, const float* base_xyz, const int32_t* quads, int64_t K, float max_angle_deg, int shard_rank,
        int shard_world, s4g_tcs_result* out) {
  if (int rc = tcs_local(c, base_xyz, quads, K, max_angle_deg, shard_rank, shard_world, out)) return rc;
  return c->comm && shard_world > 1 ? reduce_shards(c, shard_rank, shard_world, out) : S4G_OK;
}

int tcs_local(s4g_ctx* c, const float* base_xyz, const int32_t* quads, int64_t K, float max_angle_deg, int shard_rank,
              int shard_world, s4g_tcs_result* out) {
  if (shard_world < 1 || shard_rank < 0 || shard_rank >= shard_world) return fail(c, S4G_ERR_ARG, "shim: bad shard");
  if (shard_world > 1) ++g_sharded_calls;
  std::memset(out, 0, sizeof *out);
  out->best_index = -1;
  out->n_q = uint32_t(c->Q.size() / 3);
  int ids[4];
  const int nP = int(c->P.size() / 3);
  for (int k = 0; k < 4; ++k) {  // the port addresses the base by index into sampled P
    ids[k] = -1;
    for (int i = 0; i < nP && ids[k] < 0; ++i)
      if (c->P[3 * i] == base_xyz[3 * k] && c->P[3 * i + 1] == base_xyz[3 * k + 1] && c->P[3 * i + 2] == base_xyz[3 * k + 2])
        ids[k] = i;
    if (ids[k] < 0) return fail(c, S4G_ERR_ARG, "shim: base point is not a point of sampled P");
  }
  for (int k = 0; k < 3; ++k)  // (b1 + b2 + b3) / 3, match4pcsBase.hpp:385
    out->centroid1[k] = ((base_xyz[k] + base_xyz[3 + k]) + base_xyz[6 + k]) / 3.f;
  if (K <= 0) return S4G_OK;
  // rigid fit of every quad, gate (ok && 0 <= rms < 2 delta), full Verify of the survivors, first maximum -- what the
  // device does.  (port_try_congruent_set is not used: like the reference it needs a running best_LCP >= 0 and then
  // reports nothing for sets whose candidates all score 0, whereas the device reports the first gate-passing quad.)
  std::vector<float> T(size_t(K) * 16), rms(static_cast<size_t>(K), 0.f);
  std::vector<int> ok(static_cast<size_t>(K), 0);
  port_rigid_batch(c->port, ids, quads, long(K), max_angle_deg, T.data(), rms.data(), ok.data());
  long best = -1;
  uint32_t good = 0;
  for (int64_t i = 0; i < K; ++i) {
    if (i % shard_world != shard_rank) continue;  // candidate-set sharding, as in csrc/rigid.cu
    if (!ok[size_t(i)] || !(rms[size_t(i)] >= 0.f) || !(rms[size_t(i)] < 2.0f * c->delta)) continue;
    out->n_gate_pass++;
    float lcp = 0;
    uint32_t g = 0;
    port_verify_batch(c->port, &T[size_t(i) * 16], 1, 0.f, 1, &lcp, &g);
    if (best < 0 || g > good) {
      best = long(i);
      good = g;
    }
  }
  if (best < 0) return S4G_OK;
  std::memcpy(out->best_T, &T[size_t(best) * 16], 16 * sizeof(float));
  out->best_rms = rms[size_t(best)];
  out->best_count = good;
  out->best_index = int32_t(best);
  out->key = (uint64_t(good) << 32) | uint64_t(0xFFFFFFFFu - uint32_t(best));
  for (int v = 0; v < 4; ++v) out->best_quad[v] = quads[4 * best + v];
  const float* q0 = &c->Q[3 * size_t(out->best_quad[0])];
  const float* q1 = &c->Q[3 * size_t(out->best_quad[1])];
  const float* q2 = &c->Q[3 * size_t(out->best_quad[2])];
  for (int k = 0; k < 3; ++k) out->centroid2[k] = ((q0[k] + q1[k]) + q2[k]) / 3.f;  // hpp:415-417
  return S4G_OK;
}

}  // namespace

extern "C" {

int s4g_abi_version(void) { return 1; }

int s4g_device_count(int* out_count) {  // S4G_SHIM_DEVICE_COUNT pretends to be a box with that many GPUs (default 1)
  if (!out_count) return S4G_ERR_ARG;
  const char* e = std::getenv("S4G_SHIM_DEVICE_COUNT");
  *out_count = e ? std::atoi(e) : 1;
  return *out_count > 0 ? S4G_OK : S4G_ERR_CUDA;
}

int s4g_create(int device, s4g_ctx** out_ctx) {
  if (!out_ctx) return S4G_ERR_ARG;
  int seen = g_max_device.load();
  while (device > seen && !g_max_device.compare_exchange_weak(seen, device)) {}
  *out_ctx = new s4g_ctx;
  (*out_ctx)->ordinal = g_created++;
  return S4G_OK;
}

void s4g_destroy(s4g_ctx* c) {
  if (!c) return;
  drop_port(c);
  delete c;
}

const char* s4g_error_string(const s4g_ctx* c) { return c ? c->err.c_str() : "null context"; }

int s4g_set_cloud_p(s4g_ctx* c, const float* xyz, int n, float delta) {
  if (!c) return S4G_ERR_ARG;
  if (!xyz || n <= 0 || !(delta > 0)) return fail(c, S4G_ERR_ARG, "shim: s4g_set_cloud_p: bad arguments (delta must be > 0)");
  c->P.assign(xyz, xyz + 3 * size_t(n));
  c->delta = delta;
  drop_port(c);
  return S4G_OK;
}

int s4g_set_cloud_q(s4g_ctx* c, const float* xyz, const float* normals, const float* rgb, int n) {
  if (!c) return S4G_ERR_ARG;
  if (!xyz || n <= 0) return fail(c, S4G_ERR_ARG, "shim: s4g_set_cloud_q: bad arguments");
  c->Q.assign(xyz, xyz + 3 * size_t(n));
  c->has_n = normals != nullptr;
  c->has_rgb = rgb != nullptr;
  if (normals) c->Qn.assign(normals, normals + 3 * size_t(n));
  if (rgb) c->Qrgb.assign(rgb, rgb + 3 * size_t(n));
  drop_port(c);
  return S4G_OK;
}

int s4g_get_q_normalization(s4g_ctx* c, float* out5) {
  if (!c || !out5) return S4G_ERR_ARG;
  if (int rc = ready(c)) return rc;
  port_get_normalization(c->port, out5);
  return S4G_OK;
}

int s4g_rigid_batch(s4g_ctx* c, const float* base_xyz, const int32_t* quads, int64_t K, float max_angle_deg, float* out_T,
                    float* out_rms, int32_t* out_ok) {
  if (!c || !base_xyz || K < 0 || (K > 0 && !quads)) return S4G_ERR_ARG;
  if (int rc = ready(c)) return rc;
  if (K == 0) return S4G_OK;
  int ids[4];
  const int nP = int(c->P.size() / 3);
  for (int k = 0; k < 4; ++k) {
    ids[k] = -1;
    for (int i = 0; i < nP && ids[k] < 0; ++i)
      if (c->P[3 * i] == base_xyz[3 * k] && c->P[3 * i + 1] == base_xyz[3 * k + 1] && c->P[3 * i + 2] == base_xyz[3 * k + 2]) ids[k] = i;
    if (ids[k] < 0) return fail(c, S4G_ERR_ARG, "shim: base point is not a point of sampled P");
  }
  std::vector<float> T(size_t(K) * 16), rms(static_cast<size_t>(K), 0.f);
  std::vector<int> ok(static_cast<size_t>(K), 0);
  port_rigid_batch(c->port, ids, quads, long(K), max_angle_deg, T.data(), rms.data(), ok.data());
  if (out_T) std::memcpy(out_T, T.data(), T.size() * sizeof(float));
  if (out_rms) std::memcpy(out_rms, rms.data(), rms.size() * sizeof(float));
  if (out_ok) std::memcpy(out_ok, ok.data(), ok.size() * sizeof(int));
  return S4G_OK;
}

int s4g_verify(s4g_ctx* c, const float* T, int K, uint32_t* counts) {
  if (!c) return S4G_ERR_ARG;
  if (int rc = ready(c)) return rc;
  if (K <= 0) return S4G_OK;
  std::vector<float> lcp(static_cast<size_t>(K), 0.f);
  port_verify_batch(c->port, T, K, 0.f, 1, lcp.data(), counts);
  return S4G_OK;
}

int s4g_extract_pairs(s4g_ctx* c, float pair_distance, float pair_normals_angle, float eps, const float* base_p1,
                      const float* base_p2, const s4g_pair_filters* f, int slot, int64_t* n_pairs) {
  if (!c) return S4G_ERR_ARG;
  if (slot < 0 || slot > 1 || !base_p1 || !base_p2 || !n_pairs) return fail(c, S4G_ERR_ARG, "shim: s4g_extract_pairs: bad arguments");
  if (int rc = ready(c)) return rc;
  InFlight guard;
  const float f4[4] = {f ? f->max_normal_difference : -1.f, f ? f->max_translation_distance : -1.f,
                       f ? f->max_angle : -1.f, f ? f->max_color_distance : -1.f};
  // S4G_SHIM_REFERENCE_ORDER=1: hand the pairs over in the reference's emission order instead of sorted (the product's
  // order), so that the candidate order -- and with it the winner among candidates with equal inlier counts -- is the
  // reference's.  Used to show that this order is the ONLY source of the rare final-result differences (DESIGN.md 4).
  static const bool reference_order = std::getenv("S4G_SHIM_REFERENCE_ORDER") != nullptr;
  const long n = reference_order
                     ? port_extract_pairs_ordered(c->port, pair_distance, pair_normals_angle, eps, base_p1, base_p2, f4)
                     : port_extract_pairs(c->port, pair_distance, pair_normals_angle, eps, base_p1, base_p2, f4);
  c->pairs[slot].resize(size_t(2 * n));
  if (n > 0) port_get_pairs(c->port, c->pairs[slot].data());
  *n_pairs = n;
  return S4G_OK;
}

int s4g_get_pairs(s4g_ctx* c, int slot, int32_t* out) {
  if (!c || slot < 0 || slot > 1) return S4G_ERR_ARG;
  if (!c->pairs[slot].empty()) std::memcpy(out, c->pairs[slot].data(), c->pairs[slot].size() * sizeof(int32_t));
  return S4G_OK;
}

int s4g_set_pairs(s4g_ctx* c, int slot, const int32_t* pairs, int64_t n) {
  if (!c || slot < 0 || slot > 1 || n < 0) return S4G_ERR_ARG;
  c->pairs[slot].assign(pairs, pairs + 2 * n);
  return S4G_OK;
}

int s4g_find_quads(s4g_ctx* c, float invariant1, float invariant2, float distance_threshold2, const float* base_xyz,
                   int64_t* n_quads) {
  if (!c || !base_xyz || !n_quads) return S4G_ERR_ARG;
  if (int rc = ready(c)) return rc;
  if (const char* e = std::getenv("S4G_SHIM_FAIL_QUADS_ON_CONTEXT"))  // one shard failing before the reduction
    if (std::atoi(e) == c->ordinal) return fail(c, S4G_ERR_CUDA, "shim: injected failure of this context");
  const long n = port_find_quads(c->port, invariant1, invariant2, distance_threshold2, base_xyz, c->pairs[0].data(),
                                 long(c->pairs[0].size() / 2), c->pairs[1].data(), long(c->pairs[1].size() / 2));
  c->quads.resize(size_t(4 * n));
  if (n > 0) port_get_quads(c->port, c->quads.data());
  *n_quads = n;
  return S4G_OK;
}

int s4g_get_quads(s4g_ctx* c, int32_t* out) {
  if (!c) return S4G_ERR_ARG;
  if (!c->quads.empty()) std::memcpy(out, c->quads.data(), c->quads.size() * sizeof(int32_t));
  return S4G_OK;
}

int s4g_try_congruent_set(s4g_ctx* c, const float* base_xyz, const int32_t* quads, int64_t K, float max_angle_deg,
                          float /*rms_threshold = 2 delta inside the port*/, int shard_rank, int shard_world,
                          s4g_tcs_result* out) {
  if (!c || !base_xyz || !out || K < 0) return S4G_ERR_ARG;
  if (int rc = ready(c)) return rc;
  return tcs(c, base_xyz, quads, K, max_angle_deg, shard_rank, shard_world, out);
}

int s4g_try_congruent_set_resident(s4g_ctx* c, const float* base_xyz, float max_angle_deg, float, int shard_rank,
                                   int shard_world, s4g_tcs_result* out) {
  if (!c || !base_xyz || !out) return S4G_ERR_ARG;
  if (int rc = ready(c)) return rc;
  return tcs(c, base_xyz, c->quads.data(), int64_t(c->quads.size() / 4), max_angle_deg, shard_rank, shard_world, out);
}

// f1: the per-base chain for every base of the batch, on private lists (the resident slots stay untouched)
int s4g_try_bases(s4g_ctx* c, const s4g_base_desc* bases, int n_bases, float eps, const s4g_pair_filters* f,
                  float distance_threshold2, float max_angle_deg, float rms_threshold, s4g_base_result* out) {
  if (!c || !bases || !out || n_bases < 1 || n_bases > 64) return S4G_ERR_ARG;
  if (int rc = ready(c)) return rc;
  const std::vector<int32_t> keep0 = c->pairs[0], keep1 = c->pairs[1], keepq = c->quads;
  int rc = S4G_OK;
  for (int b = 0; b < n_bases && rc == S4G_OK; ++b) {
    const s4g_base_desc& d = bases[b];
    std::memset(&out[b], 0, sizeof out[b]);
    out[b].tcs.best_index = -1;
    out[b].tcs.n_q = uint32_t(c->Q.size() / 3);
    for (int k = 0; k < 3; ++k) out[b].tcs.centroid1[k] = ((d.base_xyz_p[k] + d.base_xyz_p[3 + k]) + d.base_xyz_p[6 + k]) / 3.f;
    for (int i = 0; i < 16; ++i) out[b].tcs.best_T[i] = (i % 5 == 0) ? 1.f : 0.f;
    out[b].tcs.best_rms = -1.f;
    for (int s = 0; s < 2 && rc == S4G_OK; ++s)
      rc = s4g_extract_pairs(c, d.pair_distance[s], d.pair_normals_angle[s], eps, d.base_p[2 * s], d.base_p[2 * s + 1], f, s,
                             &out[b].n_pairs[s]);
    if (rc != S4G_OK || out[b].n_pairs[0] == 0 || out[b].n_pairs[1] == 0) continue;
    float bx[12];
    for (int k = 0; k < 4; ++k)
      for (int cc = 0; cc < 3; ++cc) bx[3 * k + cc] = d.base_p[k][cc];
    rc = s4g_find_quads(c, d.invariant1, d.invariant2, distance_threshold2, bx, &out[b].n_quads);
    if (rc != S4G_OK || out[b].n_quads == 0) continue;
    rc = s4g_try_congruent_set_resident(c, d.base_xyz_p, max_angle_deg, rms_threshold, 0, 1, &out[b].tcs);
  }
  c->pairs[0] = keep0;
  c->pairs[1] = keep1;
  c->quads = keepq;
  return rc;
}

// row e inside the library: the in-process communicator has a stand-in (threads meet at a condition variable); there is
// no NCCL here, so the process-per-GPU form reports S4G_ERR_COMM like the product does when NCCL is missing
int s4g_comm_unique_id(unsigned char*) { return S4G_ERR_COMM; }
int s4g_comm_init_rank(s4g_ctx* c, const unsigned char*, int, int) {
  return c ? fail(c, S4G_ERR_COMM, "shim: no NCCL in the CPU stand-in") : S4G_ERR_ARG;
}
int s4g_comm_init_all(s4g_ctx** ctxs, int n) {
  if (!ctxs || n < 1) return S4G_ERR_ARG;
  if (std::getenv("S4G_SHIM_NO_NCCL")) return fail(ctxs[0], S4G_ERR_COMM, "shim: NCCL is not loadable (S4G_SHIM_NO_NCCL)");
  auto comm = std::make_shared<ShimComm>();
  comm->n = n;
  comm->slot.resize(size_t(n));
  for (int r = 0; r < n; ++r) {
    ctxs[r]->comm = comm;
    ctxs[r]->comm_rank = r;
  }
  return S4G_OK;
}
int s4g_comm_destroy(s4g_ctx* c) {
  if (!c) return S4G_ERR_ARG;
  c->comm.reset();
  return S4G_OK;
}
int s4g_comm_info(s4g_ctx* c, int* out4) {
  if (!c || !out4) return S4G_ERR_ARG;
  out4[0] = c->comm ? c->comm->n : 0;
  out4[1] = c->comm_rank;
  out4[2] = 0;
  out4[3] = g_collectives.load();
  return S4G_OK;
}
int s4g_comm_set_timeout(s4g_ctx* c, int) { return c ? S4G_OK : S4G_ERR_ARG; }

int s4g_get_timings(s4g_ctx* c, double* out5) {  // no device, no device time: every stage reports 1 ms per call made
  if (!c || !out5) return S4G_ERR_ARG;
  for (int k = 0; k < 5; ++k) out5[k] = 1.0;
  return S4G_OK;
}

int s4g_voxel_sample(s4g_ctx* c, const float*, int64_t, float, int32_t*, int64_t*) {
  return c ? fail(c, S4G_ERR_STATE, "shim: s4g_voxel_sample is not provided (inputs < 200K points stay on the host)") : S4G_ERR_ARG;
}

// ---- the point-cloud utilities, answered by their restatements

int s4g_verify_nearest(s4g_ctx* c, const float* T, int K, int32_t* index, float* sq_dist, uint32_t* counts) {
  if (!c) return S4G_ERR_ARG;
  if (K < 0 || (K > 0 && (!T || !index))) return fail(c, S4G_ERR_ARG, "shim: s4g_verify_nearest: bad arguments");
  if (c->P.empty() || c->Q.empty())
    return fail(c, S4G_ERR_STATE, "shim: call s4g_set_cloud_p and s4g_set_cloud_q first");
  if (K > 0)
    nearest_bruteforce(c->P.data(), n_p(c), c->Q.data(), long(c->Q.size() / 3), c->delta, T, K, index, sq_dist, counts);
  return S4G_OK;
}

int s4g_nearest(s4g_ctx* c, const float* xyz, int n, const float* T, float sq_radius, const int32_t* exclude,
                int32_t* index, float* sq_dist) {
  if (!c) return S4G_ERR_ARG;
  if (n < 0 || (n > 0 && (!xyz || !index)) || std::isnan(sq_radius))
    return fail(c, S4G_ERR_ARG, "shim: s4g_nearest: bad arguments");
  if (int rc = need_p(c)) return rc;
  if (n > 0) nearest_any_bruteforce(c->P.data(), n_p(c), xyz, n, T, sq_radius, exclude, index, sq_dist);
  return S4G_OK;
}

int s4g_knn(s4g_ctx* c, const float* xyz, int n, const float* T, int k, float sq_radius, const int32_t* exclude,
            int32_t* index, float* sq_dist) {
  if (!c) return S4G_ERR_ARG;
  if (n < 0 || (n > 0 && (!xyz || !index)) || k < 1 || k > 64 || std::isnan(sq_radius))
    return fail(c, S4G_ERR_ARG, "shim: s4g_knn: bad arguments");
  if (int rc = need_p(c)) return rc;
  knn_bruteforce(c->P.data(), n_p(c), xyz, n, T, k, sq_radius, exclude, index, sq_dist);
  return S4G_OK;
}

int s4g_range(s4g_ctx* c, const float* xyz, int n, const float* T, float sq_radius, int64_t* offsets, int64_t* total) {
  if (!c) return S4G_ERR_ARG;
  if (n < 0 || (n > 0 && !xyz) || !offsets || !total || std::isnan(sq_radius))
    return fail(c, S4G_ERR_ARG, "shim: s4g_range: bad arguments");
  if (int rc = need_p(c)) return rc;
  range_bruteforce_count(c->P.data(), n_p(c), xyz, n, T, sq_radius, offsets);
  c->range_index.resize(size_t(offsets[n]));
  c->range_sq.resize(size_t(offsets[n]));
  range_bruteforce_fill(c->P.data(), n_p(c), xyz, n, T, sq_radius, offsets, c->range_index.data(), c->range_sq.data());
  c->has_range = true;
  *total = offsets[n];
  return S4G_OK;
}

int s4g_get_range(s4g_ctx* c, int32_t* indices, float* sq_dist) {
  if (!c) return S4G_ERR_ARG;
  if (!c->has_range) return fail(c, S4G_ERR_STATE, "shim: call s4g_range first");
  if (c->range_index.empty()) return S4G_OK;
  if (!indices) return fail(c, S4G_ERR_ARG, "shim: s4g_get_range: bad arguments");
  std::memcpy(indices, c->range_index.data(), c->range_index.size() * sizeof(int32_t));
  if (sq_dist) std::memcpy(sq_dist, c->range_sq.data(), c->range_sq.size() * sizeof(float));
  return S4G_OK;
}

int s4g_normals(s4g_ctx* c, int k, float sq_radius, const float* viewpoint, float* normals, float* eigenvalues) {
  if (!c) return S4G_ERR_ARG;
  if (k < 3 || k > 64 || std::isnan(sq_radius) || sq_radius < 0.f || !normals)
    return fail(c, S4G_ERR_ARG, "shim: s4g_normals: bad arguments");
  if (int rc = need_p(c)) return rc;
  normals_port(c->P.data(), n_p(c), nullptr, n_p(c), k, sq_radius, viewpoint, normals, eigenvalues, nullptr);
  return S4G_OK;
}

int s4g_orient_normals(s4g_ctx* c, const float* normals, int k, float sq_radius, const float* viewpoint,
                       float* normals_out, int32_t* root, int64_t* out2, int32_t* tree_edges) {
  if (!c) return S4G_ERR_ARG;
  if (int rc = need_p(c)) return rc;
  if (orient_normals_port(c->P.data(), n_p(c), normals, k, sq_radius, viewpoint, nullptr, normals_out, root, out2,
                          tree_edges) != 0)
    return fail(c, S4G_ERR_ARG, "shim: s4g_orient_normals: bad arguments");
  return S4G_OK;
}

int s4g_statistical_outliers(s4g_ctx* c, int k, double std_ratio, int32_t* keep, int64_t* n_kept, double* mean_dist,
                             double* out2) {
  if (!c) return S4G_ERR_ARG;
  if (k < 1 || k > 64 || !std::isfinite(std_ratio) || !keep || !n_kept)
    return fail(c, S4G_ERR_ARG, "shim: s4g_statistical_outliers: bad arguments");
  if (int rc = need_p(c)) return rc;
  const long n = n_p(c);
  std::vector<uint8_t> flags(static_cast<size_t>(n), 0);
  std::vector<double> mean(static_cast<size_t>(n));
  double o2[2];
  statistical_port(c->P.data(), n, k, std_ratio, flags.data(), mean.data(), o2);
  compact(flags, keep, n_kept);
  if (mean_dist) std::memcpy(mean_dist, mean.data(), mean.size() * sizeof(double));
  if (out2) out2[0] = o2[0], out2[1] = o2[1];
  return S4G_OK;
}

int s4g_radius_outliers(s4g_ctx* c, float sq_radius, int min_neighbors, int32_t* keep, int64_t* n_kept, int32_t* counts) {
  if (!c) return S4G_ERR_ARG;
  if (std::isnan(sq_radius) || min_neighbors < 1 || !keep || !n_kept)
    return fail(c, S4G_ERR_ARG, "shim: s4g_radius_outliers: bad arguments");
  if (int rc = need_p(c)) return rc;
  const long n = n_p(c);
  std::vector<uint8_t> flags(static_cast<size_t>(n), 0);
  std::vector<int32_t> cnt(static_cast<size_t>(n));
  radius_port(c->P.data(), n, sq_radius, min_neighbors, nullptr, cnt.data(), flags.data());
  compact(flags, keep, n_kept);
  if (counts) std::memcpy(counts, cnt.data(), cnt.size() * sizeof(int32_t));
  return S4G_OK;
}

int s4g_euclidean_clusters(s4g_ctx* c, float sq_radius, int min_size, int max_size, int32_t* labels, int32_t* root,
                           int64_t* n_clusters, int64_t* offsets, int32_t* members) {
  if (!c) return S4G_ERR_ARG;
  if (std::isnan(sq_radius) || min_size < 1 || max_size < min_size || !labels || !n_clusters)
    return fail(c, S4G_ERR_ARG, "shim: s4g_euclidean_clusters: bad arguments");
  if (int rc = need_p(c)) return rc;
  const long n = n_p(c);
  std::vector<int64_t> off(static_cast<size_t>(n) + 1);
  std::vector<int32_t> mem(static_cast<size_t>(n));
  clusters_port(c->P.data(), n, sq_radius, min_size, max_size, labels, root, n_clusters, off.data(), mem.data());
  if (offsets) std::memcpy(offsets, off.data(), size_t(*n_clusters + 1) * sizeof(int64_t));
  if (members) std::memcpy(members, mem.data(), size_t(off[size_t(*n_clusters)]) * sizeof(int32_t));
  return S4G_OK;
}

int s4g_segment_planes(s4g_ctx* c, float threshold, int n_hypotheses, uint64_t seed, int refine, int max_planes,
                       int64_t min_inliers, int32_t* labels, s4g_plane* planes, int* n_planes, int64_t* offsets,
                       int32_t* members, uint32_t* hyp_counts) {
  if (!c) return S4G_ERR_ARG;
  if (std::isnan(threshold) || threshold < 0.f || n_hypotheses < 1 || n_hypotheses > (1 << 20) || max_planes < 1 ||
      min_inliers < 1 || !labels || !planes || !n_planes)
    return fail(c, S4G_ERR_ARG, "shim: s4g_segment_planes: bad arguments");
  if (int rc = need_p(c)) return rc;
  const long n = n_p(c);
  std::vector<int64_t> off(static_cast<size_t>(max_planes) + 1);
  std::vector<int32_t> mem(static_cast<size_t>(n));
  planes_port(c->P.data(), n, threshold, n_hypotheses, seed, refine, max_planes, min_inliers, labels, planes, n_planes,
              off.data(), mem.data(), hyp_counts);
  if (offsets) std::memcpy(offsets, off.data(), size_t(*n_planes + 1) * sizeof(int64_t));
  if (members) std::memcpy(members, mem.data(), size_t(off[size_t(*n_planes)]) * sizeof(int32_t));
  return S4G_OK;
}

// needs no cloud: the points are arguments
int s4g_voxel_grid(s4g_ctx* c, const float* xyz, const float* normals, const float* rgb, int64_t n, float leaf,
                   int min_points, float* xyz_out, float* normals_out, float* rgb_out, int32_t* counts, int32_t* first,
                   int32_t* voxel_of, int64_t* n_out) {
  if (!c || !xyz || !xyz_out || !n_out) return S4G_ERR_ARG;
  return voxel_grid_port(xyz, normals, rgb, long(n), leaf, min_points, xyz_out, normals_out, rgb_out, counts, first,
                         voxel_of, n_out);
}

int s4g_fpfh(s4g_ctx* c, const float* normals, int k, float sq_radius, float* fpfh) {
  if (!c) return S4G_ERR_ARG;
  if (int rc = need_p(c)) return rc;
  if (fpfh_port(c->P.data(), n_p(c), normals, k, sq_radius, nullptr, nullptr, fpfh, nullptr) != 0)
    return fail(c, S4G_ERR_ARG, "shim: s4g_fpfh: bad arguments");
  return S4G_OK;
}

// needs no cloud: the descriptors are arguments
int s4g_fpfh_match(s4g_ctx* c, const float* a, int64_t n_a, const float* b, int64_t n_b, int mutual, int32_t* index,
                   float* sq_dist) {
  if (!c || n_a < 0 || n_b < 0 || (n_a > 0 && (!a || !index)) || (n_a > 0 && n_b > 0 && !b)) return S4G_ERR_ARG;
  if (n_a > 0) fpfh_match_port(a, long(n_a), b, long(n_b), mutual, index, sq_dist);
  return S4G_OK;
}

}  // extern "C"
