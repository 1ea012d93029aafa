/*
 * s4g.h -- C ABI of libs4g.so, the H100-native (sm_90a) implementation of the Super4PCS
 * congruent-set extraction + LCP verification hot path.
 *
 * The reference (nmellado/Super4PCS) has no FFI: its drop-in boundary is the C++ class
 * GlobalRegistration::Match4PCSBase / MatchSuper4PCS.  The header-compatible C++ layer in
 * include/super4pcs/ sits on top of THIS ABI; every entry point below names the reference
 * function it replaces (file:line relative to the reference's src/super4pcs/).
 *
 * Conventions
 *  - plain pointers and sizes only; no C++ / torch types.  Every function returns an int
 *    status (S4G_OK == 0); s4g_error_string() gives the text of the last failure of a context.
 *    Nothing throws across this boundary (the C++ layer turns failures into
 *    std::runtime_error, which the reference's demo maps to exit code -2,
 *    demos/Super4PCS/super4pcs_test.cc:147-155).
 *  - 4x4 transforms cross as 16 floats, COLUMN-major (Eigen's default storage of
 *    Match4PCSBase::MatrixType, algorithms/match4pcsBase.h:71).
 *  - "host" pointers are ordinary CPU memory; functions with the suffix _dev take device
 *    pointers on the context's device and enqueue on the context's stream without
 *    synchronising (the caller owns ordering; see s4g_set_stream / s4g_synchronize).
 *  - clouds are the CENTRED sampled clouds, i.e. what Match4PCSBase::init leaves in
 *    sampled_P_3D_ / sampled_Q_3D_ (algorithms/match4pcsBase.hpp:112-149).
 *  - there is no CPU fallback anywhere behind this ABI: without a CUDA device s4g_create fails.
 *  - a context is NOT re-entrant (like a reference matcher instance, match4pcsBase.h mutable state):
 *    one thread at a time per context; distinct contexts are independent (also on the same GPU).
 *  - device pointers passed to *_dev entry points must be 16-byte aligned (cudaMalloc alignment).
 */
#ifndef S4G_H_
#define S4G_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define S4G_ABI_VERSION 1

#define S4G_OK 0
#define S4G_ERR_CUDA 1        /* a CUDA runtime call or kernel failed            */
#define S4G_ERR_ARG 2         /* invalid argument                                */
#define S4G_ERR_STATE 3       /* call order violated (e.g. verify before set_p)  */
#define S4G_ERR_NOMEM 4       /* device allocation failed / capacity exceeded    */
#define S4G_ERR_COMM 5        /* NCCL not loadable, a collective failed or timed out */

typedef struct s4g_ctx s4g_ctx;

int s4g_abi_version(void);
/* number of CUDA devices this process can open contexts on (0 and S4G_ERR_CUDA when there is none or the driver
 * is missing).  The C++ layer uses it for S4PCS_DEVICES=all (candidate-set sharding, SURVEY.md 8(e)). */
int s4g_device_count(int* out_count);

/* One context = one GPU + one stream + the resident clouds/grids of one matcher instance
 * (the device-side counterpart of the reference's per-instance state: kd_tree_, pcfunctor_,
 * sampled_*_3D_; algorithms/match4pcsBase.h:141-165, algorithms/super4pcs.h:76). */
int s4g_create(int device, s4g_ctx** out_ctx);
void s4g_destroy(s4g_ctx* ctx);
const char* s4g_error_string(const s4g_ctx* ctx);

/* Use an external CUDA stream (cudaStream_t as void*; NULL restores the context's own NON-BLOCKING stream -- note that the
 * legacy default stream's handle IS NULL: a caller that works on the default stream passes cudaStreamLegacy /
 * cudaStreamPerThread explicitly, or synchronises with s4g_synchronize). */
int s4g_set_stream(s4g_ctx* ctx, void* cuda_stream);
int s4g_synchronize(s4g_ctx* ctx);

/* ---- clouds ------------------------------------------------------------------------------
 * s4g_set_cloud_p replaces Match4PCSBase::initKdTree (algorithms/match4pcsBase.cc:353-363,
 * accelerators/kdtree.h:349-364,554-635): uploads the centred sampled P and builds the
 * brick-sorted uniform grid (cell edge ~2*delta) that Verify probes.
 * s4g_set_cloud_q replaces MatchSuper4PCS::Initialize -> PairCreationFunctor::synch3DContent
 * (algorithms/super4pcs.cc:230-234, algorithms/pairCreationFunctor.h:90-122): uploads the
 * centred sampled Q (+ optional normals / rgb, NULL = Point3D defaults 0 / -1), computes the
 * unit-cube normalisation (_gcenter, _ratio) and the Morton-ordered copy Verify streams.   */
int s4g_set_cloud_p(s4g_ctx* ctx, const float* xyz, int n, float delta);
int s4g_set_cloud_q(s4g_ctx* ctx, const float* xyz, const float* normals, const float* rgb, int n);
/* out5 = { _gcenter.x, _gcenter.y, _gcenter.z, _ratio, reserved } */
int s4g_get_q_normalization(s4g_ctx* ctx, float* out5);

/* grid statistics for the roofline arithmetic (SURVEY.md 8(d)):
 * out[0]=cell edge h, [1]=#occupied bricks, [2]=brick edge in cells, [3]=#cells allocated,
 * [4]=mean #P points per occupied cell, [5]=grid bytes resident (points+tables)            */
int s4g_get_grid_stats(s4g_ctx* ctx, double* out6);

/* ---- a8: Match4PCSBase::Verify (algorithms/match4pcsBase.cc:508-567) -----------------------
 * For each of K transforms: counts[k] = #{ q in sampled_Q : exists p in sampled_P with
 * ||T q - p||^2 <= delta^2 } (float arithmetic in the reference's association order, no FMA).
 * No early exit: full counts (the reference's partial counts only ever belong to
 * candidates that cannot win; LCP = counts[k] / n_Q).
 * s4g_verify_probe_stats runs the statistics variant of the same kernel: out5 = totals over all
 * (query, candidate) pairs of { P points distance-tested, cell ranges read, brick-table entries
 * read, occupancy / delta-field words read } -- the measured k-bar / C of SURVEY.md 8(d) -- and
 * out5[4] = number of (32-query sub-tile, candidate) pairs culled on the coarse occupancy.    */
int s4g_verify(s4g_ctx* ctx, const float* T_colmajor, int K, uint32_t* counts);
int s4g_verify_dev(s4g_ctx* ctx, const float* d_T_colmajor, int K, uint32_t* d_counts);
int s4g_verify_probe_stats(s4g_ctx* ctx, const float* T_colmajor, int K, uint64_t* out5);
/* Verify + the first-maximum rule of TryCongruentSet (algorithms/match4pcsBase.hpp:467-484) in one stream-ordered chain:
 * counts as s4g_verify*, then key = max_k (counts[k] << 32) | (0xFFFFFFFF - index[k])  (index = the candidates' positions
 * in the caller's whole list; NULL = k), then -- when a communicator is attached, s4g_comm_* below -- the maximum over all
 * ranks.  _dev: everything device-resident, nothing is synchronised (d_key: 8 bytes of device memory, valid in stream
 * order); host form: T / index / counts (may be NULL) / key are host buffers, returns after the read-back.          */
int s4g_verify_best_dev(s4g_ctx* ctx, const float* d_T_colmajor, int K, const uint32_t* d_index,
                        uint32_t* d_counts, uint64_t* d_key);
int s4g_verify_best(s4g_ctx* ctx, const float* T_colmajor, int K, const uint32_t* index, uint32_t* counts,
                    uint64_t* out_key);

/* ---- a6: Match4PCSBase::ComputeRigidTransformation (algorithms/match4pcsBase.cc:365-500) --
 * batched exactly as TryCongruentSet prepares it (algorithms/match4pcsBase.hpp:373-434):
 * base_xyz = the four base points sampled_P[base_id1..4] (12 floats), quads = K x 4 indices
 * into sampled_Q.  max_angle_deg is options.max_angle (degrees, <0 = off).
 * Outputs (host, any may be NULL): T K x 16 column-major, rms K, ok K (the bool returned).  */
int s4g_rigid_batch(s4g_ctx* ctx, const float* base_xyz, const int32_t* quads, int64_t K,
                    float max_angle_deg, float* out_T, float* out_rms, int32_t* out_ok);

/* ---- a7: Match4PCSBase::TryCongruentSet (algorithms/match4pcsBase.hpp:363-497) -------------
 * rigid fit (a6) -> gate ok && 0 <= rms < rms_threshold -> Verify (a8) -> best candidate,
 * all on the device.  Winner rule = the reference's: highest LCP, ties -> first in quad
 * order (strict '>' at hpp:468).  best_count_in = inlier count the winner must strictly beat
 * (= the count behind best_LCP_).  shard_rank/shard_world: this call only processes quads
 * with index % shard_world == shard_rank (candidate-set sharding across GPUs); the caller
 * combines ranks with ONE max-allreduce of `key`.                                          */
typedef struct s4g_tcs_result {
  uint64_t key;          /* (count << 32) | (0xFFFFFFFF - quad_index); 0 when nothing verified */
  uint32_t best_count;   /* inlier count of this shard's winner (0 if none)          */
  int32_t best_index;    /* index into `quads`, -1 if no gate-passing quad           */
  uint32_t n_gate_pass;  /* quads of this shard that passed the rms gate (= Verify calls) */
  uint32_t n_q;          /* |sampled_Q| (LCP = best_count / n_q)                     */
  float best_T[16];      /* column-major transform of the winner (centred frames)    */
  float best_rms;
  float centroid1[3];    /* (b1+b2+b3)/3, hpp:385                                    */
  float centroid2[3];    /* (q0+q1+q2)/3 of the winner, hpp:415-417                  */
  int32_t best_quad[4];  /* the winner's four sampled_Q indices (current_congruent_)  */
} s4g_tcs_result;

int s4g_try_congruent_set(s4g_ctx* ctx, const float* base_xyz, const int32_t* quads, int64_t K,
                          float max_angle_deg, float rms_threshold, int shard_rank,
                          int shard_world, s4g_tcs_result* out);
/* same, quads already resident (device pointer, K x 4 int32) */
int s4g_try_congruent_set_dev(s4g_ctx* ctx, const float* base_xyz, const int32_t* d_quads,
                              int64_t K, float max_angle_deg, float rms_threshold,
                              int shard_rank, int shard_world, s4g_tcs_result* out);
/* same, on the quads left resident by the last s4g_find_quads call */
int s4g_try_congruent_set_resident(s4g_ctx* ctx, const float* base_xyz, float max_angle_deg,
                                   float rms_threshold, int shard_rank, int shard_world,
                                   s4g_tcs_result* out);

/* ---- a2 + a3: MatchSuper4PCS::ExtractPairs (algorithms/super4pcs.cc:183-224) with the pair
 * predicate of PairCreationFunctor::process (algorithms/pairCreationFunctor.h:151-218) --------
 * All ordered pairs (j,i),(i,j) of sampled_Q with |dist - pair_distance| <= epsilon (+ the
 * optional normal / colour / translation / angle filters).  base_p1 / base_p2 = the two base
 * points base_3D_[base_point1], base_3D_[base_point2], 9 floats each (pos, normal, rgb).
 * The result stays resident in pair slot `slot` (0 or 1) and is returned sorted
 * lexicographically by s4g_get_pairs (the reference's order is a traversal artefact; its own
 * test sorts before comparing, tests/pair_extraction.cc:282-283).                           */
typedef struct s4g_pair_filters {
  float max_normal_difference;     /* Match4PCSOptions fields, shared4pcs.h:155-162 */
  float max_translation_distance;
  float max_angle;
  float max_color_distance;
} s4g_pair_filters;

int s4g_extract_pairs(s4g_ctx* ctx, float pair_distance, float pair_normals_angle,
                      float pair_distance_epsilon, const float* base_p1, const float* base_p2,
                      const s4g_pair_filters* filters, int slot, int64_t* n_pairs);
int s4g_get_pairs(s4g_ctx* ctx, int slot, int32_t* out_pairs /* 2*n */);
int s4g_set_pairs(s4g_ctx* ctx, int slot, const int32_t* pairs, int64_t n);
/* counting-only shell query (SURVEY.md 8(d) cfg4): number of ordered pairs, nothing written */
int s4g_count_pairs(s4g_ctx* ctx, float pair_distance, float pair_distance_epsilon,
                    int64_t* n_pairs);
/* same query, additionally out_rows[a] (host, n_Q entries) = number of ordered pairs (a, .): the per-point rows of the
 * list ExtractPairs would write (sum = *n_pairs).  Lets a test check sampled rows of a query whose list is too large to
 * materialise (cfg4: 10M points) against brute force, reference criterion tests/pair_extraction.cc:172-194.          */
int s4g_count_pairs_rows(s4g_ctx* ctx, float pair_distance, float pair_distance_epsilon,
                         uint32_t* out_rows, int64_t* n_pairs);

/* ---- a4 + a5: MatchSuper4PCS::FindCongruentQuadrilaterals (algorithms/super4pcs.cc:80-177)
 * over IndexedNormalSet<Point,3,7,float> (accelerators/normalset.h:71-153, normalset.hpp) ----
 * P_pairs = slot 0, Q_pairs = slot 1.  base_xyz = base_3D_[0..3] positions (12 floats).
 * Quads stay resident, sorted by (v0,v1,v2,v3) (= the std::set<(id,i)> order of
 * super4pcs.cc:127,166-174 when the pair lists are sorted), fetched with s4g_get_quads.     */
int s4g_find_quads(s4g_ctx* ctx, float invariant1, float invariant2,
                   float distance_threshold2, const float* base_xyz, int64_t* n_quads);
int s4g_get_quads(s4g_ctx* ctx, int32_t* out_quads /* 4*n */);

/* ---- f1 (SURVEY.md 8(f)): several RANSAC bases per launch chain -------------------------------
 * One s4g_base_desc = the arguments of the per-base chain  s4g_extract_pairs(slot 0) -> s4g_extract_pairs(slot 1)
 * -> s4g_find_quads -> s4g_try_congruent_set_resident  (reference match4pcsBase.hpp:281-360, one iteration of
 * match4pcsBase.hpp:236-256).  s4g_try_bases runs that chain for n_bases bases at once: the base index is a grid
 * dimension / a key prefix of every kernel, the lists of all bases share buffers, sizes stay on the device, and the
 * host reads back once per stage (3 per batch instead of ~7 per base).  Per base the result equals the per-base
 * chain's (same pair sets, same quads in the same order, same winner).  Limits: n_bases <= 64, |sampled_Q| < 2^26,
 * distance_threshold2 / _ratio >= 2^-14; beyond them S4G_ERR_ARG (callers fall back to the per-base chain).
 * The resident pair slots / quads of the context are left untouched.                                              */
typedef struct s4g_base_desc {
  float pair_distance[2];       /* |b0-b1|, |b2-b3|                                        */
  float pair_normals_angle[2];
  float base_p[4][9];           /* base_3D_[0..3]: pos, normal, rgb (ExtractPairs, FindCongruentQuadrilaterals) */
  float base_xyz_p[12];         /* sampled_P[base ids] positions (TryCongruentSet)          */
  float invariant1, invariant2;
} s4g_base_desc;
typedef struct s4g_base_result {
  int64_t n_pairs[2];
  int64_t n_quads;
  s4g_tcs_result tcs;
} s4g_base_result;
int s4g_try_bases(s4g_ctx* ctx, const s4g_base_desc* bases, int n_bases, float pair_distance_epsilon,
                  const s4g_pair_filters* filters, float distance_threshold2, float max_angle_deg,
                  float rms_threshold, s4g_base_result* out);

/* ---- f2 (SURVEY.md 8(f)): Sampling::UniformDistSampler (sampling.h:59-121) on the device -----
 * keeps the first point (smallest index) of every voxel of edge `voxel`; out_indices (capacity n)
 * receives the kept input indices in ascending order (= the reference's output order).      */
int s4g_voxel_sample(s4g_ctx* ctx, const float* xyz, int64_t n, float voxel, int32_t* out_indices,
                     int64_t* n_out);

/* ---- row e (SURVEY.md 8(e)): the reduction of a sharded candidate set inside the library -----------------------------
 * The reference runs the candidates of a base through one loop (OpenMP-optional, match4pcsBase.hpp:390-393, strict '>' in
 * index order at :467-484).  Here W contexts -- the GPUs of one box -- take the candidates with index % W == rank (the
 * shard_rank / shard_world arguments above).  Without a communicator every shard returns its own winner and the caller
 * takes the maximum key.  With one attached, s4g_try_congruent_set* (when shard_world == the communicator's size, every
 * rank calling with its own rank) and s4g_verify_best* finish on the device with ncclAllReduce(ncclMax) of the packed
 * 64-bit key followed, for TryCongruentSet, by one ncclAllReduce(ncclSum) of the record the non-owners have zeroed: every
 * rank returns the SAME global result (n_gate_pass = the sum over the shards).  NCCL (libnccl.so.2) is loaded on the first
 * s4g_comm_* call; S4G_ERR_COMM when it is missing -- there is no substitute transport.
 *   one process per GPU:   rank 0 calls s4g_comm_unique_id, ships the 128 bytes to the others (MPI, torch.distributed,
 *                          a file ...), every rank calls s4g_comm_init_rank (collective);
 *   one process, W GPUs:   s4g_comm_init_all on the W contexts (ncclCommInitAll; one host thread per context afterwards).
 * s4g_comm_info: out4 = { size (0 = none attached), rank, NCCL version code, collectives enqueued so far }.
 * The first collective of a communicator (NCCL's transport set-up, a blocking exchange) is run by the init calls.  A rank
 * that later waits longer than the time limit (default 60 s, s4g_comm_set_timeout) for its peers aborts the communicator
 * and returns S4G_ERR_COMM instead of blocking for ever; the context is then only good for s4g_destroy.              */
#define S4G_COMM_ID_BYTES 128
int s4g_comm_unique_id(unsigned char* out_id /* S4G_COMM_ID_BYTES */);
int s4g_comm_init_rank(s4g_ctx* ctx, const unsigned char* id, int n_ranks, int rank);
int s4g_comm_init_all(s4g_ctx** ctxs, int n);
int s4g_comm_destroy(s4g_ctx* ctx);
int s4g_comm_info(s4g_ctx* ctx, int* out4);
int s4g_comm_set_timeout(s4g_ctx* ctx, int seconds);

/* ---- timing of the last enqueued hot-path kernels (CUDA events on the context's stream) ----
 * out[0] = ms of the last Verify kernel(s), out[1] = ms of the last rigid-fit kernel,
 * out[2] = ms of the last pair extraction, out[3] = ms of the last quad extraction,
 * out[4] = number of kernel launches this context has made since creation.                 */
int s4g_get_timings(s4g_ctx* ctx, double* out5);

#ifdef __cplusplus
}
#endif
#endif /* S4G_H_ */
