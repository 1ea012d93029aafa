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
 *    The one exception is s4g_try_congruent_set_dev: it returns its record in host memory
 *    (and reads the gate count back to size Verify), so it waits for the context's stream.
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
/* The neighbour Verify looks up and drops: for every sampled-Q point i (the order of s4g_set_cloud_q) and each of K
 * transforms, the sampled-P point nearest to T q_i within delta (reference match4pcsBase.cc:531-536, the query of
 * KdTree::doQueryRestrictedClosestIndex, accelerators/kdtree.h:388-453).  T q and d^2 = dx^2 + (dy^2 + dz^2) use the
 * arithmetic of s4g_verify (fp32, reference operation order, no FMA; kdtree.h:417-418).
 *   index[k * n_Q + i]   = j, the position in the array passed to s4g_set_cloud_p (= in sampled_P_3D_, the order
 *                          initKdTree adds the points in, match4pcsBase.cc:353-363) with the smallest d^2 <= delta^2;
 *                          -1 when there is none
 *   sq_dist[k * n_Q + i] = that d^2, bit for bit; +inf when index = -1 (sq_dist may be NULL)
 *   counts[k]            = #{i : index[k * n_Q + i] >= 0} = s4g_verify's count for the same T (counts may be NULL)
 * Tie rule -- the one deliberate difference from the reference: among points of equal d^2 the SMALLEST j wins.  The
 * kd-tree keeps the last one its traversal visits (sqdist <= cl_dist, kdtree.h:417), an artefact of the tree's shape.
 * So sq_dist equals the reference's wherever it finds a neighbour, and index equals it wherever the minimum is unique.
 * _dev: device buffers (d_index / d_sq_dist: K x n_Q), enqueued on the context's stream, nothing synchronised.       */
int s4g_verify_nearest(s4g_ctx* ctx, const float* T_colmajor, int K, int32_t* index, float* sq_dist, uint32_t* counts);
int s4g_verify_nearest_dev(s4g_ctx* ctx, const float* d_T_colmajor, int K, int32_t* d_index, float* d_sq_dist,
                           uint32_t* d_counts);
/* The restricted closest-point query of the reference's kd-tree (KdTree::doQueryRestrictedClosestIndex,
 * accelerators/kdtree.h:388-453) on the resident sampled P, for n arbitrary query points xyz (n x 3):
 *   index[i]   = j with the smallest d^2 = |y_i - p_j|^2 <= sq_radius and j != exclude[i]  (-1: none),
 *                y_i = T x_i (fp32, reference order, no FMA) or x_i when T is NULL; d^2 = dx^2 + (dy^2 + dz^2) in fp32
 *   sq_dist[i] = that d^2 bit for bit, +inf for -1 (may be NULL)
 * j is the position in the array passed to s4g_set_cloud_p.  sq_radius is the kd-tree's RangeQuery::sqdist: any value,
 * +inf = unbounded; NaN -> S4G_ERR_ARG.  exclude: NULL or n entries (-1 = none) -- the kd-tree's currentId.  Ties: the
 * smallest j (as s4g_verify_nearest).  A query with a NaN coordinate finds nothing.  The kd-tree never takes a point whose
 * d^2 equals sq_radius when its pruning test (strict <) stops first, so at sq_radius = 0 it finds nothing at all; here
 * d^2 <= sq_radius holds exactly.  Needs s4g_set_cloud_p only (S4G_ERR_STATE before it); n == 0 is a no-op.
 * _dev: device buffers, enqueued on the context's stream, nothing synchronised.
 * _probe_stats: as s4g_nearest, and out2 = {P points tested, coarse blocks scanned} summed over the queries.          */
int s4g_nearest(s4g_ctx* ctx, const float* xyz, int n, const float* T_colmajor, float sq_radius, const int32_t* exclude,
                int32_t* index, float* sq_dist);
int s4g_nearest_dev(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T_colmajor, float sq_radius,
                    const int32_t* d_exclude, int32_t* d_index, float* d_sq_dist);
int s4g_nearest_probe_stats(s4g_ctx* ctx, const float* xyz, int n, const float* T_colmajor, float sq_radius,
                            const int32_t* exclude, int32_t* index, float* sq_dist, uint64_t* out2);
/* The k nearest neighbours on the resident sampled P, for n arbitrary query points xyz (n x 3).  Row i is
 * index[i*k .. i*k+k) / sq_dist[i*k .. i*k+k) (64-bit offsets: n*k may exceed 2^31): the k lexicographically smallest
 * (d^2, j) over the P points with d^2 = |y_i - p_j|^2 <= sq_radius and j != exclude[i], in ascending (d^2, j); y_i, d^2
 * and j as in s4g_nearest (sq_dist bit for bit what it computes).  A row with fewer such points is padded at its end with
 * index -1 and sq_dist +inf; a query with a NaN coordinate gets a row of padding.  k = 1 is s4g_nearest bit for bit.  For
 * a finite radius, row i is the first k entries of the s4g_range list at nextafterf(sq_radius, +inf) with j = exclude[i]
 * removed, ordered by (d^2, j).  1 <= k <= 64, sq_radius any value but NaN (+inf = unbounded), exclude NULL or n entries
 * (-1 = none); otherwise S4G_ERR_ARG.  Needs s4g_set_cloud_p only (S4G_ERR_STATE before it); n == 0 is a no-op; an
 * output the device cannot stage -> S4G_ERR_NOMEM.  sq_dist may be NULL.
 * _dev: device buffers, enqueued on the context's stream, nothing synchronised.
 * _probe_stats: as s4g_knn, and out2 = {P points tested, coarse blocks scanned} summed over the queries.              */
int s4g_knn(s4g_ctx* ctx, const float* xyz, int n, const float* T_colmajor, int k, float sq_radius,
            const int32_t* exclude, int32_t* index, float* sq_dist);
int s4g_knn_dev(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T_colmajor, int k, float sq_radius,
                const int32_t* d_exclude, int32_t* d_index, float* d_sq_dist);
int s4g_knn_probe_stats(s4g_ctx* ctx, const float* xyz, int n, const float* T_colmajor, int k, float sq_radius,
                        const int32_t* exclude, int32_t* index, float* sq_dist, uint64_t* out2);
/* Normals of the resident sampled P by PCA of k-nearest neighbourhoods, for every point j in the order of the array passed
 * to s4g_set_cloud_p: normals[3j .. 3j+3), eigenvalues[3j .. 3j+3).
 *   Neighbourhood: exactly the s4g_knn row of the query p_j (no T, no exclusion, the same k and sq_radius), so p_j itself
 *   is in it unless more than k points coincide with it; the padding is skipped; m >= 1 real entries.
 *   Arithmetic, all in double, sums from 0 in row order (ascending (d^2, j)): c = sum p / m, C = sum (p - c)(p - c)^T / m,
 *   then cyclic Jacobi rotations on C (pairs (0,1), (0,2), (1,2) per sweep; an off-diagonal entry is zeroed when 100 |a_pq|
 *   is lost against both |a_pp| and |a_qq|) until the off-diagonal is exactly zero, at most 50 sweeps.  Only + - * /,
 *   sqrt and comparisons: a CPU restatement with no FMA gives the same bits.
 *   eigenvalues = lambda0 <= lambda1 <= lambda2, the diagonal sorted stably (equal values keep the order of the Jacobi
 *   columns, which start as the x, y, z axes), rounded to float.  Curvature is lambda0 / (lambda0 + lambda1 + lambda2).
 *   normal = the Jacobi column of lambda0 (ties: the first of the equal columns in that order), normalised in double,
 *   rounded to float.  Sign: with a viewpoint v (3 floats), negated when (v - p_j) . n < 0 in double; with viewpoint NULL,
 *   the returned float normal's component of largest magnitude is made positive, ties to the lowest axis.
 *   No normal: m < 3 or C exactly zero (e.g. coincident points) -> (0, 0, 0), which the pair filter skips; the
 *   eigenvalues are written all the same.
 * 3 <= k <= 64, sq_radius >= 0 and not NaN (+inf = unbounded), normals != NULL; otherwise S4G_ERR_ARG.  Needs
 * s4g_set_cloud_p (S4G_ERR_STATE before it); scratch the device cannot hold (nP x (k + 3) 4-byte words) -> S4G_ERR_NOMEM.
 * eigenvalues may be NULL.
 * _dev: device buffers (nP x 3 floats each), enqueued on the context's stream, nothing synchronised; viewpoint is 3 host
 * floats (or NULL), read before the call returns.                                                                      */
int s4g_normals(s4g_ctx* ctx, int k, float sq_radius, const float* viewpoint, float* normals, float* eigenvalues);
int s4g_normals_dev(s4g_ctx* ctx, int k, float sq_radius, const float* viewpoint, float* d_normals, float* d_eigenvalues);
/* Consistent orientation of the normals of the resident sampled P (Hoppe et al. 1992; Open3D's
 * orient_normals_consistent_tangent_plane), made exact: signs propagated along the minimum spanning forest of the
 * symmetrised k-nearest graph.  j is the position in the array passed to s4g_set_cloud_p; normals holds nP x 3 floats in
 * that order (what s4g_normals writes); any non-zero vector is a normal, its length does not matter.
 *   Vertices: the points whose normal is not (0, 0, 0).  The others keep it, get root[j] = -1 and belong to no component.
 *   Edges: row j is exactly the s4g_knn row of the query p_j with exclude = j, no T, the caller's k and sq_radius; the
 *   undirected edge {i, j} exists iff j is in row i or i is in row j, and both ends are vertices (padding skipped).
 *   Edge values, fp32, no FMA, from the input normals: dot = (xi xj + yi yj) + zi zj (the same float from either end);
 *   flip f(i, j) = dot < 0 (strict: 0 and -0 are no flip).
 *   Order: |dot| descending, then lo = min(i, j) ascending, then hi = max(i, j) ascending (Hoppe's weight 1 - |dot|
 *   without the rounding of 1 - x).  It is total, so the minimum spanning forest is unique.  A NaN dot (products that
 *   overflow to opposite infinities) ranks above +inf and is no flip.
 *   Components: those of the graph; root[j] = the smallest j in j's component (the rule of s4g_euclidean_clusters).
 *   Anchor of a component: without a viewpoint, its root, which keeps the sign of its input normal; with a viewpoint v
 *   (3 finite floats), the member with the smallest d^2 = dx^2 + (dy^2 + dz^2), d = p - v in fp32 without FMA, ties to
 *   the smallest j, whose normal is negated when (v - p_a) . n_a < 0 in double (s4g_normals' viewpoint rule).
 *   Output: normals_out[j] = the input normal, negated iff (the anchor's negation) xor (the xor of f over the edges of the
 *   forest path from the anchor to j).  Every output float is + or - its input float, bit for bit.
 *   out2 = {n_components, n_tree_edges}, n_tree_edges = (number of vertices) - n_components.  tree_edges: the forest as
 *   (lo, hi) int32 pairs in ascending (lo, hi), capacity 2 (nP - 1) int32.  root and tree_edges may be NULL.
 *   Every output is integer work on the forest, which the edge set and the order fix, plus one double comparison per
 *   component: the same bits on every run.
 * 1 <= k <= 64, sq_radius >= 0 and not NaN (+inf = unbounded), normals, normals_out and out2 != NULL, viewpoint NULL or
 * finite; otherwise S4G_ERR_ARG.  A normal component that is not finite -> S4G_ERR_ARG.  normals_out may equal normals
 * (in place).  Needs s4g_set_cloud_p (S4G_ERR_STATE before it); scratch the device cannot hold (nP x (k + 13) 4-byte
 * words plus CUB's radix sort storage, and 24 more bytes per point in the host form) -> S4G_ERR_NOMEM.
 * _dev: device buffers (d_out2 two int64), enqueued on the context's stream, nothing synchronised; viewpoint is 3 host
 * floats (or NULL), read before the call returns.  A non-finite normal component cannot be returned as a code: the call
 * then writes d_out2[0] = -1 and the other outputs are undefined.                                                      */
int s4g_orient_normals(s4g_ctx* ctx, const float* normals, int k, float sq_radius, const float* viewpoint,
                       float* normals_out, int32_t* root, int64_t* out2, int32_t* tree_edges);
int s4g_orient_normals_dev(s4g_ctx* ctx, const float* d_normals, int k, float sq_radius, const float* viewpoint,
                           float* d_normals_out, int32_t* d_root, int64_t* d_out2, int32_t* d_tree_edges);
/* FPFH descriptors of the resident sampled P (Rusu et al. 2009; PCL's FPFHEstimation, Open3D's compute_fpfh_feature),
 * made exact.  j is the position in the array passed to s4g_set_cloud_p; normals holds nP x 3 floats in that order (what
 * s4g_normals writes); fpfh receives nP x 33 floats in the same order: bins 0-10 f1, 11-21 f2, 22-32 f3.  The descriptors
 * depend on the signs of the normals (negating them all mirrors the f1 and f3 blocks), so orient them consistently first
 * (s4g_orient_normals).
 *   Row of j: exactly the s4g_knn row of the query p_j with exclude = j, no T, the caller's k and sq_radius, in ascending
 *   (d^2, index), padding skipped, d^2 the float s4g_knn returns (Open3D's hybrid search with max_nn = k + 1).
 *   Normals: (0, 0, 0) or a non-finite component is no normal; any other is divided by sqrt(n . n) in double.  A point
 *   without a normal gets an all-zero descriptor; row entries without a normal are left out, and m_j is the number of
 *   entries that remain.
 *   Arithmetic: double, from the float inputs, + - * /, sqrt, floor and comparisons only, no FMA; every dot product is
 *   (a0 b0 + a1 b1) + a2 b2 and every cross product the textbook component formula.
 *   Pair feature of (p1, n1) = (p_j, n_j), (p2, n2) = (p_e, n_e) (Open3D's ComputePairFeatures with its two rounded
 *   transcendental decisions made exact): dp = p2 - p1, d = sqrt(dp . dp), degenerate if d = 0; a1 = n1 . dp / d,
 *   a2 = n2 . dp / d; swap iff |a1| < |a2| (Open3D's acos(|a1|) > acos(|a2|)): then (u, n') = (n2, n1), dp = -dp and
 *   f3 = -a2, else (u, n') = (n1, n2) and f3 = a1; v = dp x u, degenerate if |v| = 0, else v = v / |v|; w = u x v;
 *   f2 = v . n'; the f1 direction is (x, y) = (u . n', w . n').  A degenerate pair lands in bins (5, 16, 27).
 *   Bins: f2, f3: floor(11 * (f + 1.0) * 0.5) left to right, clamped to [0, 10].  f1: floor(11 (atan2(y, x) + pi) / 2pi)
 *   replaced by exact half-plane tests against beta_i = -pi + 2 pi i / 11, c_i = cos beta_i and s_i = sin beta_i correctly
 *   rounded to double, c_{11-i} = c_i and s_{11-i} = -s_i:
 *     i = 1: c -0x1.aeb8c8764f0bap-1, s -0x1.14cedf8bb580bp-1    i = 4: c 0x1.4f49e7f775887p-1, s -0x1.82f19bb3a28a1p-1
 *     i = 2: c -0x1.a9628d9c712b6p-2, s -0x1.d1bb48eee2c13p-1    i = 5: c 0x1.eb42a9bcd5057p-1, s -0x1.207e7fd768dbfp-2
 *     i = 3: c  0x1.2375f640f44dbp-3, s -0x1.fac9e043842efp-1
 *   y = 0 (either sign): bin 10 if x < 0, else 5; y > 0: 5 + #{i in 6..10 : c_i y - s_i x >= 0};
 *   y < 0: #{i in 1..5 : c_i y - s_i x >= 0}.
 *   SPFH of j: cnt_j[b] the pairs of j's row in bin b; spfh_j[b] = (100.0 cnt_j[b]) / m_j (all zero when m_j = 0).
 *   FPFH of j: acc[b] = the sum, over the entries e of j's row with d^2_e > 0, in row order from 0.0, of
 *   spfh_e[b] / d^2_e (the inverse squared distance, as PCL's and Open3D's code weigh); S_h = acc[11h] + ... + acc[11h+10]
 *   left to right; fpfh[j][b] = (float)(acc[b] * (100.0 / S_h) + spfh_j[b]), or (float)spfh_j[b] when S_h = 0.  Open3D
 *   sums S_h interleaved with acc; the per-bin form lets bins be reduced independently and differs only in rounding.
 *   Every output is fixed by these operations: the same bits on every run and on a CPU restatement without contraction.
 * 1 <= k <= 64, sq_radius >= 0 and not NaN (+inf = unbounded), normals and fpfh != NULL; otherwise S4G_ERR_ARG.  Needs
 * s4g_set_cloud_p (S4G_ERR_STATE before it); scratch the device cannot hold (nP x (8k + 48) bytes, and nP x 144 more in
 * the host form) -> S4G_ERR_NOMEM.
 * _dev: device buffers, enqueued on the context's stream, nothing synchronised.                                       */
int s4g_fpfh(s4g_ctx* ctx, const float* normals, int k, float sq_radius, float* fpfh);
int s4g_fpfh_dev(s4g_ctx* ctx, const float* d_normals, int k, float sq_radius, float* d_fpfh);
/* Nearest descriptor by brute force (Open3D's correspondence search of its feature RANSAC), on arbitrary arrays (no
 * resident cloud needed): a is n_a x 33 floats, b is n_b x 33.  d^2(i, j) in fp32 without FMA, from 0.0f, over
 * c = 0 .. 32 left to right: s = s + (a_c - b_c) * (a_c - b_c).  index[i] = the j of the lexicographically smallest
 * (d^2, j) over the finite d^2 (a NaN or +inf never wins), sq_dist[i] = that d^2; a row with no finite d^2 gets -1 and
 * +inf.  mutual != 0: index[i] becomes -1 unless the nearest a-row of b_{index[i]}, by the same rule, is i; sq_dist keeps
 * the nearest d^2 either way.  0 <= n_a, n_b < 2^31; n_a = 0 does nothing; n_b = 0 gives all -1.  sq_dist may be NULL.
 * a NULL a or index with n_a > 0, or b with n_a, n_b > 0 -> S4G_ERR_ARG; scratch the device cannot hold (8 bytes per
 * row of a, and per row of b when mutual; the host form stages a, b and the outputs too) -> S4G_ERR_NOMEM.
 * _dev: device buffers, enqueued on the context's stream, nothing synchronised.                                       */
int s4g_fpfh_match(s4g_ctx* ctx, const float* a, int64_t n_a, const float* b, int64_t n_b, int mutual, int32_t* index,
                   float* sq_dist);
int s4g_fpfh_match_dev(s4g_ctx* ctx, const float* d_a, int64_t n_a, const float* d_b, int64_t n_b, int mutual,
                       int32_t* d_index, float* d_sq_dist);
/* Outlier removal on the resident sampled P.  j is the position in the array passed to s4g_set_cloud_p.  Both filters
 * write the kept j in ascending order to keep[0 .. *n_kept) (capacity nP; the output form of s4g_voxel_sample).
 *
 * Statistical filter (PCL's StatisticalOutlierRemoval, made exact):
 *   Row of j: exactly the s4g_knn row of the query p_j with exclude = j, no T, sq_radius = +inf: m = min(k, nP - 1) real
 *   entries, d2_e the floats s4g_knn returns.
 *   mean_dist[j] = (sum over the row in row order, from 0.0, of sqrt((double) d2_e)) / m.
 *   mu and sigma in double, each sum in this fixed order: the j in ascending order are cut into runs of 1024 (the last
 *   may be shorter), each run summed left to right from 0.0, then the run sums left to right from 0.0.
 *     mu = (sum of mean_dist) / nP;  sigma = sqrt((sum of (mean_dist - mu)^2) / (nP - 1)), a second pass in that order.
 *   j is kept iff mean_dist[j] <= mu + std_ratio * sigma, in double.  Only + - * /, sqrt and comparisons, no FMA: a CPU
 *   restatement compiled without contraction gives the same bits.  nP = 1: the point is kept, mean_dist = mu = sigma = 0.
 *   out2 = {mu, sigma}.  mean_dist (nP doubles) and out2 may be NULL.
 *   1 <= k <= 64 and std_ratio finite (any sign), keep and n_kept != NULL; otherwise S4G_ERR_ARG.  Needs s4g_set_cloud_p
 *   (S4G_ERR_STATE before it); scratch the device cannot hold (about nP x (2k + 6) 4-byte words) -> S4G_ERR_NOMEM.
 *
 * Radius filter (PCL's RadiusOutlierRemoval, made exact):
 *   c_j = #{i != j : d^2(p_i, p_j) < sq_radius}, d^2 and the strict test exactly as in s4g_range: for sq_radius > 0, c_j
 *   is the length of the s4g_range list of the query p_j minus 1 (p_j's own d^2 is exactly 0).  sq_radius <= 0: c_j = 0;
 *   +inf: every other point with a finite d^2.
 *   j is kept iff c_j >= min_neighbors.  counts[j] = min(c_j, min_neighbors): the count stops there (this is what makes
 *   the filter cheap in dense regions), so the value is capped.  counts (nP int32) may be NULL.
 *   sq_radius not NaN, min_neighbors >= 1, keep and n_kept != NULL; otherwise S4G_ERR_ARG.  STATE and NOMEM as above.
 *
 * _dev: device buffers (d_n_kept one int64), enqueued on the context's stream, nothing synchronised.                    */
int s4g_statistical_outliers(s4g_ctx* ctx, int k, double std_ratio, int32_t* keep, int64_t* n_kept, double* mean_dist,
                             double* out2);
int s4g_statistical_outliers_dev(s4g_ctx* ctx, int k, double std_ratio, int32_t* d_keep, int64_t* d_n_kept,
                                 double* d_mean_dist, double* d_out2);
int s4g_radius_outliers(s4g_ctx* ctx, float sq_radius, int min_neighbors, int32_t* keep, int64_t* n_kept,
                        int32_t* counts);
int s4g_radius_outliers_dev(s4g_ctx* ctx, float sq_radius, int min_neighbors, int32_t* d_keep, int64_t* d_n_kept,
                            int32_t* d_counts);
/* Euclidean clusters of the resident sampled P (PCL's EuclideanClusterExtraction, made exact).  j is the position in the
 * array passed to s4g_set_cloud_p.
 *   Graph: an edge (i, j), i != j, iff d^2(p_i, p_j) < sq_radius, d^2 and the strict test exactly as in s4g_range (fp32,
 *   dx^2 + (dy^2 + dz^2), no FMA).  The graph is symmetric bit for bit: under round to nearest fl(a - b) = -fl(b - a), so
 *   d^2(p_i, p_j) and d^2(p_j, p_i) are the same float, and the search takes each edge once, from its larger end.
 *   sq_radius <= 0: no edges; +inf: every pair with a finite d^2 (s4g_set_cloud_p refuses non-finite coordinates).
 *   Components: root[j] = the smallest j' in j's connected component, before any size filter.
 *   A component is a cluster iff min_size <= size <= max_size.  Clusters are ordered by size, descending, ties by root,
 *   ascending (PCL sorts by size and leaves ties unspecified).  labels[j] = the rank of j's cluster in that order, -1 when
 *   j's component is not a cluster; *n_clusters = their number.
 *   Members in CSR form: cluster c is members[offsets[c] .. offsets[c + 1]), in ascending j.  Capacities nP + 1 (offsets)
 *   and nP (members); only offsets[0 .. n_clusters] and members[0 .. offsets[n_clusters]) are defined.
 *   Every output is integer work on the component partition, which depends on the edge set alone: the same bits on
 *   every run.
 * min_size >= 1 and max_size >= min_size (INT_MAX: no limit), sq_radius not NaN, labels and n_clusters != NULL;
 * otherwise S4G_ERR_ARG.  root, offsets and members may be NULL.  Needs s4g_set_cloud_p (S4G_ERR_STATE before it);
 * scratch the device cannot hold (24 bytes per P point, 44 in the host form, plus CUB's radix sort and scan storage)
 * -> S4G_ERR_NOMEM.
 * _dev: device buffers (d_n_clusters one int64), enqueued on the context's stream, nothing synchronised.             */
int s4g_euclidean_clusters(s4g_ctx* ctx, float sq_radius, int min_size, int max_size, int32_t* labels, int32_t* root,
                           int64_t* n_clusters, int64_t* offsets, int32_t* members);
int s4g_euclidean_clusters_dev(s4g_ctx* ctx, float sq_radius, int min_size, int max_size, int32_t* d_labels,
                               int32_t* d_root, int64_t* d_n_clusters, int64_t* d_offsets, int32_t* d_members);
/* One plane found by s4g_segment_planes (64 bytes, no padding). */
typedef struct s4g_plane {
  float coefficients[4];       /* final (a, b, c, d): a x + b y + c z + d = 0, |(a, b, c)| = 1 in double before rounding */
  float hypothesis[4];         /* the winning hypothesis' plane, before the refit                                        */
  int32_t hypothesis_index;    /* its h                                                                                  */
  int32_t sample[3];           /* its three positions j                                                                  */
  int64_t hypothesis_inliers;  /* its count                                                                              */
  int64_t n_inliers;           /* final count = the length of this plane's member list                                  */
} s4g_plane;
/* Plane segmentation of the resident sampled P (PCL's SACSegmentation with SACMODEL_PLANE and optimize_coefficients,
 * made exact): RANSAC with every hypothesis scored, no early termination, so the result is a pure function of (cloud,
 * threshold, n_hypotheses, seed, refine, max_planes, min_inliers).  j is the position in the array passed to
 * s4g_set_cloud_p; H = n_hypotheses.
 *   Rounds r = 0, 1, ..., max_planes - 1.  A_r = the ascending list of the j that no earlier plane claimed (all of P for
 *   r = 0), m = |A_r|.  m < 3: stop.
 *   Draws.  seed_r = seed + r (mod 2^64).  Hypothesis h (0 <= h < H) takes draws t = 0, 1, 2; draw t is the k-th
 *   SplitMix64 output, k = 3h + t + 1 (all mod 2^64):
 *     z = seed_r + k * 0x9E3779B97F4A7C15;  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;
 *     z = (z ^ (z >> 27)) * 0x94D049BB133111EB;  z = z ^ (z >> 31);
 *   its point is A_r[((z >> 32) * m) >> 32].
 *   Hypothesis plane, in double from the three float points p0, p1, p2: u = p1 - p0, v = p2 - p0, n = u x v
 *   (nx = uy vz - uz vy, ny = uz vx - ux vz, nz = ux vy - uy vx), len = sqrt((nx nx + ny ny) + nz nz).  len == 0
 *   (repeated draws, coincident or collinear points): the hypothesis is invalid and counts 0.  Otherwise n = n / len; if
 *   n's component of largest magnitude is negative (ties to the lowest axis), n = -n; d = -((nx x0 + ny y0) + nz z0);
 *   the four values rounded to float.
 *   Inlier test, fp32, no FMA: r = ((a x + b y) + c z) + d; p is an inlier iff |r| < threshold (strict, as s4g_range
 *   and PCL's and Open3D's plane models), for the points of A_r only.  hyp_counts[r H + h] = the count of hypothesis h.
 *   Winner: the valid hypothesis with the largest count, ties to the smallest h.  No valid hypothesis: stop.
 *   Refit (refine != 0): I = the winner's inliers in ascending j.  In double, c = sum p / |I|, then a second pass C =
 *   sum (p - c)(p - c)^T / |I|; each sum in this fixed order: the I in ascending j cut into runs of 1024 (the last may be
 *   shorter), each run summed left to right from 0.0, then the run sums left to right from 0.0.  The eigenvector of C's
 *   smallest eigenvalue as in s4g_normals (its Jacobi rotations, stable sort and column rule), normalised in double, the
 *   sign rule above, d = -((nx cx + ny cy) + nz cz), rounded to float.  |I| < 3 or C exactly zero: the hypothesis plane.
 *   refine == 0: the hypothesis plane.
 *   Final inliers: the test above with the final coefficients over A_r (PCL's re-selection after its refit).  Plane r is
 *   accepted iff their number >= min_inliers; otherwise stop (a rejected plane is not reported).  An accepted plane's
 *   points get labels[j] = r and leave the active set.
 *   Outputs: labels[j] = the plane that claimed j, -1 for none.  planes[0 .. *n_planes) (capacity max_planes).  Members
 *   in CSR form: plane r is members[offsets[r] .. offsets[r + 1]), in ascending j (capacities max_planes + 1 and nP;
 *   only offsets[0 .. n_planes] and members[0 .. offsets[n_planes]) are defined).  hyp_counts: max_planes x H entries,
 *   the rows of rounds that drew nothing all zero.
 *   Every count is an integer and every value is made of IEEE basic operations in a stated order, compiled without
 *   FMA: a CPU restatement compiled without contraction gives the same bits.
 * threshold not NaN and >= 0 (+inf: every active point), 1 <= n_hypotheses <= 2^20, max_planes >= 1, min_inliers >= 1,
 * labels, planes and n_planes != NULL; otherwise S4G_ERR_ARG.  offsets, members and hyp_counts may be NULL.  Needs
 * s4g_set_cloud_p (S4G_ERR_STATE before it); scratch the device cannot hold (37 bytes per P point, 45 in the host form, 36 per
 * hypothesis, plus CUB's select and radix sort storage) -> S4G_ERR_NOMEM.
 * _dev: device buffers (d_n_planes one int32), enqueued on the context's stream, nothing synchronised; after a stop the
 * later rounds are no-ops that read a device flag.                                                                        */
int s4g_segment_planes(s4g_ctx* ctx, float threshold, int n_hypotheses, uint64_t seed, int refine, int max_planes,
                       int64_t min_inliers, int32_t* labels, s4g_plane* planes, int* n_planes, int64_t* offsets,
                       int32_t* members, uint32_t* hyp_counts);
int s4g_segment_planes_dev(s4g_ctx* ctx, float threshold, int n_hypotheses, uint64_t seed, int refine, int max_planes,
                           int64_t min_inliers, int32_t* d_labels, s4g_plane* d_planes, int* d_n_planes,
                           int64_t* d_offsets, int32_t* d_members, uint32_t* d_hyp_counts);
/* The range query of the reference's kd-tree (KdTree::doQueryDist / doQueryDistIndices / doQueryDistProcessIndices,
 * accelerators/kdtree.h:231-262, body :462-514) on the resident sampled P, for n arbitrary query points xyz (n x 3):
 * the list of query i is every j with d^2 = |y_i - p_j|^2 < sq_radius (strict, the kd-tree's point test kdtree.h:485),
 * y_i and d^2 as in s4g_nearest, j the position in the array passed to s4g_set_cloud_p, in ascending j.  sq_radius <= 0:
 * empty lists; +inf: every point with a finite d^2; NaN -> S4G_ERR_ARG.  A query with a NaN coordinate gets an empty
 * list.  No index is excluded.  Output in CSR form: offsets [n + 1] (offsets[0] = 0, offsets[n] = total), list i =
 * indices[offsets[i] .. offsets[i + 1]), sq_dist the same positions (d^2 bit for bit).  Needs s4g_set_cloud_p only
 * (S4G_ERR_STATE before it); n == 0 writes offsets[0] = 0; a result the device cannot hold -> S4G_ERR_NOMEM.
 *   s4g_range       writes offsets and *total, keeps the lists in the context (replacing the previous result);
 *   s4g_get_range   copies the last s4g_range result out (indices [total], sq_dist [total] or NULL); S4G_ERR_STATE when
 *                   there is none (none after a failed s4g_range).
 *   _count_dev / _fill_dev: device buffers, enqueued on the context's stream, nothing synchronised.  count writes
 *   d_offsets [n + 1]; the caller reads d_offsets[n] (= total), allocates, and passes it to fill, which writes the
 *   sorted lists (d_sq_dist may be NULL).                                                                             */
int s4g_range(s4g_ctx* ctx, const float* xyz, int n, const float* T_colmajor, float sq_radius, int64_t* offsets,
              int64_t* total);
int s4g_get_range(s4g_ctx* ctx, int32_t* indices, float* sq_dist);
int s4g_range_count_dev(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T_colmajor, float sq_radius,
                        int64_t* d_offsets);
int s4g_range_fill_dev(s4g_ctx* ctx, const float* d_xyz, int n, const float* d_T_colmajor, float sq_radius,
                       const int64_t* d_offsets, int64_t total, int32_t* d_indices, float* d_sq_dist);
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
 * fewer than 2^26 pairs in every extraction (the quad keys hold a pair's index in 26 bits), quad grid depth <= 14
 * (distance_threshold2 / _ratio above about 2^-15); beyond them S4G_ERR_ARG.  More than 2^32 - 1 pairs or 2^31 - 1
 * quads in one batch: S4G_ERR_NOMEM.  Callers fall back to the per-base chain on either code.
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
/* Voxel-grid downsampling to centroids (PCL's VoxelGrid with setMinimumPointsNumberPerVoxel, Open3D's voxel_down_sample
 * with its trace, made exact) of n arbitrary points xyz (n x 3; no resident cloud needed: it shrinks a cloud before
 * s4g_set_cloud_p).  i is the input index.
 *   Voxel of a point: (floor(x s), floor(y s), floor(z s)) with s = 1.0f / leaf and each product one fp32 rounding, the
 *   arithmetic of s4g_voxel_sample (and PCL's).  The key is 3 x 21 bits, relative to the voxel of the bounding-box
 *   minimum, as in s4g_voxel_sample.  A coordinate that is not finite, a scaled coordinate whose floor is outside the
 *   int32 range, or a span of 2^21 or more voxels along an axis -> S4G_ERR_ARG.
 *   Members of a voxel: its points in ascending i; m their number.  A voxel with m < min_points is dropped.
 *   Sums, in double, each in this fixed order: the members cut into runs of 1024 (the last may be shorter), each run
 *   summed left to right from 0.0, then the run sums left to right from 0.0.  Only + - * /, sqrt and comparisons, no
 *   FMA: a CPU restatement compiled without contraction gives the same bits.
 *     centroid = (sum p) / m, rounded to float;  rgb = (sum rgb) / m, rounded to float;
 *     normal: S = sum n, len = sqrt((Sx Sx + Sy Sy) + Sz Sz); len == 0: (0, 0, 0), which the pair filter reads as "no
 *     normal"; otherwise S / len, rounded to float.  Zero normals add nothing; opposite normals cancel, so averaging
 *     assumes consistently oriented normals: the recommended chain downsamples first and estimates normals afterwards.
 *   Output order: the surviving voxels in ascending order of their first (smallest) member i, i.e. input order.
 *     xyz_out / normals_out / rgb_out [v] as above; counts[v] = m; first[v] = the smallest member i (with min_points = 1
 *     exactly the output of s4g_voxel_sample); voxel_of[i] = the output index of i's voxel, -1 when it was dropped
 *     (Open3D's trace: it averages any other attribute).  *n_out = the number of surviving voxels.
 *   normals / normals_out and rgb / rgb_out are pairs, both NULL or both given; counts, first and voxel_of may be NULL.
 *   Output capacity n (voxel_of: n entries).  leaf finite and > 0, min_points >= 1, 0 <= n < 2^31, xyz, xyz_out and
 *   n_out != NULL; otherwise S4G_ERR_ARG.  n == 0: *n_out = 0.
 *   Device scratch: 36 bytes per point plus 12 per attribute array given (48 for xyz alone, 72 with normals and rgb),
 *   plus CUB's radix sort and scan storage; the host form also holds its inputs and outputs on the device (12 bytes
 *   per point per attribute array each way, 4 per index array).  Scratch the device cannot hold -> S4G_ERR_NOMEM.
 * _dev: device buffers (d_n_out one int64), enqueued on the context's stream, nothing synchronised.  So an invalid
 * coordinate or too wide a span cannot be returned as a code: the call then writes *d_n_out = -1 and the outputs are
 * undefined.                                                                                                            */
int s4g_voxel_grid(s4g_ctx* ctx, const float* xyz, const float* normals, const float* rgb, int64_t n, float leaf,
                   int min_points, float* xyz_out, float* normals_out, float* rgb_out, int32_t* counts, int32_t* first,
                   int32_t* voxel_of, int64_t* n_out);
int s4g_voxel_grid_dev(s4g_ctx* ctx, const float* d_xyz, const float* d_normals, const float* d_rgb, int64_t n, float leaf,
                       int min_points, float* d_xyz_out, float* d_normals_out, float* d_rgb_out, int32_t* d_counts,
                       int32_t* d_first, int32_t* d_voxel_of, int64_t* d_n_out);

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
