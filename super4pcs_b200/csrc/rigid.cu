// a6 -- Match4PCSBase::ComputeRigidTransformation (reference algorithms/match4pcsBase.cc:365-500)
// a7 -- Match4PCSBase::TryCongruentSet            (reference algorithms/match4pcsBase.hpp:363-497)
//
// One thread per candidate quad: gather the quad's first three sampled_Q points, build the two
// orthonormal frames, R = Fp^T Fq, singular check, optional Euler bounds, rms of the three
// residuals / 4, T = translate(c1) * R * translate(-c2).  Every Eigen expression of the
// reference is spelled out in the association order its binary evaluates (3-vector redux =
// a0 + (a1 + a2); pinned bit-for-bit against the compiled reference, tests/test_rigid.py).
// Gate-passing candidates (ok && 0 <= rms < 2 delta, hpp:436-439) are compacted with
// warp-aggregated atomics together with their quad index; Verify (verify.cu) runs on the compacted
// list and a packed-key max picks the winner:  key = (count << 32) | (0xFFFFFFFF - quad_index)
// => highest count, ties -> smallest quad index = the reference's strict-'>' first-max rule.
#include "s4g_internal.cuh"
#include <algorithm>
#include <cmath>
#include <vector>

namespace {

struct BaseArgs {
  float3 p0, p1, p2;   // sampled_P[base_id1..3]
  float3 c1;           // (b1+b2+b3)/3
  float max_angle;     // radians (already converted like hpp:426), < 0 = off
  float rms_threshold; // distance_factor * delta
};

struct Rigid {
  float R[3][3];
  float3 t;
  float rms;
  bool ok;
  float3 c2;
};

__device__ __forceinline__ float coeff3(const float a[3][3], const float b[3][3], int i, int j) {
  return s4_sum3(__fmul_rn(a[i][0], b[0][j]), __fmul_rn(a[i][1], b[1][j]), __fmul_rn(a[i][2], b[2][j]));
}
__device__ __forceinline__ float3 mulMV(const float a[3][3], float3 v) {
  return make_float3(s4_sum3(__fmul_rn(a[0][0], v.x), __fmul_rn(a[0][1], v.y), __fmul_rn(a[0][2], v.z)),
                     s4_sum3(__fmul_rn(a[1][0], v.x), __fmul_rn(a[1][1], v.y), __fmul_rn(a[1][2], v.z)),
                     s4_sum3(__fmul_rn(a[2][0], v.x), __fmul_rn(a[2][1], v.y), __fmul_rn(a[2][2], v.z)));
}

// returns false only where the reference returns false; the "return kLargeNumber" exits of a
// bool function (cc:417-434) are ok == true with rms == 1e9.
__device__ void rigid_fit(const BaseArgs& B, float3 q0, float3 q1, float3 q2, Rigid& o) {
  const float kLarge = 1e9f;
  o.rms = kLarge;
  o.ok = true;
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) o.R[i][j] = 0.f;
  o.t = make_float3(0.f, 0.f, 0.f);
  o.c2 = s4_div(s4_add(s4_add(q0, q1), q2), 3.f);          // hpp:415-417

  float3 vp1 = s4_sub(B.p1, B.p0);                          // cc:415
  if (s4_sqnorm(vp1) == 0.f) return;
  vp1 = s4_normalized(vp1);
  float3 d = s4_sub(B.p2, B.p0);
  float3 vp2 = s4_sub(d, s4_scale(s4_dot(d, vp1), vp1));
  if (s4_sqnorm(vp2) == 0.f) return;
  vp2 = s4_normalized(vp2);
  float3 vp3 = s4_cross(vp1, vp2);
  if (s4_sqnorm(vp3) == 0.f) return;
  vp3 = s4_normalized(vp3);

  float3 vq1 = s4_sub(q1, q0);                              // cc:425
  if (s4_sqnorm(vq1) == 0.f) return;
  vq1 = s4_normalized(vq1);
  float3 e = s4_sub(q2, q0);
  float3 vq2 = s4_sub(e, s4_scale(s4_dot(e, vq1), vq1));
  if (s4_sqnorm(vq2) == 0.f) return;
  vq2 = s4_normalized(vq2);
  float3 vq3 = s4_cross(vq1, vq2);
  if (s4_sqnorm(vq3) == 0.f) return;
  vq3 = s4_normalized(vq3);

  // frames as rows (cc:439-447); R = rotate_p^T * rotate_q
  float fpt[3][3] = {{vp1.x, vp2.x, vp3.x}, {vp1.y, vp2.y, vp3.y}, {vp1.z, vp2.z, vp3.z}};
  float fq[3][3] = {{vq1.x, vq1.y, vq1.z}, {vq2.x, vq2.y, vq2.z}, {vq3.x, vq3.y, vq3.z}};
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) o.R[i][j] = coeff3(fpt, fq, i, j);

  // cc:453: ((R*R).diagonal() - 1 > 1e-6).any()
#pragma unroll
  for (int i = 0; i < 3; ++i)
    if (__fsub_rn(coeff3(o.R, o.R, i, i), 1.f) > 1e-6f) { o.ok = false; return; }

  if (B.max_angle >= 0.f) {                                 // cc:457-472 (non-default option)
    // the reference evaluates these in float via libm; device atan2f differs by <= 2 ulp,
    // which only matters within 2 ulp of the bound (documented in DESIGN.md)
    bool ok = fabsf(atan2f(o.R[2][1], o.R[2][2])) <= B.max_angle &&
              fabsf(atan2f(-o.R[2][0], __fsqrt_rn(__fadd_rn(__fmul_rn(o.R[2][1], o.R[2][1]),
                                                           __fmul_rn(o.R[2][2], o.R[2][2]))))) <= B.max_angle &&
              fabsf(atan2f(o.R[1][0], o.R[0][0])) <= B.max_angle;
    if (!ok) { o.ok = false; return; }
  }

  float rms = 0.f;                                          // cc:477-489
  const float3 qs[3] = {q0, q1, q2};
  const float3 ps[3] = {B.p0, B.p1, B.p2};
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    float3 first = s4_sub(qs[i], o.c2);                     // scaleEst == 1
    float3 tr = mulMV(o.R, first);
    float3 r = s4_add(s4_sub(tr, ps[i]), B.c1);
    rms = __fadd_rn(rms, __fsqrt_rn(s4_sqnorm(r)));
  }
  o.rms = __fdiv_rn(rms, 4.f);                              // / ref.size()
  // translation = c1 + R * (-c2)   (cc:491-497)
  o.t = s4_add(B.c1, mulMV(o.R, make_float3(-o.c2.x, -o.c2.y, -o.c2.z)));
}

// rigid fit of quad qd; returns whether it passes the gate.  A quad with an index outside sampled Q is not fitted
// (r.ok == false, r.rms == -1).
__device__ __forceinline__ bool fit_quad(const BaseArgs& B, const float4* __restrict__ Q, int nQ, int4 qd, Rigid& r) {
  r.ok = false;
  r.rms = -1.f;
  bool inb = (unsigned)qd.x < (unsigned)nQ && (unsigned)qd.y < (unsigned)nQ && (unsigned)qd.z < (unsigned)nQ &&
             (unsigned)qd.w < (unsigned)nQ;
  if (!inb) return false;
  float3 q0 = s4_xyz(__ldg(&Q[qd.x])), q1 = s4_xyz(__ldg(&Q[qd.y])), q2 = s4_xyz(__ldg(&Q[qd.z]));
  rigid_fit(B, q0, q1, q2, r);
  return r.ok && r.rms >= 0.f && r.rms < B.rms_threshold;  // hpp:436-439
}

// warp-aggregated append of the warp's gate-passing candidates (every lane calls it): quad index i, the Verify record
// (row-major 3x4 + what Verify derives from it) and the rms go to the next free slots of the compacted list
__device__ __forceinline__ void append_candidate(bool pass, uint32_t i, const Rigid& r, const VerifyRecArgs& ra,
                                                 uint32_t* __restrict__ nCand, uint32_t* __restrict__ candIdx,
                                                 VerifyCand* __restrict__ outRec, float* __restrict__ outRms) {
  unsigned b = __ballot_sync(0xffffffffu, pass);
  if (b == 0u) return;
  int lane = threadIdx.x & 31;
  int leader = __ffs(b) - 1;
  uint32_t base = 0;
  if (lane == leader) base = atomicAdd(nCand, (uint32_t)__popc(b));
  base = __shfl_sync(0xffffffffu, base, leader);
  if (pass) {
    uint32_t slot = base + __popc(b & ((1u << lane) - 1u));
    candIdx[slot] = i;
    float m[12] = {r.R[0][0], r.R[0][1], r.R[0][2], r.t.x, r.R[1][0], r.R[1][1], r.R[1][2], r.t.y,
                   r.R[2][0], r.R[2][1], r.R[2][2], r.t.z};
    s4g_verify_record(m, ra, &outRec[slot]);
    outRms[slot] = r.rms;
  }
}

// packed arg-max key of a verified candidate (see the top of this file)
__device__ __forceinline__ unsigned long long cand_key(uint32_t count, uint32_t index) {
  return ((unsigned long long)count << 32) | (unsigned long long)(0xFFFFFFFFu - index);
}

// mode 0: write dense outputs (T16 column-major, rms, ok) for every quad (s4g_rigid_batch)
// mode 1: compact gate-passing candidates (append_candidate)
template <int kMode>
__global__ void k_rigid(BaseArgs B, const float4* __restrict__ Q, int nQ, const int4* __restrict__ quads,
                        long long K, int shard_rank, int shard_world, float* __restrict__ outT,
                        float* __restrict__ outRms, int* __restrict__ outOk, uint32_t* __restrict__ candIdx,
                        uint32_t* __restrict__ nCand, VerifyRecArgs ra, VerifyCand* __restrict__ outRec) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  bool active = i < K;
  if (kMode == 1 && active && shard_world > 1) active = (i % shard_world) == shard_rank;
  Rigid r;
  bool pass = active && fit_quad(B, Q, nQ, quads[i], r);
  if (kMode == 0) {
    if (!active) return;
    float* T = outT ? outT + i * 16 : nullptr;
    if (T) {
      // column-major; a rejected candidate leaves the zero matrix the harness passes in
      bool filled = r.ok && r.rms < 1e9f;
#pragma unroll
      for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int rr = 0; rr < 3; ++rr) T[4 * c + rr] = filled ? r.R[rr][c] : 0.f;
      T[3] = T[7] = T[11] = 0.f;
      T[12] = filled ? r.t.x : 0.f;
      T[13] = filled ? r.t.y : 0.f;
      T[14] = filled ? r.t.z : 0.f;
      T[15] = filled ? 1.f : 0.f;
    }
    if (outRms) outRms[i] = r.rms;
    if (outOk) outOk[i] = r.ok ? 1 : 0;
    return;
  }
  append_candidate(pass, (uint32_t)i, r, ra, nCand, candIdx, outRec, outRms);
}

// packed-key arg-max over n verified candidates (*nCand when given); the key's index is index[i] (nullptr: i)
__global__ void k_argmax(const uint32_t* __restrict__ counts, const uint32_t* __restrict__ index,
                         const uint32_t* __restrict__ nCand, uint32_t n, unsigned long long* __restrict__ best) {
  if (nCand) n = *nCand;
  unsigned long long key = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    unsigned long long k = cand_key(counts[i], index ? index[i] : i);
    key = k > key ? k : key;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
    key = other > key ? other : key;
  }
  if ((threadIdx.x & 31) == 0 && key) atomicMax(best, key);
}

// the result record of one congruent set from its arg-max key: the candidates are candIdx[0, n) (with their Verify
// records and rms), the key's quad index counts from quads[quadOff], gate = the set's gate-passing candidates.
// Grid-stride over the candidates: the thread that holds the winner writes its part.
__device__ __forceinline__ void write_result(unsigned long long key, uint32_t gate, int nQ, const BaseArgs& B,
                                             const uint32_t* __restrict__ candIdx, uint32_t n,
                                             const VerifyCand* __restrict__ recs, const float* __restrict__ rms,
                                             const float4* __restrict__ Q, const int4* __restrict__ quads,
                                             uint32_t quadOff, s4g_tcs_result* __restrict__ out) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    out->key = key;
    out->n_gate_pass = gate;
    out->n_q = (uint32_t)nQ;
    out->centroid1[0] = B.c1.x; out->centroid1[1] = B.c1.y; out->centroid1[2] = B.c1.z;
    if (key == 0ull) {
      out->best_count = 0;
      out->best_index = -1;
      out->best_rms = -1.f;
      for (int i = 0; i < 16; ++i) out->best_T[i] = (i % 5 == 0) ? 1.f : 0.f;
      out->centroid2[0] = out->centroid2[1] = out->centroid2[2] = 0.f;
      out->best_quad[0] = out->best_quad[1] = out->best_quad[2] = out->best_quad[3] = 0;
    }
  }
  if (key == 0ull) return;
  const uint32_t widx = 0xFFFFFFFFu - (uint32_t)(key & 0xFFFFFFFFull);
  const uint32_t target = quadOff + widx;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (candIdx[i] == target) {
      const float* T = recs[i].T;
      out->best_count = (uint32_t)(key >> 32);
      out->best_index = (int32_t)widx;
      out->best_rms = rms[i];
      // row-major 3x4 -> column-major 4x4
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 4; ++c) out->best_T[4 * c + r] = T[4 * r + c];
      out->best_T[3] = out->best_T[7] = out->best_T[11] = 0.f;
      out->best_T[15] = 1.f;
      const int4 qd = quads[target];
      float3 c2 = s4_div(s4_add(s4_add(s4_xyz(Q[qd.x]), s4_xyz(Q[qd.y])), s4_xyz(Q[qd.z])), 3.f);
      out->centroid2[0] = c2.x; out->centroid2[1] = c2.y; out->centroid2[2] = c2.z;
      out->best_quad[0] = qd.x; out->best_quad[1] = qd.y; out->best_quad[2] = qd.z; out->best_quad[3] = qd.w;
    }
  }
}

// find the compacted slot of the winner and assemble the result record
__global__ void k_finish(const uint32_t* __restrict__ candIdx, const uint32_t* __restrict__ nCand,
                         const VerifyCand* __restrict__ recs, const float* __restrict__ rms,
                         const unsigned long long* __restrict__ best, BaseArgs B,
                         const float4* __restrict__ Q, const int4* __restrict__ quads, int nQ,
                         s4g_tcs_result* __restrict__ out) {
  const uint32_t n = *nCand;
  write_result(*best, n, nQ, B, candIdx, n, recs, rms, Q, quads, 0u, out);
}

BaseArgs make_base(const float* b, float max_angle_deg, float rms_threshold) {
  BaseArgs B;
  B.p0 = make_float3(b[0], b[1], b[2]);
  B.p1 = make_float3(b[3], b[4], b[5]);
  B.p2 = make_float3(b[6], b[7], b[8]);
  // (b1 + b2 + b3) / 3 in float, hpp:385 (host IEEE float ops == device _rn ops)
  volatile float sx = B.p0.x + B.p1.x, sy = B.p0.y + B.p1.y, sz = B.p0.z + B.p1.z;
  sx = sx + B.p2.x; sy = sy + B.p2.y; sz = sz + B.p2.z;
  B.c1 = make_float3(sx / 3.f, sy / 3.f, sz / 3.f);
  static const double pi = std::acos(-1);
  // options_.max_angle * pi / 180.0 is a double narrowed to the Scalar parameter, hpp:426
  B.max_angle = (float)((double)max_angle_deg * pi / 180.0);
  B.rms_threshold = rms_threshold;
  return B;
}

}  // namespace

// ============================================================================================
// f1: TryCongruentSet of B bases at once (s4g_try_bases).  The shared quad list is ordered by (base, id, i); the base of
// quad t is the prefix of its key, its first quad quadOff[base].  Rigid fit + gate compacts the candidates of ALL bases
// into one list, ONE Verify launch counts them (the candidate count stays on the device), the arg-max is taken per
// base with the quad index LOCAL to the base (= the per-base chain's key), and B result records are read back.
// ============================================================================================
namespace {

__global__ void k_brigid(const BaseArgs* __restrict__ args, const float4* __restrict__ Q, int nQ, const int4* __restrict__ quads,
                         const unsigned long long* __restrict__ qkeys, long long K, VerifyRecArgs ra,
                         VerifyCand* __restrict__ outRec, float* __restrict__ outRms, uint32_t* __restrict__ candIdx,
                         uint32_t* __restrict__ nCand, uint32_t* __restrict__ gateCnt) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  Rigid r;
  bool pass = false;
  uint32_t base = 0;
  if (i < K) {
    base = (uint32_t)(qkeys[i] >> kBatchSegShift);
    pass = fit_quad(args[base], Q, nQ, quads[i], r);
  }
  append_candidate(pass, (uint32_t)i, r, ra, nCand, candIdx, outRec, outRms);
  if (pass) atomicAdd(&gateCnt[base], 1u);
}

__global__ void k_bargmax(const uint32_t* __restrict__ counts, const uint32_t* __restrict__ candIdx, const uint32_t* __restrict__ nCand,
                          const unsigned long long* __restrict__ qkeys, const uint32_t* __restrict__ quadOff,
                          unsigned long long* __restrict__ best) {
  const uint32_t n = *nCand;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t t = candIdx[i], base = (uint32_t)(qkeys[t] >> kBatchSegShift);
    atomicMax(&best[base], cand_key(counts[i], t - quadOff[base]));
  }
}

// blockIdx.y = base; the key's quad index is local to the base
__global__ void k_bfinish(const uint32_t* __restrict__ candIdx, const uint32_t* __restrict__ nCand, const VerifyCand* __restrict__ recs,
                          const float* __restrict__ rms, const unsigned long long* __restrict__ best, const BaseArgs* __restrict__ args,
                          const float4* __restrict__ Q, const int4* __restrict__ quads, const uint32_t* __restrict__ quadOff,
                          const uint32_t* __restrict__ gateCnt, int nQ, s4g_base_result* __restrict__ outs) {
  const int base = blockIdx.y;
  write_result(best[base], gateCnt[base], nQ, args[base], candIdx, *nCand, recs, rms, Q, quads, quadOff[base],
               &outs[base].tcs);
}

}  // namespace

int s4g_batch_tcs(s4g_ctx* ctx, const s4g_base_desc* bases, float max_angle_deg, float rms_threshold, BatchHost& bh,
                  s4g_base_result* out) {
  cudaStream_t st = ctx->stream;
  const int B = bh.B;
  const long long K = (long long)bh.nQuads;
  std::vector<BaseArgs> args((size_t)B);
  for (int b = 0; b < B; ++b) args[(size_t)b] = make_base(bases[b].base_xyz_p, max_angle_deg, rms_threshold);
  S4G_TRY(s4g_reserve(ctx, ctx->bArgs, std::max<size_t>(args.size() * sizeof(BaseArgs), 64 * 1024)));
  S4G_TRY(s4g_reserve(ctx, ctx->bMisc, 4096));
  S4G_TRY(s4g_reserve(ctx, ctx->bResults, (size_t)kBatchMaxBases * sizeof(s4g_base_result)));
  S4G_TRY(s4g_reserve(ctx, ctx->bCounts, 4096));
  uint32_t* d_quadOff = ctx->bMisc.as<uint32_t>() + 256;            // written by the quad stage
  // bCounts: [0] nCand (uint32), [64..] gate counters (uint32 x B), [512 bytes ..] best keys (uint64 x B)
  uint32_t* d_nCand = ctx->bCounts.as<uint32_t>();
  uint32_t* d_gate = d_nCand + 16;
  unsigned long long* d_best = ctx->bCounts.as<unsigned long long>() + 64;
  S4G_CUDA(cudaMemsetAsync(ctx->bCounts.p, 0, 4096, st));
  S4G_CUDA(cudaMemsetAsync(ctx->bResults.p, 0, (size_t)B * sizeof(s4g_base_result), st));
  S4G_CUDA(cudaMemcpyAsync(ctx->bArgs.p, args.data(), args.size() * sizeof(BaseArgs), cudaMemcpyHostToDevice, st));
  if (K == 0) S4G_CUDA(cudaMemcpyAsync(d_quadOff, bh.quadOff, (size_t)(B + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  const long long cap = std::max<long long>(K, 1);
  S4G_TRY(s4g_reserve(ctx, ctx->dVrec, (size_t)cap * sizeof(VerifyCand)));
  S4G_TRY(s4g_reserve(ctx, ctx->dRms, (size_t)cap * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dCandIdx, (size_t)cap * sizeof(uint32_t)));
  S4G_TRY(s4g_reserve(ctx, ctx->dCounts, (size_t)cap * sizeof(uint32_t)));
  const BaseArgs* d_args = ctx->bArgs.as<BaseArgs>();
  if (K > 0) {
    const unsigned long long* qk = ctx->bQuadKeys[1].as<unsigned long long>();
    S4G_EV_START(ctx, S4G_EV_RIGID);
    k_brigid<<<(unsigned)((K + 127) / 128), 128, 0, st>>>(d_args, ctx->dQ.as<float4>(), ctx->nQ, ctx->bQuads.as<int4>(), qk, K,
                                                         s4g_verify_rec_args(ctx), ctx->dVrec.as<VerifyCand>(), ctx->dRms.as<float>(),
                                                         ctx->dCandIdx.as<uint32_t>(), d_nCand, d_gate);
    S4G_EV_STOP(ctx, S4G_EV_RIGID);
    // Verify over the compacted candidates of all bases; their number stays on the device (K quads is the upper bound)
    if (K <= 0x7fffffffll) {
      S4G_TRY(s4g_launch_verify(ctx, ctx->dVrec.as<VerifyCand>(), (int)K, ctx->dCounts.as<uint32_t>(), true, d_nCand));
    } else {                                                        // beyond Verify's int K: the count has to come to the host
      uint32_t nCand = 0;
      S4G_CUDA(cudaMemcpyAsync(&nCand, d_nCand, sizeof nCand, cudaMemcpyDeviceToHost, st));
      S4G_CUDA(cudaStreamSynchronize(st));
      if (nCand > 0x7fffffffu) { ctx->err = "s4g_try_bases: more than 2^31-1 gate-passing quads in one call"; return S4G_ERR_NOMEM; }
      S4G_TRY(s4g_launch_verify(ctx, ctx->dVrec.as<VerifyCand>(), (int)nCand, ctx->dCounts.as<uint32_t>(), true, nullptr));
    }
    k_bargmax<<<64, 256, 0, st>>>(ctx->dCounts.as<uint32_t>(), ctx->dCandIdx.as<uint32_t>(), d_nCand, qk, d_quadOff, d_best);
    ctx->launches += 2;
  }
  k_bfinish<<<dim3(K > 0 ? 32 : 1, (unsigned)B, 1), 256, 0, st>>>(ctx->dCandIdx.as<uint32_t>(), d_nCand, ctx->dVrec.as<VerifyCand>(),
                                                                  ctx->dRms.as<float>(), d_best, d_args, ctx->dQ.as<float4>(),
                                                                  ctx->bQuads.as<int4>(), d_quadOff, d_gate, ctx->nQ,
                                                                  ctx->bResults.as<s4g_base_result>());
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  S4G_CUDA(cudaMemcpyAsync(out, ctx->bResults.p, (size_t)B * sizeof(s4g_base_result), cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));                              // read-back 3 of 3
  for (int b = 0; b < B; ++b) {
    out[b].n_pairs[0] = bh.segCount[2 * b];
    out[b].n_pairs[1] = bh.segCount[2 * b + 1];
    out[b].n_quads = (int64_t)bh.quadOff[b + 1] - (int64_t)bh.quadOff[b];
  }
  return S4G_OK;
}

extern "C" int s4g_try_bases(s4g_ctx* ctx, const s4g_base_desc* bases, int n_bases, float pair_distance_epsilon,
                             const s4g_pair_filters* filters, float distance_threshold2, float max_angle_deg,
                             float rms_threshold, s4g_base_result* out) {
  if (!ctx) return S4G_ERR_ARG;
  if (!bases || !out || n_bases < 1 || n_bases > kBatchMaxBases) { ctx->err = "s4g_try_bases: need 1..64 bases"; return S4G_ERR_ARG; }
  if (ctx->nP <= 0 || ctx->nQ <= 0) { ctx->err = "s4g_try_bases: call s4g_set_cloud_p and s4g_set_cloud_q first"; return S4G_ERR_STATE; }
  if (ctx->nQ >= (1 << kBatchIdBits)) { ctx->err = "s4g_try_bases: |sampled_Q| must be < 2^26"; return S4G_ERR_ARG; }
  if (!(pair_distance_epsilon > 0.f)) { ctx->err = "s4g_try_bases: need epsilon > 0"; return S4G_ERR_ARG; }
  for (int b = 0; b < n_bases; ++b)
    if (!(bases[b].pair_distance[0] >= 0.f) || !(bases[b].pair_distance[1] >= 0.f)) { ctx->err = "s4g_try_bases: need distance >= 0"; return S4G_ERR_ARG; }
  S4G_CUDA(cudaSetDevice(ctx->device));
  BatchHost bh;
  S4G_TRY(s4g_batch_pairs(ctx, bases, n_bases, pair_distance_epsilon, filters, bh));
  S4G_TRY(s4g_batch_quads(ctx, bases, distance_threshold2, bh));
  return s4g_batch_tcs(ctx, bases, max_angle_deg, rms_threshold, bh, out);
}

extern "C" int s4g_rigid_batch(s4g_ctx* ctx, const float* base_xyz, const int32_t* quads, int64_t K,
                               float max_angle_deg, float* out_T, float* out_rms, int32_t* out_ok) {
  if (!ctx) return S4G_ERR_ARG;
  if (!base_xyz || K < 0 || (K > 0 && !quads)) { ctx->err = "s4g_rigid_batch: bad arguments"; return S4G_ERR_ARG; }
  if (ctx->nQ <= 0) { ctx->err = "s4g_rigid_batch: call s4g_set_cloud_q first"; return S4G_ERR_STATE; }
  if (K == 0) return S4G_OK;
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, (size_t)K * sizeof(int4)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, (size_t)K * 16 * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dRms, (size_t)K * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dOk, (size_t)K * sizeof(int)));
  S4G_CUDA(cudaMemcpyAsync(ctx->dScratchA.p, quads, (size_t)K * sizeof(int4), cudaMemcpyHostToDevice, st));
  BaseArgs B = make_base(base_xyz, max_angle_deg, 0.f);
  S4G_EV_START(ctx, S4G_EV_RIGID);
  k_rigid<0><<<(unsigned)((K + 127) / 128), 128, 0, st>>>(B, ctx->dQ.as<float4>(), ctx->nQ, ctx->dScratchA.as<int4>(), K,
                                                         0, 1, ctx->dScratchB.as<float>(), ctx->dRms.as<float>(),
                                                         ctx->dOk.as<int>(), nullptr, nullptr, VerifyRecArgs{}, nullptr);
  S4G_EV_STOP(ctx, S4G_EV_RIGID);
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  if (out_T) S4G_CUDA(cudaMemcpyAsync(out_T, ctx->dScratchB.p, (size_t)K * 16 * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (out_rms) S4G_CUDA(cudaMemcpyAsync(out_rms, ctx->dRms.p, (size_t)K * sizeof(float), cudaMemcpyDeviceToHost, st));
  if (out_ok) S4G_CUDA(cudaMemcpyAsync(out_ok, ctx->dOk.p, (size_t)K * sizeof(int), cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  return S4G_OK;
}

extern "C" int s4g_try_congruent_set_dev(s4g_ctx* ctx, const float* base_xyz, const int32_t* d_quads, int64_t K,
                                         float max_angle_deg, float rms_threshold, int shard_rank,
                                         int shard_world, s4g_tcs_result* out) {
  if (!ctx) return S4G_ERR_ARG;
  if (!base_xyz || !out || K < 0 || (K > 0 && !d_quads) || shard_world < 1 || shard_rank < 0 ||
      shard_rank >= shard_world) {
    ctx->err = "s4g_try_congruent_set: bad arguments";
    return S4G_ERR_ARG;
  }
  if (ctx->nP <= 0 || ctx->nQ <= 0) {
    ctx->err = "s4g_try_congruent_set: call s4g_set_cloud_p and s4g_set_cloud_q first";
    return S4G_ERR_STATE;
  }
  if (K >= (1ll << 32) - 1) { ctx->err = "s4g_try_congruent_set: K must be < 2^32-1"; return S4G_ERR_ARG; }
  S4G_TRY(s4g_comm_check_shard(ctx, shard_rank, shard_world));
  const bool reduce = s4g_comm_active(ctx, shard_world);  // the shards' winners meet on the device (comm.cu)
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  BaseArgs B = make_base(base_xyz, max_angle_deg, rms_threshold);
  long long cap = shard_world > 1 ? (K + shard_world - 1) / shard_world : K;
  if (cap < 1) cap = 1;
  S4G_TRY(s4g_reserve(ctx, ctx->dVrec, (size_t)cap * sizeof(VerifyCand)));
  S4G_TRY(s4g_reserve(ctx, ctx->dRms, (size_t)cap * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dCandIdx, (size_t)cap * sizeof(uint32_t)));
  S4G_TRY(s4g_reserve(ctx, ctx->dCounts, (size_t)cap * sizeof(uint32_t)));
  S4G_TRY(s4g_reserve(ctx, ctx->dResult, sizeof(s4g_tcs_result) + 64));
  S4G_TRY(s4g_reserve(ctx, ctx->dMisc, 256));
  uint32_t* d_nCand = ctx->dMisc.as<uint32_t>() + 8;
  unsigned long long* d_best = ctx->dMisc.as<unsigned long long>() + 8;
  S4G_CUDA(cudaMemsetAsync(ctx->dMisc.p, 0, 256, st));
  if (reduce) S4G_CUDA(cudaMemsetAsync(ctx->dResult.p, 0, sizeof(s4g_tcs_result), st));  // (padding bytes are summed too)
  uint32_t nCand = 0;
  if (K > 0) {
    S4G_EV_START(ctx, S4G_EV_RIGID);
    k_rigid<1><<<(unsigned)((K + 127) / 128), 128, 0, st>>>(B, ctx->dQ.as<float4>(), ctx->nQ,
                                                           reinterpret_cast<const int4*>(d_quads), K, shard_rank,
                                                           shard_world, nullptr, ctx->dRms.as<float>(), nullptr,
                                                           ctx->dCandIdx.as<uint32_t>(), d_nCand, s4g_verify_rec_args(ctx),
                                                           ctx->dVrec.as<VerifyCand>());
    S4G_EV_STOP(ctx, S4G_EV_RIGID);
    ctx->launches++;
    // the candidate count sizes the Verify grid: one 4-byte readback
    S4G_CUDA(cudaMemcpyAsync(&nCand, d_nCand, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    S4G_CUDA(cudaStreamSynchronize(st));
  }
  if (nCand > 0x7fffffffu) {  // s4g_verify* take `int K`; 2^31 records would be 240 GB anyway
    ctx->err = "s4g_try_congruent_set: more than 2^31-1 gate-passing quads in one call (shard the set)";
    return S4G_ERR_NOMEM;
  }
  if (nCand > 0) {
    S4G_TRY(s4g_launch_verify(ctx, ctx->dVrec.as<VerifyCand>(), (int)nCand, ctx->dCounts.as<uint32_t>(), true, nullptr));
    k_argmax<<<64, 256, 0, st>>>(ctx->dCounts.as<uint32_t>(), ctx->dCandIdx.as<uint32_t>(), d_nCand, 0u, d_best);
    ctx->launches++;
  }
  k_finish<<<64, 256, 0, st>>>(ctx->dCandIdx.as<uint32_t>(), d_nCand, ctx->dVrec.as<VerifyCand>(), ctx->dRms.as<float>(),
                               d_best, B, ctx->dQ.as<float4>(), reinterpret_cast<const int4*>(d_quads), ctx->nQ,
                               ctx->dResult.as<s4g_tcs_result>());
  ctx->launches++;
  S4G_CUDA(cudaGetLastError());
  if (reduce) {
    S4G_TRY(s4g_comm_reduce_result(ctx, d_best, d_best + 1, ctx->dResult.as<s4g_tcs_result>(), st));
    S4G_TRY(s4g_comm_wait(ctx, st));  // with its deadline -- BEFORE the copy: a D2H copy into pageable memory blocks the host
  }
  S4G_CUDA(cudaMemcpyAsync(out, ctx->dResult.p, sizeof(s4g_tcs_result), cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  return S4G_OK;
}

// Verify + first-maximum key (+ the maximum over the ranks of an attached communicator), stream-ordered
extern "C" int s4g_verify_best_dev(s4g_ctx* ctx, const float* d_T, int K, const uint32_t* d_index, uint32_t* d_counts,
                                   uint64_t* d_key) {
  if (!ctx) return S4G_ERR_ARG;
  if (K < 0 || !d_key || (K > 0 && (!d_T || !d_counts))) { ctx->err = "s4g_verify_best_dev: bad arguments"; return S4G_ERR_ARG; }
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  unsigned long long* key = reinterpret_cast<unsigned long long*>(d_key);
  S4G_CUDA(cudaMemsetAsync(key, 0, sizeof(unsigned long long), st));
  if (K > 0) {
    S4G_TRY(s4g_verify_dev(ctx, d_T, K, d_counts));
    k_argmax<<<64, 256, 0, st>>>(d_counts, d_index, nullptr, (uint32_t)K, key);
    ctx->launches++;
    S4G_CUDA(cudaGetLastError());
  }
  if (ctx->comm) S4G_TRY(s4g_comm_max_u64(ctx, key, key, st));
  return S4G_OK;
}

extern "C" int s4g_verify_best(s4g_ctx* ctx, const float* T, int K, const uint32_t* index, uint32_t* counts,
                               uint64_t* out_key) {
  if (!ctx) return S4G_ERR_ARG;
  if (K < 0 || !out_key || (K > 0 && !T)) { ctx->err = "s4g_verify_best: bad arguments"; return S4G_ERR_ARG; }
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, (size_t)(K > 0 ? K : 1) * 16 * sizeof(float)));
  S4G_TRY(s4g_reserve(ctx, ctx->dCounts, (size_t)(K > 0 ? K : 1) * sizeof(uint32_t)));
  S4G_TRY(s4g_reserve(ctx, ctx->dCandIdx, (size_t)(K > 0 ? K : 1) * sizeof(uint32_t)));
  S4G_TRY(s4g_reserve(ctx, ctx->dMisc, 256));
  if (K > 0) {
    S4G_CUDA(cudaMemcpyAsync(ctx->dScratchA.p, T, (size_t)K * 16 * sizeof(float), cudaMemcpyHostToDevice, st));
    if (index) S4G_CUDA(cudaMemcpyAsync(ctx->dCandIdx.p, index, (size_t)K * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
  }
  uint64_t* d_key = ctx->dMisc.as<uint64_t>() + 16;
  S4G_TRY(s4g_verify_best_dev(ctx, ctx->dScratchA.as<float>(), K, index ? ctx->dCandIdx.as<uint32_t>() : nullptr,
                              ctx->dCounts.as<uint32_t>(), d_key));
  if (ctx->comm) S4G_TRY(s4g_comm_wait(ctx, st));  // deadline first: the copies below block the host when `counts` is pageable
  if (K > 0 && counts) S4G_CUDA(cudaMemcpyAsync(counts, ctx->dCounts.p, (size_t)K * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaMemcpyAsync(out_key, d_key, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  S4G_CUDA(cudaStreamSynchronize(st));
  return S4G_OK;
}

extern "C" int s4g_try_congruent_set(s4g_ctx* ctx, const float* base_xyz, const int32_t* quads, int64_t K,
                                     float max_angle_deg, float rms_threshold, int shard_rank, int shard_world,
                                     s4g_tcs_result* out) {
  if (!ctx) return S4G_ERR_ARG;
  if (K < 0 || (K > 0 && !quads)) { ctx->err = "s4g_try_congruent_set: bad arguments"; return S4G_ERR_ARG; }
  S4G_CUDA(cudaSetDevice(ctx->device));
  int32_t* d_quads = nullptr;
  if (K > 0) {
    S4G_TRY(s4g_reserve(ctx, ctx->dScratchD, (size_t)K * sizeof(int4)));
    S4G_CUDA(cudaMemcpyAsync(ctx->dScratchD.p, quads, (size_t)K * sizeof(int4), cudaMemcpyHostToDevice, ctx->stream));
    d_quads = ctx->dScratchD.as<int32_t>();
  }
  return s4g_try_congruent_set_dev(ctx, base_xyz, d_quads, K, max_angle_deg, rms_threshold, shard_rank,
                                   shard_world, out);
}

extern "C" int s4g_try_congruent_set_resident(s4g_ctx* ctx, const float* base_xyz, float max_angle_deg,
                                              float rms_threshold, int shard_rank, int shard_world,
                                              s4g_tcs_result* out) {
  if (!ctx) return S4G_ERR_ARG;
  return s4g_try_congruent_set_dev(ctx, base_xyz, ctx->dQuads.as<int32_t>(), ctx->nQuads, max_angle_deg,
                                   rms_threshold, shard_rank, shard_world, out);
}
