// a2 + a3 -- MatchSuper4PCS::ExtractPairs (reference algorithms/super4pcs.cc:183-224) with the
// pair predicate of PairCreationFunctor::process (reference algorithms/pairCreationFunctor.h:
// 151-218) and the accelerator's point test HyperSphere::intersectPoint (reference
// accelerators/pairExtraction/intersectionPrimitive.h:154-157, epsilon rounded as in
// intersectionFunctor.h:59-67).
//
// The reference rasterises sphere shells into an octree; here the shell query runs on the
// Morton (grid-hash) order of sampled_Q that s4g_set_cloud_q builds: consecutive runs of 64
// points form "groups" (the leaves), runs of 64 groups form "supergroups", each with a tight
// AABB.  A CTA of 256 threads owns one group A and a slice of the partner groups B >= A: it scans
// the supergroup / group boxes, keeping only boxes whose distance range to AABB(A) meets
// [d-eps, d+eps]; the 64 points of four surviving groups at a time are staged through shared memory
// and every UNORDERED point pair is tested once (squared-distance band into a register mask, survivors
// compacted into a shared queue, then the reference's exact float/double predicate densely); both
// orientations are emitted from that one test, in ONE pass, with warp-aggregated appends (see k_pairs).
// The output order is arbitrary; every consumer sorts the slot (s4g_sort_pairs).
#include "s4g_internal.cuh"
#include <cub/cub.cuh>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace {

constexpr int kGroup = 64;  // points per group == threads per CTA

struct PairArgs {
  float pair_distance, pair_normals_angle, pair_distance_epsilon;
  float nRadius;        // pair_distance / _ratio        (pairCreationFunctor.h:124-129)
  float eps_round_sq;   // SQR(rounded unit-cube epsilon) (intersectionFunctor.h:59-67,126)
  float lo_sq, hi_sq;   // squared pre-filter band (conservative)
  float lo, hi;         // un-squared band for the box tests
  float3 b1_pos, b1_rgb, b2_pos, b2_rgb;
  float3 segment1;      // (base[b2] - base[b1]).normalized(), h:135-143
  float max_normal_difference, max_translation_distance, max_angle, max_color_distance;
  float norm_threshold; // float(0.5 * max_normal_difference * M_PI / 180.0), h:167-168
  float cos_angle_min;  // smallest float x with acosf(x) <= max_angle*pi/180 (host libm), see below
  int use_angle;
};

struct QViews {
  const float4* qm;     // world, Morton order, w = original index
  const float4* qmunit; // unit cube, Morton order
  const float4* qmn;    // normals, Morton order
  const float4* qmrgb;  // rgb, Morton order
  const float4* glo;    // group AABB lo / hi
  const float4* ghi;
  const float4* sglo;   // supergroup AABB
  const float4* sghi;
  int n, nGroups, nSuper;
  int nSplit;           // every group A is served by nSplit CTAs, each owning a slice of the partner groups
};

struct PairPoint {   // everything the predicate needs about one point
  float3 pos, unit, nrm, rgb;
};

// bit 0: emit (j,i); bit 1: emit (i,j); I is the point with the LARGER original index (the
// reference's process(i, j) is only called with i > j, pairCreationFunctor.h:152)
__device__ int pair_exact(const PairArgs& A, const PairPoint& I, const PairPoint& J) {
  // (1) accelerator point test in unit coordinates: SQR(|pos - center| - radius) < SQR(eps)
  {
    float3 d = s4_sub(J.unit, I.unit);
    float dn = __fsub_rn(__fsqrt_rn(s4_sqnorm(d)), A.nRadius);
    if (!(__fmul_rn(dn, dn) < A.eps_round_sq)) return 0;
  }
  // (2) PairCreationFunctor::process(i, j): p = Q_[j], q = Q_[i]
  const float3 p = J.pos, q = I.pos;
  float distance = __fsqrt_rn(s4_sqnorm(s4_sub(q, p)));                       // h:160
  if (fabs((double)distance - (double)A.pair_distance) > (double)A.pair_distance_epsilon) return 0;  // h:162
  if (A.max_normal_difference > 0.f) {                                          // h:165-180
    const float3 pn = J.nrm, qn = I.nrm;
    if (s4_sqnorm(qn) > 0.f && s4_sqnorm(pn) > 0.f) {
      double first = (double)__fsqrt_rn(s4_sqnorm(s4_sub(qn, pn)));
      double second = (double)__fsqrt_rn(s4_sqnorm(s4_add(qn, pn)));
      double pna = (double)A.pair_normals_angle;
      float nd = (float)fmin(fabs(first - pna), fabs(second - pna));
      if (nd > A.norm_threshold) return 0;
    }
  }
  if (A.max_color_distance > 0.f) {                                             // h:182-192
    const float3 pc = J.rgb, qc = I.rgb;
    bool use_rgb = pc.x >= 0.f && qc.x >= 0.f && A.b1_rgb.x >= 0.f && A.b2_rgb.x >= 0.f;
    bool good = __fsqrt_rn(s4_sqnorm(s4_sub(pc, A.b1_rgb))) < A.max_color_distance &&
                __fsqrt_rn(s4_sqnorm(s4_sub(qc, A.b2_rgb))) < A.max_color_distance;
    if (use_rgb && !good) return 0;
  }
  if (A.max_translation_distance > 0.f) {                                       // h:194-200
    bool good = __fsqrt_rn(s4_sqnorm(s4_sub(p, A.b1_pos))) < A.max_translation_distance &&
                __fsqrt_rn(s4_sqnorm(s4_sub(q, A.b2_pos))) < A.max_translation_distance;
    if (!good) return 0;
  }
  if (A.use_angle) {                                                            // h:203-212
    // acos(x) <= theta  <=>  x >= cos_angle_min (acosf is monotone; the threshold float was
    // found on the host with the same libm the reference uses); x > 1 gives NaN -> false.
    float3 seg2 = s4_normalized(s4_sub(q, p));
    float dt = s4_dot(A.segment1, seg2);
    float dtn = s4_dot(A.segment1, make_float3(-seg2.x, -seg2.y, -seg2.z));
    int r = 0;
    if (dt >= A.cos_angle_min && dt <= 1.f) r |= 1;
    if (dtn >= A.cos_angle_min && dtn <= 1.f) r |= 2;
    return r;
  }
  return 3;
}

__device__ __forceinline__ bool box_meets_band(float3 alo, float3 ahi, float4 blo, float4 bhi, float lo, float hi) {
  float gx = fmaxf(0.f, fmaxf(blo.x - ahi.x, alo.x - bhi.x));
  float gy = fmaxf(0.f, fmaxf(blo.y - ahi.y, alo.y - bhi.y));
  float gz = fmaxf(0.f, fmaxf(blo.z - ahi.z, alo.z - bhi.z));
  float fx = fmaxf(bhi.x - alo.x, ahi.x - blo.x);
  float fy = fmaxf(bhi.y - alo.y, ahi.y - blo.y);
  float fz = fmaxf(bhi.z - alo.z, ahi.z - blo.z);
  float dmin2 = gx * gx + gy * gy + gz * gz;
  float dmax2 = fx * fx + fy * fy + fz * fz;
  return dmin2 <= hi * hi * 1.0001f && dmax2 * 1.0001f >= lo * lo;
}

// ---- the shell query ---------------------------------------------------------------------------
// CTA (A, y): group A (64 Morton-consecutive points, in shared memory) against the partner groups B >= A of slice y of
// [A, nGroups) -- every unordered point pair is visited ONCE and both orientations are emitted from it (the exact
// predicate returns both orientation bits).  256 threads:
//   scan   : 256 partner groups per step, one per thread: supergroup box, then group box, against the distance band;
//            survivors are compacted into a shared list (warp ballots + prefix);
//   test   : 4 surviving groups (256 points, one per thread) are staged in shared memory; thread (a = t & 63, s = t >> 6)
//            runs point a against the 64 points of staged group s with the cheap squared-distance band test and records
//            the survivors in a 64-bit register mask (no divergent work in this loop);
//   compact: mask bits -> shared queue of (a, slot) entries (warp scan + one shared atomic per warp);
//   exact  : one queue entry per thread, densely: the reference's unit-cube point test + PairCreationFunctor::process,
//            then a warp-aggregated append of the 0..2 ordered pairs to the output (one global atomic per warp).
// kFill == false counts only.  The output order is arbitrary (atomics): every consumer sorts the slot first
// (s4g_sort_pairs), which is what makes results deterministic.  If the list does not fit `cap` the kernel keeps counting
// and the host re-runs it with a larger buffer.
constexpr int kPT = 256;             // threads per CTA
constexpr int kStage = kPT / kGroup; // partner groups staged per test step (4)
constexpr int kPairQueue = 4096;     // survivor entries per exact step (uint16: slot << 6 | a)
// S4G_PAIRS_TMA=1: the 4 x 1 KB partner groups of a test step are fetched with cp.async.bulk (1-D TMA, one elected
// thread, completion on an mbarrier) into a double buffer, one step ahead of the tests -- instead of one LDG.128 +
// STS per thread followed by a CTA barrier (-DS4G_PAIRS_TMA=0, kept for A/B).  Numbers in DESIGN.md section 3.3.
#ifndef S4G_PAIRS_TMA
#define S4G_PAIRS_TMA 1
#endif

#if S4G_PAIRS_TMA
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
#endif

// kMode 0: count; 1: fill; 2: count + per-point row counts (rows[a] = number of ordered pairs (a, .), test instrument);
// 3: several extractions per launch (s4g_try_bases): blockIdx.z = segment, its arguments come from argsArr, the output
// is ONE list of keys  segment << 52 | first << 26 | second  (pairs = the key array), rows[segment] counts its pairs
template <int kMode>
__global__ void __launch_bounds__(kPT)
k_pairs(QViews V, PairArgs A0, unsigned long long* __restrict__ total, unsigned long long cap, int2* __restrict__ pairs,
        uint32_t* __restrict__ rows, const PairArgs* __restrict__ argsArr) {
  constexpr bool kFill = kMode == 1 || kMode == 3;
  const PairArgs& A = kMode == 3 ? argsArr[blockIdx.z] : A0;
  __shared__ float4 sA[4][kGroup];           // group A: world pos (w = original index) | unit | normal | rgb
#if S4G_PAIRS_TMA
  __shared__ __align__(128) float4 sBuf[2][kPT];   // double-buffered partner points (bulk-copied)
  __shared__ int sStageBuf[2][kStage];
  __shared__ __align__(8) unsigned long long sBar[2];
#else
  __shared__ float4 sB[kPT];                 // staged partner points: world pos, w = original index
  __shared__ int sStageG[kStage];            // the groups staged in sB
#endif
  __shared__ int sList[kPT];                 // surviving partner groups of the current scan step
  __shared__ uint32_t sWarp[kPT / 32];
  __shared__ uint16_t sQueue[kPairQueue];
  __shared__ uint32_t sQn[2];
  const int g = blockIdx.x, y = blockIdx.y;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int a = t & (kGroup - 1), sidx = t >> 6;
  const bool need_n = A.max_normal_difference > 0.f, need_c = A.max_color_distance > 0.f;
  {
    const int ia = g * kGroup + a;
    const bool va = ia < V.n;
    if (sidx == 0) sA[0][a] = va ? V.qm[ia] : make_float4(3.0e38f, 3.0e38f, 3.0e38f, __int_as_float(-1));
    if (sidx == 1) sA[1][a] = va ? V.qmunit[ia] : make_float4(0.f, 0.f, 0.f, 0.f);
    if (sidx == 2) sA[2][a] = (va && need_n) ? V.qmn[ia] : make_float4(0.f, 0.f, 0.f, 0.f);
    if (sidx == 3) sA[3][a] = (va && need_c) ? V.qmrgb[ia] : make_float4(-1.f, -1.f, -1.f, 0.f);
  }
  if (t < 2) sQn[t] = 0;
#if S4G_PAIRS_TMA
  if (t == 0) {
    mbar_init(&sBar[0], 1);
    mbar_init(&sBar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  uint32_t par0 = 0, par1 = 0;               // CTA-uniform phase parities of the two buffers
#endif
  const float3 alo = s4_xyz(V.glo[g]), ahi = s4_xyz(V.ghi[g]);
  const long long span = (long long)V.nGroups - g;
  const int gLo = g + (int)(((long long)y * span) / V.nSplit), gHi = g + (int)(((long long)(y + 1) * span) / V.nSplit);
  __syncthreads();
  const float4 a4 = sA[0][a];
  const bool va = __float_as_int(a4.w) >= 0;
  uint32_t cur = 0;                           // CTA-uniform: which queue counter is in use
  unsigned long long my_out = 0;              // ordered pairs this thread produced (count-only mode sums them)

  for (int gb0 = gLo; gb0 < gHi; gb0 += kPT) {        // CTA-uniform loop
    // ---- scan: one partner group per thread
    const int gb = gb0 + t;
    bool keep = false;
    if (gb < gHi) {
      const int sg = gb / kGroup;
      keep = box_meets_band(alo, ahi, V.sglo[sg], V.sghi[sg], A.lo, A.hi) &&
             box_meets_band(alo, ahi, V.glo[gb], V.ghi[gb], A.lo, A.hi);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    __syncthreads();                          // previous step's readers of sList / sWarp are done
    if (lane == 0) sWarp[warp] = (uint32_t)__popc(bal);
    __syncthreads();
    uint32_t before = 0, nList = 0;
#pragma unroll
    for (int w = 0; w < kPT / 32; ++w) {
      const uint32_t c = sWarp[w];
      before += w < warp ? c : 0u;
      nList += c;
    }
    if (keep) sList[before + __popc(bal & ((1u << lane) - 1u))] = gb;
    __syncthreads();

#if S4G_PAIRS_TMA
    // fetch of the test step starting at list position l0 into buffer `buf` (all threads call it; the buffer's previous
    // readers passed a CTA barrier): slots without data get the sentinel from their own thread, the rest arrives by TMA
    auto fetch = [&](uint32_t l0, int buf) {
      const uint32_t li = l0 + (uint32_t)sidx;
      const int gs = li < nList ? sList[li] : -1;
      if (a == 0) sStageBuf[buf][sidx] = gs;
      const int have = gs >= 0 ? min(kGroup, V.n - gs * kGroup) : 0;
      if (a >= have) sBuf[buf][t] = make_float4(3.0e38f, 3.0e38f, 3.0e38f, __int_as_float(-1));
      if (t == 0) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // earlier generic accesses of this buffer before the async writes
        uint32_t bytes[kStage], total = 0;
        int gsk[kStage];
#pragma unroll
        for (int k = 0; k < kStage; ++k) {
          gsk[k] = l0 + k < nList ? sList[l0 + k] : -1;
          bytes[k] = gsk[k] >= 0 ? (uint32_t)min(kGroup, V.n - gsk[k] * kGroup) * 16u : 0u;
          total += bytes[k];
        }
        mbar_expect_tx(&sBar[buf], total);
#pragma unroll
        for (int k = 0; k < kStage; ++k)
          if (bytes[k]) bulk_g2s(&sBuf[buf][k * kGroup], &V.qm[(size_t)gsk[k] * kGroup], bytes[k], &sBar[buf]);
      }
    };
    if (nList) fetch(0, 0);
    __syncthreads();                                   // sStageBuf / sentinel writes of the first fetch
    int buf = 0;
#endif
    for (uint32_t l0 = 0; l0 < nList; l0 += kStage) {  // CTA-uniform loop
#if S4G_PAIRS_TMA
      if (l0 + kStage < nList) fetch(l0 + kStage, buf ^ 1);   // one step ahead (that buffer's readers are past the barrier that ended the last round)
      mbar_wait(&sBar[buf], buf ? par1 : par0);
      if (buf) par1 ^= 1u; else par0 ^= 1u;
      const float4* __restrict__ sB = sBuf[buf];
      const int* __restrict__ sStageG = sStageBuf[buf];
#else
      // ---- stage 4 surviving groups: one point per thread
      {
        const uint32_t li = l0 + (uint32_t)sidx;
        const int gs = li < nList ? sList[li] : -1;
        if (a == 0) sStageG[sidx] = gs;
        const int ib = gs * kGroup + a;
        sB[t] = (gs >= 0 && ib < V.n) ? V.qm[ib] : make_float4(3.0e38f, 3.0e38f, 3.0e38f, __int_as_float(-1));
      }
      __syncthreads();
#endif
      // ---- test: point a against the 64 points of staged group sidx
      unsigned long long mask = 0ull;
      {
        const int gs = sStageG[sidx];
        if (va && gs >= 0) {
          const float4* __restrict__ b = &sB[sidx * kGroup];
          const int jmin = gs == g ? a + 1 : 0;       // diagonal group: each unordered pair once
#pragma unroll 8
          for (int j = 0; j < kGroup; ++j) {
            const float4 b4 = b[j];
            const float dx = a4.x - b4.x, dy = a4.y - b4.y, dz = a4.z - b4.z;
            const float sq = __fadd_rn(__fmul_rn(dx, dx), __fadd_rn(__fmul_rn(dy, dy), __fmul_rn(dz, dz)));
            const bool hit = sq >= A.lo_sq && sq <= A.hi_sq && j >= jmin;
            mask |= hit ? (1ull << j) : 0ull;
          }
        }
      }
      // ---- rounds of { compact survivors -> queue ; exact predicate + emission }
      bool again;
      do {
        if (__any_sync(0xffffffffu, mask != 0ull)) {
          const uint32_t cnt = (uint32_t)__popcll(mask);
          uint32_t incl = cnt;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
          }
          const uint32_t tot = __shfl_sync(0xffffffffu, incl, 31);
          uint32_t base = 0;
          if (lane == 31) base = atomicAdd(&sQn[cur], tot);
          base = __shfl_sync(0xffffffffu, base, 31) + incl - cnt;
          while (mask && base < (uint32_t)kPairQueue) {
            const int j = __ffsll((long long)mask) - 1;
            mask &= mask - 1ull;
            sQueue[base++] = (uint16_t)(((sidx * kGroup + j) << 6) | a);
          }
        }
        again = __syncthreads_or(mask != 0ull) != 0;   // queue complete; leftovers => another round
        const uint32_t n = min(sQn[cur], (uint32_t)kPairQueue);
        if (t == 0) sQn[cur ^ 1u] = 0;
        // ---- exact: one surviving unordered pair per thread
        for (uint32_t i0 = 0; i0 < n; i0 += kPT) {     // CTA-uniform loop
          const uint32_t i = i0 + (uint32_t)t;
          int r = 0, i_orig = 0, j_orig = 0;
          if (i < n) {
            const uint32_t e = sQueue[i];
            const int al = (int)(e & 63u), slot = (int)(e >> 6);
            const float4 pa = sA[0][al], pb = sB[slot];
            const int ibm = sStageG[slot >> 6] * kGroup + (slot & 63);
            PairPoint PA, PB;
            PA.pos = s4_xyz(pa);
            PA.unit = s4_xyz(sA[1][al]);
            PA.nrm = s4_xyz(sA[2][al]);
            PA.rgb = s4_xyz(sA[3][al]);
            PB.pos = s4_xyz(pb);
            PB.unit = s4_xyz(V.qmunit[ibm]);
            PB.nrm = need_n ? s4_xyz(V.qmn[ibm]) : make_float3(0.f, 0.f, 0.f);
            PB.rgb = need_c ? s4_xyz(V.qmrgb[ibm]) : make_float3(-1.f, -1.f, -1.f);
            const int ao = __float_as_int(pa.w), bo = __float_as_int(pb.w);
            // process(i, j) is called with i > j (pairCreationFunctor.h:152): I = the larger original index
            const bool a_is_i = ao > bo;
            r = a_is_i ? pair_exact(A, PA, PB) : pair_exact(A, PB, PA);
            i_orig = a_is_i ? ao : bo;
            j_orig = a_is_i ? bo : ao;
          }
          const int no = (r & 1) + ((r >> 1) & 1);
          my_out += (unsigned long long)no;
          if (kMode == 2) {
            if (r & 2) atomicAdd(&rows[i_orig], 1u);
            if (r & 1) atomicAdd(&rows[j_orig], 1u);
          }
          if (kFill) {
            // warp-aggregated append: bit 0 -> (j, i), bit 1 -> (i, j)   (pairCreationFunctor.h:203-215)
            uint32_t incl = (uint32_t)no;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
              const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
              if (lane >= o) incl += v;
            }
            const uint32_t tot = __shfl_sync(0xffffffffu, incl, 31);
            unsigned long long base = 0;
            if (lane == 31 && tot) base = atomicAdd(total, (unsigned long long)tot);
            base = __shfl_sync(0xffffffffu, base, 31) + incl - (uint32_t)no;
            if (kMode == 3) {
              unsigned long long* __restrict__ keys = reinterpret_cast<unsigned long long*>(pairs);
              const unsigned long long seg = (unsigned long long)blockIdx.z << kBatchSegShift;
              if (lane == 31 && tot) atomicAdd(&rows[blockIdx.z], tot);
              if ((r & 1) && base < cap) keys[base] = seg | ((unsigned long long)j_orig << kBatchIdBits) | (unsigned long long)i_orig;
              if (r & 1) ++base;
              if ((r & 2) && base < cap) keys[base] = seg | ((unsigned long long)i_orig << kBatchIdBits) | (unsigned long long)j_orig;
            } else {
              if ((r & 1) && base < cap) pairs[base] = make_int2(j_orig, i_orig);
              if (r & 1) ++base;
              if ((r & 2) && base < cap) pairs[base] = make_int2(i_orig, j_orig);
            }
          }
        }
        __syncthreads();                               // queue / sB / sStageG free; sQn[cur ^ 1] == 0 visible
        cur ^= 1u;
      } while (again);
#if S4G_PAIRS_TMA
      buf ^= 1;
#endif
    }
  }
  if (!kFill) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) my_out += __shfl_xor_sync(0xffffffffu, my_out, o);
    if (lane == 0 && my_out) atomicAdd(total, my_out);
  }
}

// AABB of every run of `run` consecutive items (float4 points, or lo/hi boxes of the level below)
__global__ void k_group_boxes(const float4* __restrict__ lo_in, const float4* __restrict__ hi_in, int n, int run,
                              float4* __restrict__ lo_out, float4* __restrict__ hi_out, int nOut) {
  int g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31;
  if (g >= nOut) return;
  float3 lo = make_float3(3.0e38f, 3.0e38f, 3.0e38f), hi = make_float3(-3.0e38f, -3.0e38f, -3.0e38f);
  for (int k = lane; k < run; k += 32) {
    int i = g * run + k;
    if (i < n) {
      float4 a = lo_in[i], b = hi_in[i];
      lo.x = fminf(lo.x, a.x); lo.y = fminf(lo.y, a.y); lo.z = fminf(lo.z, a.z);
      hi.x = fmaxf(hi.x, b.x); hi.y = fmaxf(hi.y, b.y); hi.z = fmaxf(hi.z, b.z);
    }
  }
  warp_aabb(lo, hi);
  if (lane == 0) {
    lo_out[g] = make_float4(lo.x, lo.y, lo.z, 0.f);
    hi_out[g] = make_float4(hi.x, hi.y, hi.z, 0.f);
  }
}

__global__ void k_pair_keys(const int2* __restrict__ pairs, long long n, unsigned long long* __restrict__ keys) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int2 p = pairs[i];
  keys[i] = ((unsigned long long)(unsigned)p.x << 32) | (unsigned long long)(unsigned)p.y;
}
__global__ void k_keys_to_pairs(const unsigned long long* __restrict__ keys, long long n, int2* __restrict__ pairs) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned long long k = keys[i];
  pairs[i] = make_int2((int)(k >> 32), (int)(k & 0xffffffffull));
}

// smallest float x in [-1, 1] with (double)acosf(x) <= thr (acosf decreasing); 2.f if none
float cos_threshold_for(double thr) {
  auto ok = [&](float x) { return (double)std::acos(x) <= thr; };
  if (!ok(1.f)) return 2.f;
  if (ok(-1.f)) return -1.f;
  // monotone bisection over the ordered float bit patterns
  auto to_ord = [](float f) { int32_t i; std::memcpy(&i, &f, 4); return i >= 0 ? (int64_t)i : (int64_t)(INT32_MIN) - (int64_t)i; };
  auto from_ord = [](int64_t o) { int32_t i = o >= 0 ? (int32_t)o : (int32_t)((int64_t)INT32_MIN - o); float f; std::memcpy(&f, &i, 4); return f; };
  int64_t lo = to_ord(-1.f), hi = to_ord(1.f);   // ok(lo) false, ok(hi) true
  while (hi - lo > 1) {
    int64_t mid = lo + (hi - lo) / 2;
    if (ok(from_ord(mid))) hi = mid; else lo = mid;
  }
  return from_ord(hi);
}

}  // namespace

// group / supergroup boxes over the Morton order of Q (called by s4g_set_cloud_q's owner)
int s4g_build_pair_index(s4g_ctx* ctx) {
  const int n = ctx->nQ;
  const int nG = (n + kGroup - 1) / kGroup, nS = (nG + kGroup - 1) / kGroup;
  S4G_TRY(s4g_reserve(ctx, ctx->dQgroups, (size_t)(2 * nG + 2 * nS) * sizeof(float4)));
  float4* glo = ctx->dQgroups.as<float4>();
  float4* ghi = glo + nG;
  float4* sglo = ghi + nG;
  float4* sghi = sglo + nS;
  const float4* qm = ctx->dQmorton.as<float4>();
  k_group_boxes<<<(nG + 3) / 4, 128, 0, ctx->stream>>>(qm, qm, n, kGroup, glo, ghi, nG);
  k_group_boxes<<<(nS + 3) / 4, 128, 0, ctx->stream>>>(glo, ghi, nG, kGroup, sglo, sghi, nS);
  ctx->launches += 2;
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;
}

// PairArgs of one ExtractPairs call (everything that needs the host's libm / double arithmetic)
static PairArgs make_pair_args(const s4g_ctx* ctx, float pair_distance, float pair_normals_angle, float eps, const float* b1,
                               const float* b2, const s4g_pair_filters* f) {
  PairArgs A;
  std::memset(&A, 0, sizeof A);
  A.pair_distance = pair_distance;
  A.pair_normals_angle = pair_normals_angle;
  A.pair_distance_epsilon = eps;
  A.nRadius = pair_distance / ctx->ratio;                       // setRadius
  {
    float eps_norm = eps / ctx->ratio;                          // getNormalizedEpsilon
    const int lvlMax = -std::log2(eps_norm);                    // intersectionFunctor.h:60
    float eps_round = 1.f / std::pow(2, lvlMax);
    A.eps_round_sq = eps_round * eps_round;
  }
  double lo = std::max(0.0, (double)pair_distance - (double)eps), hi = (double)pair_distance + (double)eps;
  A.lo = (float)(lo * (1.0 - 1e-5));
  A.hi = (float)(hi * (1.0 + 1e-5));
  A.lo_sq = (float)(lo * lo * (1.0 - 4e-5));
  A.hi_sq = (float)(hi * hi * (1.0 + 4e-5));
  static const float d9[9] = {0, 0, 0, 0, 0, 0, -1, -1, -1};
  if (!b1) b1 = d9;
  if (!b2) b2 = d9;
  A.b1_pos = make_float3(b1[0], b1[1], b1[2]);
  A.b1_rgb = make_float3(b1[6], b1[7], b1[8]);
  A.b2_pos = make_float3(b2[0], b2[1], b2[2]);
  A.b2_rgb = make_float3(b2[6], b2[7], b2[8]);
  {
    // (base[b2].pos - base[b1].pos).normalized() in float, Eigen order (host IEEE == device _rn)
    volatile float dx = b2[0] - b1[0], dy = b2[1] - b1[1], dz = b2[2] - b1[2];
    volatile float yy = dy * dy, zz = dz * dz, xx = dx * dx;
    volatile float yz = yy + zz;
    volatile float z = xx + yz;
    if (z > 0.f) {
      float s = std::sqrt((float)z);
      A.segment1 = make_float3(dx / s, dy / s, dz / s);
    } else {
      A.segment1 = make_float3(dx, dy, dz);
    }
  }
  s4g_pair_filters ff = {-1.f, -1.f, -1.f, -1.f};
  if (f) ff = *f;
  A.max_normal_difference = ff.max_normal_difference;
  A.max_translation_distance = ff.max_translation_distance;
  A.max_angle = ff.max_angle;
  A.max_color_distance = ff.max_color_distance;
  A.norm_threshold = (float)(0.5 * ff.max_normal_difference * M_PI / 180.0);
  A.use_angle = ff.max_angle > 0.f ? 1 : 0;
  A.cos_angle_min = A.use_angle ? cos_threshold_for((double)ff.max_angle * M_PI / 180.0) : -1.f;
  return A;
}

// views of the Morton-ordered Q arrays + the split of every group's partner range; `segments` = extractions per launch
static int make_views(s4g_ctx* ctx, int segments, QViews& V) {
  const int n = ctx->nQ;
  const int nG = (n + kGroup - 1) / kGroup, nS = (nG + kGroup - 1) / kGroup;
  if (ctx->dQgroups.p == nullptr || !ctx->pair_index_ready) {
    S4G_TRY(s4g_build_pair_index(ctx));
    ctx->pair_index_ready = true;
  }
  V.qm = ctx->dQmorton.as<float4>();
  V.qmunit = ctx->dQmside.as<float4>();
  V.qmn = V.qmunit + n;
  V.qmrgb = V.qmn + n;
  V.glo = ctx->dQgroups.as<float4>();
  V.ghi = V.glo + nG;
  V.sglo = V.ghi + nG;
  V.sghi = V.sglo + nS;
  V.n = n;
  V.nGroups = nG;
  V.nSuper = nS;
  // a few waves of CTAs even when the cloud has few groups: the partner range [A, nGroups) of every group is split
  const long long want = (8ll * ctx->sm_count + (long long)nG * segments - 1) / ((long long)nG * segments);
  V.nSplit = (int)std::max(1ll, std::min<long long>(std::min(nG, 64), want));
  return S4G_OK;
}

static int pairs_common(s4g_ctx* ctx, float pair_distance, float pair_normals_angle, float eps, const float* b1,
                        const float* b2, const s4g_pair_filters* f, int slot, bool count_only, int64_t* n_pairs,
                        uint32_t* host_rows = nullptr) {
  if (ctx->nQ <= 0) { ctx->err = "s4g_extract_pairs: call s4g_set_cloud_q first"; return S4G_ERR_STATE; }
  if (!(eps > 0.f) || !(pair_distance >= 0.f)) { ctx->err = "s4g_extract_pairs: need epsilon > 0, distance >= 0"; return S4G_ERR_ARG; }
  S4G_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const int n = ctx->nQ;
  const PairArgs A = make_pair_args(ctx, pair_distance, pair_normals_angle, eps, b1, b2, f);
  QViews V;
  S4G_TRY(make_views(ctx, 1, V));
  const int nG = V.nGroups;

  S4G_TRY(s4g_reserve(ctx, ctx->dMisc, 256));
  unsigned long long* d_total = ctx->dMisc.as<unsigned long long>() + 16;   // byte 128 (TryCongruentSet uses 0..71)
  const dim3 pgrid((unsigned)nG, (unsigned)V.nSplit, 1);
  unsigned long long total = 0;
  S4G_EV_START(ctx, S4G_EV_PAIRS);
  if (count_only) {
    S4G_CUDA(cudaMemsetAsync(d_total, 0, sizeof(unsigned long long), st));
    if (host_rows) {
      S4G_TRY(s4g_reserve(ctx, ctx->dScratchC, (size_t)n * sizeof(uint32_t)));
      S4G_CUDA(cudaMemsetAsync(ctx->dScratchC.p, 0, (size_t)n * sizeof(uint32_t), st));
      k_pairs<2><<<pgrid, kPT, 0, st>>>(V, A, d_total, 0ull, nullptr, ctx->dScratchC.as<uint32_t>(), nullptr);
    } else {
      k_pairs<0><<<pgrid, kPT, 0, st>>>(V, A, d_total, 0ull, nullptr, nullptr, nullptr);
    }
    ctx->launches++;
    S4G_EV_STOP(ctx, S4G_EV_PAIRS);
    S4G_CUDA(cudaGetLastError());
    S4G_CUDA(cudaMemcpyAsync(&total, d_total, sizeof total, cudaMemcpyDeviceToHost, st));
    if (host_rows) S4G_CUDA(cudaMemcpyAsync(host_rows, ctx->dScratchC.p, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    S4G_CUDA(cudaStreamSynchronize(st));
    if (n_pairs) *n_pairs = (int64_t)total;
    return S4G_OK;
  }
  // single pass into the slot's buffer (grow-only, so it fits after the first few bases); if the list does not fit the
  // kernel has still counted it: grow and run once more
  ctx->nPairs[slot] = 0;
  S4G_TRY(s4g_reserve(ctx, ctx->dPairs[slot], (size_t)1 << 20));
  for (int attempt = 0; attempt < 2; ++attempt) {
    const unsigned long long cap = ctx->dPairs[slot].cap / sizeof(int2);
    S4G_CUDA(cudaMemsetAsync(d_total, 0, sizeof(unsigned long long), st));
    k_pairs<1><<<pgrid, kPT, 0, st>>>(V, A, d_total, cap, ctx->dPairs[slot].as<int2>(), nullptr, nullptr);
    ctx->launches++;
    S4G_CUDA(cudaGetLastError());
    S4G_CUDA(cudaMemcpyAsync(&total, d_total, sizeof total, cudaMemcpyDeviceToHost, st));
    S4G_CUDA(cudaStreamSynchronize(st));
    if (total <= cap) break;
    if (total >= (1ull << 32)) { ctx->err = "s4g_extract_pairs: more than 2^32-1 ordered pairs"; return S4G_ERR_NOMEM; }
    S4G_TRY(s4g_reserve(ctx, ctx->dPairs[slot], (size_t)total * sizeof(int2)));
  }
  S4G_EV_STOP(ctx, S4G_EV_PAIRS);
  if (n_pairs) *n_pairs = (int64_t)total;
  ctx->nPairs[slot] = (long long)total;
  ctx->pairs_sorted[slot] = false;
  return S4G_OK;
}

extern "C" int s4g_extract_pairs(s4g_ctx* ctx, float pair_distance, float pair_normals_angle,
                                 float pair_distance_epsilon, const float* base_p1, const float* base_p2,
                                 const s4g_pair_filters* filters, int slot, int64_t* n_pairs) {
  if (!ctx) return S4G_ERR_ARG;
  if (slot < 0 || slot > 1) { ctx->err = "s4g_extract_pairs: slot must be 0 or 1"; return S4G_ERR_ARG; }
  return pairs_common(ctx, pair_distance, pair_normals_angle, pair_distance_epsilon, base_p1, base_p2, filters, slot,
                      false, n_pairs);
}

extern "C" int s4g_count_pairs(s4g_ctx* ctx, float pair_distance, float pair_distance_epsilon, int64_t* n_pairs) {
  if (!ctx) return S4G_ERR_ARG;
  return pairs_common(ctx, pair_distance, 0.f, pair_distance_epsilon, nullptr, nullptr, nullptr, 0, true, n_pairs);
}

// ---- f1: the 2B pair extractions of B bases in ONE launch (blockIdx.z = segment 2b + slot), one shared key list,
// one radix sort that leaves every segment contiguous and in (first, second) order
int s4g_batch_pairs(s4g_ctx* ctx, const s4g_base_desc* bases, int B, float eps, const s4g_pair_filters* f, BatchHost& bh) {
  cudaStream_t st = ctx->stream;
  const int nSeg = 2 * B;
  std::vector<PairArgs> args((size_t)nSeg);
  for (int b = 0; b < B; ++b)
    for (int s = 0; s < 2; ++s)
      args[(size_t)(2 * b + s)] = make_pair_args(ctx, bases[b].pair_distance[s], bases[b].pair_normals_angle[s], eps,
                                                 bases[b].base_p[2 * s], bases[b].base_p[2 * s + 1], f);
  QViews V;
  S4G_TRY(make_views(ctx, nSeg, V));
  S4G_TRY(s4g_reserve(ctx, ctx->bArgs, std::max<size_t>(args.size() * sizeof(PairArgs), 64 * 1024)));
  S4G_TRY(s4g_reserve(ctx, ctx->bCounts, 4096));
  S4G_CUDA(cudaMemcpyAsync(ctx->bArgs.p, args.data(), args.size() * sizeof(PairArgs), cudaMemcpyHostToDevice, st));
  unsigned long long* d_total = ctx->bCounts.as<unsigned long long>();          // [0] total, then 2B uint32 segment counts
  uint32_t* d_seg = reinterpret_cast<uint32_t*>(d_total + 1);
  S4G_TRY(s4g_reserve(ctx, ctx->bPairKeys[0], (size_t)1 << 20));
  const dim3 pgrid((unsigned)V.nGroups, (unsigned)V.nSplit, (unsigned)nSeg);
  struct { unsigned long long total; uint32_t seg[2 * kBatchMaxBases]; } h;
  S4G_EV_START(ctx, S4G_EV_PAIRS);
  for (int attempt = 0; attempt < 2; ++attempt) {
    const unsigned long long cap = ctx->bPairKeys[0].cap / sizeof(unsigned long long);
    S4G_CUDA(cudaMemsetAsync(d_total, 0, 8 + 4 * (size_t)nSeg, st));
    k_pairs<3><<<pgrid, kPT, 0, st>>>(V, PairArgs(), d_total, cap, ctx->bPairKeys[0].as<int2>(), d_seg,
                                      ctx->bArgs.as<PairArgs>());
    ctx->launches++;
    S4G_CUDA(cudaGetLastError());
    S4G_CUDA(cudaMemcpyAsync(&h, d_total, 8 + 4 * (size_t)nSeg, cudaMemcpyDeviceToHost, st));
    S4G_CUDA(cudaStreamSynchronize(st));                                         // read-back 1 of 3
    // the batched quad keys hold a pair's index inside its extraction in 26 bits (base << 52 | id << 26 | i)
    for (int s = 0; s < nSeg; ++s)
      if (h.seg[s] >= (1u << kBatchIdBits)) { ctx->err = "s4g_try_bases: an extraction has 2^26 or more pairs"; return S4G_ERR_ARG; }
    if (h.total <= cap) break;
    if (h.total >= (1ull << 32)) { ctx->err = "s4g_try_bases: more than 2^32-1 ordered pairs in one batch"; return S4G_ERR_NOMEM; }
    S4G_TRY(s4g_reserve(ctx, ctx->bPairKeys[0], (size_t)h.total * sizeof(unsigned long long)));
  }
  bh.B = B;
  bh.nPairs = h.total;
  bh.nPPairs = 0;
  bh.segOff[0] = 0;
  for (int s = 0; s < nSeg; ++s) {
    bh.segCount[s] = h.seg[s];
    bh.segOff[s + 1] = bh.segOff[s] + h.seg[s];
    if ((s & 1) == 0) bh.nPPairs += h.seg[s];
  }
  if (bh.segOff[nSeg] != bh.nPairs) { ctx->err = "s4g_try_bases: internal error (segment counts)"; return S4G_ERR_CUDA; }
  if (bh.nPairs > 1) {
    S4G_TRY(s4g_reserve(ctx, ctx->bPairKeys[1], (size_t)bh.nPairs * sizeof(unsigned long long)));
    int segBits = 1;
    while ((1 << segBits) < nSeg) ++segBits;
    size_t cub_bytes = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, cub_bytes, ctx->bPairKeys[0].as<unsigned long long>(),
                                   ctx->bPairKeys[1].as<unsigned long long>(), (long long)bh.nPairs, 0, kBatchSegShift + segBits, st);
    S4G_TRY(s4g_reserve(ctx, ctx->dCub, cub_bytes));
    cub::DeviceRadixSort::SortKeys(ctx->dCub.p, cub_bytes, ctx->bPairKeys[0].as<unsigned long long>(),
                                   ctx->bPairKeys[1].as<unsigned long long>(), (long long)bh.nPairs, 0, kBatchSegShift + segBits, st);
    ctx->launches++;
  } else if (bh.nPairs == 1) {
    S4G_TRY(s4g_reserve(ctx, ctx->bPairKeys[1], 64));
    S4G_CUDA(cudaMemcpyAsync(ctx->bPairKeys[1].p, ctx->bPairKeys[0].p, 8, cudaMemcpyDeviceToDevice, st));
  }
  S4G_EV_STOP(ctx, S4G_EV_PAIRS);
  S4G_CUDA(cudaGetLastError());
  return S4G_OK;                       // sorted keys: ctx->bPairKeys[1]
}

extern "C" int s4g_count_pairs_rows(s4g_ctx* ctx, float pair_distance, float pair_distance_epsilon, uint32_t* out_rows,
                                    int64_t* n_pairs) {
  if (!ctx) return S4G_ERR_ARG;
  if (!out_rows) { ctx->err = "s4g_count_pairs_rows: null output"; return S4G_ERR_ARG; }
  return pairs_common(ctx, pair_distance, 0.f, pair_distance_epsilon, nullptr, nullptr, nullptr, 0, true, n_pairs, out_rows);
}

// sorts the slot lexicographically by (first, second) in place (device)
int s4g_sort_pairs(s4g_ctx* ctx, int slot) {
  long long n = ctx->nPairs[slot];
  if (n <= 1 || ctx->pairs_sorted[slot]) { ctx->pairs_sorted[slot] = true; return S4G_OK; }
  cudaStream_t st = ctx->stream;
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchA, (size_t)n * sizeof(unsigned long long)));
  S4G_TRY(s4g_reserve(ctx, ctx->dScratchB, (size_t)n * sizeof(unsigned long long)));
  unsigned long long* k0 = ctx->dScratchA.as<unsigned long long>();
  unsigned long long* k1 = ctx->dScratchB.as<unsigned long long>();
  k_pair_keys<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ctx->dPairs[slot].as<int2>(), n, k0);
  int bits = 1;
  while ((1ll << bits) < ctx->nQ && bits < 31) ++bits;
  size_t cub_bytes = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, cub_bytes, k0, k1, (long long)n, 0, 32 + bits, st);
  S4G_TRY(s4g_reserve(ctx, ctx->dCub, cub_bytes));
  cub::DeviceRadixSort::SortKeys(ctx->dCub.p, cub_bytes, k0, k1, (long long)n, 0, 32 + bits, st);
  k_keys_to_pairs<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(k1, n, ctx->dPairs[slot].as<int2>());
  ctx->launches += 4;
  S4G_CUDA(cudaGetLastError());
  ctx->pairs_sorted[slot] = true;
  return S4G_OK;
}

extern "C" int s4g_get_pairs(s4g_ctx* ctx, int slot, int32_t* out_pairs) {
  if (!ctx) return S4G_ERR_ARG;
  if (slot < 0 || slot > 1) { ctx->err = "s4g_get_pairs: slot must be 0 or 1"; return S4G_ERR_ARG; }
  long long n = ctx->nPairs[slot];
  if (n == 0) return S4G_OK;
  if (!out_pairs) { ctx->err = "s4g_get_pairs: null output"; return S4G_ERR_ARG; }
  S4G_CUDA(cudaSetDevice(ctx->device));
  S4G_TRY(s4g_sort_pairs(ctx, slot));
  S4G_CUDA(cudaMemcpyAsync(out_pairs, ctx->dPairs[slot].p, (size_t)n * sizeof(int2), cudaMemcpyDeviceToHost, ctx->stream));
  S4G_CUDA(cudaStreamSynchronize(ctx->stream));
  return S4G_OK;
}

extern "C" int s4g_set_pairs(s4g_ctx* ctx, int slot, const int32_t* pairs, int64_t n) {
  if (!ctx) return S4G_ERR_ARG;
  if (slot < 0 || slot > 1 || n < 0 || (n > 0 && !pairs)) { ctx->err = "s4g_set_pairs: bad arguments"; return S4G_ERR_ARG; }
  if (ctx->nQ <= 0) { ctx->err = "s4g_set_pairs: call s4g_set_cloud_q first"; return S4G_ERR_STATE; }
  for (int64_t i = 0; i < 2 * n; ++i)
    if ((unsigned)pairs[i] >= (unsigned)ctx->nQ) { ctx->err = "s4g_set_pairs: index out of range"; return S4G_ERR_ARG; }
  S4G_CUDA(cudaSetDevice(ctx->device));
  ctx->nPairs[slot] = 0;
  S4G_TRY(s4g_reserve(ctx, ctx->dPairs[slot], (size_t)std::max<int64_t>(n, 1) * sizeof(int2)));
  if (n > 0) {
    S4G_CUDA(cudaMemcpyAsync(ctx->dPairs[slot].p, pairs, (size_t)n * sizeof(int2), cudaMemcpyHostToDevice, ctx->stream));
    S4G_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  ctx->nPairs[slot] = n;
  ctx->pairs_sorted[slot] = true;   // uploaded lists keep the caller's order (ids index into THEM)
  return S4G_OK;
}
