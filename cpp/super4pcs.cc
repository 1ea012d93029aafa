// super4pcs-b200: GlobalRegistration::MatchSuper4PCS on top of the C ABI of include/s4g.h.
// Behavioural contract: reference src/super4pcs/algorithms/super4pcs.cc (ExtractPairs :183-224,
// FindCongruentQuadrilaterals :80-177, Initialize :230-234).
#include "super4pcs/algorithms/super4pcs.h"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>

#include "pair_order.h"
#include "s4g.h"
#include "shards.h"

namespace GlobalRegistration {

namespace {
void Point9(const Point3D& p, float* o) {
  for (int c = 0; c < 3; ++c) {
    o[c] = p.pos()[c];
    o[3 + c] = p.normal()[c];
    o[6 + c] = p.rgb()[c];
  }
}
s4g_pair_filters Filters(const Match4PCSOptions& o) {
  s4g_pair_filters f;
  f.max_normal_difference = o.max_normal_difference;
  f.max_translation_distance = o.max_translation_distance;
  f.max_angle = o.max_angle;
  f.max_color_distance = o.max_color_distance;
  return f;
}
}  // namespace

MatchSuper4PCS::MatchSuper4PCS(const Match4PCSOptions& options, const Utils::Logger& logger)
    : Base(options, logger, 1), fused_(true) {
  if (const char* e = std::getenv("S4PCS_FUSED")) fused_ = std::atoi(e) != 0;
  if (const char* e = std::getenv("S4PCS_EXACT_ORDER")) exact_order_ = std::atoi(e) != 0;
}

MatchSuper4PCS::~MatchSuper4PCS() {}

// The clouds (incl. the unit-cube normalisation the reference's PairCreationFunctor::synch3DContent
// computes here) were uploaded by Match4PCSBase::init; nothing else to prepare.
void MatchSuper4PCS::Initialize(const std::vector<Point3D>&, const std::vector<Point3D>&) {
  order_.reset();
  const size_t kMaxPoints = 50000;  // the replay is sequential host work: O(|sampled Q|) per level and call
  if (!exact_order_ || sampled_Q_3D_.empty() || sampled_Q_3D_.size() > kMaxPoints) return;
  EnsureDevice();
  float norm[5];
  if (s4g_get_q_normalization(gpu_, norm) != S4G_OK) ThrowLaneError(gpu_, "s4g_get_q_normalization");
  std::vector<float> unit(3 * sampled_Q_3D_.size());
  for (size_t i = 0; i < sampled_Q_3D_.size(); ++i)
    for (int c = 0; c < 3; ++c) unit[3 * i + size_t(c)] = (sampled_Q_3D_[i].pos()[c] - norm[c]) / norm[3] + 0.5f;  // worldToUnit
  order_.reset(new detail::PairOrder);
  order_->Reset(unit, norm[3]);
}

void MatchSuper4PCS::PrepareBaseOrder(Scalar distance1, Scalar distance2, BaseOrder* out) {
  out->valid = false;
  if (!order_ || !fused_) return;  // (the generic path replays inside ExtractPairs)
  const Scalar eps = distance_factor * options_.delta;
  order_->Replay(distance1, eps, &out->pos1);
  order_->Replay(distance2, eps, &out->pos2);
  out->state_after = order_->state();
  out->valid = true;
}

void MatchSuper4PCS::SnapshotBaseOrder(BaseOrder* out) const {
  out->valid = bool(order_);
  if (order_) out->state_after = order_->state();
}

void MatchSuper4PCS::RestoreBaseOrder(const BaseOrder& consumed) {
  if (order_ && consumed.valid && consumed.state_after.size() == order_->size()) order_->set_state(consumed.state_after);
}

// `best` is the first candidate with the highest inlier count in the DEVICE's candidate order (sorted pair lists).  The
// reference keeps the first one in ITS order.  Only called for a base that is about to be adopted: all counts of the
// base are recomputed through the staged ABI (quads -> rigid fits -> gate -> Verify), and among the candidates that
// reach best->count the one with the smallest (pair-1 key, pair-2 key) takes over.
void MatchSuper4PCS::ResolveTies(s4g_ctx* lane, const BaseOrder& order, const int base_ids[4], DeviceBest* best) const {
  const long kMaxQuads = 1L << 21;
  if (!order.valid || lane == nullptr || !best->any || best->n_quads <= 1 || best->n_quads > kMaxQuads) return;
  const size_t n = size_t(best->n_quads);
  std::vector<int32_t> quads(4 * n);
  if (s4g_get_quads(lane, quads.data()) != S4G_OK) ThrowLaneError(lane, "s4g_get_quads");
  float base_xyz[12];
  for (int k = 0; k < 4; ++k)
    for (int c = 0; c < 3; ++c) base_xyz[3 * k + c] = sampled_P_3D_[size_t(base_ids[k])].pos()[c];
  std::vector<float> T(16 * n), rms(n);
  std::vector<int32_t> ok(n);
  if (s4g_rigid_batch(lane, base_xyz, quads.data(), int64_t(n), options_.max_angle, T.data(), rms.data(), ok.data()) != S4G_OK)
    ThrowLaneError(lane, "s4g_rigid_batch");
  const float gate = distance_factor * options_.delta;
  std::vector<size_t> passing;
  for (size_t i = 0; i < n; ++i)
    if (ok[i] && rms[i] >= 0.f && rms[i] < gate) passing.push_back(i);
  if (passing.size() <= 1) return;
  std::vector<float> Tg(16 * passing.size());
  for (size_t k = 0; k < passing.size(); ++k) std::memcpy(&Tg[16 * k], &T[16 * passing[k]], 16 * sizeof(float));
  std::vector<uint32_t> counts(passing.size());
  if (s4g_verify(lane, Tg.data(), int(passing.size()), counts.data()) != S4G_OK) ThrowLaneError(lane, "s4g_verify");
  bool have = false;
  size_t winner = 0;
  uint64_t key1 = 0, key2 = 0;
  for (size_t k = 0; k < passing.size(); ++k) {
    if (counts[k] != best->count) continue;
    const int32_t* q = &quads[4 * passing[k]];
    const uint64_t a = detail::PairOrder::Key(order.pos1, q[0], q[1]), b = detail::PairOrder::Key(order.pos2, q[2], q[3]);
    if (!have || a < key1 || (a == key1 && b < key2)) {
      have = true;
      winner = passing[k];
      key1 = a;
      key2 = b;
    }
  }
  if (!have || long(winner) == best->index) return;
  best->index = long(winner);
  std::memcpy(best->quad, &quads[4 * winner], 4 * sizeof(int));
  best->T = Eigen::Map<const MatrixType>(&T[16 * winner]);
  const VectorType &q0 = sampled_Q_3D_[size_t(best->quad[0])].pos(), &q1 = sampled_Q_3D_[size_t(best->quad[1])].pos(),
                   &q2 = sampled_Q_3D_[size_t(best->quad[2])].pos();
  best->centroid2 = (q0 + q1 + q2) / Scalar(3);  // match4pcsBase.hpp:415-417
}

void MatchSuper4PCS::ExtractPairs(Scalar pair_distance, Scalar pair_normals_angle, Scalar pair_distance_epsilon,
                                  int base_point1, int base_point2, PairsVector* pairs) const {
  EnsureDevice();
  pairs->clear();
  float b1[9], b2[9];
  Point9(base_3D_[base_point1], b1);
  Point9(base_3D_[base_point2], b2);
  const s4g_pair_filters f = Filters(options_);
  int64_t n = 0;
  if (s4g_extract_pairs(gpu_, pair_distance, pair_normals_angle, pair_distance_epsilon, b1, b2, &f, 0, &n) != S4G_OK)
    ThrowLaneError(gpu_, "s4g_extract_pairs");
  static_assert(sizeof(std::pair<int, int>) == 2 * sizeof(int), "pair<int,int> must be two packed ints");
  pairs->resize(size_t(n));
  if (n > 0 && s4g_get_pairs(gpu_, 0, reinterpret_cast<int32_t*>(pairs->data())) != S4G_OK)
    ThrowLaneError(gpu_, "s4g_get_pairs");
  if (order_) {  // S4PCS_EXACT_ORDER: hand the list over in the reference's emission order instead of sorted
    std::vector<uint32_t> pos;
    order_->Replay(pair_distance, pair_distance_epsilon, &pos);
    std::sort(pairs->begin(), pairs->end(), [&pos](const std::pair<int, int>& x, const std::pair<int, int>& y) {
      return detail::PairOrder::Key(pos, x.first, x.second) < detail::PairOrder::Key(pos, y.first, y.second);
    });
  }
}

bool MatchSuper4PCS::FindCongruentQuadrilaterals(Scalar invariant1, Scalar invariant2, Scalar /*distance_threshold1*/,
                                                 Scalar distance_threshold2, const PairsVector& P_pairs,
                                                 const PairsVector& Q_pairs,
                                                 std::vector<Quadrilateral>* quadrilaterals) const {
  if (quadrilaterals == nullptr) return false;
  quadrilaterals->clear();
  EnsureDevice();
  if (s4g_set_pairs(gpu_, 0, reinterpret_cast<const int32_t*>(P_pairs.data()), int64_t(P_pairs.size())) != S4G_OK ||
      s4g_set_pairs(gpu_, 1, reinterpret_cast<const int32_t*>(Q_pairs.data()), int64_t(Q_pairs.size())) != S4G_OK)
    ThrowLaneError(gpu_, "s4g_set_pairs");
  float base_xyz[12];
  for (int k = 0; k < 4; ++k)
    for (int c = 0; c < 3; ++c) base_xyz[3 * k + c] = base_3D_[k].pos()[c];
  int64_t n = 0;
  if (s4g_find_quads(gpu_, invariant1, invariant2, distance_threshold2, base_xyz, &n) != S4G_OK)
    ThrowLaneError(gpu_, "s4g_find_quads");
  quadrilaterals->assign(size_t(n), Quadrilateral(0, 0, 0, 0));
  if (n > 0 && s4g_get_quads(gpu_, quadrilaterals->front().vertices.data()) != S4G_OK)
    ThrowLaneError(gpu_, "s4g_get_quads");
  return !quadrilaterals->empty();
}

bool MatchSuper4PCS::TryBaseOnLane(s4g_ctx* lane, const SelectedBase& base, DeviceBest* out) const {
  if (!fused_) return false;
  const Scalar eps = distance_factor * options_.delta;
  const s4g_pair_filters f = Filters(options_);
  float b[4][9];
  for (int k = 0; k < 4; ++k) Point9(base.base3d[k], b[k]);
  float base_xyz[12], basep_xyz[12];  // TryCongruentSet works on sampled_P[base ids] (== base3d after the reordering)
  for (int k = 0; k < 4; ++k)
    for (int c = 0; c < 3; ++c) {
      base_xyz[3 * k + c] = base.base3d[k].pos()[c];
      basep_xyz[3 * k + c] = sampled_P_3D_[base.ids[k]].pos()[c];
    }
  // One pass per device context (S4PCS_DEVICES; a single one by default): pairs and quads are replicated, the
  // candidates of TryCongruentSet are sharded by quad index (SURVEY.md section 8, row e; cpp/shards.h).
  struct Pass {
    int64_t n1 = 0, n2 = 0, nq = 0;
    double ms_pairs1 = 0, ms[5] = {0, 0, 0, 0, 0};
    s4g_tcs_result r = s4g_tcs_result();
  };
  const std::vector<s4g_ctx*>* peers = PeersOf(lane);
  std::vector<Pass> pass(1 + (peers ? peers->size() : 0));
  detail::ShardGate gate(int(pass.size()));  // S4PCS_NCCL: all shards enter the reduction, or none (cpp/shards.h)
  const bool gated = nccl_ && pass.size() > 1;
  detail::ForEachShard(lane, peers, [&](s4g_ctx* ctx, int rank, int world) {
    Pass& p = pass[size_t(rank)];
    const bool timed = timings_ && rank == 0;  // S4PCS_TIMINGS: the events of the context that also holds the result
    if (s4g_extract_pairs(ctx, base.distance1, base.normal_angle1, eps, b[0], b[1], &f, 0, &p.n1) != S4G_OK)
      ThrowLaneError(ctx, "s4g_extract_pairs");
    if (timed && s4g_get_timings(ctx, p.ms) == S4G_OK) p.ms_pairs1 = p.ms[2];  // (the slot-1 call re-uses the event pair)
    if (s4g_extract_pairs(ctx, base.distance2, base.normal_angle2, eps, b[2], b[3], &f, 1, &p.n2) != S4G_OK)
      ThrowLaneError(ctx, "s4g_extract_pairs");
    struct ReadTimings {  // on every way out of this pass
      s4g_ctx* ctx; Pass* p; bool on;
      ~ReadTimings() { if (on) (void)s4g_get_timings(ctx, p->ms); }
    } read_timings{ctx, &p, timed};
    if (p.n1 == 0 || p.n2 == 0) return;
    if (s4g_find_quads(ctx, base.invariant1, base.invariant2, eps, base_xyz, &p.nq) != S4G_OK) ThrowLaneError(ctx, "s4g_find_quads");
    if (p.nq == 0) return;
    if (gated && !gate.Pass(rank)) return;  // a peer left early: its error (or the count check below) reports it
    if (s4g_try_congruent_set_resident(ctx, basep_xyz, options_.max_angle, eps, rank, world, &p.r) != S4G_OK)
      ThrowLaneError(ctx, "s4g_try_congruent_set_resident");
  }, gated ? &gate : nullptr);
  for (const Pass& p : pass)  // replicated stages on identical inputs: anything else is a broken device / context
    if (p.n1 != pass[0].n1 || p.n2 != pass[0].n2 || p.nq != pass[0].nq)
      throw std::runtime_error("super4pcs-b200: S4PCS_DEVICES: the devices disagree on the pair / quad counts of a base");
  out->any = false;
  out->n_pairs[0] = long(pass[0].n1);
  out->n_pairs[1] = long(pass[0].n2);
  if (timings_) {  // s4g_get_timings: [0] Verify, [1] rigid fit, [2] last pair extraction, [3] quads
    const bool quads_ran = pass[0].n1 > 0 && pass[0].n2 > 0, tcs_ran = quads_ran && pass[0].nq > 0;
    out->stage_ms[0] = pass[0].ms_pairs1 + pass[0].ms[2];
    out->stage_ms[1] = quads_ran ? pass[0].ms[3] : 0.0;
    out->stage_ms[2] = tcs_ran ? pass[0].ms[1] : 0.0;
    out->stage_ms[3] = tcs_ran && pass[0].r.n_gate_pass > 0 ? pass[0].ms[0] : 0.0;  // (no survivor: no Verify launch)
  }
  if (pass[0].n1 == 0 || pass[0].n2 == 0) return true;
  out->n_quads = long(pass[0].nq);
  if (pass[0].nq == 0) return true;
  std::vector<s4g_tcs_result> shard;
  for (const Pass& p : pass) shard.push_back(p.r);
  out->SetFrom(detail::CombineShards(shard, nccl_));
  return true;
}

// Row f1, single-launch form: the whole per-base chain of TryBaseOnLane for every base of `bases` in one call of
// s4g_try_bases (base index = grid dimension / key prefix, three read-backs per batch).  Same results per base.
bool MatchSuper4PCS::TryBasesOnLane(s4g_ctx* lane, const std::vector<SelectedBase*>& bases) const {
  if (!fused_ || bases.empty() || bases.size() > 64) return false;
  const Scalar eps = distance_factor * options_.delta;
  const s4g_pair_filters f = Filters(options_);
  std::vector<s4g_base_desc> desc(bases.size());
  for (size_t b = 0; b < bases.size(); ++b) {
    const SelectedBase& sb = *bases[b];
    s4g_base_desc& d = desc[b];
    d.pair_distance[0] = sb.distance1;
    d.pair_distance[1] = sb.distance2;
    d.pair_normals_angle[0] = sb.normal_angle1;
    d.pair_normals_angle[1] = sb.normal_angle2;
    for (int k = 0; k < 4; ++k) {
      Point9(sb.base3d[size_t(k)], d.base_p[k]);
      for (int c = 0; c < 3; ++c) d.base_xyz_p[3 * k + c] = sampled_P_3D_[size_t(sb.ids[k])].pos()[c];
    }
    d.invariant1 = sb.invariant1;
    d.invariant2 = sb.invariant2;
  }
  std::vector<s4g_base_result> res(bases.size());
  const int rc = s4g_try_bases(lane, desc.data(), int(desc.size()), eps, &f, eps, options_.max_angle, eps, res.data());
  // outside the limits of the batched pass (see include/s4g.h), or its shared lists would not fit (> 2^32 pairs / 2^31 quads
  // in one batch, allocation failure): the per-base chain handles it
  if (rc == S4G_ERR_ARG || rc == S4G_ERR_NOMEM) return false;
  if (rc != S4G_OK) ThrowLaneError(lane, "s4g_try_bases");
  for (size_t b = 0; b < bases.size(); ++b) {
    SelectedBase& sb = *bases[b];
    const s4g_base_result& r = res[b];
    DeviceBest& out = sb.best;
    out = DeviceBest();
    out.n_pairs[0] = long(r.n_pairs[0]);
    out.n_pairs[1] = long(r.n_pairs[1]);
    out.n_quads = long(r.n_quads);
    out.SetFrom(r.tcs);
    sb.lane = lane;
    sb.handled = true;
    sb.batched = true;
  }
  if (timings_) {  // S4PCS_TIMINGS: the device time of the batch's stages is booked on its first base (the report sums over bases)
    double ms[5] = {0, 0, 0, 0, 0};
    if (s4g_get_timings(lane, ms) == S4G_OK) {
      DeviceBest& first = bases[0]->best;
      unsigned long long quads = 0, gate = 0;
      for (const s4g_base_result& r : res) { quads += (unsigned long long)r.n_quads; gate += r.tcs.n_gate_pass; }
      first.stage_ms[0] = ms[2];
      first.stage_ms[1] = ms[3];
      first.stage_ms[2] = quads ? ms[1] : 0.0;
      first.stage_ms[3] = gate ? ms[0] : 0.0;
    }
  }
  return true;
}

}  // namespace GlobalRegistration

namespace GlobalRegistration {
namespace Sampling {
namespace detail {

std::size_t GpuSamplerThreshold() {
  if (const char* e = std::getenv("S4PCS_GPU_SAMPLER_MIN")) return std::size_t(std::atoll(e));
  return 200000;
}

void GpuVoxelSample(const float* xyz, std::size_t n, float voxel, std::vector<int>& keep) {
  int device = 0;
  if (const char* e = std::getenv("S4PCS_DEVICE")) device = std::atoi(e);
  s4g_ctx* ctx = nullptr;
  if (s4g_create(device, &ctx) != S4G_OK)
    throw std::runtime_error("super4pcs-b200: voxel sampler: no CUDA device (there is no CPU fallback for large inputs)");
  keep.resize(n);
  int64_t kept = 0;
  const int rc = s4g_voxel_sample(ctx, xyz, int64_t(n), voxel, keep.data(), &kept);
  const std::string msg = rc == S4G_OK ? std::string() : std::string(s4g_error_string(ctx));
  s4g_destroy(ctx);
  if (rc != S4G_OK) throw std::runtime_error("super4pcs-b200: voxel sampler: " + msg);
  keep.resize(std::size_t(kept));
}

}  // namespace detail
}  // namespace Sampling
}  // namespace GlobalRegistration
