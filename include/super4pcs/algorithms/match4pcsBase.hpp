// super4pcs-b200: member templates of Match4PCSBase (the parts that depend on the caller's
// Sampler / Visitor types and therefore have to live in a header, SURVEY.md H6).
// Behavioural contract: reference src/super4pcs/algorithms/match4pcsBase.hpp --
//   ComputeTransformation :61-86, init :90-203, Perform_N_steps :208-274, TryOneBase :281-360,
//   TryCongruentSet :363-497.
// Provenance: init() RESTATES the reference's init (match4pcsBase.hpp:90-203) statement by statement -- sampler calls,
// shuffle, centring, diameter estimate, trial count, log strings -- because RNG consumption, float arithmetic and console
// output are parity-forced (SURVEY.md A.5/A.6); it is host control code, not an independent design.  The device path,
// speculative bases (lanes), candidate sharding and the timings report are new.
#ifndef SUPER4PCS_B200_ALGO_MATCH4PCSBASE_HPP_
#define SUPER4PCS_B200_ALGO_MATCH4PCSBASE_HPP_

#ifndef SUPER4PCS_B200_ALGO_MATCH4PCSBASE_H_
#include "super4pcs/algorithms/match4pcsBase.h"
#endif

#include <algorithm>
#include <chrono>
#include <cmath>
#include <iterator>
#include <type_traits>

namespace GlobalRegistration {

template <typename Sampler, typename Visitor>
Match4PCSBase::Scalar Match4PCSBase::ComputeTransformation(const std::vector<Point3D>& P, std::vector<Point3D>* Q,
                                                           Eigen::Ref<MatrixType> transformation,
                                                           const Sampler& sampler, const Visitor& v) {
  if (Q == nullptr || P.empty() || Q->empty()) return kLargeNumber;
  const std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
#ifdef TEST_GLOBAL_TIMINGS
  timings_ = true;  // the reference's compile-time switch, seen where the CALLER instantiates this template
#endif
  stats_ = StageStats();
  init(P, *Q, sampler);
  if (best_LCP_ != Scalar(1.)) Perform_N_steps(number_of_trials_, transformation, Q, v);
  if (timings_) {
    stats_.ms_total = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    LogTimings();
  }
  return best_LCP_;
}

template <typename Sampler>
void Match4PCSBase::init(const std::vector<Point3D>& P, const std::vector<Point3D>& Q, const Sampler& sampler) {
  const Scalar kSmallError = 0.00001;
  const int kMinNumberOfTrials = 4;
  const Scalar kDiameterFraction = 0.3;

  DiscardSpeculation();
  lanes_stale_ = true;
  batch_now_ = 4;
  centroid_P_ = VectorType::Zero();
  centroid_Q_ = VectorType::Zero();
  sampled_P_3D_.clear();
  sampled_Q_3D_.clear();

  // P: sampled, never truncated.  Q: sampled, shuffled with the member RNG, truncated.
  if (P.size() > options_.sample_size) {
    sampler(P, options_, sampled_P_3D_);
  } else {
    Log<LogLevel::ErrorReport>("(P) More samples requested than available: use whole cloud");
    sampled_P_3D_ = P;
  }
  if (Q.size() > options_.sample_size) {
    std::vector<Point3D> uniform_Q;
    sampler(Q, options_, uniform_Q);
    std::shuffle(uniform_Q.begin(), uniform_Q.end(), randomGenerator_);
    const size_t keep = std::min(uniform_Q.size(), options_.sample_size);
    sampled_Q_3D_.assign(uniform_Q.begin(), uniform_Q.begin() + keep);
  } else {
    Log<LogLevel::ErrorReport>("(Q) More samples requested than available: use whole cloud");
    sampled_Q_3D_ = Q;
  }

  // centre both sampled clouds on their centroids (sequential float accumulation)
  auto centre = [](std::vector<Point3D>& cloud, VectorType& c) {
    for (const Point3D& p : cloud) c += p.pos();
    c /= Scalar(cloud.size());
    for (Point3D& p : cloud) p.pos() -= c;
  };
  centre(sampled_P_3D_, centroid_P_);
  centre(sampled_Q_3D_, centroid_Q_);

  // device-side acceleration structures (replace the reference's kd-tree build)
  UploadClouds();

  // "diameter of P": largest of 1000 random pair distances -- of sampled Q, as in the reference
  P_diameter_ = 0.0;
  for (int i = 0; i < kNumberOfDiameterTrials; ++i) {
    const int at = randomGenerator_() % sampled_Q_3D_.size();
    const int bt = randomGenerator_() % sampled_Q_3D_.size();
    const Scalar l = (sampled_Q_3D_[bt].pos() - sampled_Q_3D_[at].pos()).norm();
    if (l > P_diameter_) P_diameter_ = l;
  }
  // The reference stores MeanDistance() here (hpp:168) and never reads it; P_mean_distance_ keeps the constructor's 1.0
  // and MeanDistance() computes the reference's value when called.
  max_base_diameter_ = P_diameter_;

  // RANSAC trial count for a failure probability of kSmallError
  const Scalar first_estimation =
      std::log(kSmallError) /
      std::log(1.0 - pow(options_.getOverlapEstimation(), static_cast<Scalar>(kMinNumberOfTrials)));
  number_of_trials_ = static_cast<int>(first_estimation * (P_diameter_ / kDiameterFraction) / max_base_diameter_);
  if (number_of_trials_ < kMinNumberOfTrials) number_of_trials_ = kMinNumberOfTrials;

  Log<LogLevel::Verbose>("norm_max_dist: ", options_.delta);
  current_trial_ = 0;
  best_LCP_ = 0.0;
  Q_copy_ = Q;
  for (int i = 0; i < 4; ++i) base_[i] = current_congruent_[i] = 0;
  transform_ = Eigen::Matrix<Scalar, 4, 4>::Identity();

  Initialize(P, Q);

  best_LCP_ = Verify(transform_);
  Log<LogLevel::Verbose>("Initial LCP: ", best_LCP_);
}

template <typename Visitor>
bool Match4PCSBase::Perform_N_steps(int n, Eigen::Ref<MatrixType> transformation, std::vector<Point3D>* Q,
                                    const Visitor& v) {
  using clock = std::chrono::system_clock;
  if (Q == nullptr) return false;

  const Scalar lcp_at_entry = best_LCP_;
  v(0, best_LCP_, transformation);

  bool ok = false;
  const clock::time_point t0 = clock::now();
  for (int i = current_trial_; i < current_trial_ + n; ++i) {
    // bases this call may still try (the loop ends at i == current_trial_ + n - 1 or right after
    // i exceeds number_of_trials_): bounds how far TryOneBase may select ahead
    spec_budget_ = std::max(1, std::min(current_trial_ + n - i, number_of_trials_ + 1 - i));
    ok = TryOneBase(v);

    const Scalar fraction_try = Scalar(i) / Scalar(number_of_trials_);
    // whole seconds / whole seconds: stays 0 until the budget is reached (reference behaviour)
    const Scalar fraction_time =
        std::chrono::duration_cast<std::chrono::seconds>(clock::now() - t0).count() / options_.max_time_seconds;
    const Scalar fraction = std::max(fraction_time, fraction_try);

    if (v.needsGlobalTransformation())
      transformation = GlobalTransform(transform_, qcentroid1_, qcentroid2_);
    else
      transformation = transform_;
    v(fraction, best_LCP_, transformation);

    if (ok || i > number_of_trials_ || fraction >= 0.99 || best_LCP_ == 1.0) break;
  }
  current_trial_ += n;
  spec_budget_ = 1;
  DiscardSpeculation();  // bases selected beyond the last one tried: as if never selected

  if (best_LCP_ > lcp_at_entry) {
    *Q = Q_copy_;
    transformation = GlobalTransform(transform_, qcentroid1_, qcentroid2_);
    for (size_t i = 0; i < Q->size(); ++i)
      (*Q)[i].pos() = (transformation * (*Q)[i].pos().homogeneous()).template head<3>();
  }
  return ok || current_trial_ >= number_of_trials_;
}

// Every base goes through here: select `depth` bases ahead in RNG order (one unless lanes or batches are on and this
// Perform_N_steps call may still try more than one base), run them, then consume the oldest.
template <typename Visitor>
bool Match4PCSBase::TryOneBase(const Visitor& v) {
  if (spec_.empty()) {
    const int depth = SpecDepth() > 1 && spec_budget_ > 1 ? std::min(spec_budget_, NextDepth()) : 1;
    rng_consumed_ = randomGenerator_;  // nothing of these bases consumed yet: a discard restores this state
    SnapshotBaseOrder(&order_consumed_);
    spec_.resize(size_t(depth));
    for (SelectedBase& sb : spec_) SelectBase(&sb);
    try {
      const std::chrono::steady_clock::time_point t_run = std::chrono::steady_clock::now();
      RunSpeculation();
      if (timings_) stats_.ms_passes += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_run).count();
    } catch (...) {  // device / lane set-up failed: leave the matcher as if no base had been selected
      DiscardSpeculation();
      throw;
    }
  }

  SelectedBase sb = std::move(spec_.front());
  spec_.pop_front();
  rng_consumed_ = sb.rng_after;
  if (sb.order.valid) order_consumed_ = sb.order;
  if (!sb.selected) return false;
  base_3D_ = sb.base3d;
  if (sb.error) {
    DiscardSpeculation();
    std::rethrow_exception(sb.error);
  }
  return ConsumeBase(sb, v);
}

template <typename Visitor>
bool Match4PCSBase::ConsumeBase(SelectedBase& sb, const Visitor& v) {
  if (!sb.handled) {  // subclass without a fused device pass (or S4PCS_FUSED=0): the three virtual stages
    std::vector<std::pair<int, int>> pairs1, pairs2;
    std::vector<Quadrilateral> congruent_quads;
    ExtractPairs(sb.distance1, sb.normal_angle1, distance_factor * options_.delta, 0, 1, &pairs1);
    ExtractPairs(sb.distance2, sb.normal_angle2, distance_factor * options_.delta, 2, 3, &pairs2);
    if (pairs1.size() == 0 || pairs2.size() == 0) return false;
    if (!FindCongruentQuadrilaterals(sb.invariant1, sb.invariant2, distance_factor * options_.delta,
                                     distance_factor * options_.delta, pairs1, pairs2, &congruent_quads))
      return false;
    size_t nb = 0;
    return TryCongruentSet(sb.ids[0], sb.ids[1], sb.ids[2], sb.ids[3], congruent_quads, v, nb);
  }

  AccountBase(sb.best);
  if (sb.best.any && Scalar(sb.best.count) / Scalar(sb.best.n_q) > best_LCP_) {
    if (sb.batched && sb.order.valid) {  // the tie resolution works on the base's RESIDENT quads: run this one base again
      DeviceBest again;                  // on the primary context (same result; only for a base about to be adopted)
      TryBaseOnLane(gpu_, sb, &again);
      sb.lane = gpu_;
    }
    ResolveTies(sb.lane, sb.order, sb.ids, &sb.best);
  }
  ReportAndAdopt(sb.ids, sb.best, v);
  // reference hpp:335-347: a base without pairs or without congruent quads returns false (the loop goes on even when
  // best_LCP_ already exceeds the threshold); only TryCongruentSet returns the threshold test
  if (sb.best.n_pairs[0] == 0 || sb.best.n_pairs[1] == 0 || sb.best.n_quads == 0) return false;
  return best_LCP_ > options_.getTerminateThreshold();
}

template <typename Visitor>
void Match4PCSBase::ReportAndAdopt(const int base_ids[4], const DeviceBest& best, const Visitor& v) {
  if (!best.any) return;
  if (!std::is_same<Visitor, DummyTransformVisitor>::value) {
    MatrixType T = best.T;
    if (v.needsGlobalTransformation()) T = GlobalTransform(T, best.centroid1, best.centroid2);
    v(-1, Scalar(best.count) / Scalar(best.n_q), T);
  }
  AdoptIfBetter(base_ids, best);
}

template <typename Visitor>
bool Match4PCSBase::TryCongruentSet(int base_id1, int base_id2, int base_id3, int base_id4,
                                    const std::vector<Quadrilateral>& congruent_quads, const Visitor& v,
                                    size_t& nbCongruent) {
  const int ids[4] = {base_id1, base_id2, base_id3, base_id4};
  DeviceBest best;
  DeviceTryCongruentSet(ids, congruent_quads, &best);
  nbCongruent = best.n_gate_pass;
  // The reference reports every verified candidate; the batched device pass reports the
  // best candidate of the set (callers in the reference tree ignore fraction < 0 reports).
  ReportAndAdopt(ids, best, v);
  return best_LCP_ > options_.getTerminateThreshold();
}

}  // namespace GlobalRegistration

#endif  // SUPER4PCS_B200_ALGO_MATCH4PCSBASE_HPP_
