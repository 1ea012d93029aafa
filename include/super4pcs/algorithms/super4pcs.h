// super4pcs-b200: GlobalRegistration::MatchSuper4PCS -- the Super4PCS matcher, with pair
// extraction, congruent-quad enumeration, rigid fitting and LCP verification on the GPU.
// Interface of the reference's src/super4pcs/algorithms/super4pcs.h:56-130.
#ifndef SUPER4PCS_B200_ALGO_SUPER4PCS_H_
#define SUPER4PCS_B200_ALGO_SUPER4PCS_H_

#include <memory>

#include "super4pcs/algorithms/match4pcsBase.h"

namespace GlobalRegistration {

namespace detail {
class PairOrder;  // cpp/pair_order.h: host replay of the reference's pair emission order
}

class MatchSuper4PCS : public Match4PCSBase {
 public:
  using Base = Match4PCSBase;
  using Scalar = typename Base::Scalar;
  using PairsVector = typename Base::PairsVector;

  explicit MatchSuper4PCS(const Match4PCSOptions& options, const Utils::Logger& logger);

  EIGEN_MAKE_ALIGNED_OPERATOR_NEW

  ~MatchSuper4PCS();

 protected:
  /// ordered pairs (j,i),(i,j) of sampled Q at distance pair_distance +- pair_distance_epsilon
  /// (+ the optional normal / colour / translation / angle filters), sorted lexicographically
  void ExtractPairs(Scalar pair_distance, Scalar pair_normals_angle, Scalar pair_distance_epsilon,
                    int base_point1, int base_point2, PairsVector* pairs) const override;

  /// congruent 4-point candidates of the two pair lists, in (index in P_pairs, index in Q_pairs) order
  bool FindCongruentQuadrilaterals(Scalar invariant1, Scalar invariant2, Scalar distance_threshold1,
                                   Scalar distance_threshold2, const PairsVector& P_pairs,
                                   const PairsVector& Q_pairs,
                                   std::vector<Quadrilateral>* quadrilaterals) const override;

  void Initialize(const std::vector<Point3D>& P, const std::vector<Point3D>& Q) override;

  bool TryBaseOnLane(s4g_ctx* lane, const SelectedBase& base, DeviceBest* out) const override;
  bool TryBasesOnLane(s4g_ctx* lane, const std::vector<SelectedBase*>& bases) const override;

  // S4PCS_EXACT_ORDER=1: candidates in the reference's order, so that even candidates with equal inlier counts are
  // resolved like the reference does (cpp/pair_order.h; DESIGN.md section 4)
  void PrepareBaseOrder(Scalar distance1, Scalar distance2, BaseOrder* out) override;
  void SnapshotBaseOrder(BaseOrder* out) const override;
  void RestoreBaseOrder(const BaseOrder& consumed) override;
  void ResolveTies(s4g_ctx* lane, const BaseOrder& order, const int base_ids[4], DeviceBest* best) const override;

 private:
  bool fused_;  ///< false when S4PCS_FUSED=0: every base goes through the three virtual stages
  bool exact_order_ = true;                           ///< resolve equal-count ties in the reference's candidate order (S4PCS_EXACT_ORDER=0 turns the host replay off)
  mutable std::unique_ptr<detail::PairOrder> order_;  ///< replay state (null: not active for the current clouds)
};

}  // namespace GlobalRegistration

#endif  // SUPER4PCS_B200_ALGO_SUPER4PCS_H_
