// super4pcs-b200: GlobalRegistration::Match4PCSBase -- the RANSAC driver of the 4PCS family.
//
// Header-compatible replacement of the reference's src/super4pcs/algorithms/match4pcsBase.h
// (+ match4pcsBase.hpp / .cc): same public entry point (ComputeTransformation, h:108-115), same
// protected extension points (Initialize / ExtractPairs / FindCongruentQuadrilaterals, h:270-326),
// same protected state names (h:120-165) so that Testing::TestMatcher-style subclasses (reference
// tests/testing.h:71-154) compile unchanged.  What is different is underneath: the kd-tree of
// sampled P (reference accelerators/kdtree.h) is replaced by the device grid behind the C ABI of
// include/s4g.h, and every hot stage (pairs, quads, rigid fit, Verify) runs as sm_90a CUDA.
// The host side below keeps the reference's control flow, RNG consumption order (SURVEY.md A.6)
// and float/double mixing (A.1-A.7) so that results are identical on the same inputs.
#ifndef SUPER4PCS_B200_ALGO_MATCH4PCSBASE_H_
#define SUPER4PCS_B200_ALGO_MATCH4PCSBASE_H_

#include <algorithm>
#include <array>
#include <cstdint>
#include <deque>
#include <exception>
#include <map>
#include <random>
#include <utility>
#include <vector>

#include <Eigen/Core>
#include <Eigen/Geometry>

#include "super4pcs/sampling.h"
#include "super4pcs/shared4pcs.h"
#include "super4pcs/utils/logger.h"

struct s4g_ctx;  // include/s4g.h (opaque here: callers need no CUDA headers)
struct s4g_tcs_result;

namespace GlobalRegistration {

class Match4PCSBase {
 public:
  using PairsVector = std::vector<std::pair<int, int>>;
  using Scalar = typename Point3D::Scalar;
  using VectorType = typename Point3D::VectorType;
  using MatrixType = Eigen::Matrix<Scalar, 4, 4>;
  using LogLevel = Utils::LogLevel;
  using DefaultSampler = Sampling::UniformDistSampler;

  /// Visitor concept: operator()(fraction, best_LCP, transform) + needsGlobalTransformation().
  /// fraction >= 0: progress report after every base; fraction == -1: a verified candidate.
  struct DummyTransformVisitor {
    inline void operator()(float, float, Eigen::Ref<Match4PCSBase::MatrixType>) const {}
    constexpr bool needsGlobalTransformation() const { return false; }
  };

  static constexpr int kNumberOfDiameterTrials = 1000;
  static constexpr Scalar kLargeNumber = 1e9;
  static constexpr Scalar distance_factor = 2.0;

  EIGEN_MAKE_ALIGNED_OPERATOR_NEW

  virtual ~Match4PCSBase();

  /// centred sampled clouds used by the registration
  inline const std::vector<Point3D>& getFirstSampled() const { return sampled_P_3D_; }
  inline const std::vector<Point3D>& getSecondSampled() const { return sampled_Q_3D_; }

  /// Approximates the best LCP between P and Q and the rigid motion realising it; on success
  /// Q is replaced by the transformed input.  Returns the LCP in [0,1], or kLargeNumber when Q is
  /// null or either cloud is empty.  Throws std::runtime_error when the GPU path fails.
  template <typename Sampler = DefaultSampler, typename Visitor = DummyTransformVisitor>
  Scalar ComputeTransformation(const std::vector<Point3D>& P, std::vector<Point3D>* Q,
                               Eigen::Ref<MatrixType> transformation, const Sampler& sampler = Sampler(),
                               const Visitor& v = Visitor());

 protected:
  // ---- state (names as in the reference, match4pcsBase.h:120-165)
  int number_of_trials_;
  Scalar max_base_diameter_;
  Scalar P_diameter_;
  Scalar P_mean_distance_;  ///< kept for layout/API; the reference computes but never uses it
  Eigen::Matrix<Scalar, 4, 4> transform_;
  Eigen::Matrix<Scalar, 3, 1> qcentroid1_, qcentroid2_;
  int base_[4];
  int current_congruent_[4];
  std::vector<Point3D> sampled_P_3D_;
  std::vector<Point3D> sampled_Q_3D_;
  std::vector<Point3D> base_3D_;
  std::vector<Point3D> Q_copy_;
  VectorType centroid_P_;
  VectorType centroid_Q_;
  Scalar best_LCP_;
  int current_trial_;
  const Match4PCSOptions options_;
  std::mt19937 randomGenerator_;
  const Utils::Logger& logger_;

  /// device context holding the resident clouds / grids (replaces the reference's kd_tree_)
  mutable s4g_ctx* gpu_ = nullptr;

  /// The trailing int mirrors the reference's OpenMP-only third argument (thread count of the
  /// candidate loop); it has no meaning here.
  Match4PCSBase(const Match4PCSOptions& options, const Utils::Logger& logger, int omp_nthread_congruent = 1);

  template <Utils::LogLevel level, typename... Args>
  inline void Log(Args... args) const { logger_.Log<level>(args...); }

  Scalar MeanDistance();
  bool SelectRandomTriangle(int& base1, int& base2, int& base3);
  bool TryQuadrilateral(Scalar& invariant1, Scalar& invariant2, int& base1, int& base2, int& base3, int& base4);
  bool SelectQuadrilateral(Scalar& invariant1, Scalar& invariant2, int& base1, int& base2, int& base3,
                           int& base4);
  const std::vector<Point3D>& base3D() const { return base_3D_; }

  /// Rigid motion from the first three of four correspondences (host version of the device
  /// kernel; same arithmetic, same results).
  bool ComputeRigidTransformation(const std::array<Point3D, 4>& ref, const std::array<Point3D, 4>& candidate,
                                  const Eigen::Matrix<Scalar, 3, 1>& centroid1,
                                  Eigen::Matrix<Scalar, 3, 1> centroid2, Scalar max_angle,
                                  Eigen::Ref<MatrixType> transform, Scalar& rms_, bool computeScale) const;

  /// LCP of one transform (fraction of sampled Q within delta of sampled P), on the device.
  Scalar Verify(const Eigen::Ref<const MatrixType>& mat) const;

  template <typename Visitor>
  bool Perform_N_steps(int n, Eigen::Ref<MatrixType> transformation, std::vector<Point3D>* Q, const Visitor& v);

  template <typename Visitor>
  bool TryOneBase(const Visitor& v);

  virtual void Initialize(const std::vector<Point3D>& P, const std::vector<Point3D>& Q) = 0;

  template <typename Sampler>
  void init(const std::vector<Point3D>& P, const std::vector<Point3D>& Q, const Sampler& sampler);

  virtual void ExtractPairs(Scalar pair_distance, Scalar pair_normals_angle, Scalar pair_distance_epsilon,
                            int base_point1, int base_point2, PairsVector* pairs) const = 0;

  virtual bool FindCongruentQuadrilaterals(Scalar invariant1, Scalar invariant2, Scalar distance_threshold1,
                                           Scalar distance_threshold2, const PairsVector& P_pairs,
                                           const PairsVector& Q_pairs,
                                           std::vector<Quadrilateral>* quadrilaterals) const = 0;

  template <typename Visitor>
  bool TryCongruentSet(int base_id1, int base_id2, int base_id3, int base_id4,
                       const std::vector<Quadrilateral>& congruent_quads, const Visitor& v, size_t& nbCongruent);

  // ---- device plumbing (new; not part of the reference interface)
  /// outcome of one TryCongruentSet pass on the device
  struct DeviceBest {
    bool any = false;          ///< at least one quad passed the rms gate
    unsigned count = 0;        ///< inliers of the best candidate
    unsigned n_q = 1;
    long index = -1;           ///< its index in the quad list
    int quad[4] = {0, 0, 0, 0};
    size_t n_gate_pass = 0;
    long n_quads = 0;          ///< quads left resident on the lane by this pass
    long n_pairs[2] = {0, 0};  ///< ordered pairs of the two ExtractPairs calls (fused pass)
    double stage_ms[4] = {0, 0, 0, 0};  ///< S4PCS_TIMINGS: device ms of pairs (both calls) / quads / rigid fit / Verify
    Eigen::Matrix<Scalar, 4, 4, Eigen::DontAlign> T;  ///< (unaligned: lives in std containers)
    VectorType centroid1, centroid2;
    /// the winner and the counts of a TryCongruentSet result record; the pair / quad counts and stage times stay as they are
    void SetFrom(const s4g_tcs_result& r);
  };
  /// The ORDER in which the reference would have seen the two pair lists of a base (it does not sort them, its
  /// candidate order -- and the winner among candidates with equal inlier counts -- follows from it; cpp/pair_order.h).
  /// Empty (valid == false) unless a subclass replays that order (MatchSuper4PCS with S4PCS_EXACT_ORDER=1).
  struct BaseOrder {
    bool valid = false;
    std::vector<uint32_t> pos1, pos2;     ///< leaf position of every sampled-Q id for the two ExtractPairs calls
    std::vector<uint32_t> state_after;    ///< the replay's history-dependent state after those calls
  };
  /// main thread, in base order: replay the two ExtractPairs calls of the fused pass
  virtual void PrepareBaseOrder(Scalar /*distance1*/, Scalar /*distance2*/, BaseOrder* /*out*/) {}
  virtual void SnapshotBaseOrder(BaseOrder* /*out*/) const {}
  virtual void RestoreBaseOrder(const BaseOrder& /*consumed*/) {}
  /// main thread, only when `best` is about to be adopted: among the candidates that tie with it, the reference's first
  virtual void ResolveTies(s4g_ctx* /*lane*/, const BaseOrder& /*order*/, const int /*base_ids*/[4], DeviceBest* /*best*/) const {}
  /// rigid fit + gate + Verify + arg-max of explicit quads on the device
  void DeviceTryCongruentSet(const int base_ids[4], const std::vector<Quadrilateral>& quads, DeviceBest* out) const;
  /// keeps the reference's first-maximum rule: adopt `b` only if its LCP beats best_LCP_
  void AdoptIfBetter(const int base_ids[4], const DeviceBest& b);
  void EnsureDevice() const;                       ///< creates gpu_ (throws std::runtime_error)
  void UploadClouds();                             ///< sampled_P/Q -> device (grid, Morton copy, unit cube)
  [[noreturn]] void ThrowLaneError(const s4g_ctx* lane, const char* where) const;
  void UploadCloudsTo(s4g_ctx* ctx) const;
  void UploadCloudsToAll(const std::vector<s4g_ctx*>& contexts) const;  ///< concurrently, one host thread per context
  Eigen::Matrix<Scalar, 4, 4> GlobalTransform(const Eigen::Matrix<Scalar, 4, 4>& centred,
                                              const VectorType& c1, const VectorType& c2) const;

  // ---- per-stage counters: the run-time analogue of the reference's compile-time TEST_GLOBAL_TIMINGS accumulators
  // (match4pcsBase.h:176-184, printed at the end of ComputeTransformation, hpp:77-83).  S4PCS_TIMINGS=1 (or building the
  // caller with -DTEST_GLOBAL_TIMINGS, the reference's switch) adds the device time of every stage -- CUDA events recorded
  // inside libs4g on the stream of the context that ran the base (s4g_get_timings; with S4PCS_DEVICES: rank 0's share) --
  // and the stage output counts over all bases tried, and logs them at LogLevel::Verbose in the reference's frame.
  struct StageStats {
    unsigned long bases = 0;          ///< bases consumed by the RANSAC loop (fused device pass)
    unsigned long long pairs = 0, quads = 0, verified = 0;  ///< stage outputs summed over the bases
    double ms_pairs = 0, ms_quads = 0, ms_rigid = 0, ms_verify = 0;
    double ms_total = 0;              ///< wall clock of ComputeTransformation (host)
    double ms_select = 0;             ///< wall clock inside SelectQuadrilateral (host: RNG, O(|sampled P|) fourth-point scan)
    double ms_passes = 0;             ///< wall clock of the device passes as the host sees them (launches, read-backs, waits)
  };
  bool timings_ = false;
  StageStats stats_;
  void AccountBase(const DeviceBest& b);
  void LogTimings() const;

  // ---- bases selected ahead (SURVEY.md section 8, row f1)
  // The reference tries one base at a time (hpp:236-256); a small sample keeps a GPU idle that
  // way (a base is a handful of tiny kernels and size read-backs).  Base selection depends only on
  // the RNG and on sampled P, and a base's best candidate does not depend on best_LCP_ (hpp:363-497
  // verifies every gate-passing quad), so TryOneBase selects `depth` bases ahead in RNG order, runs
  // them -- one device context ("lane") and one host thread each (S4PCS_LANES, default 1 = off), or
  // one launch chain (S4PCS_BATCH); at depth one, the reference's loop, the per-base chain on gpu_ --
  // and consumes them strictly in order with the reference's adoption and termination checks between
  // bases.  Bases selected beyond the terminating one are discarded and the RNG is put back to the
  // state right after the last consumed base, so that every observable (result, visitor calls, RNG,
  // base_3D_) is the same at any depth.
  struct SelectedBase {
    bool selected = false;   ///< SelectQuadrilateral succeeded
    bool handled = false;    ///< the fused device pass ran (else: the three virtual stages when consumed)
    Scalar invariant1 = 0, invariant2 = 0, distance1 = 0, distance2 = 0, normal_angle1 = 0, normal_angle2 = 0;
    int ids[4] = {0, 0, 0, 0};
    std::vector<Point3D> base3d;
    std::mt19937 rng_after;  ///< RNG state right after this base was selected
    DeviceBest best;
    BaseOrder order;
    s4g_ctx* lane = nullptr;  ///< the context that ran it (its quads stay resident until the next batch)
    bool batched = false;     ///< ran inside one s4g_try_bases launch chain: the lane holds no resident lists of this base
    std::exception_ptr error;
  };
  std::deque<SelectedBase> spec_;        ///< selected, not yet consumed
  std::mt19937 rng_consumed_;            ///< RNG state after the last consumed base
  BaseOrder order_consumed_;             ///< pair-order replay state after the last consumed base
  int spec_budget_ = 1;                  ///< bases the current Perform_N_steps call may still try
  int lane_count_ = 1;
  // Bases per launch chain (s4g_try_bases): S4PCS_BATCH = the maximum (default 32, 1 = off).  Used while the sampled Q cloud
  // has at most S4PCS_BATCH_MAX_Q points (default 4096: the regime where a base is launch- / read-back-bound; beyond it a
  // base's lists are millions of entries and its kernels fill the GPU on their own).  The batches of a run grow 4, 8, 16, ...
  // so that a run that terminates after a few bases does not pay for many speculative ones.
  int batch_ = 32;
  int batch_max_q_ = 4096;
  int batch_now_ = 4;                    ///< size of the next batch (doubles up to batch_)
  bool BatchOn() const { return batch_ > 1 && devices_.size() == 1 && int(sampled_Q_3D_.size()) <= batch_max_q_; }
  int SpecDepth() const { return BatchOn() ? batch_ : lane_count_; }   ///< upper bound of the bases selected ahead
  int NextDepth() {                      ///< bases to select ahead now
    if (!BatchOn()) return lane_count_;
    const int d = std::min(batch_, batch_now_);
    batch_now_ = std::min(batch_, 2 * batch_now_);
    return d;
  }
  /// One fused pass pairs -> quads -> rigid fit -> Verify of `base` entirely on the context `lane`; false (the default):
  /// no fused pass, the base goes through the three virtual stages.  Reads only immutable state (options_,
  /// sampled_P_3D_), so several lanes may run it concurrently from different threads, each on its own context.
  virtual bool TryBaseOnLane(s4g_ctx* lane, const SelectedBase& base, DeviceBest* out) const;
  /// Runs every base of `bases` (selected ahead, in RNG order) in ONE device launch chain on `lane`; fills handled / best /
  /// batched of each.  Returns false when the matcher has no batched device pass (the lanes / per-base chain is used).
  virtual bool TryBasesOnLane(s4g_ctx* lane, const std::vector<SelectedBase*>& bases) const;
  mutable std::vector<s4g_ctx*> lanes_;  ///< extra device contexts (lane 0 is gpu_), same clouds
  bool lanes_stale_ = true;              ///< clouds changed since the lanes were loaded
  void SelectBase(SelectedBase* sb);     ///< the next base in RNG order, with its distances and pair-order replay
  void RunSpeculation();                 ///< runs the selected bases of spec_
  void DiscardSpeculation();             ///< drops unconsumed bases, restores the RNG
  /// the rest of the reference's TryOneBase for a selected base (hpp:317-359): adoption, visitor report, return value
  template <typename Visitor>
  bool ConsumeBase(SelectedBase& sb, const Visitor& v);
  /// visitor report of a best candidate (fraction -1), then AdoptIfBetter
  template <typename Visitor>
  void ReportAndAdopt(const int base_ids[4], const DeviceBest& best, const Visitor& v);

  // ---- candidate-set sharding across the GPUs of one box (SURVEY.md section 8, row e) inside this layer
  // S4PCS_DEVICES = a count ("4": the S4PCS_DEVICE ordinal and the three after it), "all" (every device of the box from
  // S4PCS_DEVICE on) or a list of CUDA ordinals ("0,2,3"; an ordinal may repeat, which shards over several contexts of
  // one GPU).  Default: one device = off.
  // The first device hosts gpu_ and the lanes; every further entry gets a context with the same clouds (a "peer" of
  // the primary context).  A base then runs on all W contexts at once, one host thread each: pairs and quads are
  // replicated (cheap next to Verify), TryCongruentSet takes the quads with index % W == r, and the W shard results
  // are combined by the maximum of the packed (count, ~index) key (cpp/shards.h) -- the reference's first-maximum
  // rule, so every observable is what one device produces.  That maximum is taken on the host by default (W records
  // of 136 bytes that each thread has read back anyway); with S4PCS_NCCL=1 the W contexts share an NCCL communicator
  // (s4g_comm_init_all = ncclCommInitAll) and libs4g reduces key and record on the devices before the one read-back
  // (include/s4g.h, row e) -- every context then returns the same record and this layer only checks that they agree.
  // (Creating the communicator costs more than a small registration: off unless asked for; numbers in DESIGN.md.)
  struct PeerSet {
    std::vector<s4g_ctx*> ctx;  ///< one context per entry of devices_[1..]
    unsigned long epoch = 0;    ///< cloud_epoch_ the contexts were loaded at
    bool comm = false;          ///< S4PCS_NCCL: the communicator over {primary, ctx...} exists
  };
  bool nccl_ = false;                                      ///< S4PCS_NCCL=1
  std::vector<int> devices_;                               ///< CUDA ordinals; [0] = primary (S4PCS_DEVICE)
  mutable std::map<const s4g_ctx*, PeerSet> peers_;        ///< per primary context (gpu_ or a lane)
  unsigned long cloud_epoch_ = 0;                          ///< bumped by UploadClouds
  /// creates / reloads the peers of `primary` (calling thread only, never concurrently); null when sharding is off
  const std::vector<s4g_ctx*>* PreparePeers(const s4g_ctx* primary) const;
  /// lookup only (safe from the lane threads once PreparePeers ran for every primary in use)
  const std::vector<s4g_ctx*>* PeersOf(const s4g_ctx* primary) const;

 private:
  Match4PCSBase(const Match4PCSBase&) = delete;
  Match4PCSBase& operator=(const Match4PCSBase&) = delete;
};

}  // namespace GlobalRegistration

#include "super4pcs/algorithms/match4pcsBase.hpp"

#endif  // SUPER4PCS_B200_ALGO_MATCH4PCSBASE_H_
