// TEST INFRASTRUCTURE ONLY -- never linked into, imported by, or called from the product.
//
// oracle/_ref/liboracle_ref_nearest.so (built by oracle/nearest.py with the reference's Release flags, linked against
// oracle/_ref/liboracle_ref.so): the neighbour the UNMODIFIED reference's Verify looks up and drops
// (match4pcsBase.cc:529-536).  A matcher is initialised on (P, Q) keeping every point, and for each transform and every
// sampled-Q point its own kd_tree_ (built by initKdTree, match4pcsBase.cc:353-363) is asked
// doQueryRestrictedClosestIndex (kdtree.h:388-453) with the query Verify builds.  The protected members are reached
// through a subclass, the pattern of the reference's own tests (tests/testing.h:71-154).
//
// No reference source is copied here: this file only #includes the reference's public headers at build time.
#include "super4pcs/algorithms/super4pcs.h"
#include "super4pcs/accelerators/kdtree.h"
#include "super4pcs/utils/logger.h"

#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>

using namespace GlobalRegistration;

namespace {

struct KeepAll {   // keeps every input point, in input order
  template <typename Point>
  void operator()(const std::vector<Point>& in, const Match4PCSOptions&, std::vector<Point>& out) const { out = in; }
};

class Matcher : public MatchSuper4PCS {
 public:
  Matcher(const Match4PCSOptions& o, const Utils::Logger& l) : MatchSuper4PCS(o, l) {}
  using Match4PCSBase::init;
  using Match4PCSBase::kd_tree_;
  using Match4PCSBase::sampled_P_3D_;
  using Match4PCSBase::sampled_Q_3D_;
};

struct Handle {
  Utils::Logger logger{Utils::NoLog};
  Match4PCSOptions opt;
  Matcher* m = nullptr;
  ~Handle() { delete m; }
};

void fill(std::vector<Point3D>& c, const float* xyz, int n) {
  c.clear();
  for (int i = 0; i < n; ++i) c.emplace_back(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
}

}  // namespace

extern "C" {

// init() on (P, Q) with every point kept (sampling, centring, kd-tree); delta = options.delta
void* nearest_ref_create(const float* Pxyz, int nP, const float* Qxyz, int nQ, float delta) {
  Handle* h = new Handle;
  h->opt.delta = delta;
  h->opt.sample_size = (size_t)nP + (size_t)nQ + 1;
  std::vector<Point3D> P, Q;
  fill(P, Pxyz, nP);
  fill(Q, Qxyz, nQ);
  h->m = new Matcher(h->opt, h->logger);
  h->m->init(P, Q, KeepAll());
  return h;
}

void nearest_ref_destroy(void* hv) { delete static_cast<Handle*>(hv); }

// the centred sampled clouds the matcher works on (nP x 3, nQ x 3)
void nearest_ref_sampled(void* hv, float* P, float* Q) {
  const Matcher* m = static_cast<Handle*>(hv)->m;
  for (size_t i = 0; i < m->sampled_P_3D_.size(); ++i)
    for (int k = 0; k < 3; ++k) P[3 * i + k] = m->sampled_P_3D_[i].pos()[k];
  for (size_t i = 0; i < m->sampled_Q_3D_.size(); ++i)
    for (int k = 0; k < 3; ++k) Q[3 * i + k] = m->sampled_Q_3D_[i].pos()[k];
}

// for K column-major transforms: out_index (K x nQ) = what the kd-tree returns for the query Verify builds (-1: none),
// out_sq = the squared distance to that sampled-P point, computed as the kd-tree's leaf test does (+inf for -1)
void nearest_ref_query(void* hv, const float* T16k, long K, int32_t* out_index, float* out_sq) {
  Handle* h = static_cast<Handle*>(hv);
  const Matcher* m = h->m;
  const long nQ = (long)m->sampled_Q_3D_.size();
  const float epsilon = h->opt.delta;                    // options_.delta, cc:516
  const float sq_eps = epsilon * epsilon;                // cc:522
  for (long c = 0; c < K; ++c) {
    Match4PCSBase::MatrixType T;
    std::memcpy(T.data(), T16k + 16 * c, 16 * sizeof(float));
    const Eigen::Ref<const Match4PCSBase::MatrixType> mat(T);   // Verify's argument type
    for (long i = 0; i < nQ; ++i) {
      KdTree<Match4PCSBase::Scalar>::RangeQuery<> query;
      query.queryPoint = (mat * m->sampled_Q_3D_[i].pos().homogeneous()).head<3>();
      query.sqdist = sq_eps;
      const auto id = m->kd_tree_.doQueryRestrictedClosestIndex(query);
      const bool hit = id != KdTree<Match4PCSBase::Scalar>::invalidIndex();
      out_index[c * nQ + i] = hit ? (int32_t)id : -1;
      out_sq[c * nQ + i] = hit ? (query.queryPoint - m->sampled_P_3D_[id].pos()).squaredNorm()
                               : std::numeric_limits<float>::infinity();
    }
  }
}

}  // extern "C"
