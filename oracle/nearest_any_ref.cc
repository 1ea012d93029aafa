// TEST INFRASTRUCTURE ONLY -- never linked into, imported by, or called from the product.
//
// oracle/_ref/liboracle_ref_nearest_any.so (built by oracle/nearest_any.py with the reference's Release flags, linked
// against oracle/_ref/liboracle_ref.so): the UNMODIFIED reference's restricted closest-point query
// (KdTree::doQueryRestrictedClosestIndex, kdtree.h:388-453) for arbitrary query points, squared radii and excluded
// indices, and the P_mean_distance_ its init stores (MeanDistance, match4pcsBase.cc:158-182).  A matcher is initialised
// on (P, Q) -- with every point kept, or with the reference's own sampler -- and its kd_tree_ (built by initKdTree on the
// centred sampled P) is asked directly.  The protected members are reached through a subclass, the pattern of the
// reference's own tests (tests/testing.h:71-154).
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
  using Match4PCSBase::P_diameter_;
  using Match4PCSBase::P_mean_distance_;
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

// init() on (P, Q) with options.delta = delta.  sample_size <= 0: every point kept, in input order; otherwise the
// reference's default sampler (UniformDistSampler) with that sample size and configureOverlap(overlap), as
// ComputeTransformation runs it
void* nearest_any_ref_create(const float* Pxyz, int nP, const float* Qxyz, int nQ, float delta, float overlap,
                             long sample_size) {
  Handle* h = new Handle;
  h->opt.delta = delta;
  std::vector<Point3D> P, Q;
  fill(P, Pxyz, nP);
  fill(Q, Qxyz, nQ);
  if (sample_size <= 0) {
    h->opt.sample_size = (size_t)nP + (size_t)nQ + 1;
    h->m = new Matcher(h->opt, h->logger);
    h->m->init(P, Q, KeepAll());
  } else {
    h->opt.sample_size = (size_t)sample_size;
    h->opt.configureOverlap(overlap);
    h->m = new Matcher(h->opt, h->logger);
    h->m->init(P, Q, Sampling::UniformDistSampler());
  }
  return h;
}

void nearest_any_ref_destroy(void* hv) { delete static_cast<Handle*>(hv); }

// the sizes of the centred sampled clouds
void nearest_any_ref_sizes(void* hv, long* out2) {
  const Matcher* m = static_cast<Handle*>(hv)->m;
  out2[0] = (long)m->sampled_P_3D_.size();
  out2[1] = (long)m->sampled_Q_3D_.size();
}

// the centred sampled clouds (nP x 3, nQ x 3)
void nearest_any_ref_sampled(void* hv, float* P, float* Q) {
  const Matcher* m = static_cast<Handle*>(hv)->m;
  for (size_t i = 0; i < m->sampled_P_3D_.size(); ++i)
    for (int k = 0; k < 3; ++k) P[3 * i + k] = m->sampled_P_3D_[i].pos()[k];
  for (size_t i = 0; i < m->sampled_Q_3D_.size(); ++i)
    for (int k = 0; k < 3; ++k) Q[3 * i + k] = m->sampled_Q_3D_[i].pos()[k];
}

// out2 = {P_diameter_, P_mean_distance_} after init
void nearest_any_ref_mean_distance(void* hv, float* out2) {
  const Matcher* m = static_cast<Handle*>(hv)->m;
  out2[0] = m->P_diameter_;
  out2[1] = m->P_mean_distance_;
}

// for n query points (T16: column-major 4x4 applied as Verify does, or null): out_index = what the kd-tree returns for
// RangeQuery{queryPoint = y, sqdist = sq_radius} and currentId = exclude[i] (-1 when exclude is null; -1 out: none),
// out_sq = the squared distance to that point, computed as the kd-tree's leaf test does (+inf for -1)
void nearest_any_ref_query(void* hv, const float* X, long n, const float* T16, float sq_radius, const int32_t* exclude,
                           int32_t* out_index, float* out_sq) {
  const Matcher* m = static_cast<Handle*>(hv)->m;
  Match4PCSBase::MatrixType T = Match4PCSBase::MatrixType::Identity();
  if (T16) std::memcpy(T.data(), T16, 16 * sizeof(float));
  const Eigen::Ref<const Match4PCSBase::MatrixType> mat(T);
  for (long i = 0; i < n; ++i) {
    KdTree<Match4PCSBase::Scalar>::RangeQuery<> query;
    const Eigen::Matrix<Match4PCSBase::Scalar, 3, 1> x(X[3 * i], X[3 * i + 1], X[3 * i + 2]);
    if (T16) query.queryPoint = (mat * x.homogeneous()).head<3>();
    else query.queryPoint = x;
    query.sqdist = sq_radius;
    const int current = exclude ? (int)exclude[i] : -1;
    const auto id = m->kd_tree_.doQueryRestrictedClosestIndex(query, current);
    const bool hit = id != KdTree<Match4PCSBase::Scalar>::invalidIndex();
    out_index[i] = hit ? (int32_t)id : -1;
    out_sq[i] = hit ? (query.queryPoint - m->sampled_P_3D_[id].pos()).squaredNorm() : std::numeric_limits<float>::infinity();
  }
}

}  // extern "C"
