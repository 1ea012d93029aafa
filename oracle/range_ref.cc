// TEST INFRASTRUCTURE ONLY -- never linked into, imported by, or called from the product.
//
// oracle/_ref/liboracle_ref_range.so (built by oracle/range.py with the reference's Release flags, linked against
// oracle/_ref/liboracle_ref.so): the UNMODIFIED reference's range query (KdTree::doQueryDistIndices, kdtree.h:242-249,
// body :462-514) for arbitrary query points and squared radii.  A matcher is initialised on (P, Q) -- with every point
// kept, or with the reference's own sampler -- and its kd_tree_ (built by initKdTree on the centred sampled P) is asked
// directly; each list is then sorted by index (the tree's order is an artefact of its traversal).  The protected members
// are reached through a subclass, the pattern of the reference's own tests (tests/testing.h:71-154).
//
// No reference source is copied here: this file only #includes the reference's public headers at build time.
#include "super4pcs/algorithms/super4pcs.h"
#include "super4pcs/accelerators/kdtree.h"
#include "super4pcs/utils/logger.h"

#include <algorithm>
#include <cstdint>
#include <cstring>
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
  std::vector<int32_t> index;   // the lists of the last query
  std::vector<float> sq;
  ~Handle() { delete m; }
};

void fill(std::vector<Point3D>& c, const float* xyz, int n) {
  c.clear();
  for (int i = 0; i < n; ++i) c.emplace_back(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
}

}  // namespace

extern "C" {

// init() on (P, Q) with options.delta = delta.  sample_size <= 0: every point kept, in input order; otherwise the
// reference's default sampler (UniformDistSampler) with that sample size and configureOverlap(overlap)
void* range_ref_create(const float* Pxyz, int nP, const float* Qxyz, int nQ, float delta, float overlap, long sample_size) {
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

void range_ref_destroy(void* hv) { delete static_cast<Handle*>(hv); }

void range_ref_sizes(void* hv, long* out2) {
  const Matcher* m = static_cast<Handle*>(hv)->m;
  out2[0] = (long)m->sampled_P_3D_.size();
  out2[1] = (long)m->sampled_Q_3D_.size();
}

// the centred sampled clouds (nP x 3, nQ x 3)
void range_ref_sampled(void* hv, float* P, float* Q) {
  const Matcher* m = static_cast<Handle*>(hv)->m;
  for (size_t i = 0; i < m->sampled_P_3D_.size(); ++i)
    for (int k = 0; k < 3; ++k) P[3 * i + k] = m->sampled_P_3D_[i].pos()[k];
  for (size_t i = 0; i < m->sampled_Q_3D_.size(); ++i)
    for (int k = 0; k < 3; ++k) Q[3 * i + k] = m->sampled_Q_3D_[i].pos()[k];
}

// for n query points (T16: column-major 4x4 applied as Verify does, or null): the kd-tree's list for RangeQuery{queryPoint
// = y, sqdist = sq_radius}, sorted by index, kept in the handle (range_ref_get); offsets: n + 1 CSR offsets
void range_ref_query(void* hv, const float* X, long n, const float* T16, float sq_radius, int64_t* offsets) {
  Handle* h = static_cast<Handle*>(hv);
  const Matcher* m = h->m;
  Match4PCSBase::MatrixType T = Match4PCSBase::MatrixType::Identity();
  if (T16) std::memcpy(T.data(), T16, 16 * sizeof(float));
  const Eigen::Ref<const Match4PCSBase::MatrixType> mat(T);
  h->index.clear();
  h->sq.clear();
  offsets[0] = 0;
  std::vector<int> list;
  for (long i = 0; i < n; ++i) {
    KdTree<Match4PCSBase::Scalar>::RangeQuery<> query;
    const Eigen::Matrix<Match4PCSBase::Scalar, 3, 1> x(X[3 * i], X[3 * i + 1], X[3 * i + 2]);
    if (T16) query.queryPoint = (mat * x.homogeneous()).head<3>();
    else query.queryPoint = x;
    query.sqdist = sq_radius;
    list.clear();
    m->kd_tree_.doQueryDistIndices(query, list);
    std::sort(list.begin(), list.end());
    for (int j : list) {
      h->index.push_back((int32_t)j);
      h->sq.push_back((query.queryPoint - m->sampled_P_3D_[j].pos()).squaredNorm());
    }
    offsets[i + 1] = (int64_t)h->index.size();
  }
}

// the lists of the last range_ref_query: index [total], sq [total] (d^2 as the kd-tree's point test computes it)
void range_ref_get(void* hv, int32_t* index, float* sq) {
  const Handle* h = static_cast<Handle*>(hv);
  std::copy(h->index.begin(), h->index.end(), index);
  std::copy(h->sq.begin(), h->sq.end(), sq);
}

}  // extern "C"
