// super4pcs-b200: non-template members of GlobalRegistration::Match4PCSBase.
//
// Host side of the RANSAC loop: base selection, plus the glue to the device stages behind include/s4g.h.
// Provenance: SegmentToSegment / SelectRandomTriangle / TryQuadrilateral / SelectQuadrilateral RESTATE the reference's
// host driver (src/super4pcs/algorithms/match4pcsBase.cc:64-131, 185-351) statement by statement -- same RNG consumption
// order, same float/double mixing, same branch structure -- because the same seed has to pick the same bases bit for bit
// (SURVEY.md A.5/A.6).  They are parity-forced host control code outside the GPU hot path, not an independent design;
// everything else in this file (device glue, lanes, shards, timings) is new.
#include "super4pcs/algorithms/match4pcsBase.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <stdexcept>
#include <string>
#include <thread>

#include "s4g.h"
#include "shards.h"

namespace GlobalRegistration {

constexpr int Match4PCSBase::kNumberOfDiameterTrials;
constexpr Match4PCSBase::Scalar Match4PCSBase::kLargeNumber;
constexpr Match4PCSBase::Scalar Match4PCSBase::distance_factor;

namespace {

using Vec3 = Match4PCSBase::VectorType;

// Closest approach of segments [p1,p2] and [q1,q2]; the parameters of the two closest points are
// the base invariants.  Scalars are double, vector arithmetic stays float -- the mix of the
// reference's distSegmentToSegment (match4pcsBase.cc:64-131, instantiated with Scalar=double).
double SegmentToSegment(const Vec3& p1, const Vec3& p2, const Vec3& q1, const Vec3& q2, double& inv1,
                        double& inv2) {
  const double kTiny = 0.0001;
  const Vec3 u = p2 - p1, v = q2 - q1, w = p1 - q1;
  const double a = u.dot(u), b = u.dot(v), c = v.dot(v), d = u.dot(w), e = v.dot(w);
  const double f = a * c - b * b;
  double sNum = 0.0, sDen = f, tNum = 0.0, tDen = f;
  if (f < kTiny) {  // (nearly) parallel: clamp s to the start of the first segment
    sNum = 0.0; sDen = 1.0; tNum = e; tDen = c;
  } else {
    sNum = b * e - c * d;
    tNum = a * e - b * d;
    if (sNum < 0.0) {
      sNum = 0.0; tNum = e; tDen = c;
    } else if (sNum > sDen) {
      sNum = sDen; tNum = e + b; tDen = c;
    }
  }
  if (tNum < 0.0) {
    tNum = 0.0;
    if (-d < 0.0) sNum = 0.0;
    else if (-d > a) sNum = sDen;
    else { sNum = -d; sDen = a; }
  } else if (tNum > tDen) {
    tNum = tDen;
    if ((-d + b) < 0.0) sNum = 0;
    else if ((-d + b) > a) sNum = sDen;
    else { sNum = (-d + b); sDen = a; }
  }
  inv1 = (std::abs(sNum) < kTiny ? 0.0 : sNum / sDen);
  inv2 = (std::abs(tNum) < kTiny ? 0.0 : tNum / tDen);
  return (w + (inv1 * u) - (inv2 * v)).norm();
}

}  // namespace

Match4PCSBase::Match4PCSBase(const Match4PCSOptions& options, const Utils::Logger& logger, int)
    : number_of_trials_(0),
      max_base_diameter_(-1),
      P_mean_distance_(1.0),
      best_LCP_(0.0),
      options_(options),
      randomGenerator_(options.randomSeed),
      logger_(logger) {
  base_3D_.resize(4);
  // The reference never initialises these two (match4pcsBase.h:137); progress reports issued before the first
  // adopted candidate read them (hpp:228).  Zero is what a freshly allocated reference object holds in practice.
  qcentroid1_.setZero();
  qcentroid2_.setZero();
  transform_.setIdentity();
  if (const char* e = std::getenv("S4PCS_LANES")) lane_count_ = std::max(1, std::min(16, std::atoi(e)));
  if (const char* e = std::getenv("S4PCS_BATCH")) batch_ = std::max(1, std::min(64, std::atoi(e)));
  if (const char* e = std::getenv("S4PCS_BATCH_MAX_Q")) batch_max_q_ = std::max(0, std::atoi(e));
  if (const char* e = std::getenv("S4PCS_TIMINGS")) timings_ = std::atoi(e) != 0;
  if (const char* e = std::getenv("S4PCS_NCCL")) nccl_ = std::atoi(e) != 0;
  int first = 0;
  if (const char* e = std::getenv("S4PCS_DEVICE")) first = std::atoi(e);
  devices_.assign(1, first);
  if (const char* e = std::getenv("S4PCS_DEVICES")) {  // "4" = first .. first + 3; "0,2,3" = exactly these ordinals
    const std::string spec(e);
    if (spec == "all") {  // every CUDA device of the box, starting at S4PCS_DEVICE
      int count = 0;
      if (s4g_device_count(&count) != S4G_OK) count = 0;  // (no device: s4g_create reports it when first needed)
      for (int k = first + 1; k < count && devices_.size() < 16; ++k) devices_.push_back(k);
    } else if (spec.find(',') == std::string::npos) {
      const int count = std::max(1, std::min(16, std::atoi(e)));
      for (int k = 1; k < count; ++k) devices_.push_back(first + k);
    } else {
      devices_.clear();
      size_t at = 0;
      while (at <= spec.size() && devices_.size() < 16) {
        const size_t comma = std::min(spec.find(',', at), spec.size());
        if (comma > at) devices_.push_back(std::atoi(spec.substr(at, comma - at).c_str()));
        at = comma + 1;
      }
      if (devices_.empty()) devices_.assign(1, first);
    }
  }
  // communicators of different lanes would interleave their collectives on the same devices in thread order: one lane
  if (nccl_ && devices_.size() > 1) lane_count_ = 1;
}

Match4PCSBase::~Match4PCSBase() {
  for (s4g_ctx* lane : lanes_)
    if (lane) s4g_destroy(lane);
  lanes_.clear();
  for (auto& entry : peers_)
    for (s4g_ctx* peer : entry.second.ctx)
      if (peer) s4g_destroy(peer);
  peers_.clear();
  if (gpu_) s4g_destroy(gpu_);
  gpu_ = nullptr;
}

void Match4PCSBase::ThrowLaneError(const s4g_ctx* lane, const char* where) const {
  throw std::runtime_error(std::string("super4pcs-b200: ") + where + ": " +
                           (lane ? s4g_error_string(lane) : "no CUDA device (there is no CPU fallback)"));
}

void Match4PCSBase::EnsureDevice() const {
  if (gpu_) return;
  if (s4g_create(devices_[0], &gpu_) != S4G_OK) {
    gpu_ = nullptr;
    ThrowLaneError(nullptr, "s4g_create");
  }
}

void Match4PCSBase::UploadClouds() {
  EnsureDevice();
  UploadCloudsTo(gpu_);
  lanes_stale_ = true;  // the extra lanes are (re)loaded when speculation first needs them
  ++cloud_epoch_;       // ... and so are the contexts on the other devices (PreparePeers)
}

const std::vector<s4g_ctx*>* Match4PCSBase::PeersOf(const s4g_ctx* primary) const {
  if (devices_.size() < 2) return nullptr;
  const auto it = peers_.find(primary);
  return it == peers_.end() ? nullptr : &it->second.ctx;
}

const std::vector<s4g_ctx*>* Match4PCSBase::PreparePeers(const s4g_ctx* primary) const {
  if (devices_.size() < 2 || primary == nullptr) return nullptr;
  PeerSet& set = peers_[primary];
  while (set.ctx.size() + 1 < devices_.size()) {
    s4g_ctx* peer = nullptr;
    const int ordinal = devices_[set.ctx.size() + 1];
    if (s4g_create(ordinal, &peer) != S4G_OK) {
      int count = 0;
      (void)s4g_device_count(&count);
      throw std::runtime_error("super4pcs-b200: S4PCS_DEVICES: cannot open CUDA device " + std::to_string(ordinal) + " (" +
                               std::to_string(count) + " device(s) visible; there is no CPU fallback)");
    }
    set.ctx.push_back(peer);
    set.epoch = 0;
  }
  if (nccl_ && !set.comm) {  // one communicator over the primary and its peers; no other transport is tried
    std::vector<s4g_ctx*> ranks(1, const_cast<s4g_ctx*>(primary));
    ranks.insert(ranks.end(), set.ctx.begin(), set.ctx.end());
    if (s4g_comm_init_all(ranks.data(), int(ranks.size())) != S4G_OK)
      throw std::runtime_error(std::string("super4pcs-b200: S4PCS_NCCL: ") + s4g_error_string(primary));
    set.comm = true;
  }
  if (set.epoch != cloud_epoch_) {  // upload + grid build on every further device at once
    UploadCloudsToAll(set.ctx);
    set.epoch = cloud_epoch_;
  }
  return &set.ctx;
}

void Match4PCSBase::UploadCloudsTo(s4g_ctx* ctx) const {
  auto flatten = [](const std::vector<Point3D>& c, int what, std::vector<float>& out) {
    out.resize(3 * c.size());
    for (size_t i = 0; i < c.size(); ++i) {
      const VectorType& v = what == 0 ? c[i].pos() : what == 1 ? c[i].normal() : c[i].rgb();
      out[3 * i] = v[0]; out[3 * i + 1] = v[1]; out[3 * i + 2] = v[2];
    }
  };
  std::vector<float> xyz, nrm, rgb;
  flatten(sampled_P_3D_, 0, xyz);
  if (s4g_set_cloud_p(ctx, xyz.data(), int(sampled_P_3D_.size()), options_.delta) != S4G_OK)
    ThrowLaneError(ctx, "s4g_set_cloud_p");
  flatten(sampled_Q_3D_, 0, xyz);
  flatten(sampled_Q_3D_, 1, nrm);
  flatten(sampled_Q_3D_, 2, rgb);
  if (s4g_set_cloud_q(ctx, xyz.data(), nrm.data(), rgb.data(), int(sampled_Q_3D_.size())) != S4G_OK)
    ThrowLaneError(ctx, "s4g_set_cloud_q");
}

// the same clouds into several contexts at once, one host thread each (the peers of S4PCS_DEVICES)
void Match4PCSBase::UploadCloudsToAll(const std::vector<s4g_ctx*>& contexts) const {
  if (contexts.size() == 1) {
    UploadCloudsTo(contexts[0]);
    return;
  }
  std::vector<std::exception_ptr> errors(contexts.size());
  std::vector<std::thread> workers;
  for (size_t k = 0; k < contexts.size(); ++k)
    workers.emplace_back([this, &contexts, &errors, k] {
      try {
        UploadCloudsTo(contexts[k]);
      } catch (...) {
        errors[k] = std::current_exception();
      }
    });
  for (std::thread& w : workers) w.join();
  for (const std::exception_ptr& e : errors)
    if (e) std::rethrow_exception(e);
}

// match4pcsBase.cc:158-182: for every sampled-P point, its nearest other sampled-P point with d^2 <= 0.2 x P_diameter_
// (a length passed as a squared radius, as the reference does), then the mean of those distances summed in index order.
// gpu_ holds sampled P since init uploaded it; the query excludes the point itself (the kd-tree's currentId = i).  Equal
// d^2 give equal norms, so the tie rule of s4g_nearest does not change the value.
Match4PCSBase::Scalar Match4PCSBase::MeanDistance() {
  const Scalar kDiameterFraction = 0.2;
  int number_of_samples = 0;
  Scalar distance = 0.0;
  const int n = int(sampled_P_3D_.size());
  if (n > 0) {
    if (gpu_ == nullptr) throw std::runtime_error("super4pcs-b200: MeanDistance: no clouds on the device (call init first)");
    std::vector<float> xyz(3 * size_t(n));
    std::vector<int32_t> self(n), nearest(n);
    for (int i = 0; i < n; ++i) {
      for (int k = 0; k < 3; ++k) xyz[3 * size_t(i) + k] = sampled_P_3D_[i].pos()[k];
      self[i] = i;
    }
    if (s4g_nearest(gpu_, xyz.data(), n, nullptr, P_diameter_ * kDiameterFraction, self.data(), nearest.data(), nullptr) !=
        S4G_OK)
      ThrowLaneError(gpu_, "s4g_nearest");
    for (int i = 0; i < n; ++i) {
      if (nearest[i] < 0) continue;
      distance += (sampled_P_3D_[i].pos() - sampled_P_3D_[nearest[i]].pos()).norm();
      number_of_samples++;
    }
  }
  return distance / number_of_samples;
}

bool Match4PCSBase::SelectRandomTriangle(int& base1, int& base2, int& base3) {
  const int n = int(sampled_P_3D_.size());
  base1 = base2 = base3 = -1;
  const int first = randomGenerator_() % n;
  const Scalar sq_limit = max_base_diameter_ * max_base_diameter_;
  const VectorType& origin = sampled_P_3D_[first].pos();
  Scalar widest = 0.0;
  for (int trial = 0; trial < kNumberOfDiameterTrials; ++trial) {
    const int second = randomGenerator_() % n;
    const int third = randomGenerator_() % n;
    const VectorType u = sampled_P_3D_[second].pos() - origin;
    const VectorType w = sampled_P_3D_[third].pos() - origin;
    const Scalar area2 = (u.cross(w)).norm();  // twice the triangle area: wide but bounded triangles
    if (area2 > widest && u.squaredNorm() < sq_limit && w.squaredNorm() < sq_limit) {
      widest = area2;
      base1 = first; base2 = second; base3 = third;
    }
  }
  return base1 != -1 && base2 != -1 && base3 != -1;
}

bool Match4PCSBase::TryQuadrilateral(Scalar& invariant1, Scalar& invariant2, int& id1, int& id2, int& id3,
                                     int& id4) {
  // among the 12 ordered ways to split the four points into two segments keep the split whose
  // segments pass closest to each other
  Scalar closest = std::numeric_limits<Scalar>::max();
  int order[4] = {-1, -1, -1, -1};
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      if (i == j) continue;
      int k = 0;
      while (k == i || k == j) ++k;
      int l = 0;
      while (l == i || l == j || l == k) ++l;
      double r1, r2;
      const Scalar gap = SegmentToSegment(base_3D_[i].pos(), base_3D_[j].pos(), base_3D_[k].pos(),
                                          base_3D_[l].pos(), r1, r2);
      if (gap < closest) {
        closest = gap;
        order[0] = i; order[1] = j; order[2] = k; order[3] = l;
        invariant1 = r1;
        invariant2 = r2;
      }
    }
  if (order[0] < 0 || order[1] < 0 || order[2] < 0 || order[3] < 0) return false;

  const std::vector<Point3D> pts = base_3D_;
  const int ids[4] = {id1, id2, id3, id4};
  for (int s = 0; s < 4; ++s) base_3D_[s] = pts[order[s]];
  id1 = ids[order[0]]; id2 = ids[order[1]]; id3 = ids[order[2]]; id4 = ids[order[3]];
  return true;
}

bool Match4PCSBase::SelectQuadrilateral(Scalar& invariant1, Scalar& invariant2, int& base1, int& base2, int& base3,
                                        int& base4) {
  const Scalar kBaseTooSmall(0.2);
  for (int attempt = 0; attempt < kNumberOfDiameterTrials; ++attempt) {
    if (!SelectRandomTriangle(base1, base2, base3)) return false;
    base_3D_[0] = sampled_P_3D_[base1];
    base_3D_[1] = sampled_P_3D_[base2];
    base_3D_[2] = sampled_P_3D_[base3];

    // plane A x + B y + C z = 1 through the triangle (Cramer, evaluated in double)
    const double x1 = base_3D_[0].x(), y1 = base_3D_[0].y(), z1 = base_3D_[0].z();
    const double x2 = base_3D_[1].x(), y2 = base_3D_[1].y(), z2 = base_3D_[1].z();
    const double x3 = base_3D_[2].x(), y3 = base_3D_[2].y(), z3 = base_3D_[2].z();
    const Scalar det = (-x3 * y2 * z1 + x2 * y3 * z1 + x3 * y1 * z2 - x1 * y3 * z2 - x2 * y1 * z3 + x1 * y2 * z3);
    if (det == 0) continue;
    const Scalar A = (-y2 * z1 + y3 * z1 + y1 * z2 - y3 * z2 - y1 * z3 + y2 * z3) / det;
    const Scalar B = (x2 * z1 - x3 * z1 - x1 * z2 + x3 * z2 + x1 * z3 - x2 * z3) / det;
    const Scalar C = (-x2 * y1 + x3 * y1 + x1 * y2 - x3 * y2 - x1 * y3 + x2 * y3) / det;

    // fourth point: the most coplanar sample that is not too close to the triangle's corners
    base4 = -1;
    Scalar flattest = std::numeric_limits<Scalar>::max();
    const Scalar too_small = std::pow(max_base_diameter_ * kBaseTooSmall, 2);
    const VectorType &c1 = sampled_P_3D_[base1].pos(), &c2 = sampled_P_3D_[base2].pos(),
                     &c3 = sampled_P_3D_[base3].pos();
    for (unsigned int i = 0; i < sampled_P_3D_.size(); ++i) {
      const Point3D& s = sampled_P_3D_[i];
      if ((s.pos() - c1).squaredNorm() < too_small || (s.pos() - c2).squaredNorm() < too_small ||
          (s.pos() - c3).squaredNorm() < too_small)
        continue;
      const Scalar off_plane = std::abs(A * s.x() + B * s.y() + C * s.z() - 1.0);
      if (off_plane < flattest) {
        flattest = off_plane;
        base4 = int(i);
      }
    }
    if (base4 != -1) {
      base_3D_[3] = sampled_P_3D_[base4];
      if (TryQuadrilateral(invariant1, invariant2, base1, base2, base3, base4)) return true;
    }
  }
  return false;
}

// Host twin of the device rigid fit (csrc/rigid.cu): identical operations in identical order.
bool Match4PCSBase::ComputeRigidTransformation(const std::array<Point3D, 4>& ref,
                                               const std::array<Point3D, 4>& candidate,
                                               const Eigen::Matrix<Scalar, 3, 1>& centroid1,
                                               Eigen::Matrix<Scalar, 3, 1> centroid2, Scalar max_angle,
                                               Eigen::Ref<MatrixType> transform, Scalar& rms_,
                                               bool computeScale) const {
  rms_ = kLargeNumber;
  if (computeScale) return false;  // multiscale matching (reference macro MULTISCALE) is not built
  auto frame = [](const VectorType& o, const VectorType& a, const VectorType& b, Eigen::Matrix<Scalar, 3, 3>& F) {
    VectorType e1 = a - o;
    if (e1.squaredNorm() == 0) return false;
    e1.normalize();
    VectorType e2 = (b - o) - ((b - o).dot(e1)) * e1;
    if (e2.squaredNorm() == 0) return false;
    e2.normalize();
    VectorType e3 = e1.cross(e2);
    if (e3.squaredNorm() == 0) return false;
    e3.normalize();
    F.row(0) = e1; F.row(1) = e2; F.row(2) = e3;
    return true;
  };
  Eigen::Matrix<Scalar, 3, 3> Fp, Fq;
  // degenerate frames: "true with rms = kLargeNumber", later rejected by the caller's rms gate
  if (!frame(ref[0].pos(), ref[1].pos(), ref[2].pos(), Fp)) return true;
  if (!frame(candidate[0].pos(), candidate[1].pos(), candidate[2].pos(), Fq)) return true;
  const Eigen::Matrix<Scalar, 3, 3> R = Fp.transpose() * Fq;
  if (((R * R).diagonal().array() - Scalar(1) > Scalar(1e-6)).any()) return false;
  if (max_angle >= 0) {
    const bool within = std::abs(std::atan2(R(2, 1), R(2, 2))) <= max_angle &&
                        std::abs(std::atan2(-R(2, 0), std::sqrt(std::pow(R(2, 1), 2) + std::pow(R(2, 2), 2)))) <= max_angle &&
                        std::abs(atan2(R(1, 0), R(0, 0))) <= max_angle;
    if (!within) return false;
  }
  Scalar sum = 0;
  for (int i = 0; i < 3; ++i) {
    const VectorType moved = R * (candidate[i].pos() - centroid2);
    sum += (moved - ref[i].pos() + centroid1).norm();
  }
  rms_ = sum / Scalar(ref.size());
  transform.setIdentity();
  transform.block<3, 3>(0, 0) = R;
  transform.block<3, 1>(0, 3) = centroid1 + R * (-centroid2);
  return true;
}

Match4PCSBase::Scalar Match4PCSBase::Verify(const Eigen::Ref<const MatrixType>& mat) const {
  EnsureDevice();
  const MatrixType T = mat;  // contiguous column-major copy
  uint32_t count = 0;
  if (s4g_verify(gpu_, T.data(), 1, &count) != S4G_OK) ThrowLaneError(gpu_, "s4g_verify");
  return Scalar(count) / Scalar(sampled_Q_3D_.size());
}

void Match4PCSBase::getCorrespondences(std::vector<int>* nearest, std::vector<float>* sq_dist) const {
  // gpu_ holds the clouds init() uploaded; transform_ is the centred transform behind best_LCP_ (the identity when
  // nothing beat it).  No context or no sampled cloud: ComputeTransformation has not run, or returned kLargeNumber.
  if (gpu_ == nullptr || sampled_P_3D_.empty() || sampled_Q_3D_.empty())
    throw std::runtime_error("super4pcs-b200: getCorrespondences: no registration has run on this matcher");
  if (nearest == nullptr) throw std::invalid_argument("super4pcs-b200: getCorrespondences: nearest is null");
  const MatrixType T = transform_;
  nearest->resize(sampled_Q_3D_.size());
  static_assert(sizeof(int) == sizeof(int32_t), "index type");
  if (sq_dist) sq_dist->resize(sampled_Q_3D_.size());
  if (s4g_verify_nearest(gpu_, T.data(), 1, reinterpret_cast<int32_t*>(nearest->data()), sq_dist ? sq_dist->data() : nullptr,
                         nullptr) != S4G_OK)
    ThrowLaneError(gpu_, "s4g_verify_nearest");
}

void Match4PCSBase::getCorrespondences(std::vector<int>* nearest, std::vector<float>* sq_dist, Scalar max_distance) const {
  if (gpu_ == nullptr || sampled_P_3D_.empty() || sampled_Q_3D_.empty())
    throw std::runtime_error("super4pcs-b200: getCorrespondences: no registration has run on this matcher");
  if (nearest == nullptr) throw std::invalid_argument("super4pcs-b200: getCorrespondences: nearest is null");
  if (std::isnan(max_distance)) throw std::invalid_argument("super4pcs-b200: getCorrespondences: max_distance is NaN");
  const MatrixType T = transform_;
  const int n = int(sampled_Q_3D_.size());
  std::vector<float> xyz(3 * size_t(n));
  for (int i = 0; i < n; ++i)
    for (int k = 0; k < 3; ++k) xyz[3 * size_t(i) + k] = sampled_Q_3D_[i].pos()[k];
  nearest->resize(n);
  if (sq_dist) sq_dist->resize(n);
  const float sq_radius = max_distance * max_distance;   // as delta * delta (match4pcsBase.cc:522)
  if (s4g_nearest(gpu_, xyz.data(), n, T.data(), sq_radius, nullptr, reinterpret_cast<int32_t*>(nearest->data()),
                  sq_dist ? sq_dist->data() : nullptr) != S4G_OK)
    ThrowLaneError(gpu_, "s4g_nearest");
}

void Match4PCSBase::getNeighbors(std::vector<int64_t>* offsets, std::vector<int>* indices, Scalar max_distance,
                                 std::vector<float>* sq_dist) const {
  if (gpu_ == nullptr || sampled_P_3D_.empty() || sampled_Q_3D_.empty())
    throw std::runtime_error("super4pcs-b200: getNeighbors: no registration has run on this matcher");
  if (offsets == nullptr || indices == nullptr) throw std::invalid_argument("super4pcs-b200: getNeighbors: null output");
  if (std::isnan(max_distance)) throw std::invalid_argument("super4pcs-b200: getNeighbors: max_distance is NaN");
  const MatrixType T = transform_;
  const int n = int(sampled_Q_3D_.size());
  std::vector<float> xyz(3 * size_t(n));
  for (int i = 0; i < n; ++i)
    for (int k = 0; k < 3; ++k) xyz[3 * size_t(i) + k] = sampled_Q_3D_[i].pos()[k];
  offsets->resize(size_t(n) + 1);
  const float sq_radius = max_distance * max_distance;   // as getCorrespondences squares it
  int64_t total = 0;
  if (s4g_range(gpu_, xyz.data(), n, T.data(), sq_radius, offsets->data(), &total) != S4G_OK)
    ThrowLaneError(gpu_, "s4g_range");
  indices->resize(size_t(total));
  if (sq_dist) sq_dist->resize(size_t(total));
  if (s4g_get_range(gpu_, reinterpret_cast<int32_t*>(indices->data()), sq_dist ? sq_dist->data() : nullptr) != S4G_OK)
    ThrowLaneError(gpu_, "s4g_get_range");
}

void Match4PCSBase::getKNearest(std::vector<int>* indices, std::vector<float>* sq_dist, int k, Scalar max_distance) const {
  if (gpu_ == nullptr || sampled_P_3D_.empty() || sampled_Q_3D_.empty())
    throw std::runtime_error("super4pcs-b200: getKNearest: no registration has run on this matcher");
  if (indices == nullptr) throw std::invalid_argument("super4pcs-b200: getKNearest: null output");
  if (std::isnan(max_distance)) throw std::invalid_argument("super4pcs-b200: getKNearest: max_distance is NaN");
  const MatrixType T = transform_;
  const int n = int(sampled_Q_3D_.size());
  std::vector<float> xyz(3 * size_t(n));
  for (int i = 0; i < n; ++i)
    for (int c = 0; c < 3; ++c) xyz[3 * size_t(i) + c] = sampled_Q_3D_[i].pos()[c];
  const size_t entries = k > 0 ? size_t(n) * size_t(k) : 0;
  indices->resize(entries);
  if (sq_dist) sq_dist->resize(entries);
  const float sq_radius = max_distance * max_distance;   // as getCorrespondences squares it
  if (s4g_knn(gpu_, xyz.data(), n, T.data(), k, sq_radius, nullptr, reinterpret_cast<int32_t*>(indices->data()),
              sq_dist ? sq_dist->data() : nullptr) != S4G_OK)
    ThrowLaneError(gpu_, "s4g_knn");
}

bool Match4PCSBase::TryBaseOnLane(s4g_ctx*, const SelectedBase&, DeviceBest*) const { return false; }

bool Match4PCSBase::TryBasesOnLane(s4g_ctx*, const std::vector<SelectedBase*>&) const { return false; }

void Match4PCSBase::SelectBase(SelectedBase* sb) {
  const std::chrono::steady_clock::time_point t_sel = std::chrono::steady_clock::now();
  sb->selected = SelectQuadrilateral(sb->invariant1, sb->invariant2, sb->ids[0], sb->ids[1], sb->ids[2], sb->ids[3]);
  if (timings_) stats_.ms_select += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_sel).count();
  if (sb->selected) {
    sb->distance1 = (base_3D_[0].pos() - base_3D_[1].pos()).norm();
    sb->distance2 = (base_3D_[2].pos() - base_3D_[3].pos()).norm();
    sb->normal_angle1 = (base_3D_[0].normal() - base_3D_[1].normal()).norm();
    sb->normal_angle2 = (base_3D_[2].normal() - base_3D_[3].normal()).norm();
    sb->base3d = base_3D_;
    PrepareBaseOrder(sb->distance1, sb->distance2, &sb->order);
  }
  sb->rng_after = randomGenerator_;
}

// Row f1.  Runs the selected bases of spec_: in one launch chain on gpu_ when batches are on and several bases were
// selected ahead, else each through TryBaseOnLane, base k on lane k (lane 0 = gpu_ on the calling thread, the others
// on one short-lived thread each: a base is a chain of stream launches with blocking size read-backs, so host threads
// are what lets the chains overlap).  One base selected: the per-base chain on gpu_.
void Match4PCSBase::RunSpeculation() {
  EnsureDevice();
  std::vector<SelectedBase*> selected;
  for (SelectedBase& sb : spec_)  // (deque elements do not move while nothing is inserted)
    if (sb.selected) selected.push_back(&sb);
  auto run = [this](SelectedBase* sb, s4g_ctx* lane) {
    sb->lane = lane;
    try {
      sb->handled = TryBaseOnLane(lane, *sb, &sb->best);
    } catch (...) {
      sb->error = std::current_exception();
    }
  };
  if (BatchOn() && spec_.size() > 1) {
    // one launch chain for all the selected bases (s4g_try_bases); candidate sharding over several devices keeps the
    // per-base chain (its quads have to be resident on every device)
    if (TryBasesOnLane(gpu_, selected)) return;
    if (lane_count_ <= 1) {  // no batched pass for this matcher and no lanes: one base after the other on the primary context
      for (SelectedBase* sb : selected) run(sb, gpu_);
      return;
    }
  }
  if (selected.size() > 1) {
    while (lanes_.size() + 1 < selected.size()) {
      s4g_ctx* lane = nullptr;
      if (s4g_create(devices_[0], &lane) != S4G_OK) ThrowLaneError(nullptr, "s4g_create (lane)");
      lanes_.push_back(lane);
      lanes_stale_ = true;
    }
    if (lanes_stale_) {
      for (s4g_ctx* lane : lanes_) UploadCloudsTo(lane);  // (sequential: the form the GPU tests run)
      lanes_stale_ = false;
    }
  }
  if (devices_.size() > 1) {  // every lane that runs below shards its candidates over the other devices
    PreparePeers(gpu_);
    for (size_t k = 0; k + 1 < selected.size() && k < lanes_.size(); ++k) PreparePeers(lanes_[k]);
  }
  std::vector<std::thread> workers;
  for (size_t k = 1; k < selected.size(); ++k) workers.emplace_back(run, selected[k], lanes_[k - 1]);
  if (!selected.empty()) run(selected[0], gpu_);
  for (std::thread& w : workers) w.join();
}

void Match4PCSBase::DiscardSpeculation() {
  if (spec_.empty()) return;
  randomGenerator_ = rng_consumed_;
  RestoreBaseOrder(order_consumed_);
  spec_.clear();
}

void Match4PCSBase::DeviceTryCongruentSet(const int base_ids[4], const std::vector<Quadrilateral>& quads,
                                          DeviceBest* out) const {
  EnsureDevice();
  float base_xyz[12];
  for (int k = 0; k < 4; ++k)
    for (int c = 0; c < 3; ++c) base_xyz[3 * k + c] = sampled_P_3D_[base_ids[k]].pos()[c];
  static_assert(sizeof(Quadrilateral) == 4 * sizeof(int), "Quadrilateral must be 4 packed ints");
  const std::vector<s4g_ctx*>* peers = PreparePeers(gpu_);
  std::vector<s4g_tcs_result> shard(1 + (peers ? peers->size() : 0));
  detail::ForEachShard(gpu_, peers, [&](s4g_ctx* ctx, int rank, int world) {  // (nothing precedes the call: no gate needed)
    if (s4g_try_congruent_set(ctx, base_xyz, quads.empty() ? nullptr : quads[0].vertices.data(), int64_t(quads.size()),
                              options_.max_angle, distance_factor * options_.delta, rank, world,
                              &shard[size_t(rank)]) != S4G_OK)
      ThrowLaneError(ctx, "s4g_try_congruent_set");
  });
  out->SetFrom(detail::CombineShards(shard, nccl_));
}

void Match4PCSBase::DeviceBest::SetFrom(const s4g_tcs_result& r) {
  any = r.best_index >= 0;
  count = r.best_count;
  n_q = r.n_q ? r.n_q : 1;
  index = r.best_index;
  n_gate_pass = r.n_gate_pass;
  if (any) {
    std::memcpy(quad, r.best_quad, sizeof r.best_quad);
    T = Eigen::Map<const MatrixType>(r.best_T);
    centroid1 = Eigen::Map<const VectorType>(r.centroid1);
    centroid2 = Eigen::Map<const VectorType>(r.centroid2);
  }
}

void Match4PCSBase::AccountBase(const DeviceBest& b) {
  if (!timings_) return;
  stats_.bases++;
  stats_.pairs += static_cast<unsigned long long>(b.n_pairs[0]) + static_cast<unsigned long long>(b.n_pairs[1]);
  stats_.quads += static_cast<unsigned long long>(b.n_quads);
  stats_.verified += static_cast<unsigned long long>(b.n_gate_pass);
  stats_.ms_pairs += b.stage_ms[0];
  stats_.ms_quads += b.stage_ms[1];
  stats_.ms_rigid += b.stage_ms[2];
  stats_.ms_verify += b.stage_ms[3];
}

// the reference's frame (hpp:77-83) with the device stages in place of its kd-tree line
void Match4PCSBase::LogTimings() const {
  Log<LogLevel::Verbose>("----------- Timings (msec) -------------");
  Log<LogLevel::Verbose>(" Total computation time  : ", stats_.ms_total);
  Log<LogLevel::Verbose>(" Total verify time       : ", stats_.ms_verify, "  (device; ", stats_.verified, " candidates)");
  Log<LogLevel::Verbose>("    Rigid fit + gate     : ", stats_.ms_rigid, "  (device; ", stats_.quads, " quads)");
  Log<LogLevel::Verbose>(" Pair extraction         : ", stats_.ms_pairs, "  (device; ", stats_.pairs, " ordered pairs)");
  Log<LogLevel::Verbose>(" Congruent quads         : ", stats_.ms_quads, "  (device)");
  Log<LogLevel::Verbose>(" Bases tried             : ", stats_.bases);
  Log<LogLevel::Verbose>(" Base selection          : ", stats_.ms_select, "  (host wall clock)");
  Log<LogLevel::Verbose>(" Device passes           : ", stats_.ms_passes, "  (host wall clock: launches, read-backs, waits)");
  Log<LogLevel::Verbose>("----------------------------------------");
}

void Match4PCSBase::AdoptIfBetter(const int base_ids[4], const DeviceBest& b) {
  const Scalar lcp = Scalar(b.count) / Scalar(b.n_q);
  if (!(lcp > best_LCP_)) return;  // strict: the first maximum wins (reference hpp:468)
  for (int k = 0; k < 4; ++k) {
    base_[k] = base_ids[k];
    current_congruent_[k] = b.quad[k];
  }
  best_LCP_ = lcp;
  transform_ = b.T;
  qcentroid1_ = b.centroid1;
  qcentroid2_ = b.centroid2;
}

// centred-frame transform -> transform between the original clouds (reference hpp:224-229)
Eigen::Matrix<Match4PCSBase::Scalar, 4, 4> Match4PCSBase::GlobalTransform(const Eigen::Matrix<Scalar, 4, 4>& centred,
                                                                          const VectorType& c1,
                                                                          const VectorType& c2) const {
  Eigen::Matrix<Scalar, 3, 3> rot, scale;
  Eigen::Transform<Scalar, 3, Eigen::Affine>(centred).computeRotationScaling(&rot, &scale);
  Eigen::Matrix<Scalar, 4, 4> out = centred;
  out.col(3) = (c1 + centroid_P_ - (rot * scale * (c2 + centroid_Q_))).homogeneous();
  return out;
}

}  // namespace GlobalRegistration
