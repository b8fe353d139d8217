// okvis_b200_estimator.hpp -- C++ host shim above the C-ABI (include/okvis_b200.h), mirroring the public surface of
// okvis::Estimator (okvis_ceres/include/okvis/Estimator.hpp:77-412).  It owns the host book-keeping the reference
// keeps in statesMap_ / landmarksMap_ / okvis::ceres::Map (id <-> block maps, which residual touches which block) and
// forwards all numeric work to the device:
//   * the keyframe window lives on the device (one slot of the context); addStates / addLandmark / addObservation /
//     removeObservation / set_* forward ONE command each (okb_window_add_frame, ...), so a frame's worth of data
//     crosses PCIe per optimize() -- never the window;
//   * optimize()                      = okb_optimize_slots + okb_window_download_slots (Estimator.cpp:843-906)
//   * applyMarginalizationStrategy()  = the reference's bookkeeping (which blocks / residuals, Estimator.cpp:434-773)
//                                       on the host + okb_window_marginalize_batch for MarginalizationError's numerics
//                                       (MarginalizationError.cpp:127-435, 507-846) + okb_window_remove_*;
//   * state prediction in addStates() = okb_imu_propagate_batch                        (ImuError.cpp:287-504).
// An EstimatorGroup (below) owns one context for many sessions, one slot each, and runs addStates / optimize /
// applyMarginalizationStrategy for a list of them with one batched device call per step, between host halves of the
// session.  A standalone Estimator is a group of one: it owns a one-window EstimatorGroup, takes its slot 0, and its
// own addStates / optimize / applyMarginalizationStrategy run the group's list bodies on the list {this}.
// Eigen-free: poses are [t(3), q_xyzw(4)] arrays exactly as PoseParameterBlock stores them
// (okvis_ceres/src/PoseParameterBlock.cpp:68-79), so an OKVIS build wraps these calls one-to-one (INTEGRATION.md
// shows the adaptor a maintainer would add; the MultiFrame / cv types stay on the OKVIS side of it).
//
// Not supported (fails loudly): online extrinsics estimation (sigma_absolute_* > 0 / sigma_c_relative_* > 0).
#pragma once
#include <algorithm>
#include <array>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <iterator>
#include <map>
#include <memory>
#include <ostream>
#include <set>
#include <stdexcept>
#include <string>
#include <vector>

#include "okvis_b200.h"

namespace okvis_b200 {

using Pose7 = std::array<double, 7>;        // [t, q_xyzw]
using SpeedAndBias = std::array<double, 9>; // [v_W, b_g, b_a]
using Vec4 = std::array<double, 4>;

struct ImuMeasurement { int64_t t_ns; double gyro[3]; double acc[3]; };

// okvis::ExtrinsicsEstimationParameters (okvis_common/include/okvis/Parameters.hpp:60-96)
struct ExtrinsicsEstimationParameters {
  double sigma_absolute_translation = 0, sigma_absolute_orientation = 0;
  double sigma_c_relative_translation = 0, sigma_c_relative_orientation = 0;
};

// okvis::KeypointIdentifier / okvis::MapPoint (okvis_common/include/okvis/FrameTypedefs.hpp)
struct KeypointIdentifier {
  uint64_t frameId = 0; size_t cameraIndex = 0, keypointIndex = 0;
  bool operator<(const KeypointIdentifier& o) const {
    if (frameId != o.frameId) return frameId < o.frameId;
    if (cameraIndex != o.cameraIndex) return cameraIndex < o.cameraIndex;
    return keypointIndex < o.keypointIndex;
  }
};
struct MapPoint {
  uint64_t id = 0;
  Vec4 point{{0, 0, 0, 1}};
  double quality = 0, distance = 0;
  std::map<KeypointIdentifier, uint64_t> observations;   // -> residual block id
};
using PointMap = std::map<uint64_t, MapPoint>;
using MapPointVector = std::vector<MapPoint>;

// Device-side capacities of an Estimator's resident window (okb_window_reserve).
// featureKeypoints > 0 also gives the window a feature store (okb_window_reserve_features) for the device-side 3D-2D
// tracking of Frontend::matchToKeyframes3D2D / matchToLastFrame3D2D: one feature slot per frame, that many keypoints
// per camera image.
struct EstimatorCapacity {
  int frames = 16, landmarks = 4096, observations = 65536, imu_samples = 8192, marg_dim = 160;
  int featureKeypoints = 0, descriptorBytes = 48;
};

// Throws std::runtime_error with the context's last error unless rc is OKB_OK.
inline void throwIfFailed(okb_ctx* ctx, int rc) {
  if (rc != OKB_OK) throw std::runtime_error(std::string("okvis_b200: ") + okb_last_error(ctx));
}

class EstimatorGroup;
class Frontend;

class Estimator {
 private:
  friend class EstimatorGroup;
  friend class Frontend;

  struct State { uint64_t id = 0; int64_t t_ns = 0; bool isKeyframe = false, hasSb = false; Pose7 T_WS{}; SpeedAndBias sb{}; bool hasImuTerm = false; std::vector<okb_imu_sample> imuFromPrev; };
  struct BlockRef { int kind; uint64_t id; };
  // addStates between its halves: the new state, and (predict) the propagation from the previous state still to run
  struct PendingState { State st; std::vector<okb_imu_sample> samples; bool predict = false; int64_t t0_ns = 0; int used = 0; };
  // applyMarginalizationStrategy between its halves: the bookkeeping's results and the device job (none: !anything)
  struct MargPlan {
    bool skip = true, anything = false, reDoFixation = false;
    std::vector<uint64_t> removeFrames, removeAllButPose, landmarksGone;
    std::vector<BlockRef> blocks;
    std::vector<int32_t> prev, kinds;
    std::vector<uint8_t> margFlag;
    std::vector<uint32_t> idx, jobTerms, jobSbPriors, jobLandmarks;
    okb_marg_job job{};
    const okb_marg_job* deviceJob() {
      if (!anything) return nullptr;
      job = okb_marg_job{};
      job.n_blocks = (int32_t)blocks.size(); job.n_imu_terms = (int32_t)jobTerms.size(); job.n_sb_priors = (int32_t)jobSbPriors.size();
      job.n_landmarks = (int32_t)jobLandmarks.size();
      job.block_kind = kinds.data(); job.block_idx = idx.data(); job.block_prev = prev.data(); job.block_marginalize = margFlag.data();
      job.imu_terms = jobTerms.data(); job.sb_priors = jobSbPriors.data(); job.landmarks = jobLandmarks.data();
      return &job;
    }
  };
  // Estimates as the download returns them, sized for the window as it is now.
  struct Estimates { std::vector<double> poses, sbs, lms, q; };

 public:
  using Capacity = EstimatorCapacity;

  // A standalone session: a group of one (its own context with one window), slot 0.
  explicit Estimator(int device = 0, Capacity cap = Capacity());
  // A session of `group`: takes the group's lowest free slot (throws std::runtime_error when the group is full) and
  // gives it back on destruction.  The slot's window from a previous occupant is replaced by this session's first
  // full upload (its first optimize / applyMarginalizationStrategy), which also drops its pending commands and prior.
  explicit Estimator(EstimatorGroup& group, Capacity cap = Capacity());
  ~Estimator();
  Estimator(const Estimator&) = delete;
  Estimator& operator=(const Estimator&) = delete;

  // ---- sensor configuration (Estimator.cpp:82-110).  The camera geometry and T_SC travel with the call because the
  // reference reads them from the MultiFrame in addStates / addObservation.
  int addCamera(const ExtrinsicsEstimationParameters& p, const okb_camera& geometry, const Pose7& T_SC) {
    if (p.sigma_absolute_translation > 1e-8 || p.sigma_absolute_orientation > 1e-8 || p.sigma_c_relative_translation > 1e-12 ||
        p.sigma_c_relative_orientation > 1e-12)
      throw std::runtime_error("okvis_b200: online extrinsics estimation is not supported by the device solver");
    if (resident_) throw std::runtime_error("okvis_b200: cameras must be added before the first optimize()");
    extrinsicsParams_.push_back(p); cameras_.push_back(geometry); T_SC_.push_back(T_SC);
    return (int)cameras_.size() - 1;
  }
  int addImu(const okb_imu_params& p) { if (hasImu_) return -1; imu_ = p; hasImu_ = true; return 0; }
  void clearCameras() { extrinsicsParams_.clear(); cameras_.clear(); T_SC_.clear(); }
  void clearImus() { hasImu_ = false; }

  // ---- Estimator::addStates (Estimator.cpp:110-343): first frame -> gravity-aligned pose + priors; later frames ->
  // propagate the last state through the IMU samples, add an ImuError term.
  // EstimatorGroup::addStates for this session alone: prepareState (checks, first-frame pose and priors), the
  // prediction (okb_imu_propagate_batch) and appendState.
  bool addStates(uint64_t frameId, int64_t timestamp_ns, const std::vector<ImuMeasurement>& imu, bool asKeyframe);

  // ---- landmarks / observations (Estimator.cpp:345-413, implementation/Estimator.hpp:43-90)
  bool addLandmark(uint64_t landmarkId, const Vec4& hp) {
    if (landmarks_.count(landmarkId)) return false;
    MapPoint mp; mp.id = landmarkId; mp.point = hp;
    mp.distance = std::fabs(hp[3]) > 1e-8 ? std::sqrt(hp[0] * hp[0] + hp[1] * hp[1] + hp[2] * hp[2]) / std::fabs(hp[3]) : 1e300;
    landmarks_[landmarkId] = mp;
    uint32_t slot;
    if (!freeSlots_.empty()) { slot = *freeSlots_.begin(); freeSlots_.erase(freeSlots_.begin()); }
    else slot = slotCount_++;
    if ((int)slot >= cap_.landmarks) throw std::runtime_error("okvis_b200: landmark capacity of the resident window exceeded");
    lmSlot_[landmarkId] = slot; slotOwner_[slot] = landmarkId;
    if (resident_) throwIfFailed(ctx_, okb_window_set_landmarks(ctx_, slot_, 1, &slot, hp.data()));
    return true;
  }
  // returns the residual block id (0 = duplicate observation, like the reference's NULL)
  uint64_t addObservation(uint64_t landmarkId, uint64_t poseId, size_t camIdx, size_t keypointIdx, const double kp[2], double keypointSize) {
    auto it = landmarks_.find(landmarkId);
    if (it == landmarks_.end() || !states_.count(poseId) || camIdx >= cameras_.size()) throw std::runtime_error("okvis_b200: addObservation on unknown ids");
    KeypointIdentifier kid; kid.frameId = poseId; kid.cameraIndex = camIdx; kid.keypointIndex = keypointIdx;
    if (it->second.observations.count(kid)) return 0;
    // one reprojection error per (landmark, frame, camera): the device grid holds one cell per such triple
    for (auto& o : it->second.observations)
      if (o.first.frameId == poseId && o.first.cameraIndex == camIdx) return 0;
    Obs o; o.lm = landmarkId; o.pose = poseId; o.cam = (uint32_t)camIdx; o.kp = keypointIdx; o.z[0] = kp[0]; o.z[1] = kp[1];
    o.sqrt_info = 8.0 / keypointSize;       // information = 64/size^2 * I2
    const uint64_t id = ++nextResidualId_;
    obs_[id] = o;
    it->second.observations[kid] = id;
    if (resident_) { okb_observation d = deviceObs(o); throwIfFailed(ctx_, okb_window_add_observations(ctx_, slot_, 1, &d)); }
    setStoreLandmark(poseId, camIdx, keypointIdx, landmarkId, true);
    return id;
  }
  bool removeObservation(uint64_t residualBlockId) {
    auto it = obs_.find(residualBlockId);
    if (it == obs_.end()) return false;
    if (resident_) {
      okb_obs_key k{posePos(it->second.pose), lmSlot_.at(it->second.lm), it->second.cam, 0};
      throwIfFailed(ctx_, okb_window_remove_observations(ctx_, slot_, 1, &k));
    }
    // the keypoint keeps its landmark but no longer holds the observation (skipB of doSetup, :238-250)
    setStoreLandmark(it->second.pose, it->second.cam, it->second.kp, it->second.lm, false);
    eraseObsHost(it);
    return true;
  }
  bool removeObservation(uint64_t landmarkId, uint64_t poseId, size_t camIdx, size_t keypointIdx) {
    auto it = landmarks_.find(landmarkId);
    if (it == landmarks_.end()) return false;
    KeypointIdentifier kid; kid.frameId = poseId; kid.cameraIndex = camIdx; kid.keypointIndex = keypointIdx;
    auto o = it->second.observations.find(kid);
    if (o == it->second.observations.end()) return false;
    return removeObservation(o->second);
  }

  // ---- Estimator::applyMarginalizationStrategy (Estimator.cpp:434-773).  Bookkeeping on the host, numerics
  // (linearisation at the first-estimate points, Schur complements, eigen-factorisation) on the device.
  // EstimatorGroup's form for this session alone: planMarginalization -> okb_window_marginalize_batch -> finishMarginalization.
  bool applyMarginalizationStrategy(size_t numKeyframes, size_t numImuFrames, MapPointVector& removedLandmarks);
  bool applyMarginalizationStrategy(size_t numKeyframes, size_t numImuFrames) { MapPointVector r; return applyMarginalizationStrategy(numKeyframes, numImuFrames, r); }

  // ---- Estimator::optimize (Estimator.cpp:843-906) + setOptimizationTimeLimit (:909-929)
  bool setOptimizationTimeLimit(double timeLimit, int minIterations) { timeLimit_ = timeLimit; minIterations_ = minIterations; return true; }
  // EstimatorGroup::optimize for this session alone.
  void optimize(size_t numIter, size_t /*numThreads*/ = 1, bool /*verbose*/ = false);
  const okb_summary& summary() const { return summary_; }
  // bytes the last commit of the window moved host -> device (a frame's worth once the window is resident; 0 before)
  int64_t lastUploadBytes() const { return resident_ ? okb_window_h2d_bytes(ctx_, slot_) : 0; }

 private:
  // applyMarginalizationStrategy, plan half: the reference's bookkeeping (removeObservation appends included) and the
  // device job.  p.skip: fewer frames than numImuFrames + 1, nothing to do.
  void planMarginalization(size_t numKeyframes, size_t numImuFrames, MapPointVector& removedLandmarks, MargPlan& p) {
    // keep the newest numImuFrames
    auto rit = states_.rbegin();
    for (size_t k = 0; k < numImuFrames; ++k) { ++rit; if (rit == states_.rend()) return; }
    p.skip = false;
    ensureResident();
    std::vector<uint64_t>& removeFrames = p.removeFrames;
    std::vector<uint64_t>& removeAllButPose = p.removeAllButPose;
    std::vector<uint64_t> allLinearizedFrames;
    size_t countedKeyframes = 0;
    for (; rit != states_.rend(); ++rit) {
      if (!rit->second.isKeyframe || countedKeyframes >= numKeyframes) removeFrames.push_back(rit->first);
      else countedKeyframes++;
      removeAllButPose.push_back(rit->first);
      allLinearizedFrames.push_back(rit->first);
    }
    auto contains = [](const std::vector<uint64_t>& v, uint64_t q) { return std::find(v.begin(), v.end(), q) != v.end(); };
    // the linear system: blocks of the current prior first (their order), newly connected blocks appended in the
    // order MarginalizationError::addResidualBlock meets them
    std::vector<BlockRef>& blocks = p.blocks;
    blocks = margBlocks_;
    std::vector<int32_t>& prev = p.prev;
    prev.resize(blocks.size());
    for (size_t i = 0; i < blocks.size(); ++i) prev[i] = (int32_t)i;
    std::vector<uint8_t>& margFlag = p.margFlag;
    margFlag.assign(blocks.size(), 0);
    auto connect = [&](int kind, uint64_t id) -> size_t {
      for (size_t i = 0; i < blocks.size(); ++i) if (blocks[i].kind == kind && blocks[i].id == id) return i;
      blocks.push_back({kind, id}); prev.push_back(-1); margFlag.push_back(0);
      return blocks.size() - 1;
    };
    std::vector<uint32_t>& jobTerms = p.jobTerms;
    std::vector<uint32_t>& jobSbPriors = p.jobSbPriors;
    std::vector<uint32_t>& jobLandmarks = p.jobLandmarks;
    std::set<size_t> termDone, sbPriorDone;
    auto linearizeTerm = [&](size_t ti) {
      if (!termDone.insert(ti).second) return;
      connect(OKB_BLOCK_POSE, terms_[ti].first); connect(OKB_BLOCK_SPEED_BIAS, terms_[ti].first);
      connect(OKB_BLOCK_POSE, terms_[ti].second); connect(OKB_BLOCK_SPEED_BIAS, terms_[ti].second);
      jobTerms.push_back((uint32_t)ti);
    };
    bool& anything = p.anything;
    // marginalize everything but pose (Estimator.cpp:483-554): the speed/bias block of every frame that left the IMU window
    for (uint64_t fid : removeAllButPose) {
      State& st = states_.at(fid);
      if (!st.hasSb) continue;
      margFlag[connect(OKB_BLOCK_SPEED_BIAS, fid)] = 1;
      anything = true;
      for (size_t ti = 0; ti < terms_.size(); ++ti)
        if (terms_[ti].first == fid || terms_[ti].second == fid) linearizeTerm(ti);
      for (size_t pi = 0; pi < sbPriors_.size(); ++pi)
        if (sbPriors_[pi].frame == fid && sbPriorDone.insert(pi).second) jobSbPriors.push_back((uint32_t)pi);
    }
    // marginalize ONLY pose now (:556-733)
    bool& reDoFixation = p.reDoFixation;
    std::vector<uint64_t>& landmarksGone = p.landmarksGone;      // marginalised or deleted (device slots to clear)
    if (!removeFrames.empty()) {
      const uint64_t currentKfId = allLinearizedFrames.at(0);
      for (uint64_t fid : removeFrames) {
        margFlag[connect(OKB_BLOCK_POSE, fid)] = 1;
        anything = true;
        for (auto& pp : posePriors_) if (pp.frame == fid) reDoFixation = true;       // PoseError is dropped, not linearised
        for (size_t ti = 0; ti < terms_.size(); ++ti)
          if (terms_[ti].first == fid || terms_[ti].second == fid) linearizeTerm(ti);
      }
      for (auto pit = landmarks_.begin(); pit != landmarks_.end();) {
        MapPoint& mp = pit->second;
        bool skipLandmark = true, hasNewObservations = false, justDelete = false, marginalize = true, errorTermAdded = false;
        size_t obsCount = 0;
        for (auto& o : mp.observations) {
          const uint64_t poseId = o.first.frameId;
          if (contains(removeFrames, poseId)) skipLandmark = false;
          if (poseId >= currentKfId) { marginalize = false; hasNewObservations = true; }
          if (contains(allLinearizedFrames, poseId)) obsCount++;
        }
        if (mp.observations.empty()) {
          removedLandmarks.push_back(mp); landmarksGone.push_back(pit->first); pit = landmarks_.erase(pit);
          continue;
        }
        if (skipLandmark) { ++pit; continue; }
        std::vector<uint64_t> toRemove;
        size_t remaining = mp.observations.size();
        for (auto& o : mp.observations) {
          const uint64_t poseId = o.first.frameId;
          if ((contains(removeFrames, poseId) && hasNewObservations) || (!contains(allLinearizedFrames, poseId) && marginalize)) {
            toRemove.push_back(o.second); --remaining;
          } else if (marginalize && contains(allLinearizedFrames, poseId)) {
            if (obsCount < 2) { toRemove.push_back(o.second); --remaining; }
            else { errorTermAdded = true; connect(OKB_BLOCK_POSE, poseId); }
          }
          if (remaining == 0) { justDelete = true; marginalize = false; }
        }
        for (uint64_t rid : toRemove) removeObservation(rid);
        if (justDelete) {
          removedLandmarks.push_back(mp); landmarksGone.push_back(pit->first); pit = landmarks_.erase(pit);
          continue;
        }
        if (marginalize && errorTermAdded) {
          jobLandmarks.push_back(lmSlot_.at(pit->first));
          removedLandmarks.push_back(mp); landmarksGone.push_back(pit->first); pit = landmarks_.erase(pit);
          continue;
        }
        ++pit;
      }
    }
    // ---- the job for the numerics on the device (positions as the window is NOW)
    if (anything) {
      p.kinds.resize(blocks.size());
      p.idx.resize(blocks.size());
      for (size_t i = 0; i < blocks.size(); ++i) { p.kinds[i] = blocks[i].kind; p.idx[i] = blocks[i].kind == OKB_BLOCK_POSE ? posePos(blocks[i].id) : sbPos(blocks[i].id); }
    }
  }
  // applyMarginalizationStrategy, finish half (after the device job ran): adopt the kept blocks, make the same
  // structural edits on the device and in the host maps, re-fix the first pose.
  void finishMarginalization(const MargPlan& p) {
    const std::vector<uint64_t>& removeFrames = p.removeFrames;
    auto contains = [](const std::vector<uint64_t>& v, uint64_t q) { return std::find(v.begin(), v.end(), q) != v.end(); };
    if (p.anything) {
      std::vector<BlockRef> kept;
      for (size_t i = 0; i < p.blocks.size(); ++i) if (!p.margFlag[i]) kept.push_back(p.blocks[i]);
      margBlocks_.swap(kept);
    }
    // ---- the same structural edits on the device and in the host maps
    for (uint64_t lid : p.landmarksGone) {
      // observations still attached to a deleted landmark die with it on the device (okb_window_remove_landmarks)
      for (auto o = obs_.begin(); o != obs_.end();) o = (o->second.lm == lid) ? obs_.erase(o) : std::next(o);
      const uint32_t slot = lmSlot_.at(lid);
      throwIfFailed(ctx_, okb_window_remove_landmarks(ctx_, slot_, 1, &slot));
      lmSlot_.erase(lid); slotOwner_.erase(slot); freeSlots_.insert(slot);
    }
    for (uint64_t fid : p.removeAllButPose) {        // newest first: positions of older blocks do not move
      State& st = states_.at(fid);
      const bool whole = contains(removeFrames, fid);
      if (whole) {
        throwIfFailed(ctx_, okb_window_remove_frame(ctx_, slot_, posePos(fid), st.hasSb ? sbPos(fid) : 0xffffffffu));
        releaseFeatures(fid);
        for (auto o = obs_.begin(); o != obs_.end();) {
          if (o->second.pose == fid) {
            auto lm = landmarks_.find(o->second.lm);
            if (lm != landmarks_.end()) eraseKey(lm->second, o->first);
            o = obs_.erase(o);
          } else ++o;
        }
      } else if (st.hasSb) {
        throwIfFailed(ctx_, okb_window_remove_speed_bias(ctx_, slot_, sbPos(fid)));
      }
      // host mirrors of the device lists (stable compaction, exactly what the interpreter does)
      eraseIf(terms_, [&](const TermRef& t) { return (t.first == fid || t.second == fid); });
      eraseIf(sbPriors_, [&](const SbPrior& q) { return q.frame == fid; });
      if (whole) { eraseIf(posePriors_, [&](const PosePrior& q) { return q.frame == fid; }); states_.erase(fid); }
      else st.hasSb = false;
    }
    if (p.reDoFixation && !states_.empty()) {
      // finally fix the first pose properly (Estimator.cpp:761-770): information diag(1e14 x3, 0, 0, 1e14); the
      // reference's LLT leaves diag(1e7,1e7,1e7,0,0,1e14) as the square root (SURVEY 8a item 8)
      const State& first = states_.begin()->second;
      okb_pose_prior pp{};
      for (int k = 0; k < 7; ++k) pp.meas[k] = first.T_WS[k];
      const double d[6] = {1e7, 1e7, 1e7, 0, 0, 1e14};
      for (int k = 0; k < 6; ++k) pp.sqrt_info[k * 6 + k] = d[k];
      posePriors_.push_back({first.id, pp});
    }
    pushPriors();
  }

  // optimize, host half before the solve: false where there is nothing to solve; else the window is resident, and opt
  // and e are the solve options and the buffers of the download
  bool prepareOptimize(size_t numIter, okb_solve_options& opt, Estimates& e) {
    if (states_.empty() || cameras_.empty()) return false;
    ensureResident();
    opt = okb_solve_options{};
    opt.max_iterations = (int)numIter; opt.min_iterations = minIterations_; opt.time_limit_s = timeLimit_; opt.use_cauchy_loss = 1;
    const size_t K = states_.size(), NSB = numSb(), L = slotCount_ ? slotCount_ : 1;
    e.poses.resize(7 * K); e.sbs.resize(9 * std::max<size_t>(NSB, 1)); e.lms.resize(4 * L); e.q.resize(L);
    return true;
  }
  // optimize, write-back half (Estimator.cpp:880-900): poses, speed/bias, and point + quality for every landmark
  void adoptEstimates(const Estimates& e) {
    size_t i = 0, j = 0;
    for (auto& kv : states_) {
      std::copy(e.poses.begin() + 7 * i, e.poses.begin() + 7 * i + 7, kv.second.T_WS.begin()); ++i;
      if (kv.second.hasSb) { std::copy(e.sbs.begin() + 9 * j, e.sbs.begin() + 9 * j + 9, kv.second.sb.begin()); ++j; }
    }
    for (auto& kv : landmarks_) {
      const uint32_t s = lmSlot_.at(kv.first);
      std::copy(e.lms.begin() + 4 * s, e.lms.begin() + 4 * s + 4, kv.second.point.begin());
      kv.second.quality = e.q[s];
      const Vec4& hp = kv.second.point;
      kv.second.distance = std::fabs(hp[3]) > 1e-8 ? std::sqrt(hp[0] * hp[0] + hp[1] * hp[1] + hp[2] * hp[2]) / std::fabs(hp[3]) : 1e300;
    }
  }

 public:

  // ---- getters / setters (Estimator.cpp:931-1230)
  bool get_T_WS(uint64_t poseId, Pose7& T) const { auto it = states_.find(poseId); if (it == states_.end()) return false; T = it->second.T_WS; return true; }
  bool getSpeedAndBias(uint64_t poseId, uint64_t /*imuIdx*/, SpeedAndBias& sb) const {
    auto it = states_.find(poseId);
    if (it == states_.end() || !it->second.hasSb) return false;
    sb = it->second.sb; return true;
  }
  bool getCameraSensorStates(uint64_t poseId, size_t cameraIdx, Pose7& T_SCi) const {
    if (!states_.count(poseId) || cameraIdx >= T_SC_.size()) return false;
    T_SCi = T_SC_[cameraIdx]; return true;
  }
  bool set_T_WS(uint64_t poseId, const Pose7& T) {
    auto it = states_.find(poseId); if (it == states_.end()) return false;
    it->second.T_WS = T;
    if (resident_) { const uint32_t p = posePos(poseId); throwIfFailed(ctx_, okb_window_set_states(ctx_, slot_, 1, &p, T.data(), 0, nullptr, nullptr)); }
    return true;
  }
  bool setSpeedAndBias(uint64_t poseId, size_t /*imuIdx*/, const SpeedAndBias& sb) {
    auto it = states_.find(poseId); if (it == states_.end() || !it->second.hasSb) return false;
    it->second.sb = sb;
    if (resident_) { const uint32_t p = sbPos(poseId); throwIfFailed(ctx_, okb_window_set_states(ctx_, slot_, 0, nullptr, nullptr, 1, &p, sb.data())); }
    return true;
  }
  bool setCameraSensorStates(uint64_t poseId, size_t cameraIdx, const Pose7& T_SCi) {
    if (!states_.count(poseId) || cameraIdx >= T_SC_.size()) return false;
    if (resident_) throw std::runtime_error("okvis_b200: extrinsics are fixed once the window is resident");
    T_SC_[cameraIdx] = T_SCi; return true;
  }
  bool getLandmark(uint64_t id, MapPoint& mp) const { auto it = landmarks_.find(id); if (it == landmarks_.end()) return false; mp = it->second; return true; }
  size_t getLandmarks(PointMap& landmarks) const { landmarks = landmarks_; return landmarks_.size(); }
  size_t getLandmarks(MapPointVector& landmarks) const {
    landmarks.clear(); landmarks.reserve(landmarks_.size());
    for (auto& kv : landmarks_) landmarks.push_back(kv.second);
    return landmarks_.size();
  }
  bool setLandmark(uint64_t id, const Vec4& hp) {
    auto it = landmarks_.find(id); if (it == landmarks_.end()) return false;
    it->second.point = hp;
    if (resident_) { const uint32_t s = lmSlot_.at(id); throwIfFailed(ctx_, okb_window_set_landmarks(ctx_, slot_, 1, &s, hp.data())); }
    return true;
  }
  bool isLandmarkAdded(uint64_t id) const { return landmarks_.count(id) != 0; }
  bool isLandmarkInitialized(uint64_t id) const { auto it = lmInitialized_.find(id); return it != lmInitialized_.end() && it->second; }
  void setLandmarkInitialized(uint64_t id, bool initialized) {
    if (!landmarks_.count(id)) return;
    lmInitialized_[id] = initialized;
    if (resident_ && featReserved_) {
      const uint32_t s = lmSlot_.at(id);
      const uint8_t f = initialized ? 1 : 0;
      throwIfFailed(ctx_, okb_window_set_landmark_initialized(ctx_, slot_, 1, &s, &f));
    }
  }

  // ---- the frame's features for device-side tracking (Capacity::featureKeypoints > 0): keypoints, descriptors
  // [n][descriptorBytes] and the landmark id of every keypoint (0: none), as the MultiFrame holds them.  The frame takes
  // a feature slot of the window's store; the slot is freed when the frame leaves the window.
  void setFrameFeatures(uint64_t frameId, size_t cam, const std::vector<okb_keypoint>& keypoints, const std::vector<uint8_t>& descriptors,
                        const std::vector<uint64_t>& landmarkIds) {
    if (cap_.featureKeypoints <= 0) throw std::runtime_error("okvis_b200: setFrameFeatures needs Capacity::featureKeypoints > 0");
    if (!states_.count(frameId) || cam >= cameras_.size()) throw std::runtime_error("okvis_b200: setFrameFeatures on unknown ids");
    const size_t n = keypoints.size();
    if (descriptors.size() != n * (size_t)cap_.descriptorBytes || landmarkIds.size() != n)
      throw std::invalid_argument("okvis_b200: setFrameFeatures: descriptor / landmark id count mismatch");
    ensureResident();
    auto fs = takeFeatureSlot(frameId);
    std::vector<int32_t> slots(n, -1);
    std::vector<uint8_t> observed(n, 0);
    for (size_t k = 0; k < n; ++k) {
      auto l = landmarks_.find(landmarkIds[k]);
      if (landmarkIds[k] == 0 || l == landmarks_.end()) continue;
      slots[k] = (int32_t)lmSlot_.at(landmarkIds[k]);
      KeypointIdentifier kid; kid.frameId = frameId; kid.cameraIndex = cam; kid.keypointIndex = k;
      observed[k] = l->second.observations.count(kid) ? 1 : 0;
    }
    throwIfFailed(ctx_, okb_window_set_features(ctx_, slot_, fs->second, (int)cam, (int)n, keypoints.data(), descriptors.data(), slots.data(), observed.data()));
    FrameFeatures& f = feats_[frameId][cam];
    f.kp = keypoints; f.lm = landmarkIds;
  }
  // MultiFrame::setLandmarkId(cam, kp, id) for a frame with features: the frame's host id and the store entry (the
  // landmark's slot if `landmarkId` names a landmark of the graph, else -1; observed as the graph holds it).  This is
  // how a RANSAC outlier is reported (setLandmarkId(..., 0), Frontend.cpp:631, 745): removeObservation alone keeps the
  // store's slot, so the keypoint would still count as matched in the keyframe decision.
  void setFrameLandmarkId(uint64_t frameId, size_t cam, size_t kp, uint64_t landmarkId) {
    auto f = feats_.find(frameId);
    if (f == feats_.end() || cam >= f->second.size() || kp >= f->second[cam].kp.size())
      throw std::runtime_error("okvis_b200: setFrameLandmarkId on a keypoint without features");
    bool observed = false;
    auto l = landmarkId ? landmarks_.find(landmarkId) : landmarks_.end();
    if (l != landmarks_.end()) {
      KeypointIdentifier kid; kid.frameId = frameId; kid.cameraIndex = cam; kid.keypointIndex = kp;
      observed = l->second.observations.count(kid) != 0;
    }
    setStoreLandmark(frameId, cam, kp, l != landmarks_.end() ? landmarkId : 0, observed);
    f->second[cam].lm[kp] = landmarkId;
  }
  // The landmark ids of a frame's keypoints as the store holds them (what the MultiFrame's landmarkId() should say).
  std::vector<uint64_t> frameLandmarkIds(uint64_t frameId, size_t cam) const {
    auto it = feats_.find(frameId);
    if (it == feats_.end() || cam >= it->second.size()) return {};
    return it->second[cam].lm;
  }
  size_t numFrames() const { return states_.size(); }
  size_t numLandmarks() const { return landmarks_.size(); }
  uint64_t currentFrameId() const { return states_.empty() ? 0 : states_.rbegin()->first; }
  uint64_t currentKeyframeId() const {
    for (auto rit = states_.rbegin(); rit != states_.rend(); ++rit) if (rit->second.isKeyframe) return rit->first;
    return 0;
  }
  uint64_t frameIdByAge(size_t age) const { auto it = states_.rbegin(); for (size_t k = 0; k < age && it != states_.rend(); ++k) ++it; return it == states_.rend() ? 0 : it->first; }
  bool isKeyframe(uint64_t id) const { auto it = states_.find(id); return it != states_.end() && it->second.isKeyframe; }
  bool isInImuWindow(uint64_t id) const { auto it = states_.find(id); return it != states_.end() && it->second.hasSb; }
  void setKeyframe(uint64_t id, bool kf) { auto it = states_.find(id); if (it != states_.end()) it->second.isKeyframe = kf; }
  int64_t timestamp(uint64_t id) const { return states_.at(id).t_ns; }
  void printStates(uint64_t poseId, std::ostream& buffer) const {
    auto it = states_.find(poseId);
    if (it == states_.end()) return;
    buffer << "GLOBAL: id=" << poseId << ":pose " << (it->second.isKeyframe ? "(keyframe) " : "") << "SENSOR: ";
    if (it->second.hasSb) buffer << "speedAndBias ";
    for (size_t c = 0; c < T_SC_.size(); ++c) buffer << "(extrinsics " << c << ") ";
    buffer << "\n";
  }

  // Estimator::initPoseFromImu (Estimator.cpp:811-840): align z_W with the mean specific force.
  static bool initPoseFromImu(const std::vector<ImuMeasurement>& imu, Pose7& T_WS) {
    T_WS = Pose7{{0, 0, 0, 0, 0, 0, 1}};
    if (imu.empty()) return false;
    double a[3] = {0, 0, 0};
    for (auto& m : imu) for (int k = 0; k < 3; ++k) a[k] += m.acc[k];
    const double n = std::sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
    if (n == 0) return false;
    const double e[3] = {a[0] / n, a[1] / n, a[2] / n};
    // poseIncrement = -(ez x e_acc).normalized() * acos(ez . e_acc), applied with Transformation::oplus
    double ax[3] = {-e[1], e[0], 0.0};
    const double an = std::sqrt(ax[0] * ax[0] + ax[1] * ax[1]);
    const double angle = std::acos(e[2]);
    if (an < 1e-15) return true;
    const double s = -angle / an;
    const double d[3] = {ax[0] * s, ax[1] * s, 0.0};
    const double half = 0.5 * std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    const double sinc = half > 1e-6 ? std::sin(half) / half : 1.0 - half * half / 6.0;
    T_WS[3] = sinc * 0.5 * d[0]; T_WS[4] = sinc * 0.5 * d[1]; T_WS[5] = sinc * 0.5 * d[2]; T_WS[6] = std::cos(half);
    return true;
  }

  // Slot of the session's window in its context (0 for a standalone Estimator).
  int slot() const { return slot_; }
  // Seconds this session spent inside C-ABI calls that run and wait for device work (prediction, optimize + download,
  // marginalisation); the rest of a call's wall time is host bookkeeping.  Group calls account on the group.
  double deviceSeconds() const { return deviceSeconds_; }

 private:

  // addStates, host check / prepare half: nothing changes; false where addStates returns false before its
  // prediction.  A prediction needs two samples at least (okb_imu_propagate_batch rejects a job with fewer): such a
  // request fails here so that it cannot fail a group's whole prediction batch.
  bool prepareState(uint64_t frameId, int64_t timestamp_ns, const std::vector<ImuMeasurement>& imu, bool asKeyframe, PendingState& p) const {
    if (!hasImu_ || states_.count(frameId)) return false;
    if (!states_.empty() && frameId < states_.rbegin()->first) return false;      // ids grow with time, as IdProvider's do
    State& st = p.st;
    st.id = frameId; st.t_ns = timestamp_ns; st.isKeyframe = asKeyframe; st.hasSb = true;
    p.samples = toSamples(imu);
    if (states_.empty()) {
      if (!initPoseFromImu(imu, st.T_WS)) return false;
      st.sb.fill(0.0);
      for (int k = 0; k < 3; ++k) st.sb[6 + k] = imu_.a0[k];
      return true;
    }
    const State& prev = states_.rbegin()->second;
    if (!prev.hasSb || p.samples.size() < 2) return false;
    st.T_WS = prev.T_WS; st.sb = prev.sb;
    p.predict = true; p.t0_ns = prev.t_ns;
    return true;
  }
  // addStates, append half: after the prediction wrote p.st's pose / speed-bias and p.used
  bool appendState(PendingState& p) {
    State& st = p.st;
    const uint64_t frameId = st.id;
    if (p.predict) {
      if (p.used < 1) return false;
      st.imuFromPrev = p.samples;
      st.hasImuTerm = true;
    } else {
      // PoseError, information diag(1e8,1e8,1e8,0,0,1e8) with the reference's LLT result (SURVEY 8a item 8)
      okb_pose_prior pp{};
      for (int k = 0; k < 7; ++k) pp.meas[k] = st.T_WS[k];
      const double d[6] = {1e4, 1e4, 1e4, 0, 0, 1e8};
      for (int k = 0; k < 6; ++k) pp.sqrt_info[k * 6 + k] = d[k];
      posePriors_.push_back({frameId, pp});
      okb_sb_prior sp{};                      // SpeedAndBiasError(speedAndBias, 1.0, sigma_bg^2, sigma_ba^2)
      for (int k = 0; k < 9; ++k) sp.meas[k] = st.sb[k];
      const double si[9] = {1, 1, 1, 1 / imu_.sigma_bg, 1 / imu_.sigma_bg, 1 / imu_.sigma_bg, 1 / imu_.sigma_ba, 1 / imu_.sigma_ba, 1 / imu_.sigma_ba};
      for (int k = 0; k < 9; ++k) sp.sqrt_info[k * 9 + k] = si[k];
      sbPriors_.push_back({frameId, sp});
    }
    const bool first = states_.empty();
    const uint64_t prevId = first ? 0 : states_.rbegin()->first;
    states_[frameId] = st;
    if (!first) terms_.push_back({prevId, frameId});
    if (resident_) {
      okb_imu_term t{};
      const State& prev = states_.at(prevId);
      t.pose0 = posePos(prevId); t.sb0 = sbPos(prevId); t.pose1 = posePos(frameId); t.sb1 = sbPos(frameId);
      t.t0_ns = prev.t_ns; t.t1_ns = st.t_ns; t.sample_offset = 0; t.sample_count = (uint32_t)p.samples.size();
      throwIfFailed(ctx_, okb_window_add_frame(ctx_, slot_, st.T_WS.data(), st.sb.data(), &t, p.samples.data(), (int)p.samples.size()));
    }
    return true;
  }
  struct Obs { uint64_t lm, pose; uint32_t cam; size_t kp; double z[2]; double sqrt_info; };
  using TermRef = std::pair<uint64_t, uint64_t>;            // ImuError between two frame ids, in the device's list order
  struct PosePrior { uint64_t frame; okb_pose_prior p; };
  struct SbPrior { uint64_t frame; okb_sb_prior p; };

  template <class V, class F> static void eraseIf(V& v, F f) { v.erase(std::remove_if(v.begin(), v.end(), f), v.end()); }
  static std::vector<okb_imu_sample> toSamples(const std::vector<ImuMeasurement>& imu) {
    std::vector<okb_imu_sample> s(imu.size());
    for (size_t i = 0; i < imu.size(); ++i) { s[i].t_ns = imu[i].t_ns; for (int k = 0; k < 3; ++k) { s[i].gyro[k] = imu[i].gyro[k]; s[i].acc[k] = imu[i].acc[k]; } }
    return s;
  }
  uint32_t posePos(uint64_t id) const { return (uint32_t)std::distance(states_.begin(), states_.find(id)); }
  uint32_t sbPos(uint64_t id) const {
    uint32_t p = 0;
    for (auto& kv : states_) { if (kv.first == id) return p; if (kv.second.hasSb) ++p; }
    return p;
  }
  size_t numSb() const { size_t n = 0; for (auto& kv : states_) n += kv.second.hasSb; return n; }
  okb_observation deviceObs(const Obs& o) const {
    okb_observation d{};
    d.pose_idx = posePos(o.pose); d.lm_idx = lmSlot_.at(o.lm); d.ext_idx = o.cam; d.cam_idx = o.cam;
    d.z[0] = o.z[0]; d.z[1] = o.z[1]; d.sqrt_info = o.sqrt_info;
    return d;
  }
  static void eraseKey(MapPoint& mp, uint64_t residualId) {
    for (auto o = mp.observations.begin(); o != mp.observations.end();) o = (o->second == residualId) ? mp.observations.erase(o) : std::next(o);
  }
  // the store's reference of one keypoint (no-op without a store, or when the frame has no features for the camera)
  void setStoreLandmark(uint64_t frameId, size_t cam, size_t kp, uint64_t landmarkId, bool observed) {
    if (!resident_ || !featReserved_) return;
    auto f = feats_.find(frameId);
    if (f == feats_.end() || cam >= f->second.size() || kp >= f->second[cam].kp.size()) return;
    auto s = lmSlot_.find(landmarkId);
    const int32_t k = (int32_t)kp, l = s == lmSlot_.end() ? -1 : (int32_t)s->second;
    const uint8_t o = observed ? 1 : 0;
    throwIfFailed(ctx_, okb_window_set_feature_landmarks(ctx_, slot_, featSlot_.at(frameId), (int)cam, 1, &k, &l, &o));
    f->second[cam].lm[kp] = landmarkId;
  }
  // the frame's feature slot, taken from the free ones when the frame has none yet
  std::map<uint64_t, int32_t>::iterator takeFeatureSlot(uint64_t frameId) {
    auto fs = featSlot_.find(frameId);
    if (fs == featSlot_.end()) {
      if (freeFeat_.empty()) throw std::runtime_error("okvis_b200: no free feature slot (Capacity::frames)");
      fs = featSlot_.emplace(frameId, *freeFeat_.begin()).first;
      freeFeat_.erase(freeFeat_.begin());
      feats_[frameId].resize(cameras_.size());
    }
    return fs;
  }
  void releaseFeatures(uint64_t frameId) {
    auto fs = featSlot_.find(frameId);
    if (fs == featSlot_.end()) return;
    throwIfFailed(ctx_, okb_window_clear_features(ctx_, slot_, fs->second));
    freeFeat_.insert(fs->second);
    featSlot_.erase(fs);
    feats_.erase(frameId);
  }
  // A round of the current frame against frame A: camera camA of frame A against camera camB of the current frame (a
  // 3D-2D tracking round, or the camera pair of a 2D-2D match).
  struct TrackRound { uint64_t frameA; size_t camA, camB; };
  // The rounds of matchToKeyframes (Frontend.cpp:389-452) or, keyframes false, of matchToLastFrame (:484-509), in the
  // reference's order: every camera im -> im against each older frame by age from 1 -- the keyframes, at most
  // maxKeyframes of them, or the last frame unless it is a keyframe.  None before the second frame (:381-384, 470-473).
  std::vector<TrackRound> olderFrameRounds(bool keyframes, size_t maxKeyframes) const {
    std::vector<uint64_t> older;
    if (keyframes) {
      for (size_t age = 1; age < states_.size() && older.size() < maxKeyframes; ++age)
        if (isKeyframe(frameIdByAge(age))) older.push_back(frameIdByAge(age));
    } else if (states_.size() > 1 && !isKeyframe(frameIdByAge(1))) {
      older.push_back(frameIdByAge(1));
    }
    std::vector<TrackRound> rounds;
    for (uint64_t a : older)
      for (size_t im = 0; im < cameras_.size(); ++im) rounds.push_back(TrackRound{a, im, im});
    return rounds;
  }
  // One okb_track_3d2d_batch job of this session: frame B = currentFrameId against `rounds`; rounds without features
  // on either side are dropped.  finishTrack applies the results through addObservation.
  struct TrackPlan {
    uint64_t frameB = 0;
    std::vector<okb_track_round> rounds;
    std::vector<okb_track_assoc> assoc;
    std::vector<uint32_t> uninit;
    std::vector<int32_t> numMatches, numUncertain;
    int32_t nAssoc = 0, nUninit = 0;
    okb_track_job job{};
  };
  bool planTrackRounds(uint64_t currentFrameId, const std::vector<TrackRound>& rounds, float threshold, TrackPlan& p) {
    auto fb = featSlot_.find(currentFrameId);
    if (fb == featSlot_.end()) return false;
    size_t sumA = 0, sumB = 0;
    const auto& B = feats_.at(currentFrameId);
    for (const TrackRound& r : rounds) {
      auto fa = featSlot_.find(r.frameA);
      if (fa == featSlot_.end()) continue;
      const auto& A = feats_.at(r.frameA);
      if (A[r.camA].kp.empty() || B[r.camB].kp.empty()) continue;
      p.rounds.push_back(okb_track_round{fa->second, (int32_t)r.camA, (int32_t)r.camB, 0});
      sumA += A[r.camA].kp.size(); sumB += B[r.camB].kp.size();
    }
    if (p.rounds.empty()) return false;
    p.frameB = currentFrameId;
    p.assoc.resize(std::max<size_t>(sumB, 1)); p.uninit.resize(std::max<size_t>(sumA, 1));
    p.numMatches.resize(p.rounds.size()); p.numUncertain.resize(p.rounds.size());
    okb_track_job& j = p.job;
    j.win = slot_; j.pose_b = (int32_t)posePos(currentFrameId);
    j.sb_b = states_.at(currentFrameId).hasSb ? (int32_t)sbPos(currentFrameId) : -1;
    j.feat_slot_b = fb->second; j.threshold = threshold; j.num_best = 4;
    j.n_rounds = (int32_t)p.rounds.size(); j.rounds = p.rounds.data();
    j.assoc = p.assoc.data(); j.assoc_cap = (int32_t)p.assoc.size(); j.n_assoc = &p.nAssoc;
    j.num_matches = p.numMatches.data(); j.num_uncertain = p.numUncertain.data();
    j.uninit = p.uninit.data(); j.uninit_cap = (int32_t)p.uninit.size(); j.n_uninit = &p.nUninit;
    return true;
  }
  // the host half of setBestMatch / doSetup, in the returned order: setLandmarkInitialized(false), addObservation
  void finishTrack(const TrackPlan& p, int& numMatches, int& numUncertainMatches) {
    for (int i = 0; i < p.nUninit; ++i) lmInitialized_[slotOwner_.at(p.uninit[i])] = false;     // the device cleared them
    for (int i = 0; i < p.nAssoc; ++i) {
      const okb_track_assoc& a = p.assoc[i];
      const uint64_t lid = slotOwner_.at((uint32_t)a.lm_slot);
      FrameFeatures& f = feats_.at(p.frameB)[a.cam_b];
      const okb_keypoint& kp = f.kp[a.kp_b];
      f.lm[a.kp_b] = lid;
      const double z[2] = {kp.x, kp.y};
      if (!addObservation(lid, p.frameB, a.cam_b, a.kp_b, z, kp.size))
        setStoreLandmark(p.frameB, a.cam_b, a.kp_b, lid, false);     // refused: the keypoint names it, no observation
    }
    for (int32_t m : p.numMatches) numMatches += m;
    for (int32_t u : p.numUncertain) numUncertainMatches += u;
  }

  // One okb_match2d2d_batch job of this session: a Match2D2D round (frameA, camA) -> (frameB, camB), setFrames(frameA,
  // frameB, camA, camB) -- an older frame against the current one (matchToKeyframes :413-452, matchToLastFrame
  // :499-509), or frameA == frameB for matchStereo's match of two cameras of one frame.  finish2D2D applies the records.
  struct Match2D2DPlan {
    uint64_t frameA = 0, frameB = 0;
    size_t camA = 0, camB = 0;
    std::vector<okb_stereo_match> out;
    int32_t nOut = 0;
    okb_match2d2d_job job{};
  };
  // Throws unless, in the frame, "the keypoint has a landmark id" is "its store slot names a landmark of the graph":
  // the device's view of setBestMatch's lmIdA / lmIdB.  Holds for the current frame before matchStereo names its
  // remaining keypoints; finish2D2D checks the weaker "store slot >= 0 <=> the id names a landmark of the graph".
  void checkFrameIds(uint64_t frameId) const {
    auto f = feats_.find(frameId);
    if (f == feats_.end()) return;
    for (size_t c = 0; c < f->second.size(); ++c)
      for (uint64_t id : f->second[c].lm)
        if (id != 0 && !landmarks_.count(id))
          throw std::runtime_error("okvis_b200: matchStereo: a keypoint of frame " + std::to_string(frameId) +
                                   " names landmark " + std::to_string(id) + ", which is not in the graph");
  }
  bool plan2D2D(uint64_t frameA, size_t camA, uint64_t frameB, size_t camB, float threshold, Match2D2DPlan& p) {
    auto fa = featSlot_.find(frameA), fb = featSlot_.find(frameB);
    if (fa == featSlot_.end() || fb == featSlot_.end()) return false;
    const auto& A = feats_.at(frameA);
    const auto& B = feats_.at(frameB);
    if (A[camA].kp.empty() || B[camB].kp.empty()) return false;
    p.frameA = frameA; p.frameB = frameB; p.camA = camA; p.camB = camB;
    p.out.resize(B[camB].kp.size());
    okb_match2d2d_job& j = p.job;
    j.win = slot_;
    j.pose_a = (int32_t)posePos(frameA); j.feat_slot_a = fa->second; j.cam_a = (int32_t)camA;
    j.pose_b = (int32_t)posePos(frameB); j.feat_slot_b = fb->second; j.cam_b = (int32_t)camB;
    // doSetup's prior (:127-142) scales with the speed of the window's current frame while it is in the IMU window
    const uint64_t cur = currentFrameId();
    j.sb_current = isInImuWindow(cur) ? (int32_t)sbPos(cur) : -1;
    j.threshold = threshold; j.num_best = 4;
    j.out = p.out.data(); j.out_cap = (int32_t)p.out.size(); j.n_out = &p.nOut;
    return true;
  }
  // The host half of setBestMatch's 2D-2D branch (VioKeyframeWindowMatchingAlgorithm.cpp:371-481), record by record.
  // Returns numMatches_, the records that reached the landmark bookkeeping.  Throws unless each record's store slots
  // agree with the host ids: slot >= 0 exactly when the id names a landmark of the graph, and then its slot.
  template <class NewId>
  int finish2D2D(const Match2D2DPlan& p, const NewId& newId) {
    auto& FA = feats_.at(p.frameA)[p.camA];
    auto& FB = feats_.at(p.frameB)[p.camB];
    auto agrees = [&](uint64_t id, int32_t slot) {
      auto s = id ? lmSlot_.find(id) : lmSlot_.end();
      return s == lmSlot_.end() ? slot < 0 : slot >= 0 && s->second == (uint32_t)slot;
    };
    int numMatches = 0;
    for (int i = 0; i < p.nOut; ++i) {
      const okb_stereo_match& r = p.out[i];
      const uint64_t idA = FA.lm[r.kp_a], idB = FB.lm[r.kp_b];
      if (!agrees(idA, r.lm_slot_a) || !agrees(idB, r.lm_slot_b))
        throw std::runtime_error("okvis_b200: 2D-2D match: the store and the frames' landmark ids disagree");
      if (idA != 0 && idB != 0) continue;          // both carry an id, on the host only at least one of them (:373-375)
      ++numMatches;
      const bool cbi = r.can_be_initialized != 0;
      const Vec4 hp{{r.hp_W[0], r.hp_W[1], r.hp_W[2], r.hp_W[3]}};
      bool insertA = idA == 0, insertB = idB == 0, insertPoint = false;
      uint64_t lmId;
      if (insertA && insertB) {
        lmId = newId();
        insertPoint = true;
      } else {
        lmId = insertA ? idB : idA;
        if (!landmarks_.count(lmId)) insertPoint = insertA = insertB = true;   // named on the host only: add it
      }
      if (insertPoint) {
        addLandmark(lmId, hp);
        setLandmarkInitialized(lmId, cbi);
      } else if (cbi) {
        setLandmarkInitialized(lmId, true);
        setLandmark(lmId, hp);
      }
      if (insertA) observeStereo(p.frameA, p.camA, r.kp_a, lmId);
      if (insertB) observeStereo(p.frameB, p.camB, r.kp_b, lmId);
      if (cbi) setLandmark(lmId, hp);
    }
    return numMatches;
  }
  void observeStereo(uint64_t frameId, size_t cam, size_t k, uint64_t lmId) {
    FrameFeatures& f = feats_.at(frameId)[cam];
    f.lm[k] = lmId;
    const double z[2] = {f.kp[k].x, f.kp[k].y};
    if (!addObservation(lmId, frameId, cam, k, z, f.kp[k].size))
      setStoreLandmark(frameId, cam, k, lmId, false);      // refused: the keypoint names it, no observation
  }
  // matchStereo's last loop (Frontend.cpp:563-571): every keypoint still without an id gets one, in (camera, keypoint)
  // order.  Frame bookkeeping only: the store keeps -1 for them, as no landmark of the graph has that id.
  template <class NewId>
  void nameRemainingKeypoints(uint64_t frameId, const NewId& newId) {
    auto f = feats_.find(frameId);
    if (f == feats_.end()) return;
    for (auto& cam : f->second)
      for (auto& id : cam.lm)
        if (id == 0) id = newId();
  }

  // One okb_keyframe_overlap_batch job of this session's frame (every camera).  Throws unless, for every keypoint of
  // the frame, "the host id is not 0" is "its store slot is >= 0" -- the device's view of landmarkId(im, k) != 0.
  void planKeyframe(uint64_t frameId, float overlapThreshold, float matchingRatioThreshold, std::vector<okb_keyframe_cam>& cams,
                    okb_keyframe_result& out, okb_keyframe_job& j) const {
    auto fs = featSlot_.find(frameId);
    if (fs == featSlot_.end()) throw std::runtime_error("okvis_b200: doWeNeedANewKeyframe: frame " + std::to_string(frameId) + " has no features");
    for (const FrameFeatures& f : feats_.at(frameId))
      for (uint64_t id : f.lm)
        if (id != 0 && !landmarks_.count(id))
          throw std::runtime_error("okvis_b200: doWeNeedANewKeyframe: a keypoint of frame " + std::to_string(frameId) + " names landmark " +
                                   std::to_string(id) + ", which is not in the graph (its store slot is -1)");
    cams.assign(cameras_.size(), okb_keyframe_cam{});
    j = okb_keyframe_job{};
    j.win = slot_; j.feat_slot = fs->second; j.n_cams = (int32_t)cameras_.size();
    j.overlap_threshold = overlapThreshold; j.matching_ratio_threshold = matchingRatioThreshold;
    j.cams = cams.data(); j.out = &out;
  }

  // One okb_ransac_3d2d_batch job of this session's frame (every camera) with Frontend::runRansac3d2d's parameters
  // (ransac.threshold_ = 9, max_iterations_ = 50) and `seed`.  finishRansac3d2d applies the device's outliers.
  struct RansacPlan {
    uint64_t frameId = 0;
    std::vector<okb_ransac_outlier> outliers;
    okb_ransac_result result{};
    okb_ransac_job job{};
  };
  void planRansac3d2d(uint64_t frameId, uint64_t seed, RansacPlan& p) {
    auto fs = featSlot_.find(frameId);
    if (fs == featSlot_.end()) throw std::runtime_error("okvis_b200: runRansac3d2d: frame " + std::to_string(frameId) + " has no features");
    size_t n = 0;
    for (const FrameFeatures& f : feats_.at(frameId)) n += f.kp.size();
    p.frameId = frameId;
    p.outliers.assign(std::max<size_t>(n, 1), okb_ransac_outlier{});
    p.result = okb_ransac_result{};
    p.job = okb_ransac_job{};
    p.job.win = slot_; p.job.feat_slot = fs->second; p.job.n_cams = (int32_t)cameras_.size();
    p.job.max_iterations = 50; p.job.threshold = 9.0; p.job.seed = seed;
    p.job.outliers = p.outliers.data(); p.job.outlier_cap = (int32_t)n; p.job.out = &p.result;
  }
  // Frontend.cpp:613-640 for the device's outliers, in correspondence order: removeObservation (when removeOutliers),
  // then the keypoint's id set to 0.  This order, not the reference's: removeObservation rewrites the store entry to
  // (landmark, not observed), which would undo an id cleared before it.  Throws unless each outlier's store slot is the
  // slot of the keypoint's host id.  Returns what runRansac3d2d returns.
  int finishRansac3d2d(const RansacPlan& p, bool removeOutliers) {
    for (int i = 0; i < p.result.n_outliers; ++i) {
      const okb_ransac_outlier& o = p.outliers[i];
      const uint64_t id = feats_.at(p.frameId)[o.cam].lm[o.kp];
      auto s = id ? lmSlot_.find(id) : lmSlot_.end();
      if (s == lmSlot_.end() || s->second != (uint32_t)o.lm_slot)
        throw std::runtime_error("okvis_b200: runRansac3d2d: the store and the frame's landmark ids disagree");
      if (removeOutliers) removeObservation(id, p.frameId, (size_t)o.cam, (size_t)o.kp);
      setFrameLandmarkId(p.frameId, (size_t)o.cam, (size_t)o.kp, 0);
    }
    return p.result.ret;
  }

  // One okb_ransac_2d2d_batch job of Frontend::runRansac2d2d(currentFrameId, olderFrameId, ...) on every camera, with
  // its parameters (threshold_ = 9, max_iterations_ = 50), initialize_pose = initializePose (the caller's
  // initializePose && !isInitialized_) and `seed`.  Returns false when either frame has no features: every camera has
  // then fewer than 10 correspondences and the reference returns -1 with rotationOnly (:802-808).
  // finishRansac2d2d applies the device's outliers and pose.
  struct Ransac2d2dPlan {
    uint64_t frameId = 0;
    std::vector<okb_ransac2d_outlier> outliers;
    okb_ransac2d_result result{};
    okb_ransac2d_job job{};
  };
  bool planRansac2d2d(uint64_t currentFrameId, uint64_t olderFrameId, bool initializePose, uint64_t seed, Ransac2d2dPlan& p) {
    if (!states_.count(currentFrameId) || !states_.count(olderFrameId))
      throw std::runtime_error("okvis_b200: runRansac2d2d: frame " + std::to_string(states_.count(currentFrameId) ? olderFrameId : currentFrameId) +
                               " is not in the window");
    auto fb = featSlot_.find(currentFrameId), fa = featSlot_.find(olderFrameId);
    if (fa == featSlot_.end() || fb == featSlot_.end()) return false;
    size_t n = 0;
    for (const FrameFeatures& f : feats_.at(olderFrameId)) n += f.kp.size();
    p.frameId = currentFrameId;
    p.outliers.assign(std::max<size_t>(n, 1), okb_ransac2d_outlier{});
    p.result = okb_ransac2d_result{};
    p.job = okb_ransac2d_job{};
    p.job.win = slot_;
    p.job.pose_b = (int32_t)posePos(currentFrameId); p.job.feat_slot_b = fb->second;
    p.job.pose_a = (int32_t)posePos(olderFrameId); p.job.feat_slot_a = fa->second;
    p.job.n_cams = (int32_t)cameras_.size(); p.job.initialize_pose = initializePose ? 1 : 0;
    p.job.max_iterations = 50; p.job.threshold = 9.0; p.job.seed = seed;
    p.job.outliers = p.outliers.data(); p.job.outlier_cap = (int32_t)n; p.job.out = &p.result;
    return true;
  }
  // Frontend.cpp:735-753 and :756-798 for the device's results.  Each outlier record names the correspondence's B
  // keypoint (okvis_b200.h's one departure): removeObservation (when removeOutliers), then the keypoint's id set to 0,
  // the order of finishRansac3d2d.  A B keypoint that several A keypoints of one landmark matched comes in more than one
  // record; the first applies it, the others find the id already 0 and are skipped.  Throws unless each applied record's
  // store slot is the slot of the keypoint's host id.  With pose_set, set_T_WS(frameId, T_WS) before returning, so the
  // next round sees the pose.  Returns what runRansac2d2d returns and sets rotationOnly.
  int finishRansac2d2d(const Ransac2d2dPlan& p, bool removeOutliers, bool& rotationOnly) {
    for (int i = 0; i < p.result.n_outliers; ++i) {
      const okb_ransac2d_outlier& o = p.outliers[i];
      const uint64_t id = feats_.at(p.frameId)[o.cam].lm[o.kp_b];
      if (id == 0) continue;
      auto s = lmSlot_.find(id);
      if (s == lmSlot_.end() || s->second != (uint32_t)o.lm_slot)
        throw std::runtime_error("okvis_b200: runRansac2d2d: the store and the frame's landmark ids disagree");
      if (removeOutliers) removeObservation(id, p.frameId, (size_t)o.cam, (size_t)o.kp_b);
      setFrameLandmarkId(p.frameId, (size_t)o.cam, (size_t)o.kp_b, 0);
    }
    if (p.result.pose_set) {
      Pose7 T;
      for (int k = 0; k < 7; ++k) T[k] = p.result.T_WS[k];
      set_T_WS(p.frameId, T);
    }
    rotationOnly = p.result.rotation_only != 0;
    return p.result.ret;
  }

  // One okb_detect_describe_store_batch job of this session's frame: images[c] for camera c, detected with `prm` into the
  // frame's feature slot.  checkDetectStore throws what planDetectStore would, without touching anything;
  // planDetectStore takes (or reuses) the frame's feature slot as setFrameFeatures does; finishDetectStore records the
  // host keypoints with every landmark id 0 (the store holds slot -1, observed 0 for them).
  struct DetectStorePlan {
    uint64_t frameId = 0;
    int maxOut = 0;
    std::vector<okb_image_desc> images;
    std::vector<okb_keypoint> kp;         // [camera][maxOut]
    std::vector<int32_t> n;
    okb_detect_store_job job{};
  };
  void checkDetectStore(uint64_t frameId, size_t nImages, const okb_detect_params& prm) const {
    if (cap_.featureKeypoints <= 0) throw std::runtime_error("okvis_b200: detectAndDescribe into the store needs Capacity::featureKeypoints > 0");
    if (!states_.count(frameId))
      throw std::runtime_error("okvis_b200: detectAndDescribe: frame " + std::to_string(frameId) + " is not in the window (call addStates first)");
    if (cap_.featureKeypoints < prm.max_keypoints)
      throw std::invalid_argument("okvis_b200: detectAndDescribe: Capacity::featureKeypoints is below the detector's maximum keypoints");
    if (prm.desc_bytes != cap_.descriptorBytes)
      throw std::invalid_argument("okvis_b200: detectAndDescribe: the descriptor length differs from Capacity::descriptorBytes");
    if (nImages != cameras_.size()) throw std::invalid_argument("okvis_b200: detectAndDescribe: one image per camera");
  }
  void planDetectStore(uint64_t frameId, const std::vector<okb_image_desc>& images, const okb_detect_params& prm, DetectStorePlan& p) {
    checkDetectStore(frameId, images.size(), prm);
    ensureResident();
    auto fs = takeFeatureSlot(frameId);
    const size_t C = cameras_.size();
    p.frameId = frameId;
    p.maxOut = prm.max_keypoints;
    p.images = images;
    p.kp.assign(C * (size_t)p.maxOut, okb_keypoint{});
    p.n.assign(C, 0);
    p.job = okb_detect_store_job{};
    p.job.win = slot_; p.job.feat_slot = fs->second; p.job.n_cams = (int32_t)C;
    p.job.images = p.images.data(); p.job.out_kp = p.kp.data(); p.job.out_desc = nullptr; p.job.n_out = p.n.data();
  }
  // Returns the keypoints per camera; a camera over the detector's candidate capacity (n = -1) keeps its features.
  std::vector<std::vector<okb_keypoint>> finishDetectStore(const DetectStorePlan& p) {
    std::vector<std::vector<okb_keypoint>> out(cameras_.size());
    for (size_t c = 0; c < cameras_.size(); ++c) {
      if (p.n[c] < 0) continue;
      const okb_keypoint* k = p.kp.data() + c * (size_t)p.maxOut;
      out[c].assign(k, k + p.n[c]);
      FrameFeatures& f = feats_.at(p.frameId)[c];
      f.kp = out[c];
      f.lm.assign(out[c].size(), 0);
    }
    return out;
  }

  void eraseObsHost(std::map<uint64_t, Obs>::iterator it) {
    auto lm = landmarks_.find(it->second.lm);
    if (lm != landmarks_.end()) eraseKey(lm->second, it->first);
    obs_.erase(it);
  }
  void pushPriors() {
    if (!resident_) return;
    std::vector<okb_pose_prior> pps; std::vector<okb_sb_prior> sps;
    for (auto& p : posePriors_) { okb_pose_prior q = p.p; q.pose_idx = posePos(p.frame); pps.push_back(q); }
    for (auto& p : sbPriors_) { okb_sb_prior q = p.p; q.sb_idx = sbPos(p.frame); sps.push_back(q); }
    throwIfFailed(ctx_, okb_window_set_priors(ctx_, slot_, (int)pps.size(), pps.data(), (int)sps.size(), sps.data(), nullptr));
  }
  // First contact with the device: the whole graph once (okb_window_upload); everything after that is incremental.
  void ensureResident() {
    if (resident_) return;
    std::vector<double> poses, sbs, ext;
    for (auto& kv : states_) { poses.insert(poses.end(), kv.second.T_WS.begin(), kv.second.T_WS.end()); if (kv.second.hasSb) sbs.insert(sbs.end(), kv.second.sb.begin(), kv.second.sb.end()); }
    for (auto& t : T_SC_) ext.insert(ext.end(), t.begin(), t.end());
    std::vector<uint8_t> extFixed(T_SC_.size(), 1);
    const size_t L = slotCount_ ? slotCount_ : 1;
    std::vector<double> lms(4 * L, 0.0);
    for (auto& kv : landmarks_) std::copy(kv.second.point.begin(), kv.second.point.end(), lms.begin() + 4 * lmSlot_.at(kv.first));
    std::vector<okb_observation> obs;
    for (auto& kv : obs_) obs.push_back(deviceObs(kv.second));
    std::vector<okb_imu_term> terms; std::vector<okb_imu_sample> samples;
    for (auto& tr : terms_) {
      const State& s0 = states_.at(tr.first); const State& s1 = states_.at(tr.second);
      okb_imu_term t{};
      t.pose0 = posePos(tr.first); t.sb0 = sbPos(tr.first); t.pose1 = posePos(tr.second); t.sb1 = sbPos(tr.second);
      t.t0_ns = s0.t_ns; t.t1_ns = s1.t_ns;
      t.sample_offset = (uint32_t)samples.size(); t.sample_count = (uint32_t)s1.imuFromPrev.size();
      samples.insert(samples.end(), s1.imuFromPrev.begin(), s1.imuFromPrev.end());
      terms.push_back(t);
    }
    std::vector<okb_pose_prior> pps; std::vector<okb_sb_prior> sps;
    for (auto& p : posePriors_) { okb_pose_prior q = p.p; q.pose_idx = posePos(p.frame); pps.push_back(q); }
    for (auto& p : sbPriors_) { okb_sb_prior q = p.p; q.sb_idx = sbPos(p.frame); sps.push_back(q); }
    okb_window_desc d{};
    d.n_poses = (int)states_.size(); d.n_speed_bias = (int)numSb(); d.n_extrinsics = (int)T_SC_.size(); d.n_landmarks = (int)L;
    d.n_cameras = (int)cameras_.size(); d.n_obs = (int)obs.size(); d.n_imu_terms = (int)terms.size(); d.n_imu_samples = (int)samples.size();
    d.n_pose_priors = (int)pps.size(); d.n_sb_priors = (int)sps.size();
    d.poses = poses.data(); d.speed_bias = sbs.data(); d.extrinsics = ext.data(); d.extrinsics_fixed = extFixed.data(); d.landmarks = lms.data();
    d.cameras = cameras_.data(); d.obs = obs.data(); d.imu_terms = terms.data(); d.imu_samples = samples.data(); d.imu_params = imu_;
    d.pose_priors = pps.data(); d.sb_priors = sps.data();
    throwIfFailed(ctx_, okb_window_reserve(ctx_, slot_, cap_.frames, cap_.landmarks, cap_.observations, cap_.imu_samples, cap_.marg_dim));
    if (cap_.featureKeypoints > 0)
      throwIfFailed(ctx_, okb_window_reserve_features(ctx_, slot_, cap_.frames, (int)cameras_.size(), cap_.featureKeypoints, cap_.descriptorBytes));
    throwIfFailed(ctx_, okb_window_upload(ctx_, slot_, &d));
    resident_ = true;
    if (cap_.featureKeypoints > 0) {
      // a slot of a group may hold a previous session's store: every feature slot empty, every flag as this session has it
      featReserved_ = true;
      for (int f = 0; f < cap_.frames; ++f) { throwIfFailed(ctx_, okb_window_clear_features(ctx_, slot_, f)); freeFeat_.insert(f); }
      std::vector<uint32_t> idx(cap_.landmarks);
      std::vector<uint8_t> flags(cap_.landmarks, 0);
      for (int s = 0; s < cap_.landmarks; ++s) idx[s] = (uint32_t)s;
      for (auto& kv : lmInitialized_) if (kv.second && lmSlot_.count(kv.first)) flags[lmSlot_.at(kv.first)] = 1;
      throwIfFailed(ctx_, okb_window_set_landmark_initialized(ctx_, slot_, cap_.landmarks, idx.data(), flags.data()));
    }
  }

  std::unique_ptr<EstimatorGroup> own_;      // a standalone session's group of one; declared first, destroyed last
  EstimatorGroup* group_;
  okb_ctx* ctx_;                             // group_'s
  int slot_;
  double deviceSeconds_ = 0;
  Capacity cap_;
  bool resident_ = false;
  std::vector<ExtrinsicsEstimationParameters> extrinsicsParams_;
  std::vector<okb_camera> cameras_;
  std::vector<Pose7> T_SC_;
  okb_imu_params imu_{};
  bool hasImu_ = false;
  std::map<uint64_t, State> states_;
  PointMap landmarks_;
  std::map<uint64_t, bool> lmInitialized_;
  // feature store: feature slot of each frame that has features, free slots, the host copy of the frames' keypoints
  // (addObservation needs their positions / sizes) and of their landmark ids
  struct FrameFeatures { std::vector<okb_keypoint> kp; std::vector<uint64_t> lm; };
  bool featReserved_ = false;
  std::map<uint64_t, int32_t> featSlot_;
  std::set<int32_t> freeFeat_;
  std::map<uint64_t, std::vector<FrameFeatures>> feats_;
  std::map<uint64_t, Obs> obs_;
  uint64_t nextResidualId_ = 0;
  // device mirrors: landmark slots, IMU term / prior lists in the device's order, blocks of the marginalisation prior
  std::map<uint64_t, uint32_t> lmSlot_;
  std::map<uint32_t, uint64_t> slotOwner_;
  std::set<uint32_t> freeSlots_;
  uint32_t slotCount_ = 0;
  std::vector<TermRef> terms_;
  std::vector<PosePrior> posePriors_;
  std::vector<SbPrior> sbPriors_;
  std::vector<BlockRef> margBlocks_;
  double timeLimit_ = -1.0; int minIterations_ = 0;
  okb_summary summary_{};
};

// Many okvis::Estimator sessions in one context: the group owns a context of `max_sessions` windows, each session of
// the group (Estimator(group)) one slot of it.  Member calls of a session work as on a standalone Estimator; the group
// calls below run one per-frame step of the ThreadedKFVio cycle for a list of its sessions with one batched device call:
//   addStates                    -> one okb_imu_propagate_batch for every request that needs a prediction
//   optimize                     -> one okb_optimize_slots per distinct option set + one okb_window_download_slots
//   applyMarginalizationStrategy -> one okb_window_marginalize_batch over the span of the sessions' slots
// Lists may be in any order and need not be contiguous.  A duplicate, a session of another group or a standalone
// Estimator throws std::invalid_argument before anything changes.  Sessions not listed are not committed, waited for,
// read or written.
// Results: each session's estimates, summary and bookkeeping equal, bit for bit, what the same member calls made one
// session at a time in a group of the same max_sessions give, as long as one optimize lists at most SMs/2 sessions
// (66 on an H100; longer batches take another launch shape of the reduced solve) and every camera of its sessions
// uses one distortion model (a batch whose cameras mix models runs the landmark kernel's run-time-switch
// instantiation, which rounds differently).  Against a standalone Estimator the bookkeeping is identical.  So are the
// estimates while a window holds at most 64 * floor(2 * SMs / max_sessions) landmarks; beyond that the one-window
// context splits the landmark sums into more chunks, and the estimates agree to rounding.
// Threading: as for the C-ABI context, the caller serialises group calls and the member calls of the group's sessions
// (what Estimator's estimator_mutex_ does for one session in the reference).  Sessions are destroyed before their group.
class EstimatorGroup {
 public:
  struct StatesRequest {
    Estimator* session;
    uint64_t frameId;
    int64_t timestamp_ns;
    std::vector<ImuMeasurement> imu;
    bool asKeyframe;
  };

  EstimatorGroup(int device, int max_sessions) : max_(max_sessions) {
    if (max_sessions < 1) throw std::invalid_argument("okvis_b200: a group holds at least one session");
    if (okb_ctx_create(device, max_sessions, &ctx_) != OKB_OK) throw std::runtime_error(std::string("okvis_b200: ") + okb_last_error(nullptr));
    for (int s = 0; s < max_sessions; ++s) free_.insert(s);
  }
  ~EstimatorGroup() { okb_ctx_destroy(ctx_); }
  EstimatorGroup(const EstimatorGroup&) = delete;
  EstimatorGroup& operator=(const EstimatorGroup&) = delete;

  int maxSessions() const { return max_; }
  int numSessions() const { return max_ - (int)free_.size(); }
  int64_t kernelLaunches() const { return okb_kernel_launches(ctx_); }
  // Seconds the group calls spent inside the batched C-ABI calls (see Estimator::deviceSeconds).
  double deviceSeconds() const { return deviceSeconds_; }

  // Estimator::addStates for each request; one result per request, as the single call returns it.
  std::vector<bool> addStates(const std::vector<StatesRequest>& requests) {
    std::vector<Estimator*> sessions;
    for (const auto& r : requests) sessions.push_back(r.session);
    validate(sessions);
    return addStates(requests, deviceSeconds_);
  }

  // Estimator::optimize(numIter) for each session: sessions with nothing to solve are skipped as the single call skips
  // them; the rest are solved with one okb_optimize_slots per distinct (numIter, minIterations, timeLimit), then
  // downloaded with one okb_window_download_slots and written back.
  void optimize(const std::vector<Estimator*>& sessions, size_t numIter) {
    validate(sessions);
    optimize(sessions, numIter, deviceSeconds_);
  }

  // Estimator::applyMarginalizationStrategy(numKeyframes, numImuFrames, removed[i]) for each session: every session
  // plans (the host bookkeeping), one okb_window_marginalize_batch runs the jobs, every session finishes.  removed is
  // resized to the list's length if shorter; removed[i] receives what sessions[i] removes.  A failing batch throws
  // std::runtime_error naming the slot (Estimator::slot()) of the session whose job it rejected.
  bool applyMarginalizationStrategy(const std::vector<Estimator*>& sessions, size_t numKeyframes, size_t numImuFrames,
                                    std::vector<MapPointVector>& removed) {
    validate(sessions);
    if (removed.size() < sessions.size()) removed.resize(sessions.size());
    std::vector<MapPointVector*> to;
    for (size_t i = 0; i < sessions.size(); ++i) to.push_back(&removed[i]);
    return applyMarginalizationStrategy(sessions, numKeyframes, numImuFrames, to, deviceSeconds_);
  }

 private:
  friend class Estimator;
  friend class Frontend;
  using Clock = std::chrono::steady_clock;
  static double seconds(Clock::time_point t0) { return std::chrono::duration<double>(Clock::now() - t0).count(); }

  // The bodies of the three group calls and of a session's own calls (on the list {session}), for a validated list.
  // The time of their device calls is added to `deviceTime`: the group's deviceSeconds_ or the session's.
  std::vector<bool> addStates(const std::vector<StatesRequest>& requests, double& deviceTime) {
    const size_t n = requests.size();
    std::vector<Estimator::PendingState> p(n);
    std::vector<char> ok(n, 0);
    std::vector<okb_propagate_job> jobs;
    std::vector<size_t> of;
    for (size_t i = 0; i < n; ++i) {
      const StatesRequest& r = requests[i];
      ok[i] = r.session->prepareState(r.frameId, r.timestamp_ns, r.imu, r.asKeyframe, p[i]);
      if (!ok[i] || !p[i].predict) continue;
      okb_propagate_job j{};
      j.params = &r.session->imu_; j.samples = p[i].samples.data(); j.n_samples = (int32_t)p[i].samples.size();
      j.t0_ns = p[i].t0_ns; j.t1_ns = r.timestamp_ns; j.pose = p[i].st.T_WS.data(); j.speed_bias = p[i].st.sb.data();
      j.n_used = &p[i].used;
      jobs.push_back(j); of.push_back(i);
    }
    if (!jobs.empty()) {
      const auto t0 = Clock::now();
      const int rc = okb_imu_propagate_batch(ctx_, (int)jobs.size(), jobs.data());
      deviceTime += seconds(t0);
      if (rc != OKB_OK) for (size_t i : of) ok[i] = 0;        // a failed prediction: addStates returns false
    }
    std::vector<bool> out(n);
    for (size_t i = 0; i < n; ++i) out[i] = ok[i] && requests[i].session->appendState(p[i]);
    return out;
  }

  void optimize(const std::vector<Estimator*>& sessions, size_t numIter, double& deviceTime) {
    std::vector<Estimator*> live;
    std::vector<okb_solve_options> opt(sessions.size());
    std::vector<Estimator::Estimates> e(sessions.size());
    for (Estimator* s : sessions)                                  // opt[i], e[i]: live[i]'s
      if (s->prepareOptimize(numIter, opt[live.size()], e[live.size()])) live.push_back(s);
    if (live.empty()) return;
    const size_t n = live.size();
    std::vector<int32_t> all(n);
    std::vector<double*> poses(n), sbs(n), lms(n), q(n);
    for (size_t i = 0; i < n; ++i) {
      all[i] = live[i]->slot_;
      poses[i] = e[i].poses.data(); sbs[i] = e[i].sbs.data(); lms[i] = e[i].lms.data(); q[i] = e[i].q.data();
    }
    std::vector<char> done(n, 0);
    const auto t0 = Clock::now();
    for (size_t i = 0; i < n; ++i) {
      if (done[i]) continue;
      std::vector<int32_t> slots;
      std::vector<size_t> members;
      for (size_t k = i; k < n; ++k)
        if (!done[k] && opt[k].min_iterations == opt[i].min_iterations && opt[k].time_limit_s == opt[i].time_limit_s) {
          slots.push_back(live[k]->slot_); members.push_back(k); done[k] = 1;
        }
      std::vector<okb_summary> summ(slots.size());
      const int rc = okb_optimize_slots(ctx_, (int)slots.size(), slots.data(), &opt[i], summ.data());
      if (rc != OKB_OK) { deviceTime += seconds(t0); throwIfFailed(ctx_, rc); }
      for (size_t m = 0; m < members.size(); ++m) live[members[m]]->summary_ = summ[m];
    }
    const int rc = okb_window_download_slots(ctx_, (int)n, all.data(), poses.data(), sbs.data(), lms.data(), q.data());
    deviceTime += seconds(t0);
    throwIfFailed(ctx_, rc);
    for (size_t i = 0; i < n; ++i) live[i]->adoptEstimates(e[i]);
  }

  bool applyMarginalizationStrategy(const std::vector<Estimator*>& sessions, size_t numKeyframes, size_t numImuFrames,
                                    const std::vector<MapPointVector*>& removed, double& deviceTime) {
    const size_t n = sessions.size();
    std::vector<Estimator::MargPlan> p(n);
    for (size_t i = 0; i < n; ++i) sessions[i]->planMarginalization(numKeyframes, numImuFrames, *removed[i], p[i]);
    int lo = max_, hi = -1;
    std::vector<const okb_marg_job*> jobs(max_, nullptr);
    for (size_t i = 0; i < n; ++i) {
      if (const okb_marg_job* j = p[i].deviceJob()) {        // none where the plan skips
        const int s = sessions[i]->slot_;
        jobs[s] = j; lo = std::min(lo, s); hi = std::max(hi, s);
      }
    }
    if (hi >= lo) {
      const auto t0 = Clock::now();
      const int rc = okb_window_marginalize_batch(ctx_, lo, hi - lo + 1, jobs.data() + lo);
      deviceTime += seconds(t0);
      throwIfFailed(ctx_, rc);
    }
    for (size_t i = 0; i < n; ++i) if (!p[i].skip) sessions[i]->finishMarginalization(p[i]);
    return true;
  }

  void validate(const std::vector<Estimator*>& sessions) const {
    std::set<const Estimator*> seen;
    for (size_t i = 0; i < sessions.size(); ++i) {
      const Estimator* e = sessions[i];
      const std::string at = "okvis_b200: EstimatorGroup: entry " + std::to_string(i);
      if (!e) throw std::invalid_argument(at + " is null");
      if (e->group_ != this) throw std::invalid_argument(at + (e->own_ ? " is a standalone Estimator" : " is a session of another group"));
      if (!seen.insert(e).second) throw std::invalid_argument(at + " lists a session twice");
    }
  }
  int takeSlot() {
    if (free_.empty()) throw std::runtime_error("okvis_b200: EstimatorGroup: all " + std::to_string(max_) + " sessions are taken");
    const int s = *free_.begin();
    free_.erase(free_.begin());
    return s;
  }

  okb_ctx* ctx_ = nullptr;
  int max_;
  std::set<int> free_;
  double deviceSeconds_ = 0;
};

inline Estimator::Estimator(int device, Capacity cap)
    : own_(new EstimatorGroup(device, 1)), group_(own_.get()), ctx_(group_->ctx_), slot_(group_->takeSlot()), cap_(cap) {}
inline Estimator::Estimator(EstimatorGroup& group, Capacity cap) : group_(&group), ctx_(group.ctx_), slot_(group.takeSlot()), cap_(cap) {}
// The slot goes back before own_, and with it a standalone session's context, is destroyed.
inline Estimator::~Estimator() { group_->free_.insert(slot_); }

inline bool Estimator::addStates(uint64_t frameId, int64_t timestamp_ns, const std::vector<ImuMeasurement>& imu, bool asKeyframe) {
  return group_->addStates({{this, frameId, timestamp_ns, imu, asKeyframe}}, deviceSeconds_)[0];
}
inline void Estimator::optimize(size_t numIter, size_t, bool) { group_->optimize({this}, numIter, deviceSeconds_); }
inline bool Estimator::applyMarginalizationStrategy(size_t numKeyframes, size_t numImuFrames, MapPointVector& removedLandmarks) {
  return group_->applyMarginalizationStrategy({this}, numKeyframes, numImuFrames, {&removedLandmarks}, deviceSeconds_);
}

}  // namespace okvis_b200
