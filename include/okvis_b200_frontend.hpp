// okvis_b200_frontend.hpp -- C++ host shims above the C-ABI (include/okvis_b200.h) for the two frontend classes the
// hot path replaces:
//   okvis_b200::Frontend      mirrors okvis::Frontend      (okvis_frontend/include/okvis/Frontend.hpp:71-255):
//       detectAndDescribe (Frontend.cpp:92-114 -> Frame::detect / Frame::describe), propagation (Frontend.cpp:274-292
//       -> ImuError::propagation) and the brisk / keyframe parameter accessors (:137-255);
//   okvis_b200::DenseMatcher  mirrors okvis::DenseMatcher  (okvis_matcher/include/okvis/DenseMatcher.hpp:59-212):
//       match<MATCHING_ALGORITHM>() with the epilogue of matchBody (implementation/DenseMatcher.hpp:48-125) on the
//       host and listBIteration + assignbest (DenseMatcher.cpp:69-110) on the device.
// Eigen- and OpenCV-free: images are raw u8 rows, keypoints are okb_keypoint (the cv::KeyPoint fields the reference
// uses), poses are [t(3), q_xyzw(4)].  INTEGRATION.md shows the adaptor an OKVIS build adds around these.
//
// Of Frontend::dataAssociationAndInitialization (Frontend.cpp:116-272) the 3D-2D tracking is provided:
// Frontend::matchToKeyframes3D2D / matchToLastFrame3D2D run the 3D-2D rounds of matchToKeyframes (:389-411) and
// matchToLastFrame (:484-494) on the device (okb_track_3d2d_batch on the window's feature store, filled by
// Estimator::setFrameFeatures) and apply them through Estimator::addObservation; the group forms make one call for many
// sessions of an EstimatorGroup.  Frontend::matchStereo creates the stereo landmarks of the current frame
// (Frontend.cpp:521-572): per overlapping camera pair the 2D-2D match on the device (okb_match2d2d_batch: backProject,
// gated match, stereoTriangulate, getUncertainty), setBestMatch's landmark bookkeeping on the host, then the pair's
// same-frame 3D-2D passes (okb_track_3d2d_batch).  Frontend::matchToKeyframes2D2D / matchToLastFrame2D2D run the 2D-2D
// rounds of matchToKeyframes (:413-452) and matchToLastFrame (:499-509) the same way (okb_match2d2d_batch, one call per
// round, setBestMatch's bookkeeping on the host before the next round).  Frontend::doWeNeedANewKeyframe (:295-369) runs
// on the device (okb_keyframe_overlap_batch on the current frame's store view), and
// Frontend::dataAssociationAndInitialization (:117-271) chains all of these for one frame.  Frontend::runRansac3d2d
// (:575-642) rejects 3D-2D outliers on the device (okb_ransac_3d2d_batch: the adapter's correspondences, the project's
// own sampler and generalised P3P, the reference's score and decision) and applies them through
// Estimator::removeObservation and Estimator::setFrameLandmarkId; with RansacHooks::device3d2d set,
// dataAssociationAndInitialization runs it at both of the reference's call points.  Frontend::runRansac2d2d (:645-810)
// rejects 2D-2D outliers and initialises the pose on the device (okb_ransac_2d2d_batch: the adapter's correspondences,
// the project's own sampler, two-point rotation and five-point solvers, the reference's scores, decision and pose
// chain), applies the outliers the same way and the pose with Estimator::set_T_WS; with RansacHooks::device2d2d set,
// dataAssociationAndInitialization runs it at both of its call points.  Without those flags the hooks keep OpenGV.  Frontend::detectAndDescribe(estimator, frameId, images) detects every camera of a
// frame straight into the frame's feature slot of the estimator's store (okb_detect_describe_store_batch: one device
// call, the descriptors stay on the device), in place of the single-image detectAndDescribe + setFrameFeatures; its
// EstimatorGroup form makes one call for many sessions.  Each call has one body: a group form validates its list once,
// before any device work, and a single form runs the same body on its session alone, in the session's group (a
// standalone Estimator's group of one).
#pragma once
#include <cmath>
#include <cstdint>
#include <functional>
#include <limits>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

#include "okvis_b200.h"
#include "okvis_b200_estimator.hpp"

namespace okvis_b200 {

// Frontend::RansacHooks (declared here so that its defaults hold in Frontend's default arguments): the three places
// where the reference runs RANSAC, each receiving the session index (0 for the single form) and that
// session's initialisation flag.  Without device3d2d / device2d2d the adaptor keeps OpenGV there and reports outliers through
// Estimator::removeObservation and Estimator::setFrameLandmarkId(..., 0).  An empty hook means no RANSAC.
struct FrontendRansacHooks {
  // true: runRansac3d2d on the device at both of its call points, before the hooks there are called -- after the
  // first keyframe's 2D-2D rounds for initialised sessions (:434-436) and after matchToLastFrame's 3D-2D rounds
  // (:496-497) -- one device call for all sessions that reach the point; afterKeyframe is then left with runRansac2d2d
  // (nothing, with device2d2d)
  bool device3d2d = false;
  // true: runRansac2d2d on the device at both of its call points, before the hooks there are called -- after each
  // keyframe's 2D-2D rounds for sessions that are not initialised, with initializePose (:438-446), and after
  // matchToLastFrame's 2D-2D rounds, without (:512-515) -- one device call per point and keyframe index for all sessions
  // that reach it; rotationOnly_tmp then comes from the device and afterKeyframe's return value is not used
  bool device2d2d = false;
  // after each keyframe's 2D-2D rounds of matchToKeyframes (:432-447): runRansac3d2d when kfcounter == 0 and
  // initialised, runRansac2d2d while not initialised; returns rotationOnly_tmp (empty hook: false)
  std::function<bool(size_t session, bool initialized, size_t kfcounter, uint64_t olderFrameId)> afterKeyframe;
  // matchToLastFrame, between its 3D-2D and 2D-2D rounds (:496-497): runRansac3d2d
  std::function<void(size_t session, bool initialized)> afterLastFrame3D2D;
  // matchToLastFrame, after its 2D-2D rounds (:512-515): runRansac2d2d while not initialised
  std::function<void(size_t session, bool initialized)> afterLastFrame2D2D;
};

class Frontend {
 public:
  // own == nullptr: the Frontend creates its own context on `device`; otherwise it borrows the caller's.
  explicit Frontend(size_t numCameras, int device = 0, okb_ctx* shared = nullptr) : numCameras_(numCameras), ctx_(shared), owns_(shared == nullptr) {
    if (owns_ && okb_ctx_create(device, 1, &ctx_) != OKB_OK) throw std::runtime_error(std::string("okvis_b200: ") + okb_last_error(nullptr));
  }
  virtual ~Frontend() { if (owns_) okb_ctx_destroy(ctx_); }
  Frontend(const Frontend&) = delete;
  Frontend& operator=(const Frontend&) = delete;

  // Frontend::detectAndDescribe(cameraIndex, frameOut, T_WC, keypoints): detects on the image of camera `cameraIndex`
  // and describes with the keypoint orientation taken from the gravity direction in that camera (Frame.hpp(impl):128-156).
  // May be called concurrently for different camera indices (one device stream per camera slot), like the reference
  // (ThreadedKFVio.cpp:131, 425).  Returns the number of keypoints; descriptors come back row-contiguous [n][bytes].
  int detectAndDescribe(size_t cameraIndex, const uint8_t* image, int width, int height, int stride, const okb_camera& geometry,
                        const double T_WC[7], std::vector<okb_keypoint>& keypoints, std::vector<uint8_t>& descriptors) {
    if (cameraIndex >= numCameras_) throw std::runtime_error("okvis_b200: camera index out of range");
    double R_CW[9];
    rotationCW(T_WC, R_CW);
    const okb_detect_params p = detectParams();
    keypoints.resize(briskDetectionMaximumKeypoints_);
    descriptors.resize(briskDetectionMaximumKeypoints_ * (size_t)descriptorBytes_);
    int n = 0;
    throwIfFailed(ctx_, okb_detect_describe(ctx_, (int)cameraIndex, image, width, height, stride, &geometry, R_CW, &p, keypoints.data(),
                                            descriptors.data(), (int)briskDetectionMaximumKeypoints_, &n));
    keypoints.resize(n);
    descriptors.resize((size_t)n * descriptorBytes_);
    isInitialized_ = true;
    return n;
  }

  // One camera's image of a frame, as the reference's detectAndDescribe(cameraIndex, frame, T_WC, ...) receives it: the
  // pixels (row stride `stride` bytes) and the camera's pose T_WC [t, q_xyzw].
  struct CameraImage {
    const uint8_t* image = nullptr;
    int width = 0, height = 0, stride = 0;
    Pose7 T_WC{};
  };
  // detectAndDescribe for every camera of a frame, straight into the frame's feature slot of the estimator's window
  // (okb_detect_describe_store_batch: one device call, the descriptors never leave the device).  images[c] is camera c
  // of the estimator, whose geometry is used.  The frame must be in the window (addStates first), and the estimator's
  // Capacity must hold this Frontend's maximum keypoints and descriptor length.  The frame's features then stand as
  // after Estimator::setFrameFeatures with every landmark id 0.  Returns the keypoints per camera, equal to the
  // single-image detectAndDescribe's.
  std::vector<std::vector<okb_keypoint>> detectAndDescribe(Estimator& estimator, uint64_t frameId, const std::vector<CameraImage>& images) {
    return detectStoreGroup(*estimator.group_, {&estimator}, {frameId}, {images})[0];
  }
  // The same for sessions of one EstimatorGroup (any order, each listed once): one okb_detect_describe_store_batch for
  // all of them; results[i] equals the single form's on sessions[i].
  std::vector<std::vector<std::vector<okb_keypoint>>> detectAndDescribe(EstimatorGroup& group, const std::vector<Estimator*>& sessions,
                                                                        const std::vector<uint64_t>& frameIds,
                                                                        const std::vector<std::vector<CameraImage>>& images) {
    group.validate(sessions);
    return detectStoreGroup(group, sessions, frameIds, images);
  }

  // Frontend::propagation (Frontend.cpp:274-292): ImuError::propagation on the device; covariance / jacobian 15x15 or null.
  bool propagation(const okb_imu_sample* imuMeasurements, int n, const okb_imu_params& imuParams, double T_WS_propagated[7], double speedAndBiases[9],
                   int64_t t_start_ns, int64_t t_end_ns, double* covariance, double* jacobian) const {
    if (n < 2) return false;
    int used = 0;
    const int rc = okb_imu_propagate(ctx_, &imuParams, imuMeasurements, n, t_start_ns, t_end_ns, T_WS_propagated, speedAndBiases, covariance, jacobian, &used);
    return rc == OKB_OK && used > 0;
  }

  // ---- accessors (Frontend.hpp:137-255)
  size_t getBriskDetectionOctaves() const { return briskDetectionOctaves_; }
  double getBriskDetectionThreshold() const { return briskDetectionThreshold_; }
  double getBriskDetectionAbsoluteThreshold() const { return briskDetectionAbsoluteThreshold_; }
  size_t getBriskDetectionMaximumKeypoints() const { return briskDetectionMaximumKeypoints_; }
  bool getBriskDescriptionRotationInvariance() const { return briskDescriptionRotationInvariance_; }
  bool getBriskDescriptionScaleInvariance() const { return briskDescriptionScaleInvariance_; }
  double getBriskMatchingThreshold() const { return briskMatchingThreshold_; }
  float getKeyframeInsertionOverlapThershold() const { return keyframeInsertionOverlapThreshold_; }
  float getKeyframeInsertionMatchingRatioThreshold() const { return keyframeInsertionMatchingRatioThreshold_; }
  bool isInitialized() const { return isInitialized_; }
  void setBriskDetectionOctaves(size_t octaves) {
    if (octaves != 0) throw std::runtime_error("okvis_b200: the device detector is single scale (octaves = 0, the value OKVIS ships)");
    briskDetectionOctaves_ = octaves;
  }
  void setBriskDetectionThreshold(double threshold) { briskDetectionThreshold_ = threshold; }
  void setBriskDetectionAbsoluteThreshold(double threshold) { briskDetectionAbsoluteThreshold_ = threshold; }
  void setBriskDetectionMaximumKeypoints(size_t maxKeypoints) { briskDetectionMaximumKeypoints_ = maxKeypoints; }
  void setBriskDescriptionRotationInvariance(bool invariance) { briskDescriptionRotationInvariance_ = invariance; }
  void setBriskDescriptionScaleInvariance(bool invariance) {
    if (invariance) throw std::runtime_error("okvis_b200: scale-invariant description is not built (OKVIS constructs the extractor with scaleInvariant = false)");
    briskDescriptionScaleInvariance_ = invariance;
  }
  void setBriskMatchingThreshold(double threshold) { briskMatchingThreshold_ = threshold; }
  void setKeyframeInsertionOverlapThreshold(float threshold) { keyframeInsertionOverlapThreshold_ = threshold; }
  void setKeyframeInsertionMatchingRatioThreshold(float threshold) { keyframeInsertionMatchingRatioThreshold_ = threshold; }
  void setDescriptorBytes(int bytes) { if (bytes != 48 && bytes != 64) throw std::runtime_error("okvis_b200: 48 or 64 byte descriptors"); descriptorBytes_ = bytes; }
  int descriptorBytes() const { return descriptorBytes_; }
  okb_ctx* context() const { return ctx_; }

  // ---- 3D-2D tracking of the current frame against the window (device: okb_track_3d2d_batch)
  // landmarkIds[cam][k]: the frame's landmark ids after tracking (write them into the MultiFrame); the counts are the sums
  // of numMatches_ / numUncertainMatches_ over the rounds.
  struct TrackResult {
    std::vector<std::vector<uint64_t>> landmarkIds;
    int numMatches = 0, numUncertainMatches = 0;
  };
  // matchToKeyframes' 3D-2D loop (Frontend.cpp:389-411): keyframes by age from 1, every camera im -> im, at most 3
  TrackResult matchToKeyframes3D2D(Estimator& estimator, uint64_t currentFrameId) {
    return trackGroup(*estimator.group_, {&estimator}, {currentFrameId}, true)[0];
  }
  // matchToLastFrame's 3D-2D pass (:484-494): nothing when the last frame is a keyframe
  TrackResult matchToLastFrame3D2D(Estimator& estimator, uint64_t currentFrameId) {
    return trackGroup(*estimator.group_, {&estimator}, {currentFrameId}, false)[0];
  }
  // The same for sessions of one EstimatorGroup (any order, each listed once): one okb_track_3d2d_batch for all of them;
  // results[i] equals the single call's on sessions[i].
  std::vector<TrackResult> matchToKeyframes3D2D(EstimatorGroup& group, const std::vector<Estimator*>& sessions,
                                                const std::vector<uint64_t>& currentFrameIds) {
    group.validate(sessions);
    return trackGroup(group, sessions, currentFrameIds, true);
  }
  std::vector<TrackResult> matchToLastFrame3D2D(EstimatorGroup& group, const std::vector<Estimator*>& sessions,
                                                const std::vector<uint64_t>& currentFrameIds) {
    group.validate(sessions);
    return trackGroup(group, sessions, currentFrameIds, false);
  }

  // ---- 2D-2D landmark initialisation against earlier frames (device: okb_match2d2d_batch)
  // matchToKeyframes' 2D-2D loop (Frontend.cpp:413-452): keyframes by age from 1, at most 2, every camera im -> im, one
  // device call per round with the records applied as setBestMatch does (new landmarks take newId() in the order
  // IdProvider::newId() would hand them out) before the next round: a round may add or initialise a landmark a later
  // round must skip or reuse.  After each keyframe's rounds, afterKeyframe(kfcounter, olderFrameId) -- where the
  // reference runs runRansac3d2d / runRansac2d2d (:432-447).  numMatches sums numMatches_ over the rounds (records that
  // reached the landmark bookkeeping), numUncertainMatches is 0; landmarkIds are the current frame's ids (an older
  // frame's: Estimator::frameLandmarkIds).  Keypoint ids that exist only on the host (matchStereo's last loop) are honoured.
  TrackResult matchToKeyframes2D2D(Estimator& estimator, uint64_t currentFrameId, const std::function<uint64_t()>& newId,
                                   const std::function<void(size_t, uint64_t)>& afterKeyframe = {}) {
    std::function<void(size_t, size_t, uint64_t)> cb;
    if (afterKeyframe) cb = [&](size_t, size_t kf, uint64_t id) { afterKeyframe(kf, id); };
    return match2D2DGroup(*estimator.group_, {&estimator}, {currentFrameId}, {newId}, true, cb)[0];
  }
  // matchToLastFrame's 2D-2D loop (:499-509): nothing when the last frame is a keyframe
  TrackResult matchToLastFrame2D2D(Estimator& estimator, uint64_t currentFrameId, const std::function<uint64_t()>& newId) {
    return match2D2DGroup(*estimator.group_, {&estimator}, {currentFrameId}, {newId}, false, {})[0];
  }
  // The same for sessions of one EstimatorGroup: one okb_match2d2d_batch per round index for every session that has
  // that round, each session's records applied in list order with its own newId; afterKeyframe(session, kfcounter,
  // olderFrameId) runs per session.  results[i] and the ids equal the single call's on sessions[i].
  std::vector<TrackResult> matchToKeyframes2D2D(EstimatorGroup& group, const std::vector<Estimator*>& sessions,
                                                const std::vector<uint64_t>& currentFrameIds,
                                                const std::vector<std::function<uint64_t()>>& newIds,
                                                const std::function<void(size_t, size_t, uint64_t)>& afterKeyframe = {}) {
    group.validate(sessions);
    return match2D2DGroup(group, sessions, currentFrameIds, newIds, true, afterKeyframe);
  }
  std::vector<TrackResult> matchToLastFrame2D2D(EstimatorGroup& group, const std::vector<Estimator*>& sessions,
                                                const std::vector<uint64_t>& currentFrameIds,
                                                const std::vector<std::function<uint64_t()>>& newIds) {
    group.validate(sessions);
    return match2D2DGroup(group, sessions, currentFrameIds, newIds, false, {});
  }

  // ---- stereo landmark initialisation of the current frame (device: okb_match2d2d_batch + okb_track_3d2d_batch)
  // Frontend::matchStereo (Frontend.cpp:521-572).  overlap[i][j]: NCameraSystem::hasOverlap(i, j).  For every pair
  // im0 < im1 that overlaps: the 2D-2D match, its records applied as setBestMatch does (new landmarks take newId() in the
  // order IdProvider::newId() would hand them out), then the 3D-2D passes (frame, im0 -> im1) and (frame, im1 -> im0).
  // Finally every keypoint of the frame still without an id gets newId(), in (camera, keypoint) order -- frame
  // bookkeeping only, reported by TrackResult::landmarkIds / Estimator::frameLandmarkIds.  Throws if a keypoint of the
  // frame names a landmark that is not in the graph.  The counts are those of the 3D-2D passes.
  TrackResult matchStereo(Estimator& estimator, uint64_t frameId, const std::function<uint64_t()>& newId,
                          const std::vector<std::vector<bool>>& overlap) {
    return stereoGroup(*estimator.group_, {&estimator}, {frameId}, {newId}, overlap)[0];
  }
  // The same for sessions of one EstimatorGroup: one okb_match2d2d_batch and one okb_track_3d2d_batch per camera
  // pair for all of them; each session's records are applied in list order with that session's newId.
  std::vector<TrackResult> matchStereo(EstimatorGroup& group, const std::vector<Estimator*>& sessions, const std::vector<uint64_t>& frameIds,
                                       const std::vector<std::function<uint64_t()>>& newIds, const std::vector<std::vector<bool>>& overlap) {
    group.validate(sessions);
    return stereoGroup(group, sessions, frameIds, newIds, overlap);
  }

  // ---- the keyframe decision (device: okb_keyframe_overlap_batch)
  // Frontend::doWeNeedANewKeyframe (Frontend.cpp:295-369) for the frame's features as the store holds them:
  // numFrames() < 2 gives true and an uninitialised Frontend false, both on the host; otherwise one device job with this
  // Frontend's two thresholds.  Throws unless every keypoint of the frame with a host id has a store slot and the reverse
  // (a removed landmark must be reported with Estimator::setFrameLandmarkId).  cams / result (optional) receive the
  // per-camera values and the maxima of the device call, and are left empty when the host answers.
  bool doWeNeedANewKeyframe(const Estimator& estimator, uint64_t currentFrameId, std::vector<okb_keyframe_cam>* cams = nullptr,
                            okb_keyframe_result* result = nullptr) {
    std::vector<std::vector<okb_keyframe_cam>> c;
    std::vector<okb_keyframe_result> r;
    const bool need = keyframeGroup(*estimator.group_, {&estimator}, {currentFrameId}, {(char)(isInitialized_ ? 1 : 0)}, &c, &r)[0];
    if (cams) *cams = c[0];
    if (result) *result = r[0];
    return need;
  }
  // The same for sessions of one EstimatorGroup: one okb_keyframe_overlap_batch for every session that needs the device.
  // One Frontend serves many sessions here, so each session's initialisation flag is passed in.
  std::vector<bool> doWeNeedANewKeyframe(EstimatorGroup& group, const std::vector<Estimator*>& sessions, const std::vector<uint64_t>& frameIds,
                                         const std::vector<char>& initialized, std::vector<std::vector<okb_keyframe_cam>>* cams = nullptr,
                                         std::vector<okb_keyframe_result>* results = nullptr) {
    std::vector<const Estimator*> cs(sessions.begin(), sessions.end());
    group.validate(sessions);
    return keyframeGroup(group, cs, frameIds, initialized, cams, results);
  }

  // ---- 3D-2D outlier rejection (device: okb_ransac_3d2d_batch)
  // Frontend::runRansac3d2d (Frontend.cpp:575-642) on the current frame's features: numFrames() < 2 returns 1 on the
  // host; otherwise one device job (threshold 9, 50 hypotheses, seed = currentFrameId) and, for every outlier,
  // Estimator::removeObservation (when removeOutliers) and then Estimator::setFrameLandmarkId(..., 0), which leaves the
  // keypoint with host id 0, store slot -1 and no observation.  Returns what the reference returns.
  int runRansac3d2d(Estimator& estimator, uint64_t currentFrameId, bool removeOutliers = true) {
    return ransacGroup(*estimator.group_, {&estimator}, {currentFrameId}, removeOutliers)[0];
  }
  // The same for sessions of one EstimatorGroup: one okb_ransac_3d2d_batch for every session with 2 frames or more;
  // results[i] and the removals equal the single call's on sessions[i].
  std::vector<int> runRansac3d2d(EstimatorGroup& group, const std::vector<Estimator*>& sessions, const std::vector<uint64_t>& currentFrameIds,
                                 bool removeOutliers = true) {
    group.validate(sessions);
    return ransacGroup(group, sessions, currentFrameIds, removeOutliers);
  }

  // ---- 2D-2D outlier rejection and pose initialisation (device: okb_ransac_2d2d_batch)
  // Frontend::runRansac2d2d (Frontend.cpp:645-810) between the current frame and an older one: one device job
  // (threshold 9, 50 hypotheses per problem, seed = currentFrameId, initialize_pose = initializePose && !isInitialized_
  // of this Frontend), then Estimator::finishRansac2d2d: every outlier's B keypoint removed (removeObservation when
  // removeOutliers, then setFrameLandmarkId(..., 0)) and, when the device initialised the pose, set_T_WS.  Returns what
  // the reference returns and sets rotationOnly.
  int runRansac2d2d(Estimator& estimator, uint64_t currentFrameId, uint64_t olderFrameId, bool initializePose, bool removeOutliers,
                    bool& rotationOnly) {
    std::vector<char> ro;
    const int r = ransac2dGroup(*estimator.group_, {&estimator}, {currentFrameId}, {olderFrameId},
                                {(char)(initializePose && !isInitialized_ ? 1 : 0)}, removeOutliers, ro)[0];
    rotationOnly = ro[0] != 0;
    return r;
  }
  // The same for sessions of one EstimatorGroup, with each session's own initialisation flag: one okb_ransac_2d2d_batch
  // for all listed sessions; results[i], rotationOnly[i], the removals and the pose equal the single call's on
  // sessions[i] with isInitialized_ = initialized[i].
  std::vector<int> runRansac2d2d(EstimatorGroup& group, const std::vector<Estimator*>& sessions, const std::vector<uint64_t>& currentFrameIds,
                                 const std::vector<uint64_t>& olderFrameIds, bool initializePose, const std::vector<char>& initialized,
                                 bool removeOutliers, std::vector<char>& rotationOnly) {
    group.validate(sessions);
    if (initialized.size() != sessions.size()) throw std::invalid_argument("okvis_b200: one initialisation flag per session");
    std::vector<char> init(sessions.size());
    for (size_t i = 0; i < sessions.size(); ++i) init[i] = initializePose && !initialized[i] ? 1 : 0;
    return ransac2dGroup(group, sessions, currentFrameIds, olderFrameIds, init, removeOutliers, rotationOnly);
  }

  // ---- one frame of Frontend::dataAssociationAndInitialization (Frontend.cpp:117-271)
  using RansacHooks = FrontendRansacHooks;
  struct FrameResult {
    std::vector<std::vector<uint64_t>> landmarkIds;   // the frame's ids per camera after matchStereo
    int num3dMatches = 0;                             // matchToKeyframes' retCtr (its 3D-2D and 2D-2D matches)
    // the keyframe decision's device values (empty when the host answered) and the frame's ids as the decision saw them
    std::vector<okb_keyframe_cam> keyframeCams;
    okb_keyframe_result keyframe{};
    std::vector<std::vector<uint64_t>> keyframeIds;
  };
  // The reference's per-frame sequence, built from the calls above: when numFrames() > 1, matchToKeyframes3D2D and
  // matchToKeyframes2D2D (rotationOnly starts true and takes the first keyframe's afterKeyframe result), isInitialized
  // as at :184-189, *asKeyframe = *asKeyframe || doWeNeedANewKeyframe, then matchToLastFrame3D2D, afterLastFrame3D2D,
  // matchToLastFrame2D2D, afterLastFrame2D2D (the matchToLastFrame part only when the last frame is not a keyframe, as
  // the reference returns early there); otherwise *asKeyframe = true.  Finally matchStereo.  Reads and sets this
  // Frontend's isInitialized_.  setKeyframe(frameId, *asKeyframe) stays with the caller (ThreadedKFVio.cpp:507-525).
  FrameResult dataAssociationAndInitialization(Estimator& estimator, uint64_t frameId, const std::function<uint64_t()>& newId,
                                               const std::vector<std::vector<bool>>& overlap, bool* asKeyframe,
                                               const RansacHooks& hooks = {}) {
    std::vector<char> init{(char)(isInitialized_ ? 1 : 0)}, kf{(char)(*asKeyframe ? 1 : 0)};
    FrameResult r = associateGroup(*estimator.group_, {&estimator}, {frameId}, {newId}, overlap, kf, hooks, init)[0];
    isInitialized_ = init[0] != 0;
    *asKeyframe = kf[0] != 0;
    return r;
  }
  // The same for sessions of one EstimatorGroup, with one flag per session in `asKeyframe` and `initialized` (read and
  // set).  Sessions may differ in camera count: matchStereo runs once per camera count, `overlap` covering the largest.
  // results[i], the flags and every hook call equal the single form's on sessions[i].
  std::vector<FrameResult> dataAssociationAndInitialization(EstimatorGroup& group, const std::vector<Estimator*>& sessions,
                                                            const std::vector<uint64_t>& frameIds,
                                                            const std::vector<std::function<uint64_t()>>& newIds,
                                                            const std::vector<std::vector<bool>>& overlap, std::vector<char>& asKeyframe,
                                                            const RansacHooks& hooks, std::vector<char>& initialized) {
    group.validate(sessions);
    return associateGroup(group, sessions, frameIds, newIds, overlap, asKeyframe, hooks, initialized);
  }

 private:
  // The bodies of the calls above, for a list the group form has validated (a single form lists its session alone
  // and passes the session's group, the group of one of a standalone Estimator included).
  std::vector<bool> keyframeGroup(EstimatorGroup& group, const std::vector<const Estimator*>& sessions, const std::vector<uint64_t>& frameIds,
                                  const std::vector<char>& initialized, std::vector<std::vector<okb_keyframe_cam>>* cams,
                                  std::vector<okb_keyframe_result>* results) {
    const size_t n = sessions.size();
    if (frameIds.size() != n || initialized.size() != n) throw std::invalid_argument("okvis_b200: one frame id and one initialisation flag per session");
    std::vector<bool> need(n, false);
    std::vector<std::vector<okb_keyframe_cam>> c(n);
    std::vector<okb_keyframe_result> r(n, okb_keyframe_result{});
    std::vector<okb_keyframe_job> jobs;
    for (size_t i = 0; i < n; ++i) {
      if (sessions[i]->numFrames() < 2) { need[i] = true; continue; }    // just starting (:299-302)
      if (!initialized[i]) continue;                                     // (:304-305)
      okb_keyframe_job j;
      sessions[i]->planKeyframe(frameIds[i], keyframeInsertionOverlapThreshold_, keyframeInsertionMatchingRatioThreshold_, c[i], r[i], j);
      jobs.push_back(j);
    }
    if (!jobs.empty()) {
      throwIfFailed(group.ctx_, okb_keyframe_overlap_batch(group.ctx_, (int)jobs.size(), jobs.data()));
      for (size_t i = 0; i < n; ++i) if (!c[i].empty()) need[i] = r[i].need_keyframe != 0;
    }
    if (cams) *cams = c;
    if (results) *results = r;
    return need;
  }

  std::vector<FrameResult> associateGroup(EstimatorGroup& group, const std::vector<Estimator*>& sessions, const std::vector<uint64_t>& frameIds,
                                          const std::vector<std::function<uint64_t()>>& newIds, const std::vector<std::vector<bool>>& overlap,
                                          std::vector<char>& asKeyframe, const RansacHooks& hooks, std::vector<char>& initialized) {
    const size_t n = sessions.size();
    if (frameIds.size() != n || newIds.size() != n || asKeyframe.size() != n || initialized.size() != n)
      throw std::invalid_argument("okvis_b200: one frame id, id source and flag pair per session");
    std::vector<FrameResult> out(n);
    // the sessions past their first frame (:142), in list order, with their positions in `sessions`
    std::vector<size_t> at;
    for (size_t i = 0; i < n; ++i) {
      if (sessions[i]->numFrames() > 1) at.push_back(i);
      else asKeyframe[i] = 1;                                            // first frame (:234-235)
    }
    if (!at.empty()) {
      std::vector<Estimator*> s;
      std::vector<uint64_t> f;
      std::vector<std::function<uint64_t()>> ni;
      for (size_t i : at) { s.push_back(sessions[i]); f.push_back(frameIds[i]); ni.push_back(newIds[i]); }
      // matchToKeyframes (:373-460)
      const std::vector<TrackResult> kf3 = trackGroup(group, s, f, true);
      std::vector<char> rotationOnly(at.size(), 1), first(at.size(), 1), deviceRotationOnly(at.size(), 0);
      auto afterKeyframe = [&](size_t k, size_t kf, uint64_t older) {
        const bool hook = hooks.afterKeyframe ? hooks.afterKeyframe(at[k], initialized[at[k]] != 0, kf, older) : false;
        const bool tmp = hooks.device2d2d ? deviceRotationOnly[k] != 0 : hook;
        if (first[k]) { rotationOnly[k] = tmp ? 1 : 0; first[k] = 0; }
      };
      std::function<void(const std::vector<size_t>&, const std::vector<uint64_t>&)> keyframeRansac2d;
      if (hooks.device2d2d)
        keyframeRansac2d = [&](const std::vector<size_t>& ks, const std::vector<uint64_t>& older) {   // !isInitialized_ (:438-442)
          std::vector<Estimator*> rs;
          std::vector<uint64_t> rf, ro;
          std::vector<size_t> rk;
          for (size_t j = 0; j < ks.size(); ++j) {
            deviceRotationOnly[ks[j]] = 0;                                 // rotationOnly_tmp = false (:437)
            if (!initialized[at[ks[j]]]) { rs.push_back(s[ks[j]]); rf.push_back(f[ks[j]]); ro.push_back(older[j]); rk.push_back(ks[j]); }
          }
          if (rs.empty()) return;
          std::vector<char> rot;
          ransac2dGroup(group, rs, rf, ro, std::vector<char>(rs.size(), 1), true, rot);
          for (size_t j = 0; j < rk.size(); ++j) deviceRotationOnly[rk[j]] = rot[j];
        };
      std::function<void(const std::vector<size_t>&)> firstKeyframeRansac;
      if (hooks.device3d2d)
        firstKeyframeRansac = [&](const std::vector<size_t>& ks) {      // kfcounter == 0 && isInitialized_ (:434-436)
          std::vector<Estimator*> rs;
          std::vector<uint64_t> rf;
          for (size_t k : ks) if (initialized[at[k]]) { rs.push_back(s[k]); rf.push_back(f[k]); }
          if (!rs.empty()) ransacGroup(group, rs, rf, true);
        };
      const std::vector<TrackResult> kf2 = match2D2DGroup(group, s, f, ni, true, afterKeyframe, firstKeyframeRansac, keyframeRansac2d);
      for (size_t k = 0; k < at.size(); ++k) {
        out[at[k]].num3dMatches = kf3[k].numMatches + kf2[k].numMatches;
        if (!initialized[at[k]] && !rotationOnly[k]) initialized[at[k]] = 1;     // (:184-189)
      }
      // the keyframe decision (:196)
      std::vector<char> init(at.size());
      for (size_t k = 0; k < at.size(); ++k) init[k] = initialized[at[k]];
      std::vector<const Estimator*> cs(s.begin(), s.end());
      std::vector<std::vector<okb_keyframe_cam>> kc;
      std::vector<okb_keyframe_result> kr;
      const std::vector<bool> need = keyframeGroup(group, cs, f, init, &kc, &kr);
      for (size_t k = 0; k < at.size(); ++k) {
        asKeyframe[at[k]] = (asKeyframe[at[k]] || need[k]) ? 1 : 0;
        FrameResult& o = out[at[k]];
        o.keyframeCams = kc[k]; o.keyframe = kr[k];
        for (size_t c = 0; c < s[k]->cameras_.size(); ++c) o.keyframeIds.push_back(s[k]->frameLandmarkIds(f[k], c));
      }
      // matchToLastFrame (:463-518): nothing when the last frame is a keyframe
      std::vector<char> last(at.size());
      for (size_t k = 0; k < at.size(); ++k) last[k] = s[k]->isKeyframe(s[k]->frameIdByAge(1)) ? 0 : 1;
      trackGroup(group, s, f, false);
      if (hooks.device3d2d) {                                              // (:496-497)
        std::vector<Estimator*> rs;
        std::vector<uint64_t> rf;
        for (size_t k = 0; k < at.size(); ++k) if (last[k]) { rs.push_back(s[k]); rf.push_back(f[k]); }
        if (!rs.empty()) ransacGroup(group, rs, rf, true);
      }
      if (hooks.afterLastFrame3D2D)
        for (size_t k = 0; k < at.size(); ++k) if (last[k]) hooks.afterLastFrame3D2D(at[k], initialized[at[k]] != 0);
      match2D2DGroup(group, s, f, ni, false, {});
      if (hooks.device2d2d) {                                              // !isInitialized_ (:512-515)
        std::vector<Estimator*> rs;
        std::vector<uint64_t> rf, ro;
        for (size_t k = 0; k < at.size(); ++k)
          if (last[k] && !initialized[at[k]]) { rs.push_back(s[k]); rf.push_back(f[k]); ro.push_back(s[k]->frameIdByAge(1)); }
        std::vector<char> rot;
        if (!rs.empty()) ransac2dGroup(group, rs, rf, ro, std::vector<char>(rs.size(), 0), true, rot);
      }
      if (hooks.afterLastFrame2D2D)
        for (size_t k = 0; k < at.size(); ++k) if (last[k]) hooks.afterLastFrame2D2D(at[k], initialized[at[k]] != 0);
    }
    // matchStereo (:237-268), once per camera count
    std::map<size_t, std::vector<size_t>> byCams;
    for (size_t i = 0; i < n; ++i) byCams[sessions[i]->cameras_.size()].push_back(i);
    for (auto& kv : byCams) {
      std::vector<Estimator*> s;
      std::vector<uint64_t> f;
      std::vector<std::function<uint64_t()>> ni;
      for (size_t i : kv.second) { s.push_back(sessions[i]); f.push_back(frameIds[i]); ni.push_back(newIds[i]); }
      std::vector<std::vector<bool>> ov(kv.first, std::vector<bool>(kv.first, false));
      for (size_t a = 0; a < kv.first && a < overlap.size(); ++a)
        for (size_t b = 0; b < kv.first && b < overlap[a].size(); ++b) ov[a][b] = overlap[a][b];
      const std::vector<TrackResult> st = stereoGroup(group, s, f, ni, ov);
      for (size_t k = 0; k < kv.second.size(); ++k) out[kv.second[k]].landmarkIds = st[k].landmarkIds;
    }
    return out;
  }

  std::vector<TrackResult> match2D2DGroup(EstimatorGroup& group, const std::vector<Estimator*>& sessions, const std::vector<uint64_t>& frameIds,
                                          const std::vector<std::function<uint64_t()>>& newIds, bool keyframes,
                                          const std::function<void(size_t, size_t, uint64_t)>& afterKeyframe,
                                          const std::function<void(const std::vector<size_t>&)>& firstKeyframeDone = {},
                                          const std::function<void(const std::vector<size_t>&, const std::vector<uint64_t>&)>& keyframeDone = {}) {
    const size_t n = sessions.size();
    if (frameIds.size() != n || newIds.size() != n) throw std::invalid_argument("okvis_b200: one frame id and one id source per session");
    std::vector<std::vector<Estimator::TrackRound>> rounds(n);
    size_t R = 0;
    for (size_t i = 0; i < n; ++i) {
      rounds[i] = sessions[i]->olderFrameRounds(keyframes, 2);
      R = std::max(R, rounds[i].size());
    }
    std::vector<TrackResult> out(n);
    for (size_t r = 0; r < R; ++r) {
      const std::vector<int> m = match2D2DRound(group, sessions, frameIds, rounds, r, newIds);
      for (size_t i = 0; i < n; ++i) out[i].numMatches += m[i];
      // the sessions whose round r is the last camera's of a keyframe: the end of keyframe r / C's rounds
      std::vector<size_t> closing;
      for (size_t i = 0; i < n; ++i)
        if (keyframes && r < rounds[i].size() && rounds[i][r].camA + 1 == sessions[i]->cameras_.size()) closing.push_back(i);
      if (firstKeyframeDone) {                         // those whose first keyframe's rounds end here, before afterKeyframe
        std::vector<size_t> done;
        for (size_t i : closing) if (r < sessions[i]->cameras_.size()) done.push_back(i);
        if (!done.empty()) firstKeyframeDone(done);
      }
      if (keyframeDone && !closing.empty()) {          // every session whose keyframe's rounds end here, with that keyframe
        std::vector<uint64_t> older;
        for (size_t i : closing) older.push_back(rounds[i][r].frameA);
        keyframeDone(closing, older);
      }
      if (afterKeyframe)
        for (size_t i : closing) afterKeyframe(i, r / sessions[i]->cameras_.size(), rounds[i][r].frameA);
    }
    for (size_t i = 0; i < n; ++i)
      for (size_t c = 0; c < sessions[i]->cameras_.size(); ++c) out[i].landmarkIds.push_back(sessions[i]->frameLandmarkIds(frameIds[i], c));
    return out;
  }

  std::vector<TrackResult> stereoGroup(EstimatorGroup& group, const std::vector<Estimator*>& sessions, const std::vector<uint64_t>& frameIds,
                                       const std::vector<std::function<uint64_t()>>& newIds, const std::vector<std::vector<bool>>& overlap) {
    const size_t n = sessions.size();
    if (frameIds.size() != n || newIds.size() != n) throw std::invalid_argument("okvis_b200: one frame id and one id source per session");
    if (n == 0) return {};
    const size_t C = sessions[0]->cameras_.size();
    if (overlap.size() < C) throw std::invalid_argument("okvis_b200: matchStereo: overlap must be numCameras x numCameras");
    for (size_t i = 0; i < n; ++i) {
      if (sessions[i]->cameras_.size() != C) throw std::invalid_argument("okvis_b200: matchStereo: sessions with different camera counts");
      sessions[i]->checkFrameIds(frameIds[i]);
    }
    std::vector<TrackResult> out(n);
    for (size_t im0 = 0; im0 < C; ++im0)
      for (size_t im1 = im0 + 1; im1 < C; ++im1) {
        if (overlap[im0].size() < C || !overlap[im0][im1]) continue;
        // the pair's rounds: the 2D-2D match (:532-546) is the first, the 3D-2D and 2D-3D passes (:547-553) are both
        std::vector<std::vector<Estimator::TrackRound>> rounds(n);
        for (size_t i = 0; i < n; ++i) rounds[i] = {{frameIds[i], im0, im1}, {frameIds[i], im1, im0}};
        match2D2DRound(group, sessions, frameIds, rounds, 0, newIds);
        track3D2D(group, sessions, frameIds, rounds, out);
      }
    for (size_t i = 0; i < n; ++i) {
      sessions[i]->nameRemainingKeypoints(frameIds[i], newIds[i]);
      for (size_t c = 0; c < C; ++c) out[i].landmarkIds.push_back(sessions[i]->frameLandmarkIds(frameIds[i], c));
    }
    return out;
  }

  // One 2D-2D round for many sessions: session i matches its round rounds[i][r] (none when r is past its rounds) into
  // its frame frameIds[i] -- plan2D2D per session, one okb_match2d2d_batch, finish2D2D per session in list order (new
  // landmarks take newIds[i]()).  Returns each session's numMatches_ of the round.
  std::vector<int> match2D2DRound(EstimatorGroup& group, const std::vector<Estimator*>& sessions, const std::vector<uint64_t>& frameIds,
                                  const std::vector<std::vector<Estimator::TrackRound>>& rounds, size_t r,
                                  const std::vector<std::function<uint64_t()>>& newIds) {
    const size_t n = sessions.size();
    std::vector<Estimator::Match2D2DPlan> plans(n);
    std::vector<char> has(n, 0);
    std::vector<okb_match2d2d_job> jobs;
    for (size_t i = 0; i < n; ++i) {
      if (r >= rounds[i].size()) continue;
      const Estimator::TrackRound& rd = rounds[i][r];
      has[i] = sessions[i]->plan2D2D(rd.frameA, rd.camA, frameIds[i], rd.camB, (float)briskMatchingThreshold_, plans[i]);
      if (has[i]) jobs.push_back(plans[i].job);
    }
    if (!jobs.empty()) throwIfFailed(group.ctx_, okb_match2d2d_batch(group.ctx_, (int)jobs.size(), jobs.data()));
    std::vector<int> numMatches(n, 0);
    for (size_t i = 0; i < n; ++i) if (has[i]) numMatches[i] = sessions[i]->finish2D2D(plans[i], newIds[i]);
    return numMatches;
  }
  // One 3D-2D call for many sessions: session i tracks its frame frameIds[i] in the rounds rounds[i] (planTrackRounds
  // per session; one whose rounds all lack features sits out), one okb_track_3d2d_batch, finishTrack per session in
  // list order, its counts added to out[i].
  void track3D2D(EstimatorGroup& group, const std::vector<Estimator*>& sessions, const std::vector<uint64_t>& frameIds,
                 const std::vector<std::vector<Estimator::TrackRound>>& rounds, std::vector<TrackResult>& out) {
    const size_t n = sessions.size();
    std::vector<Estimator::TrackPlan> plans(n);
    std::vector<char> has(n, 0);
    std::vector<okb_track_job> jobs;
    for (size_t i = 0; i < n; ++i) {
      has[i] = sessions[i]->planTrackRounds(frameIds[i], rounds[i], (float)briskMatchingThreshold_, plans[i]);
      if (has[i]) jobs.push_back(plans[i].job);
    }
    if (!jobs.empty()) throwIfFailed(group.ctx_, okb_track_3d2d_batch(group.ctx_, (int)jobs.size(), jobs.data()));
    for (size_t i = 0; i < n; ++i) if (has[i]) sessions[i]->finishTrack(plans[i], out[i].numMatches, out[i].numUncertainMatches);
  }

  // R_CW = C_WC^T from the quaternion of T_WC
  static void rotationCW(const double T_WC[7], double R_CW[9]) {
    const double x = T_WC[3], y = T_WC[4], z = T_WC[5], w = T_WC[6];
    const double C[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                         2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                         2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
    const double R[9] = {C[0], C[3], C[6], C[1], C[4], C[7], C[2], C[5], C[8]};
    for (int k = 0; k < 9; ++k) R_CW[k] = R[k];
  }
  okb_detect_params detectParams() const {
    okb_detect_params p{};
    p.uniformity_radius = briskDetectionThreshold_;          // the "detection threshold" of the yaml is brisk's uniformity radius (Frontend.cpp:828-831)
    p.absolute_threshold = briskDetectionAbsoluteThreshold_;
    p.max_keypoints = (int32_t)briskDetectionMaximumKeypoints_;
    p.desc_bytes = descriptorBytes_;
    p.rotation_invariance = briskDescriptionRotationInvariance_ ? 1 : 0;
    return p;
  }

  std::vector<std::vector<std::vector<okb_keypoint>>> detectStoreGroup(EstimatorGroup& group, const std::vector<Estimator*>& sessions,
                                                                       const std::vector<uint64_t>& frameIds,
                                                                       const std::vector<std::vector<CameraImage>>& images) {
    const size_t n = sessions.size();
    if (frameIds.size() != n || images.size() != n) throw std::invalid_argument("okvis_b200: one frame id and one image list per session");
    const okb_detect_params prm = detectParams();
    for (size_t i = 0; i < n; ++i) sessions[i]->checkDetectStore(frameIds[i], images[i].size(), prm);   // before any device work
    std::vector<Estimator::DetectStorePlan> plans(n);
    std::vector<okb_detect_store_job> jobs(n);
    for (size_t i = 0; i < n; ++i) {
      Estimator& e = *sessions[i];
      std::vector<okb_image_desc> ims(images[i].size());
      for (size_t c = 0; c < ims.size(); ++c) {
        const CameraImage& im = images[i][c];
        ims[c].img = im.image; ims[c].width = im.width; ims[c].height = im.height; ims[c].stride = im.stride;
        ims[c].cam = e.cameras_[c];
        rotationCW(im.T_WC.data(), ims[c].R_CW);
      }
      e.planDetectStore(frameIds[i], ims, prm, plans[i]);
      jobs[i] = plans[i].job;
    }
    std::vector<std::vector<std::vector<okb_keypoint>>> out(n);
    if (n == 0) return out;
    const int rc = okb_detect_describe_store_batch(group.ctx_, (int)n, jobs.data(), &prm, prm.max_keypoints, 0);
    if (rc != OKB_ERR_CAPACITY) throwIfFailed(group.ctx_, rc);
    for (size_t i = 0; i < n; ++i) out[i] = sessions[i]->finishDetectStore(plans[i]);   // the store and the host agree, also on capacity
    throwIfFailed(group.ctx_, rc);
    isInitialized_ = true;
    return out;
  }

  std::vector<int> ransacGroup(EstimatorGroup& group, const std::vector<Estimator*>& sessions, const std::vector<uint64_t>& frameIds,
                               bool removeOutliers) {
    const size_t n = sessions.size();
    if (frameIds.size() != n) throw std::invalid_argument("okvis_b200: one current frame id per session");
    std::vector<int> out(n, 1);                        // nothing to match against, just starting (:579-582)
    std::vector<Estimator::RansacPlan> plans(n);
    std::vector<char> has(n, 0);
    std::vector<okb_ransac_job> jobs;
    for (size_t i = 0; i < n; ++i) {
      if (sessions[i]->numFrames() < 2) continue;
      sessions[i]->planRansac3d2d(frameIds[i], frameIds[i], plans[i]);
      has[i] = 1;
      jobs.push_back(plans[i].job);
    }
    if (!jobs.empty()) throwIfFailed(group.ctx_, okb_ransac_3d2d_batch(group.ctx_, (int)jobs.size(), jobs.data()));
    for (size_t i = 0; i < n; ++i) if (has[i]) out[i] = sessions[i]->finishRansac3d2d(plans[i], removeOutliers);
    return out;
  }

  std::vector<int> ransac2dGroup(EstimatorGroup& group, const std::vector<Estimator*>& sessions, const std::vector<uint64_t>& frameIds,
                                 const std::vector<uint64_t>& olderIds, const std::vector<char>& initializePose, bool removeOutliers,
                                 std::vector<char>& rotationOnly) {
    const size_t n = sessions.size();
    if (frameIds.size() != n || olderIds.size() != n || initializePose.size() != n)
      throw std::invalid_argument("okvis_b200: one current frame id, older frame id and pose flag per session");
    std::vector<int> out(n, -1);                      // no features: no camera reaches 10 correspondences (:802-808)
    rotationOnly.assign(n, 1);
    std::vector<Estimator::Ransac2d2dPlan> plans(n);
    std::vector<char> has(n, 0);
    std::vector<okb_ransac2d_job> jobs;
    for (size_t i = 0; i < n; ++i) {
      has[i] = sessions[i]->planRansac2d2d(frameIds[i], olderIds[i], initializePose[i] != 0, frameIds[i], plans[i]) ? 1 : 0;
      if (has[i]) jobs.push_back(plans[i].job);
    }
    if (!jobs.empty()) throwIfFailed(group.ctx_, okb_ransac_2d2d_batch(group.ctx_, (int)jobs.size(), jobs.data()));
    for (size_t i = 0; i < n; ++i)
      if (has[i]) {
        bool ro = true;
        out[i] = sessions[i]->finishRansac2d2d(plans[i], removeOutliers, ro);
        rotationOnly[i] = ro ? 1 : 0;
      }
    return out;
  }

  std::vector<TrackResult> trackGroup(EstimatorGroup& group, const std::vector<Estimator*>& sessions, const std::vector<uint64_t>& frameIds,
                                      bool keyframes) {
    if (sessions.size() != frameIds.size()) throw std::invalid_argument("okvis_b200: one current frame id per session");
    const size_t n = sessions.size();
    std::vector<std::vector<Estimator::TrackRound>> rounds(n);
    for (size_t i = 0; i < n; ++i) rounds[i] = sessions[i]->olderFrameRounds(keyframes, 3);
    std::vector<TrackResult> out(n);
    track3D2D(group, sessions, frameIds, rounds, out);
    for (size_t i = 0; i < n; ++i)
      for (size_t c = 0; c < sessions[i]->cameras_.size(); ++c) out[i].landmarkIds.push_back(sessions[i]->frameLandmarkIds(frameIds[i], c));
    return out;
  }

  size_t numCameras_;
  okb_ctx* ctx_;
  bool owns_;
  bool isInitialized_ = false;
  // defaults of Frontend::Frontend (Frontend.cpp:59-81)
  size_t briskDetectionOctaves_ = 0;
  double briskDetectionThreshold_ = 50.0;
  double briskDetectionAbsoluteThreshold_ = 800.0;
  size_t briskDetectionMaximumKeypoints_ = 450;
  bool briskDescriptionRotationInvariance_ = true;
  bool briskDescriptionScaleInvariance_ = false;
  double briskMatchingThreshold_ = 60.0;
  float keyframeInsertionOverlapThreshold_ = 0.6f;
  float keyframeInsertionMatchingRatioThreshold_ = 0.2f;
  int descriptorBytes_ = 48;
};

// okvis::DenseMatcher.  MATCHING_ALGORITHM_T provides what okvis::MatchingAlgorithm provides (doSetup, sizeA, sizeB,
// skipA, skipB, distanceThreshold, distanceRatioThreshold, reserveMatches, setBestMatch) plus direct access to the
// binary descriptors instead of the per-pair distance() callback:
//   const uint8_t* descriptorsA() / descriptorsB()   row-contiguous [size][descriptorBytes()]
// (with the pure Hamming MatchingAlgorithm of testMatcher.cpp / cfg-3 the two are the same thing; the production
// VioKeyframeWindowMatchingAlgorithm gates distance() geometrically -- use candidates() below for that one).
class DenseMatcher {
 public:
  typedef float distance_t;
  struct Pairing {
    Pairing() : indexA(-1), distance(std::numeric_limits<float>::max()) {}
    Pairing(int ia, distance_t d) : indexA(ia), distance(d) {}
    bool operator<(const Pairing& rhs) const { return distance < rhs.distance; }
    int indexA;
    distance_t distance;
  };
  DenseMatcher(okb_ctx* ctx, unsigned char /*numMatcherThreads*/ = 8, unsigned char numBest = 4, bool useDistanceRatioThreshold = false)
      : ctx_(ctx), numBest_(numBest), useDistanceRatioThreshold_(useDistanceRatioThreshold) {}

  // DenseMatcher::match (implementation/DenseMatcher.hpp:48-122) for a matching algorithm whose distance() is the plain
  // descriptor distance.
  template <typename MATCHING_ALGORITHM_T>
  void match(MATCHING_ALGORITHM_T& matchingAlgorithm) {
    matchingAlgorithm.doSetup();
    matchImpl(matchingAlgorithm, nullptr);
  }

  // The same for a geometry-gated algorithm (VioKeyframeWindowMatchingAlgorithm: distance() = Hamming AND verifyMatch,
  // src/VioKeyframeWindowMatchingAlgorithm.cpp:304-339): the algorithm hands over what its doSetup() prepared --
  // projections + uncertainties (3D-2D) or bearings, ray sigmas and T_AB (2D-2D) -- as an okb_match_gate through
  // matchGate(); the gate runs on the device inside the top-k kernel (okb_hamming_match_gated).
  template <typename MATCHING_ALGORITHM_T>
  void matchGated(MATCHING_ALGORITHM_T& matchingAlgorithm) {
    matchingAlgorithm.doSetup();
    const okb_match_gate& gate = matchingAlgorithm.matchGate();
    matchImpl(matchingAlgorithm, &gate);
  }

  // Candidate lists for a geometry-gated matching algorithm: every B with Hamming distance < threshold per A, ascending
  // B (CSR).  The caller applies verifyMatch (VioKeyframeWindowMatchingAlgorithm.cpp:304-339) on these pairs only.
  void candidates(const uint8_t* A, int nA, const uint8_t* B, int nB, int descriptorBytes, float threshold, std::vector<uint32_t>& rowPtr,
                  std::vector<uint32_t>& colIdx, std::vector<uint16_t>& dist) {
    rowPtr.assign((size_t)nA + 1, 0);
    size_t cap = (size_t)std::max(1024, 8 * (nA + nB));
    for (int attempt = 0; attempt < 2; ++attempt) {
      colIdx.resize(cap); dist.resize(cap);
      const int rc = okb_hamming_candidates(ctx_, A, nA, B, nB, descriptorBytes, threshold, rowPtr.data(), colIdx.data(), dist.data(), (int)cap);
      if (rc == OKB_OK) { colIdx.resize(rowPtr[nA]); dist.resize(rowPtr[nA]); return; }
      if (rc != OKB_ERR_CAPACITY) throwIfFailed(ctx_, rc);
      cap = rowPtr[nA];
    }
    throw std::runtime_error("okvis_b200: candidate capacity");
  }

 private:
  template <typename MATCHING_ALGORITHM_T>
  void matchImpl(MATCHING_ALGORITHM_T& matchingAlgorithm, const okb_match_gate* gate) {
    const int nA = (int)matchingAlgorithm.sizeA(), nB = (int)matchingAlgorithm.sizeB();
    if (nA == 0 || nB == 0) return;
    std::vector<uint8_t> skipA(nA), skipB(nB);
    for (int i = 0; i < nA; ++i) skipA[i] = matchingAlgorithm.skipA(i) ? 1 : 0;
    for (int i = 0; i < nB; ++i) skipB[i] = matchingAlgorithm.skipB(i) ? 1 : 0;
    std::vector<okb_pair> topk((size_t)nA * numBest_), pairs(nB);
    const distance_t thr = matchingAlgorithm.distanceThreshold();
    const int rc = gate ? okb_hamming_match_gated(ctx_, matchingAlgorithm.descriptorsA(), nA, matchingAlgorithm.descriptorsB(), nB,
                                                  matchingAlgorithm.descriptorBytes(), skipA.data(), skipB.data(), thr, numBest_, 0, 0.f, gate,
                                                  topk.data(), pairs.data())
                        : okb_hamming_match(ctx_, matchingAlgorithm.descriptorsA(), nA, matchingAlgorithm.descriptorsB(), nB,
                                            matchingAlgorithm.descriptorBytes(), skipA.data(), skipB.data(), thr, numBest_, 0, 0.f, topk.data(),
                                            pairs.data());
    throwIfFailed(ctx_, rc);
    // epilogue of matchBody (implementation/DenseMatcher.hpp:92-122), ascending B
    matchingAlgorithm.reserveMatches((size_t)nB);
    const distance_t ratio = matchingAlgorithm.distanceRatioThreshold();
    for (int b = 0; b < nB; ++b) {
      if (!(pairs[b].distance < thr)) continue;
      if (useDistanceRatioThreshold_) {
        const okb_pair* best = &topk[(size_t)pairs[b].index_a * numBest_];
        if (numBest_ > 1 && best[1].index_a != -1) {
          if (!(best[0].distance == 0 || best[1].distance / best[0].distance > ratio)) continue;
        }
      }
      matchingAlgorithm.setBestMatch((size_t)pairs[b].index_a, (size_t)b, pairs[b].distance);
    }
  }

  okb_ctx* ctx_;
  int numBest_;
  bool useDistanceRatioThreshold_;
};

}  // namespace okvis_b200
