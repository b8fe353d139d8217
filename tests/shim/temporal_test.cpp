// Exercises the 2D-2D rounds across time through the C++ mirror: Frontend::matchToKeyframes2D2D / matchToLastFrame2D2D
// and their EstimatorGroup forms, in the reference's per-frame order (addStates -> features -> matchToKeyframes3D2D ->
// matchToKeyframes2D2D -> matchToLastFrame3D2D -> matchToLastFrame2D2D -> matchStereo -> optimize ->
// applyMarginalizationStrategy(5, 3)).  No landmark is created from the scene's truth.  Prints one JSON line per mode;
// tests/test_gpu_temporal_mirror.py checks them.
//   temporal_test.bin --no-gpu   the mirror fails loudly without a device
//   temporal_test.bin --cases    one round between two frames with one record of each host-id combination
//   temporal_test.bin --stereo   stereo_test's scene with a fifth of the points masked out of camera 1, 24 frames
//   temporal_test.bin --mono     one camera, starting at rest and accelerating sideways, 24 frames
// --stereo and --mono run 3 standalone sessions and the same 3 sessions in one EstimatorGroup and compare them frame by
// frame, ids and afterKeyframe calls included.
#include <algorithm>
#include <array>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <random>
#include <set>
#include <string>

#include "okvis_b200_frontend.hpp"

using namespace okvis_b200;

namespace {

constexpr double kG = 9.81007, kDt = 0.2;
constexpr int kLandmarks = 300, kDistractors = 40, kFrames = 24, kSessions = 3, kDesc = 48;

okb_camera camera() {
  okb_camera cam{};
  cam.model = OKB_DIST_NONE; cam.width = 752; cam.height = 480; cam.fu = 450; cam.fv = 450; cam.cu = 376; cam.cv = 240;
  return cam;
}

Estimator::Capacity capacity() {
  Estimator::Capacity c;
  c.frames = 12; c.landmarks = 4096; c.observations = 16384; c.imu_samples = 4096;
  c.featureKeypoints = 400; c.descriptorBytes = kDesc;
  return c;
}

struct Image { std::vector<okb_keypoint> kp; std::vector<uint8_t> desc; std::vector<uint64_t> truth; };

// A rig moving along +y: y(t) = vy t + acc t^2 / 2 from the first frame on, the IMU measuring acc after it (the first
// frame's samples see the rig at rest, so that the initial attitude from gravity is level).  Camera c sits
// at y = +-0.055 m and looks along +x.  In `mask` scenes every fifth point is hidden from camera 1.
struct Scene {
  int cams;
  double vy, acc;
  bool mask;
  std::mt19937 rng;
  std::vector<std::array<double, 3>> lmk;
  std::vector<std::array<uint8_t, kDesc>> base;
  int k = 0;
  Scene(int s, int nCams, double v, double a, bool m) : cams(nCams), vy(v), acc(a), mask(m), rng(23 + 31 * s) {
    const double span = vy * kDt * kFrames + 0.5 * acc * (kDt * kFrames) * (kDt * kFrames);
    std::uniform_real_distribution<double> ux(2.0, 6.0), uy(-4.0, 4.0 + span), uz(-1.5, 1.5);
    std::uniform_int_distribution<int> byte(0, 255);
    lmk.resize(kLandmarks); base.resize(kLandmarks);
    for (int l = 0; l < kLandmarks; ++l) {
      lmk[l] = {ux(rng), uy(rng), uz(rng)};
      for (auto& b : base[l]) b = (uint8_t)byte(rng);
    }
  }
  uint64_t frameId() const { return 100 + k; }
  int64_t t(int j) const { return 1000000000LL + (int64_t)(j * kDt * 1e9); }
  double yCam() const { const double tt = k * kDt; return vy * tt + 0.5 * acc * tt * tt; }
  std::vector<ImuMeasurement> imu() const {
    std::vector<ImuMeasurement> meas;
    for (int64_t s = (k == 0 ? t(k) - 50000000LL : t(k - 1) - 5000000LL); s <= t(k) + (k == 0 ? 0 : 5000000LL); s += 5000000LL) {
      ImuMeasurement m{}; m.t_ns = s; m.acc[1] = s > t(0) ? acc : 0.0; m.acc[2] = kG; meas.push_back(m);
    }
    return meas;
  }
  bool keyframe() const { return k % 3 == 0; }
  void configure(Estimator& est) const {
    const okb_camera cam = camera();
    est.addCamera(ExtrinsicsEstimationParameters(), cam, Pose7{{0.0, 0.055, 0.0, -0.5, 0.5, -0.5, 0.5}});
    if (cams > 1) est.addCamera(ExtrinsicsEstimationParameters(), cam, Pose7{{0.0, -0.055, 0.0, -0.5, 0.5, -0.5, 0.5}});
    okb_imu_params imu{};
    imu.a_max = 176; imu.g_max = 7.8; imu.sigma_g_c = 12e-4; imu.sigma_a_c = 8e-3; imu.sigma_bg = 0.03; imu.sigma_ba = 0.1;
    imu.sigma_gw_c = 4e-6; imu.sigma_aw_c = 4e-5; imu.tau = 3600; imu.g = kG; imu.rate = 200;
    est.addImu(imu);
  }
  // the keypoints of frame k in camera c: visible landmarks (pixel noise, a few descriptor bits flipped) and distractors
  Image image(int c) {
    const okb_camera cam = camera();
    std::normal_distribution<double> noise(0.0, 0.3);
    std::uniform_int_distribution<int> flips(0, 4), bit(0, 8 * kDesc - 1), byte(0, 255);
    std::uniform_real_distribution<double> ux(0, 752), uy(0, 480);
    Image im;
    const double y_cam = yCam();
    for (int l = 0; l < kLandmarks; ++l) {
      if (mask && c == 1 && l % 5 == 0) continue;
      const double xs = lmk[l][0], ys = lmk[l][1] - y_cam - (c == 0 ? 0.055 : -0.055), zs = lmk[l][2];
      const double xc = -ys, yc = -zs, zc = xs;
      const double px[2] = {cam.fu * xc / zc + cam.cu, cam.fv * yc / zc + cam.cv};
      if (!(zc > 0.5 && px[0] >= 1 && px[0] < 751 && px[1] >= 1 && px[1] < 479)) continue;
      okb_keypoint kp{};
      kp.x = (float)(px[0] + noise(rng)); kp.y = (float)(px[1] + noise(rng)); kp.size = 8.0f;
      im.kp.push_back(kp);
      std::array<uint8_t, kDesc> d = base[l];
      for (int f = flips(rng); f > 0; --f) { const int b = bit(rng); d[b / 8] ^= (uint8_t)(1u << (b % 8)); }
      im.desc.insert(im.desc.end(), d.begin(), d.end());
      im.truth.push_back(100000 + l);
    }
    for (int i = 0; i < kDistractors; ++i) {
      okb_keypoint kp{};
      kp.x = (float)ux(rng); kp.y = (float)uy(rng); kp.size = 8.0f;
      im.kp.push_back(kp);
      for (int b = 0; b < kDesc; ++b) im.desc.push_back((uint8_t)byte(rng));
      im.truth.push_back(0);
    }
    return im;
  }
};

// What a session's caller sees of one frame.
struct FrameRecord {
  int kf3 = 0, kf2 = 0, last3 = 0, last2 = 0, stereo = 0;
  std::vector<std::vector<uint64_t>> ids;
  std::vector<std::pair<size_t, uint64_t>> callbacks;     // afterKeyframe(kfcounter, olderFrameId)
  bool operator==(const FrameRecord& o) const {
    return kf3 == o.kf3 && kf2 == o.kf2 && last3 == o.last3 && last2 == o.last2 && stereo == o.stereo && ids == o.ids &&
           callbacks == o.callbacks;
  }
};

struct Totals {
  long landmarks = 0, mixed = 0, distractorObs = 0, framesTracked = 0, minMatches = 1 << 30, initChecked = 0,
       maskedInit = 0, temporalMatches = 0, callbackErrors = 0;
  double maxRel = 0, sumRel = 0, maxPoseErr = 0;
  std::vector<double> rels;
  std::string perFrame;
};

// every landmark's observations must see one true point; initialised ones with 3+ observations must lie near it
void checkLandmarks(const Estimator& est, const Scene& sc, const std::map<uint64_t, std::vector<Image>>& truth, Totals& tot) {
  PointMap lms;
  est.getLandmarks(lms);
  const double y_cam = sc.yCam();
  Pose7 T;
  if (est.get_T_WS(sc.frameId(), T))          // the current frame's position against the rig's
    tot.maxPoseErr = std::max(tot.maxPoseErr, std::sqrt(T[0] * T[0] + (T[1] - y_cam) * (T[1] - y_cam) + T[2] * T[2]));
  for (auto& kv : lms) {
    std::set<uint64_t> seen;
    for (auto& o : kv.second.observations) {
      const uint64_t t = truth.at(o.first.frameId)[o.first.cameraIndex].truth.at(o.first.keypointIndex);
      seen.insert(t);
      if (t == 0) ++tot.distractorObs;
    }
    ++tot.landmarks;
    if (seen.size() > 1) { ++tot.mixed; continue; }
    if (seen.empty() || *seen.begin() == 0 || !est.isLandmarkInitialized(kv.first)) continue;
    const int l = (int)(*seen.begin() - 100000);
    if (sc.mask && l % 5 == 0) ++tot.maskedInit;
    if (kv.second.observations.size() < 3) continue;
    const auto& P = sc.lmk[l];
    const auto& X = kv.second.point;
    const double e[3] = {X[0] / X[3] - P[0], X[1] / X[3] - P[1], X[2] / X[3] - P[2]};
    const double d = std::sqrt(P[0] * P[0] + (P[1] - y_cam) * (P[1] - y_cam) + P[2] * P[2]);
    const double rel = std::sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]) / d;
    tot.maxRel = std::max(tot.maxRel, rel); tot.sumRel += rel; ++tot.initChecked; tot.rels.push_back(rel);
  }
}

// The sessions one by one (standalone Estimators) or together (one EstimatorGroup, group forms of every call).
std::vector<std::vector<FrameRecord>> run(bool grouped, int cams, bool mono, Totals& tot) {
  std::unique_ptr<EstimatorGroup> g;
  if (grouped) g.reset(new EstimatorGroup(0, kSessions));
  Frontend fe(cams);
  std::vector<std::unique_ptr<Estimator>> est;
  std::vector<std::unique_ptr<Scene>> sc;
  std::vector<uint64_t> next(kSessions);
  std::vector<std::function<uint64_t()>> newIds;
  for (int s = 0; s < kSessions; ++s) {
    est.emplace_back(grouped ? new Estimator(*g, capacity()) : new Estimator(0, capacity()));
    sc.emplace_back(mono ? new Scene(s, 1, 0.0, 1.0 + 0.1 * s, false) : new Scene(s, 2, 1.0 + 0.1 * s, 0.0, true));
    sc[s]->configure(*est[s]);
    next[s] = 1000000000ULL * (s + 1);                  // each session has its own id source
    uint64_t* n = &next[s];
    newIds.push_back([n]() { return ++*n; });
  }
  const std::vector<std::vector<bool>> overlap(cams, std::vector<bool>(cams, true));
  std::vector<std::map<uint64_t, std::vector<Image>>> truth(kSessions);
  std::vector<std::vector<FrameRecord>> rec(kSessions);
  std::vector<Estimator*> all;
  for (auto& e : est) all.push_back(e.get());
  for (int f = 0; f < kFrames; ++f) {
    std::vector<uint64_t> ids;
    if (grouped) {
      std::vector<EstimatorGroup::StatesRequest> req;
      for (int s = 0; s < kSessions; ++s) req.push_back({all[s], sc[s]->frameId(), sc[s]->t(sc[s]->k), sc[s]->imu(), sc[s]->keyframe()});
      for (bool ok : g->addStates(req)) if (!ok) throw std::runtime_error("addStates failed");
    } else {
      for (int s = 0; s < kSessions; ++s)
        if (!est[s]->addStates(sc[s]->frameId(), sc[s]->t(sc[s]->k), sc[s]->imu(), sc[s]->keyframe())) throw std::runtime_error("addStates failed");
    }
    for (int s = 0; s < kSessions; ++s) {
      auto& ims = truth[s][sc[s]->frameId()];
      ims.clear();
      for (int c = 0; c < cams; ++c) ims.push_back(sc[s]->image(c));
      for (int c = 0; c < cams; ++c) est[s]->setFrameFeatures(sc[s]->frameId(), c, ims[c].kp, ims[c].desc, std::vector<uint64_t>(ims[c].kp.size(), 0));
      ids.push_back(sc[s]->frameId());
    }
    std::vector<FrameRecord> r(kSessions);
    std::vector<Frontend::TrackResult> kf3, kf2, l3, l2, st;
    if (grouped) {
      kf3 = fe.matchToKeyframes3D2D(*g, all, ids);
      kf2 = fe.matchToKeyframes2D2D(*g, all, ids, newIds, [&](size_t s, size_t kf, uint64_t older) { r[s].callbacks.push_back({kf, older}); });
      l3 = fe.matchToLastFrame3D2D(*g, all, ids);
      l2 = fe.matchToLastFrame2D2D(*g, all, ids, newIds);
      st = fe.matchStereo(*g, all, ids, newIds, overlap);
    } else {
      for (int s = 0; s < kSessions; ++s) {
        kf3.push_back(fe.matchToKeyframes3D2D(*est[s], ids[s]));
        kf2.push_back(fe.matchToKeyframes2D2D(*est[s], ids[s], newIds[s], [&](size_t kf, uint64_t older) { r[s].callbacks.push_back({kf, older}); }));
        l3.push_back(fe.matchToLastFrame3D2D(*est[s], ids[s]));
        l2.push_back(fe.matchToLastFrame2D2D(*est[s], ids[s], newIds[s]));
        st.push_back(fe.matchStereo(*est[s], ids[s], newIds[s], overlap));
      }
    }
    std::vector<MapPointVector> removed(kSessions);
    if (grouped) g->optimize(all, 5);
    else for (int s = 0; s < kSessions; ++s) est[s]->optimize(5);
    for (int s = 0; s < kSessions; ++s) {
      r[s].kf3 = kf3[s].numMatches; r[s].kf2 = kf2[s].numMatches; r[s].last3 = l3[s].numMatches; r[s].last2 = l2[s].numMatches;
      r[s].stereo = st[s].numMatches; r[s].ids = st[s].landmarkIds;
      // afterKeyframe runs once per keyframe matched, kfcounter 0, 1, ... on the keyframes by age
      for (size_t i = 0; i < r[s].callbacks.size(); ++i)
        if (r[s].callbacks[i].first != i || !est[s]->isKeyframe(r[s].callbacks[i].second)) ++tot.callbackErrors;
      if (f > 0 && r[s].callbacks.empty()) ++tot.callbackErrors;
      tot.temporalMatches += r[s].kf2 + r[s].last2;
      rec[s].push_back(r[s]);
      if (f > 0) {
        ++tot.framesTracked;
        const int m = r[s].kf3 + r[s].last3;
        if (f >= 6) tot.minMatches = std::min<long>(tot.minMatches, m);
        tot.perFrame += (tot.perFrame.empty() ? "" : ",") + std::to_string(m);
      }
      if (f == kFrames - 1 || f % 6 == 5) checkLandmarks(*est[s], *sc[s], truth[s], tot);
    }
    if (grouped) g->applyMarginalizationStrategy(all, 5, 3, removed);
    else for (int s = 0; s < kSessions; ++s) est[s]->applyMarginalizationStrategy(5, 3, removed[s]);
    for (int s = 0; s < kSessions; ++s) sc[s]->k++;
  }
  est.clear();
  return rec;
}

int slide(bool mono) {
  Totals ts, tg;
  const int cams = mono ? 1 : 2;
  const auto single = run(false, cams, mono, ts);
  const auto grouped = run(true, cams, mono, tg);
  int same = 1;
  for (int s = 0; s < kSessions; ++s) same &= (single[s] == grouped[s]) ? 1 : 0;
  std::sort(ts.rels.begin(), ts.rels.end());
  const double median = ts.rels.empty() ? 0.0 : ts.rels[ts.rels.size() / 2];
  std::printf("{\"mode\":\"%s\",\"frames\":%d,\"sessions\":%d,\"landmarks\":%ld,\"mixed\":%ld,\"distractor_obs\":%ld,"
              "\"frames_tracked\":%ld,\"min_matches_from_6\":%ld,\"init_checked\":%ld,\"max_rel\":%.6g,\"mean_rel\":%.6g,"
              "\"masked_initialised\":%ld,\"temporal_matches\":%ld,\"callback_errors\":%ld,\"group_mixed\":%ld,"
              "\"group_equals_single\":%d,\"median_rel\":%.6g,\"max_pose_err\":%.6g,\"matches\":[%s]}\n",
              mono ? "mono" : "stereo", kFrames, kSessions, ts.landmarks, ts.mixed, ts.distractorObs, ts.framesTracked,
              ts.minMatches, ts.initChecked, ts.maxRel, ts.initChecked ? ts.sumRel / ts.initChecked : 0.0, ts.maskedInit,
              ts.temporalMatches, ts.callbackErrors + tg.callbackErrors, tg.mixed, same, median, ts.maxPoseErr, ts.perFrame.c_str());
  return 0;
}

// --cases: one keyframe (100) and the current frame (101), one camera, six points seen in both with 0.2 m of
// parallax.  The keypoints carry every combination of host ids the reference meets in setBestMatch:
//   p0 (0, 0)                  a new id from newId(), addLandmark, observations in A and B
//   p1 (host-only X1, 0)       X1 added to the graph, observations in A and B, B takes X1
//   p2 (graph L2, 0)           B observes L2 and takes its id
//   p3 (0, graph L3)           A observes L3 and takes its id
//   p4 (host-only X4, graph L4) both carry an id: dropped
//   p5 (host-only X5, host-only Y5) both carry an id: dropped
int cases() {
  const okb_camera cam = camera();
  const double acc = 10.0;                              // 0.2 m along +y in the first 0.2 s
  Estimator est(0, capacity());
  est.addCamera(ExtrinsicsEstimationParameters(), cam, Pose7{{0.0, 0.0, 0.0, -0.5, 0.5, -0.5, 0.5}});
  okb_imu_params imu{};
  imu.a_max = 176; imu.g_max = 7.8; imu.sigma_g_c = 12e-4; imu.sigma_a_c = 8e-3; imu.sigma_bg = 0.03; imu.sigma_ba = 0.1;
  imu.sigma_gw_c = 4e-6; imu.sigma_aw_c = 4e-5; imu.tau = 3600; imu.g = kG; imu.rate = 200;
  est.addImu(imu);
  auto samples = [&](int64_t t0, int64_t t1) {
    std::vector<ImuMeasurement> m;
    for (int64_t s = t0; s <= t1; s += 5000000LL) { ImuMeasurement x{}; x.t_ns = s; x.acc[1] = s > 1000000000LL ? acc : 0.0; x.acc[2] = kG; m.push_back(x); }
    return m;
  };
  const int64_t t0 = 1000000000LL, t1 = t0 + 200000000LL;
  if (!est.addStates(100, t0, samples(t0 - 50000000LL, t0), true)) throw std::runtime_error("addStates failed");
  if (!est.addStates(101, t1, samples(t0 - 5000000LL, t1 + 5000000LL), false)) throw std::runtime_error("addStates failed");
  const double P[6][3] = {{3.0, -0.6, 0.3}, {3.5, 0.2, -0.4}, {4.0, 0.9, 0.5}, {2.5, -0.2, -0.2}, {4.5, -1.0, 0.1}, {3.2, 0.5, 0.6}};
  auto image = [&](double y, std::vector<okb_keypoint>& kp, std::vector<uint8_t>& desc) {
    for (int i = 0; i < 6; ++i) {
      const double xc = -(P[i][1] - y), yc = -P[i][2], zc = P[i][0];
      okb_keypoint k{}; k.x = (float)(cam.fu * xc / zc + cam.cu); k.y = (float)(cam.fv * yc / zc + cam.cv); k.size = 8.0f;
      kp.push_back(k);
      for (int b = 0; b < kDesc; ++b) desc.push_back((uint8_t)(37 * i + 11 * b + (b * b) % 7));
    }
  };
  std::vector<okb_keypoint> kpA, kpB;
  std::vector<uint8_t> dA, dB;
  image(0.0, kpA, dA);
  image(0.5 * acc * 0.04, kpB, dB);
  const uint64_t L2 = 500, L3 = 501, L4 = 502, X1 = 601, X4 = 604, X5 = 605, Y5 = 705;
  for (uint64_t l : {L2, L3, L4}) {
    const int i = (int)(l - 500) + 2;
    est.addLandmark(l, Vec4{{P[i][0], P[i][1], P[i][2], 1.0}});
    est.setLandmarkInitialized(l, false);
  }
  est.setFrameFeatures(100, 0, kpA, dA, {0, X1, 0, 0, X4, X5});
  est.setFrameFeatures(101, 0, kpB, dB, {0, 0, 0, 0, 0, Y5});
  const double z2[2] = {kpA[2].x, kpA[2].y}, z3[2] = {kpB[3].x, kpB[3].y}, z4[2] = {kpB[4].x, kpB[4].y};
  est.addObservation(L2, 100, 0, 2, z2, 8.0);          // names A's keypoint 2 on the host and in the store
  est.addObservation(L3, 101, 0, 3, z3, 8.0);
  est.addObservation(L4, 101, 0, 4, z4, 8.0);
  uint64_t next = 9000;
  Frontend fe(1);
  std::vector<std::pair<size_t, uint64_t>> calls;
  const auto r = fe.matchToKeyframes2D2D(est, 101, [&]() { return ++next; }, [&](size_t kf, uint64_t id) { calls.push_back({kf, id}); });
  const auto idsA = est.frameLandmarkIds(100, 0), idsB = est.frameLandmarkIds(101, 0);
  auto observes = [&](uint64_t l, uint64_t frame, size_t k) {
    MapPoint mp;
    if (!est.getLandmark(l, mp)) return false;
    for (auto& o : mp.observations)
      if (o.first.frameId == frame && o.first.cameraIndex == 0 && o.first.keypointIndex == k) return true;
    return false;
  };
  int fails = 0;
  std::string why;
  auto expect = [&](bool ok, const char* what) { if (!ok) { ++fails; why += std::string(why.empty() ? "" : ";") + what; } };
  expect(r.numMatches == 4 && r.numUncertainMatches == 0, "numMatches");
  expect(calls.size() == 1 && calls[0].first == 0 && calls[0].second == 100, "afterKeyframe");
  expect(next == 9001 && idsA[0] == 9001 && idsB[0] == 9001 && observes(9001, 100, 0) && observes(9001, 101, 0), "p0");
  expect(idsA[1] == X1 && idsB[1] == X1 && observes(X1, 100, 1) && observes(X1, 101, 1), "p1");
  expect(idsA[2] == L2 && idsB[2] == L2 && observes(L2, 101, 2), "p2");
  expect(idsA[3] == L3 && idsB[3] == L3 && observes(L3, 100, 3), "p3");
  MapPoint m4;
  est.getLandmark(L4, m4);
  expect(idsA[4] == X4 && idsB[4] == L4 && m4.observations.size() == 1 && !est.getLandmark(X4, m4), "p4");
  expect(idsA[5] == X5 && idsB[5] == Y5 && !est.getLandmark(X5, m4) && !est.getLandmark(Y5, m4), "p5");
  PointMap lms;
  expect(est.getLandmarks(lms) == 5, "graph size");
  // the store now names the new landmarks on both sides: a second round finds nothing to initialise, and its records
  // pass finish2D2D's check that every store slot agrees with the host ids
  const auto again = fe.matchToKeyframes2D2D(est, 101, [&]() { return ++next; });
  expect(again.numMatches == 0 && next == 9001 && est.getLandmarks(lms) == 5, "second round");
  std::printf("{\"mode\":\"cases\",\"num_matches\":%d,\"fails\":%d,\"why\":\"%s\"}\n", r.numMatches, fails, why.c_str());
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  const std::string mode = argc > 1 ? argv[1] : "--stereo";
  try {
    if (mode == "--no-gpu") {
      try {
        Estimator e(0, capacity());
        std::printf("{\"mode\":\"no-gpu\",\"threw\":false}\n");
      } catch (const std::runtime_error& e) {
        std::printf("{\"mode\":\"no-gpu\",\"threw\":true}\n");
      }
      return 0;
    }
    if (mode == "--cases") return cases();
    if (mode == "--stereo" || mode == "--mono") return slide(mode == "--mono");
    std::printf("{\"error\":\"unknown mode\"}\n");
    return 1;
  } catch (const std::exception& e) {
    std::printf("{\"error\":\"%s\"}\n", e.what());
    return 1;
  }
}
