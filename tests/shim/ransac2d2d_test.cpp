// Exercises the device 2D-2D RANSAC and pose initialisation through the C++ mirror: Frontend::runRansac2d2d
// (okb_ransac_2d2d_batch), its EstimatorGroup form and RansacHooks::device2d2d inside
// Frontend::dataAssociationAndInitialization, on sessions that start uninitialised at rest (no translation: the
// rotation-only model wins) and then accelerate sideways (parallax: the five-point model wins), with injected wrong
// associations (look-alike keypoints).  Prints one JSON line per mode; tests/test_gpu_ransac2d2d_mirror.py checks them.
//   ransac2d2d_test.bin --no-gpu     the mirror fails loudly without a device
//   ransac2d2d_test.bin --slide      two stereo sessions and one monocular session, 16 frames, with device2d2d, standalone
//                                    and as one group (compared frame by frame); and, as one group, sessions initialised
//                                    from the start with and without device2d2d (compared frame by frame)
//   ransac2d2d_test.bin --direct     runRansac2d2d called by an afterKeyframe hook at the reference's call point while
//                                    the session is not initialised: the end state of every outlier (host id 0, store
//                                    slot -1, observation gone), the return values and the initialised pose's direction
//                                    of translation against the truth
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <random>
#include <string>

#include "okvis_b200_frontend.hpp"

using namespace okvis_b200;

namespace {

constexpr double kG = 9.81007, kDt = 0.2;
constexpr int kLandmarks = 300, kDistractors = 40, kFrames = 16, kRest = 6, kDesc = 48;
constexpr double kWrong = 0.1;      // share of a frame's visible landmarks given a look-alike

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

// lm[k]: the scene landmark keypoint k shows (-1: distractor); wrong[k]: a look-alike of that landmark
struct Image { std::vector<okb_keypoint> kp; std::vector<uint8_t> desc; std::vector<int> lm; std::vector<char> wrong; };

// The temporal driver's scene: a rig looking along +x, at rest for kRest frames and then accelerating along +y
// (y(t) = acc (t - t_rest)^2 / 2), camera c at y = +-0.055 m; landmarks with noisy keypoints and a few flipped
// descriptor bits, plus distractors.
struct Scene {
  int cams;
  double acc;
  std::mt19937 rng;
  std::vector<std::array<double, 3>> lmk;
  std::vector<std::array<uint8_t, kDesc>> base;
  int k = 0;
  Scene(int s, int nCams, double a) : cams(nCams), acc(a), rng(29 + 31 * s) {
    const double tm = kDt * (kFrames - kRest), span = 0.5 * acc * tm * tm;
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
  double yCam() const { const double tt = std::max(0, k - kRest) * kDt; return 0.5 * acc * tt * tt; }
  std::vector<ImuMeasurement> imu() const {
    std::vector<ImuMeasurement> meas;
    for (int64_t s = (k == 0 ? t(k) - 50000000LL : t(k - 1) - 5000000LL); s <= t(k) + (k == 0 ? 0 : 5000000LL); s += 5000000LL) {
      ImuMeasurement m{}; m.t_ns = s; m.acc[1] = s > t(kRest) ? acc : 0.0; m.acc[2] = kG; meas.push_back(m);
    }
    return meas;
  }
  void configure(Estimator& est) const {
    const okb_camera cam = camera();
    est.addCamera(ExtrinsicsEstimationParameters(), cam, Pose7{{0.0, 0.055, 0.0, -0.5, 0.5, -0.5, 0.5}});
    if (cams > 1) est.addCamera(ExtrinsicsEstimationParameters(), cam, Pose7{{0.0, -0.055, 0.0, -0.5, 0.5, -0.5, 0.5}});
    okb_imu_params imu{};
    imu.a_max = 176; imu.g_max = 7.8; imu.sigma_g_c = 12e-4; imu.sigma_a_c = 8e-3; imu.sigma_bg = 0.03; imu.sigma_ba = 0.1;
    imu.sigma_gw_c = 4e-6; imu.sigma_aw_c = 4e-5; imu.tau = 3600; imu.g = kG; imu.rate = 200;
    est.addImu(imu);
  }
  // Keypoints of camera c; with `wrong`, kWrong of the visible landmarks also get a look-alike: the landmark's own
  // descriptor 6-10 px from its projection, while the true keypoint's descriptor is replaced by a random one, so the
  // 3D-2D match associates the landmark with the look-alike (an injected wrong association).
  Image image(int c, bool wrong) {
    const okb_camera cam = camera();
    std::normal_distribution<double> noise(0.0, 0.3);
    std::uniform_int_distribution<int> flips(0, 4), bit(0, 8 * kDesc - 1), byte(0, 255);
    std::uniform_real_distribution<double> ux(0, 752), uy(0, 480), u01(0, 1), off(6, 10), ang(0, 6.283185307179586);
    Image im;
    const double y_cam = yCam();
    auto push = [&](double x, double y, const uint8_t* d, int l, char w) {
      okb_keypoint kp{};
      kp.x = (float)x; kp.y = (float)y; kp.size = 8.0f;
      im.kp.push_back(kp); im.desc.insert(im.desc.end(), d, d + kDesc); im.lm.push_back(l); im.wrong.push_back(w);
    };
    for (int l = 0; l < kLandmarks; ++l) {
      const double xs = lmk[l][0], ys = lmk[l][1] - y_cam - (c == 0 ? 0.055 : -0.055), zs = lmk[l][2];
      const double xc = -ys, yc = -zs, zc = xs;
      const double px[2] = {cam.fu * xc / zc + cam.cu, cam.fv * yc / zc + cam.cv};
      if (!(zc > 0.5 && px[0] >= 12 && px[0] < 740 && px[1] >= 12 && px[1] < 468)) continue;
      std::array<uint8_t, kDesc> d = base[l];
      for (int f = flips(rng); f > 0; --f) { const int b = bit(rng); d[b / 8] ^= (uint8_t)(1u << (b % 8)); }
      const bool lookalike = wrong && u01(rng) < kWrong;
      if (lookalike) {
        std::array<uint8_t, kDesc> r;
        for (auto& b : r) b = (uint8_t)byte(rng);
        push(px[0] + noise(rng), px[1] + noise(rng), r.data(), l, 0);
        const double o = off(rng), a = ang(rng);
        push(px[0] + o * std::cos(a), px[1] + o * std::sin(a), d.data(), l, 1);
      } else {
        push(px[0] + noise(rng), px[1] + noise(rng), d.data(), l, 0);
      }
    }
    for (int i = 0; i < kDistractors; ++i) {
      std::array<uint8_t, kDesc> r;
      for (auto& b : r) b = (uint8_t)byte(rng);
      push(ux(rng), uy(rng), r.data(), -1, 0);
    }
    return im;
  }
};

// What a session's caller sees of one frame.
struct FrameRecord {
  int keyframe = 0, num3d = 0, initialized = 0;
  std::vector<std::vector<uint64_t>> ids, keyframeIds;
  std::vector<std::string> hooks;
  std::array<uint64_t, 7> pose{};
  bool operator==(const FrameRecord& o) const {
    return keyframe == o.keyframe && num3d == o.num3d && initialized == o.initialized && ids == o.ids && keyframeIds == o.keyframeIds &&
           hooks == o.hooks && pose == o.pose;
  }
};

uint64_t bits(double v) { uint64_t u; std::memcpy(&u, &v, 8); return u; }

bool observes(const Estimator& e, uint64_t lm, uint64_t frame, size_t cam, size_t k) {
  MapPoint mp;
  if (!e.getLandmark(lm, mp)) return false;
  KeypointIdentifier kid; kid.frameId = frame; kid.cameraIndex = cam; kid.keypointIndex = k;
  return mp.observations.count(kid) != 0;
}

const int kCams[3] = {2, 2, 1};

// C (row-major) of a quaternion [x, y, z, w]
void rotation(const double* q, double* C) {
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                       2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                       2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
  for (int k = 0; k < 9; ++k) C[k] = R[k];
}     // two stereo sessions and a monocular one

// firstInit[s]: the frame at which session s became initialised (-1: never)
std::vector<std::vector<FrameRecord>> run(bool grouped, bool device, bool startInitialized, std::vector<int>& firstInit) {
  const int nSessions = 3;
  std::unique_ptr<EstimatorGroup> g;
  if (grouped) g.reset(new EstimatorGroup(0, nSessions));
  std::vector<std::unique_ptr<Frontend>> fe;
  std::vector<std::unique_ptr<Estimator>> est;
  std::vector<std::unique_ptr<Scene>> sc;
  std::vector<uint64_t> next(nSessions);
  std::vector<std::function<uint64_t()>> newIds;
  for (int s = 0; s < nSessions; ++s) {
    est.emplace_back(grouped ? new Estimator(*g, capacity()) : new Estimator(0, capacity()));
    sc.emplace_back(new Scene(s, kCams[s], 1.5 + 0.25 * s));
    sc[s]->configure(*est[s]);
    if (!grouped || s == 0) fe.emplace_back(new Frontend(2));
    next[s] = 1000000000ULL * (s + 1);
    uint64_t* n = &next[s];
    newIds.push_back([n]() { return ++*n; });
  }
  const std::vector<std::vector<bool>> overlap(2, std::vector<bool>(2, true));
  std::vector<std::vector<FrameRecord>> rec(nSessions);
  std::vector<Estimator*> all;
  for (auto& e : est) all.push_back(e.get());
  std::vector<char> initialized(nSessions, startInitialized ? 1 : 0);
  firstInit.assign(nSessions, startInitialized ? 0 : -1);
  for (int f = 0; f < kFrames; ++f) {
    std::vector<uint64_t> fid;
    if (grouped) {
      std::vector<EstimatorGroup::StatesRequest> req;
      for (int s = 0; s < nSessions; ++s) req.push_back({all[s], sc[s]->frameId(), sc[s]->t(sc[s]->k), sc[s]->imu(), false});
      for (bool ok : g->addStates(req)) if (!ok) throw std::runtime_error("addStates failed");
    } else {
      for (int s = 0; s < nSessions; ++s)
        if (!est[s]->addStates(sc[s]->frameId(), sc[s]->t(sc[s]->k), sc[s]->imu(), false)) throw std::runtime_error("addStates failed");
    }
    for (int s = 0; s < nSessions; ++s) {
      for (int c = 0; c < kCams[s]; ++c) {
        const Image im = sc[s]->image(c, f >= 2);
        est[s]->setFrameFeatures(sc[s]->frameId(), c, im.kp, im.desc, std::vector<uint64_t>(im.kp.size(), 0));
      }
      fid.push_back(sc[s]->frameId());
    }
    std::vector<FrameRecord> r(nSessions);
    int cur = 0;
    auto who = [&](size_t s) { return grouped ? (int)s : cur; };
    Frontend::RansacHooks hooks;
    hooks.device2d2d = device;
    hooks.afterKeyframe = [&](size_t s, bool init, size_t kf, uint64_t older) {
      r[who(s)].hooks.push_back("K" + std::to_string(init) + "/" + std::to_string(kf) + "/" + std::to_string(older));
      return false;
    };
    hooks.afterLastFrame2D2D = [&](size_t s, bool init) { r[who(s)].hooks.push_back("L2/" + std::to_string(init)); };
    std::vector<Frontend::FrameResult> res(nSessions);
    std::vector<char> kf(nSessions, 0);
    if (grouped) {
      res = fe[0]->dataAssociationAndInitialization(*g, all, fid, newIds, overlap, kf, hooks, initialized);
    } else {
      for (int s = 0; s < nSessions; ++s) {
        cur = s;
        bool k = false;
        res[s] = fe[s]->dataAssociationAndInitialization(*est[s], fid[s], newIds[s], overlap, &k, hooks);
        kf[s] = k ? 1 : 0;
        initialized[s] = fe[s]->isInitialized() ? 1 : 0;
      }
    }
    for (int s = 0; s < nSessions; ++s) {
      if (initialized[s] && firstInit[s] < 0) firstInit[s] = f;
      est[s]->setKeyframe(fid[s], kf[s] != 0);
    }
    if (grouped) g->optimize(all, 5);
    else for (int s = 0; s < nSessions; ++s) est[s]->optimize(5);
    for (int s = 0; s < nSessions; ++s) {
      Pose7 T;
      est[s]->get_T_WS(fid[s], T);
      for (int i = 0; i < 7; ++i) r[s].pose[i] = bits(T[i]);
      r[s].keyframe = kf[s]; r[s].num3d = res[s].num3dMatches; r[s].ids = res[s].landmarkIds; r[s].keyframeIds = res[s].keyframeIds;
      r[s].initialized = initialized[s];
      rec[s].push_back(r[s]);
    }
    std::vector<MapPointVector> removed(nSessions);
    if (grouped) g->applyMarginalizationStrategy(all, 5, 3, removed);
    else for (int s = 0; s < nSessions; ++s) est[s]->applyMarginalizationStrategy(5, 3, removed[s]);
    for (int s = 0; s < nSessions; ++s) sc[s]->k++;
  }
  est.clear();
  return rec;
}

int slide() {
  std::vector<int> fs, fg, fi, fn;
  const auto single = run(false, true, false, fs);
  const auto grouped = run(true, true, false, fg);
  const auto initDev = run(true, true, true, fi);
  const auto initOff = run(true, false, true, fn);
  int same = 1, initSame = 1;
  for (size_t s = 0; s < single.size(); ++s) {
    same &= (single[s] == grouped[s]) ? 1 : 0;
    initSame &= (initDev[s] == initOff[s]) ? 1 : 0;
  }
  std::string first;
  for (size_t s = 0; s < fg.size(); ++s) first += (s ? "," : "") + std::to_string(fg[s]);
  std::printf("{\"mode\":\"slide\",\"frames\":%d,\"rest\":%d,\"sessions\":3,\"group_equals_single\":%d,\"first_initialized\":[%s],"
              "\"initialized_unchanged\":%d}\n", kFrames, kRest, same, first.c_str(), initSame);
  return 0;
}

// One session (stereo or monocular) without device2d2d whose afterKeyframe hook calls runRansac2d2d itself while the
// session is not initialised, as the reference does at :438-446 (initializePose = true).  Every keypoint whose id the
// call cleared must end with host id 0, no observation of its former landmark and store slot -1 (the keyframe decision
// that follows counts as matched exactly the keypoints with a host id).  When the call initialised the pose from the
// five-point model with a translation, its direction from the older frame is compared with the truth (+y in the world).
int direct(int cams) {
  Estimator est(0, capacity());
  Scene sc(7 + cams, cams, 1.5);
  sc.configure(est);
  Frontend fe(2);
  uint64_t next = 7000000000ULL;
  const std::vector<std::vector<bool>> overlap(2, std::vector<bool>(2, true));
  long removed = 0, endStateFails = 0, storeFails = 0, calls = 0, lookalikesRemoved = 0, rotationOnlyCalls = 0, poseSets = 0, retNeg = 0;
  long retRotMismatch = 0;
  double maxAngle = 0.0;
  bool initialized = false;
  std::map<uint64_t, double> yOf;
  for (int f = 0; f < kFrames; ++f) {
    if (!est.addStates(sc.frameId(), sc.t(sc.k), sc.imu(), false)) throw std::runtime_error("addStates failed");
    yOf[sc.frameId()] = sc.yCam();
    std::vector<Image> ims;
    for (int c = 0; c < cams; ++c) {
      ims.push_back(sc.image(c, f >= 2));
      est.setFrameFeatures(sc.frameId(), c, ims[c].kp, ims[c].desc, std::vector<uint64_t>(ims[c].kp.size(), 0));
    }
    const uint64_t id = sc.frameId();
    Frontend::RansacHooks hooks;
    hooks.afterKeyframe = [&](size_t, bool init, size_t, uint64_t older) {
      bool tmp = false;
      if (init) return tmp;
      std::vector<std::vector<uint64_t>> before;
      for (int c = 0; c < cams; ++c) before.push_back(est.frameLandmarkIds(id, c));
      Pose7 A{}, B0{}, B1{};
      est.get_T_WS(older, A);
      est.get_T_WS(id, B0);
      const int ret = fe.runRansac2d2d(est, id, older, true, true, tmp);
      ++calls;
      if (tmp) ++rotationOnlyCalls;
      if (ret < 0 && !tmp) ++retRotMismatch;              // -1 always comes with rotationOnly (:802-808)
      if (ret < 0) ++retNeg;
      est.get_T_WS(id, B1);
      if (B1 != B0) ++poseSets;
      // T_C1C2 = (T_WSA T_SC0)^-1 T_WS0 T_SC0 recovers the device's relative pose from the poses; its translation (camera
      // 0's frame at A) against the true motion, +y of the world and body frames seen in camera 0 (R_SC^T e_y)
      Pose7 T_SC{};
      est.getCameraSensorStates(id, 0, T_SC);
      double CA[9], CB[9], CS[9];
      rotation(A.data() + 3, CA); rotation(B1.data() + 3, CB); rotation(T_SC.data() + 3, CS);
      double pa[3], pb[3], d[3], t[3];
      for (int i = 0; i < 3; ++i) {
        pa[i] = A[i] + CA[3 * i] * T_SC[0] + CA[3 * i + 1] * T_SC[1] + CA[3 * i + 2] * T_SC[2];
        pb[i] = B1[i] + CB[3 * i] * T_SC[0] + CB[3 * i + 1] * T_SC[1] + CB[3 * i + 2] * T_SC[2];
        d[i] = pb[i] - pa[i];
      }
      double C_WC[9];                                      // C_WS_A C_SC
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C_WC[3 * i + j] = CA[3 * i] * CS[j] + CA[3 * i + 1] * CS[3 + j] + CA[3 * i + 2] * CS[6 + j];
      for (int j = 0; j < 3; ++j) t[j] = C_WC[j] * d[0] + C_WC[3 + j] * d[1] + C_WC[6 + j] * d[2];
      const double truth[3] = {CS[3], CS[4], CS[5]};       // R_SC^T e_y
      const double tn = std::sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
      if (!tmp && B1 != B0 && tn > 0.0 && yOf[id] - yOf[older] > 0.0) {
        const double c = (t[0] * truth[0] + t[1] * truth[1] + t[2] * truth[2]) / tn;
        maxAngle = std::max(maxAngle, std::acos(std::min(1.0, std::max(-1.0, c))) * 180.0 / 3.14159265358979323846);
      }
      for (int c = 0; c < cams; ++c) {
        const std::vector<uint64_t> after = est.frameLandmarkIds(id, c);
        for (size_t k = 0; k < after.size(); ++k) {
          if (before[c][k] == after[k]) continue;
          ++removed;
          if (ims[c].wrong[k]) ++lookalikesRemoved;
          if (after[k] != 0 || observes(est, before[c][k], id, c, k)) ++endStateFails;
        }
      }
      return tmp;
    };
    bool kfb = false;
    const Frontend::FrameResult res = fe.dataAssociationAndInitialization(est, id, [&]() { return ++next; }, overlap, &kfb, hooks);
    initialized = fe.isInitialized();
    if (!res.keyframeCams.empty())
      for (int c = 0; c < cams; ++c) {
        int named = 0;
        for (uint64_t v : res.keyframeIds[c]) named += v != 0 ? 1 : 0;
        if (res.keyframeCams[c].n_matched != named) ++storeFails;
      }
    est.setKeyframe(id, kfb);
    est.optimize(5);
    MapPointVector rm;
    est.applyMarginalizationStrategy(5, 3, rm);
    sc.k++;
  }
  std::printf("{\"mode\":\"direct\",\"cams\":%d,\"calls\":%ld,\"rotation_only_calls\":%ld,\"ret_negative\":%ld,\"ret_rot_mismatch\":%ld,"
              "\"pose_sets\":%ld,\"removed\":%ld,\"lookalikes_removed\":%ld,\"end_state_fails\":%ld,\"store_fails\":%ld,"
              "\"max_translation_angle_deg\":%.4f,\"initialized\":%d}\n",
              cams, calls, rotationOnlyCalls, retNeg, retRotMismatch, poseSets, removed, lookalikesRemoved, endStateFails, storeFails, maxAngle,
              initialized ? 1 : 0);
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  const std::string mode = argc > 1 ? argv[1] : "--slide";
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
    if (mode == "--slide") return slide();
    if (mode == "--direct") return direct(argc > 2 ? std::atoi(argv[2]) : 2);
    std::printf("{\"error\":\"unknown mode\"}\n");
    return 1;
  } catch (const std::exception& e) {
    std::printf("{\"error\":\"%s\"}\n", e.what());
    return 1;
  }
}
