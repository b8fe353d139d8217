// Exercises the keyframe decision through the C++ mirror: Frontend::dataAssociationAndInitialization (which calls
// Frontend::doWeNeedANewKeyframe, okb_keyframe_overlap_batch) and its EstimatorGroup form, with the keyframes chosen by
// the decision instead of a fixed schedule, through optimize and applyMarginalizationStrategy(5, 3).  Prints one JSON
// line per mode; tests/test_gpu_keyframe_mirror.py checks them.
//   keyframe_test.bin --no-gpu        the mirror fails loudly without a device
//   keyframe_test.bin --slide DIR     three stereo sessions and one monocular session, at rest for 8 frames and then
//                                     accelerating sideways, 24 frames; standalone (one Frontend per session) and as one
//                                     group, compared frame by frame (ids, decisions, hook calls); every device decision
//                                     of the standalone run is written to DIR with the keypoints and matched flags it saw
//   keyframe_test.bin --reject        a RANSAC hook that rejects keypoints through setFrameLandmarkId changes the matched
//                                     count of the frame's decision; removeObservation alone does not
#include <algorithm>
#include <array>
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
constexpr int kLandmarks = 300, kDistractors = 40, kFrames = 24, kRest = 8, kDesc = 48;

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

struct Image { std::vector<okb_keypoint> kp; std::vector<uint8_t> desc; };

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
  Image image(int c) {
    const okb_camera cam = camera();
    std::normal_distribution<double> noise(0.0, 0.3);
    std::uniform_int_distribution<int> flips(0, 4), bit(0, 8 * kDesc - 1), byte(0, 255);
    std::uniform_real_distribution<double> ux(0, 752), uy(0, 480);
    Image im;
    const double y_cam = yCam();
    for (int l = 0; l < kLandmarks; ++l) {
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
    }
    for (int i = 0; i < kDistractors; ++i) {
      okb_keypoint kp{};
      kp.x = (float)ux(rng); kp.y = (float)uy(rng); kp.size = 8.0f;
      im.kp.push_back(kp);
      for (int b = 0; b < kDesc; ++b) im.desc.push_back((uint8_t)byte(rng));
    }
    return im;
  }
};

// What a session's caller sees of one frame.
struct FrameRecord {
  int keyframe = 0, num3d = 0;
  std::vector<std::vector<uint64_t>> ids;
  std::vector<std::string> hooks;
  bool operator==(const FrameRecord& o) const { return keyframe == o.keyframe && num3d == o.num3d && ids == o.ids && hooks == o.hooks; }
};

uint64_t bits(double v) { uint64_t u; std::memcpy(&u, &v, 8); return u; }

// one device decision with the keypoints and matched flags it saw, for tests/keyframe_reference.py
void dump(const std::string& dir, int s, int f, const std::map<uint64_t, std::vector<Image>>& images, uint64_t frameId,
          const Frontend::FrameResult& r) {
  const std::string path = dir + "/s" + std::to_string(s) + "_f" + std::to_string(f) + ".txt";
  FILE* o = std::fopen(path.c_str(), "w");
  if (!o) throw std::runtime_error("cannot write " + path);
  std::fprintf(o, "%d %016llx %016llx %zu\n", r.keyframe.need_keyframe, (unsigned long long)bits(r.keyframe.overlap),
               (unsigned long long)bits(r.keyframe.ratio), r.keyframeCams.size());
  for (size_t c = 0; c < r.keyframeCams.size(); ++c) {
    const okb_keyframe_cam& v = r.keyframeCams[c];
    const auto& kp = images.at(frameId)[c].kp;
    std::fprintf(o, "%d %d %d %d %d %d %016llx %016llx %016llx %016llx\n", v.n_points, v.n_matched, v.hull_all, v.hull_matched,
                 v.inside, v.skipped, (unsigned long long)bits(v.area_all), (unsigned long long)bits(v.area_matched),
                 (unsigned long long)bits(v.overlap), (unsigned long long)bits(v.ratio));
    for (size_t k = 0; k < kp.size(); ++k) std::fprintf(o, "%a %a %d\n", (double)kp[k].x, (double)kp[k].y, r.keyframeIds[c][k] != 0 ? 1 : 0);
  }
  std::fclose(o);
}

struct Totals { long restKeyframes = 0, motionKeyframes = 0, deviceDecisions = 0, landmarks = 0; std::string schedule; };

// The sessions one by one (a standalone Estimator and Frontend each) or together (one EstimatorGroup and one Frontend).
std::vector<std::vector<FrameRecord>> run(bool grouped, const std::string& dir, Totals& tot) {
  const int nSessions = 4;
  std::unique_ptr<EstimatorGroup> g;
  if (grouped) g.reset(new EstimatorGroup(0, nSessions));
  std::vector<std::unique_ptr<Frontend>> fe;
  std::vector<std::unique_ptr<Estimator>> est;
  std::vector<std::unique_ptr<Scene>> sc;
  std::vector<uint64_t> next(nSessions);
  std::vector<std::function<uint64_t()>> newIds;
  for (int s = 0; s < nSessions; ++s) {
    const int cams = s < 3 ? 2 : 1;
    est.emplace_back(grouped ? new Estimator(*g, capacity()) : new Estimator(0, capacity()));
    sc.emplace_back(new Scene(s, cams, 1.5 + 0.25 * s));
    sc[s]->configure(*est[s]);
    if (!grouped || s == 0) fe.emplace_back(new Frontend(2));
    next[s] = 1000000000ULL * (s + 1);
    uint64_t* n = &next[s];
    newIds.push_back([n]() { return ++*n; });
  }
  const std::vector<std::vector<bool>> overlap(2, std::vector<bool>(2, true));
  std::vector<std::map<uint64_t, std::vector<Image>>> images(nSessions);
  std::vector<std::vector<FrameRecord>> rec(nSessions);
  std::vector<Estimator*> all;
  for (auto& e : est) all.push_back(e.get());
  std::vector<char> initialized(nSessions, 0);
  for (int f = 0; f < kFrames; ++f) {
    std::vector<uint64_t> ids;
    if (grouped) {
      std::vector<EstimatorGroup::StatesRequest> req;
      for (int s = 0; s < nSessions; ++s) req.push_back({all[s], sc[s]->frameId(), sc[s]->t(sc[s]->k), sc[s]->imu(), false});
      for (bool ok : g->addStates(req)) if (!ok) throw std::runtime_error("addStates failed");
    } else {
      for (int s = 0; s < nSessions; ++s)
        if (!est[s]->addStates(sc[s]->frameId(), sc[s]->t(sc[s]->k), sc[s]->imu(), false)) throw std::runtime_error("addStates failed");
    }
    for (int s = 0; s < nSessions; ++s) {
      auto& ims = images[s][sc[s]->frameId()];
      ims.clear();
      for (int c = 0; c < sc[s]->cams; ++c) ims.push_back(sc[s]->image(c));
      for (int c = 0; c < sc[s]->cams; ++c)
        est[s]->setFrameFeatures(sc[s]->frameId(), c, ims[c].kp, ims[c].desc, std::vector<uint64_t>(ims[c].kp.size(), 0));
      ids.push_back(sc[s]->frameId());
    }
    std::vector<FrameRecord> r(nSessions);
    int cur = 0;                                          // the standalone session being run (hooks receive 0 there)
    auto who = [&](size_t s) { return grouped ? (int)s : cur; };
    Frontend::RansacHooks hooks;
    hooks.afterKeyframe = [&](size_t s, bool init, size_t kf, uint64_t older) {
      r[who(s)].hooks.push_back("K" + std::to_string(init) + "/" + std::to_string(kf) + "/" + std::to_string(older));
      return false;
    };
    hooks.afterLastFrame3D2D = [&](size_t s, bool init) { r[who(s)].hooks.push_back("L3/" + std::to_string(init)); };
    hooks.afterLastFrame2D2D = [&](size_t s, bool init) { r[who(s)].hooks.push_back("L2/" + std::to_string(init)); };
    std::vector<Frontend::FrameResult> res(nSessions);
    std::vector<char> kf(nSessions, 0);
    if (grouped) {
      res = fe[0]->dataAssociationAndInitialization(*g, all, ids, newIds, overlap, kf, hooks, initialized);
    } else {
      for (int s = 0; s < nSessions; ++s) {
        cur = s;
        bool k = false;
        res[s] = fe[s]->dataAssociationAndInitialization(*est[s], ids[s], newIds[s], overlap, &k, hooks);
        kf[s] = k ? 1 : 0;
      }
    }
    for (int s = 0; s < nSessions; ++s) est[s]->setKeyframe(ids[s], kf[s] != 0);      // ThreadedKFVio.cpp:507-525
    std::vector<MapPointVector> removed(nSessions);
    if (grouped) g->optimize(all, 5);
    else for (int s = 0; s < nSessions; ++s) est[s]->optimize(5);
    for (int s = 0; s < nSessions; ++s) {
      r[s].keyframe = kf[s]; r[s].num3d = res[s].num3dMatches; r[s].ids = res[s].landmarkIds;
      rec[s].push_back(r[s]);
      if (!res[s].keyframeCams.empty()) {
        ++tot.deviceDecisions;
        if (!grouped && !dir.empty()) dump(dir, s, f, images[s], ids[s], res[s]);
      }
      if (f > 0 && f < kRest) tot.restKeyframes += kf[s];
      if (f >= kRest + 2) tot.motionKeyframes += kf[s];
      tot.schedule += kf[s] ? "K" : ".";
    }
    tot.schedule += " ";
    if (grouped) g->applyMarginalizationStrategy(all, 5, 3, removed);
    else for (int s = 0; s < nSessions; ++s) est[s]->applyMarginalizationStrategy(5, 3, removed[s]);
    for (int s = 0; s < nSessions; ++s) sc[s]->k++;
  }
  for (auto& e : est) tot.landmarks += (long)e->numLandmarks();
  est.clear();
  return rec;
}

int slide(const std::string& dir) {
  Totals ts, tg;
  const auto single = run(false, dir, ts);
  const auto grouped = run(true, "", tg);
  int same = 1;
  for (size_t s = 0; s < single.size(); ++s) same &= (single[s] == grouped[s]) ? 1 : 0;
  std::printf("{\"mode\":\"slide\",\"frames\":%d,\"rest_frames\":%d,\"sessions\":%zu,\"rest_keyframes\":%ld,\"motion_keyframes\":%ld,"
              "\"motion_frames\":%d,\"device_decisions\":%ld,\"landmarks\":%ld,\"group_equals_single\":%d,\"schedule\":\"%s\"}\n",
              kFrames, kRest, single.size(), ts.restKeyframes, ts.motionKeyframes, kFrames - kRest - 2, ts.deviceDecisions,
              ts.landmarks, same, ts.schedule.c_str());
  return 0;
}

// One stereo session at rest for 5 frames; at the last one, a hook after the first keyframe's 2D-2D rounds rejects
// the first 5 matched keypoints of the current frame's camera 0.  With setFrameLandmarkId(..., 0) the decision sees 5
// fewer matched points than without the hook; with removeObservation alone it sees as many.
int reject() {
  auto runOnce = [](int mode) {               // 0: no hook, 1: removeObservation only, 2: removeObservation + setFrameLandmarkId
    Estimator est(0, capacity());
    Scene sc(7, 2, 0.0);
    sc.configure(est);
    Frontend fe(2);
    uint64_t next = 5000000000ULL;
    const std::vector<std::vector<bool>> overlap(2, std::vector<bool>(2, true));
    Frontend::FrameResult last;
    int rejected = 0;
    for (int f = 0; f < 5; ++f) {
      if (!est.addStates(sc.frameId(), sc.t(sc.k), sc.imu(), false)) throw std::runtime_error("addStates failed");
      for (int c = 0; c < 2; ++c) {
        const Image im = sc.image(c);
        est.setFrameFeatures(sc.frameId(), c, im.kp, im.desc, std::vector<uint64_t>(im.kp.size(), 0));
      }
      const uint64_t id = sc.frameId();
      Frontend::RansacHooks hooks;
      if (mode && f == 4)
        hooks.afterKeyframe = [&](size_t, bool, size_t kf, uint64_t) {
          if (kf != 0) return false;
          const std::vector<uint64_t> ids = est.frameLandmarkIds(id, 0);
          for (size_t k = 0; k < ids.size() && rejected < 5; ++k) {
            if (ids[k] == 0) continue;
            est.removeObservation(ids[k], id, 0, k);
            if (mode == 2) est.setFrameLandmarkId(id, 0, k, 0);
            ++rejected;
          }
          return false;
        };
      bool kf = false;
      last = fe.dataAssociationAndInitialization(est, id, [&]() { return ++next; }, overlap, &kf, hooks);
      est.setKeyframe(id, kf);
      est.optimize(5);
      MapPointVector removed;
      est.applyMarginalizationStrategy(5, 3, removed);
      sc.k++;
    }
    if (last.keyframeCams.empty()) throw std::runtime_error("no device decision at the last frame");
    return std::make_pair(last.keyframeCams[0].n_matched, rejected);
  };
  const auto plain = runOnce(0), removeOnly = runOnce(1), withId = runOnce(2);
  std::printf("{\"mode\":\"reject\",\"matched\":%d,\"matched_remove_only\":%d,\"matched_set_id\":%d,\"rejected\":%d}\n",
              plain.first, removeOnly.first, withId.first, withId.second);
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
    if (mode == "--slide") return slide(argc > 2 ? argv[2] : "");
    if (mode == "--reject") return reject();
    std::printf("{\"error\":\"unknown mode\"}\n");
    return 1;
  } catch (const std::exception& e) {
    std::printf("{\"error\":\"%s\"}\n", e.what());
    return 1;
  }
}
