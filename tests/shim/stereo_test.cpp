// Exercises stereo landmark initialisation through the C++ mirror: Frontend::matchStereo and its EstimatorGroup form
// over a sliding window (addStates -> features -> matchToKeyframes3D2D / matchToLastFrame3D2D -> matchStereo ->
// optimize -> applyMarginalizationStrategy(5, 3)).  No landmark is created from the scene's truth: matchStereo makes
// every one of them.  Each session sees a stereo rig (0.11 m baseline) moving along +y past 300 points; every point has
// its own 48-byte descriptor (a few bits flipped per observation), and every image also holds 40 unrelated keypoints.
// Prints one JSON line per mode; tests/test_gpu_stereo_mirror.py checks them.
//   stereo_test.bin --no-gpu    the mirror fails loudly without a device
//   stereo_test.bin --slide     3 standalone sessions against the same 3 sessions in one EstimatorGroup, 24 frames
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
  c.frames = 12; c.landmarks = 2048; c.observations = 16384; c.imu_samples = 4096;
  c.featureKeypoints = 400; c.descriptorBytes = kDesc;
  return c;
}

struct Image { std::vector<okb_keypoint> kp; std::vector<uint8_t> desc; std::vector<uint64_t> truth; };

struct Scene {
  int seed;
  double vy;
  std::mt19937 rng;
  std::vector<std::array<double, 3>> lmk;
  std::vector<std::array<uint8_t, kDesc>> base;
  int k = 0;
  explicit Scene(int s) : seed(s), vy(1.0 + 0.1 * s), rng(23 + 31 * s) {
    std::uniform_real_distribution<double> ux(2.0, 6.0), uy(-4.0, 4.0 + vy * kDt * kFrames), uz(-1.5, 1.5);
    std::uniform_int_distribution<int> byte(0, 255);
    lmk.resize(kLandmarks); base.resize(kLandmarks);
    for (int l = 0; l < kLandmarks; ++l) {
      lmk[l] = {ux(rng), uy(rng), uz(rng)};
      for (auto& b : base[l]) b = (uint8_t)byte(rng);
    }
  }
  uint64_t frameId() const { return 100 + k; }
  int64_t t(int j) const { return 1000000000LL + (int64_t)(j * kDt * 1e9); }
  std::vector<ImuMeasurement> imu() const {
    std::vector<ImuMeasurement> meas;
    for (int64_t s = (k == 0 ? t(k) - 50000000LL : t(k - 1) - 5000000LL); s <= t(k) + 5000000LL; s += 5000000LL) {
      ImuMeasurement m{}; m.t_ns = s; m.acc[2] = kG; meas.push_back(m);
    }
    return meas;
  }
  bool keyframe() const { return k % 3 == 0; }
  void configure(Estimator& est) const {
    const okb_camera cam = camera();
    est.addCamera(ExtrinsicsEstimationParameters(), cam, Pose7{{0.0, 0.055, 0.0, -0.5, 0.5, -0.5, 0.5}});
    est.addCamera(ExtrinsicsEstimationParameters(), cam, Pose7{{0.0, -0.055, 0.0, -0.5, 0.5, -0.5, 0.5}});
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
    const double y_cam = vy * k * kDt;
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
  int kfMatches = 0, lastMatches = 0, stereoMatches = 0;
  std::vector<std::vector<uint64_t>> ids;
  bool operator==(const FrameRecord& o) const {
    return kfMatches == o.kfMatches && lastMatches == o.lastMatches && stereoMatches == o.stereoMatches && ids == o.ids;
  }
};

struct Totals {
  long landmarks = 0, observations = 0, mixed = 0, distractorObs = 0, framesTracked = 0, minMatches = 1 << 30, initChecked = 0;
  double maxRel = 0, sumRel = 0;
  std::string perFrame;
};

// every landmark's observations must see one true point; initialised ones must lie near it
void checkLandmarks(const Estimator& est, const Scene& sc, const std::map<uint64_t, std::vector<Image>>& truth, Totals& tot) {
  PointMap lms;
  est.getLandmarks(lms);
  const double y_cam = sc.vy * sc.k * kDt;
  for (auto& kv : lms) {
    std::set<uint64_t> seen;
    for (auto& o : kv.second.observations) {
      const uint64_t t = truth.at(o.first.frameId)[o.first.cameraIndex].truth.at(o.first.keypointIndex);
      seen.insert(t);
      ++tot.observations;
      if (t == 0) ++tot.distractorObs;
    }
    ++tot.landmarks;
    if (seen.size() > 1) { ++tot.mixed; continue; }
    if (seen.empty() || *seen.begin() == 0 || !est.isLandmarkInitialized(kv.first) || kv.second.observations.size() < 3) continue;
    const auto& P = sc.lmk[*seen.begin() - 100000];
    const auto& X = kv.second.point;
    const double e[3] = {X[0] / X[3] - P[0], X[1] / X[3] - P[1], X[2] / X[3] - P[2]};
    const double d = std::sqrt(P[0] * P[0] + (P[1] - y_cam) * (P[1] - y_cam) + P[2] * P[2]);
    const double rel = std::sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]) / d;
    tot.maxRel = std::max(tot.maxRel, rel); tot.sumRel += rel; ++tot.initChecked;
  }
}

// The sessions one by one (standalone Estimators) or together (one EstimatorGroup, group forms of every call).
std::vector<std::vector<FrameRecord>> run(bool grouped, Totals& tot) {
  std::unique_ptr<EstimatorGroup> g;
  if (grouped) g.reset(new EstimatorGroup(0, kSessions));
  Frontend fe(2);
  std::vector<std::unique_ptr<Estimator>> est;
  std::vector<std::unique_ptr<Scene>> sc;
  std::vector<uint64_t> next(kSessions);
  std::vector<std::function<uint64_t()>> newIds;
  for (int s = 0; s < kSessions; ++s) {
    est.emplace_back(grouped ? new Estimator(*g, capacity()) : new Estimator(0, capacity()));
    sc.emplace_back(new Scene(s));
    sc[s]->configure(*est[s]);
    next[s] = 1000000000ULL * (s + 1);                  // each session has its own id source
    uint64_t* n = &next[s];
    newIds.push_back([n]() { return ++*n; });
  }
  const std::vector<std::vector<bool>> overlap{{true, true}, {true, true}};
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
      ims = {sc[s]->image(0), sc[s]->image(1)};
      for (int c = 0; c < 2; ++c) est[s]->setFrameFeatures(sc[s]->frameId(), c, ims[c].kp, ims[c].desc, std::vector<uint64_t>(ims[c].kp.size(), 0));
      ids.push_back(sc[s]->frameId());
    }
    std::vector<Frontend::TrackResult> kf, last, st;
    if (grouped) {
      kf = fe.matchToKeyframes3D2D(*g, all, ids);
      last = fe.matchToLastFrame3D2D(*g, all, ids);
      st = fe.matchStereo(*g, all, ids, newIds, overlap);
    } else {
      for (int s = 0; s < kSessions; ++s) {
        kf.push_back(fe.matchToKeyframes3D2D(*est[s], ids[s]));
        last.push_back(fe.matchToLastFrame3D2D(*est[s], ids[s]));
        st.push_back(fe.matchStereo(*est[s], ids[s], newIds[s], overlap));
      }
    }
    std::vector<MapPointVector> removed(kSessions);
    if (grouped) g->optimize(all, 5);
    else for (int s = 0; s < kSessions; ++s) est[s]->optimize(5);
    for (int s = 0; s < kSessions; ++s) {
      FrameRecord r;
      r.kfMatches = kf[s].numMatches; r.lastMatches = last[s].numMatches; r.stereoMatches = st[s].numMatches;
      r.ids = st[s].landmarkIds;
      rec[s].push_back(r);
      if (f > 0) {
        ++tot.framesTracked;
        const int m = r.kfMatches + r.lastMatches;
        // min_matches counts from frame 4 on: before that the velocity is still being learnt
        if (f >= 4) tot.minMatches = std::min<long>(tot.minMatches, m);
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
    Totals ts, tg;
    const auto single = run(false, ts);
    const auto grouped = run(true, tg);
    int same = 1;
    for (int s = 0; s < kSessions; ++s) same &= (single[s] == grouped[s]) ? 1 : 0;
    std::printf("{\"mode\":\"slide\",\"frames\":%d,\"sessions\":%d,\"landmarks\":%ld,\"observations\":%ld,\"mixed\":%ld,"
                "\"distractor_obs\":%ld,\"frames_tracked\":%ld,\"min_matches\":%ld,\"init_checked\":%ld,\"max_rel\":%.6g,"
                "\"mean_rel\":%.6g,\"group_mixed\":%ld,\"group_equals_single\":%d,\"matches\":[%s]}\n",
                kFrames, kSessions, ts.landmarks, ts.observations, ts.mixed, ts.distractorObs, ts.framesTracked, ts.minMatches,
                ts.initChecked, ts.maxRel, ts.initChecked ? ts.sumRel / ts.initChecked : 0.0, tg.mixed, same, ts.perFrame.c_str());
  } catch (const std::exception& e) {
    std::printf("{\"error\":\"%s\"}\n", e.what());
    return 1;
  }
  return 0;
}
