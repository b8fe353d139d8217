// Exercises Frontend::detectAndDescribe's store form (okb_detect_describe_store_batch) through the C++ mirror on real
// images: three stereo sessions slide over a textured plane, each frame addStates -> detectAndDescribe (store form) ->
// dataAssociationAndInitialization -> optimize -> applyMarginalizationStrategy, against twin sessions fed by the
// single-image detectAndDescribe + Estimator::setFrameFeatures.  Prints one JSON line per mode;
// tests/test_gpu_detect_store_mirror.py checks them.
//   detect_store_test.bin --no-gpu     the mirror fails loudly without a device
//   detect_store_test.bin --slide      store form standalone and as one group, twins standalone: everything a caller sees
//                                      compared frame by frame, bit for bit
//   detect_store_test.bin --refusals   the store form's refusals throw before anything changes
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

constexpr double kG = 9.81007, kDt = 0.2, kFu = 450.0, kDepth = 4.125;   // 12 px stereo disparity on the plane
constexpr int kW = 752, kH = 480, kFrames = 14, kRest = 3, kTexW = 1400;

okb_camera camera() {
  okb_camera cam{};
  cam.model = OKB_DIST_NONE; cam.width = kW; cam.height = kH; cam.fu = kFu; cam.fv = kFu; cam.cu = 376; cam.cv = 240;
  return cam;
}

Estimator::Capacity capacity(int keypoints = 450, int descBytes = 48) {
  Estimator::Capacity c;
  c.frames = 12; c.landmarks = 4096; c.observations = 16384; c.imu_samples = 4096;
  c.featureKeypoints = keypoints; c.descriptorBytes = descBytes;
  return c;
}

const Pose7 kT_SC[2] = {Pose7{{0.0, 0.055, 0.0, -0.5, 0.5, -0.5, 0.5}}, Pose7{{0.0, -0.055, 0.0, -0.5, 0.5, -0.5, 0.5}}};

// T_A * T_B for poses [t, q_xyzw]
Pose7 compose(const Pose7& a, const Pose7& b) {
  const double ax = a[3], ay = a[4], az = a[5], aw = a[6], bx = b[3], by = b[4], bz = b[5], bw = b[6];
  const double R[9] = {1 - 2 * (ay * ay + az * az), 2 * (ax * ay - az * aw), 2 * (ax * az + ay * aw),
                       2 * (ax * ay + az * aw), 1 - 2 * (ax * ax + az * az), 2 * (ay * az - ax * aw),
                       2 * (ax * az - ay * aw), 2 * (ay * az + ax * aw), 1 - 2 * (ax * ax + ay * ay)};
  Pose7 r;
  for (int i = 0; i < 3; ++i) r[i] = a[i] + R[3 * i] * b[0] + R[3 * i + 1] * b[1] + R[3 * i + 2] * b[2];
  r[3] = aw * bx + ax * bw + ay * bz - az * by;
  r[4] = aw * by - ax * bz + ay * bw + az * bx;
  r[5] = aw * bz + ax * by - ay * bx + az * bw;
  r[6] = aw * bw - ax * bx - ay * by - az * bz;
  return r;
}

// A rig looking along +x at a textured plane kDepth ahead, at rest for kRest frames and then accelerating along +y
// (y(t) = acc (t - t_rest)^2 / 2); camera c at body y = +-0.055 m.  The plane's texture (rectangles and discs on a
// shaded background) has one pixel per kDepth / fu metres, so camera c's image is the texture row-for-row, columns
// mirrored and shifted by the camera's y in pixels (rounded), with sensor noise.
struct Scene {
  double acc;
  int seed;
  std::vector<uint8_t> tex;          // [kH][kTexW]
  int k = 0;
  Scene(int s, double a) : acc(a), seed(s), tex((size_t)kH * kTexW) {
    std::mt19937 rng(1000 + 77 * s);
    std::vector<double> img((size_t)kH * kTexW);
    for (int y = 0; y < kH; ++y)
      for (int x = 0; x < kTexW; ++x) img[(size_t)y * kTexW + x] = 110.0 + 25.0 * std::sin(x / 97.0) * std::cos(y / 71.0);
    std::uniform_real_distribution<double> ux(0, kTexW), uy(0, kH), us(4, 40), uv(20, 235), u01(0, 1);
    for (int i = 0; i < 1700; ++i) {
      const double cx = ux(rng), cy = uy(rng), w = us(rng), h = us(rng), v = uv(rng);
      const bool rect = u01(rng) < 0.6;
      const double r = std::max(w, h);
      for (int y = std::max(0, (int)(cy - r)); y < std::min(kH, (int)(cy + r) + 1); ++y)
        for (int x = std::max(0, (int)(cx - r)); x < std::min(kTexW, (int)(cx + r) + 1); ++x) {
          const bool in = rect ? (std::fabs(x - cx) < w / 2 && std::fabs(y - cy) < h / 2) : ((x - cx) * (x - cx) + (y - cy) * (y - cy) < w * w / 4);
          if (in) img[(size_t)y * kTexW + x] = v;
        }
    }
    for (size_t i = 0; i < img.size(); ++i) tex[i] = (uint8_t)std::min(255.0, std::max(0.0, std::rint(img[i])));
  }
  uint64_t frameId() const { return 100 + k; }
  int64_t t(int j) const { return 1000000000LL + (int64_t)(j * kDt * 1e9); }
  double yRig() const { const double tt = std::max(0, k - kRest) * kDt; return 0.5 * acc * tt * tt; }
  std::vector<ImuMeasurement> imu() const {
    std::vector<ImuMeasurement> meas;
    for (int64_t s = (k == 0 ? t(k) - 50000000LL : t(k - 1) - 5000000LL); s <= t(k) + (k == 0 ? 0 : 5000000LL); s += 5000000LL) {
      ImuMeasurement m{}; m.t_ns = s; m.acc[1] = s > t(kRest) ? acc : 0.0; m.acc[2] = kG; meas.push_back(m);
    }
    return meas;
  }
  void configure(Estimator& est) const {
    for (int c = 0; c < 2; ++c) est.addCamera(ExtrinsicsEstimationParameters(), camera(), kT_SC[c]);
    okb_imu_params imu{};
    imu.a_max = 176; imu.g_max = 7.8; imu.sigma_g_c = 12e-4; imu.sigma_a_c = 8e-3; imu.sigma_bg = 0.03; imu.sigma_ba = 0.1;
    imu.sigma_gw_c = 4e-6; imu.sigma_aw_c = 4e-5; imu.tau = 3600; imu.g = kG; imu.rate = 200;
    est.addImu(imu);
  }
  // camera c's image of frame k, row stride kW + 8 (the padding holds 0)
  std::vector<uint8_t> image(int c) const {
    // image column x shows the plane at world y = y_cam - (x - cu) kDepth / fu: texture column s - x
    const double yCam = yRig() + (c == 0 ? 0.055 : -0.055);
    const int s = 1380 - (int)std::lround(yCam * kFu / kDepth);     // 1047..1386 over the run: s - x stays on the texture
    std::mt19937 rng(seed * 7919 + k * 31 + c);
    std::normal_distribution<double> noise(0.0, 2.0);
    std::vector<uint8_t> im((size_t)kH * (kW + 8), 0);
    for (int y = 0; y < kH; ++y)
      for (int x = 0; x < kW; ++x)
        im[(size_t)y * (kW + 8) + x] = (uint8_t)std::min(255.0, std::max(0.0, std::rint(tex[(size_t)y * kTexW + (s - x)] + noise(rng))));
    return im;
  }
};

uint64_t bits(double v) { uint64_t u; std::memcpy(&u, &v, 8); return u; }
uint64_t bitsf(float v) { uint32_t u; std::memcpy(&u, &v, 4); return u; }

// Everything a caller sees of one session's frame, as raw bits.
struct Digest {
  std::vector<uint64_t> w;
  void kp(const std::vector<okb_keypoint>& k) {
    w.push_back(k.size());
    for (const okb_keypoint& p : k) for (float f : {p.x, p.y, p.size, p.angle, p.response}) w.push_back(bitsf(f)), w.push_back((uint64_t)p.octave);
  }
  void ids(const std::vector<std::vector<uint64_t>>& v) { for (auto& c : v) { w.push_back(c.size()); w.insert(w.end(), c.begin(), c.end()); } }
};

struct Totals { long keypoints = 0, num3d = 0, decisions = 0, trackedLandmarks = 0; double maxPosErr = 0; };

enum class Mode { Store, StoreGroup, Twin };

std::vector<std::vector<Digest>> run(Mode mode, Totals& tot) {
  const int nSessions = 3;
  const bool grouped = mode == Mode::StoreGroup;
  std::unique_ptr<EstimatorGroup> g;
  if (grouped) g.reset(new EstimatorGroup(0, nSessions));
  std::vector<std::unique_ptr<Frontend>> fe;
  std::vector<std::unique_ptr<Estimator>> est;
  std::vector<std::unique_ptr<Scene>> sc;
  std::vector<uint64_t> next(nSessions);
  std::vector<std::function<uint64_t()>> newIds;
  for (int s = 0; s < nSessions; ++s) {
    est.emplace_back(grouped ? new Estimator(*g, capacity()) : new Estimator(0, capacity()));
    sc.emplace_back(new Scene(s, 1.0 + 0.25 * s));
    sc[s]->configure(*est[s]);
    if (!grouped || s == 0) fe.emplace_back(new Frontend(2));
    next[s] = 1000000000ULL * (s + 1);
    uint64_t* n = &next[s];
    newIds.push_back([n]() { return ++*n; });
  }
  const std::vector<std::vector<bool>> overlap(2, std::vector<bool>(2, true));
  std::vector<std::vector<Digest>> rec(nSessions);
  std::vector<Estimator*> all;
  for (auto& e : est) all.push_back(e.get());
  std::vector<char> initialized(nSessions, 0);
  for (int f = 0; f < kFrames; ++f) {
    std::vector<uint64_t> fid;
    for (int s = 0; s < nSessions; ++s) fid.push_back(sc[s]->frameId());
    if (grouped) {
      std::vector<EstimatorGroup::StatesRequest> req;
      for (int s = 0; s < nSessions; ++s) req.push_back({all[s], fid[s], sc[s]->t(sc[s]->k), sc[s]->imu(), false});
      for (bool ok : g->addStates(req)) if (!ok) throw std::runtime_error("addStates failed");
    } else {
      for (int s = 0; s < nSessions; ++s)
        if (!est[s]->addStates(fid[s], sc[s]->t(sc[s]->k), sc[s]->imu(), false)) throw std::runtime_error("addStates failed");
    }
    // the frame's images with T_WC from the propagated T_WS, as frameConsumerLoop hands them over
    std::vector<std::vector<std::vector<uint8_t>>> pix(nSessions);
    std::vector<std::vector<Frontend::CameraImage>> images(nSessions);
    for (int s = 0; s < nSessions; ++s) {
      Pose7 T_WS;
      est[s]->get_T_WS(fid[s], T_WS);
      for (int c = 0; c < 2; ++c) pix[s].push_back(sc[s]->image(c));
      for (int c = 0; c < 2; ++c) {
        Frontend::CameraImage im;
        im.image = pix[s][c].data(); im.width = kW; im.height = kH; im.stride = kW + 8; im.T_WC = compose(T_WS, kT_SC[c]);
        images[s].push_back(im);
      }
    }
    std::vector<std::vector<std::vector<okb_keypoint>>> kps(nSessions);
    if (mode == Mode::StoreGroup) {
      kps = fe[0]->detectAndDescribe(*g, all, fid, images);
    } else if (mode == Mode::Store) {
      for (int s = 0; s < nSessions; ++s) kps[s] = fe[s]->detectAndDescribe(*est[s], fid[s], images[s]);
    } else {
      for (int s = 0; s < nSessions; ++s)
        for (int c = 0; c < 2; ++c) {
          const Frontend::CameraImage& im = images[s][c];
          std::vector<okb_keypoint> kp;
          std::vector<uint8_t> desc;
          fe[s]->detectAndDescribe(c, im.image, im.width, im.height, im.stride, camera(), im.T_WC.data(), kp, desc);
          est[s]->setFrameFeatures(fid[s], c, kp, desc, std::vector<uint64_t>(kp.size(), 0));
          kps[s].push_back(kp);
        }
    }
    std::vector<Frontend::FrameResult> res(nSessions);
    std::vector<char> kf(nSessions, 0);
    if (grouped) {
      res = fe[0]->dataAssociationAndInitialization(*g, all, fid, newIds, overlap, kf, {}, initialized);
    } else {
      for (int s = 0; s < nSessions; ++s) {
        bool k = false;
        res[s] = fe[s]->dataAssociationAndInitialization(*est[s], fid[s], newIds[s], overlap, &k);
        kf[s] = k ? 1 : 0;
      }
    }
    std::vector<Digest> d(nSessions);
    for (int s = 0; s < nSessions; ++s) {
      for (int c = 0; c < 2; ++c) { d[s].kp(kps[s][c]); tot.keypoints += (long)kps[s][c].size(); }
      d[s].ids(res[s].landmarkIds);
      d[s].ids(res[s].keyframeIds);
      d[s].w.push_back((uint64_t)kf[s]);
      d[s].w.push_back((uint64_t)res[s].num3dMatches);
      tot.num3d += res[s].num3dMatches;
      for (const okb_keyframe_cam& k : res[s].keyframeCams)
        for (uint64_t v : {(uint64_t)k.n_points, (uint64_t)k.n_matched, (uint64_t)k.hull_all, (uint64_t)k.hull_matched, (uint64_t)k.inside,
                           (uint64_t)k.skipped, bits(k.area_all), bits(k.area_matched), bits(k.overlap), bits(k.ratio)})
          d[s].w.push_back(v);
      if (!res[s].keyframeCams.empty()) {
        ++tot.decisions;
        for (uint64_t v : {bits(res[s].keyframe.overlap), bits(res[s].keyframe.ratio), (uint64_t)res[s].keyframe.need_keyframe}) d[s].w.push_back(v);
      }
      est[s]->setKeyframe(fid[s], kf[s] != 0);
    }
    if (grouped) g->optimize(all, 5);
    else for (int s = 0; s < nSessions; ++s) est[s]->optimize(5);
    for (int s = 0; s < nSessions; ++s) {
      // the estimates: the frame's pose and speed/bias, and every landmark the frame names with its observations
      Pose7 T;
      est[s]->get_T_WS(fid[s], T);
      for (double v : T) d[s].w.push_back(bits(v));
      SpeedAndBias sb;
      if (est[s]->getSpeedAndBias(fid[s], 0, sb)) for (double v : sb) d[s].w.push_back(bits(v));
      tot.maxPosErr = std::max(tot.maxPosErr, std::sqrt(T[0] * T[0] + (T[1] - sc[s]->yRig()) * (T[1] - sc[s]->yRig()) + T[2] * T[2]));
      for (int c = 0; c < 2; ++c)
        for (uint64_t id : est[s]->frameLandmarkIds(fid[s], c)) {
          MapPoint mp;
          if (!id || !est[s]->getLandmark(id, mp)) continue;
          for (double v : mp.point) d[s].w.push_back(bits(v));
          d[s].w.push_back(mp.observations.size());
          for (auto& o : mp.observations) for (uint64_t v : {o.first.frameId, (uint64_t)o.first.cameraIndex, (uint64_t)o.first.keypointIndex}) d[s].w.push_back(v);
          if (f > 0 && mp.observations.begin()->first.frameId < fid[s]) ++tot.trackedLandmarks;
        }
      rec[s].push_back(d[s]);
    }
    std::vector<MapPointVector> removed(nSessions);
    if (grouped) g->applyMarginalizationStrategy(all, 5, 3, removed);
    else for (int s = 0; s < nSessions; ++s) est[s]->applyMarginalizationStrategy(5, 3, removed[s]);
    for (int s = 0; s < nSessions; ++s) sc[s]->k++;
  }
  est.clear();
  return rec;
}

// the first (session, frame) where two runs differ, or -1
int firstDiff(const std::vector<std::vector<Digest>>& a, const std::vector<std::vector<Digest>>& b) {
  for (size_t f = 0; f < (size_t)kFrames; ++f)
    for (size_t s = 0; s < a.size(); ++s)
      if (a[s][f].w != b[s][f].w) return (int)(s * 1000 + f);
  return -1;
}

int slide() {
  Totals ts, tg, tt;
  const auto store = run(Mode::Store, ts);
  const auto group = run(Mode::StoreGroup, tg);
  const auto twin = run(Mode::Twin, tt);
  std::printf("{\"mode\":\"slide\",\"frames\":%d,\"sessions\":3,\"store_vs_twin_first_diff\":%d,\"group_vs_single_first_diff\":%d,"
              "\"keypoints\":%ld,\"num3d\":%ld,\"decisions\":%ld,\"tracked_landmarks\":%ld,\"max_pos_err\":%.6f}\n",
              kFrames, firstDiff(store, twin), firstDiff(group, store), ts.keypoints, ts.num3d, ts.decisions, ts.trackedLandmarks,
              ts.maxPosErr);
  return 0;
}

// Each refusal throws, and leaves the frame without features: the session then takes the valid call as a fresh one.
int refusals() {
  Scene sc(9, 1.0);
  std::vector<uint8_t> px[2] = {sc.image(0), sc.image(1)};
  std::vector<Frontend::CameraImage> ims(2);
  for (int c = 0; c < 2; ++c) { ims[c].image = px[c].data(); ims[c].width = kW; ims[c].height = kH; ims[c].stride = kW + 8; ims[c].T_WC = kT_SC[c]; }
  int thrown = 0, cases = 0;
  auto expectThrow = [&](const std::function<void()>& f) { ++cases; try { f(); } catch (const std::exception&) { ++thrown; } };
  Frontend fe(2);
  {
    Estimator est(0, capacity());
    sc.configure(est);
    expectThrow([&]() { fe.detectAndDescribe(est, sc.frameId(), ims); });                    // frame not in the window
    if (!est.addStates(sc.frameId(), sc.t(0), sc.imu(), false)) throw std::runtime_error("addStates failed");
    expectThrow([&]() { fe.detectAndDescribe(est, sc.frameId(), {ims[0]}); });               // one image for two cameras
    fe.setDescriptorBytes(64);
    expectThrow([&]() { fe.detectAndDescribe(est, sc.frameId(), ims); });                    // 64-byte descriptors, 48-byte store
    fe.setDescriptorBytes(48);
    fe.setBriskDetectionMaximumKeypoints(451);
    expectThrow([&]() { fe.detectAndDescribe(est, sc.frameId(), ims); });                    // 451 keypoints, store of 450
    fe.setBriskDetectionMaximumKeypoints(450);
    const bool untouched = est.frameLandmarkIds(sc.frameId(), 0).empty();
    const auto kp = fe.detectAndDescribe(est, sc.frameId(), ims);
    std::vector<okb_keypoint> single;
    std::vector<uint8_t> desc;
    fe.detectAndDescribe(0, ims[0].image, kW, kH, kW + 8, camera(), ims[0].T_WC.data(), single, desc);
    bool same = kp[0].size() == single.size() && std::memcmp(kp[0].data(), single.data(), single.size() * sizeof(okb_keypoint)) == 0;
    same = same && est.frameLandmarkIds(sc.frameId(), 0) == std::vector<uint64_t>(single.size(), 0);
    std::printf("{\"mode\":\"refusals\",\"cases\":%d,\"thrown\":%d,\"untouched\":%d,\"valid_after\":%d,\"keypoints\":%zu}\n", cases, thrown,
                untouched ? 1 : 0, same ? 1 : 0, single.size());
  }
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
    if (mode == "--refusals") return refusals();
    std::printf("{\"error\":\"unknown mode\"}\n");
    return 1;
  } catch (const std::exception& e) {
    std::printf("{\"error\":\"%s\"}\n", e.what());
    return 1;
  }
}
