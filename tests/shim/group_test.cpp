// Exercises okvis_b200::EstimatorGroup (include/okvis_b200_estimator.hpp): many sessions of the ThreadedKFVio cycle
// (addStates -> addLandmark / addObservation -> optimize -> applyMarginalizationStrategy(5, 3)) in one context.  Every
// session runs the scene of shim_test.cpp --sliding (stereo, 600 landmarks, constant velocity along +y, a keyframe every
// third frame), parameterised by seed, velocity and keyframe phase.  Prints one JSON line per mode;
// tests/test_gpu_estimator_group.py checks them and tools/bench_estimator_group.py drives --bench.
//   group_test.bin --no-gpu        a group fails loudly without a device
//   group_test.bin --arms          group batched vs one session per group call vs standalone Estimators, slot reuse
//   group_test.bin --rules         unlisted sessions untouched, launch count, list errors
//   group_test.bin --bench N F     host wall time per frame of N sessions over F frames, three ways
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <random>
#include <set>
#include <string>

#include "okvis_b200_estimator.hpp"

using namespace okvis_b200;

namespace {

constexpr double kG = 9.81007, kDt = 0.2;
constexpr int kLandmarks = 600;

okb_camera camera() {
  okb_camera cam{};
  cam.model = OKB_DIST_NONE; cam.width = 752; cam.height = 480; cam.fu = 450; cam.fv = 450; cam.cu = 376; cam.cv = 240;
  return cam;
}

// One session's scene and its host-side state (what a frontend would hold).
struct Scene {
  int seed = 0, phase = 0;
  double vy = 1.5;
  std::mt19937 rng;
  std::vector<std::array<double, 3>> lmk;
  std::set<uint64_t> gone;      // marginalised / dropped landmark ids do not come back
  int k = 0;                    // frames added so far
  explicit Scene(int s) : seed(s), phase(s % 3), vy(1.2 + 0.1 * (s % 7)), rng(11 + 17 * s) {
    const int n_frames = 64;
    std::uniform_real_distribution<double> ux(3.0, 9.0), uy(-4.0, 4.0 + vy * kDt * n_frames), uz(-1.5, 1.5);
    lmk.resize(kLandmarks);
    for (auto& p : lmk) p = {ux(rng), uy(rng), uz(rng)};
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
  bool keyframe() const { return (k + phase) % 3 == 0; }
  void configure(Estimator& est) const {
    const okb_camera cam = camera();
    est.addCamera(ExtrinsicsEstimationParameters(), cam, Pose7{{0.0, 0.055, 0.0, -0.5, 0.5, -0.5, 0.5}});
    est.addCamera(ExtrinsicsEstimationParameters(), cam, Pose7{{0.0, -0.055, 0.0, -0.5, 0.5, -0.5, 0.5}});
    okb_imu_params imu{};
    imu.a_max = 176; imu.g_max = 7.8; imu.sigma_g_c = 12e-4; imu.sigma_a_c = 8e-3; imu.sigma_bg = 0.03; imu.sigma_ba = 0.1;
    imu.sigma_gw_c = 4e-6; imu.sigma_aw_c = 4e-5; imu.tau = 3600; imu.g = kG; imu.rate = 200;
    est.addImu(imu);
  }
  // addLandmark / addObservation of frame k (after its addStates)
  void observe(Estimator& est) {
    const okb_camera cam = camera();
    std::normal_distribution<double> noise(0.0, 0.05);
    const double y_cam = vy * k * kDt;
    for (int l = 0; l < kLandmarks; ++l)
      for (int c = 0; c < 2; ++c) {
        const double xs = lmk[l][0], ys = lmk[l][1] - y_cam - (c == 0 ? 0.055 : -0.055), zs = lmk[l][2];
        const double xc = -ys, yc = -zs, zc = xs;
        const double px[2] = {cam.fu * xc / zc + cam.cu, cam.fv * yc / zc + cam.cv};
        if (!(zc > 0.5 && px[0] >= 0 && px[0] < 752 && px[1] >= 0 && px[1] < 480)) continue;
        const uint64_t lid = 100000 + l;
        if (!est.isLandmarkAdded(lid)) {
          if (gone.count(lid)) continue;
          est.addLandmark(lid, Vec4{{lmk[l][0] + noise(rng), lmk[l][1] + noise(rng), lmk[l][2] + noise(rng), 1.0}});
        }
        est.addObservation(lid, frameId(), c, l, px, 8.0);
      }
  }
};

// What a session's caller sees after a frame: ids and flags (bookkeeping) and numbers (estimates).
struct Record {
  std::vector<uint64_t> ids;
  std::vector<double> pose, sb, lm, cost;
  std::vector<int> iters;
};

void record(const Estimator& est, const MapPointVector& removed, Record& r) {
  r.ids.push_back(0xFFFF0000ull + est.numFrames());
  for (size_t a = 0; a < est.numFrames(); ++a) {
    const uint64_t id = est.frameIdByAge(a);
    r.ids.push_back(id * 4 + (est.isInImuWindow(id) ? 2 : 0) + (est.isKeyframe(id) ? 1 : 0));
    Pose7 T; est.get_T_WS(id, T);
    r.pose.insert(r.pose.end(), T.begin(), T.end());
    SpeedAndBias sb;
    if (est.getSpeedAndBias(id, 0, sb)) r.sb.insert(r.sb.end(), sb.begin(), sb.end());
  }
  MapPointVector lms;
  est.getLandmarks(lms);
  r.ids.push_back(0xEEEE0000ull + lms.size());
  for (auto& mp : lms) {
    r.ids.push_back(mp.id);
    r.lm.insert(r.lm.end(), mp.point.begin(), mp.point.end());
    r.lm.push_back(mp.quality);
  }
  r.ids.push_back(0xDDDD0000ull + removed.size());
  for (auto& mp : removed) r.ids.push_back(mp.id);
  const okb_summary& s = est.summary();
  r.cost.push_back(s.initial_cost); r.cost.push_back(s.final_cost); r.cost.push_back(s.final_radius);
  r.iters.push_back(s.iterations); r.iters.push_back(s.num_successful_steps); r.iters.push_back(s.termination);
}

bool same_bits(const std::vector<double>& a, const std::vector<double>& b) {
  return a.size() == b.size() && (a.empty() || !std::memcmp(a.data(), b.data(), sizeof(double) * a.size()));
}
bool same(const Record& a, const Record& b) {
  return a.ids == b.ids && a.iters == b.iters && same_bits(a.pose, b.pose) && same_bits(a.sb, b.sb) && same_bits(a.lm, b.lm) &&
         same_bits(a.cost, b.cost);
}

// ---- the 8-session schedule over 30 frames
constexpr int kSessions = 8, kFrames = 30, kLeaver = 3, kLeaveFrame = 12, kNewcomer = 8;
int join_frame(int s) { static const int j[kSessions + 1] = {0, 0, 1, 2, 3, 5, 6, 8, kLeaveFrame + 1}; return j[s]; }
bool active(int s, int f) { return f >= join_frame(s) && !(s == kLeaver && f > kLeaveFrame); }
// every fourth frame some sessions sit out optimize / applyMarginalizationStrategy
bool listed(int s, int f) { return f % 4 != 3 || (s + f / 4) % 3 != 0; }
// list order: rotated and reversed, so it is neither slot order nor contiguous
std::vector<int> order(const std::vector<int>& v, int f) {
  std::vector<int> o(v.rbegin(), v.rend());
  if (!o.empty()) std::rotate(o.begin(), o.begin() + (f % o.size()), o.end());
  return o;
}

enum class Arm { Batched, OneByOne, Standalone };

// Runs the schedule with the sessions in `which`; records[s][frame] per session.
std::vector<std::vector<Record>> run_arm(Arm arm, const std::set<int>& which, std::vector<int>* slots = nullptr) {
  std::unique_ptr<EstimatorGroup> g;
  if (arm != Arm::Standalone) g.reset(new EstimatorGroup(0, kSessions));
  std::vector<std::unique_ptr<Estimator>> est(kSessions + 1);
  std::vector<std::unique_ptr<Scene>> sc(kSessions + 1);
  std::vector<std::vector<Record>> rec(kSessions + 1);
  if (slots) slots->assign(kSessions + 1, -1);
  for (int f = 0; f < kFrames; ++f) {
    std::vector<int> act;
    for (int s = 0; s <= kSessions; ++s) {
      if (!which.count(s) || !active(s, f)) continue;
      if (!est[s]) {
        est[s].reset(g ? new Estimator(*g) : new Estimator(0));
        sc[s].reset(new Scene(s));
        sc[s]->configure(*est[s]);
        if (slots) (*slots)[s] = est[s]->slot();
      }
      act.push_back(s);
    }
    const std::vector<int> o = order(act, f);
    // addStates
    if (arm == Arm::Batched) {
      std::vector<EstimatorGroup::StatesRequest> req;
      for (int s : o) req.push_back({est[s].get(), sc[s]->frameId(), sc[s]->t(sc[s]->k), sc[s]->imu(), sc[s]->keyframe()});
      for (bool ok : g->addStates(req)) if (!ok) throw std::runtime_error("addStates failed");
    } else {
      for (int s : o) {
        bool ok;
        if (arm == Arm::OneByOne) ok = g->addStates({{est[s].get(), sc[s]->frameId(), sc[s]->t(sc[s]->k), sc[s]->imu(), sc[s]->keyframe()}})[0];
        else ok = est[s]->addStates(sc[s]->frameId(), sc[s]->t(sc[s]->k), sc[s]->imu(), sc[s]->keyframe());
        if (!ok) throw std::runtime_error("addStates failed");
      }
    }
    for (int s : o) sc[s]->observe(*est[s]);
    // the leaver goes with its frame's commands still pending
    if (f == kLeaveFrame && est[kLeaver]) {
      est[kLeaver].reset();
      act.erase(std::remove(act.begin(), act.end(), kLeaver), act.end());
    }
    std::vector<int> lst;
    for (int s : order(act, f + 1)) if (listed(s, f)) lst.push_back(s);
    std::vector<MapPointVector> removed(kSessions + 1);
    if (arm == Arm::Batched) {
      std::vector<Estimator*> l;
      for (int s : lst) l.push_back(est[s].get());
      g->optimize(l, 10);
      std::vector<MapPointVector> r;
      g->applyMarginalizationStrategy(l, 5, 3, r);
      for (size_t i = 0; i < lst.size(); ++i) removed[lst[i]] = r[i];
    } else {
      for (int s : lst) {
        if (arm == Arm::OneByOne) g->optimize({est[s].get()}, 10);
        else est[s]->optimize(10);
      }
      for (int s : lst) {
        if (arm == Arm::OneByOne) { std::vector<MapPointVector> r; g->applyMarginalizationStrategy({est[s].get()}, 5, 3, r); removed[s] = r[0]; }
        else est[s]->applyMarginalizationStrategy(5, 3, removed[s]);
      }
    }
    for (int s : act) {
      for (auto& mp : removed[s]) sc[s]->gone.insert(mp.id);
      Record r;
      record(*est[s], removed[s], r);
      rec[s].push_back(r);
      sc[s]->k++;
    }
  }
  est.clear();
  return rec;
}

int arms() {
  std::set<int> all;
  for (int s = 0; s <= kSessions; ++s) all.insert(s);
  std::vector<int> slotsA, slotsB;
  const auto A = run_arm(Arm::Batched, all, &slotsA);
  const auto B = run_arm(Arm::OneByOne, all, &slotsB);
  const auto C = run_arm(Arm::Standalone, all);
  const auto D = run_arm(Arm::Batched, {kNewcomer});           // the newcomer alone in a fresh group
  int records = 0, a_eq_b = 1, first_diff_session = -1, first_diff_frame = -1, ids_eq_c = 1, iter_diff = 0;
  double dpose = 0, dsb = 0, dcost = 0, dlm = 0;
  for (int s = 0; s <= kSessions; ++s) {
    if (A[s].size() != B[s].size() || A[s].size() != C[s].size()) { a_eq_b = 0; ids_eq_c = 0; continue; }
    for (size_t f = 0; f < A[s].size(); ++f) {
      ++records;
      if (!same(A[s][f], B[s][f]) && a_eq_b) { a_eq_b = 0; first_diff_session = s; first_diff_frame = (int)f; }
      const Record &a = A[s][f], &c = C[s][f];
      if (a.ids != c.ids || a.pose.size() != c.pose.size() || a.sb.size() != c.sb.size() || a.lm.size() != c.lm.size()) { ids_eq_c = 0; continue; }
      for (size_t i = 0; i < a.pose.size(); ++i) dpose = std::max(dpose, std::fabs(a.pose[i] - c.pose[i]));
      for (size_t i = 0; i < a.sb.size(); ++i) dsb = std::max(dsb, std::fabs(a.sb[i] - c.sb[i]));
      for (size_t i = 0; i < a.lm.size(); ++i) dlm = std::max(dlm, std::fabs(a.lm[i] - c.lm[i]));
      for (int i = 0; i < 2; ++i) dcost = std::max(dcost, std::fabs(a.cost[i] - c.cost[i]) / std::max(1e-300, std::fabs(c.cost[i])));
      if (a.iters[0] != c.iters[0]) ++iter_diff;
    }
  }
  int reuse_eq = A[kNewcomer].size() == D[kNewcomer].size() && !A[kNewcomer].empty();
  for (size_t f = 0; reuse_eq && f < A[kNewcomer].size(); ++f) reuse_eq = same(A[kNewcomer][f], D[kNewcomer][f]);
  int slots_eq = slotsA == slotsB;
  std::printf("{\"mode\": \"arms\", \"records\": %d, \"group_equals_one_by_one\": %d, \"first_diff_session\": %d, \"first_diff_frame\": %d, "
              "\"same_slots\": %d, \"leaver_slot\": %d, \"newcomer_slot\": %d, \"bookkeeping_equals_standalone\": %d, "
              "\"max_dpose\": %.3e, \"max_dsb\": %.3e, \"max_dlandmark\": %.3e, \"max_rel_dcost\": %.3e, \"iteration_diffs\": %d, "
              "\"reuse_equals_fresh\": %d, \"newcomer_frames\": %zu, \"final_frames\": %zu}\n",
              records, a_eq_b, first_diff_session, first_diff_frame, slots_eq, slotsA[kLeaver], slotsA[kNewcomer], ids_eq_c, dpose, dsb, dlm,
              dcost, iter_diff, reuse_eq, A[kNewcomer].size(), A[0].empty() ? (size_t)0 : A[0].back().pose.size() / 7);
  return 0;
}

// ---- unlisted sessions, launch count, errors
struct Snapshot { int64_t bytes; Record r; };
Snapshot snap(const Estimator& e) { Snapshot s; s.bytes = e.lastUploadBytes(); record(e, MapPointVector(), s.r); return s; }
bool same(const Snapshot& a, const Snapshot& b) { return a.bytes == b.bytes && same(a.r, b.r); }

// n sessions of group g stepped together for `frames` frames with group calls
void step_all(EstimatorGroup& g, std::vector<std::unique_ptr<Estimator>>& est, std::vector<std::unique_ptr<Scene>>& sc, int frames) {
  for (int f = 0; f < frames; ++f) {
    std::vector<EstimatorGroup::StatesRequest> req;
    std::vector<Estimator*> l;
    for (size_t s = 0; s < est.size(); ++s) {
      req.push_back({est[s].get(), sc[s]->frameId(), sc[s]->t(sc[s]->k), sc[s]->imu(), sc[s]->keyframe()});
      l.push_back(est[s].get());
    }
    g.addStates(req);
    for (size_t s = 0; s < est.size(); ++s) sc[s]->observe(*est[s]);
    g.optimize(l, 10);
    std::vector<MapPointVector> r;
    g.applyMarginalizationStrategy(l, 5, 3, r);
    for (size_t s = 0; s < est.size(); ++s) { for (auto& mp : r[s]) sc[s]->gone.insert(mp.id); sc[s]->k++; }
  }
}

int rules() {
  const int n = 4;
  auto make = [&](EstimatorGroup& g, std::vector<std::unique_ptr<Estimator>>& est, std::vector<std::unique_ptr<Scene>>& sc) {
    for (int s = 0; s < n; ++s) {
      est.emplace_back(new Estimator(g));
      sc.emplace_back(new Scene(s));
      sc[s]->configure(*est[s]);
    }
    step_all(g, est, sc, 6);
  };
  EstimatorGroup g1(0, n), g2(0, n);
  std::vector<std::unique_ptr<Estimator>> e1, e2;
  std::vector<std::unique_ptr<Scene>> s1, s2;
  make(g1, e1, s1);
  make(g2, e2, s2);
  // 4. session 2 adds its next frame (commands pending) and is left out of a group optimize of the others
  Snapshot before = snap(*e1[2]);
  if (!g1.addStates({{e1[2].get(), s1[2]->frameId(), s1[2]->t(s1[2]->k), s1[2]->imu(), s1[2]->keyframe()}})[0]) throw std::runtime_error("addStates");
  s1[2]->observe(*e1[2]);
  const Snapshot pending = snap(*e1[2]);
  for (int s : {0, 1, 3}) {
    g1.addStates({{e1[s].get(), s1[s]->frameId(), s1[s]->t(s1[s]->k), s1[s]->imu(), s1[s]->keyframe()}});
    s1[s]->observe(*e1[s]);
  }
  g1.optimize({e1[3].get(), e1[0].get(), e1[1].get()}, 10);
  const int64_t pending_bytes = pending.bytes;
  const int unlisted_ok = same(pending, snap(*e1[2])) && pending.bytes == before.bytes && e1[3]->summary().iterations > 0;
  // 5. launches: a group optimize of all sessions (one run of slots, one option set) vs one session alone, same state
  for (int s = 0; s < n; ++s) {
    g2.addStates({{e2[s].get(), s2[s]->frameId(), s2[s]->t(s2[s]->k), s2[s]->imu(), s2[s]->keyframe()}});
    s2[s]->observe(*e2[s]);
  }
  EstimatorGroup g3(0, n);
  std::vector<std::unique_ptr<Estimator>> e3;
  std::vector<std::unique_ptr<Scene>> s3;
  make(g3, e3, s3);
  for (int s = 0; s < n; ++s) {
    g3.addStates({{e3[s].get(), s3[s]->frameId(), s3[s]->t(s3[s]->k), s3[s]->imu(), s3[s]->keyframe()}});
    s3[s]->observe(*e3[s]);
  }
  int64_t l0 = g2.kernelLaunches();
  g2.optimize({e2[0].get(), e2[1].get(), e2[2].get(), e2[3].get()}, 10);
  const int64_t launches_all = g2.kernelLaunches() - l0;
  l0 = g3.kernelLaunches();
  g3.optimize({e3[0].get()}, 10);
  const int64_t launches_one = g3.kernelLaunches() - l0;
  // 6. errors: nothing changes
  std::vector<Snapshot> snaps;
  for (auto& e : e2) snaps.push_back(snap(*e));
  l0 = g2.kernelLaunches();
  Estimator standalone(0);
  int thrown = 0;
  std::vector<std::string> msgs;
  auto expect = [&](auto fn) {
    try { fn(); } catch (const std::invalid_argument& ex) { ++thrown; msgs.push_back(ex.what()); }
  };
  std::vector<MapPointVector> r;
  expect([&] { g2.optimize({e2[1].get(), e2[0].get(), e2[1].get()}, 10); });
  expect([&] { g2.optimize({e2[0].get(), e1[0].get()}, 10); });
  expect([&] { g2.optimize({e2[0].get(), &standalone}, 10); });
  expect([&] { g2.applyMarginalizationStrategy({e2[0].get(), e2[0].get()}, 5, 3, r); });
  expect([&] { g2.applyMarginalizationStrategy({e1[1].get()}, 5, 3, r); });
  expect([&] { g2.addStates({{e2[0].get(), 900, s2[0]->t(s2[0]->k), s2[0]->imu(), false}, {&standalone, 900, 0, {}, false}}); });
  expect([&] { g2.addStates({{e2[0].get(), 900, s2[0]->t(s2[0]->k), s2[0]->imu(), false}, {e2[0].get(), 901, 0, {}, false}}); });
  int full_throws = 0;
  try { Estimator extra(g2); } catch (const std::runtime_error&) { full_throws = 1; }
  int unchanged = g2.kernelLaunches() == l0 && g2.numSessions() == n && r.empty();
  for (int s = 0; s < n; ++s) unchanged = unchanged && same(snaps[s], snap(*e2[s])) && e2[s]->numFrames() == snaps[s].r.pose.size() / 7;
  // the group still works
  g2.optimize({e2[2].get(), e2[0].get()}, 10);
  std::string m;
  for (auto& x : msgs) m += (m.empty() ? "" : " | ") + x;
  std::printf("{\"mode\": \"rules\", \"unlisted_untouched\": %d, \"pending_bytes\": %lld, \"launches_all\": %lld, \"launches_one\": %lld, "
              "\"errors_thrown\": %d, \"full_group_throws\": %d, \"errors_change_nothing\": %d, \"still_works\": %d, \"messages\": \"%s\"}\n",
              unlisted_ok, (long long)pending_bytes, (long long)launches_all, (long long)launches_one, thrown, full_throws, unchanged,
              e2[2]->summary().iterations > 0 ? 1 : 0, m.c_str());
  return 0;
}

// ---- host wall time per frame of N sessions, three ways
using Clock = std::chrono::steady_clock;
double since(Clock::time_point t0) { return std::chrono::duration<double>(Clock::now() - t0).count(); }

struct Times { double add = 0, obs = 0, opt = 0, marg = 0, device = 0; int frames = 0; };

Times bench_arm(Arm arm, int N, int F, int skip) {
  std::unique_ptr<EstimatorGroup> g;
  if (arm != Arm::Standalone) g.reset(new EstimatorGroup(0, N));
  std::vector<std::unique_ptr<Estimator>> est;
  std::vector<std::unique_ptr<Scene>> sc;
  for (int s = 0; s < N; ++s) {
    est.emplace_back(g ? new Estimator(*g) : new Estimator(0));
    sc.emplace_back(new Scene(s));
    sc[s]->configure(*est[s]);
  }
  std::vector<Estimator*> all;
  for (auto& e : est) all.push_back(e.get());
  auto device = [&]() {
    if (g) return g->deviceSeconds();
    double d = 0;
    for (auto& e : est) d += e->deviceSeconds();
    return d;
  };
  Times T;
  for (int f = 0; f < F; ++f) {
    const bool timed = f >= skip;
    const double d0 = device();
    auto t0 = Clock::now();
    if (arm == Arm::Batched) {
      std::vector<EstimatorGroup::StatesRequest> req;
      for (int s = 0; s < N; ++s) req.push_back({all[s], sc[s]->frameId(), sc[s]->t(sc[s]->k), sc[s]->imu(), sc[s]->keyframe()});
      g->addStates(req);
    } else {
      for (int s = 0; s < N; ++s) {
        if (arm == Arm::OneByOne) g->addStates({{all[s], sc[s]->frameId(), sc[s]->t(sc[s]->k), sc[s]->imu(), sc[s]->keyframe()}});
        else all[s]->addStates(sc[s]->frameId(), sc[s]->t(sc[s]->k), sc[s]->imu(), sc[s]->keyframe());
      }
    }
    const double t_add = since(t0);
    t0 = Clock::now();
    for (int s = 0; s < N; ++s) sc[s]->observe(*all[s]);
    const double t_obs = since(t0);
    t0 = Clock::now();
    if (arm == Arm::Batched) g->optimize(all, 10);
    else for (int s = 0; s < N; ++s) { if (arm == Arm::OneByOne) g->optimize({all[s]}, 10); else all[s]->optimize(10); }
    const double t_opt = since(t0);
    t0 = Clock::now();
    std::vector<MapPointVector> removed(N);
    if (arm == Arm::Batched) g->applyMarginalizationStrategy(all, 5, 3, removed);
    else
      for (int s = 0; s < N; ++s) {
        if (arm == Arm::OneByOne) { std::vector<MapPointVector> r; g->applyMarginalizationStrategy({all[s]}, 5, 3, r); removed[s] = r[0]; }
        else all[s]->applyMarginalizationStrategy(5, 3, removed[s]);
      }
    const double t_marg = since(t0);
    for (int s = 0; s < N; ++s) { for (auto& mp : removed[s]) sc[s]->gone.insert(mp.id); sc[s]->k++; }
    if (timed) { T.add += t_add; T.obs += t_obs; T.opt += t_opt; T.marg += t_marg; T.device += device() - d0; T.frames++; }
  }
  est.clear();
  return T;
}

void print_times(const char* name, const Times& T) {
  const double k = 1e3 / std::max(1, T.frames);
  const double calls = T.add + T.opt + T.marg;
  std::printf("\"%s\": {\"ms_per_frame\": %.3f, \"add_states_ms\": %.3f, \"optimize_ms\": %.3f, \"marginalize_ms\": %.3f, "
              "\"device_calls_ms\": %.3f, \"host_bookkeeping_ms\": %.3f, \"observations_ms\": %.3f, \"frames\": %d}",
              name, k * calls, k * T.add, k * T.opt, k * T.marg, k * T.device, k * (calls - T.device), k * T.obs, T.frames);
}

int bench(int N, int F, int standalone_max) {
  const int skip = std::min(F - 1, 8);       // the first frames upload whole windows and capture solver graphs
  bench_arm(Arm::Batched, std::min(N, 8), std::min(F, skip + 2), skip);      // warm-up: modules, graphs
  const Times c = bench_arm(Arm::Batched, N, F, skip);
  const Times b = bench_arm(Arm::OneByOne, N, F, skip);
  std::printf("{\"mode\": \"bench\", \"sessions\": %d, \"frames\": %d, \"timed_frames\": %d, ", N, F, c.frames);
  print_times("group_batched", c);
  std::printf(", ");
  print_times("group_one_per_call", b);
  if (N <= standalone_max) {
    const Times a = bench_arm(Arm::Standalone, N, F, skip);
    std::printf(", ");
    print_times("standalone_loop", a);
  } else {
    std::printf(", \"standalone_loop\": null");
  }
  std::printf("}\n");
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  const std::string mode = argc > 1 ? argv[1] : "";
  try {
    if (mode == "--no-gpu") {
      try { EstimatorGroup g(0, 2); Estimator e(g); std::printf("{\"created\": true}\n"); }
      catch (const std::exception& ex) { std::printf("{\"created\": false, \"error\": \"%s\"}\n", ex.what()); }
      return 0;
    }
    if (mode == "--arms") return arms();
    if (mode == "--rules") return rules();
    if (mode == "--bench" && argc > 3) return bench(std::atoi(argv[2]), std::atoi(argv[3]), argc > 4 ? std::atoi(argv[4]) : 132);
  } catch (const std::exception& ex) {
    std::printf("{\"error\": \"%s\"}\n", ex.what());
    return 1;
  }
  std::fprintf(stderr, "usage: group_test.bin --no-gpu | --arms | --rules | --bench N F [standalone_max]\n");
  return 2;
}
