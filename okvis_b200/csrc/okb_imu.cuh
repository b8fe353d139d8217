// IMU preintegration / propagation / residual for the CUDA estimator path, written ONCE against a
// tiny "cooperative context" so the same code runs (a) warp-cooperatively inside kernels (32 lanes
// share the 15x15 products through shared memory, small 3x3 algebra is replicated per lane) and
// (b) sequentially on the host for the GPU-less host check (tests/hostcheck).
//
// Mirrors, re-organised: ImuError::redoPreintegration (okvis_ceres/src/ImuError.cpp:76-284), the static
// ImuError::propagation (:287-504) and ImuError::EvaluateWithMinimalJacobians (:514-685).
#pragma once
#include "okb_math.cuh"

namespace okb {

struct SeqCtx {  // host / single thread
  OKB_HD int lane() const { return 0; }
  OKB_HD int lanes() const { return 1; }
  OKB_HD void sync() const {}
};
#if defined(__CUDACC__)
struct WarpCtx {  // one warp
  __device__ __forceinline__ int lane() const { return threadIdx.x & 31; }
  __device__ __forceinline__ int lanes() const { return 32; }
  __device__ __forceinline__ void sync() const { __syncwarp(); }
};
// G lanes of a warp (G = 8, 16, 32): 32 / G independent groups share one warp, each working on its own term.  The
// small algebra every lane replicates is then issued once for 32 / G terms; the groups may diverge freely (sync()
// only names the group's own lanes).
template <int G>
struct GroupCtx {
  __device__ __forceinline__ int lane() const { return threadIdx.x & (G - 1); }
  __device__ __forceinline__ int lanes() const { return G; }
  __device__ __forceinline__ void sync() const {
    const unsigned m = (G == 32) ? 0xffffffffu : (((1u << (G & 31)) - 1u) << ((threadIdx.x & 31) & ~(G - 1)));
    __syncwarp(m);
  }
};
#endif

// Device-resident cache of one ImuError term (the reference's mutable members, ImuError.hpp:251-276).
struct ImuCache {
  double Delta_q[4];
  double C_integral[9], C_doubleintegral[9];
  double acc_integral[3], acc_doubleintegral[3];
  double dalpha_db_g[9], dv_db_g[9], dp_db_g[9];
  double sqrt_info[225];   // upper triangular L^T of the information matrix
  double sb_ref[9];
  int valid;               // 0 = redo_ (never preintegrated)
  int redo_count;
};

// replicated small state of the integration loop
struct ImuInt {
  double Delta_q[4];
  double C_integral[9], C_doubleintegral[9];
  double acc_integral[3], acc_doubleintegral[3];
  double cross[9];
  double dalpha_db_g[9], dv_db_g[9], dp_db_g[9];
  double Delta_t;
};

OKB_HD double ns_to_sec(int64_t ns) {
  int64_t sec = ns / 1000000000LL, nsec = ns % 1000000000LL;
  if (nsec < 0) { nsec += 1000000000LL; sec -= 1; }
  return (double)sec + 1e-9 * (double)nsec;
}

// imu_integrate works through the samples in batches of kImuBatch.  Each sample has a record of kImuRec doubles:
// first its precompute (kImuPre doubles: valid, dt, sigma_g, sigma_a, ac(3), dq(4), Jr(9), R(dq^-1)(9), last), then,
// written over it by the state step, what the covariance step needs: flag (0 skip, 1 integrate, 2 integrate and
// stop), dt, sigma_g, sigma_a, add(3), 0.5 CCa dt(3), F09, F012, C1, sumA, CC (3x3 each).
constexpr int kImuPre = 30;
constexpr int kImuRec = 55;
constexpr int kImuBatch = 8;
constexpr int kImuState = (int)(sizeof(ImuInt) / sizeof(double));

// Workspace of one term (shared memory on the device).
struct ImuWork {
  double* P;    // covariance (result), 15x15
  double* F;    // 15x15 scratch
  double* T;    // 15x15 scratch
  double* St;   // the running ImuInt of imu_integrate (kImuState doubles), read by every lane afterwards
  double* S;    // kImuBatch x kImuRec per-sample records; only imu_integrate uses them, so they may overlay F and T
  OKB_HD ImuInt& state() const { return *reinterpret_cast<ImuInt*>(St); }
};

// One term's shared scratch of kImuScratch doubles: P | F | T with the records over F | T and the state behind T.  Once
// the preintegration has stored sqrt_info all of that is dead, and the evaluation's [F0|F1] (450), sqrt_info [F0|F1]
// (450) and r15 (15 + 1 pad) reuse the space.
constexpr int kImuScratch = 450 + 450 + 16;
static_assert(kImuBatch * kImuRec <= 450 && 675 + kImuState <= kImuScratch, "IMU scratch layout");
struct ImuScratch {
  ImuWork wk;
  double* F01;
  double* SF;
  double* r15;
};
OKB_HD ImuScratch imu_scratch(double* buf) {
  return ImuScratch{ImuWork{buf, buf + 225, buf + 450, buf + 675, buf + 225}, buf, buf + 450, buf + 900};
}

// y = F x for the 15-vector x with F = I + N (N as listed in imu_integrate): rows 0..8 only.
OKB_HD void imu_apply_F(const double* x, double* y, double dt, const double* X03, const double* F09,
                               const double* F012, const double* C1, const double* X63, const double* sumA,
                               const double* CC) {
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    double r0 = x[a] + dt * x[6 + a], r1 = 0.0, r2 = x[6 + a], r2b = 0.0, r2c = 0.0;
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      r0 -= X03[a * 3 + b] * x[3 + b];
      r0 += F09[a * 3 + b] * x[9 + b];
      r0 += F012[a * 3 + b] * x[12 + b];
      r1 += C1[a * 3 + b] * x[9 + b];
      r2 -= X63[a * 3 + b] * x[3 + b];
      r2b += sumA[a * 3 + b] * x[9 + b];
      r2c += CC[a * 3 + b] * x[12 + b];
    }
    y[a] = r0;
    y[3 + a] = x[3 + a] - dt * r1;
    y[6 + a] = r2 + 0.5 * dt * (r2b - r2c);
  }
#pragma unroll
  for (int k = 9; k < 15; ++k) y[k] = x[k];
}

// Integrates the samples over [t0,t1].  PREINT selects the redoPreintegration variant
// (dalpha_db_g uses the right Jacobian; sigma2_v = dt*sigma_a_c^2), otherwise the propagation variant.
// Returns the number of steps (-1 if the samples do not reach t1).  The final state is left in wk.state(); with
// WANT_COV the covariance is accumulated in wk.P.
template <bool PREINT, bool WANT_COV, class Ctx>
OKB_HD int imu_integrate(const Ctx& cx, const okb_imu_sample* s, int n, const okb_imu_params& prm, int64_t t0,
                         int64_t t1, const double* sb, ImuWork wk) {
  if (!(s[n - 1].t_ns >= t1)) return -1;
  ImuInt& st = wk.state();
  if (cx.lane() == 0) {
    st.Delta_q[0] = st.Delta_q[1] = st.Delta_q[2] = 0; st.Delta_q[3] = 1;
    for (int k = 0; k < 9; ++k) {
      st.C_integral[k] = st.C_doubleintegral[k] = st.cross[k] = 0;
      st.dalpha_db_g[k] = st.dv_db_g[k] = st.dp_db_g[k] = 0;
    }
    for (int k = 0; k < 3; ++k) st.acc_integral[k] = st.acc_doubleintegral[k] = 0;
    st.Delta_t = 0;
  }
  double* Pc = wk.P;   // covariance, updated in place
  if (WANT_COV)
    for (int e = cx.lane(); e < 225; e += cx.lanes()) wk.P[e] = 0.0;
  cx.sync();
  // Three passes per batch of samples, with the same formulas and the same order of operations per sample as the
  // reference loop:
  //  1. the quantities that do not depend on the running state (interpolated rates, dt, the rotation increment dq
  //     with its sinc/cos, the right Jacobian, R(dq^-1), saturation flags), one sample per lane;
  //  2. the state recursion (3x3 algebra) on lane 0, which leaves in each sample's record the blocks of N;
  //  3. the covariance recursion, which reads those blocks as broadcast loads.
  // The state does not depend on the covariance, so 2 can run ahead of 3; keeping them apart keeps the running state
  // out of the registers of the 15-wide covariance products.
  int i = 0;
  bool finished = false;
  for (int base = 0; base < n && !finished; base += kImuBatch) {
    for (int j = cx.lane(); j < kImuBatch; j += cx.lanes()) {
      const int it = base + j;
      double* o = wk.S + j * kImuRec;
      o[0] = 0.0;
      if (it >= n) continue;
      const bool last = (it + 1 == n);
      double w0[3], a0[3], w1[3], a1[3];
      for (int k = 0; k < 3; ++k) {
        w0[k] = s[it].gyro[k]; a0[k] = s[it].acc[k];
        w1[k] = s[last ? it : it + 1].gyro[k]; a1[k] = s[last ? it : it + 1].acc[k];
      }
      // `time` of the reference loop: t0 for the first integrated interval, the sample's own stamp afterwards
      const int64_t start = (s[it].t_ns > t0) ? s[it].t_ns : t0;
      int64_t nexttime = last ? t1 : s[it + 1].t_ns;
      double dt = ns_to_sec(nexttime - start);
      if (t1 < nexttime) {
        const double interval = ns_to_sec(nexttime - s[it].t_ns);
        nexttime = t1;
        dt = ns_to_sec(nexttime - start);
        const double r = dt / interval;
        for (int k = 0; k < 3; ++k) { w1[k] = (1.0 - r) * w0[k] + r * w1[k]; a1[k] = (1.0 - r) * a0[k] + r * a1[k]; }
      }
      if (dt <= 0.0) continue;
      if (s[it].t_ns <= t0) {   // first integrated interval (hasStarted == false in the reference)
        const double r = dt / ns_to_sec(nexttime - s[it].t_ns);
        for (int k = 0; k < 3; ++k) { w0[k] = r * w0[k] + (1.0 - r) * w1[k]; a0[k] = r * a0[k] + (1.0 - r) * a1[k]; }
      }
      double sigma_g_c = prm.sigma_g_c, sigma_a_c = prm.sigma_a_c;
      bool gsat = false, asat = false;
      for (int k = 0; k < 3; ++k) {
        if (fabs(w0[k]) > prm.g_max || fabs(w1[k]) > prm.g_max) gsat = true;
        if (fabs(a0[k]) > prm.a_max || fabs(a1[k]) > prm.a_max) asat = true;
      }
      if (gsat) sigma_g_c *= 100;
      if (asat) sigma_a_c *= 100;
      double om[3];
      for (int k = 0; k < 3; ++k) { om[k] = 0.5 * (w0[k] + w1[k]) - sb[3 + k]; o[4 + k] = 0.5 * (a0[k] + a1[k]) - sb[6 + k]; }
      const double th = sqrt(om[0] * om[0] + om[1] * om[1] + om[2] * om[2]) * 0.5 * dt;
      const double sc = sinc(th) * 0.5 * dt;
      const double dq[4] = {sc * om[0], sc * om[1], sc * om[2], cos(th)};
      const double wdt[3] = {om[0] * dt, om[1] * dt, om[2] * dt};
      double Jr[9], dqi[4], Rdqi[9];
      rightJacobian(wdt, Jr);
      qinv(dq, dqi);
      q2R(dqi, Rdqi);
      o[1] = dt; o[2] = sigma_g_c; o[3] = sigma_a_c;
      for (int k = 0; k < 4; ++k) o[7 + k] = dq[k];
      for (int k = 0; k < 9; ++k) { o[11 + k] = Jr[k]; o[20 + k] = Rdqi[k]; }
      o[29] = (nexttime == t1) ? 1.0 : 0.0;
      o[0] = 1.0;
    }
    cx.sync();
    for (int j = 0; cx.lane() == 0 && j < kImuBatch && base + j < n; ++j) {   // the state recursion: lane 0 only
      double* o = wk.S + j * kImuRec;
      if (o[0] == 0.0) continue;
      const double dt = o[1];
      const double ac[3] = {o[4], o[5], o[6]};
      const double dq[4] = {o[7], o[8], o[9], o[10]};
      const double* Jr = o + 11;
      const double* Rdqi = o + 20;
      const bool last = (o[29] != 0.0);
      st.Delta_t += dt;
      double q1[4];
      qmul(st.Delta_q, dq, q1);
      double C[9], C1[9], CC[9], CCa[3];
      q2R(st.Delta_q, C);
      q2R(q1, C1);
      for (int k = 0; k < 9; ++k) CC[k] = C[k] + C1[k];
      mat3vec(CC, ac, CCa);
      double Ci1[9], ai1[3], add[3];
      for (int k = 0; k < 9; ++k) Ci1[k] = st.C_integral[k] + 0.5 * CC[k] * dt;
      for (int k = 0; k < 3; ++k) ai1[k] = st.acc_integral[k] + 0.5 * CCa[k] * dt;
      double F012[9];
      for (int k = 0; k < 9; ++k) {
        F012[k] = -st.C_integral[k] * dt + 0.25 * CC[k] * dt * dt;
        st.C_doubleintegral[k] += st.C_integral[k] * dt + 0.25 * CC[k] * dt * dt;
      }
      for (int k = 0; k < 3; ++k) {
        add[k] = st.acc_integral[k] * dt + 0.25 * CCa[k] * dt * dt;
        st.acc_doubleintegral[k] += add[k];
      }
      if (PREINT) {
        double CJ[9];
        mat3mul(C1, Jr, CJ);
        for (int k = 0; k < 9; ++k) st.dalpha_db_g[k] += CJ[k] * dt;
      } else {
        for (int k = 0; k < 9; ++k) st.dalpha_db_g[k] += dt * C1[k];
      }
      double cross1[9];
      mat3mul(Rdqi, st.cross, cross1);
      for (int k = 0; k < 9; ++k) cross1[k] += Jr[k] * dt;
      double ax[9], t1m[9], t2m[9], A1[9], A2[9], sumA[9];
      crossMx(ac, ax);
      mat3mul(C, ax, t1m); mat3mul(t1m, st.cross, A1);
      mat3mul(C1, ax, t2m); mat3mul(t2m, cross1, A2);
      for (int k = 0; k < 9; ++k) sumA[k] = A1[k] + A2[k];
      double dv1[9], F09[9];
      for (int k = 0; k < 9; ++k) {
        dv1[k] = st.dv_db_g[k] + 0.5 * dt * sumA[k];
        F09[k] = dt * st.dv_db_g[k] + 0.25 * dt * dt * sumA[k];
        st.dp_db_g[k] += F09[k];
      }
      for (int k = 0; k < 4; ++k) st.Delta_q[k] = q1[k];
      for (int k = 0; k < 9; ++k) { st.C_integral[k] = Ci1[k]; st.cross[k] = cross1[k]; st.dv_db_g[k] = dv1[k]; }
      for (int k = 0; k < 3; ++k) st.acc_integral[k] = ai1[k];
      // the record of the covariance step, over the precompute (read completely above)
      if (WANT_COV) {
        for (int k = 0; k < 3; ++k) { o[4 + k] = add[k]; o[7 + k] = 0.5 * CCa[k] * dt; }
        for (int k = 0; k < 9; ++k) { o[10 + k] = F09[k]; o[19 + k] = F012[k]; o[28 + k] = C1[k]; o[37 + k] = sumA[k]; o[46 + k] = CC[k]; }
      }
      o[0] = last ? 2.0 : 1.0;
      if (last) break;
    }
    cx.sync();
    for (int j = 0; j < kImuBatch && base + j < n; ++j) {
      const double* o = wk.S + j * kImuRec;
      if (o[0] == 0.0) continue;
      if (WANT_COV) {
        // P <- F P F^T + Q with F = I + N, N nonzero only in rows 0..8:
        //   N = {(0,3):-[add]x, (0,6): dt I, (0,9): F09, (0,12): F012, (3,9): -dt C1,
        //        (6,3): -[0.5 CCa dt]x, (6,9): 0.5 dt sumA, (6,12): -0.5 CC dt}
        // One lane per column: P(:,c) <- F P(:,c), then one lane per row: P(l,:) <- F P(l,:)^T + Q(l,:).  Each lane
        // reads its whole column (row) before it writes it back, so P is updated in place.  Each lane does
        // 2 x 66 multiply-adds per sample.
        const double dt = o[1], sigma_g_c = o[2], sigma_a_c = o[3];
        double X03[9], X63[9];
        crossMx(o + 4, X03);
        crossMx(o + 7, X63);
        const double *F09 = o + 10, *F012 = o + 19, *C1 = o + 28, *sumA = o + 37, *CC = o + 46;
        const double s2_dalpha = dt * sigma_g_c * sigma_g_c;
        const double s2_v = PREINT ? dt * sigma_a_c * sigma_a_c : dt * sigma_a_c * prm.sigma_a_c;
        const double s2_p = 0.5 * dt * dt * s2_v;
        const double s2_bg = dt * prm.sigma_gw_c * prm.sigma_gw_c;
        const double s2_ba = dt * prm.sigma_aw_c * prm.sigma_aw_c;
        for (int c = cx.lane(); c < 15; c += cx.lanes()) {
          double x[15], y[15];
#pragma unroll
          for (int k = 0; k < 15; ++k) x[k] = Pc[k * 15 + c];
          imu_apply_F(x, y, dt, X03, F09, F012, C1, X63, sumA, CC);
#pragma unroll
          for (int k = 0; k < 15; ++k) Pc[k * 15 + c] = y[k];
        }
        cx.sync();
        for (int l = cx.lane(); l < 15; l += cx.lanes()) {
          double x[15], y[15];
#pragma unroll
          for (int k = 0; k < 15; ++k) x[k] = Pc[l * 15 + k];
          imu_apply_F(x, y, dt, X03, F09, F012, C1, X63, sumA, CC);
          const int bq = l / 3;
          const double qd = (bq == 0) ? s2_p : (bq == 1) ? s2_dalpha : (bq == 2) ? s2_v : (bq == 3) ? s2_bg : s2_ba;
#pragma unroll
          for (int k = 0; k < 15; ++k) Pc[l * 15 + k] = y[k] + ((k == l) ? qd : 0.0);
        }
        cx.sync();
      }
      ++i;
      if (o[0] == 2.0) { finished = true; break; }
    }
    cx.sync();   // the records are rewritten by the next batch
  }
  return i;
}

// In-place lower Cholesky of a 15x15 SPD matrix in M (cooperative).  Returns false on failure.
template <class Ctx>
OKB_HD bool chol15(const Ctx& cx, double* M) {
  bool ok = true;
  for (int k = 0; k < 15; ++k) {
    const double x = M[k * 15 + k];
    if (!(x > 0.0)) { ok = false; break; }   // uniform across lanes (all read the same value)
    const double sx = sqrt(x);
    cx.sync();
    for (int i = k + cx.lane(); i < 15; i += cx.lanes()) M[i * 15 + k] = (i == k) ? sx : M[i * 15 + k] / sx;
    cx.sync();
    // trailing update, lower part
    const int nt = 14 - k;
    for (int e = cx.lane(); e < nt * nt; e += cx.lanes()) {
      const int i = k + 1 + e / nt, j = k + 1 + e % nt;
      if (j <= i) M[i * 15 + j] -= M[i * 15 + k] * M[j * 15 + k];
    }
    cx.sync();
  }
  return ok;
}

// redoPreintegration: integrates at `sb`, then information = sym(P^-1), sqrt_info = LLT(information)^T.
// The inverse is taken through the Cholesky factor of the (symmetrised) covariance.
template <class Ctx>
OKB_HD int imu_preintegrate(const Ctx& cx, const okb_imu_sample* s, int n, const okb_imu_params& prm, int64_t t0,
                            int64_t t1, const double* sb, ImuCache* cache, ImuWork wk) {
  const int steps = imu_integrate<true, true>(cx, s, n, prm, t0, t1, sb, wk);
  if (steps < 0) return steps;
  const ImuInt& st = wk.state();
  // symmetrise P into F (workspace)
  for (int e = cx.lane(); e < 225; e += cx.lanes()) {
    const int rr = e / 15, cc = e % 15;
    wk.F[e] = 0.5 * wk.P[rr * 15 + cc] + 0.5 * wk.P[cc * 15 + rr];
  }
  cx.sync();
  chol15(cx, wk.F);                       // F = L (lower), P = L L^T
  // T = L^-1 (lower), column by column (each lane owns columns)
  for (int c = cx.lane(); c < 15; c += cx.lanes()) {
    for (int r = 0; r < 15; ++r) {
      double v = 0.0;
      if (r >= c) {
        double sacc = (r == c) ? 1.0 : 0.0;
        for (int k = c; k < r; ++k) sacc -= wk.F[r * 15 + k] * wk.T[k * 15 + c];
        v = sacc / wk.F[r * 15 + r];
      }
      wk.T[r * 15 + c] = v;
    }
  }
  cx.sync();
  // information = L^-T L^-1 (symmetric by construction) -> P
  for (int e = cx.lane(); e < 225; e += cx.lanes()) {
    const int rr = e / 15, cc = e % 15;
    double sacc = 0;
    const int k0 = rr > cc ? rr : cc;
    for (int k = k0; k < 15; ++k) sacc += wk.T[k * 15 + rr] * wk.T[k * 15 + cc];
    wk.P[e] = sacc;
  }
  cx.sync();
  chol15(cx, wk.P);                       // lower factor of the information
  // store sqrt_info = L^T (upper)
  for (int e = cx.lane(); e < 225; e += cx.lanes()) {
    const int rr = e / 15, cc = e % 15;
    cache->sqrt_info[e] = (cc >= rr) ? wk.P[cc * 15 + rr] : 0.0;
  }
  if (cx.lane() == 0) {
    for (int k = 0; k < 4; ++k) cache->Delta_q[k] = st.Delta_q[k];
    for (int k = 0; k < 9; ++k) {
      cache->C_integral[k] = st.C_integral[k]; cache->C_doubleintegral[k] = st.C_doubleintegral[k];
      cache->dalpha_db_g[k] = st.dalpha_db_g[k]; cache->dv_db_g[k] = st.dv_db_g[k]; cache->dp_db_g[k] = st.dp_db_g[k];
      cache->sb_ref[k] = sb[k];
    }
    for (int k = 0; k < 3; ++k) { cache->acc_integral[k] = st.acc_integral[k]; cache->acc_doubleintegral[k] = st.acc_doubleintegral[k]; }
    cache->valid = 1;
    cache->redo_count += 1;
  }
  cx.sync();
  return steps;
}

// Evaluates one ImuError at (pose0, sb0, pose1, sb1).  Mutates the cache like the reference (redo
// when never preintegrated or |db_g|*Dt > 1e-4, then db := 0).
// Outputs (cooperative, in the caller's buffers; any may be null):
//   e15   : unweighted error (15)                 r15: sqrt_info * e
//   SF    : [15][30] = sqrt_info * [F0 | F1]  (the four minimal Jacobians side by side:
//           cols 0-5 pose0, 6-14 sb0, 15-20 pose1, 21-29 sb1)
// F01 needs 450 doubles (F0|F1 unweighted, [15][30]); it and SF may overlay wk (see imu_scratch).
template <class Ctx>
OKB_HD void imu_evaluate(const Ctx& cx, const okb_imu_sample* s, int n, const okb_imu_params& prm, int64_t t0, int64_t t1,
                         const double* pose0, const double* sb0, const double* pose1, const double* sb1, ImuCache* cache,
                         ImuWork wk, double* F01, double* e15, double* r15, double* SF) {
  const double Delta_t = ns_to_sec(t1 - t0);
  double db[6];
  bool redo = (cache->valid == 0);
  for (int k = 0; k < 6; ++k) db[k] = sb0[3 + k] - cache->sb_ref[3 + k];
  if (!redo) redo = sqrt(db[0] * db[0] + db[1] * db[1] + db[2] * db[2]) * Delta_t > 0.0001;
  cx.sync();
  if (redo) {
    imu_preintegrate(cx, s, n, prm, t0, t1, sb0, cache, wk);
    for (int k = 0; k < 6; ++k) db[k] = 0.0;
  }
  // small algebra, replicated per lane
  double q0[4] = {pose0[3], pose0[4], pose0[5], pose0[6]}, q1[4] = {pose1[3], pose1[4], pose1[5], pose1[6]};
  qnormalize(q0); qnormalize(q1);
  double C_WS0[9];
  q2R(q0, C_WS0);
  const double C_S0W[9] = {C_WS0[0], C_WS0[3], C_WS0[6], C_WS0[1], C_WS0[4], C_WS0[7], C_WS0[2], C_WS0[5], C_WS0[8]};
  const double g = prm.g;
  double dp[3], dv[3];
  for (int k = 0; k < 3; ++k) {
    const double gk = (k == 2) ? g : 0.0;
    dp[k] = pose0[k] - pose1[k] + sb0[k] * Delta_t - 0.5 * gk * Delta_t * Delta_t;
    dv[k] = sb0[k] - sb1[k] - gk * Delta_t;
  }
  double mdb[3], dqb[4], Dq[4];
  mat3vec(cache->dalpha_db_g, db, mdb);
  mdb[0] = -mdb[0]; mdb[1] = -mdb[1]; mdb[2] = -mdb[2];
  deltaQ(mdb, dqb);
  qmul(dqb, cache->Delta_q, Dq);
  double q1i[4], q1i_q0[4], Dq_q1i[4], qe[4];
  qinv(q1, q1i);
  qmul(q1i, q0, q1i_q0);
  qmul(Dq, q1i, Dq_q1i);
  qmul(Dq, q1i_q0, qe);
  // 3x3 blocks
  double B03[9], B63[9], X[9];
  crossMx(dp, X); mat3mul(C_S0W, X, B03);
  crossMx(dv, X); mat3mul(C_S0W, X, B63);
  // F0(3,3) = (plus(Dq*q1^-1) * oplus(q0))_3x3 ; plus(a)oplus(b) p = a*p*b
  // F1(3,3) = -(plus(Dq) * oplus(q0) * plus(q1^-1))_3x3 : p -> Dq*(q1^-1 * p)*q0
  // F0(3,9) = -(oplus(q1^-1 q0) * oplus(Dq))_3x3 * dalpha_db_g : p -> (p*Dq)*(q1^-1 q0)
  double B33[9], B133[9], B39[9], T39[9];
  for (int c = 0; c < 3; ++c) {
    double e[4] = {0, 0, 0, 0}, t[4], u[4];
    e[c] = 1.0;
    qmul(Dq_q1i, e, t); qmul(t, q0, u);
    B33[0 * 3 + c] = u[0]; B33[1 * 3 + c] = u[1]; B33[2 * 3 + c] = u[2];
    qmul(q1i, e, t); qmul(Dq, t, u); qmul(u, q0, t);
    B133[0 * 3 + c] = -t[0]; B133[1 * 3 + c] = -t[1]; B133[2 * 3 + c] = -t[2];
    qmul(e, Dq, t); qmul(t, q1i_q0, u);
    T39[0 * 3 + c] = u[0]; T39[1 * 3 + c] = u[1]; T39[2 * 3 + c] = u[2];
  }
  mat3mul(T39, cache->dalpha_db_g, B39);
  for (int k = 0; k < 9; ++k) B39[k] = -B39[k];
  // assemble [F0 | F1] (15 x 30) cooperatively: the lanes write the identity, the zeros and the blocks read from the
  // cache; lane 0 writes the blocks computed above, with constant indices so that they stay in registers
  for (int e = cx.lane(); e < 450; e += cx.lanes()) {
    const int rr = e / 30, c30 = e % 30;
    const int which = c30 / 15, cc = c30 % 15;
    const int br = rr / 3, bc = cc / 3, a = rr % 3, b = cc % 3;
    double v;
    bool lane0 = false;
    if (which == 0) {
      v = (rr == cc) ? 1.0 : 0.0;
      if (br == 0) {
        if (bc <= 2) lane0 = true;
        else if (bc == 3) v = cache->dp_db_g[a * 3 + b];
        else v = -cache->C_doubleintegral[a * 3 + b];
      } else if (br == 1) {
        lane0 = (bc == 1 || bc == 3);
      } else if (br == 2) {
        if (bc == 1 || bc == 2) lane0 = true;
        else if (bc == 3) v = cache->dv_db_g[a * 3 + b];
        else if (bc == 4) v = -cache->C_integral[a * 3 + b];
        else v = 0.0;
      }
    } else {
      v = (rr == cc) ? -1.0 : 0.0;
      lane0 = (br == bc && br < 3);
    }
    if (!lane0) F01[e] = v;
  }
  if (cx.lane() == 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
      for (int b = 0; b < 3; ++b) {
        const int k = a * 3 + b;
        F01[a * 30 + b] = C_S0W[k];                      // F0 (0,0)
        F01[a * 30 + 3 + b] = B03[k];                    // F0 (0,1)
        F01[a * 30 + 6 + b] = C_S0W[k] * Delta_t;        // F0 (0,2)
        F01[(3 + a) * 30 + 3 + b] = B33[k];              // F0 (1,1)
        F01[(3 + a) * 30 + 9 + b] = B39[k];              // F0 (1,3)
        F01[(6 + a) * 30 + 3 + b] = B63[k];              // F0 (2,1)
        F01[(6 + a) * 30 + 6 + b] = C_S0W[k];            // F0 (2,2)
        F01[a * 30 + 15 + b] = -C_S0W[k];                // F1 (0,0)
        F01[(3 + a) * 30 + 18 + b] = B133[k];            // F1 (1,1)
        F01[(6 + a) * 30 + 21 + b] = -C_S0W[k];          // F1 (2,2)
      }
    }
  }
  cx.sync();
  // error vector (replicated), uses F0 rows 0..2 / 6..8, cols 9..14
  double err[15];
  {
    double t[3];
    mat3vec(C_S0W, dp, t);
    for (int a = 0; a < 3; ++a) {
      double fb = 0;
      for (int b = 0; b < 6; ++b) fb += F01[(0 + a) * 30 + 9 + b] * db[b];
      err[a] = t[a] + cache->acc_doubleintegral[a] + fb;
    }
    err[3] = 2 * qe[0]; err[4] = 2 * qe[1]; err[5] = 2 * qe[2];
    mat3vec(C_S0W, dv, t);
    for (int a = 0; a < 3; ++a) {
      double fb = 0;
      for (int b = 0; b < 6; ++b) fb += F01[(6 + a) * 30 + 9 + b] * db[b];
      err[6 + a] = t[a] + cache->acc_integral[a] + fb;
    }
    for (int a = 0; a < 6; ++a) err[9 + a] = sb0[3 + a] - sb1[3 + a];
  }
  if (e15) for (int e = cx.lane(); e < 15; e += cx.lanes()) e15[e] = err[e];
  if (r15) {
    for (int e = cx.lane(); e < 15; e += cx.lanes()) {
      double sacc = 0;
#pragma unroll
      for (int k = 0; k < 15; ++k)
        if (k >= e) sacc += cache->sqrt_info[e * 15 + k] * err[k];   // constant index: err stays in registers
      r15[e] = sacc;
    }
  }
  if (SF) {
    for (int e = cx.lane(); e < 450; e += cx.lanes()) {
      const int rr = e / 30, cc = e % 30;
      double sacc = 0;
      for (int k = rr; k < 15; ++k) sacc += cache->sqrt_info[rr * 15 + k] * F01[k * 30 + cc];
      SF[e] = sacc;
    }
  }
  cx.sync();
}

// Static ImuError::propagation: pose/sb in-out; optional covariance (15x15) and Jacobian (15x15).
template <class Ctx>
OKB_HD int imu_propagate(const Ctx& cx, const okb_imu_sample* s, int n, const okb_imu_params& prm, int64_t t0, int64_t t1,
                         double* pose, double* sb, double* covariance, double* jacobian, ImuWork wk) {
  int steps;
  if (covariance) steps = imu_integrate<false, true>(cx, s, n, prm, t0, t1, sb, wk);
  else steps = imu_integrate<false, false>(cx, s, n, prm, t0, t1, sb, wk);
  if (steps < 0) return steps;
  const ImuInt& st = wk.state();
  double q0[4] = {pose[3], pose[4], pose[5], pose[6]};
  qnormalize(q0);
  double C0[9];
  q2R(q0, C0);
  const double r0[3] = {pose[0], pose[1], pose[2]};
  const double Dt = st.Delta_t, g = prm.g;
  double Cadd[3], Cai[3], qn[4];
  mat3vec(C0, st.acc_doubleintegral, Cadd);
  mat3vec(C0, st.acc_integral, Cai);
  qmul(q0, st.Delta_q, qn);
  qnormalize(qn);
  cx.sync();
  if (jacobian) {
    double X03[9], X63[9], M09[9], M012[9], M39[9], M69[9], M612[9];
    crossMx(Cadd, X03); crossMx(Cai, X63);
    mat3mul(C0, st.dp_db_g, M09); mat3mul(C0, st.C_doubleintegral, M012); mat3mul(C0, st.dalpha_db_g, M39);
    mat3mul(C0, st.dv_db_g, M69); mat3mul(C0, st.C_integral, M612);
    for (int e = cx.lane(); e < 225; e += cx.lanes()) {
      const int rr = e / 15, cc = e % 15, br = rr / 3, bc = cc / 3, a = rr % 3, b = cc % 3;
      double v = (rr == cc) ? 1.0 : 0.0;
      if (br == 0) {
        if (bc == 1) v = -X03[a * 3 + b];
        else if (bc == 2) v = (a == b) ? Dt : 0.0;
        else if (bc == 3) v = M09[a * 3 + b];
        else if (bc == 4) v = -M012[a * 3 + b];
      } else if (br == 1) {
        if (bc == 3) v = -M39[a * 3 + b];
      } else if (br == 2) {
        if (bc == 1) v = -X63[a * 3 + b];
        else if (bc == 3) v = M69[a * 3 + b];
        else if (bc == 4) v = -M612[a * 3 + b];
      }
      jacobian[e] = v;
    }
  }
  if (covariance) {
    // P = T P_delta T^T, T = blockdiag(C0, C0, C0, I, I)
    for (int e = cx.lane(); e < 225; e += cx.lanes()) {
      const int rr = e / 15, cc = e % 15, br = rr / 3, a = rr % 3;
      double v;
      if (br < 3) { v = 0; for (int k = 0; k < 3; ++k) v += C0[a * 3 + k] * wk.P[(br * 3 + k) * 15 + cc]; }
      else v = wk.P[e];
      wk.T[e] = v;
    }
    cx.sync();
    for (int e = cx.lane(); e < 225; e += cx.lanes()) {
      const int rr = e / 15, cc = e % 15, bc = cc / 3, b = cc % 3;
      double v;
      if (bc < 3) { v = 0; for (int k = 0; k < 3; ++k) v += wk.T[rr * 15 + bc * 3 + k] * C0[b * 3 + k]; }
      else v = wk.T[e];
      covariance[e] = v;
    }
  }
  cx.sync();
  if (cx.lane() == 0) {
    for (int k = 0; k < 3; ++k) {
      const double gk = (k == 2) ? g : 0.0;
      pose[k] = r0[k] + sb[k] * Dt + Cadd[k] - 0.5 * gk * Dt * Dt;
    }
    for (int k = 0; k < 4; ++k) pose[3 + k] = qn[k];
    for (int k = 0; k < 3; ++k) sb[k] += Cai[k] - ((k == 2) ? g : 0.0) * Dt;
  }
  cx.sync();
  return steps;
}

}  // namespace okb
