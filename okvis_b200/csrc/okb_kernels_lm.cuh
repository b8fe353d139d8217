// Landmark-side kernels of the solver round (sm_90a):
//   k_landmarks ("A1"): one CTA per 128 landmarks.  Candidate landmark, reprojection residuals + Jacobian factors of
//       the cameras of every frame its tiles see, Cauchy weighting, per-frame M_f = sum rho' A^T A (stored tile-major,
//       see lm_M_index) and m_f = sum rho' A^T r, the pose-block contributions H_pp,f = G^T M_f G and g_p,f = G^T m_f
//       reduced per (CTA, frame), then H_ll = sum_f M_f, g_l = -sum_f m_f and (H_ll + mu E)^-1 by 3x3 Cholesky.
//   k_schur ("A2"): one CTA per (landmark chunk, window), tiles of 32 landmarks staged by TMA bulk copies:
//       Y_f = W_f L^-T into a shared-memory tile, then the Schur complement as a block-sparse SYRK
//       S += Y^T Y on the FP64 tensor cores, the 6K pose columns packed into 8-column blocks, one 8x8 block per block
//       pair (details at the kernel).
//   k_quality: post-solve landmark quality (Estimator.cpp:880-894), one thread per landmark.
#pragma once
#include <cooperative_groups.h>

#include "okb_estimator.cuh"

namespace okb {

constexpr int L1_THREADS = 128;          // landmarks per k_landmarks CTA: one partH record per (CTA, frame)
constexpr int A2_TILE = 32;              // landmarks per Y tile
constexpr int kPartH = 32;               // doubles per (cx, frame) record: 27 H_pp/g_p + cost + stepnorm2 + pad

struct SlotCtx {
  SlotXf xf;
  CamIntr cam;
  int frame;
  int valid;
};
static_assert(sizeof(SlotCtx) % 8 == 0, "SlotCtx is copied as doubles");

// (frame, camera) contexts at the candidate poses: computed once per round by the kernel that writes the
// candidate (k_reset / k_solve) instead of by every k_landmarks CTA.
__device__ inline void build_slot_ctx(const WinDev& W, int tid, int nthr) {
  for (int s = tid; s < W.NS; s += nthr) {
    const SlotInfo si = W.slots[s];
    SlotCtx sc;
    sc.valid = si.valid; sc.frame = s / W.CP;
    if (si.valid) { make_slot_xf(W.pose_c + 7 * si.pose_idx, W.ext + 7 * si.ext_idx, sc.xf); cam_load(W.cams[si.cam_idx], sc.cam); }
    else { for (int k = 0; k < 9; ++k) sc.xf.R[k] = 0; for (int k = 0; k < 3; ++k) sc.xf.t[k] = 0; cam_load(W.cams[0], sc.cam); }
    W.slot_ctx[s] = sc;
  }
}

// ------------------------------------------------------------------------------------------------
// A1: CS CTAs (one cluster) per (128 sorted landmarks, window), FG groups of 128 threads each; thread (g, t) owns
// landmark t.  Walk lane p = crank * FG + g (crank = rank in the cluster), P = CS * FG lanes.
//   1. per landmark (group 0): candidate X = lm + a g/E + b GN; CTA 0 also stores lm_c and the step-norm partial;
//   2. frame walk in rounds: in round k lane p takes the walked frame of rank k P + p (the frames seen by the 4
//      tiles, ascending), so P frames are in flight.  Per (landmark, frame): <= CP projections, M_f / m_f, the lm_M
//      store, the 27 pose-block values and the cost.  Each warp reduces its 32 landmarks' 28 values with a
//      reduce-scatter butterfly (lane e ends with value e) and stores them as the warp's partial; after the round's
//      barrier warp 0 of the group adds the four partials in warp order into the (cx, f) record.  M_f / m_f are staged
//      in shared memory; group 0 of CTA 0 adds them to H_ll / g_l in frame order after the same barrier (the other
//      CTA's through distributed shared memory).  Partials and staging are double-buffered by round;
//   3. group 0 of CTA 0 runs the landmark-block epilogue: metric E, R = H_ll + mu E, 3x3 Cholesky, R^-1, L^-1 | z.
// H_ll and g_l are summed frame by frame in ascending order whatever P is, and a record's sum order depends only on
// the landmark's position in the tile, so a window gives the same bits alone or in a batch of any size.  The running
// sums live in shared memory.
// Every (cx, f < K) record is written (zeros for frames no tile of the CTA sees); slot 28 of frame 0's record
// holds the CTA's step norm.
// MODEL is the distortion model of every camera in the launch (OKB_DIST_*), or kDistAny to switch per camera.
// ------------------------------------------------------------------------------------------------
constexpr int kLmRows = 28;     // values reduced per (landmark, frame): 27 H_pp / g_p + cost

// dynamic shared memory of k_landmarks<FG>: the step-norm row, X [4][128], the running H_ll | g_l [9][128], staged
// M_f | m_f [2 rounds][FG][9][128], warp partials [2 rounds][FG][4 warps][32]
__host__ __device__ inline size_t smemL_bytes(int groups) {
  return ((size_t)L1_THREADS + 4 * L1_THREADS + 9 * L1_THREADS + (size_t)2 * groups * 9 * L1_THREADS + (size_t)2 * groups * L1_THREADS) *
         sizeof(double);
}

// Reduce-scatter of 32 values over a warp: on return lane e holds the sum over the warp's lanes of value e.  A fixed
// butterfly (xor 16, 8, 4, 2, 1), 31 shuffles, so the summation order is the same on every launch.
template <int O, int N>
__device__ __forceinline__ void reduce_scatter_step(double (&v)[N]) {      // v[0, 2 O) -> v[0, O): this lane's half
  const bool hi = (threadIdx.x & O) != 0;
#pragma unroll
  for (int i = 0; i < O; ++i) {
    const double keep = hi ? v[i + O] : v[i], send = hi ? v[i] : v[i + O];
    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, O);
  }
}
__device__ __forceinline__ double warp_reduce_scatter32(double (&v)[32]) {
  reduce_scatter_step<16>(v);
  reduce_scatter_step<8>(v);
  reduce_scatter_step<4>(v);
  reduce_scatter_step<2>(v);
  reduce_scatter_step<1>(v);
  return v[0];
}

// <FG = 2, CS = 1>: 256 threads, three CTAs (24 warps) per SM at <= 80 registers.  <4, 2> (launches whose tiles
// would fill less than half the SMs): clusters of two 512-thread CTAs, one CTA per SM, 8 frames in flight per tile.
template <int FG, int CS, int MODEL>
__global__ void __launch_bounds__(FG * L1_THREADS, FG == 2 ? 3 : 1) k_landmarks(const WinDev* __restrict__ wins, const int32_t* __restrict__ win_slots) {
  const WinDev& W = wins[win_slots[blockIdx.y]];
  SolverState* st = W.st;
  if (st->done) return;                // (uniform over a cluster: same window, same landmark tile)
  const int cx = blockIdx.x / CS, crank = blockIdx.x % CS;
  const int L = W.L, K = W.K, CP = W.CP;
  if (cx * L1_THREADS >= L) return;
  const int tid = threadIdx.x, g = tid / L1_THREADS, t = tid % L1_THREADS;
  constexpr int P = CS * FG;
  const int lane = crank * FG + g;
  const int l = cx * L1_THREADS + t;
  const int mode = st->mode, cur = st->cur;
  const bool cauchy = W.use_cauchy != 0;
  double* rec = W.partH + (size_t)cx * K * kPartH;        // this CTA's records [K][kPartH]

  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* sdn = reinterpret_cast<double*>(smem_raw);                     // step norm per landmark
  double* sX = sdn + L1_THREADS;                                         // [4][128] candidate landmarks
  double* sHg = sX + 4 * L1_THREADS;                                     // [9][128] running H_ll (6) | g_l (3)
  double* sstage = sHg + 9 * L1_THREADS;                                 // [2][FG][9][128] M_f (6) | m_f (3) per lane
  double* spart = sstage + 2 * FG * 9 * L1_THREADS;                      // [2][FG][4][32] warp partials of the 28 values
  const bool owner = crank == 0 && g == 0;                               // adds the staged blocks, runs the epilogue
  if (owner) {
#pragma unroll
    for (int k = 0; k < 9; ++k) sHg[k * L1_THREADS + t] = 0.0;
  }

  // frames seen by the CTA's 4 tiles (landmarks are sorted by observing-frame range)
  uint32_t fmask = 0;
#pragma unroll
  for (int q = 0; q < L1_THREADS / 32; ++q) {
    const int tile = cx * (L1_THREADS / 32) + q;
    if (tile * 32 < L) {
      const uint32_t tr = W.tile_range[tile];
      const uint32_t fa = tr & 0xffu, fb = tr >> 8;
      if (fa <= fb) fmask |= ((2u << fb) - 1u) & ~((1u << fa) - 1u);
    }
  }
  const uint32_t vmask = (l < L) ? W.lm_vis[l] : 0u;

  // ---- 1. per-landmark work (group 0)
  if (g == 0) {
    double dn = 0.0;
    if (l < L) {
      const double4 x4 = *reinterpret_cast<const double4*>(W.lm + 4 * (size_t)l);
      double X[4] = {x4.x, x4.y, x4.z, x4.w};
      if (mode == MODE_STEP) {
        const double a = st->a, b = st->b;
        const double* gp = W.lm_g[cur] + 3 * (size_t)l;
        const double* Ep = W.lm_E[cur] + 3 * (size_t)l;
        const double* gn = W.lm_gn + 3 * (size_t)l;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const double dlt = a * gp[c] / Ep[c] + b * gn[c];
          X[c] += dlt;
          dn += dlt * dlt;
        }
      }
      if (crank == 0) *reinterpret_cast<double4*>(W.lm_c + 4 * (size_t)l) = make_double4(X[0], X[1], X[2], X[3]);
#pragma unroll
      for (int c = 0; c < 4; ++c) sX[c * L1_THREADS + t] = X[c];
    }
    sdn[t] = dn;
  }
  // records of frames no tile sees, and slot 28 (step norm) of frames other than 0
  for (int i = tid; crank == 0 && i < K * 29; i += FG * L1_THREADS) {
    const int f = i / 29, e = i % 29;
    if (e == 28 ? f != 0 : !((fmask >> f) & 1u)) rec[(size_t)f * kPartH + e] = 0.0;
  }
  __syncthreads();
  if (crank == 0 && tid < 4) {      // step norm into slot 28 of frame 0's record: 4 lanes x 32 columns, then two shuffle steps
    const int q = tid;
    double s = 0.0;
#pragma unroll 8
    for (int i = 0; i < 32; ++i) s += sdn[q * 32 + ((i + 4 * q) & 31)];
    s += __shfl_xor_sync(0xfu, s, 1);
    s += __shfl_xor_sync(0xfu, s, 2);
    if (q == 0) rec[28] = s;
  }

  // ---- 2. frame walk in rounds of P frames
  const int nf = __popc(fmask);
  uint32_t rest = fmask;
  for (int i = 0; i < lane && rest; ++i) rest &= rest - 1;
  for (int r0 = 0; r0 < nf; r0 += P) {
    const int buf = (r0 / P) & 1;
    double* stg = sstage + (size_t)((buf * FG + g) * 9) * L1_THREADS + t;     // element k at stg[k * L1_THREADS]
    double* part = spart + (size_t)(buf * FG + g) * L1_THREADS;              // [4 warps][32]
    const bool walks = r0 + lane < nf;     // (uniform over the group)
    const int f = __ffs(rest) - 1;
    if (walks) {
#pragma unroll
      for (int i = 0; i < P; ++i) rest &= rest - 1;
      double v[32];
      if ((vmask >> f) & 1u) {
        const size_t gi0 = (size_t)(f * CP) * L + l;
        const SlotCtx* sc = W.slot_ctx + f * CP;
        // M_f | m_f are accumulated in this lane's staging slot, not in registers: with one distortion model the
        // observation loop then fits in the 80 registers of three CTAs per SM without spilling
#pragma unroll
        for (int k = 0; k < 9; ++k) stg[k * L1_THREADS] = 0.0;
        double cost = 0, lprod = 1.0;
        for (int c = 0; c < CP; ++c) {
          const double wobs = W.obs_w[gi0 + (size_t)c * L];
          if (wobs > 0.0 && sc[c].valid) {
            const double2 z = W.obs_z[gi0 + (size_t)c * L];
            const double X[4] = {sX[t], sX[L1_THREADS + t], sX[2 * L1_THREADS + t], sX[3 * L1_THREADS + t]};
            double r[2], A[6];
            reproj_slot<true, MODEL>(sc[c].xf, sc[c].cam, X, z.x, z.y, wobs, r, A);
            const double sq = r[0] * r[0] + r[1] * r[1];
            double rho1 = 1.0;
            if (cauchy) {          // 0.5 log(1 + s) per block: the logs of a frame's cameras are taken as one log of the product
              rho1 = 1.0 / (1.0 + sq);
              lprod *= 1.0 + sq;
              if (lprod > 1e250) { cost += 0.5 * log(lprod); lprod = 1.0; }
            } else cost += 0.5 * sq;
            stg[0] += rho1 * (A[0] * A[0] + A[3] * A[3]);
            stg[L1_THREADS] += rho1 * (A[0] * A[1] + A[3] * A[4]);
            stg[2 * L1_THREADS] += rho1 * (A[0] * A[2] + A[3] * A[5]);
            stg[3 * L1_THREADS] += rho1 * (A[1] * A[1] + A[4] * A[4]);
            stg[4 * L1_THREADS] += rho1 * (A[1] * A[2] + A[4] * A[5]);
            stg[5 * L1_THREADS] += rho1 * (A[2] * A[2] + A[5] * A[5]);
            stg[6 * L1_THREADS] += rho1 * (A[0] * r[0] + A[3] * r[1]);
            stg[7 * L1_THREADS] += rho1 * (A[1] * r[0] + A[4] * r[1]);
            stg[8 * L1_THREADS] += rho1 * (A[2] * r[0] + A[5] * r[1]);
          }
        }
        if (cauchy) cost += 0.5 * log(lprod);
        const double M0 = stg[0], M1 = stg[L1_THREADS], M2 = stg[2 * L1_THREADS], M3 = stg[3 * L1_THREADS], M4 = stg[4 * L1_THREADS];
        const double M5 = stg[5 * L1_THREADS], m0 = stg[6 * L1_THREADS], m1 = stg[7 * L1_THREADS], m2 = stg[8 * L1_THREADS];
        double* Mo = W.lm_M + lm_M_index(l, f, K);          // tile-major: a warp stores 256-byte rows
        Mo[0] = M0; Mo[32] = M1; Mo[64] = M2; Mo[96] = M3; Mo[128] = M4; Mo[160] = M5;
        // pose-block contributions: G = [w I, -[p]x], p = X - t_WS w
        const double* tw = W.pose_c + 7 * f;
        const double w = sX[3 * L1_THREADS + t];
        const double p0 = sX[t] - tw[0] * w, p1 = sX[L1_THREADS + t] - tw[1] * w, p2 = sX[2 * L1_THREADS + t] - tw[2] * w;
        const double Q00 = M1 * p2 - M2 * p1, Q01 = -M0 * p2 + M2 * p0, Q02 = M0 * p1 - M1 * p0;
        const double Q10 = M3 * p2 - M4 * p1, Q11 = -M1 * p2 + M4 * p0, Q12 = M1 * p1 - M3 * p0;
        const double Q20 = M4 * p2 - M5 * p1, Q21 = -M2 * p2 + M5 * p0, Q22 = M2 * p1 - M4 * p0;
        const double w2 = w * w;
        v[0] = w2 * M0; v[1] = w2 * M1; v[2] = w2 * M2; v[3] = w2 * M3; v[4] = w2 * M4; v[5] = w2 * M5;
        v[6] = -w * Q00; v[7] = -w * Q01; v[8] = -w * Q02;
        v[9] = -w * Q10; v[10] = -w * Q11; v[11] = -w * Q12;
        v[12] = -w * Q20; v[13] = -w * Q21; v[14] = -w * Q22;
        v[15] = p2 * Q10 - p1 * Q20; v[16] = p2 * Q11 - p1 * Q21; v[17] = p2 * Q12 - p1 * Q22;
        v[18] = -p2 * Q01 + p0 * Q21; v[19] = -p2 * Q02 + p0 * Q22;
        v[20] = p1 * Q02 - p0 * Q12;
        v[21] = w * m0; v[22] = w * m1; v[23] = w * m2;
        v[24] = p1 * m2 - p2 * m1; v[25] = p2 * m0 - p0 * m2; v[26] = p0 * m1 - p1 * m0;
        v[27] = cost;
      } else {
#pragma unroll
        for (int e = 0; e < kLmRows; ++e) v[e] = 0.0;
#pragma unroll
        for (int k = 0; k < 9; ++k) stg[k * L1_THREADS] = 0.0;
      }
#pragma unroll
      for (int e = kLmRows; e < 32; ++e) v[e] = 0.0;
      part[t] = warp_reduce_scatter32(v);      // part[32 w + e]: warp w's sum of value e
    }
    // the round's blocks and partials are staged (buffer buf is rewritten two rounds later, after the next round's
    // barrier, which their readers reach only when these reads are done)
    if constexpr (CS > 1) cooperative_groups::this_cluster().sync();
    else __syncthreads();
    if (walks && t < kLmRows) {      // warp 0 of the group: the four warps' partials in warp order
      rec[(size_t)f * kPartH + t] = ((part[t] + part[32 + t]) + part[64 + t]) + part[96 + t];
    }
    if (owner) {
      double v[9];
#pragma unroll
      for (int k = 0; k < 9; ++k) v[k] = sHg[k * L1_THREADS + t];
      for (int q = 0; q < P && r0 + q < nf; ++q) {
        const double* src = sstage + (size_t)((buf * FG + q % FG) * 9) * L1_THREADS + t;
        if constexpr (CS > 1) src = cooperative_groups::this_cluster().map_shared_rank(src, q / FG);
#pragma unroll
        for (int k = 0; k < 6; ++k) v[k] += src[k * L1_THREADS];
#pragma unroll
        for (int k = 6; k < 9; ++k) v[k] -= src[k * L1_THREADS];
      }
#pragma unroll
      for (int k = 0; k < 9; ++k) sHg[k * L1_THREADS + t] = v[k];
    }
  }
  if constexpr (CS > 1) cooperative_groups::this_cluster().sync();     // the peers' staging stays until it is read

  // ---- 3. landmark-block epilogue (group 0 of CTA 0)
  if (!owner || l >= L) return;
  double v[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) v[k] = sHg[k * L1_THREADS + t];
  const double H0 = v[0], H1 = v[1], H2 = v[2], H3 = v[3], H4 = v[4], H5 = v[5], gl0 = v[6], gl1 = v[7], gl2 = v[8];
  const double mu = (mode == MODE_STEP) ? fmax(kMinMu, 2.0 * st->mu / kMuIncrease) : st->mu;
  const double gl[3] = {gl0, gl1, gl2};
  double sc3[3], E[3];
  const double hd[3] = {H0, H3, H5};
  if (mode == MODE_INIT) {
#pragma unroll
    for (int c = 0; c < 3; ++c) { sc3[c] = 1.0 / (1.0 + sqrt(hd[c])); W.lm_scale[3 * (size_t)l + c] = sc3[c]; }
  } else {
#pragma unroll
    for (int c = 0; c < 3; ++c) sc3[c] = W.lm_scale[3 * (size_t)l + c];
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double s2 = sc3[c] * sc3[c];
    E[c] = fmin(fmax(s2 * hd[c], kMinDiag), kMaxDiag) / s2;
  }
  const double R[6] = {H0 + mu * E[0], H1, H2, H3 + mu * E[1], H4, H5 + mu * E[2]};
  double Lc[6], Li[6];
  if (chol3(R, Lc)) linv3(Lc, Li);
  else {
#pragma unroll
    for (int i = 0; i < 6; ++i) Li[i] = 0.0;
    st->numeric_fail = 1;
  }
  double* Ro = W.lm_Rinv + 6 * (size_t)l;
  Ro[0] = Li[0] * Li[0] + Li[1] * Li[1] + Li[3] * Li[3];
  Ro[1] = Li[1] * Li[2] + Li[3] * Li[4];
  Ro[2] = Li[3] * Li[5];
  Ro[3] = Li[2] * Li[2] + Li[4] * Li[4];
  Ro[4] = Li[4] * Li[5];
  Ro[5] = Li[5] * Li[5];
  double* gs = W.lm_g[cur ^ 1] + 3 * (size_t)l;
  double* Es = W.lm_E[cur ^ 1] + 3 * (size_t)l;
#pragma unroll
  for (int c = 0; c < 3; ++c) { gs[c] = gl[c]; Es[c] = E[c]; }
  double* Lo = W.lm_Li + 9 * (size_t)l;     // L^-1 (6) | z (3)
#pragma unroll
  for (int i = 0; i < 6; ++i) Lo[i] = Li[i];
  Lo[6] = Li[0] * gl[0];
  Lo[7] = Li[1] * gl[0] + Li[2] * gl[1];
  Lo[8] = Li[3] * gl[0] + Li[4] * gl[1] + Li[5] * gl[2];
}

// ------------------------------------------------------------------------------------------------
// A2: Schur complement of the landmark blocks,  S = sum_l Y_l^T Y_l  with  Y_l = W_l L_l^-T, and the reduced
// right-hand side  sum_l Y_l^T z_l  with  z_l = L_l^-1 g_l.
//
// Landmarks arrive sorted by (first, last) observing frame, so a tile of 32 consecutive landmarks only touches the
// frames [a, b] listed in W.tile_range.  The window's 6K pose columns are packed densely into nB = ceil(6K / 8) blocks
// of 8 columns: pose column (f, e) is column 6f + e, in block (6f + e) / 8.  Per tile, Y is built over the tile's 96
// rows (3 per landmark) for the blocks [6a / 8, (6b + 5) / 8] the range touches; the columns of those blocks that lie
// outside the range's frames (or past 6K) are written as zero.  The SYRK runs on the FP64 tensor cores
// (mma.sync.m8n8k4.f64): block pair (bi, bj), bi >= bj, is one 8x8 block Y_bi^T Y_bj.  Every block pair owns a fixed
// 8x8 accumulator for the whole chunk (shared memory, or the chunk's global partial for windows with many frames); a
// tile adds one DMMA chain per pair of its blocks, so the accumulation order is the tile order whatever the ranges =>
// deterministic, and nothing moves when the range changes.  The right-hand side is formed in the Y build: the warp that
// builds frame f of a tile holds its 32 landmarks, and sums Y_f^T z over them with a fixed butterfly into frame f's
// accumulator (one writer per frame and tile).
// ------------------------------------------------------------------------------------------------
constexpr int kLiStride = 9;                   // L^-1 (6) | z (3), as in global memory (one bulk copy per tile)
// Y is stored column-major, one column of the tile's 96 rows (3 per landmark) every kYCol doubles, so pose column
// (f, e) starts at the fixed offset (6f + e) kYCol.  The 4 doubles of padding make both accesses free of
// bank conflicts: the Y build stores one column at rows 3 ll + c over a warp's 32 landmarks (3 ll mod 16 is a
// permutation), and a m8n8k4 fragment read (lane 4g + t: row 4s + t, column g of the block, i.e. A[g][t] of Y_bi^T
// and B[t][g] of Y_bj alike) hits 4g + t mod 16.
constexpr int kYCol = 3 * A2_TILE + 4;
constexpr int kYBlock = 8 * kYCol;             // doubles of one 8-column Y block

__host__ __device__ inline int schur_blocks(int K) { return (6 * K + 7) / 8; }

// Element (r, c) of block pair (bi, bj)'s 8x8 block, i.e. pose entry (R, C) = (8 bi + r, 8 bj + c), in the chunk's
// partial (dcp x dcp, the full 6x6 block of every frame pair fR >= fC), or -1 for columns past the poses and the
// entries above the diagonal of a diagonal block pair that belong to no stored frame pair.
__device__ __forceinline__ int schur_elem(int bi, int bj, int r, int c, int K, int dcp) {
  const int R = 8 * bi + r, C = 8 * bj + c;
  if (R >= 6 * K || C >= 6 * K || R / 6 < C / 6) return -1;
  return R * dcp + C;
}
// The mirror (C, R) of an entry of a frame's diagonal 6x6 block that the lower block triangle reaches only from below:
// the frame straddles blocks bj < bi.  -1 for every other entry.
__device__ __forceinline__ int schur_mirror(int bi, int bj, int r, int c, int K, int dcp) {
  const int R = 8 * bi + r, C = 8 * bj + c;
  if (bi == bj || R >= 6 * K || R / 6 != C / 6) return -1;
  return C * dcp + R;
}

// acc_smem: 1 = the block-pair accumulators (nB(nB+1)/2 blocks of 64 doubles) and the right-hand side (6K doubles)
// live in shared memory; 0 = accumulate in the chunk's global partial instead (windows with many frames).
__host__ __device__ inline size_t smemA2_bytes(int K, int acc_smem) {
  const size_t nB = (size_t)schur_blocks(K);
  size_t b = 16;                                                    // mbarrier (TMA completion)
  b += nB * kYBlock * sizeof(double);                               // Y, column-major, 8-column blocks
  b += (size_t)K * 6 * A2_TILE * sizeof(double);                   // M tile [f][e][ll]
  b += (size_t)A2_TILE * kLiStride * sizeof(double);               // L^-1 | z
  b += (size_t)A2_TILE * 4 * sizeof(double);                       // X
  b += (size_t)K * 4 * sizeof(double);                             // frame translations
  b += (size_t)acc_smem * (nB * (nB + 1) / 2 * 64 + 6 * (size_t)K) * sizeof(double);
  return b;
}

// Sum over the warp of v[0..5] (v[6], v[7] zero): a reduce-scatter over the lane bits 4, 2, 1, then xor 8 and 16; lane
// e < 6 ends with the sum of value e.  A fixed butterfly, so the summation order is the same on every launch.
__device__ __forceinline__ double warp_sum6(double (&v)[8]) {
  reduce_scatter_step<4>(v);
  reduce_scatter_step<2>(v);
  reduce_scatter_step<1>(v);
  double s = v[0];
  s += __shfl_xor_sync(0xffffffffu, s, 8);
  s += __shfl_xor_sync(0xffffffffu, s, 16);
  return s;
}

// ---- TMA bulk copies (cp.async.bulk, 1-D) completing on an mbarrier
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
               "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok)
                 : "r"(smem_u32(bar)), "r"(parity)
                 : "memory");
  } while (!ok);
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void dmma_8x8x4(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

// NT = 256 where two CTAs fit an SM (cfg-2), else 512: 16 warps per SM either way.
template <int NT>
__global__ void __launch_bounds__(NT, NT == 256 ? 2 : 1) k_schur(const WinDev* __restrict__ wins, const int32_t* __restrict__ win_slots, int acc_smem, int max_iterations) {
  const WinDev& W = wins[win_slots[blockIdx.y]];
  SolverState* st = W.st;
  if (st->done) return;
  // the step being judged in this round is the last one (iteration limit): k_solve will not build another
  // reduced system, so the Schur complement of this linearisation is never used
  if (st->iteration >= max_iterations) return;
  const int chunk = blockIdx.x;
  if (chunk >= W.n_chunks) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  constexpr int NW = NT / 32;
  const int K = W.K, dc = W.dc, dcp = W.dcp, L = W.L;
  const int nB = schur_blocks(K);
  const int n_pairs = nB * (nB + 1) / 2;

  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint64_t* mbar = reinterpret_cast<uint64_t*>(smem_raw);            // TMA completion of the staged tile
  double* Yt = reinterpret_cast<double*>(smem_raw + 16);             // [nB][kYBlock]
  double* sM = Yt + (size_t)nB * kYBlock;                            // [K][6][32]
  double* sLi = sM + (size_t)K * 6 * A2_TILE;
  double* sX = sLi + A2_TILE * kLiStride;
  double* tws = sX + A2_TILE * 4;
  double* Sacc = tws + 4 * K;                                        // [n_pairs][64] when acc_smem
  double* Sp = W.partA + (size_t)chunk * W.partA_stride;
  double* rhs = acc_smem ? Sacc + (size_t)n_pairs * 64 : Sp + (size_t)dc * dcp;     // [6K] right-hand side

  for (int f = tid; f < K; f += NT) {
    tws[4 * f] = W.pose_c[7 * f]; tws[4 * f + 1] = W.pose_c[7 * f + 1]; tws[4 * f + 2] = W.pose_c[7 * f + 2];
  }
  if (acc_smem) for (int i = tid; i < n_pairs * 64 + 6 * K; i += NT) Sacc[i] = 0.0;
  else for (int i = tid; i < dcp * dcp; i += NT) Sp[i] = 0.0;

  const int lm_begin = chunk * W.lm_per_chunk;     // multiple of A2_TILE
  const int lm_end = min(L, lm_begin + W.lm_per_chunk);

  // Asynchronous staging of one tile by the TMA engine (cp.async.bulk, issued by thread 0, completion on mbar);
  // frames [fa, fb] only.  Global and shared layouts agree, so every piece is one contiguous copy:
  //   M  [tile][f][6][32] -> sM[f][6][32] : frames [fa, fb] are one contiguous block
  //   Li [l][9] -> sLi[32][9] (2304 B),  X = lm_c [l][4] -> sX[32][4] (1024 B)
  // Rows beyond the chunk's last landmark read allocated padding (Lp) and are never used.  The staging buffer is only
  // read by the Y build, so the next tile's copies are issued right after it and land while the SYRK runs.
  if (tid == 0) { mbar_init(mbar, 1); fence_proxy_async(); }
  __syncthreads();
  uint32_t parity = 0;
  auto stage = [&](int base, uint32_t tr) {
    const int fa = tr & 0xffu, fb = tr >> 8;
    if (fa > fb || tid != 0) return;       // (the buffer's last generic-proxy reads are ordered before this point by a CTA barrier)
    const uint32_t m_bytes = (uint32_t)(fb - fa + 1) * 6 * A2_TILE * 8;
    mbar_arrive_expect_tx(mbar, m_bytes + A2_TILE * kLiStride * 8 + A2_TILE * 4 * 8);
    bulk_g2s(sM + (size_t)fa * 6 * A2_TILE, W.lm_M + lm_M_index(base, fa, K), m_bytes, mbar);
    bulk_g2s(sLi, W.lm_Li + (size_t)kLiStride * base, A2_TILE * kLiStride * 8, mbar);
    bulk_g2s(sX, W.lm_c + 4 * (size_t)base, A2_TILE * 4 * 8, mbar);
  };

  // Block pair (i, j)'s accumulator as this lane's C[g][2t], C[g][2t+1] of the 8x8 block: read before a DMMA chain
  // (the global-memory latency overlaps the chain), written back with the chain added (and to the mirrored entry where
  // the block holds the lower half of a straddling frame's diagonal block).  Each pair is taken by one warp per tile
  // and tiles are separated by CTA barriers: one writer per element at a time.
  const int g = lane >> 2, t2 = 2 * (lane & 3);
  auto acc_load = [&](int i, int j, double& v0, double& v1) {
    if (acc_smem) {
      const double2 v = reinterpret_cast<const double2*>(Sacc + (size_t)(i * (i + 1) / 2 + j) * 64)[lane];
      v0 = v.x; v1 = v.y;
    } else {
      const int e0 = schur_elem(i, j, g, t2, K, dcp), e1 = schur_elem(i, j, g, t2 + 1, K, dcp);
      v0 = e0 >= 0 ? Sp[e0] : 0.0;
      v1 = e1 >= 0 ? Sp[e1] : 0.0;
    }
  };
  auto acc_store = [&](int i, int j, double v0, double v1) {
    if (acc_smem) {
      reinterpret_cast<double2*>(Sacc + (size_t)(i * (i + 1) / 2 + j) * 64)[lane] = make_double2(v0, v1);
    } else {
      const int e0 = schur_elem(i, j, g, t2, K, dcp), e1 = schur_elem(i, j, g, t2 + 1, K, dcp);
      const int m0 = schur_mirror(i, j, g, t2, K, dcp), m1 = schur_mirror(i, j, g, t2 + 1, K, dcp);
      if (e0 >= 0) Sp[e0] = v0;
      if (e1 >= 0) Sp[e1] = v1;
      if (m0 >= 0) Sp[m0] = v0;
      if (m1 >= 0) Sp[m1] = v1;
    }
  };

#ifdef OKB_SCHUR_PROF     // per-phase cycle counters of chunk 0 / thread 0 (diagnostics builds only):
  // 0 staging wait, 1 Y build, 2 barrier after the Y build, 3 DMMA + accumulator adds, 4 barrier after the SYRK,
  // 5 write-back of the accumulators
  const bool prof = (tid == 0 && chunk == 0);
  unsigned long long t_ph = 0, ph[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  auto now = []() { return (unsigned long long)clock64(); };
#define SCHUR_MARK(i) do { if (prof) { const unsigned long long n_ = now(); ph[i] += n_ - t_ph; t_ph = n_; } } while (0)
  if (prof) t_ph = now();
#else
#define SCHUR_MARK(i) do { } while (0)
#endif
  uint32_t tr_next = (lm_begin < lm_end) ? W.tile_range[lm_begin >> 5] : 1u;
  if (lm_begin < lm_end) stage(lm_begin, tr_next);
  for (int base = lm_begin; base < lm_end; base += A2_TILE) {
    const uint32_t tr = tr_next;
    if (base + A2_TILE < lm_end) tr_next = W.tile_range[(base >> 5) + 1];
    const int fa = tr & 0xffu, fb = tr >> 8;
    const bool live = fa <= fb;            // some landmark of the tile is observed (CTA-uniform)
    const int nl = min(A2_TILE, lm_end - base);
    const int ba = (6 * fa) >> 3, bb = (6 * fb + 5) >> 3;      // the blocks the range touches
    if (live) {
      mbar_wait(mbar, parity);
      parity ^= 1u;
      SCHUR_MARK(0);
      // ---- Y_f = W_f L^-T for every (landmark, frame) pair of the tile, frames [fa, fb], and Y_f^T z.  A warp takes
      // one frame of the 32 landmarks, so each store writes one column (conflict-free, see kYCol).  The warps of
      // frames fa and fb also zero the columns of blocks ba and bb outside the range.
      for (int pidx = tid; pidx < A2_TILE * (fb - fa + 1); pidx += NT) {
        const int ll = pidx % A2_TILE, f = fa + pidx / A2_TILE;      // landmark fastest: conflict-free reads of sM
        const int k0 = 3 * ll, k1 = k0 + 1, k2 = k0 + 2;
        auto zero_column = [&](int c) {
          double* y = Yt + (size_t)c * kYCol;
          y[k0] = 0.0; y[k1] = 0.0; y[k2] = 0.0;
        };
        if (f == fa) for (int c = 8 * ba; c < 6 * fa; ++c) zero_column(c);            // (warp-uniform)
        if (f == fb) for (int c = 6 * fb + 6; c < 8 * bb + 8; ++c) zero_column(c);
        double M0 = 0, M1 = 0, M2 = 0, M3 = 0, M4 = 0, M5 = 0;
        if (ll < nl) {
          const double* sp = sM + (size_t)(f * 6) * A2_TILE + ll;
          M0 = sp[0]; M1 = sp[A2_TILE]; M2 = sp[2 * A2_TILE]; M3 = sp[3 * A2_TILE]; M4 = sp[4 * A2_TILE]; M5 = sp[5 * A2_TILE];
        }
        const double* Li = sLi + ll * kLiStride;
        double y0[6], y1[6], y2[6];      // rows k0, k1, k2 of Y_f
        if (M0 != 0.0 || M3 != 0.0 || M5 != 0.0) {
          const double w = sX[ll * 4 + 3];
          const double p0 = sX[ll * 4] - tws[4 * f] * w, p1 = sX[ll * 4 + 1] - tws[4 * f + 1] * w, p2 = sX[ll * 4 + 2] - tws[4 * f + 2] * w;
          const double N00 = M0 * Li[0], N01 = M0 * Li[1] + M1 * Li[2], N02 = M0 * Li[3] + M1 * Li[4] + M2 * Li[5];
          const double N10 = M1 * Li[0], N11 = M1 * Li[1] + M3 * Li[2], N12 = M1 * Li[3] + M3 * Li[4] + M4 * Li[5];
          const double N20 = M2 * Li[0], N21 = M2 * Li[1] + M4 * Li[2], N22 = M2 * Li[3] + M4 * Li[4] + M5 * Li[5];
          y0[0] = -w * N00; y0[1] = -w * N10; y0[2] = -w * N20;
          y1[0] = -w * N01; y1[1] = -w * N11; y1[2] = -w * N21;
          y2[0] = -w * N02; y2[1] = -w * N12; y2[2] = -w * N22;
          y0[3] = -(p1 * N20 - p2 * N10); y0[4] = -(p2 * N00 - p0 * N20); y0[5] = -(p0 * N10 - p1 * N00);
          y1[3] = -(p1 * N21 - p2 * N11); y1[4] = -(p2 * N01 - p0 * N21); y1[5] = -(p0 * N11 - p1 * N01);
          y2[3] = -(p1 * N22 - p2 * N12); y2[4] = -(p2 * N02 - p0 * N22); y2[5] = -(p0 * N12 - p1 * N02);
        } else {
#pragma unroll
          for (int e = 0; e < 6; ++e) { y0[e] = 0.0; y1[e] = 0.0; y2[e] = 0.0; }
        }
        const double z0 = ll < nl ? Li[6] : 0.0, z1 = ll < nl ? Li[7] : 0.0, z2 = ll < nl ? Li[8] : 0.0;
        double* y = Yt + (size_t)(6 * f) * kYCol;
        double v[8];
#pragma unroll
        for (int e = 0; e < 6; ++e) {
          y[e * kYCol + k0] = y0[e]; y[e * kYCol + k1] = y1[e]; y[e * kYCol + k2] = y2[e];
          v[e] = (y0[e] * z0 + y1[e] * z1) + y2[e] * z2;
        }
        v[6] = 0.0; v[7] = 0.0;
        const double r = warp_sum6(v);
        if (lane < 6) rhs[6 * f + lane] += r;
      }
      SCHUR_MARK(1);
    }
    __syncthreads();                       // Y is complete; the staging buffer is free
    SCHUR_MARK(2);
    if (base + A2_TILE < lm_end) stage(base + A2_TILE, tr_next);
    if (!live) continue;
    // ---- SYRK: items of one or two block pairs (i, j0), (i, j0 + 1) sharing row block i, dealt to the warps in a
    // fixed order.  Per k-step a two-pair item loads three fragments for two DMMAs.  Rows past the tile's last
    // landmark are zero and are skipped.
    const int ub = bb - ba + 1;
    const int ns = (3 * nl + 3) >> 2;
    const int n_items = (ub + 1) * (ub + 1) / 4;    // sum over the rows il of ceil((il + 1) / 2)
    for (int it = warp; it < n_items; it += NW) {
      int il = 0, q = it;
      while (q >= ((il + 2) >> 1)) { q -= (il + 2) >> 1; ++il; }
      const int i = ba + il, j0 = ba + 2 * q;
      const double* ya = Yt + (size_t)i * kYBlock + g * kYCol + (lane & 3);      // this lane's fragment slot
      const double* yb = Yt + (size_t)j0 * kYBlock + g * kYCol + (lane & 3);
      double c0 = 0.0, c1 = 0.0, o0, o1;
      acc_load(i, j0, o0, o1);
      if (j0 < i) {                        // (warp-uniform)
        double e0 = 0.0, e1 = 0.0, q0, q1;
        acc_load(i, j0 + 1, q0, q1);
#pragma unroll 4
        for (int s = 0; s < ns; ++s) {
          const double a = ya[4 * s], b0 = yb[4 * s], b1 = yb[kYBlock + 4 * s];
          dmma_8x8x4(c0, c1, a, b0);
          dmma_8x8x4(e0, e1, a, b1);
        }
        acc_store(i, j0 + 1, q0 + e0, q1 + e1);
      } else {
#pragma unroll 4
        for (int s = 0; s < ns; ++s) {
          const double a = ya[4 * s];
          dmma_8x8x4(c0, c1, a, a);
        }
      }
      acc_store(i, j0, o0 + c0, o1 + c1);
    }
    SCHUR_MARK(3);
    __syncthreads();                       // Y may be rebuilt
    SCHUR_MARK(4);
  }
  if (acc_smem) {
    __syncthreads();
    // unpack the 8x8 blocks into the frame-pair blocks k_reduce_partials / k_solve read, and the right-hand side
    for (int e = tid; e < n_pairs * 64; e += NT) {
      const int p = e >> 6;
      int i = (int)((sqrtf(8.0f * (float)p + 1.0f) - 1.0f) * 0.5f);
      while (i * (i + 1) / 2 > p) --i;
      while ((i + 1) * (i + 2) / 2 <= p) ++i;
      const int j = p - i * (i + 1) / 2;
      const int ln = (e & 63) >> 1, r = ln >> 2, c = 2 * (ln & 3) + (e & 1);
      const int idx = schur_elem(i, j, r, c, K, dcp), mir = schur_mirror(i, j, r, c, K, dcp);
      if (idx >= 0) Sp[idx] = Sacc[e];
      if (mir >= 0) Sp[mir] = Sacc[e];
    }
    for (int e = tid; e < 6 * K; e += NT) Sp[(size_t)dc * dcp + e] = rhs[e];
  }
  SCHUR_MARK(5);
#ifdef OKB_SCHUR_PROF
  if (prof) for (int i = 0; i < 8; ++i) st->phase_ns[8 + i] += ph[i];
#endif
#undef SCHUR_MARK
}

// Sums the per-chunk Schur accumulators of a window into chunk 0 (fixed order => deterministic), in
// parallel over the matrix elements, so that k_solve reads one partial regardless of the chunk count.
__global__ void __launch_bounds__(256) k_reduce_partials(const WinDev* __restrict__ wins, const int32_t* __restrict__ win_slots) {
  const WinDev& W = wins[win_slots[blockIdx.y]];
  if (W.st->done || W.n_chunks <= 1) return;
  const int n = W.dcp * W.dcp;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double s = W.partA[i];
    for (int c = 1; c < W.n_chunks; ++c) s += W.partA[(size_t)c * W.partA_stride + i];
    W.partA[i] = s;
  }
}

// ------------------------------------------------------------------------------------------------
// Landmark-sharded window: k_reduce_partials fused with the push half of the all-reduce.  Every rank sums its
// chunk partials (Schur accumulator) and its per-CTA pose-block records in fixed order and stores the result with
// plain stores into box [parity][rank] of EVERY rank's mailbox (its own included) -- remote stores travel over
// NVLink / NVSwitch and are not waited for.  The last CTA of the window fences at system scope and releases the
// `world` ready flags.  The sum over ranks happens in k_solve's prologue (every rank adds the boxes in rank order
// => bit-identical reduced systems, so the redundant reduced solves stay in lock step).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double* shard_box(const WinDev& W, int dst, int parity, int src) {
  return reinterpret_cast<double*>(W.shard_mail[dst] + kShardHeaderBytes) + ((size_t)parity * W.shard_world + src) * W.shard_box_cap;
}
__device__ __forceinline__ double* shard_marg_box(const WinDev& W, int dst, int parity, int src) {
  return reinterpret_cast<double*>(W.shard_mail[dst] + kShardHeaderBytes) + 2 * (size_t)W.shard_world * W.shard_box_cap +
         ((size_t)parity * W.shard_world + src) * W.shard_marg_cap;
}
__device__ __forceinline__ unsigned long long* shard_flag(const WinDev& W, int dst, size_t which, int parity, int src) {
  return reinterpret_cast<unsigned long long*>(W.shard_mail[dst] + which) + parity * kMaxShard + src;
}

__global__ void __launch_bounds__(256) k_shard_push(const WinDev* __restrict__ wins, const int32_t* __restrict__ win_slots) {
  const WinDev& W = wins[win_slots[blockIdx.y]];
  SolverState* st = W.st;
  if (st->done) return;
  const int world = W.shard_world, me = W.shard_rank;
  const unsigned long long epoch = st->shard_epoch + 1;
  const int par = (int)(epoch & 1ull);
  const int K = W.K, nA = W.dcp * W.dcp, nH = K * kPartH;
  const int n = nA + nH + 8;
  const int n_cx = (W.L + L1_THREADS - 1) / L1_THREADS;
  double* dst[kMaxShard];
#pragma unroll
  for (int r = 0; r < kMaxShard; ++r) dst[r] = (r < world) ? shard_box(W, r, par, me) : nullptr;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double s = 0.0;
    if (i < nA) {
      s = W.partA[i];
      for (int c = 1; c < W.n_chunks; ++c) s += W.partA[(size_t)c * W.partA_stride + i];
    } else if (i < nA + nH) {
      const int j = i - nA, f = j / kPartH, e = j % kPartH;
      if (e < 29)
        for (int c = 0; c < n_cx; ++c) s += W.partH[((size_t)c * K + f) * kPartH + e];
    } else if (i == nA + nH) {
      s = st->numeric_fail ? 1.0 : 0.0;
    }
#pragma unroll
    for (int r = 0; r < kMaxShard; ++r)
      if (r < world) dst[r][i] = s;
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int* counter = reinterpret_cast<unsigned int*>(W.shard_mail[me] + kShardCounter);
    const unsigned int prev = atomicAdd(counter, 1u);
    if (prev == gridDim.x - 1) {
      *counter = 0u;
      __threadfence_system();
      for (int r = 0; r < world; ++r) st_release_sys_u64(shard_flag(W, r, kShardFlags1, par, me), epoch);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Post-solve landmark quality: H = sum J_lm^T J_lm (sqrt-information weighted, no robust weight)
// at the final estimate; quality = sqrt(lambda_min)/sqrt(lambda_max), 0 if lambda_min < 1e-12.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_quality(const WinDev* __restrict__ wins, const int32_t* __restrict__ win_slots) {
  const WinDev& W = wins[win_slots[blockIdx.y]];
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SlotCtx* slots = reinterpret_cast<SlotCtx*>(smem_raw);
  const int tid = threadIdx.x;
  for (int s = tid; s < W.NS; s += blockDim.x) {
    const SlotInfo si = W.slots[s];
    SlotCtx& sc = slots[s];
    sc.valid = si.valid; sc.frame = si.valid ? si.pose_idx : 0;
    if (si.valid) { make_slot_xf(W.pose + 7 * si.pose_idx, W.ext + 7 * si.ext_idx, sc.xf); cam_load(W.cams[si.cam_idx], sc.cam); }
  }
  __syncthreads();
  const int L = W.L, CP = W.CP;
  for (int l = blockIdx.x * blockDim.x + tid; l < L; l += gridDim.x * blockDim.x) {
    const double4 x4 = *reinterpret_cast<const double4*>(W.lm + 4 * (size_t)l);
    const double X[4] = {x4.x, x4.y, x4.z, x4.w};
    double H[6] = {0, 0, 0, 0, 0, 0};
    uint32_t vis = W.lm_vis[l];
    while (vis) {
      const int f = __ffs(vis) - 1;
      vis &= vis - 1;
      for (int c = 0; c < CP; ++c) {
        const int s = f * CP + c;
        const double wobs = W.obs_w[(size_t)s * L + l];
        if (wobs > 0.0 && slots[s].valid) {
          const double2 z = W.obs_z[(size_t)s * L + l];
          double r[2], A[6];
          reproj_slot<true>(slots[s].xf, slots[s].cam, X, z.x, z.y, wobs, r, A);
          H[0] += A[0] * A[0] + A[3] * A[3]; H[1] += A[0] * A[1] + A[3] * A[4]; H[2] += A[0] * A[2] + A[3] * A[5];
          H[3] += A[1] * A[1] + A[4] * A[4]; H[4] += A[1] * A[2] + A[4] * A[5]; H[5] += A[2] * A[2] + A[5] * A[5];
        }
      }
    }
    double ev[3];
    eig3sym_closed(H, ev);
    const double q = (ev[0] < 1.0e-12) ? 0.0 : sqrt(ev[0]) / sqrt(ev[2]);
    W.quality[l] = q;
    // write-back in the caller's order: the master copy (next compile) and the packed download block
    const uint32_t lc = W.perm[l];
    *reinterpret_cast<double4*>(W.m_lm + 4 * (size_t)lc) = x4;
    double* o = W.out + out_lm_offset(W.K, W.NSB);
    *reinterpret_cast<double4*>(o + 4 * (size_t)lc) = x4;
    o[4 * (size_t)L + lc] = q;
  }
  if (blockIdx.x == 0) {
    for (int i = tid; i < 7 * W.K; i += blockDim.x) W.out[i] = W.pose[i];
    for (int i = tid; i < 9 * W.NSB; i += blockDim.x) W.out[7 * W.K + i] = W.sb[i];
  }
}

}  // namespace okb
