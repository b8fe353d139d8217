// Device-side marginalisation (sm_90a): the numeric work of okvis::ceres::MarginalizationError that
// Estimator::applyMarginalizationStrategy (okvis_ceres/src/Estimator.cpp:434-773) drives once per frame --
//   addResidualBlock       okvis_ceres/src/MarginalizationError.cpp:127-435  (linearise residual blocks at the
//                          first-estimate linearisation points, Cauchy correction :313-365, H += J^T J, b0 -= J^T r)
//   marginalizeOut         :507-802  (landmark blocks: per-3x3 pseudo-inverse; dense blocks: eigen pseudo-inverse;
//                          Schur complements in a diagonally preconditioned system)
//   updateErrorComputation :806-846  (H = U S U^T,  J = (p U sqrt(S))^T,  e0 = -sqrt(S)^+ U^T p^-1 b0)
//   pseudoInverseSymmSqrt  okvis_ceres/include/okvis/ceres/implementation/MarginalizationError.hpp:215-243
// -- so that the window stays resident on the device across frames: the result replaces the window's
// marginalisation prior in place (marg_J / marg_e0 / marg_H0 / block list / linearisation points) and is what the
// next okb_optimize evaluates (row M).  One CTA per window:
//   phase 0  linearisation points (kept from the current prior or the current estimate), column layout
//   phase 1  the current prior's H / b0 scattered into the new ordering
//   phase 2  SpeedAndBiasError terms                      (J = -sqrt_info)
//   phase 3  ImuError terms (warp 0, the same imu_evaluate the solver uses; the term's cache is mutated
//            exactly like the reference's functor)
//   phase 4  reprojection errors of the landmarks to marginalise, loss-corrected; per landmark the 3x3 block V is
//            pseudo-inverted in its preconditioned form and eliminated:  H_pp -= W V^+ W^T,  b_p -= W V^+ b_l
//            (the preconditioner of the kept coordinates cancels, only p_b = sqrt(diag V) matters)
//   phase 5  dense blocks to marginalise: V^+ through a parallel cyclic Jacobi eigen-decomposition, Schur complement
//   phase 6  eigen-decomposition of the preconditioned reduced H -> J, e0, H0 = J^T J
// All sums run in a fixed order: bit-reproducible.
// Landmark-sharded windows run k_marginalize<true> on every rank: phases 0-3 see only replicated inputs, phase 4 sees
// the rank's own landmarks.  Its per-element sums over them (pose x pose entries of H, pose rows of b) are pushed into
// box [parity][rank] of every rank's mailbox instead of being added; after the flag exchange every rank adds the
// `world` boxes in rank order and runs phases 5-6 on bit-identical inputs.  A job fingerprint and each rank's error word
// travel with the boxes: a mismatch, an error on any rank or a peer time-out abandons the step on every rank before
// phase 5 with one status, and the previous prior stays.
#pragma once
#include "okb_estimator.cuh"
#include "okb_graph.cuh"
#include "okb_kernels.cuh"

namespace okb {

constexpr int kMargWork = 256;          // largest linear system (dense coordinates) built before marginalising
constexpr int M_THREADS = 256;
constexpr int kMargRec = 72;            // doubles per (landmark, frame) record: W 18 | Z 18 | U 21 | bp 6 | Wy 6 | pad
enum { MERR_BLOCK = 1, MERR_PREV = 2, MERR_TERM = 3, MERR_POSE_NOT_CONNECTED = 4, MERR_DIM = 5,
       MERR_SHARD_JOB = 6,         // the ranks' jobs differ in their replicated part (fingerprint)
       MERR_SHARD_TIMEOUT = 7 };   // a peer did not arrive within kShardTimeoutNs

// Job as laid out in the batch buffer of the call (header, then the index lists, 16-byte aligned).
struct MargJobHeader {
  int32_t n_blocks, n_imu, n_sbp, n_lm;
  int32_t N;              // dimension of the system before marginalising
  int32_t n_keep;         // dimension after
  int32_t lm_cap;         // landmark records the scratch can hold
  int32_t _pad;
};

struct MargScratch {
  // the job: in the batch buffer of the call
  MargJobHeader* hdr;
  int32_t* kind; uint32_t* idx; int32_t* prev; uint8_t* marg;
  uint32_t* imu_terms; uint32_t* sb_priors; uint32_t* landmarks;
  // work arrays and status: carved out of one device buffer per slot (WinStore::marg_scratch)
  double* H;              // [N][N] work system
  double* b;              // [N]
  double* A;              // [N][N] eigen work
  double* Q;              // [N][N] eigenvectors
  double* T;              // [N][N] temp
  double* Hn;             // [N][N] reduced system
  double* bn;             // [N]
  double* xlin;           // [n_blocks][9]
  double* lmrec;          // [lm_cap][K][kMargRec]
  double* lmV;            // [lm_cap][16]: Veff^+ (9) | y = Veff^+ b_l (3) | pad
  uint32_t* lmvis;        // [lm_cap] frames with a record
  int32_t* lmslot;        // [Lcap] landmark -> slot + 1 (all zero between calls)
  int32_t* clist;         // [Ocap] indices of the observations to linearise, list order
  int32_t* status;        // [4]: error code, rank of the final H, rank of the dense V, Jacobi sweeps (max of phases 5, 6)
};

// One entry of k_marginalize's task table per CTA: the window it marginalises and where its job and scratch lie.
// fingerprint: landmark-sharded windows only, the host's hash of the job's replicated part (MargJobHeader has no
// 64-bit spare field).
struct alignas(16) MargTask {
  int32_t win, _pad;
  uint64_t fingerprint;
  MargScratch sc;
};
static_assert(sizeof(MargTask) % 16 == 0, "MargTask is copied as 16-byte words");

// 3x3 symmetric eigen-decomposition by cyclic Jacobi (S packed: 00 01 02 11 12 22); Q columns = eigenvectors
__device__ inline void eig3_jacobi(const double* S, double* ev, double* Q) {
  double a[3][3] = {{S[0], S[1], S[2]}, {S[1], S[3], S[4]}, {S[2], S[4], S[5]}};
  double q[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int sweep = 0; sweep < 32; ++sweep) {
    const double off = a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2];
    const double dg = a[0][0] * a[0][0] + a[1][1] * a[1][1] + a[2][2] * a[2][2];
    if (off <= 1e-32 * (dg + off) || off == 0.0) break;
    for (int p = 0; p < 2; ++p)
      for (int r = p + 1; r < 3; ++r) {
        const double apq = a[p][r];
        if (apq == 0.0) continue;
        const double theta = (a[r][r] - a[p][p]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 3; ++k) { const double x = a[k][p], y = a[k][r]; a[k][p] = c * x - s * y; a[k][r] = s * x + c * y; }
        for (int k = 0; k < 3; ++k) { const double x = a[p][k], y = a[r][k]; a[p][k] = c * x - s * y; a[r][k] = s * x + c * y; }
        for (int k = 0; k < 3; ++k) { const double x = q[k][p], y = q[k][r]; q[k][p] = c * x - s * y; q[k][r] = s * x + c * y; }
      }
  }
  for (int i = 0; i < 3; ++i) { ev[i] = a[i][i]; for (int j = 0; j < 3; ++j) Q[i * 3 + j] = q[i][j]; }
}

// Parallel cyclic Jacobi on A (n x n, row-major, leading dimension n, symmetric, in global scratch).  On return the
// diagonal of A holds the eigenvalues and column k of Q the matching eigenvector.  All threads of the CTA call it.
// Round-robin ordering: n/2 disjoint rotations per round, applied as A <- R^T (A R) in two conflict-free passes.
__device__ inline int jacobi_eig(double* A, double* Q, int n, double* s_cs /* [2 * 128] */, int* s_pq /* [2 * 128] */, double* red) {
  const int tid = threadIdx.x, NT = blockDim.x;
  for (int i = tid; i < n * n; i += NT) Q[i] = ((i / n) == (i % n)) ? 1.0 : 0.0;
  __syncthreads();
  if (n < 2) return 0;
  const int m = (n + 1) & ~1, half = m / 2;
  int sweep = 0;
  for (; sweep < 40; ++sweep) {
    double off = 0.0, dg = 0.0;
    for (int i = tid; i < n * n; i += NT) {
      const int r = i / n, c = i % n;
      const double v = A[i];
      if (c > r) off += v * v; else if (c == r) dg += v * v;
    }
    off = block_sum(off, red);
    dg = block_sum(dg, red);
    if (off <= 1e-32 * (dg + off) || off == 0.0) break;
    for (int round = 0; round < m - 1; ++round) {
      if (tid < half) {
        int p, q;
        if (tid == 0) { p = m - 1; q = round; }
        else { p = (round + tid) % (m - 1); q = (round - tid + (m - 1)) % (m - 1); }
        if (p > q) { const int t = p; p = q; q = t; }
        double c = 1.0, s = 0.0;
        if (q < n) {
          const double apq = A[(size_t)p * n + q];
          if (apq != 0.0) {
            const double theta = (A[(size_t)q * n + q] - A[(size_t)p * n + p]) / (2.0 * apq);
            const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
            c = 1.0 / sqrt(t * t + 1.0); s = t * c;
          }
        } else { p = -1; }
        s_pq[2 * tid] = p; s_pq[2 * tid + 1] = q;
        s_cs[2 * tid] = c; s_cs[2 * tid + 1] = s;
      }
      __syncthreads();
      // columns p, q of A and of Q
      for (int w = tid; w < half * n; w += NT) {
        const int pr = w / n, k = w % n;
        const int p = s_pq[2 * pr], q = s_pq[2 * pr + 1];
        if (p < 0) continue;
        const double c = s_cs[2 * pr], s = s_cs[2 * pr + 1];
        const double akp = A[(size_t)k * n + p], akq = A[(size_t)k * n + q];
        A[(size_t)k * n + p] = c * akp - s * akq;
        A[(size_t)k * n + q] = s * akp + c * akq;
        const double vkp = Q[(size_t)k * n + p], vkq = Q[(size_t)k * n + q];
        Q[(size_t)k * n + p] = c * vkp - s * vkq;
        Q[(size_t)k * n + q] = s * vkp + c * vkq;
      }
      __syncthreads();
      // rows p, q of A
      for (int w = tid; w < half * n; w += NT) {
        const int pr = w / n, k = w % n;
        const int p = s_pq[2 * pr], q = s_pq[2 * pr + 1];
        if (p < 0) continue;
        const double c = s_cs[2 * pr], s = s_cs[2 * pr + 1];
        const double apk = A[(size_t)p * n + k], aqk = A[(size_t)q * n + k];
        A[(size_t)p * n + k] = c * apk - s * aqk;
        A[(size_t)q * n + k] = s * apk + c * aqk;
      }
      __syncthreads();
    }
  }
  return sweep;
}

__device__ __forceinline__ double marg_precond(double hii) { return (hii > 1.0e-9) ? sqrt(hii) : 1.0e-3; }

// Box parity of a landmark-sharded window's next marginalisation exchange (the epoch lives in the rank's own mailbox
// header, so it survives okb_window_reset and uploads like the solver's shard_epoch).
__device__ __forceinline__ int marg_shard_parity(const WinDev& W) {
  return (int)((*reinterpret_cast<const unsigned long long*>(W.shard_mail[W.shard_rank] + kShardMargEpoch) + 1ull) & 1ull);
}

// One CTA per task: CTA b marginalises window tasks[b].win with the job and scratch of tasks[b].sc.  The task is
// copied to shared memory once; the phases read its pointers from there.  kShard: the window is landmark-sharded (see
// the top of this file); an error in phases 0-4 is pushed to the peers instead of ending the CTA early, so no peer
// waits for a rank that has left.
#pragma nv_diag_suppress 177      // label `exchange` is only jumped to in the sharded instantiation
template <bool kShard>
__global__ void __launch_bounds__(M_THREADS) k_marginalize(const WinDev* __restrict__ wins, const MargTask* __restrict__ tasks) {
  __shared__ MargTask s_task;
  if (threadIdx.x < sizeof(MargTask) / 16)
    reinterpret_cast<int4*>(&s_task)[threadIdx.x] = reinterpret_cast<const int4*>(tasks + blockIdx.x)[threadIdx.x];
  __syncthreads();
  const MargScratch& sc = s_task.sc;
  const WinDev& W = wins[s_task.win];
  GraphState* g = &W.st->g;
  const MargJobHeader J = *sc.hdr;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int NB = J.n_blocks, N = J.N, K = g->K, NSB = g->NSB;
  __shared__ double s_imu[kImuScratch];
  __shared__ double s_red[64];
  __shared__ double s_cs[256];
  __shared__ int s_pq[256];
  __shared__ int s_col[kMaxMargBlocks + 1], s_dim[kMaxMargBlocks];
  __shared__ int s_pose_blk[kMaxFrames], s_sb_blk[kMaxFrames];
  __shared__ short s_ia[kMargWork], s_ib[kMargWork], s_oldrow[kMargWork], s_rowblk[kMargWork];
  __shared__ int s_i[8];
  const double eps = 2.220446049250313e-16;

  // ---------------- phase 0: layout + linearisation points
  if (tid == 0) {
    int col = 0, err = 0;
    for (int k = 0; k < 4; ++k) sc.status[k] = 0;     // this call's status word (read by okb_window_download_marg)
    for (int f = 0; f < kMaxFrames; ++f) { s_pose_blk[f] = -1; s_sb_blk[f] = -1; }
    for (int b = 0; b < NB; ++b) {
      const int kind = sc.kind[b];
      const int dim = (kind == OKB_BLOCK_SPEED_BIAS) ? 9 : 6;
      s_col[b] = col; s_dim[b] = dim;
      const int lim = (kind == OKB_BLOCK_POSE) ? K : (kind == OKB_BLOCK_SPEED_BIAS) ? NSB : -1;
      if (lim < 0 || (int)sc.idx[b] >= lim) { err = MERR_BLOCK; break; }
      int* slot = (kind == OKB_BLOCK_POSE) ? &s_pose_blk[sc.idx[b]] : &s_sb_blk[sc.idx[b]];
      if (*slot != -1) { err = MERR_BLOCK; break; }
      *slot = b;
      const int pv = sc.prev[b];
      if (pv >= 0 && (pv >= g->marg_nb || W.marg_kind[pv] != kind || W.marg_idx[pv] != sc.idx[b] || W.marg_col[pv] < 0)) { err = MERR_PREV; break; }
      col += dim;
    }
    s_col[NB] = col;
    if (!err && col != N) err = MERR_DIM;
    // every non-fixed block of the current prior must be carried over exactly once
    if (!err) {
      int seen = 0;
      for (int b = 0; b < NB; ++b) if (sc.prev[b] >= 0) ++seen;
      int live = 0;
      for (int p = 0; p < g->marg_nb; ++p) if (W.marg_col[p] >= 0) ++live;
      if (seen != live) err = MERR_PREV;
    }
    s_i[0] = err;
  }
  __syncthreads();
  if (s_i[0]) {
    if (tid == 0) { sc.status[0] = s_i[0]; graph_error(g, GERR_DIMS); }
    if constexpr (kShard) goto exchange; else return;
  }
  for (int b = tid; b < NB; b += M_THREADS) {
    const int kind = sc.kind[b], pv = sc.prev[b];
    const int w = (kind == OKB_BLOCK_SPEED_BIAS) ? 9 : 7;
    const double* src = (pv >= 0) ? W.marg_x0 + W.marg_off[pv] : (kind == OKB_BLOCK_POSE) ? W.pose + 7 * sc.idx[b] : W.sb + 9 * sc.idx[b];
    for (int k = 0; k < w; ++k) sc.xlin[9 * b + k] = src[k];
  }
  for (int b = tid; b < NB; b += M_THREADS) {
    const int pv = sc.prev[b];
    for (int k = 0; k < s_dim[b]; ++k) { s_rowblk[s_col[b] + k] = (short)b; s_oldrow[s_col[b] + k] = (short)((pv >= 0) ? W.marg_col[pv] + k : -1); }
  }
  __syncthreads();
  // ---------------- phase 1: the current prior (H, b0 as left by the previous marginalisation) in the new ordering
  {
    const int n_old = g->marg_n;
    for (int i = tid; i < N * N; i += M_THREADS) {
      const int r = i / N, c = i % N;
      const int orow = s_oldrow[r], ocol = s_oldrow[c];
      sc.H[i] = (orow >= 0 && ocol >= 0) ? W.marg_Hs[(size_t)orow * n_old + ocol] : 0.0;
    }
    for (int r = tid; r < N; r += M_THREADS) sc.b[r] = (s_oldrow[r] >= 0) ? W.marg_b0[s_oldrow[r]] : 0.0;
  }
  __syncthreads();
  // ---------------- phase 2: SpeedAndBiasError terms  r = S (meas - x),  J = -S
  for (int i = 0; i < J.n_sbp; ++i) {
    const uint32_t pi = sc.sb_priors[i];
    if ((int)pi >= g->n_sbp) {
      if (tid == 0) { sc.status[0] = MERR_TERM; graph_error(g, GERR_INDEX); }
      if constexpr (kShard) goto exchange; else return;
    }
    const okb_sb_prior& pr = W.sbp[pi];
    const int blk = ((int)pr.sb_idx < kMaxFrames) ? s_sb_blk[pr.sb_idx] : -1;
    if (blk < 0) {
      if (tid == 0) { sc.status[0] = MERR_TERM; graph_error(g, GERR_INDEX); }
      if constexpr (kShard) goto exchange; else return;
    }
    const int o = s_col[blk];
    const double* x = sc.xlin + 9 * blk;
    if (tid < 81) {
      const int a = tid / 9, bb = tid % 9;
      double s = 0;
      for (int k = 0; k < 9; ++k) s += pr.sqrt_info[k * 9 + a] * pr.sqrt_info[k * 9 + bb];
      sc.H[(size_t)(o + a) * N + o + bb] += s;
    } else if (tid >= 96 && tid < 105) {
      const int a = tid - 96;
      double s = 0;
      for (int k = 0; k < 9; ++k) {
        double rk = 0;
        for (int j = 0; j < 9; ++j) rk += pr.sqrt_info[k * 9 + j] * (pr.meas[j] - x[j]);
        s += pr.sqrt_info[k * 9 + a] * rk;       // b0 -= J^T r = +S^T r
      }
      sc.b[o + a] += s;
    }
    __syncthreads();
  }
  // ---------------- phase 3: ImuError terms
  for (int i = 0; i < J.n_imu; ++i) {
    const uint32_t t = sc.imu_terms[i];
    if ((int)t >= g->n_imu) {
      if (tid == 0) { sc.status[0] = MERR_TERM; graph_error(g, GERR_INDEX); }
      if constexpr (kShard) goto exchange; else return;
    }
    const okb_imu_term& T = W.imu_terms[t];
    const int blks[4] = {s_pose_blk[T.pose0], s_sb_blk[T.sb0], s_pose_blk[T.pose1], s_sb_blk[T.sb1]};
    if (blks[0] < 0 || blks[1] < 0 || blks[2] < 0 || blks[3] < 0) {
      if (tid == 0) { sc.status[0] = MERR_TERM; graph_error(g, GERR_INDEX); }
      if constexpr (kShard) goto exchange; else return;
    }
    const ImuScratch isc = imu_scratch(s_imu);
    double* SF = isc.SF;
    double* r15 = isc.r15;
    if (warp == 0) {
      WarpCtx cx;
      imu_evaluate(cx, W.samples + T.sample_offset, (int)T.sample_count, W.imu_params, T.t0_ns, T.t1_ns, sc.xlin + 9 * blks[0], sc.xlin + 9 * blks[1],
                   sc.xlin + 9 * blks[2], sc.xlin + 9 * blks[3], W.imu_cache + t, isc.wk, isc.F01, (double*)nullptr, r15, SF);
    }
    __syncthreads();
    const int offs[4] = {s_col[blks[0]], s_col[blks[1]], s_col[blks[2]], s_col[blks[3]]};
    for (int e = tid; e < 930; e += M_THREADS) {
      const int a = (e < 900) ? e / 30 : e - 900, bcol = (e < 900) ? e % 30 : 0;
      const int ba = (a < 6) ? 0 : (a < 15) ? 1 : (a < 21) ? 2 : 3;
      const int la = a - ((ba == 0) ? 0 : (ba == 1) ? 6 : (ba == 2) ? 15 : 21);
      if (e < 900) {
        const int bb = (bcol < 6) ? 0 : (bcol < 15) ? 1 : (bcol < 21) ? 2 : 3;
        const int lb = bcol - ((bb == 0) ? 0 : (bb == 1) ? 6 : (bb == 2) ? 15 : 21);
        double s = 0;
#pragma unroll
        for (int k = 0; k < 15; ++k) s += SF[k * 30 + a] * SF[k * 30 + bcol];
        sc.H[(size_t)(offs[ba] + la) * N + offs[bb] + lb] += s;
      } else {
        double s = 0;
#pragma unroll
        for (int k = 0; k < 15; ++k) s += SF[k * 30 + a] * r15[k];
        sc.b[offs[ba] + la] -= s;
      }
    }
    __syncthreads();
  }
  // ---------------- phase 4: landmarks to marginalise (sharded: the rank's own; a rank with none still pushes zeros)
  if (const int n_lm = J.n_lm; kShard || n_lm > 0) {
    const int n_obs = g->n_obs;
    const int mpar = kShard ? marg_shard_parity(W) : 0;
    if constexpr (kShard) {       // packed pose coordinate of each row of H (s_ia is free until phase 5), count in s_i[3]
      if (tid == 0) {
        int p = 0;
        for (int r = 0; r < N; ++r) s_ia[r] = (short)((sc.kind[s_rowblk[r]] == OKB_BLOCK_POSE) ? p++ : -1);
        s_i[3] = p;
      }
    }
    for (int j = tid; j < n_lm; j += M_THREADS) {
      const uint32_t l = sc.landmarks[j];
      if ((int)l < g->L) sc.lmslot[l] = j + 1;
      sc.lmvis[j] = 0u;
    }
    for (size_t i = tid; i < (size_t)n_lm * K * kMargRec; i += M_THREADS) sc.lmrec[i] = 0.0;
    __syncthreads();
    // observations to linearise, in list order
    int n_c = 0;
    {
      int* s_warp = s_pq;       // 32 ints of scan scratch
      for (int base = 0; base < n_obs; base += M_THREADS) {
        const int i = base + tid;
        int keep = 0;
        if (i < n_obs) {
          const okb_observation& ob = W.m_obs[i];
          keep = (ob.sqrt_info != 0.0 && (int)ob.lm_idx < g->L && sc.lmslot[ob.lm_idx] > 0) ? 1 : 0;
        }
        // exclusive scan over the CTA (8 warps)
        int x = keep;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
        __syncthreads();
        if (lane == 31) s_warp[warp] = x;
        __syncthreads();
        int wbase = 0, total = 0;
        for (int w2 = 0; w2 < M_THREADS / 32; ++w2) { if (w2 < warp) wbase += s_warp[w2]; total += s_warp[w2]; }
        if (keep) sc.clist[n_c + wbase + x - 1] = i;
        n_c += total;
      }
    }
    __syncthreads();
    const bool cauchy = W.use_cauchy != 0;
    // one thread per landmark: its observations in list order
    for (int j = tid; j < n_lm; j += M_THREADS) {
      const uint32_t l = sc.landmarks[j];
      double Vp[6] = {0, 0, 0, 0, 0, 0}, bl[3] = {0, 0, 0};
      uint32_t vis = 0u;
      bool bad = (int)l >= g->L;
      const double* X = W.m_lm + 4 * (size_t)(bad ? 0 : l);
      for (int ci = 0; ci < n_c && !bad; ++ci) {
        const okb_observation ob = W.m_obs[sc.clist[ci]];
        if (ob.lm_idx != l) continue;
        const int f = (int)ob.pose_idx;
        const int blk = s_pose_blk[f];
        if (blk < 0) { bad = true; break; }
        double r[2], J0[12], J1[6];
        reproj_full(W.cams[ob.cam_idx], sc.xlin + 9 * blk, X, W.ext + 7 * ob.ext_idx, ob.z, ob.sqrt_info, r, J0, J1, (double*)nullptr);
        if (cauchy) {         // Corrector with rho'' < 0: residual and Jacobians scaled by sqrt(rho')
          const double wq = sqrt(1.0 / (1.0 + r[0] * r[0] + r[1] * r[1]));
          for (int k = 0; k < 12; ++k) J0[k] *= wq;
          for (int k = 0; k < 6; ++k) J1[k] *= wq;
          r[0] *= wq; r[1] *= wq;
        }
        Vp[0] += J1[0] * J1[0] + J1[3] * J1[3]; Vp[1] += J1[0] * J1[1] + J1[3] * J1[4]; Vp[2] += J1[0] * J1[2] + J1[3] * J1[5];
        Vp[3] += J1[1] * J1[1] + J1[4] * J1[4]; Vp[4] += J1[1] * J1[2] + J1[4] * J1[5]; Vp[5] += J1[2] * J1[2] + J1[5] * J1[5];
        for (int a = 0; a < 3; ++a) bl[a] -= J1[a] * r[0] + J1[3 + a] * r[1];
        double* rec = sc.lmrec + ((size_t)j * K + f) * kMargRec;
        for (int a = 0; a < 6; ++a)
          for (int c3 = 0; c3 < 3; ++c3) rec[a * 3 + c3] += J0[a] * J1[c3] + J0[6 + a] * J1[3 + c3];          // W_f = J_p^T J_l
        int u = 36;
        for (int a = 0; a < 6; ++a)
          for (int c6 = 0; c6 <= a; ++c6) rec[u++] += J0[a] * J0[c6] + J0[6 + a] * J0[6 + c6];              // U_f lower triangle
        for (int a = 0; a < 6; ++a) rec[57 + a] -= J0[a] * r[0] + J0[6 + a] * r[1];                         // b_p,f
        vis |= 1u << f;
      }
      if (bad) { sc.status[0] = MERR_POSE_NOT_CONNECTED; graph_error(g, GERR_INDEX); vis = 0u; }
      // V^+ in the preconditioned form: Veff^+ = P^-1 (P^-1 V P^-1)^+ P^-1,  P = diag(p_b)
      const double p[3] = {marg_precond(Vp[0]), marg_precond(Vp[3]), marg_precond(Vp[5])};
      const double Vs[6] = {Vp[0] / p[0] / p[0], Vp[1] / p[0] / p[1], Vp[2] / p[0] / p[2], Vp[3] / p[1] / p[1], Vp[4] / p[1] / p[2], Vp[5] / p[2] / p[2]};
      double ev[3], Qm[9];
      eig3_jacobi(Vs, ev, Qm);
      const double lmax = fmax(ev[0], fmax(ev[1], ev[2]));
      const double tol = eps * 3.0 * lmax;
      double Vi[9];
      for (int a = 0; a < 3; ++a)
        for (int c3 = 0; c3 < 3; ++c3) {
          double s = 0;
          for (int k = 0; k < 3; ++k) s += (ev[k] > tol) ? Qm[a * 3 + k] * Qm[c3 * 3 + k] / ev[k] : 0.0;
          Vi[a * 3 + c3] = s / p[a] / p[c3];
        }
      double y[3];
      for (int a = 0; a < 3; ++a) y[a] = Vi[a * 3] * bl[0] + Vi[a * 3 + 1] * bl[1] + Vi[a * 3 + 2] * bl[2];
      for (int k = 0; k < 9; ++k) sc.lmV[(size_t)j * 16 + k] = Vi[k];
      for (int k = 0; k < 3; ++k) sc.lmV[(size_t)j * 16 + 9 + k] = y[k];
      sc.lmvis[j] = vis;
      uint32_t m = vis;
      while (m) {
        const int f = __ffs((int)m) - 1;
        m &= m - 1;
        double* rec = sc.lmrec + ((size_t)j * K + f) * kMargRec;
        for (int a = 0; a < 6; ++a) {
          for (int c3 = 0; c3 < 3; ++c3) rec[18 + a * 3 + c3] = rec[a * 3] * Vi[c3] + rec[a * 3 + 1] * Vi[3 + c3] + rec[a * 3 + 2] * Vi[6 + c3];   // Z_f = W_f Veff^+
          rec[63 + a] = rec[a * 3] * y[0] + rec[a * 3 + 1] * y[1] + rec[a * 3 + 2] * y[2];                                                            // W_f y
        }
      }
    }
    __syncthreads();
    if constexpr (!kShard) { if (sc.status[0]) return; }
    // fixed-order reduction over the landmarks into the pose rows of H and b (sharded: into every rank's box)
    for (int i = tid; i < N * N; i += M_THREADS) {
      const int r = i / N, c = i % N;
      const int br = s_rowblk[r], bc = s_rowblk[c];
      if (sc.kind[br] != OKB_BLOCK_POSE || sc.kind[bc] != OKB_BLOCK_POSE) continue;
      const int fr = (int)sc.idx[br], fc = (int)sc.idx[bc], a = r - s_col[br], bb = c - s_col[bc];
      const uint32_t need = (1u << fr) | (1u << fc);
      double s = 0.0;
      for (int j = 0; j < n_lm; ++j) {
        if ((sc.lmvis[j] & need) != need) continue;
        const double* zr = sc.lmrec + ((size_t)j * K + fr) * kMargRec + 18 + a * 3;
        const double* wc = sc.lmrec + ((size_t)j * K + fc) * kMargRec + bb * 3;
        s -= zr[0] * wc[0] + zr[1] * wc[1] + zr[2] * wc[2];
        if (fr == fc) {
          const int hi = max(a, bb), lo = min(a, bb);
          s += sc.lmrec[((size_t)j * K + fr) * kMargRec + 36 + hi * (hi + 1) / 2 + lo];
        }
      }
      if constexpr (kShard) {
        const size_t o = kMargBoxHeader + (size_t)s_ia[r] * s_i[3] + s_ia[c];
        for (int q = 0; q < W.shard_world; ++q) shard_marg_box(W, q, mpar, W.shard_rank)[o] = s;
      } else {
        sc.H[i] += s;
      }
    }
    for (int r = tid; r < N; r += M_THREADS) {
      const int br = s_rowblk[r];
      if (sc.kind[br] != OKB_BLOCK_POSE) continue;
      const int fr = (int)sc.idx[br], a = r - s_col[br];
      double s = 0.0;
      for (int j = 0; j < n_lm; ++j) {
        if (!((sc.lmvis[j] >> fr) & 1u)) continue;
        const double* rec = sc.lmrec + ((size_t)j * K + fr) * kMargRec;
        s += rec[57 + a] - rec[63 + a];
      }
      if constexpr (kShard) {
        const size_t o = kMargBoxHeader + (size_t)s_i[3] * s_i[3] + s_ia[r];
        for (int q = 0; q < W.shard_world; ++q) shard_marg_box(W, q, mpar, W.shard_rank)[o] = s;
      } else {
        sc.b[r] += s;
      }
    }
    for (int j = tid; j < n_lm; j += M_THREADS) { const uint32_t l = sc.landmarks[j]; if ((int)l < g->L) sc.lmslot[l] = 0; }
    __syncthreads();
  }
exchange:
  if constexpr (kShard) {
    // Push the header (job fingerprint, this rank's phase 0-4 error word), release this rank's flag in every mailbox,
    // acquire the `world` flags in this rank's own; then every rank reads the same boxes.
    __syncthreads();
    const int world = W.shard_world, me = W.shard_rank;
    unsigned long long* ep = reinterpret_cast<unsigned long long*>(W.shard_mail[me] + kShardMargEpoch);
    const unsigned long long epoch = *ep + 1;
    const int par = (int)(epoch & 1ull);
    if (tid == 0) s_i[4] = 0;
    if (tid < world) {
      unsigned long long* hb = reinterpret_cast<unsigned long long*>(shard_marg_box(W, tid, par, me));
      hb[0] = s_task.fingerprint;
      hb[1] = (unsigned long long)(unsigned)sc.status[0];
      hb[2] = epoch;
    }
    __threadfence_system();
    __syncthreads();
    if (tid < world) {
      st_release_sys_u64(shard_flag(W, tid, kShardFlagsM, par, me), epoch);
      const unsigned long long t0 = globaltimer_ns();
      const unsigned long long* fl = shard_flag(W, me, kShardFlagsM, par, tid);
      while (ld_acquire_sys_u64(fl) < epoch)
        if (globaltimer_ns() - t0 > kShardTimeoutNs) { s_i[4] = MERR_SHARD_TIMEOUT; break; }
    }
    __syncthreads();
    int st = s_i[4];
    // a box pushed at another epoch: the ranks are out of step (a rank's earlier call never launched, or timed out)
    for (int q = 0; q < world && !st; ++q)
      if (__ldcg(reinterpret_cast<const unsigned long long*>(shard_marg_box(W, me, par, q)) + 2) != epoch) st = MERR_SHARD_TIMEOUT;
    if (!st) {
      const unsigned long long fp0 = __ldcg(reinterpret_cast<const unsigned long long*>(shard_marg_box(W, me, par, 0)));
      for (int q = 0; q < world && !st; ++q)
        if (__ldcg(reinterpret_cast<const unsigned long long*>(shard_marg_box(W, me, par, q))) != fp0) st = MERR_SHARD_JOB;
      for (int q = 0; q < world && !st; ++q) st = (int)__ldcg(reinterpret_cast<const unsigned long long*>(shard_marg_box(W, me, par, q)) + 1);
    }
    if (st) {       // every rank took the same decision from the same boxes: the previous prior stays everywhere
      if (tid == 0) { sc.status[0] = st; graph_error(g, GERR_SHARD_MARG); *ep = epoch; }
      return;
    }
    const int P = s_i[3];
    for (int i = tid; i < N * N; i += M_THREADS) {
      const int r = i / N, c = i % N;
      if (s_ia[r] < 0 || s_ia[c] < 0) continue;
      const size_t o = kMargBoxHeader + (size_t)s_ia[r] * P + s_ia[c];
      double s = 0.0;
      for (int q = 0; q < world; ++q) s += __ldcg(shard_marg_box(W, me, par, q) + o);
      sc.H[i] += s;
    }
    for (int r = tid; r < N; r += M_THREADS) {
      if (s_ia[r] < 0) continue;
      const size_t o = kMargBoxHeader + (size_t)P * P + s_ia[r];
      double s = 0.0;
      for (int q = 0; q < world; ++q) s += __ldcg(shard_marg_box(W, me, par, q) + o);
      sc.b[r] += s;
    }
    if (tid == 0) *ep = epoch;
    __syncthreads();
  }
  // ---------------- phase 5: dense blocks to marginalise
  if (tid == 0) {
    int na = 0, nb = 0;
    for (int r = 0; r < N; ++r) { if (sc.marg[s_rowblk[r]]) s_ib[nb++] = (short)r; else s_ia[na++] = (short)r; }
    s_i[1] = na; s_i[2] = nb;
  }
  __syncthreads();
  const int na = s_i[1], nb = s_i[2];
  if (na != J.n_keep) { if (tid == 0) { sc.status[0] = MERR_DIM; graph_error(g, GERR_DIMS); } return; }
  if (nb > 0) {
    // A = P_b^-1 sym(V) P_b^-1
    for (int i = tid; i < nb * nb; i += M_THREADS) {
      const int r = s_ib[i / nb], c = s_ib[i % nb];
      sc.A[i] = 0.5 * (sc.H[(size_t)r * N + c] + sc.H[(size_t)c * N + r]) / marg_precond(sc.H[(size_t)r * N + r]) / marg_precond(sc.H[(size_t)c * N + c]);
    }
    __syncthreads();
    const int sw = jacobi_eig(sc.A, sc.Q, nb, s_cs, s_pq, s_red);
    double lmax = -1e300;
    for (int k = tid; k < nb; k += M_THREADS) lmax = fmax(lmax, sc.A[(size_t)k * nb + k]);
    lmax = block_max(lmax, s_red);
    const double tol = eps * nb * lmax;
    if (tid == 0) { int rk = 0; for (int k = 0; k < nb; ++k) rk += sc.A[(size_t)k * nb + k] > tol; sc.status[2] = rk; sc.status[3] = sw; }
    // T = Veff^+ = P^-1 Q diag(1/lambda | 0) Q^T P^-1
    for (int i = tid; i < nb * nb; i += M_THREADS) {
      const int r = i / nb, c = i % nb;
      double s = 0;
      for (int k = 0; k < nb; ++k) { const double lam = sc.A[(size_t)k * nb + k]; if (lam > tol) s += sc.Q[(size_t)r * nb + k] * sc.Q[(size_t)c * nb + k] / lam; }
      sc.T[i] = s / marg_precond(sc.H[(size_t)s_ib[r] * N + s_ib[r]]) / marg_precond(sc.H[(size_t)s_ib[c] * N + s_ib[c]]);
    }
    __syncthreads();
    // M = W Veff^+  (na x nb) into A
    for (int i = tid; i < na * nb; i += M_THREADS) {
      const int r = s_ia[i / nb], c = i % nb;
      double s = 0;
      for (int k = 0; k < nb; ++k) s += sc.H[(size_t)r * N + s_ib[k]] * sc.T[(size_t)k * nb + c];
      sc.A[i] = s;
    }
    __syncthreads();
    for (int i = tid; i < na * na; i += M_THREADS) {
      const int r = i / na, c = i % na;
      double s = 0;
      for (int k = 0; k < nb; ++k) s += sc.A[(size_t)r * nb + k] * sc.H[(size_t)s_ia[c] * N + s_ib[k]];
      sc.Hn[i] = sc.H[(size_t)s_ia[r] * N + s_ia[c]] - s;
    }
    for (int r = tid; r < na; r += M_THREADS) {
      double s = 0;
      for (int k = 0; k < nb; ++k) s += sc.A[(size_t)r * nb + k] * sc.b[s_ib[k]];
      sc.bn[r] = sc.b[s_ia[r]] - s;
    }
  } else {
    for (int i = tid; i < na * na; i += M_THREADS) sc.Hn[i] = sc.H[(size_t)s_ia[i / na] * N + s_ia[i % na]];
    for (int r = tid; r < na; r += M_THREADS) sc.bn[r] = sc.b[s_ia[r]];
  }
  __syncthreads();
  // ---------------- phase 6: updateErrorComputation on (Hn, bn), n = na
  const int n = na;
  for (int i = tid; i < n * n; i += M_THREADS) {
    const int r = i / n, c = i % n;
    sc.A[i] = 0.5 * (sc.Hn[i] + sc.Hn[(size_t)c * n + r]) / marg_precond(sc.Hn[(size_t)r * n + r]) / marg_precond(sc.Hn[(size_t)c * n + c]);
  }
  __syncthreads();
  const int sw6 = jacobi_eig(sc.A, sc.Q, n, s_cs, s_pq, s_red);
  if (tid == 0) sc.status[3] = max(sc.status[3], sw6);       // 40: one of the two decompositions did not converge
  double lmax = -1e300;
  for (int k = tid; k < n; k += M_THREADS) lmax = fmax(lmax, sc.A[(size_t)k * n + k]);
  lmax = (n > 0) ? block_max(lmax, s_red) : 0.0;
  const double tol = eps * n * lmax;
  if (tid == 0) { int rk = 0; for (int k = 0; k < n; ++k) rk += sc.A[(size_t)k * n + k] > tol; sc.status[1] = rk; }
  // the new prior replaces the old one in the arena
  for (int i = tid; i < n * n; i += M_THREADS) {
    const int k = i / n, c = i % n;                 // residual row k <- eigenpair k
    const double lam = sc.A[(size_t)k * n + k];
    W.marg_J[i] = (lam > tol) ? sqrt(lam) * sc.Q[(size_t)c * n + k] * marg_precond(sc.Hn[(size_t)c * n + c]) : 0.0;
    W.marg_Hs[i] = sc.Hn[i];
  }
  for (int k = tid; k < n; k += M_THREADS) {
    const double lam = sc.A[(size_t)k * n + k];
    double acc = 0.0;
    for (int i = 0; i < n; ++i) acc += sc.Q[(size_t)i * n + k] / marg_precond(sc.Hn[(size_t)i * n + i]) * sc.bn[i];
    W.marg_e0[k] = (lam > tol) ? -sqrt(1.0 / lam) * acc : 0.0;
    W.marg_b0[k] = sc.bn[k];
  }
  __syncthreads();
  for (int e = tid; e < n * n; e += M_THREADS) {      // H0 = J^T J (fixed summation order), as CMD_SET_MARG does
    const int i = e / n, j = e % n;
    if (j > i) continue;
    double s = 0;
    for (int r = 0; r < n; ++r) s += W.marg_J[(size_t)r * n + i] * W.marg_J[(size_t)r * n + j];
    W.marg_H0[(size_t)i * n + j] = s; W.marg_H0[(size_t)j * n + i] = s;
  }
  if (tid == 0) {
    int nbk = 0, col = 0, xo = 0;
    for (int b = 0; b < NB; ++b) {
      if (sc.marg[b]) continue;
      const int kind = sc.kind[b];
      W.marg_kind[nbk] = kind; W.marg_idx[nbk] = sc.idx[b]; W.marg_col[nbk] = col; W.marg_off[nbk] = xo;
      const int w = (kind == OKB_BLOCK_SPEED_BIAS) ? 9 : 7;
      for (int k = 0; k < w; ++k) W.marg_x0[xo + k] = sc.xlin[9 * b + k];
      col += s_dim[b]; xo += w; ++nbk;
    }
    g->marg_n = n; g->marg_nb = nbk; g->marg_xdim = xo;
  }
}
#pragma nv_diag_default 177

// CMD_REMOVE_SB of the graph interpreter lives in okb_graph.cuh; the download of the prior for tests / the host shim:
__global__ void k_marg_export(const WinDev* __restrict__ wins, int win, double* out /* header 8 | kind nb | idx nb | x0 | J | e0 | H | b0 */, int cap) {
  const WinDev& W = wins[win];
  const GraphState* g = &W.st->g;
  const int n = g->marg_n, nb = g->marg_nb, xd = g->marg_xdim;
  const int need = 8 + 2 * nb + xd + 2 * n * n + 2 * n;
  if (threadIdx.x == 0) { out[0] = n; out[1] = nb; out[2] = xd; out[3] = need; }
  if (need > cap) return;
  double* o = out + 8;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) { o[i] = W.marg_kind[i]; o[nb + i] = W.marg_idx[i]; }
  o += 2 * nb;
  for (int i = threadIdx.x; i < xd; i += blockDim.x) o[i] = W.marg_x0[i];
  o += xd;
  for (int i = threadIdx.x; i < n * n; i += blockDim.x) { o[i] = W.marg_J[i]; o[n * n + n + i] = W.marg_Hs[i]; }
  for (int i = threadIdx.x; i < n; i += blockDim.x) { o[n * n + i] = W.marg_e0[i]; o[2 * n * n + n + i] = W.marg_b0[i]; }
}

}  // namespace okb
