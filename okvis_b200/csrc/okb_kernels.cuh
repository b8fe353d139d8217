// Kernels of the batched dogleg/Schur solver (sm_90a).  One solver round is
//   k_imu (side stream) || k_landmarks -> k_schur -> k_reduce_partials   (okb_kernels_lm.cuh), then
//   k_solve ("S"): one CTA of 256 threads per window, two CTAs per SM.  IMU / prior / marginalisation terms
//       assembled directly in the shared-memory system buffer (packed lower triangle), step acceptance
//       (Ceres 1.9 trust-region logic), blocked Cholesky with the right-hand side as an appended row,
//       backward substitution, landmark back-substitution, traditional dogleg step, candidate state and
//       the (frame, camera) contexts of the next linearisation.
// plus k_imu (IMU_G lanes per IMU term), k_zero / k_prepare (upload epilogue on the transfer stream), k_reset.
#pragma once
#include "okb_chol.cuh"
#include "okb_estimator.cuh"
#include "okb_kernels_lm.cuh"

namespace okb {

constexpr int S_THREADS = 256;    // two k_solve CTAs per SM (packed system: ~112 KB of shared memory each)
constexpr int S_WARPS = S_THREADS / 32;
constexpr int kImuOut = 932;     // doubles per IMU term produced by k_imu: H30 | g30 | cost | pad
static_assert(OKB_IMU_TERM_OUT == 900 + 30 + 1 && OKB_IMU_TERM_OUT < kImuOut, "okb_debug_imu_terms copies H30 | g30 | cost");

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// block-wide sum; `red` is shared scratch of >= 32 doubles; result valid in all threads
__device__ __forceinline__ double block_sum(double v, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0;
  for (int i = 0; i < nw; ++i) s += red[i];   // fixed order: deterministic
  return s;
}
__device__ __forceinline__ double block_max(double v, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = red[0];
  for (int i = 1; i < nw; ++i) s = fmax(s, red[i]);
  return s;
}

// ------------------------------------------------------------------------------------------------
// Kernel I: IMU_G lanes per IMU term: residual, the four minimal Jacobians, and the term's contribution
// [J0 J1 J2 J3]^T [J0 J1 J2 J3] (30x30), J^T r (30), cost.  Re-preintegrates exactly when the reference's Evaluate()
// would.  A term's shared scratch is kImuScratch doubles (7.3 KB) and the kernel is held to 168 registers, so that
// 12 CTAs (24 terms) fit on an SM.
// ------------------------------------------------------------------------------------------------
constexpr int IMU_G = 16;      // lanes per IMU term: 32 / IMU_G terms per warp
__host__ __device__ inline size_t smemI_bytes() { return (size_t)(32 / IMU_G) * kImuScratch * sizeof(double); }
__global__ void __launch_bounds__(32, 12) k_imu(const WinDev* __restrict__ wins, const int32_t* __restrict__ win_slots) {
  const WinDev& W = wins[win_slots[blockIdx.y]];
  if (W.st->done) return;
  const int grp = (threadIdx.x & 31) / IMU_G;
  const int t = blockIdx.x * (32 / IMU_G) + grp;
  if (t >= W.n_imu) return;
  extern __shared__ __align__(16) double imu_buf[];
  GroupCtx<IMU_G> cx;
  const ImuScratch sc = imu_scratch(imu_buf + (size_t)grp * kImuScratch);
  double* SF = sc.SF;
  double* r15 = sc.r15;
  const okb_imu_term& T = W.imu_terms[t];
  imu_evaluate(cx, W.samples + T.sample_offset, (int)T.sample_count, W.imu_params, T.t0_ns, T.t1_ns, W.pose_c + 7 * T.pose0,
               W.sb_c + 9 * T.sb0, W.pose_c + 7 * T.pose1, W.sb_c + 9 * T.sb1, W.imu_cache + t, sc.wk, sc.F01, (double*)nullptr,
               r15, SF);
  double* out = W.imu_out + (size_t)t * kImuOut;
  const int lane = cx.lane();
  for (int e = lane; e < 900; e += IMU_G) {
    const int a = e / 30, b = e % 30;
    double s = 0;
#pragma unroll
    for (int k = 0; k < 15; ++k) s += SF[k * 30 + a] * SF[k * 30 + b];
    out[e] = s;
  }
  for (int e = lane; e < 30; e += IMU_G) {
    double s = 0;
#pragma unroll
    for (int k = 0; k < 15; ++k) s += SF[k * 30 + e] * r15[k];
    out[900 + e] = s;
  }
  if (lane == 0) {
    double c = 0;
    for (int k = 0; k < 15; ++k) c += r15[k] * r15[k];
    out[930] = 0.5 * c;
  }
}

// ------------------------------------------------------------------------------------------------
// Kernel S
// ------------------------------------------------------------------------------------------------
struct SShared {
  double red[64];
  // broadcast scalars
  double cand_cost, cost_lm, stepn2_lm, cost_dense;
  int adopt, terminate, commit_only, fail, spec, chol_flag;
  int shard_fault, chain_ok;
  double x2[8];         // landmark-sharded windows: step scalars combined over the ranks
};

// Landmark-sharded window, second exchange of a round (inside k_solve): the landmark parts of the dogleg scalars
// [N2, GU, G2, VHV, ||x||^2, max|g|, #non-finite, elapsed+last (time-limit callback)] of every rank.  Each rank stores
// its 8 doubles into slot [parity][rank] of every mailbox and releases the matching flag; then it acquires the
// `world` flags of its own mailbox and combines the slots in rank order (sum, max for v[5], rank 0's clock for v[7]):
// every rank obtains the same bits.  Called by all threads of the CTA; returns 0 on a time-out.
__device__ inline int shard_exchange_scalars(const WinDev& W, SolverState* st, SShared* sh, double* v) {
  const int tid = threadIdx.x, world = W.shard_world, me = W.shard_rank;
  const unsigned long long epoch = st->shard_epoch;        // set by the prologue of this round
  const int par = (int)(epoch & 1ull);
  if (tid == 0) sh->shard_fault = 0;
  __syncthreads();
  if (tid < world) {
    double* box = reinterpret_cast<double*>(W.shard_mail[tid] + kShardScalars) + ((size_t)par * kMaxShard + me) * 16;
#pragma unroll
    for (int k = 0; k < 8; ++k) box[k] = v[k];
    __threadfence_system();
    st_release_sys_u64(shard_flag(W, tid, kShardFlags2, par, me), epoch);
    const unsigned long long t0 = globaltimer_ns();
    const unsigned long long* fl = shard_flag(W, me, kShardFlags2, par, tid);
    while (ld_acquire_sys_u64(fl) < epoch)
      if (globaltimer_ns() - t0 > kShardTimeoutNs) { sh->shard_fault = 1; break; }
  }
  __syncthreads();
  if (sh->shard_fault) return 0;
  if (tid < 8) {
    double acc = 0.0;
    for (int r = 0; r < world; ++r) {
      const double x = __ldcg(reinterpret_cast<const double*>(W.shard_mail[me] + kShardScalars) + ((size_t)par * kMaxShard + r) * 16 + tid);
      if (tid == 5) acc = (r == 0) ? x : fmax(acc, x);
      else if (tid == 7) acc = (r == 0) ? x : acc;
      else acc += x;
    }
    sh->x2[tid] = acc;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 8; ++k) v[k] = sh->x2[k];
  return 1;
}

// r = S e etc. are tiny; one warp handles all priors.
// The dense Hessian lives in packed lower-triangular storage: contributions to the upper triangle are dropped
// (their mirror images are always added as well).
__device__ __forceinline__ void hd_add(double* Hd, int r, int c, double v) {
  if (r >= c) Hd[tri_row(r) + c] += v;
}

__device__ void dense_priors(const WinDev& W, double* Hd, double* gd, double* cost_out) {
  const int lane = threadIdx.x & 31;
  double cost = 0.0;
  for (int i = 0; i < W.n_pp; ++i) {
    const okb_pose_prior& pr = W.pp[i];
    double r[6], J[36];
    pose_error(pr.meas, pr.sqrt_info, W.pose_c + 7 * pr.pose_idx, r, J);   // replicated per lane (tiny)
    const int o = 6 * pr.pose_idx;
    for (int e = lane; e < 36; e += 32) {
      const int a = e / 6, b = e % 6;
      double s = 0;
      for (int k = 0; k < 6; ++k) s += J[k * 6 + a] * J[k * 6 + b];
      hd_add(Hd, (o + a), o + b, s);
    }
    if (lane < 6) {
      double s = 0;
      for (int k = 0; k < 6; ++k) s += J[k * 6 + lane] * r[k];
      gd[o + lane] += s;
    }
    for (int k = 0; k < 6; ++k) cost += 0.5 * r[k] * r[k];
    __syncwarp();
  }
  for (int i = 0; i < W.n_sbp; ++i) {
    const okb_sb_prior& pr = W.sbp[i];
    const double* x = W.sb_c + 9 * pr.sb_idx;
    double e9[9], r[9];
    for (int k = 0; k < 9; ++k) e9[k] = pr.meas[k] - x[k];
    for (int a = 0; a < 9; ++a) {
      double s = 0;
      for (int k = 0; k < 9; ++k) s += pr.sqrt_info[a * 9 + k] * e9[k];
      r[a] = s;
    }
    const int o = W.dc + 9 * pr.sb_idx;
    for (int e = lane; e < 81; e += 32) {   // J = -S  => J^T J = S^T S
      const int a = e / 9, b = e % 9;
      double s = 0;
      for (int k = 0; k < 9; ++k) s += pr.sqrt_info[k * 9 + a] * pr.sqrt_info[k * 9 + b];
      hd_add(Hd, (o + a), o + b, s);
    }
    if (lane < 9) {
      double s = 0;
      for (int k = 0; k < 9; ++k) s -= pr.sqrt_info[k * 9 + lane] * r[k];
      gd[o + lane] += s;
    }
    for (int k = 0; k < 9; ++k) cost += 0.5 * r[k] * r[k];
    __syncwarp();
  }
  *cost_out = cost;
}

// solve_mode: 1 = the packed reduced system lives in shared memory (d <= ~150); 2 = system in global memory, the
// speed/bias chain band and the dc x dc pose system (after the chain elimination) in shared memory; 0 = system and
// pose system in global memory, only the chain band in shared memory.
__host__ __device__ inline size_t smemS_bytes(int d, int dc, int K, int n_marg, int n_imu, int solve_mode) {
  size_t b = sizeof(SShared);
  b = (b + 15) & ~(size_t)15;
  b += (size_t)8 * d * sizeof(double);                     // gd, Ed, ud, rhs, vd, tmp, delta, colk
  b += (size_t)K * 4 * sizeof(double);                     // committed frame translations
  b += (size_t)3 * (((n_marg > 0 ? n_marg : 1) + 1) & ~1) * sizeof(double);   // marg: dchi, e, Jte (even length each: 16-byte loads stay inside)
  b = (b + 31) & ~(size_t)31;
  b += (size_t)CH_NB * ((d + 1 + 3) & ~3) * sizeof(double);  // Cholesky panel (k-major)
  if (solve_mode == 1) b += tri_row(d + 1) * sizeof(double) + 16;        // the reduced system (packed lower triangle) + appended rhs row
  else {
    b += (size_t)(d - dc) * 18 * sizeof(double) + 16;                    // chain band
    if (solve_mode == 2) b += tri_row(dc + 1) * sizeof(double);          // pose system + appended rhs row
  }
  return b;
}

// NT = 256: two CTAs per SM (batched throughput); NT = 512: one CTA per SM with twice the threads for small batches
// (latency: the parallel phases -- assembly, trailing updates, landmark back-substitution -- run twice as wide).
template <int NT>
__global__ void __launch_bounds__(NT, NT == 256 ? 2 : 1) k_solve(const WinDev* __restrict__ wins, const int32_t* __restrict__ win_slots, okb_solve_options opt,
                                                        int solve_mode) {
  const int chol_in_smem = (solve_mode == 1);
  const WinDev& W = wins[win_slots[blockIdx.x]];
  SolverState* st = W.st;
  if (st->done) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int K = W.K, d = W.d, dc = W.dc, dcp = W.dcp, L = W.L;

  extern __shared__ __align__(16) unsigned char smem_raw[];
  size_t off = 0;
  SShared* sh = reinterpret_cast<SShared*>(smem_raw); off += sizeof(SShared);
  off = (off + 15) & ~(size_t)15;
  double* s_g = reinterpret_cast<double*>(smem_raw + off); off += (size_t)d * 8;
  double* s_E = reinterpret_cast<double*>(smem_raw + off); off += (size_t)d * 8;
  double* s_u = reinterpret_cast<double*>(smem_raw + off); off += (size_t)d * 8;
  double* s_rhs = reinterpret_cast<double*>(smem_raw + off); off += (size_t)d * 8;
  double* s_v = reinterpret_cast<double*>(smem_raw + off); off += (size_t)d * 8;
  double* s_tmp = reinterpret_cast<double*>(smem_raw + off); off += (size_t)d * 8;
  double* s_delta = reinterpret_cast<double*>(smem_raw + off); off += (size_t)d * 8;
  double* s_col = reinterpret_cast<double*>(smem_raw + off); off += (size_t)d * 8;
  double* s_tws = reinterpret_cast<double*>(smem_raw + off); off += (size_t)K * 4 * 8;
  const int nm = ((W.marg_n > 0 ? W.marg_n : 1) + 1) & ~1;     // even: the compiler reads these vectors two doubles at a time
  double* s_dchi = reinterpret_cast<double*>(smem_raw + off); off += (size_t)nm * 8;
  double* s_me = reinterpret_cast<double*>(smem_raw + off); off += (size_t)nm * 8;
  double* s_mJte = reinterpret_cast<double*>(smem_raw + off); off += (size_t)nm * 8;
  const int ld_p = (d + 1 + 3) & ~3;
  off = (off + 31) & ~(size_t)31;
  double* s_panel = reinterpret_cast<double*>(smem_raw + off); off += (size_t)CH_NB * ld_p * 8;
  double* s_big = reinterpret_cast<double*>(smem_raw + off);   // the reduced system (when it fits)

  unsigned long long t_ph = globaltimer_ns();
#define PHASE_MARK(i) do { if (tid == 0) { const unsigned long long n_ = globaltimer_ns(); st->phase_ns[i] += n_ - t_ph; t_ph = n_; } } while (0)
  const int mode = st->mode;
  const int spec = st->cur ^ 1;
  double* gd = W.gd[spec];

  // ================= phase 1: dense terms at the candidate =================
  // The dense Hessian is assembled directly in the shared-memory buffer that later holds the reduced system (packed
  // lower triangle; an appended row carries the right-hand side through the factorisation); windows whose system
  // does not fit keep it in global memory.
  double* Hd = chol_in_smem ? s_big : W.Hd;
  for (int i = tid; i < (int)tri_row(d); i += NT) Hd[i] = 0.0;
  for (int i = tid; i < d; i += NT) gd[i] = 0.0;
  __syncthreads();
  double cost_dense_local = 0.0;   // accumulated by thread 0
  // IMU terms were evaluated by k_imu; add their 30x30 blocks.  Terms that form a chain over consecutive frames
  // (term t ends where term t+1 starts, indices strictly increasing -- what Estimator::addStates builds) are added in
  // two passes, even terms then odd terms: terms of equal parity touch disjoint blocks.  Anything else goes term by term.
  bool imu_chain = true;
  for (int t = 0; t < W.n_imu; ++t) {
    const okb_imu_term& T = W.imu_terms[t];
    if (!(T.pose1 > T.pose0 && T.sb1 > T.sb0)) imu_chain = false;
    if (t + 1 < W.n_imu && (W.imu_terms[t + 1].pose0 < T.pose1 || W.imu_terms[t + 1].sb0 < T.sb1)) imu_chain = false;
  }
  const int n_pass = imu_chain ? min(2, W.n_imu) : W.n_imu;
  for (int pass = 0; pass < n_pass; ++pass) {
    const int t_stride = imu_chain ? 2 : 1;
    const int n_in_pass = imu_chain ? (W.n_imu - pass + 1) / 2 : 1;
    for (int ee = tid; ee < n_in_pass * 931; ee += NT) {
      const int t = pass + t_stride * (ee / 931), e = ee % 931;
      const okb_imu_term& T = W.imu_terms[t];
      const double* out = W.imu_out + (size_t)t * kImuOut;
      if (e < 900) {
        const int a = e / 30, b = e % 30;
        const int ba = (a < 6) ? 0 : (a < 15) ? 1 : (a < 21) ? 2 : 3;
        const int bb = (b < 6) ? 0 : (b < 15) ? 1 : (b < 21) ? 2 : 3;
        const int la = a - ((ba == 0) ? 0 : (ba == 1) ? 6 : (ba == 2) ? 15 : 21);
        const int lb = b - ((bb == 0) ? 0 : (bb == 1) ? 6 : (bb == 2) ? 15 : 21);
        const int oa = (ba == 0) ? 6 * (int)T.pose0 : (ba == 1) ? dc + 9 * (int)T.sb0 : (ba == 2) ? 6 * (int)T.pose1 : dc + 9 * (int)T.sb1;
        const int ob = (bb == 0) ? 6 * (int)T.pose0 : (bb == 1) ? dc + 9 * (int)T.sb0 : (bb == 2) ? 6 * (int)T.pose1 : dc + 9 * (int)T.sb1;
        hd_add(Hd, oa + la, ob + lb, out[e]);
      } else if (e < 930) {
        const int a = e - 900;
        const int ba = (a < 6) ? 0 : (a < 15) ? 1 : (a < 21) ? 2 : 3;
        const int la = a - ((ba == 0) ? 0 : (ba == 1) ? 6 : (ba == 2) ? 15 : 21);
        const int oa = (ba == 0) ? 6 * (int)T.pose0 : (ba == 1) ? dc + 9 * (int)T.sb0 : (ba == 2) ? 6 * (int)T.pose1 : dc + 9 * (int)T.sb1;
        gd[oa + la] += out[e];
      }
    }
    __syncthreads();
  }
  if (tid == 0) for (int t = 0; t < W.n_imu; ++t) cost_dense_local += W.imu_out[(size_t)t * kImuOut + 930];
  // priors (warp 0)
  if (warp == 0) {
    double c = 0;
    dense_priors(W, Hd, gd, &c);
    if (lane == 0) cost_dense_local += c;
  }
  __syncthreads();
  // marginalisation prior
  if (W.marg_n > 0) {
    const int n = W.marg_n;
    // Delta chi
    for (int b = tid; b < W.marg_nb; b += NT) {
      const int kind = W.marg_kind[b], col = W.marg_col[b], xo = W.marg_off[b];
      if (col < 0) continue;
      if (kind == OKB_BLOCK_SPEED_BIAS) {
        const double* x = W.sb_c + 9 * W.marg_idx[b];
        for (int k = 0; k < 9; ++k) s_dchi[col + k] = x[k] - W.marg_x0[xo + k];
      } else {
        const double* x = (kind == OKB_BLOCK_POSE) ? W.pose_c + 7 * W.marg_idx[b] : W.ext + 7 * W.marg_idx[b];
        pose_minus(W.marg_x0 + xo, x, s_dchi + col);
      }
    }
    __syncthreads();
    for (int r0 = tid; r0 < n; r0 += NT) {
      double s = W.marg_e0[r0];
      for (int c = 0; c < n; ++c) s += W.marg_J[(size_t)r0 * n + c] * s_dchi[c];
      s_me[r0] = s;
    }
    __syncthreads();
    for (int c = tid; c < n; c += NT) {   // J^T e
      double s = 0;
      for (int r0 = 0; r0 < n; ++r0) s += W.marg_J[(size_t)r0 * n + c] * s_me[r0];
      s_mJte[c] = s;
    }
    __syncthreads();
    // H_eff = B^T H0 B, g_eff = B^T J^T e, B = blockdiag(I3, Brot) for poses, I9 for speed/bias.
    // Work block-pair by block-pair; each thread computes entries of one (bi,bj) pair.
    for (int bp = 0; bp < W.marg_nb * W.marg_nb; ++bp) {
      const int bi = bp / W.marg_nb, bj = bp % W.marg_nb;
      const int ci = W.marg_col[bi], cj = W.marg_col[bj];
      if (ci < 0 || cj < 0) continue;
      const int ki = W.marg_kind[bi], kj = W.marg_kind[bj];
      if (ki == OKB_BLOCK_EXTRINSICS || kj == OKB_BLOCK_EXTRINSICS) continue;  // fixed extrinsics only (v1)
      const int mi = (ki == OKB_BLOCK_SPEED_BIAS) ? 9 : 6, mj = (kj == OKB_BLOCK_SPEED_BIAS) ? 9 : 6;
      const int oi = (ki == OKB_BLOCK_POSE) ? 6 * (int)W.marg_idx[bi] : dc + 9 * (int)W.marg_idx[bi];
      const int oj = (kj == OKB_BLOCK_POSE) ? 6 * (int)W.marg_idx[bj] : dc + 9 * (int)W.marg_idx[bj];
      double Bi[9], Bj[9];
      if (ki == OKB_BLOCK_POSE) marg_pose_rot_block(W.marg_x0 + W.marg_off[bi], W.pose_c + 7 * W.marg_idx[bi], Bi);
      if (kj == OKB_BLOCK_POSE) marg_pose_rot_block(W.marg_x0 + W.marg_off[bj], W.pose_c + 7 * W.marg_idx[bj], Bj);
      for (int e = tid; e < mi * mj; e += NT) {
        const int a = e / mj, b = e % mj;
        // (B_i^T H0_ij B_j)[a][b]
        double s = 0;
        const bool ra = (ki == OKB_BLOCK_POSE && a >= 3), rb = (kj == OKB_BLOCK_POSE && b >= 3);
        if (!ra && !rb) s = W.marg_H0[(size_t)(ci + a) * n + cj + b];
        else if (ra && !rb) { for (int k = 0; k < 3; ++k) s += Bi[k * 3 + (a - 3)] * W.marg_H0[(size_t)(ci + 3 + k) * n + cj + b]; }
        else if (!ra && rb) { for (int k = 0; k < 3; ++k) s += W.marg_H0[(size_t)(ci + a) * n + cj + 3 + k] * Bj[k * 3 + (b - 3)]; }
        else {
          for (int k = 0; k < 3; ++k)
            for (int k2 = 0; k2 < 3; ++k2) s += Bi[k * 3 + (a - 3)] * W.marg_H0[(size_t)(ci + 3 + k) * n + cj + 3 + k2] * Bj[k2 * 3 + (b - 3)];
        }
        hd_add(Hd, (oi + a), oj + b, s);
      }
      if (bi == bj) {
        for (int a = tid; a < mi; a += NT) {
          double s = 0;
          if (ki == OKB_BLOCK_POSE && a >= 3) { for (int k = 0; k < 3; ++k) s += Bi[k * 3 + (a - 3)] * s_mJte[ci + 3 + k]; }
          else s = s_mJte[ci + a];
          gd[oi + a] += s;
        }
      }
      __syncthreads();
    }
    if (tid == 0) {
      double c = 0;
      for (int r0 = 0; r0 < n; ++r0) c += s_me[r0] * s_me[r0];
      cost_dense_local += 0.5 * c;
    }
  }
  const double cost_dense = block_sum(cost_dense_local, sh->red);

  PHASE_MARK(0);
  // ================= phase 2: gather the landmark-kernel partials =================
  const bool sharded = W.shard_world > 1;
  if (sharded) {
    // receive half of the all-reduce: wait for every rank's box of this round (flags live in THIS rank's memory),
    // add the boxes in rank order into the local partials.  The dense terms above did not depend on them.
    const unsigned long long epoch = st->shard_epoch + 1;
    const int par = (int)(epoch & 1ull), world = W.shard_world, me = W.shard_rank;
    const unsigned long long t_w0 = globaltimer_ns();
    if (tid == 0) sh->shard_fault = 0;
    __syncthreads();
    if (tid < world) {
      const unsigned long long* fl = shard_flag(W, me, kShardFlags1, par, tid);
      while (ld_acquire_sys_u64(fl) < epoch)
        if (globaltimer_ns() - t_w0 > kShardTimeoutNs) { sh->shard_fault = 1; break; }
    }
    __syncthreads();
    if (sh->shard_fault) {
      if (tid == 0) { st->shard_fault = 1; st->termination = OKB_TERM_FAILURE; st->done = 1; st->shard_epoch = epoch; }
      return;
    }
    const int nA = dcp * dcp, nH = K * kPartH;
    for (int i = tid; i < nA + nH + 1; i += NT) {
      double s = 0.0;
      for (int r = 0; r < world; ++r) s += __ldcg(shard_box(W, me, par, r) + i);
      if (i < nA) W.partA[i] = s;
      else if (i < nA + nH) W.partH[i - nA] = s;          // record (cx = 0, frame f): the gather below runs with n_cx = 1
      else st->numeric_fail = (s > 0.0) ? 1 : 0;
    }
    __syncthreads();
    if (tid == 0) { st->shard_epoch = epoch; st->shard_wait_ns += globaltimer_ns() - t_w0; st->shard_rounds += 1; }
  }
  const int n_cx = sharded ? 1 : (L + L1_THREADS - 1) / L1_THREADS;
  if (warp == 0) {     // cost and step-norm sums of the landmark kernels: lane-strided partials, fixed shuffle tree
    double c_ = 0.0, s_ = 0.0;
    for (int i = lane; i < n_cx * K; i += 32) {
      c_ += W.partH[(size_t)i * kPartH + 27];
      s_ += W.partH[(size_t)i * kPartH + 28];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { c_ += __shfl_xor_sync(0xffffffffu, c_, o); s_ += __shfl_xor_sync(0xffffffffu, s_, o); }
    if (lane == 0) { sh->cost_lm = c_; sh->stepn2_lm = s_; }
  }
  // H_pp / g_p block contributions
  for (int i = tid; i < 27 * K; i += NT) {
    const int e = i / K, f = i % K, o = 6 * f;
    double s = 0;
    for (int c = 0; c < n_cx; ++c) s += W.partH[((size_t)c * K + f) * kPartH + e];
    if (e < 6) {          // H_tt symmetric packed
      const int a = (e < 3) ? 0 : (e < 5) ? 1 : 2;
      const int b = (e < 3) ? e : (e < 5) ? e - 2 : 2;
      hd_add(Hd, (o + a), o + b, s);
      if (a != b) hd_add(Hd, (o + b), o + a, s);
    } else if (e < 15) {  // H_tr 3x3
      const int a = (e - 6) / 3, b = (e - 6) % 3;
      hd_add(Hd, (o + a), o + 3 + b, s);
      hd_add(Hd, (o + 3 + b), o + a, s);
    } else if (e < 21) {  // H_rr symmetric packed
      const int q = e - 15;
      const int a = (q < 3) ? 0 : (q < 5) ? 1 : 2;
      const int b = (q < 3) ? q : (q < 5) ? q - 2 : 2;
      hd_add(Hd, (o + 3 + a), o + 3 + b, s);
      if (a != b) hd_add(Hd, (o + 3 + b), o + 3 + a, s);
    } else {              // g_p
      gd[o + (e - 21)] += s;
    }
  }
  __syncthreads();
  PHASE_MARK(1);
  // ================= phase 3: judge =================
  if (tid == 0) {
    const unsigned long long now = globaltimer_ns();
    sh->adopt = 0; sh->terminate = 0; sh->commit_only = 0; sh->fail = 0;
    const double cost_lm = sh->cost_lm, stepn2_lm = sh->stepn2_lm;
    const double cand_cost = cost_lm + cost_dense;
    sh->cand_cost = cand_cost;
    if (mode == MODE_INIT) {
      st->t_start_ns = now; st->t_iter_begin_ns = now; st->t_last_iter_ns = 0;
      st->cost = cand_cost; st->initial_cost = cand_cost;
      sh->adopt = 1;
    } else if (mode == MODE_REBUILD) {
      st->cost = cand_cost;
      sh->adopt = 1;
    } else {
      const double step_norm = sqrt(stepn2_lm + st->cand_step_norm2_dense);
      const double cost_change = st->cost - cand_cost;
      if (step_norm <= kParameterTolerance * (sqrt(st->x_norm2) + kParameterTolerance)) {
        st->termination = OKB_TERM_PARAMETER_TOL; sh->terminate = 1;
      } else if (fabs(cost_change) < kFunctionTolerance * st->cost) {
        st->termination = OKB_TERM_FUNCTION_TOL; sh->terminate = 1;
      } else {
        const double rel = cost_change / st->model_cost_change;
        if (rel > kMinRelativeDecrease) {
          st->num_successful += 1;
          if (rel < 0.25) st->radius *= 0.5;
          if (rel > 0.75) st->radius = fmax(st->radius, 3.0 * st->dogleg_step_norm);
          st->mu = fmax(kMinMu, 2.0 * st->mu / kMuIncrease);
          st->reuse = 0;
          st->cost = cand_cost;
          sh->adopt = 1;
        } else {
          st->radius *= 0.5;
          st->reuse = 1;
        }
        if (st->radius < kMinRadius) {
          st->termination = OKB_TERM_MIN_RADIUS;
          if (sh->adopt) sh->commit_only = 1; else sh->terminate = 1;
        }
      }
      st->t_last_iter_ns = now - st->t_iter_begin_ns;
    }
    if (st->numeric_fail && sh->adopt) sh->fail = 1;
    st->numeric_fail = 0;
  }
  __syncthreads();
  if (sh->terminate) {
    if (tid == 0) {
      int redo = 0;
      for (int t = 0; t < W.n_imu; ++t) redo += W.imu_cache[t].redo_count;
      st->imu_redo_final = redo - st->imu_redo;
      st->done = 1;
      st->solve_time_s = 1e-9 * (double)(globaltimer_ns() - st->t_start_ns);
    }
    return;
  }
  const int adopt = sh->adopt;
  int cur = st->cur;
  double xs[8] = {0, 0, 0, 0, 0, 0, 0, 0};     // N2, GU, G2, VHV, ||x||^2, max|g|, #non-finite, (sharded: rank clock)
  int chol_fail_adopt = 0;
  const bool dense_owner = !sharded || W.shard_rank == 0;   // sharded: the dense blocks are counted once

  // ================= phase 4: adopt the speculative linearisation =================
  if (adopt) {
    // commit dense parameters
    for (int i = tid; i < 7 * K; i += NT) W.pose[i] = W.pose_c[i];
    for (int i = tid; i < 9 * W.NSB; i += NT) W.sb[i] = W.sb_c[i];
    cur = spec;
    __syncthreads();
    if (tid == 0) st->cur = cur;
    for (int f = tid; f < K; f += NT) {
      s_tws[4 * f] = W.pose[7 * f]; s_tws[4 * f + 1] = W.pose[7 * f + 1]; s_tws[4 * f + 2] = W.pose[7 * f + 2];
    }
    // metric E_d (and, once, the Jacobi scale)
    for (int i = tid; i < d; i += NT) {
      const double hjj = Hd[tri_row(i) + i];
      double sc;
      if (mode == MODE_INIT) { sc = 1.0 / (1.0 + sqrt(hjj)); W.scale_d[i] = sc; }
      else sc = W.scale_d[i];
      const double s2 = sc * sc;
      const double E = fmin(fmax(s2 * hjj, kMinDiag), kMaxDiag) / s2;
      W.Ed[cur][i] = E;
      s_E[i] = E;
      s_g[i] = gd[i];
      s_v[i] = gd[i] / E;
    }
    __syncthreads();
    // If the iteration limit is reached, the step that was just judged is the last one: the new linearisation
    // is only committed (state, gradient norm for the tolerance test) -- no reduced system, no factorisation,
    // no new step (k_schur skips the same rounds).
    const bool skip_solve = (st->iteration >= opt.max_iterations) && !sh->fail;
    double VHV_dd = 0.0;
    int chol_fail = sh->fail;
    if (!skip_solve) {
      // One pass over the packed dense Hessian, a warp per row (lanes over the columns: no index arithmetic, coalesced
      // partials): v^T H v of the dense-dense part, and the reduced system M = Hd + mu E - [Sacc] written in place
      // when the system lives in shared memory.
      double* Mx = chol_in_smem ? s_big : W.chol;
      const double mu = st->mu;
      double vhv_loc = 0.0;
      for (int r0 = warp; r0 < d; r0 += NT / 32) {
        const double* hrow = Hd + tri_row(r0);
        double* mrow = Mx + tri_row(r0);
        const double* arow = W.partA + (size_t)r0 * dcp;      // chunk partials were summed by k_reduce_partials
        double sacc = 0.0;
        for (int c0 = lane; c0 <= r0; c0 += 32) {
          const double h = hrow[c0];
          double v = h;
          if (c0 < r0) sacc += h * s_v[c0];
          else { vhv_loc += s_v[r0] * h * s_v[r0]; v += mu * s_E[r0]; }
          if (r0 < dc) v -= arow[c0];
          mrow[c0] = v;
        }
        vhv_loc += 2.0 * s_v[r0] * sacc;
      }
      VHV_dd = block_sum(vhv_loc, sh->red);
      for (int i = tid; i < d; i += NT) {
        double v = s_g[i];
        if (i < dc) {
          v -= W.partA[(size_t)dc * dcp + i];
        }
        s_rhs[i] = v;
        Mx[tri_row(d) + i] = v;            // appended row: the right-hand side
      }
      __syncthreads();
      PHASE_MARK(2);
      if (tid == 0) {
        // the chain elimination needs a block-tridiagonal speed/bias part: IMU terms between consecutive blocks,
        // at most two neighbouring blocks in the marginalisation prior (anything else takes the plain dense path)
        int ok = (W.NSB > 0) ? 1 : 0;
        for (int t = 0; t < W.n_imu; ++t) {
          const int dsb = (int)W.imu_terms[t].sb1 - (int)W.imu_terms[t].sb0;
          if (dsb > 1 || dsb < -1) ok = 0;
        }
        int lo = 1 << 30, hi = -1;
        for (int b = 0; b < W.marg_nb; ++b)
          if (W.marg_kind[b] == OKB_BLOCK_SPEED_BIAS && W.marg_col[b] >= 0) { lo = min(lo, (int)W.marg_idx[b]); hi = max(hi, (int)W.marg_idx[b]); }
        if (hi - lo > 1) ok = 0;
        sh->chain_ok = ok;
      }
      __syncthreads();
      if (sh->chain_ok) {
        // ---- speed/bias chain first (okb_chol.cuh), then the dense blocked Cholesky of the dc x dc pose system
        const int nsb = W.NSB, ns = 9 * nsb;
        double* s_band = chol_in_smem ? nullptr : s_big;
        double* Cp = (solve_mode == 2) ? s_big + (((size_t)ns * 18 + 1) & ~(size_t)1) : Mx;     // pose system C'
        int* s_yo = reinterpret_cast<int*>(s_delta + dc);       // row offset tables (okb_chol.cuh) in the idle tail of s_delta
        int* s_ao = s_yo + ns;
        const ChainView A{s_band ? s_band : Mx, s_ao, Mx, s_yo, dc};
        for (int i = tid; i < ns; i += NT) {
          const int yo = (int)tri_row(dc + i);
          s_yo[i] = yo;
          s_ao[i] = s_band ? 18 * i : yo + dc + 9 * (i / 9) - 9;
        }
        if (s_band) {
          for (int e = tid; e < ns * 18; e += NT) {
            const int i = e / 18, j = 9 * (i / 9) - 9 + e % 18;
            s_band[e] = (j >= 0 && j <= i) ? Mx[tri_row(dc + i) + dc + j] : 0.0;
          }
        }
#ifdef OKB_CHOL_PROF
        unsigned long long t_cp = clock64();
#define CHAIN_MARK(i) do { if (tid == 0) { const unsigned long long n_ = clock64(); st->phase_ns[i] += n_ - t_cp; t_cp = n_; } } while (0)
#else
#define CHAIN_MARK(i) do { } while (0)
#endif
        if (tid == 0) sh->chol_flag = 0;
        __syncthreads();
        if (!chol_fail) {
          // warp 0 factors the chain; the other warps follow one block behind with Y over B and z over the rhs
          // (named barriers 1..nsb; long chains or very wide pose parts run the two steps one after the other)
          const bool pipelined = nsb <= 15 && dc + 1 <= NT - 32;
          if (warp == 0) chain_factor(A, nsb, s_col + dc, &sh->chol_flag, pipelined);
          else if (pipelined) chain_forward(A, nsb, s_col + dc, s_rhs + dc, true);
          if (!pipelined) {
            __syncthreads();
            chain_forward(A, nsb, s_col + dc, s_rhs + dc, false);
          }
        }
        __syncthreads();
        if (sh->chol_flag) chol_fail = 1;
        CHAIN_MARK(11);
        if (!chol_fail) {
          CHAIN_MARK(12);
          chain_schur(A, Cp, ns, s_rhs, s_rhs + dc);
          __syncthreads();
          CHAIN_MARK(13);
          // appended right-hand side row of the pose system; in place it takes the slot of Y's first row, which
          // is parked in s_delta until the pose solve is done
          for (int i = tid; i < dc; i += NT) {
            if (Cp == Mx) s_delta[i] = Mx[tri_row(dc) + i];
            Cp[tri_row(dc) + i] = s_rhs[i];
          }
          __syncthreads();
          chol_fail = block_cholesky(Cp, dc, dc + 1, s_panel, ld_p, s_col, &sh->chol_flag, st->phase_ns + 8, solve_mode != 0);
        }
        PHASE_MARK(3);
        if (!chol_fail) {
          for (int i = tid; i < dc; i += NT) s_tmp[i] = Cp[tri_row(dc) + i];
          __syncthreads();
          CHAIN_MARK(7);      // row swap + dense factorisation (its sub-phases are slots 8..10)
          block_cholesky_backward(Cp, dc, s_col, s_tmp);
          CHAIN_MARK(14);
          if (Cp == Mx) for (int i = tid; i < dc; i += NT) Mx[tri_row(dc) + i] = s_delta[i];
          __syncthreads();
          for (int r = tid; r < ns; r += NT) {        // z - Y u_p
            const double* yr = Mx + s_yo[r];
            double sacc = s_rhs[dc + r];
            for (int i = 0; i < dc; ++i) sacc -= yr[i] * s_tmp[i];
            s_tmp[dc + r] = sacc;
          }
          __syncthreads();
          if (warp == 0) chain_backward(A, nsb, s_col + dc, s_tmp);
          __syncthreads();
          CHAIN_MARK(15);
          for (int i = tid; i < d; i += NT) { s_u[i] = s_tmp[i]; W.ud[i] = s_tmp[i]; }
          __syncthreads();
        }
      } else {
        // ---- dense Cholesky (lower), blocked right-looking (okb_chol.cuh); row d comes out as z = L^-1 rhs
        if (!chol_fail) chol_fail = block_cholesky(Mx, d, d + 1, s_panel, ld_p, s_col, &sh->chol_flag, st->phase_ns + 8, chol_in_smem != 0);
        PHASE_MARK(3);
        if (!chol_fail) {
          for (int i = tid; i < d; i += NT) s_tmp[i] = Mx[tri_row(d) + i];
          __syncthreads();
          block_cholesky_backward(Mx, d, s_col, s_tmp);
          for (int i = tid; i < d; i += NT) { s_u[i] = s_tmp[i]; W.ud[i] = s_tmp[i]; }
          __syncthreads();
        }
      }
    }
    PHASE_MARK(4);
    // ---- landmarks: commit, back-substitute, scalar reductions
    double N2 = 0, GU = 0, G2 = 0, VHV = 0, xn2 = 0, gmax = 0;
    int bad = 0;
    const double* gl_ = W.lm_g[cur];
    const double* El_ = W.lm_E[cur];
    for (int l = tid; l < L; l += NT) {
      const double4 X = *reinterpret_cast<const double4*>(W.lm_c + 4 * (size_t)l);
      *reinterpret_cast<double4*>(W.lm + 4 * (size_t)l) = X;
      xn2 += X.x * X.x + X.y * X.y + X.z * X.z + X.w * X.w;
      if (chol_fail) continue;
      const double g0 = gl_[3 * (size_t)l], g1 = gl_[3 * (size_t)l + 1], g2 = gl_[3 * (size_t)l + 2];
      if (skip_solve) { gmax = fmax(gmax, fmax(fabs(g0), fmax(fabs(g1), fabs(g2)))); continue; }
      const double E0 = El_[3 * (size_t)l], E1 = El_[3 * (size_t)l + 1], E2 = El_[3 * (size_t)l + 2];
      const double v0 = g0 / E0, v1 = g1 / E1, v2 = g2 / E2;
      double q0 = 0, q1 = 0, q2 = 0;        // sum_f M_f (G_f u_f)
      double hv = 0;                        // sum_f v^T M_f (v - 2 G_f v_f)
      // landmarks are sorted by observing-frame range, so the visibility test is warp-coherent; M is
      // tile-major (lm_M_index): every load is a 256-byte row per warp
      const uint32_t vis = W.lm_vis[l];
      for (int f = 0; f < K; ++f) {
        if (!((vis >> f) & 1u)) continue;
        const double* Mo = W.lm_M + lm_M_index(l, f, K);
        const double M0 = Mo[0], M1 = Mo[32], M2 = Mo[64], M3 = Mo[96], M4 = Mo[128], M5 = Mo[160];
        const double p0 = X.x - s_tws[4 * f] * X.w, p1 = X.y - s_tws[4 * f + 1] * X.w, p2 = X.z - s_tws[4 * f + 2] * X.w;
        const double* uf = s_u + 6 * f;
        const double* vf = s_v + 6 * f;
        // G y = w y_t + y_r x p
        const double a0 = X.w * uf[0] + (uf[4] * p2 - uf[5] * p1);
        const double a1 = X.w * uf[1] + (uf[5] * p0 - uf[3] * p2);
        const double a2 = X.w * uf[2] + (uf[3] * p1 - uf[4] * p0);
        q0 += M0 * a0 + M1 * a1 + M2 * a2;
        q1 += M1 * a0 + M3 * a1 + M4 * a2;
        q2 += M2 * a0 + M4 * a1 + M5 * a2;
        const double b0 = v0 - 2.0 * (X.w * vf[0] + (vf[4] * p2 - vf[5] * p1));
        const double b1 = v1 - 2.0 * (X.w * vf[1] + (vf[5] * p0 - vf[3] * p2));
        const double b2 = v2 - 2.0 * (X.w * vf[2] + (vf[3] * p1 - vf[4] * p0));
        hv += v0 * (M0 * b0 + M1 * b1 + M2 * b2) + v1 * (M1 * b0 + M3 * b1 + M4 * b2) + v2 * (M2 * b0 + M4 * b1 + M5 * b2);
      }
      const double* Ri = W.lm_Rinv + 6 * (size_t)l;
      const double t0 = g0 + q0, t1 = g1 + q1, t2 = g2 + q2;
      const double u0 = Ri[0] * t0 + Ri[1] * t1 + Ri[2] * t2;
      const double u1 = Ri[1] * t0 + Ri[3] * t1 + Ri[4] * t2;
      const double u2 = Ri[2] * t0 + Ri[4] * t1 + Ri[5] * t2;
      W.lm_gn[3 * (size_t)l] = -u0; W.lm_gn[3 * (size_t)l + 1] = -u1; W.lm_gn[3 * (size_t)l + 2] = -u2;
      if (!(isfinite(u0) && isfinite(u1) && isfinite(u2))) bad = 1;
      N2 += E0 * u0 * u0 + E1 * u1 * u1 + E2 * u2 * u2;
      GU += g0 * u0 + g1 * u1 + g2 * u2;
      G2 += g0 * v0 + g1 * v1 + g2 * v2;
      VHV += hv;
      gmax = fmax(gmax, fmax(fabs(g0), fmax(fabs(g1), fabs(g2))));
    }
    for (int i = tid; i < d; i += NT) {
      if (chol_fail || !dense_owner) break;
      const double g = s_g[i], E = s_E[i];
      if (skip_solve) { gmax = fmax(gmax, fabs(g)); continue; }
      const double u = s_u[i];
      if (!isfinite(u)) bad = 1;
      N2 += E * u * u; GU += g * u; G2 += g * g / E;
      gmax = fmax(gmax, fabs(g));
    }
    if (dense_owner) {
      for (int i = tid; i < 7 * K; i += NT) xn2 += W.pose[i] * W.pose[i];
      for (int i = tid; i < 9 * W.NSB; i += NT) xn2 += W.sb[i] * W.sb[i];
    }
    xs[0] = block_sum(N2, sh->red);
    xs[1] = block_sum(GU, sh->red);
    xs[2] = block_sum(G2, sh->red);
    xs[3] = block_sum(VHV, sh->red) + (dense_owner ? VHV_dd : 0.0);
    xs[4] = block_sum(xn2, sh->red);
    xs[5] = block_max(gmax, sh->red);
    xs[6] = block_sum((double)bad, sh->red);
    chol_fail_adopt = chol_fail;
  }
  if (sharded) {
    // second exchange of the round: the landmark parts of the step scalars live on their shards; rank 0's clock
    // drives the time-limit callback on every rank (the ranks must take identical decisions)
    xs[7] = 1e-9 * ((double)(globaltimer_ns() - st->t_start_ns) + (double)st->t_last_iter_ns);
    if (!shard_exchange_scalars(W, st, sh, xs)) {
      if (tid == 0) { st->shard_fault = 1; st->termination = OKB_TERM_FAILURE; st->done = 1; }
      return;
    }
  }
  if (adopt) {
    if (tid == 0) {
      st->x_norm2 = xs[4];
      st->grad_max = xs[5];
      st->numeric_fail = 0;
      if (chol_fail_adopt || xs[6] > 0) {
        sh->fail = 1;
      } else {
        st->G2 = xs[2]; st->VHV = xs[3]; st->GU = xs[1]; st->N2 = xs[0];
        sh->fail = 0;
      }
    }
    __syncthreads();
  }

  PHASE_MARK(5);
  // ================= phase 5: loop top (callbacks, iteration limit), dogleg step =================
  if (tid == 0) {
    const unsigned long long now = globaltimer_ns();
    int finish = 0;
    if (sh->commit_only) finish = 1;                       // min radius reached after an accepted step
    else if (sh->fail) {
      // linear solver failure: DoglegStrategy raises mu and retries inside ComputeStep; if mu is
      // exhausted the step is invalid (counts as an iteration, StepIsInvalid raises mu again).
      st->mu *= kMuIncrease;
      if (st->mu >= kMaxMu) {
        st->iteration += 1;
        st->num_invalid += 1;
        if (st->num_invalid >= kMaxConsecutiveInvalid) { st->termination = OKB_TERM_FAILURE; finish = 1; }
        st->mu *= kMuIncrease;
      }
      st->reuse = 0;
      st->mode = MODE_REBUILD;
      st->a = 0; st->b = 0;
      sh->spec = -1;   // no candidate computation
    } else {
      if (adopt && st->grad_max <= kGradientTolerance) { st->termination = OKB_TERM_GRADIENT_TOL; finish = 1; }
      // IterationCallback on the summary of the iteration that just ended
      const double elapsed = 1e-9 * (double)(now - st->t_start_ns);
      const double last = 1e-9 * (double)st->t_last_iter_ns;
      const double t_cb = sharded ? sh->x2[7] : elapsed + last;     // sharded: rank 0's clock, exchanged above
      if (!finish && opt.time_limit_s >= 0.0 && st->iteration >= opt.min_iterations && t_cb > opt.time_limit_s) {
        st->termination = OKB_TERM_TIME_LIMIT; finish = 1;
      }
      if (!finish && st->iteration >= opt.max_iterations) { st->termination = OKB_TERM_NO_CONVERGENCE; finish = 1; }
      if (!finish) {
        st->iteration += 1;
        st->t_iter_begin_ns = now;
        // ---- traditional dogleg in the metric E (== Ceres' diagonal-scaled space)
        const double G2 = st->G2, VHV = st->VHV, GU = st->GU, N2 = st->N2, mu = st->mu, radius = st->radius;
        const double alpha = G2 / VHV;
        const double gnorm = sqrt(G2), gn_norm = sqrt(N2);
        double a, b, dl;
        if (gn_norm <= radius) { a = 0.0; b = 1.0; dl = gn_norm; }
        else if (gnorm * alpha >= radius) { a = -radius / gnorm; b = 0.0; dl = radius; }
        else {
          const double b_dot_a = alpha * GU;                   // -alpha * (ghat . GN), ghat.GN = -GU
          const double a_sq = alpha * alpha * G2;
          const double bma = a_sq - 2.0 * b_dot_a + N2;
          const double c = b_dot_a - a_sq;
          const double dd = sqrt(c * c + bma * (radius * radius - a_sq));
          const double beta = (c <= 0) ? (dd - c) / bma : (radius * radius - a_sq) / (dd + c);
          a = -alpha * (1.0 - beta); b = beta;
          dl = sqrt(fmax(0.0, a * a * G2 - 2.0 * a * b * GU + b * b * N2));
        }
        // model cost change = -step^T g - 0.5 step^T H step, step = a v + b (-u)
        const double sg = a * G2 - b * GU;
        const double vHu = G2 - mu * GU, uHu = GU - mu * N2;
        const double sHs = a * a * VHV - 2.0 * a * b * vHu + b * b * uHu;
        const double mcc = -sg - 0.5 * sHs;
        st->a = a; st->b = b; st->dogleg_step_norm = dl; st->model_cost_change = mcc;
        if (!(mcc >= 0.0)) {
          st->num_invalid += 1;
          if (st->num_invalid >= kMaxConsecutiveInvalid) { st->termination = OKB_TERM_FAILURE; finish = 1; }
          st->mu *= kMuIncrease;          // StepIsInvalid
          st->reuse = 0;
          st->mode = MODE_REBUILD;
          st->a = 0; st->b = 0;
          sh->spec = -1;
        } else {
          st->num_invalid = 0;
          st->mode = MODE_STEP;
          sh->spec = 1;
        }
      }
    }
    if (finish) {
      int redo = 0;
      for (int t = 0; t < W.n_imu; ++t) redo += W.imu_cache[t].redo_count;
      st->imu_redo_final = redo - st->imu_redo;
      st->done = 1;
      st->solve_time_s = 1e-9 * (double)(globaltimer_ns() - st->t_start_ns);
      sh->spec = 0;
    }
  }
  __syncthreads();
  const int what = sh->spec;
  if (what == 0) return;

  // ================= phase 6: candidate dense parameters =================
  {
    const double a = st->a, b = st->b;
    const double* gcur = W.gd[cur];
    const double* Ecur = W.Ed[cur];
    for (int i = tid; i < d; i += NT) s_delta[i] = (what == 1) ? (a * gcur[i] / Ecur[i] - b * W.ud[i]) : 0.0;
    __syncthreads();
    double sn2 = 0.0;
    for (int f = tid; f < K; f += NT) {
      double o[7];
      if (what == 1) pose_plus(W.pose + 7 * f, s_delta + 6 * f, o);
      else for (int k = 0; k < 7; ++k) o[k] = W.pose[7 * f + k];
      for (int k = 0; k < 7; ++k) {
        const double dlt = o[k] - W.pose[7 * f + k];
        sn2 += dlt * dlt;
        W.pose_c[7 * f + k] = o[k];
      }
    }
    for (int i = tid; i < 9 * W.NSB; i += NT) {
      const double dlt = s_delta[dc + i];
      W.sb_c[i] = W.sb[i] + dlt;
      sn2 += dlt * dlt;
    }
    sn2 = block_sum(sn2, sh->red);
    if (tid == 0) st->cand_step_norm2_dense = sn2;
    build_slot_ctx(W, tid, NT);        // (frame, camera) contexts of the next linearisation
  }
  PHASE_MARK(6);
#undef PHASE_MARK
}

// Compile epilogue on the transfer stream, batched over windows (blockIdx.y), for windows whose graph changed
// (W.dirty): k_zero clears the observation grid and the M blocks; k_prepare scatters the compacted observation
// list (k_compile_obs) into the slot-major grid through the landmark permutation (k_compile_sort), refreshes the packed
// output block and, after a full upload, keeps the initial state for okb_window_reset.
__global__ void __launch_bounds__(256) k_zero(const WinDev* __restrict__ wins, int win_first) {
  const WinDev& W = wins[win_first + blockIdx.y];
  if (!W.dirty) return;
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    uint4* p = reinterpret_cast<uint4*>(W.zero_ptr[r]);
    const size_t n = W.zero_bytes[r] / sizeof(uint4);         // regions are 256-byte multiples
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) p[i] = z;
  }
}
// packed estimates for the download: pose [K][7] | sb [NSB][9] | landmarks [L][4] | quality [L] (caller's order)
__device__ __forceinline__ double* out_lm(const WinDev& W) { return W.out + out_lm_offset(W.K, W.NSB); }
__device__ __forceinline__ double* out_quality(const WinDev& W) { return W.out + out_lm_offset(W.K, W.NSB) + 4 * (size_t)W.L; }

__global__ void __launch_bounds__(256) k_prepare(const WinDev* __restrict__ wins, int win_first) {
  const WinDev& W = wins[win_first + blockIdx.y];
  if (!W.dirty) return;
  const int n_obs = W.st->g.n_obs;
  const int work = max(max(n_obs, 4 * W.L), max(7 * W.K, 9 * W.NSB));
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < work; i += gridDim.x * blockDim.x) {
    if (i < n_obs) {
      const okb_observation ob = W.m_obs[i];
      const size_t g = (size_t)((int)ob.pose_idx * W.CP + (int)ob.cam_idx) * W.L + W.lm_inv[ob.lm_idx];
      W.obs_z[g] = make_double2(ob.z[0], ob.z[1]);
      W.obs_w[g] = ob.sqrt_info;
    }
    if (i < 7 * W.K) { W.out[i] = W.pose[i]; if (W.full) W.pose_init[i] = W.pose[i]; }
    if (i < 9 * W.NSB) { W.out[7 * W.K + i] = W.sb[i]; if (W.full) W.sb_init[i] = W.sb[i]; }
    if (i < 4 * W.L) { out_lm(W)[i] = W.m_lm[i]; if (W.full) W.m_lm_init[i] = W.m_lm[i]; }
    if (i < W.L) out_quality(W)[i] = 0.0;
  }
}

// resets the solver state (and optionally the parameter state: the one of the last full upload) of the windows
// wins[win_slots[blockIdx.x]]
__global__ void k_reset(const WinDev* __restrict__ wins, const int32_t* __restrict__ win_slots, int restore_params) {
  const WinDev& W = wins[win_slots[blockIdx.x]];
  const int tid = threadIdx.x;
  if (restore_params) {
    for (int i = tid; i < 7 * W.K; i += blockDim.x) { W.pose[i] = W.pose_init[i]; W.out[i] = W.pose_init[i]; }
    for (int i = tid; i < 9 * W.NSB; i += blockDim.x) { W.sb[i] = W.sb_init[i]; W.out[7 * W.K + i] = W.sb_init[i]; }
    for (int j = tid; j < W.L; j += blockDim.x) {
      const uint32_t l = W.perm[j];
      const double4 x = *reinterpret_cast<const double4*>(W.m_lm_init + 4 * (size_t)l);
      *reinterpret_cast<double4*>(W.m_lm + 4 * (size_t)l) = x;
      *reinterpret_cast<double4*>(W.lm + 4 * (size_t)j) = x;
      *reinterpret_cast<double4*>(out_lm(W) + 4 * (size_t)l) = x;
      out_quality(W)[l] = 0.0;
    }
    const int nb = (int)(sizeof(ImuCache) / sizeof(double));
    for (int i = tid; i < nb * W.n_imu; i += blockDim.x) reinterpret_cast<double*>(W.imu_cache)[i] = 0.0;   // valid = 0, as uploaded
  }
  __syncthreads();
  for (int i = tid; i < 7 * W.K; i += blockDim.x) W.pose_c[i] = W.pose[i];
  for (int i = tid; i < 9 * W.NSB; i += blockDim.x) W.sb_c[i] = W.sb[i];
  __syncthreads();
  build_slot_ctx(W, tid, blockDim.x);
  if (tid == 0) {
    SolverState* st = W.st;
    st->mode = MODE_INIT; st->done = 0; st->cur = 0;
    st->iteration = 0; st->num_successful = 0; st->num_invalid = 0; st->termination = OKB_TERM_NO_CONVERGENCE;
    if (st->g.err) { st->done = 1; st->termination = OKB_TERM_FAILURE; }    // a rejected graph is never solved
    st->reuse = 0; st->numeric_fail = 0;
    st->radius = kInitialRadius; st->mu = kMinMu; st->mu_spec = kMinMu;
    st->cost = 0; st->initial_cost = 0; st->x_norm2 = 0;
    st->G2 = st->VHV = st->GU = st->N2 = 0; st->a = 0; st->b = 0;
    st->model_cost_change = 0; st->dogleg_step_norm = 0; st->cand_step_norm2_dense = 0; st->grad_max = 0;
    for (int i = 0; i < 16; ++i) st->phase_ns[i] = 0;
    st->shard_wait_ns = 0; st->shard_rounds = 0; st->shard_fault = 0;     // shard_epoch is never reset
    st->t_start_ns = 0; st->t_last_iter_ns = 0; st->t_iter_begin_ns = 0; st->solve_time_s = 0;
    int redo = 0;
    for (int t = 0; t < W.n_imu; ++t) redo += W.imu_cache[t].redo_count;
    st->imu_redo = redo;   // baseline; the summary reports the difference
    st->imu_redo_final = 0;
  }
}

}  // namespace okb
