// Device-resident window graph (sm_90a): the "master" copy of a keyframe window in the caller's index space,
// edited by a command interpreter and compiled into the solver's working layout on the device.
//
//   host (okb_window_upload / okb_window_add_frame / ... in okb_estimator.cu) only appends COMMANDS + payload to a
//   pinned per-slot buffer; okb_window_commit ships the buffer with one H2D copy and launches, batched over windows:
//     k_apply_commands : one CTA per window interprets the commands in order (set / add / remove frames, landmarks,
//                        observations, IMU terms, priors) on the master arrays -- replaces the reference's
//                        Estimator::addStates / addLandmark / addObservation / removeObservation bookkeeping
//                        (okvis_ceres/src/Estimator.cpp:110-413, implementation/Estimator.hpp:43-90) and the Map's
//                        pointer graph (okvis_ceres/include/okvis/ceres/Map.hpp:348-402);
//     k_compile_obs    : validates + compacts the observation list (order preserving), builds the per-landmark frame
//                        visibility masks, the (frame, camera) slot table and rejects duplicate observations;
//     k_compile_sort   : stable counting sort of the landmarks by (first, last) observing frame (same order as
//                        okb_hostpack.hpp: sort_landmarks_by_frame_range), tile frame ranges, sorted landmark copy;
//     k_zero / k_prepare (okb_kernels.cuh) : clear and scatter the slot-major observation grid.
//   The solver kernels never see the master copy; k_quality writes the estimates back in the caller's order.
#pragma once
#include "okb_estimator.cuh"

namespace okb {

enum {
  CMD_RESET_GRAPH = 1,      // a = n_extrinsics, b = n_cameras; payload: extrinsics [a][7], cameras [b]
  CMD_SET_FRAMES = 2,       // a = K, b = NSB; payload poses [K][7], speed_bias [NSB][9] (replaces all frames)
  CMD_SET_POSE = 3,         // a = idx; payload 7
  CMD_SET_SB = 4,           // a = idx; payload 9
  CMD_SET_EXT = 5,          // a = idx; payload 7
  CMD_ADD_FRAME = 6,        // b & 1: has speed/bias; payload pose 7 (+ speed_bias 9)
  CMD_REMOVE_FRAME = 7,     // a = pose index, b = speed/bias index (0xffffffff: none)
  CMD_SET_LANDMARKS = 8,    // n landmarks; b = 1: indices are a, a+1, ... (no list) else payload idx [n] u32 (8-byte padded); then xyzw [n][4]
  CMD_REMOVE_LANDMARKS = 9, // n; payload idx [n] u32
  CMD_ADD_OBS = 10,         // n; payload okb_observation [n]
  CMD_REMOVE_OBS = 11,      // n; payload {pose_idx, lm_idx, cam_idx, _} u32 x 4 [n]
  CMD_SET_IMU = 12,         // a = terms, b = samples; payload okb_imu_term [a] (absolute offsets), okb_imu_sample [b]; replaces all, caches cleared
  CMD_ADD_IMU_TERM = 13,    // n = samples; payload okb_imu_term (sample_offset relative to the payload's samples), okb_imu_sample [n]
  CMD_SET_POSE_PRIORS = 14, // n; payload okb_pose_prior [n]
  CMD_SET_SB_PRIORS = 15,   // n; payload okb_sb_prior [n]
  CMD_REMOVE_SB = 17,       // a = speed/bias index: the block, the IMU terms and SpeedAndBiasError priors attached to it
  CMD_SET_MARG = 16,        // a = n, b = n_blocks; payload kind [b] i32, idx [b] u32 (each 8-byte padded), x0, J [n][n], e0 [n]
  // feature store (FeatStore, okb_estimator.cuh); every array of a payload is 8-byte padded
  CMD_SET_FEATURES = 18,    // n keypoints of image (a = feature slot, b = camera); payload x, y, size [n][3] f64, lm [n] i32, observed [n] u8, desc [n][D]
  CMD_SET_FEATURE_LMS = 19, // n; a = feature slot, b = camera; payload kp_idx [n] i32, lm [n] i32, observed [n] u8
  CMD_CLEAR_FEATURES = 20,  // a = feature slot: every camera's image emptied
  CMD_SET_LM_INIT = 21      // n; payload idx [n] u32, flags [n] u8
};
struct CmdHeader { uint32_t op, n, a, b; uint64_t payload_bytes; };   // payload follows, 8-byte aligned
static_assert(sizeof(CmdHeader) == 24, "command header layout");

enum { GERR_INDEX = 1, GERR_DUPLICATE = 2, GERR_SLOT_EXT = 3, GERR_CAPACITY = 4, GERR_SQRT_INFO = 5, GERR_DIMS = 6, GERR_MARG_REF = 7,
       GERR_SHARD_MARG = 8 };

__device__ __forceinline__ void graph_error(GraphState* g, int code) { atomicCAS(&g->err, 0, code); }

__device__ __forceinline__ int block_excl_scan_1024(int v, int* s_warp, int* total) {
  // exclusive scan of one int per thread over a 1024-thread CTA; *total = sum (valid in all threads)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  __syncthreads();
  if (lane == 31) s_warp[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = s_warp[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
    s_warp[lane] = w;
  }
  __syncthreads();
  const int base = warp ? s_warp[warp - 1] : 0;
  *total = s_warp[31];
  return base + x - v;
}

// ------------------------------------------------------------------------------------------------
// command interpreter: one CTA of 1024 threads per window
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_apply_commands(const WinDev* __restrict__ wins, int win_first) {
  const WinDev& W = wins[win_first + blockIdx.x];
  if (W.cmd_bytes <= 0) return;
  GraphState* g = &W.st->g;
  const int tid = threadIdx.x, NT = blockDim.x;
  __shared__ int s_map[kMaxFrames];          // IMU term compaction map
  __shared__ int s_i[4];
  __shared__ uint32_t s_keys[256 * 3];
  const unsigned char* p = W.cmd;
  const unsigned char* end = W.cmd + W.cmd_bytes;
  while (p < end) {
    __syncthreads();
    const CmdHeader h = *reinterpret_cast<const CmdHeader*>(p);
    const unsigned char* pay = p + sizeof(CmdHeader);
    const double* pd = reinterpret_cast<const double*>(pay);
    p = pay + h.payload_bytes;
    const int K = g->K, NSB = g->NSB, n_obs = g->n_obs;
    __syncthreads();
    switch (h.op) {
      case CMD_RESET_GRAPH: {
        const double* ext = pd;
        const double* cams = ext + 7 * h.a;
        for (int i = tid; i < 7 * (int)h.a; i += NT) W.ext[i] = ext[i];
        for (int i = tid; i < (int)(h.b * sizeof(okb_camera) / 8); i += NT) reinterpret_cast<double*>(W.cams)[i] = cams[i];
        for (int i = tid; i < 4 * W.Lcap; i += NT) W.m_lm[i] = 0.0;
        if (tid == 0) {
          g->K = 0; g->NSB = 0; g->L = 0; g->n_obs = 0; g->n_imu = 0; g->n_samples = 0; g->n_pp = 0; g->n_sbp = 0;
          g->marg_n = 0; g->marg_nb = 0; g->marg_xdim = 0; g->err = 0; g->NE = (int)h.a; g->NC = (int)h.b;
          if ((int)h.a > W.NEcap || (int)h.b > W.NCcap) graph_error(g, GERR_CAPACITY);
        }
        break;
      }
      case CMD_SET_FRAMES: {
        if ((int)h.a > W.Kcap || (int)h.b > W.Kcap) { if (tid == 0) graph_error(g, GERR_CAPACITY); break; }
        for (int i = tid; i < 7 * (int)h.a; i += NT) W.pose[i] = pd[i];
        for (int i = tid; i < 9 * (int)h.b; i += NT) W.sb[i] = pd[7 * h.a + i];
        if (tid == 0) { g->K = (int)h.a; g->NSB = (int)h.b; }
        break;
      }
      case CMD_SET_POSE:
        if ((int)h.a >= K) { if (tid == 0) graph_error(g, GERR_INDEX); break; }
        if (tid < 7) W.pose[7 * h.a + tid] = pd[tid];
        break;
      case CMD_SET_SB:
        if ((int)h.a >= NSB) { if (tid == 0) graph_error(g, GERR_INDEX); break; }
        if (tid < 9) W.sb[9 * h.a + tid] = pd[tid];
        break;
      case CMD_SET_EXT:
        if ((int)h.a >= g->NE) { if (tid == 0) graph_error(g, GERR_INDEX); break; }
        if (tid < 7) W.ext[7 * h.a + tid] = pd[tid];
        break;
      case CMD_ADD_FRAME: {
        const bool has_sb = h.b & 1u;
        if (K >= W.Kcap || (has_sb && NSB >= W.Kcap)) { if (tid == 0) graph_error(g, GERR_CAPACITY); break; }
        if (tid < 7) W.pose[7 * K + tid] = pd[tid];
        if (has_sb && tid < 9) W.sb[9 * NSB + tid] = pd[7 + tid];
        if (tid == 0) { g->K = K + 1; if (has_sb) g->NSB = NSB + 1; }
        break;
      }
      case CMD_REMOVE_FRAME: {
        const int pf = (int)h.a;
        const int sbi = (h.b == 0xffffffffu) ? -1 : (int)h.b;
        if (pf >= K || sbi >= NSB) { if (tid == 0) graph_error(g, GERR_INDEX); break; }
        // states: shift down (all values fit one pass of the CTA: read, barrier, write)
        {
          const int np = 7 * (K - pf - 1), ns = (sbi >= 0) ? 9 * (NSB - sbi - 1) : 0;
          double vp = 0, vs = 0;
          if (tid < np) vp = W.pose[7 * (pf + 1) + tid];
          if (tid < ns) vs = W.sb[9 * (sbi + 1) + tid];
          __syncthreads();
          if (tid < np) W.pose[7 * pf + tid] = vp;
          if (tid < ns) W.sb[9 * sbi + tid] = vs;
        }
        // observations of the frame die; later frames move down one position
        for (int i = tid; i < n_obs; i += NT) {
          okb_observation* ob = W.m_obs + i;
          const uint32_t f = ob->pose_idx;
          if ((int)f == pf) ob->sqrt_info = 0.0;
          else if ((int)f > pf) ob->pose_idx = f - 1;
        }
        // IMU terms touching the frame are dropped, the others re-indexed; caches follow their terms
        const int n_imu = g->n_imu;
        if (tid == 0) {
          int o = 0;
          for (int t = 0; t < n_imu; ++t) {
            okb_imu_term T = W.imu_terms[t];
            const bool drop = (int)T.pose0 == pf || (int)T.pose1 == pf || (sbi >= 0 && ((int)T.sb0 == sbi || (int)T.sb1 == sbi));
            s_map[t] = drop ? -1 : o;
            if (drop) continue;
            if ((int)T.pose0 > pf) T.pose0--;
            if ((int)T.pose1 > pf) T.pose1--;
            if (sbi >= 0 && (int)T.sb0 > sbi) T.sb0--;
            if (sbi >= 0 && (int)T.sb1 > sbi) T.sb1--;
            W.imu_terms[o++] = T;
          }
          s_i[0] = o;
        }
        __syncthreads();
        const int n_new = s_i[0];
        constexpr int CW = (int)(sizeof(ImuCache) / sizeof(double));
        for (int t = 0; t < n_imu; ++t) {           // ascending: destinations never overtake unread sources
          const int o = s_map[t];
          if (o < 0 || o == t) continue;
          double v[(CW + 1023) / 1024];
#pragma unroll
          for (int q = 0; q < (CW + 1023) / 1024; ++q) { const int i = tid + q * 1024; if (i < CW) v[q] = reinterpret_cast<const double*>(W.imu_cache + t)[i]; }
          __syncthreads();
#pragma unroll
          for (int q = 0; q < (CW + 1023) / 1024; ++q) { const int i = tid + q * 1024; if (i < CW) reinterpret_cast<double*>(W.imu_cache + o)[i] = v[q]; }
          __syncthreads();
        }
        // sample pool: reclaim the samples in front of the first sample still referenced
        if (tid == 0) {
          uint32_t lo = 0xffffffffu, hi = 0;
          for (int t = 0; t < n_new; ++t) { lo = min(lo, W.imu_terms[t].sample_offset); hi = max(hi, W.imu_terms[t].sample_offset + W.imu_terms[t].sample_count); }
          if (n_new == 0) { lo = 0; hi = 0; }
          s_i[1] = (int)lo; s_i[2] = (int)hi;
          for (int t = 0; t < n_new; ++t) W.imu_terms[t].sample_offset -= lo;
        }
        __syncthreads();
        {
          const int lo = s_i[1], hi = s_i[2];
          constexpr int SW = (int)(sizeof(okb_imu_sample) / 8);
          const int words = (hi - lo) * SW;
          double* pool = reinterpret_cast<double*>(W.samples);
          if (lo > 0)
            for (int base = 0; base < words; base += NT) {
              const int i = base + tid;
              double v = 0;
              if (i < words) v = pool[(size_t)lo * SW + i];
              __syncthreads();
              if (i < words) pool[i] = v;
              __syncthreads();
            }
          if (tid == 0) { g->n_samples = hi - lo; g->n_imu = n_new; }
        }
        if (tid == 0) {
          int o = 0;
          for (int i = 0; i < g->n_pp; ++i) {
            okb_pose_prior P = W.pp[i];
            if ((int)P.pose_idx == pf) continue;
            if ((int)P.pose_idx > pf) P.pose_idx--;
            W.pp[o++] = P;
          }
          g->n_pp = o;
          o = 0;
          for (int i = 0; i < g->n_sbp; ++i) {
            okb_sb_prior P = W.sbp[i];
            if (sbi >= 0 && (int)P.sb_idx == sbi) continue;
            if (sbi >= 0 && (int)P.sb_idx > sbi) P.sb_idx--;
            W.sbp[o++] = P;
          }
          g->n_sbp = o;
          for (int b = 0; b < g->marg_nb; ++b) {
            const int kind = W.marg_kind[b];
            const int ref = (kind == OKB_BLOCK_POSE) ? pf : (kind == OKB_BLOCK_SPEED_BIAS) ? sbi : -1;
            if (ref < 0) continue;
            if ((int)W.marg_idx[b] == ref) graph_error(g, GERR_MARG_REF);
            else if ((int)W.marg_idx[b] > ref) W.marg_idx[b]--;
          }
          g->K = K - 1;
          if (sbi >= 0) g->NSB = NSB - 1;
        }
        break;
      }
      case CMD_SET_LANDMARKS: {
        const int n = (int)h.n;
        const bool range = h.b & 1u;
        const uint32_t* idx = reinterpret_cast<const uint32_t*>(pay);
        const double* x = range ? pd : reinterpret_cast<const double*>(pay + (((size_t)n * 4 + 7) & ~(size_t)7));
        if (tid == 0) s_i[0] = g->L;
        __syncthreads();
        int lmax = 0;
        for (int i = tid; i < n; i += NT) {
          const uint32_t l = range ? h.a + (uint32_t)i : idx[i];
          if ((int)l >= W.Lcap) { graph_error(g, GERR_CAPACITY); continue; }
          *reinterpret_cast<double4*>(W.m_lm + 4 * (size_t)l) = make_double4(x[4 * i], x[4 * i + 1], x[4 * i + 2], x[4 * i + 3]);
          lmax = max(lmax, (int)l + 1);
        }
        if (lmax) atomicMax(&s_i[0], lmax);
        __syncthreads();
        if (tid == 0) g->L = s_i[0];
        break;
      }
      case CMD_REMOVE_LANDMARKS: {
        const int n = (int)h.n, L = g->L;
        const uint32_t* idx = reinterpret_cast<const uint32_t*>(pay);
        for (int i = tid; i < n; i += NT) { if ((int)idx[i] < L) W.m_mark[idx[i]] = 1; else graph_error(g, GERR_INDEX); }
        __syncthreads();
        for (int i = tid; i < n_obs; i += NT) {
          okb_observation* ob = W.m_obs + i;
          if ((int)ob->lm_idx < L && W.m_mark[ob->lm_idx]) ob->sqrt_info = 0.0;
        }
        if (W.feat && W.shard_world > 1) {
          // landmark-sharded: the store names global slots and is replicated; the removal reaches only the owner, so
          // the slot is marked (bit 1) and every rank's store forgets it at the next landmark exchange (okb_frontend.cu)
          for (int i = tid; i < n; i += NT)
            if ((int)idx[i] < W.feat->lm_cap) W.feat->lm_init[idx[i]] = 2;
        } else if (W.feat) {
          // the store forgets the removed slots (the reference's isLandmarkAdded(id) == false for a gone id), so a slot
          // reused later is never reached through a keypoint that referred to its previous occupant
          const FeatStore& F = *W.feat;
          const int n_ent = F.F * F.C * F.N;
          for (int e = tid; e < n_ent; e += NT) {
            const int l = F.lm[e];
            if (l >= 0 && l < L && W.m_mark[l]) { F.lm[e] = -1; F.observed[e] = 0; }
          }
          for (int i = tid; i < n; i += NT)
            if ((int)idx[i] < F.lm_cap) F.lm_init[idx[i]] = 0;
        }
        __syncthreads();
        for (int i = tid; i < n; i += NT)
          if ((int)idx[i] < L) { W.m_mark[idx[i]] = 0; *reinterpret_cast<double4*>(W.m_lm + 4 * (size_t)idx[i]) = make_double4(0, 0, 0, 0); }
        break;
      }
      case CMD_ADD_OBS: {
        const int n = (int)h.n;
        if (n_obs + n > W.Ocap) { if (tid == 0) graph_error(g, GERR_CAPACITY); break; }
        constexpr int OW = (int)(sizeof(okb_observation) / 8);
        const unsigned long long* src = reinterpret_cast<const unsigned long long*>(pay);
        unsigned long long* dst = reinterpret_cast<unsigned long long*>(W.m_obs + n_obs);
        for (int i = tid; i < n * OW; i += NT) dst[i] = src[i];
        if (tid == 0) g->n_obs = n_obs + n;
        break;
      }
      case CMD_REMOVE_OBS: {
        const int n = (int)h.n;
        const uint32_t* keys = reinterpret_cast<const uint32_t*>(pay);
        for (int kb = 0; kb < n; kb += 256) {
          const int nk = min(256, n - kb);
          __syncthreads();
          for (int i = tid; i < nk * 3; i += NT) s_keys[i] = keys[4 * (kb + i / 3) + (i % 3)];
          __syncthreads();
          for (int i = tid; i < n_obs; i += NT) {
            okb_observation* ob = W.m_obs + i;
            const uint32_t f = ob->pose_idx, l = ob->lm_idx, cm = ob->cam_idx;
            for (int k = 0; k < nk; ++k)
              if (s_keys[3 * k] == f && s_keys[3 * k + 1] == l && s_keys[3 * k + 2] == cm) { ob->sqrt_info = 0.0; break; }
          }
        }
        break;
      }
      case CMD_SET_IMU: {
        const int nt = (int)h.a, ns = (int)h.b;
        if (nt > W.Tcap || ns > W.Scap) { if (tid == 0) graph_error(g, GERR_CAPACITY); break; }
        const double* tsrc = pd;
        const double* ssrc = pd + (size_t)nt * (sizeof(okb_imu_term) / 8);
        for (int i = tid; i < nt * (int)(sizeof(okb_imu_term) / 8); i += NT) reinterpret_cast<double*>(W.imu_terms)[i] = tsrc[i];
        for (int i = tid; i < ns * (int)(sizeof(okb_imu_sample) / 8); i += NT) reinterpret_cast<double*>(W.samples)[i] = ssrc[i];
        for (int i = tid; i < nt * (int)(sizeof(ImuCache) / 8); i += NT) reinterpret_cast<double*>(W.imu_cache)[i] = 0.0;
        if (tid == 0) { g->n_imu = nt; g->n_samples = ns; }
        break;
      }
      case CMD_ADD_IMU_TERM: {
        const int ns = (int)h.n, n_imu = g->n_imu, n_s = g->n_samples;
        if (n_imu >= W.Tcap || n_s + ns > W.Scap) { if (tid == 0) graph_error(g, GERR_CAPACITY); break; }
        const double* ssrc = pd + sizeof(okb_imu_term) / 8;
        for (int i = tid; i < ns * (int)(sizeof(okb_imu_sample) / 8); i += NT) reinterpret_cast<double*>(W.samples + n_s)[i] = ssrc[i];
        for (int i = tid; i < (int)(sizeof(ImuCache) / 8); i += NT) reinterpret_cast<double*>(W.imu_cache + n_imu)[i] = 0.0;
        if (tid == 0) {
          okb_imu_term T = *reinterpret_cast<const okb_imu_term*>(pay);
          T.sample_offset += (uint32_t)n_s;
          W.imu_terms[n_imu] = T;
          g->n_imu = n_imu + 1; g->n_samples = n_s + ns;
        }
        break;
      }
      case CMD_SET_POSE_PRIORS: {
        if ((int)h.n > W.PPcap) { if (tid == 0) graph_error(g, GERR_CAPACITY); break; }
        for (int i = tid; i < (int)(h.n * sizeof(okb_pose_prior) / 8); i += NT) reinterpret_cast<double*>(W.pp)[i] = pd[i];
        if (tid == 0) g->n_pp = (int)h.n;
        break;
      }
      case CMD_SET_SB_PRIORS: {
        if ((int)h.n > W.PPcap) { if (tid == 0) graph_error(g, GERR_CAPACITY); break; }
        for (int i = tid; i < (int)(h.n * sizeof(okb_sb_prior) / 8); i += NT) reinterpret_cast<double*>(W.sbp)[i] = pd[i];
        if (tid == 0) g->n_sbp = (int)h.n;
        break;
      }
      case CMD_SET_MARG: {
        const int n = (int)h.a, nb = (int)h.b;
        if (n > kMaxMarg || nb > kMaxMargBlocks) { if (tid == 0) graph_error(g, GERR_CAPACITY); break; }
        const size_t kb = ((size_t)nb * 4 + 7) & ~(size_t)7;
        const int32_t* kinds = reinterpret_cast<const int32_t*>(pay);
        const uint32_t* idx = reinterpret_cast<const uint32_t*>(pay + kb);
        if (tid == 0) {
          int col = 0, xo = 0;
          for (int b = 0; b < nb; ++b) {
            W.marg_kind[b] = kinds[b]; W.marg_idx[b] = idx[b]; W.marg_off[b] = xo;
            const bool fixed = kinds[b] == OKB_BLOCK_EXTRINSICS;       // extrinsics are fixed in the device solver
            W.marg_col[b] = fixed ? -1 : col;
            if (!fixed) col += (kinds[b] == OKB_BLOCK_SPEED_BIAS) ? 9 : 6;
            xo += (kinds[b] == OKB_BLOCK_SPEED_BIAS) ? 9 : 7;
          }
          if (col != n) graph_error(g, GERR_DIMS);
          s_i[0] = xo;
          g->marg_n = n; g->marg_nb = nb; g->marg_xdim = xo;
        }
        __syncthreads();
        const int xdim = s_i[0];
        const double* x0 = reinterpret_cast<const double*>(pay + 2 * kb);
        const double* J = x0 + xdim;
        const double* e0 = J + (size_t)n * n;
        for (int i = tid; i < xdim; i += NT) W.marg_x0[i] = x0[i];
        for (int i = tid; i < n * n; i += NT) W.marg_J[i] = J[i];
        for (int i = tid; i < n; i += NT) W.marg_e0[i] = e0[i];
        for (int e = tid; e < n * n; e += NT) {        // H0 = J^T J (fixed summation order)
          const int i = e / n, j = e % n;
          if (j > i) continue;
          double s = 0;
          for (int r = 0; r < n; ++r) s += J[(size_t)r * n + i] * J[(size_t)r * n + j];
          W.marg_H0[(size_t)i * n + j] = s; W.marg_H0[(size_t)j * n + i] = s;
          W.marg_Hs[(size_t)i * n + j] = s; W.marg_Hs[(size_t)j * n + i] = s;
        }
        for (int i = tid; i < n; i += NT) {            // b0 = -J^T e0: what a later okb_window_marginalize starts from
          double s = 0;
          for (int r = 0; r < n; ++r) s += J[(size_t)r * n + i] * e0[r];
          W.marg_b0[i] = -s;
        }
        break;
      }
      case CMD_REMOVE_SB: {
        const int sbi = (int)h.a;
        if (sbi >= NSB) { if (tid == 0) graph_error(g, GERR_INDEX); break; }
        {
          const int ns = 9 * (NSB - sbi - 1);
          double vs = 0;
          if (tid < ns) vs = W.sb[9 * (sbi + 1) + tid];
          __syncthreads();
          if (tid < ns) W.sb[9 * sbi + tid] = vs;
        }
        const int n_imu = g->n_imu;
        if (tid == 0) {
          int o = 0;
          for (int t = 0; t < n_imu; ++t) {
            okb_imu_term T = W.imu_terms[t];
            const bool drop = (int)T.sb0 == sbi || (int)T.sb1 == sbi;
            s_map[t] = drop ? -1 : o;
            if (drop) continue;
            if ((int)T.sb0 > sbi) T.sb0--;
            if ((int)T.sb1 > sbi) T.sb1--;
            W.imu_terms[o++] = T;
          }
          s_i[0] = o;
        }
        __syncthreads();
        const int n_new = s_i[0];
        constexpr int CW2 = (int)(sizeof(ImuCache) / sizeof(double));
        for (int t = 0; t < n_imu; ++t) {
          const int o = s_map[t];
          if (o < 0 || o == t) continue;
          double v[(CW2 + 1023) / 1024];
#pragma unroll
          for (int q = 0; q < (CW2 + 1023) / 1024; ++q) { const int i = tid + q * 1024; if (i < CW2) v[q] = reinterpret_cast<const double*>(W.imu_cache + t)[i]; }
          __syncthreads();
#pragma unroll
          for (int q = 0; q < (CW2 + 1023) / 1024; ++q) { const int i = tid + q * 1024; if (i < CW2) reinterpret_cast<double*>(W.imu_cache + o)[i] = v[q]; }
          __syncthreads();
        }
        if (tid == 0) {
          uint32_t lo = 0xffffffffu, hi = 0;
          for (int t = 0; t < n_new; ++t) { lo = min(lo, W.imu_terms[t].sample_offset); hi = max(hi, W.imu_terms[t].sample_offset + W.imu_terms[t].sample_count); }
          if (n_new == 0) { lo = 0; hi = 0; }
          s_i[1] = (int)lo; s_i[2] = (int)hi;
          for (int t = 0; t < n_new; ++t) W.imu_terms[t].sample_offset -= lo;
        }
        __syncthreads();
        {
          const int lo = s_i[1], hi = s_i[2];
          constexpr int SW2 = (int)(sizeof(okb_imu_sample) / 8);
          const int words = (hi - lo) * SW2;
          double* pool = reinterpret_cast<double*>(W.samples);
          if (lo > 0)
            for (int base = 0; base < words; base += NT) {
              const int i = base + tid;
              double v = 0;
              if (i < words) v = pool[(size_t)lo * SW2 + i];
              __syncthreads();
              if (i < words) pool[i] = v;
              __syncthreads();
            }
          if (tid == 0) { g->n_samples = hi - lo; g->n_imu = n_new; }
        }
        if (tid == 0) {
          int o = 0;
          for (int i = 0; i < g->n_sbp; ++i) {
            okb_sb_prior P = W.sbp[i];
            if ((int)P.sb_idx == sbi) continue;
            if ((int)P.sb_idx > sbi) P.sb_idx--;
            W.sbp[o++] = P;
          }
          g->n_sbp = o;
          for (int b = 0; b < g->marg_nb; ++b) {
            if (W.marg_kind[b] != OKB_BLOCK_SPEED_BIAS) continue;
            if ((int)W.marg_idx[b] == sbi) graph_error(g, GERR_MARG_REF);
            else if ((int)W.marg_idx[b] > sbi) W.marg_idx[b]--;
          }
          g->NSB = NSB - 1;
        }
        break;
      }
      case CMD_SET_FEATURES: {
        const int n = (int)h.n, f = (int)h.a, cm = (int)h.b;
        if (!W.feat || f >= W.feat->F || cm >= W.feat->C || n > W.feat->N) { if (tid == 0) graph_error(g, GERR_INDEX); break; }
        const FeatStore& F = *W.feat;
        const size_t base = ((size_t)f * F.C + cm) * F.N;
        const size_t bl = ((size_t)4 * n + 7) & ~(size_t)7, bo = ((size_t)n + 7) & ~(size_t)7;
        const int32_t* lm = reinterpret_cast<const int32_t*>(pay + 24 * (size_t)n);
        const uint8_t* ob = pay + 24 * (size_t)n + bl;
        const uint32_t* desc = reinterpret_cast<const uint32_t*>(pay + 24 * (size_t)n + bl + bo);
        for (int i = tid; i < n; i += NT) {
          F.kp[2 * (base + i)] = pd[3 * i]; F.kp[2 * (base + i) + 1] = pd[3 * i + 1]; F.size[base + i] = pd[3 * i + 2];
          F.lm[base + i] = lm[i]; F.observed[base + i] = ob[i];
        }
        const int dw = F.D / 4;
        for (int i = tid; i < n * dw; i += NT) F.desc[base * dw + i] = desc[i];
        if (tid == 0) F.n[f * F.C + cm] = n;
        break;
      }
      case CMD_SET_FEATURE_LMS: {
        const int n = (int)h.n, f = (int)h.a, cm = (int)h.b;
        if (!W.feat || f >= W.feat->F || cm >= W.feat->C) { if (tid == 0) graph_error(g, GERR_INDEX); break; }
        const FeatStore& F = *W.feat;
        const size_t base = ((size_t)f * F.C + cm) * F.N;
        const size_t b4 = ((size_t)4 * n + 7) & ~(size_t)7;
        const int32_t* k = reinterpret_cast<const int32_t*>(pay);
        const int32_t* lm = reinterpret_cast<const int32_t*>(pay + b4);
        const uint8_t* ob = pay + 2 * b4;
        const int nk = F.n[f * F.C + cm];
        for (int i = tid; i < n; i += NT) {
          if (k[i] < 0 || k[i] >= nk) { graph_error(g, GERR_INDEX); continue; }
          F.lm[base + k[i]] = lm[i]; F.observed[base + k[i]] = ob[i];
        }
        break;
      }
      case CMD_CLEAR_FEATURES: {
        if (!W.feat || (int)h.a >= W.feat->F) { if (tid == 0) graph_error(g, GERR_INDEX); break; }
        if (tid < W.feat->C) W.feat->n[(int)h.a * W.feat->C + tid] = -1;
        break;
      }
      case CMD_SET_LM_INIT: {
        const int n = (int)h.n;
        if (!W.feat) { if (tid == 0) graph_error(g, GERR_INDEX); break; }
        const uint32_t* idx = reinterpret_cast<const uint32_t*>(pay);
        const uint8_t* fl = pay + (((size_t)4 * n + 7) & ~(size_t)7);
        for (int i = tid; i < n; i += NT) {
          if ((int)idx[i] >= W.feat->lm_cap) { graph_error(g, GERR_INDEX); continue; }
          W.feat->lm_init[idx[i]] = (W.feat->lm_init[idx[i]] & 2) | (fl[i] ? 1 : 0);   // keeps a sharded removal mark
        }
        break;
      }
      default:
        if (tid == 0) graph_error(g, GERR_DIMS);
        p = end;
        break;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// compile, pass 1: observation list -> validated, compacted list + visibility masks + slot table
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_compile_obs(const WinDev* __restrict__ wins, int win_first) {
  const WinDev& W = wins[win_first + blockIdx.x];
  if (!W.dirty) return;
  GraphState* g = &W.st->g;
  const int tid = threadIdx.x, NT = blockDim.x;
  __shared__ int s_warp[32];
  const int K = W.K, L = W.L, CP = W.CP, NS = W.NS;
  // the host mirrors every dimension; a mismatch means the command stream was not what the host thinks it was
  if (tid == 0 && (g->K != K || g->NSB != W.NSB || g->L != L || g->n_imu != W.n_imu || g->n_samples != W.n_samples || g->n_pp != W.n_pp ||
                   g->n_sbp != W.n_sbp || g->marg_n != W.marg_n || g->marg_nb != W.marg_nb || g->NE != W.NE || g->NC != W.NC))
    graph_error(g, GERR_DIMS);
  for (int i = tid; i < L; i += NT) W.m_vis[i] = 0u;
  const size_t n_words = ((size_t)NS * L + 31) / 32;
  for (size_t i = tid; i < n_words; i += NT) W.m_bitmap[i] = 0u;
  for (int s = tid; s < W.NSP; s += NT) W.slots[s] = SlotInfo{s / CP, -1, s % CP, 0};
  __syncthreads();
  const int n = g->n_obs;
  int out = 0;
  for (int base = 0; base < n; base += NT) {
    const int i = base + tid;
    okb_observation ob;
    int keep = 0;
    if (i < n) {
      ob = W.m_obs[i];
      if (ob.sqrt_info != 0.0) {                                    // 0 marks a removed observation
        if ((int)ob.pose_idx >= K || (int)ob.lm_idx >= L || (int)ob.ext_idx >= W.NE || (int)ob.cam_idx >= W.NC) graph_error(g, GERR_INDEX);
        else if (!(ob.sqrt_info > 0.0)) graph_error(g, GERR_SQRT_INFO);
        else keep = 1;
      }
    }
    int total;
    const int pos = block_excl_scan_1024(keep, s_warp, &total);      // barriers inside: all reads of this chunk are done
    if (keep) {
      W.m_obs[out + pos] = ob;
      atomicOr(&W.m_vis[ob.lm_idx], 1u << ob.pose_idx);
      const int s = (int)ob.pose_idx * CP + (int)ob.cam_idx;
      const size_t cell = (size_t)s * L + ob.lm_idx;
      const uint32_t bit = 1u << (cell & 31);
      if (atomicOr(&W.m_bitmap[cell >> 5], bit) & bit) graph_error(g, GERR_DUPLICATE);
      const int old = atomicCAS(&W.slots[s].ext_idx, -1, (int)ob.ext_idx);
      if (old != -1 && old != (int)ob.ext_idx) graph_error(g, GERR_SLOT_EXT);
      W.slots[s].valid = 1;
    }
    out += total;
    __syncthreads();
  }
  if (tid == 0) g->n_obs = out;
  __syncthreads();
  for (int s = tid; s < W.NSP; s += NT)
    if (!W.slots[s].valid) W.slots[s] = SlotInfo{0, 0, 0, 0};
}

// ------------------------------------------------------------------------------------------------
// compile, pass 2: stable counting sort of the landmarks by (first, last) observing frame
// (identical order to okb_hostpack.hpp: sort_landmarks_by_frame_range), tile ranges, sorted copies
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t frame_range_key_dev(uint32_t m) {
  if (!m) return 32u * 32u;
  return (uint32_t)(__ffs((int)m) - 1) * 32u + (31u - (uint32_t)__clz((int)m));
}

__global__ void __launch_bounds__(1024) k_compile_sort(const WinDev* __restrict__ wins, int win_first) {
  const WinDev& W = wins[win_first + blockIdx.x];
  if (!W.dirty) return;
  const int tid = threadIdx.x, NT = blockDim.x, lane = tid & 31, warp = tid >> 5;
  const int L = W.L;
  __shared__ uint32_t cursor[32 * 32 + 1];
  for (int i = tid; i < 32 * 32 + 1; i += NT) cursor[i] = 0u;
  __syncthreads();
  for (int l = tid; l < L; l += NT) atomicAdd(&cursor[frame_range_key_dev(W.m_vis[l])], 1u);
  __syncthreads();
  if (warp == 0) {          // exclusive scan of the 1025 bucket counts: 33 per lane, then a warp scan of the lane sums
    uint32_t loc[33];
    uint32_t s = 0;
#pragma unroll
    for (int q = 0; q < 33; ++q) { const int b = lane * 33 + q; loc[q] = (b < 1025) ? cursor[b] : 0u; s += loc[q]; }
    uint32_t x = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    uint32_t run = x - s;
#pragma unroll
    for (int q = 0; q < 33; ++q) { const int b = lane * 33 + q; if (b < 1025) cursor[b] = run; run += loc[q]; }
  }
  __syncthreads();
  // stable placement: landmarks in ascending caller index; inside a chunk of 1024 the warps take turns
  for (int base = 0; base < L; base += NT) {
    const int l = base + tid;
    const uint32_t key = (l < L) ? frame_range_key_dev(W.m_vis[l]) : 0xffffu;
    const uint32_t grp = __match_any_sync(0xffffffffu, key);
    const int rank = __popc(grp & ((1u << lane) - 1u));
    const int leader = __ffs((int)grp) - 1;
    uint32_t start = 0;
    for (int w = 0; w < NT / 32; ++w) {
      if (warp == w && lane == leader && l < L) { start = cursor[key]; cursor[key] = start + (uint32_t)__popc(grp); }
      __syncthreads();
    }
    start = __shfl_sync(0xffffffffu, start, leader);
    if (l < L) {
      const uint32_t j = start + (uint32_t)rank;
      W.perm[j] = (uint32_t)l;
      W.lm_inv[l] = j;
    }
  }
  __syncthreads();
  // sorted copies + frame range per tile of 32
  const int n_tiles = (L + 31) / 32;
  for (int t = warp; t < n_tiles; t += NT / 32) {
    const int j = t * 32 + lane;
    uint32_t m = 0u;
    if (j < L) {
      const uint32_t l = W.perm[j];
      m = W.m_vis[l];
      W.lm_vis[j] = m;
      *reinterpret_cast<double4*>(W.lm + 4 * (size_t)j) = *reinterpret_cast<const double4*>(W.m_lm + 4 * (size_t)l);
    }
    uint32_t fi = m ? (uint32_t)(__ffs((int)m) - 1) : 255u, la = m ? 31u - (uint32_t)__clz((int)m) : 0u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { fi = min(fi, __shfl_xor_sync(0xffffffffu, fi, o)); la = max(la, __shfl_xor_sync(0xffffffffu, la, o)); }
    if (lane == 0) W.tile_range[t] = (fi == 255u) ? 1u : (fi | (la << 8));
  }
}

}  // namespace okb
