// Device-side data model of one keyframe window and of the batched dogleg/Schur solver.
// See DESIGN.md ("Data layout in HBM", "Kernels") for the rationale.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "okb_imu.cuh"

namespace okb {

// ---- compile-time limits ------------------------------------------------------------------
constexpr int kMaxFrames = 32;        // frame visibility mask is one u32
constexpr int kMaxChunks = 64;        // landmark chunks (CTAs) per window in kernel A
constexpr int kMaxDense = 512;        // reduced-system dimension limit
constexpr int kMaxMarg = 160;         // marginalisation prior dimension limit
constexpr int kMaxMargBlocks = 64;    // parameter blocks connected to the marginalisation prior
constexpr int kMaxShard = 8;          // ranks of a landmark-sharded window (one NVSwitch domain)

// Ceres 1.9 defaults used by Estimator::optimize (SURVEY.md 3.1)
constexpr double kInitialRadius = 1e4;
constexpr double kMinRadius = 1e-32;
constexpr double kMinRelativeDecrease = 1e-3;
constexpr double kFunctionTolerance = 1e-6;
constexpr double kGradientTolerance = 1e-10;
constexpr double kParameterTolerance = 1e-8;
constexpr double kMinDiag = 1e-6;
constexpr double kMaxDiag = 1e32;
constexpr double kMinMu = 1e-8;
constexpr double kMaxMu = 1.0;
constexpr double kMuIncrease = 10.0;
constexpr int kMaxConsecutiveInvalid = 5;

enum Mode { MODE_INIT = 0, MODE_STEP = 1, MODE_REBUILD = 2 };

struct SlotInfo { int pose_idx, ext_idx, cam_idx, valid; };

// Dimensions of the device-resident window graph as the command interpreter left them (okb_graph.cuh); the host
// mirrors the same arithmetic, k_compile_obs cross-checks.  err: first GERR_* raised by a command or by the compile.
struct GraphState { int K, NSB, L, n_obs, n_imu, n_samples, n_pp, n_sbp, marg_n, marg_nb, marg_xdim, NE, NC, err; };

// Per-window solver state (device resident, one per window; also read back as the summary).
struct SolverState {
  int mode;            // what kernel A must evaluate next / what kernel S must judge
  int done;            // 1 = terminated
  int cur;             // buffer index of the linearisation at the committed state (lm_g / lm_E / gd / Ed)
  int iteration, num_successful, num_invalid, termination;
  int reuse;           // dogleg reuse_ flag
  int numeric_fail;    // set by kernel A when a landmark block is not positive definite
  int imu_redo;
  int imu_redo_final;
  double radius, mu, mu_spec;
  double cost, initial_cost;
  double x_norm2;      // ||x||^2 of the committed state (ambient)
  // dogleg scalars of the current linearisation (metric E):
  double G2, VHV, GU, N2;
  double a, b;         // step = a * g/E + b * (-u)
  double model_cost_change, dogleg_step_norm;
  double cand_step_norm2_dense;   // ||x - x_cand||^2 over the dense blocks
  double grad_max;
  unsigned long long t_start_ns, t_last_iter_ns, t_iter_begin_ns;
  double solve_time_s;
  unsigned long long phase_ns[16];  // accumulated phase times (diagnostics): 0..7 k_solve, 8..13 k_schur (chunk 0, thread 0)
  // Landmark-sharded windows: exchange epoch (one per solver round; never reset, so stale mailbox flags of an earlier
  // optimize can not match) and the accumulated device time spent waiting for / summing the peers' partial systems.
  unsigned long long shard_epoch;
  unsigned long long shard_wait_ns, shard_rounds;
  int shard_fault;     // 1 = a peer did not arrive within the time-out (the window terminates with FAILURE)
  GraphState g;
};

// ---- landmark-sharded single window (SURVEY 8e row 2): per-window mailbox in every rank's device memory.
// Rank s PUSHES its reduced landmark partial (Schur accumulator, pose-block sums, cost) into box [parity][s] of every
// rank's mailbox with plain stores over NVLink, then releases flag [parity][s]; the consumer (k_solve) acquires the
// `world` flags in its own memory and adds the boxes in rank order, so every rank forms the bit-identical reduced
// system.  Boxes are double-buffered by the parity of the round's epoch (see DESIGN.md, "Multi-GPU").
constexpr size_t kShardHeaderBytes = 4096;
constexpr size_t kShardFlags1 = 0;       // u64 [2][kMaxShard]   reduced-system boxes ready
constexpr size_t kShardFlags2 = 128;     // u64 [2][kMaxShard]   step scalars ready
constexpr size_t kShardCounter = 256;    // u32                  last-CTA counter of k_shard_push (local use)
constexpr size_t kShardMargEpoch = 384;  // u64                  epoch of the last marginalisation exchange (local use)
constexpr size_t kShardScalars = 512;    // f64 [2][kMaxShard][16]
constexpr size_t kShardFlagsM = 2560;    // u64 [2][kMaxShard]   marginalisation boxes ready
constexpr size_t kShardFlagsL = 2688;    // u64 [2][kMaxShard]   landmark replica pushed (frontend calls)
constexpr size_t kShardLmEpoch = 2816;   // u64                  epoch of the last landmark exchange (local use)
constexpr size_t kShardLmCounter = 2824; // u32                  last-CTA counter of k_shard_lm_push (local use)
constexpr size_t kShardLmStatus = 2828;  // i32                  0, or 7: a peer did not arrive (local use)
static_assert(kShardScalars + 2 * kMaxShard * 16 * sizeof(double) <= kShardFlagsM &&
              kShardFlagsM + 2 * kMaxShard * sizeof(unsigned long long) <= kShardFlagsL &&
              kShardFlagsL + 2 * kMaxShard * sizeof(unsigned long long) <= kShardLmEpoch &&
              kShardLmStatus + 4 <= kShardHeaderBytes, "shard mailbox header layout");
constexpr unsigned long long kShardTimeoutNs = 4000000000ull;   // a peer that does not arrive within 4 s: FAILURE, no hang
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void st_release_sys_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__host__ __device__ inline size_t shard_box_doubles(int K, int dcp) { return (size_t)dcp * dcp + (size_t)K * 32 + 8; }
// Marginalisation box (k_marginalize<true>): header [fingerprint, error word, epoch, pad] | pose-pose sums [P][P] | pose
// rows of b [P], P = 6 * (pose blocks of the job) <= 6 * max_frames.  A region of [2][world] such boxes follows the
// solver boxes, so a peer's marginalisation push never lands in a box a rank may still be reading for its last round.
constexpr int kMargBoxHeader = 4;
__host__ __device__ inline size_t shard_marg_box_doubles(int max_frames) {
  const size_t p = 6 * (size_t)max_frames;
  return kMargBoxHeader + p * p + p;
}
// Landmark replica of the frontend calls (okb_frontend.cu): the state the store kernels read of every global landmark
// slot g < lm_cap, all-gathered from the owners (rank g mod world, local slot g div world) at the start of a call.  A
// region of two halves follows the marginalisation boxes, double-buffered by the parity of the exchange epoch: a peer
// already in its next call never writes the half a rank may still be reading.  A half holds the homogeneous points
// [lm_cap][4] (zero: not in the graph, Estimator::isLandmarkAdded) and then ShardLmAux [lm_cap]: 40 bytes per slot,
// the half rounded up to 256 bytes.
struct ShardLmAux {
  int32_t n_obs;      // observations of the landmark in the graph
  uint8_t init;       // Estimator::isLandmarkInitialized
  uint8_t removed;    // removed since the last exchange: every rank forgets the slot's store references
  uint8_t _pad[2];
};
static_assert(sizeof(ShardLmAux) == 8, "landmark replica record");
__host__ __device__ inline size_t shard_lm_offset(int world, size_t box_cap, size_t marg_cap) {
  return (kShardHeaderBytes + 2 * (size_t)world * (box_cap + marg_cap) * sizeof(double) + 255) & ~(size_t)255;
}
__host__ __device__ inline size_t shard_lm_half_bytes(size_t lm_cap) { return (40 * lm_cap + 255) & ~(size_t)255; }
__host__ __device__ inline size_t shard_win_bytes(int world, size_t box_cap, size_t marg_cap, size_t lm_cap = 0) {
  return (shard_lm_offset(world, box_cap, marg_cap) + 2 * shard_lm_half_bytes(lm_cap) + 255) & ~(size_t)255;
}

// Everything kernels need to know about one window.  All pointers are device pointers into the
// window's arena.
// lm_M is tile-major: [tile of 32 landmarks][frame][element][32] -- a warp's accesses are 256-byte rows and
// the frames [a, b] of one tile are ONE contiguous block (a single TMA bulk copy in k_schur).
__host__ __device__ inline size_t lm_M_index(int l, int f, int K) { return ((size_t)(l >> 5) * K + f) * 192 + (l & 31); }   // + 32 * element (0..5)

// packed download block: pose [K][7] | speed/bias [NSB][9] | pad to 4 doubles | landmarks [L][4] | quality [L]
// (the landmark part is written with 32-byte vector stores)
__host__ __device__ inline size_t out_lm_offset(int K, int NSB) { return ((size_t)7 * K + (size_t)9 * NSB + 3) & ~(size_t)3; }

struct SlotCtx;   // per (frame, camera) transform + intrinsics at the candidate state (okb_kernels_lm.cuh)

// Per-window feature store of okb_track_3d2d_batch (one device allocation per window that reserved it; the struct heads
// it).  Image (f, c) = feature slot f, camera c; keypoint k of it is entry (f * C + c) * N + k.  Edited by the graph
// commands CMD_SET_FEATURES .. CMD_SET_LM_INIT (okb_graph.cuh), read and written by the tracking kernels
// (okb_frontend.cu).  Keypoints are kept in double, as Frame::getKeypoint / getKeypointSize hand them to the matcher.
struct FeatStore {
  int F, C, N, D;               // feature slots, cameras, keypoints per image, descriptor bytes
  int lm_cap;                   // landmark slots covered by lm_init
  int _pad;
  int* n;                       // [F][C] keypoints of the image, -1: none
  double* kp;                   // [F][C][N][2]
  double* size;                 // [F][C][N]
  uint32_t* desc;               // [F][C][N][D/4]
  int32_t* lm;                  // [F][C][N] landmark slot, -1: none
  uint8_t* observed;            // [F][C][N]
  uint8_t* lm_init;             // [lm_cap] Estimator::isLandmarkInitialized
};

struct WinDev {
  // capacities the arena was planned for (okb_window_reserve / the largest upload); the current dimensions below
  // change with the graph commands
  int Kcap, Lcap, Ocap, Scap, Tcap, NEcap, NCcap, PPcap;
  // master graph in the caller's index space (okb_graph.cuh); pose / sb / ext below are master and working copy at once
  double* m_lm;                                // [Lcap][4] landmark estimates, caller's order (written back after every optimize)
  double* m_lm_init;                           // [Lcap][4] as of the last full upload (okb_window_reset)
  unsigned char* m_mark;                       // [Lcap] scratch marks of the command interpreter (all zero between commands)
  okb_observation* m_obs;                      // [Ocap] observation list; sqrt_info == 0: removed, compacted by k_compile_obs
  uint32_t* m_vis;                             // [Lcap] frame-visibility masks, caller's order (compile scratch)
  uint32_t* m_bitmap;                          // one bit per observation-grid cell (duplicate detection)
  uint32_t* perm;                              // [Lcap] internal (sorted) landmark index -> caller's index
  double* out;                                 // packed estimates for the download: pose [K][7] | sb [NSB][9] | landmarks [L][4] | quality [L]
  const unsigned char* cmd;                    // command buffer of the pending commit
  int cmd_bytes;
  int dirty;                                   // 1 = the graph changed: compile before the next optimize
  int full;                                    // 1 = the pending commit is a full upload: snapshot the initial state
  int K, NSB, NE, L, NC;
  int Lp;              // L rounded up to whole tiles of 32: leading dimension of lm_M, rows of lm_Li / lm_c (bulk copies stay aligned)
  int CP;              // cameras per frame padded to a power of two
  int NS;              // slots = K * CP  (slot = frame * CP + cam)
  int NG;              // slot groups of 32 lanes
  int NSP;             // NG * 32: padded slots per landmark in the observation grid
  int d, dc, dcp;      // reduced dims: dc = 6K (pose part), d = dc + 9 NSB, dcp = 4*ceil((dc+1)/4)
  int n_imu, n_samples, n_pp, n_sbp;
  int marg_n, marg_nb, marg_xdim;
  int n_chunks, lm_per_chunk;
  int use_cauchy;
  // state
  double *pose, *sb, *ext, *lm;                // committed  [K][7] [NSB][9] [NE][7] [L][4]
  double *pose_init, *sb_init;                 // as of the last full upload (okb_window_reset); landmarks: m_lm_init
  double *pose_c, *sb_c, *lm_c;                // candidate
  // graph
  SlotInfo* slots;                             // [NSP]
  okb_camera* cams;                            // [NC]
  double2* obs_z;                              // [NS][L]  slot-major: coalesced for thread-per-landmark kernels
  double* obs_w;                               // [NS][L] sqrt information, 0 = no observation
  uint32_t* lm_vis;                            // [L] bit f set = observed in frame f
  int n_obs;                                   // host's upper bound of the list length (launch sizing); exact: st->g.n_obs
  // Landmarks are stored sorted by (first, last) observing frame (okb_window_upload): tracks are runs of
  // consecutive frames, so neighbouring landmarks see nearly the same frames -> warp-coherent visibility
  // in k_landmarks and block-sparse Schur tiles in k_schur.
  unsigned char* zero_ptr[3];                  // regions cleared by k_zero at every compile: observation grid (z, w), M blocks
  size_t zero_bytes[3];
  uint32_t* lm_inv;                            // [L] caller's landmark index -> internal (sorted) index
  uint32_t* tile_range;                  // [ceil(L/32)] frames seen by the tile: first | last << 8 (first > last: none)
  // per-landmark solver data
  double* lm_g[2];                             // [L][3] gradient block (double buffered: cur / speculative)
  double* lm_E[2];                             // [L][3] metric (Ceres diagonal^2 / scale^2)
  double* lm_Rinv;                             // [L][6] (H_ll + mu E)^-1, symmetric packed
  double* lm_M;                                // [Lp/32][K][6][32] per-frame sum of rho' A^T A (lm_M_index)
  SlotCtx* slot_ctx;                           // [NS] built by k_reset / k_solve whenever the candidate poses change
  double* lm_Li;                               // [L][9] L^-1 of (H_ll + mu E) (6) and z = L^-1 g_l (3)
  double* lm_gn;                               // [L][3] Gauss-Newton step of the current linearisation
  double* lm_scale;                            // [L][3] Jacobi scale (fixed after the first linearisation)
  double* quality;                             // [L]
  // kernel A -> kernel S partial sums, one record per chunk
  double* partA;                               // [n_chunks][dcp*dcp] Schur accumulator per chunk (k_schur)
  int partA_stride;                            // dcp*dcp
  double* partH;                               // [ceil(L/128)][K][32] pose-block sums, cost, step norm (k_landmarks)
  // dense part
  double* Hd;                                  // [d][d] J^T J restricted to dense blocks (speculative)
  double* gd[2];                               // [d]
  double* Ed[2];                               // [d]
  double* ud;                                  // [d] (H+mu E)^-1 g, dense part
  double* scale_d;                             // [d]
  double* chol;                                // [d][d] workspace (used when it does not fit in shared memory)
  // IMU
  okb_imu_term* imu_terms;
  okb_imu_sample* samples;
  okb_imu_params imu_params;
  ImuCache* imu_cache;                         // all zero (valid = 0) after an upload / okb_window_reset
  double* imu_out;                             // [n_imu][kImuOut] written by k_imu, consumed by k_solve
  int *sb_off;                                 // unused placeholder for alignment
  // priors
  okb_pose_prior* pp;
  okb_sb_prior* sbp;
  // marginalisation prior
  int32_t* marg_kind;
  uint32_t* marg_idx;
  int32_t* marg_col;                           // [marg_nb] first column of each block
  int32_t* marg_off;                           // [marg_nb] offset into x0
  double *marg_x0, *marg_J, *marg_e0, *marg_H0;  // H0 = J^T J
  double *marg_Hs, *marg_b0;                   // H / b0 as MarginalizationError keeps them between calls (okb_marg.cuh); host-supplied priors: J^T J, -J^T e0
  // landmark sharding: this rank holds the landmarks / observations of its shard and all dense blocks
  int shard_rank, shard_world;                 // world <= 1: not sharded
  int shard_box_cap;                           // doubles per box
  int shard_marg_cap;                          // doubles per marginalisation box (shard_marg_box_doubles)
  int shard_lm_cap;                            // global landmark slots of the replica (ShardLmAux), 0: none
  unsigned char* shard_mail[kMaxShard];       // this window's mailbox in every rank's memory, as mapped on this device
  SolverState* st;
  FeatStore* feat;                             // feature store (okb_window_reserve_features), nullptr: none
};

}  // namespace okb
