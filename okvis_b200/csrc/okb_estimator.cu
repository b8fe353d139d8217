// Host side of the estimator path of libokvis_b200.so: context, window packing/upload, the solver
// launch sequence, download, and the single-residual-block test hooks.  C-ABI: include/okvis_b200.h.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "okb_ctx.h"
#include "okb_hostpack.hpp"
#include "okb_graph.cuh"
#include "okb_kernels.cuh"
#include "okb_marg.cuh"

using namespace okb;

static std::string g_create_error;

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// ---------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------
template <int MODEL>
static void set_landmarks_attributes() {
  cudaFuncSetAttribute(k_landmarks<2, 1, MODEL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemL_bytes(2));
  cudaFuncSetAttribute(k_landmarks<2, 1, MODEL>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  cudaFuncSetAttribute(k_landmarks<4, 2, MODEL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemL_bytes(4));
}

// The transfer stream gets the highest priority: its small kernels (k_zero / k_prepare) are scheduled as soon
// as CTA slots free up instead of waiting behind the solver kernels of other slots.  The propagation stream gets it for
// the same reason: its one-warp jobs are latency-bound.
static cudaError_t create_high_priority_stream(cudaStream_t* s) {
  int lo = 0, hi = 0;
  cudaDeviceGetStreamPriorityRange(&lo, &hi);
  return cudaStreamCreateWithPriority(s, cudaStreamNonBlocking, hi);
}

extern "C" int okb_ctx_create(int device_id, int max_windows, okb_ctx** out) {
  if (!out || max_windows < 1) return OKB_ERR_INVALID_ARG;
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    g_create_error = std::string("no CUDA device: ") + cudaGetErrorString(e);
    return OKB_ERR_NO_DEVICE;
  }
  if (device_id < 0 || device_id >= n) { g_create_error = "bad device id"; return OKB_ERR_INVALID_ARG; }
  okb_ctx* c = new okb_ctx();
  c->device = device_id;
  c->max_windows = max_windows;
  // the landmark / solve chain is the critical path of a round: it runs at the highest stream priority, the IMU terms
  // (side stream, a long tail of one-warp CTAs) at the lowest, so they fill what the chain leaves idle
  int prio_least = 0, prio_greatest = 0;
  if (cudaSetDevice(device_id) == cudaSuccess) cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest);
  if (cudaSetDevice(device_id) != cudaSuccess || cudaStreamCreateWithPriority(&c->stream, cudaStreamNonBlocking, prio_greatest) != cudaSuccess) {
    g_create_error = "cudaSetDevice / cudaStreamCreate failed";
    okb_ctx_destroy(c);
    return OKB_ERR_CUDA;
  }
  if (cudaStreamCreateWithPriority(&c->stream_imu, cudaStreamNonBlocking, prio_least) != cudaSuccess ||
      cudaEventCreateWithFlags(&c->ev_round, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&c->ev_imu, cudaEventDisableTiming) != cudaSuccess ||
      create_high_priority_stream(&c->stream_xfer) != cudaSuccess ||
      cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming) != cudaSuccess) {
    g_create_error = "cudaStreamCreate / cudaEventCreate failed";
    okb_ctx_destroy(c);
    return OKB_ERR_CUDA;
  }
  c->group_stream[0] = c->stream; c->group_imu[0] = c->stream_imu;
  c->group_round[0] = c->ev_round; c->group_imu_done[0] = c->ev_imu;
  for (int g = 0; g < okb_ctx::kMaxSolveGroups; ++g) {      // further groups: the same priorities as group 0
    bool ok = cudaEventCreateWithFlags(&c->group_stagger[g], cudaEventDisableTiming) == cudaSuccess;
    if (g > 0)
      ok = ok && cudaStreamCreateWithPriority(&c->group_stream[g], cudaStreamNonBlocking, prio_greatest) == cudaSuccess &&
           cudaStreamCreateWithPriority(&c->group_imu[g], cudaStreamNonBlocking, prio_least) == cudaSuccess &&
           cudaEventCreateWithFlags(&c->group_round[g], cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&c->group_imu_done[g], cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&c->group_done[g], cudaEventDisableTiming) == cudaSuccess;
    if (!ok) {
      g_create_error = "cudaStreamCreate / cudaEventCreate failed";
      okb_ctx_destroy(c);
      return OKB_ERR_CUDA;
    }
  }
  for (int k = 0; k < okb_ctx::kDoneRing; ++k) cudaEventCreateWithFlags(&c->done_ring[k], cudaEventDisableTiming);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, device_id);
  c->sm_count = prop.multiProcessorCount;
  c->smem_optin = (int)prop.sharedMemPerBlockOptin;
  c->smem_per_sm = (int)prop.sharedMemPerMultiprocessor;
  c->wins.resize(max_windows);
  c->host.assign(max_windows, WinDev());
  std::memset(c->host.data(), 0, sizeof(WinDev) * max_windows);
  c->chunk_cap = std::max(1, std::min(kMaxChunks, (2 * c->sm_count) / max_windows));
  if (cudaMalloc(&c->d_wins, sizeof(WinDev) * max_windows) != cudaSuccess ||
      cudaMalloc(&c->d_states, sizeof(SolverState) * max_windows) != cudaSuccess ||
      cudaMallocHost(&c->h_states, sizeof(SolverState) * max_windows) != cudaSuccess ||
      cudaMalloc(&c->d_slot_tab, sizeof(int32_t) * max_windows) != cudaSuccess ||
      cudaMalloc(&c->d_ident, sizeof(int32_t) * max_windows) != cudaSuccess ||
      cudaMallocHost(&c->h_slot_ring, sizeof(int32_t) * okb_ctx::kDoneRing * max_windows) != cudaSuccess) {
    g_create_error = "cudaMalloc failed";
    okb_ctx_destroy(c);
    return OKB_ERR_CUDA;
  }
  cudaMemset(c->d_states, 0, sizeof(SolverState) * max_windows);
  c->ident.resize(max_windows);
  for (int i = 0; i < max_windows; ++i) c->ident[i] = i;
  cudaMemcpy(c->d_ident, c->ident.data(), sizeof(int32_t) * max_windows, cudaMemcpyHostToDevice);
  cudaFuncSetAttribute(k_schur<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, c->smem_optin);
  cudaFuncSetAttribute(k_schur<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, c->smem_optin);
  cudaFuncSetAttribute(k_imu, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemI_bytes());
  cudaFuncSetAttribute(k_imu, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  cudaFuncSetAttribute(k_solve<S_THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, c->smem_optin);
  cudaFuncSetAttribute(k_solve<S_THREADS>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  cudaFuncSetAttribute(k_solve<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, c->smem_optin);
  cudaFuncSetAttribute(k_solve<512>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  cudaFuncSetAttribute(k_schur<256>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  cudaFuncSetAttribute(k_schur<512>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  cudaFuncSetAttribute(k_quality, cudaFuncAttributeMaxDynamicSharedMemorySize, c->smem_optin);
  set_landmarks_attributes<OKB_DIST_NONE>();
  set_landmarks_attributes<OKB_DIST_RADTAN>();
  set_landmarks_attributes<OKB_DIST_EQUIDISTANT>();
  set_landmarks_attributes<OKB_DIST_RADTAN8>();
  set_landmarks_attributes<kDistAny>();
  *out = c;
  return OKB_OK;
}

extern "C" void okb_ctx_destroy(okb_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);      // null when okb_ctx_create failed before creating it
  if (c->stream_xfer) cudaStreamSynchronize(c->stream_xfer);
  for (auto& w : c->wins) {
    if (w.arena) cudaFree(w.arena);
    if (w.marg_scratch) cudaFree(w.marg_scratch);
    if (w.feat_mem) cudaFree(w.feat_mem);
    if (w.staging) cudaFreeHost(w.staging);
    if (w.out_staging) cudaFreeHost(w.out_staging);
    if (w.copied) cudaEventDestroy(w.copied);
    if (w.down) cudaEventDestroy(w.down);
  }
  for (int k = 0; k < okb_ctx::kDoneRing; ++k) if (c->done_ring[k]) cudaEventDestroy(c->done_ring[k]);
  if (c->ev_join) cudaEventDestroy(c->ev_join);
  if (c->stream_xfer) cudaStreamDestroy(c->stream_xfer);
  okb_frontend_release(c);
  for (int r = 0; r < kMaxShard; ++r)
    if (c->shard_peer_ipc[r] && c->shard_peer[r]) cudaIpcCloseMemHandle(c->shard_peer[r]);
  if (c->shard_local) cudaFree(c->shard_local);
  if (c->d_wins) cudaFree(c->d_wins);
  if (c->d_states) cudaFree(c->d_states);
  if (c->h_states) cudaFreeHost(c->h_states);
  if (c->d_slot_tab) cudaFree(c->d_slot_tab);
  if (c->d_ident) cudaFree(c->d_ident);
  if (c->h_slot_ring) cudaFreeHost(c->h_slot_ring);
  if (c->hook_buf) cudaFree(c->hook_buf);
  if (c->marg_host) cudaFreeHost(c->marg_host);
  if (c->marg_dev) cudaFree(c->marg_dev);
  if (c->marg_copied) cudaEventDestroy(c->marg_copied);
  for (unsigned char* p : c->marg_retired_dev) cudaFree(p);
  for (unsigned char* p : c->marg_retired_host) cudaFreeHost(p);
  for (auto& e : c->marg_pool) { cudaFreeHost(e.p); cudaEventDestroy(e.done); }
  c->prop_one.release();
  c->prop_batch.release();
  if (c->stream_prop) cudaStreamDestroy(c->stream_prop);
  for (auto& g : c->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
  for (auto e : c->prof_events) cudaEventDestroy(e);
  for (int g = 0; g < okb_ctx::kMaxSolveGroups; ++g) {
    if (c->group_stagger[g]) cudaEventDestroy(c->group_stagger[g]);
    if (g == 0) continue;      // entry 0 aliases the context's own stream and events
    if (c->group_round[g]) cudaEventDestroy(c->group_round[g]);
    if (c->group_imu_done[g]) cudaEventDestroy(c->group_imu_done[g]);
    if (c->group_done[g]) cudaEventDestroy(c->group_done[g]);
    if (c->group_imu[g]) cudaStreamDestroy(c->group_imu[g]);
    if (c->group_stream[g]) cudaStreamDestroy(c->group_stream[g]);
  }
  if (c->ev_round) cudaEventDestroy(c->ev_round);
  if (c->ev_imu) cudaEventDestroy(c->ev_imu);
  if (c->stream_imu) cudaStreamDestroy(c->stream_imu);
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;
}

extern "C" const char* okb_last_error(const okb_ctx* c) { return c ? c->error.c_str() : g_create_error.c_str(); }
extern "C" int64_t okb_kernel_launches(const okb_ctx* c) {
  return c ? c->launches + c->prop_launches.load() + okb_frontend_launches(c) : 0;
}
extern "C" void* okb_stream(const okb_ctx* c) { return c ? (void*)c->stream : nullptr; }

// ---------------------------------------------------------------------------------------------
// window graph: capacities, arena, command staging, commit (device side: okb_graph.cuh)
// ---------------------------------------------------------------------------------------------
namespace {
// Orders the solver stream after every transfer issued so far.
int join_transfers(okb_ctx* c) {
  if (cudaEventRecord(c->ev_join, c->stream_xfer) != cudaSuccess) return 1;
  return cudaStreamWaitEvent(c->stream, c->ev_join, 0) != cudaSuccess;
}
// Marks solver-stream work on the n listed windows: later transfers of these windows wait for it.
void mark_work(okb_ctx* c, const int32_t* slots, int n) {
  const int k = c->done_next;
  c->done_next = (k + 1) % okb_ctx::kDoneRing;
  cudaEventRecord(c->done_ring[k], c->stream);
  for (int t = 0; t < n; ++t) c->wins[slots[t]].done_idx = k;
}
inline bool caps_cover(const WinCaps& a, const WinCaps& b) {
  return a.K >= b.K && a.L >= b.L && a.O >= b.O && a.S >= b.S && a.T >= b.T && a.NE >= b.NE && a.NC >= b.NC && a.PP >= b.PP && a.MN >= b.MN;
}
inline WinCaps caps_max(const WinCaps& a, const WinCaps& b) {
  return WinCaps{std::max(a.K, b.K), std::max(a.L, b.L), std::max(a.O, b.O), std::max(a.S, b.S), std::max(a.T, b.T),
                 std::max(a.NE, b.NE), std::max(a.NC, b.NC), std::max(a.PP, b.PP), std::max(a.MN, b.MN)};
}
inline size_t full_upload_bytes(const WinCaps& q) {      // command stream of a full upload at these sizes
  return 12 * sizeof(CmdHeader) + 8 * ((size_t)7 * q.NE + 16 * (size_t)q.K + 4 * (size_t)q.L + 2 * kMaxMargBlocks + 16 * kMaxMargBlocks +
                                        (size_t)q.MN * q.MN + q.MN) +
         sizeof(okb_camera) * q.NC + sizeof(okb_observation) * (size_t)q.O + sizeof(okb_imu_term) * q.T + sizeof(okb_imu_sample) * (size_t)q.S +
         (sizeof(okb_pose_prior) + sizeof(okb_sb_prior)) * q.PP + 4096;
}

// Dimensions that follow from the current K / L / NC ... of the host mirror.
void derive_dims(WinDev& W) {
  int CP = 1;
  while (CP < W.NC) CP <<= 1;
  W.CP = CP;
  W.NS = W.K * CP; W.NG = (W.NS + 31) / 32; W.NSP = W.NG * 32;
  W.dc = 6 * W.K; W.d = W.dc + 9 * W.NSB; W.dcp = 4 * ((W.dc + 1 + 3) / 4);
  W.Lp = (W.L + 31) & ~31;
  W.partA_stride = W.dcp * W.dcp;
  W.zero_bytes[0] = align_up(sizeof(double2) * (size_t)W.L * W.NS, 256);
  W.zero_bytes[1] = align_up(sizeof(double) * (size_t)W.L * W.NS, 256);
  W.zero_bytes[2] = align_up(sizeof(double) * 6 * (size_t)W.Lp * W.K, 256);
}

// (Re)plans the slot's arena for `q` and points the host mirror at it.  Contents are lost (callers follow up with a
// full upload).
int plan_arena(okb_ctx* c, int win, const WinCaps& q) {
  WinStore& S = c->wins[win];
  Carve P;
  auto take = [&P](size_t bytes) { return P.take(bytes, 256); };     // every array on a 256-byte boundary
  int CPc = 1;
  while (CPc < q.NC) CPc <<= 1;
  const int Kc = q.K, Lc = q.L, Lpc = (Lc + 31) & ~31;
  const int NSc = Kc * CPc, NSPc = (NSc + 31) / 32 * 32;
  const int dcc = 6 * Kc, dcap = 15 * Kc, dcpc = 4 * ((dcc + 1 + 3) / 4);
  const int MN = std::max(q.MN, 1), MB = kMaxMargBlocks;
  const size_t o_pose = take(8 * 7 * Kc), o_sb = take(8 * 9 * Kc), o_ext = take(8 * 7 * q.NE), o_mlm = take(8 * 4 * (size_t)Lpc);
  const size_t o_out = take(8 * (16 * (size_t)Kc + 4 + 5 * (size_t)Lc));
  const size_t o_cams = take(sizeof(okb_camera) * q.NC), o_obs = take(sizeof(okb_observation) * (size_t)std::max(q.O, 1));
  const size_t o_imut = take(sizeof(okb_imu_term) * std::max(q.T, 1)), o_samp = take(sizeof(okb_imu_sample) * (size_t)std::max(q.S, 1));
  const size_t o_pp = take(sizeof(okb_pose_prior) * std::max(q.PP, 1)), o_sbp = take(sizeof(okb_sb_prior) * std::max(q.PP, 1));
  const size_t o_mkind = take(4 * MB), o_midx = take(4 * MB), o_mcol = take(4 * MB), o_moff = take(4 * MB);
  const size_t o_mx0 = take(8 * 9 * MB), o_mJ = take(8 * (size_t)MN * MN), o_me0 = take(8 * MN), o_mH0 = take(8 * (size_t)MN * MN);
  const size_t o_mHs = take(8 * (size_t)MN * MN), o_mb0 = take(8 * MN);
  const size_t o_mlmi = take(8 * 4 * (size_t)Lpc), o_mark = take(Lpc), o_mvis = take(4 * (size_t)Lpc);
  const size_t o_bitmap = take(4 * (((size_t)NSc * Lc + 31) / 32 + 1));
  const size_t o_perm = take(4 * (size_t)Lpc), o_inv = take(4 * (size_t)Lpc), o_trange = take(4 * (size_t)(Lpc / 32 + 1)), o_vis = take(4 * (size_t)Lpc);
  const size_t o_slots = take(sizeof(SlotInfo) * NSPc);
  const size_t cmd_cap = align_up(full_upload_bytes(q) + S.feat_frame_bytes + 65536, 256);
  const size_t o_cmd = take(cmd_cap);
  // working state / scratch
  const size_t o_lm = take(8 * 4 * (size_t)Lpc), o_pose_i = take(8 * 7 * Kc), o_sb_i = take(8 * 9 * Kc);
  const size_t o_pose_c = take(8 * 7 * Kc), o_sb_c = take(8 * 9 * Kc), o_lm_c = take(8 * 4 * (size_t)Lpc);
  size_t o_lmg[2], o_lmE[2], o_gd[2], o_Ed[2];
  for (int b = 0; b < 2; ++b) { o_lmg[b] = take(8 * 3 * (size_t)Lc); o_lmE[b] = take(8 * 3 * (size_t)Lc); }
  const size_t o_Rinv = take(8 * 6 * (size_t)Lc), o_slotctx = take(sizeof(SlotCtx) * NSPc);
  const size_t o_gn = take(8 * 3 * (size_t)Lc), o_Li = take(8 * 9 * (size_t)Lpc), o_scale = take(8 * 3 * (size_t)Lc);
  const int n_cx = (Lc + L1_THREADS - 1) / L1_THREADS;
  const size_t o_partH = take(8 * (size_t)n_cx * Kc * kPartH), o_part = take(8 * (size_t)dcpc * dcpc * c->chunk_cap);
  const size_t o_Hd = take(8 * (size_t)dcap * dcap);
  for (int b = 0; b < 2; ++b) { o_gd[b] = take(8 * dcap); o_Ed[b] = take(8 * dcap); }
  const size_t o_ud = take(8 * dcap), o_scd = take(8 * dcap), o_chol = take(8 * (size_t)(dcap + 1) * (dcap + 1));
  const size_t o_obsz = take(sizeof(double2) * (size_t)Lc * NSc), o_obsw = take(8 * (size_t)Lc * NSc), o_M = take(8 * 6 * (size_t)Lpc * Kc);
  const size_t o_quality = take(8 * (size_t)Lc);
  const size_t o_cache = take(sizeof(ImuCache) * std::max(q.T, 1)), o_imu_out = take(8 * kImuOut * std::max(q.T, 1));

  int rc;
  if ((rc = grow(c, &S.arena, &S.arena_bytes, P.off)) ||
      (rc = grow_pinned(c, &S.out_staging, &S.out_bytes, 8 * (16 * (size_t)Kc + 4 + 5 * (size_t)Lc))))
    return rc;
  if (!S.down) OKB_CUDA(c, cudaEventCreateWithFlags(&S.down, cudaEventDisableTiming));
  if (!S.copied) OKB_CUDA(c, cudaEventCreateWithFlags(&S.copied, cudaEventDisableTiming));
  // the m_mark scratch must be all zero between commands; dead landmark slots must hold finite values
  OKB_CUDA(c, cudaMemsetAsync(S.arena + o_mark, 0, Lpc, c->stream_xfer));
  OKB_CUDA(c, cudaMemsetAsync(S.arena + o_mlm, 0, 8 * 4 * (size_t)Lpc, c->stream_xfer));
  S.caps = q;
  S.cmd_cap_dev = cmd_cap;

  unsigned char* A = S.arena;
  WinDev W;
  std::memset(&W, 0, sizeof W);
  auto dp = [&](size_t o) { return reinterpret_cast<double*>(A + o); };
  auto up = [&](size_t o) { return reinterpret_cast<uint32_t*>(A + o); };
  W.Kcap = q.K; W.Lcap = q.L; W.Ocap = q.O; W.Scap = q.S; W.Tcap = q.T; W.NEcap = q.NE; W.NCcap = q.NC; W.PPcap = q.PP;
  W.pose = dp(o_pose); W.sb = dp(o_sb); W.ext = dp(o_ext); W.m_lm = dp(o_mlm); W.out = dp(o_out);
  W.cams = reinterpret_cast<okb_camera*>(A + o_cams);
  W.m_obs = reinterpret_cast<okb_observation*>(A + o_obs);
  W.imu_terms = reinterpret_cast<okb_imu_term*>(A + o_imut);
  W.samples = reinterpret_cast<okb_imu_sample*>(A + o_samp);
  W.pp = reinterpret_cast<okb_pose_prior*>(A + o_pp);
  W.sbp = reinterpret_cast<okb_sb_prior*>(A + o_sbp);
  W.marg_kind = reinterpret_cast<int32_t*>(A + o_mkind); W.marg_idx = up(o_midx);
  W.marg_col = reinterpret_cast<int32_t*>(A + o_mcol); W.marg_off = reinterpret_cast<int32_t*>(A + o_moff);
  W.marg_x0 = dp(o_mx0); W.marg_J = dp(o_mJ); W.marg_e0 = dp(o_me0); W.marg_H0 = dp(o_mH0); W.marg_Hs = dp(o_mHs); W.marg_b0 = dp(o_mb0);
  W.m_lm_init = dp(o_mlmi); W.m_mark = A + o_mark; W.m_vis = up(o_mvis); W.m_bitmap = up(o_bitmap);
  W.perm = up(o_perm); W.lm_inv = up(o_inv); W.tile_range = up(o_trange); W.lm_vis = up(o_vis);
  W.slots = reinterpret_cast<SlotInfo*>(A + o_slots);
  W.cmd = A + o_cmd;
  W.lm = dp(o_lm); W.pose_init = dp(o_pose_i); W.sb_init = dp(o_sb_i);
  W.pose_c = dp(o_pose_c); W.sb_c = dp(o_sb_c); W.lm_c = dp(o_lm_c);
  for (int b = 0; b < 2; ++b) { W.lm_g[b] = dp(o_lmg[b]); W.lm_E[b] = dp(o_lmE[b]); W.gd[b] = dp(o_gd[b]); W.Ed[b] = dp(o_Ed[b]); }
  W.lm_Rinv = dp(o_Rinv); W.slot_ctx = reinterpret_cast<SlotCtx*>(A + o_slotctx); W.lm_gn = dp(o_gn);
  W.lm_Li = dp(o_Li); W.lm_scale = dp(o_scale); W.partH = dp(o_partH); W.partA = dp(o_part);
  W.Hd = dp(o_Hd); W.ud = dp(o_ud); W.scale_d = dp(o_scd); W.chol = dp(o_chol);
  W.obs_z = reinterpret_cast<double2*>(A + o_obsz); W.obs_w = dp(o_obsw); W.lm_M = dp(o_M); W.quality = dp(o_quality);
  W.zero_ptr[0] = A + o_obsz; W.zero_ptr[1] = A + o_obsw; W.zero_ptr[2] = A + o_M;
  W.imu_cache = reinterpret_cast<ImuCache*>(A + o_cache); W.imu_out = dp(o_imu_out);
  W.st = c->d_states + win;
  W.feat = S.feat_mem ? reinterpret_cast<FeatStore*>(S.feat_mem) : nullptr;
  W.n_chunks = 1; W.use_cauchy = 1;
  c->host[win] = W;
  return OKB_OK;
}

// ---- command staging (pinned, per slot)
int cmd_reserve(okb_ctx* c, WinStore& S, size_t extra) {
  if (S.staging_busy) {          // the previous commit's H2D copy reads the buffer: wait before it is rewritten
    OKB_CUDA(c, cudaEventSynchronize(S.copied));
    S.staging_busy = false;
  }
  const size_t need = S.cmd_used + extra;
  if (need <= S.staging_bytes) return OKB_OK;
  const size_t cap = align_up(std::max(need, 2 * S.staging_bytes), 4096);
  unsigned char* nb = nullptr;
  OKB_CUDA(c, cudaMallocHost(&nb, cap));
  if (S.cmd_used) std::memcpy(nb, S.staging, S.cmd_used);
  if (S.staging) cudaFreeHost(S.staging);
  S.staging = nb; S.staging_bytes = cap;
  return OKB_OK;
}
// Appends a command header and returns the payload pointer (8-byte aligned); payload_bytes is rounded up to 8.
unsigned char* cmd_put(WinStore& S, uint32_t op, uint32_t n, uint32_t a, uint32_t b, size_t payload_bytes) {
  payload_bytes = align_up(payload_bytes, 8);
  CmdHeader h{op, n, a, b, payload_bytes};
  std::memcpy(S.staging + S.cmd_used, &h, sizeof h);
  unsigned char* pay = S.staging + S.cmd_used + sizeof h;
  S.cmd_used += sizeof h + payload_bytes;
  return pay;
}
}  // namespace

static const char* graph_error_text(int e) {
  switch (e) {
    case GERR_INDEX: return "window graph: index out of range";
    case GERR_DUPLICATE: return "window graph: duplicate observation of a landmark in one (frame,camera)";
    case GERR_SLOT_EXT: return "window graph: inconsistent extrinsics block for a (frame,camera) slot";
    case GERR_CAPACITY: return "window graph: capacity exceeded (okb_window_reserve)";
    case GERR_SQRT_INFO: return "window graph: observation with non-positive sqrt information";
    case GERR_DIMS: return "window graph: host / device dimension mismatch";
    case GERR_MARG_REF: return "window graph: a removed frame is still referenced by the marginalisation prior";
    case GERR_SHARD_MARG: return "window graph: a landmark-sharded marginalisation was abandoned on every rank (okb_window_download_marg status)";
    default: return "window graph: unknown error";
  }
}
static int graph_error_status(int e) {
  return e == GERR_DUPLICATE ? OKB_ERR_UNSUPPORTED : e == GERR_CAPACITY ? OKB_ERR_CAPACITY : OKB_ERR_INVALID_ARG;
}

extern "C" int okb_window_reserve(okb_ctx* c, int win, int max_frames, int max_landmarks, int max_observations, int max_imu_samples,
                                  int max_marg_dim) {
  if (!c || win < 0 || win >= c->max_windows || max_frames < 0 || max_landmarks < 0 || max_observations < 0 || max_imu_samples < 0 ||
      max_marg_dim < 0) return OKB_ERR_INVALID_ARG;
  if (max_frames > kMaxFrames || max_marg_dim > kMaxMarg) { c->set_error("okb_window_reserve: beyond the compiled-in limits"); return OKB_ERR_CAPACITY; }
  WinCaps& r = c->wins[win].reserve;
  r.K = max_frames; r.L = max_landmarks; r.O = max_observations; r.S = max_imu_samples; r.T = max_frames; r.MN = max_marg_dim;
  r.PP = std::max(r.PP, 4);
  return OKB_OK;
}

// Commits the pending commands of slots [first, first+count): H2D copies + interpreter + compile on the transfer stream.
static int commit_range(okb_ctx* c, int first, int count) {
  cudaSetDevice(c->device);
  cudaStream_t xs = c->stream_xfer;
  bool any = false;
  int max_work = 1;
  for (int i = first; i < first + count; ++i) {
    WinStore& S = c->wins[i];
    WinDev& W = c->host[i];
    W.cmd_bytes = 0; W.dirty = 0; W.full = 0;
    if (!S.cmd_used) continue;
    if (S.cmd_used > S.cmd_cap_dev) { c->set_error("pending window commands exceed the device command buffer (commit more often)"); return OKB_ERR_CAPACITY; }
    any = true;
    if (S.done_idx >= 0) OKB_CUDA(c, cudaStreamWaitEvent(xs, c->done_ring[S.done_idx], 0));   // solver work on this slot finishes first
    OKB_CUDA(c, cudaMemcpyAsync(const_cast<unsigned char*>(W.cmd), S.staging, S.cmd_used, cudaMemcpyHostToDevice, xs));
    OKB_CUDA(c, cudaEventRecord(S.copied, xs));
    S.staging_busy = true;
    S.h2d_bytes = S.cmd_used;
    W.cmd_bytes = (int)S.cmd_used; W.dirty = 1; W.full = S.full_pending ? 1 : 0;
    W.n_obs = S.obs_bound;
    S.cmd_used = 0; S.full_pending = false; S.committed = true;
    S.feat_n = S.feat_n_pending;
    max_work = std::max(max_work, std::max(std::max(W.n_obs, 4 * W.L), std::max(7 * W.K, 9 * W.NSB)));
  }
  if (!any) return OKB_OK;
  OKB_CUDA(c, cudaMemcpyAsync(c->d_wins + first, &c->host[first], sizeof(WinDev) * count, cudaMemcpyHostToDevice, xs));
  const int gx = std::max(1, std::min((max_work + 255) / 256, std::max(4, (8 * c->sm_count + count - 1) / count)));
  k_apply_commands<<<count, 1024, 0, xs>>>(c->d_wins, first);
  k_compile_obs<<<count, 1024, 0, xs>>>(c->d_wins, first);
  k_compile_sort<<<count, 1024, 0, xs>>>(c->d_wins, first);
  k_zero<<<dim3(gx, count), 256, 0, xs>>>(c->d_wins, first);
  k_prepare<<<dim3(gx, count), 256, 0, xs>>>(c->d_wins, first);
  c->launches += 5;
  OKB_CUDA(c, cudaGetLastError());
  for (int i = first; i < first + count; ++i) { c->host[i].cmd_bytes = 0; c->host[i].dirty = 0; c->host[i].full = 0; }
  return OKB_OK;
}

int okb_commit_windows(okb_ctx* c, const int32_t* wins, int n) {
  std::vector<int32_t> sorted(wins, wins + n);
  std::sort(sorted.begin(), sorted.end());
  const int rc = for_runs(sorted.data(), n, [&](int f, int m) { return commit_range(c, f, m); });
  if (rc) return rc;
  return wait_solver_work(c, c->stream_xfer, wins, n);
}

extern "C" int okb_window_commit(okb_ctx* c, int first, int count) {
  if (!c || first < 0 || count < 1 || first + count > c->max_windows) return OKB_ERR_INVALID_ARG;
  const int rc = commit_range(c, first, count);
  // landmark-sharded: the edits are applied before the call returns, so that no rank's graph compile is still queued
  // when a peer's solver kernels start spinning on the exchange (a rank whose commit ran beside them arrived seconds
  // late and its peers timed out)
  if (!rc && c->shard_world > 1) OKB_CUDA(c, cudaStreamSynchronize(c->stream_xfer));
  return rc;
}

// Full upload = a command stream that rebuilds the whole graph (host side: validation of what only the host can
// reject synchronously + one pass of memcpy into the pinned command buffer; sorting / slot tables / duplicate
// detection happen on the device).
// An IMU term's samples must cover [t0, t1] with t0 < t1 (ImuError.cpp:86-89 asserts the first and refuses the last).
// A term ending before t1 would never preintegrate and silently add nothing to every solve; one starting after t0
// would integrate a shorter interval than the Delta_t its residual uses.
static const char* imu_term_coverage(const okb_imu_term& T, const okb_imu_sample* s) {
  if (!(T.t1_ns > T.t0_ns)) return "t1 is not after t0";
  if (s[0].t_ns > T.t0_ns) return "first sample is after t0";
  if (s[T.sample_count - 1].t_ns < T.t1_ns) return "last sample is before t1";
  return nullptr;
}

static int upload_pack(okb_ctx* c, int win, const okb_window_desc* D) {
  if (!c || !D || win < 0 || win >= c->max_windows) return OKB_ERR_INVALID_ARG;
  cudaSetDevice(c->device);
  const int K = D->n_poses, NSB = D->n_speed_bias, NE = D->n_extrinsics, L = D->n_landmarks, NC = D->n_cameras;
  if (K < 1 || L < 1 || NC < 1 || NE < 1) { c->set_error("empty window"); return OKB_ERR_INVALID_ARG; }
  if (K > kMaxFrames || NSB > kMaxFrames) { c->set_error("more than 32 frames per window"); return OKB_ERR_CAPACITY; }
  for (int e = 0; e < NE; ++e)
    if (!D->extrinsics_fixed || !D->extrinsics_fixed[e]) {
      c->set_error("device solver requires fixed extrinsics (sigma_absolute_* = 0 as in the shipped configs)");
      return OKB_ERR_UNSUPPORTED;
    }
  if (D->n_relpose_terms > 0) { c->set_error("relative-pose terms need free extrinsics"); return OKB_ERR_UNSUPPORTED; }
  if (NC > 32) { c->set_error("more than 32 cameras"); return OKB_ERR_CAPACITY; }
  if (6 * K + 9 * NSB > kMaxDense) { c->set_error("reduced system too large"); return OKB_ERR_CAPACITY; }
  int marg_n = 0, marg_nb = 0, marg_xdim = 0;
  if (D->marg && D->marg->n > 0) {
    marg_n = D->marg->n; marg_nb = D->marg->n_blocks;
    if (marg_n > kMaxMarg || marg_nb > kMaxMargBlocks) { c->set_error("marginalisation prior too large"); return OKB_ERR_CAPACITY; }
    int col = 0;
    for (int b = 0; b < marg_nb; ++b) {
      const int kind = D->marg->block_kind[b];
      const uint32_t idx = D->marg->block_idx[b];
      const int lim = kind == OKB_BLOCK_POSE ? K : kind == OKB_BLOCK_SPEED_BIAS ? NSB : kind == OKB_BLOCK_EXTRINSICS ? NE : -1;
      if (lim < 0) { c->set_error("marginalisation prior: unknown block kind"); return OKB_ERR_INVALID_ARG; }
      if ((int)idx >= lim) { c->set_error("marginalisation prior: block index out of range"); return OKB_ERR_INVALID_ARG; }
      if (kind != OKB_BLOCK_EXTRINSICS) col += (kind == OKB_BLOCK_SPEED_BIAS) ? 9 : 6;
      marg_xdim += (kind == OKB_BLOCK_SPEED_BIAS) ? 9 : 7;
    }
    if (col != marg_n) { c->set_error("marginalisation prior dimension mismatch"); return OKB_ERR_INVALID_ARG; }
  }
  for (int i = 0; i < D->n_pose_priors; ++i)
    if ((int)D->pose_priors[i].pose_idx >= K) { c->set_error("pose prior index out of range"); return OKB_ERR_INVALID_ARG; }
  for (int i = 0; i < D->n_sb_priors; ++i)
    if ((int)D->sb_priors[i].sb_idx >= NSB) { c->set_error("speed/bias prior index out of range"); return OKB_ERR_INVALID_ARG; }
  for (int t = 0; t < D->n_imu_terms; ++t) {
    const okb_imu_term& T = D->imu_terms[t];
    if ((int)T.pose0 >= K || (int)T.pose1 >= K || (int)T.sb0 >= NSB || (int)T.sb1 >= NSB ||
        (uint64_t)T.sample_offset + (uint64_t)T.sample_count > (uint64_t)D->n_imu_samples || T.sample_count < 2) {
      c->set_error("IMU term index out of range");
      return OKB_ERR_INVALID_ARG;
    }
    if (const char* why = imu_term_coverage(T, D->imu_samples + T.sample_offset)) {
      c->set_error("IMU term " + std::to_string(t) + ": " + why);
      return OKB_ERR_INVALID_ARG;
    }
  }
  for (int i = 0; i < D->n_obs; ++i) {
    const okb_observation& ob = D->obs[i];
    if ((int)ob.pose_idx >= K || (int)ob.lm_idx >= L || (int)ob.ext_idx >= NE || (int)ob.cam_idx >= NC) {
      c->set_error("observation index out of range");
      return OKB_ERR_INVALID_ARG;
    }
    if (!(ob.sqrt_info > 0.0)) { c->set_error("observation with non-positive sqrt information"); return OKB_ERR_INVALID_ARG; }
  }
  if (smemA2_bytes(K, 0) > (size_t)c->smem_optin) { c->set_error("window does not fit kernel A shared memory"); return OKB_ERR_CAPACITY; }

  WinStore& S = c->wins[win];
  S.uploaded = false;        // true again only when the whole upload has been issued successfully
  WinCaps need{K, L, D->n_obs, D->n_imu_samples, D->n_imu_terms, NE, NC, std::max(D->n_pose_priors, D->n_sb_priors), marg_n};
  need = caps_max(need, S.reserve);
  need.T = std::max(need.T, need.K);
  if (!S.arena || !caps_cover(S.caps, need)) {
    if (S.done_idx >= 0) OKB_CUDA(c, cudaEventSynchronize(c->done_ring[S.done_idx]));    // the old arena may still be in use
    int rc = plan_arena(c, win, S.arena ? caps_max(S.caps, need) : need);
    if (rc) return rc;
  }
  // a full upload supersedes the graph edits still pending; feature-store edits are kept and follow it
  std::vector<unsigned char> store_cmds;
  for (size_t o = 0; S.feat_mem && o < S.cmd_used;) {
    CmdHeader h;
    std::memcpy(&h, S.staging + o, sizeof h);
    const size_t len = sizeof h + h.payload_bytes;
    if (h.op >= CMD_SET_FEATURES && h.op <= CMD_SET_LM_INIT) store_cmds.insert(store_cmds.end(), S.staging + o, S.staging + o + len);
    o += len;
  }
  S.cmd_used = 0;
  int rc = cmd_reserve(c, S, full_upload_bytes(need) + store_cmds.size());
  if (rc) return rc;
  unsigned char* q;
  q = cmd_put(S, CMD_RESET_GRAPH, 0, (uint32_t)NE, (uint32_t)NC, 8 * 7 * (size_t)NE + sizeof(okb_camera) * NC);
  std::memcpy(q, D->extrinsics, 8 * 7 * (size_t)NE);
  std::memcpy(q + 8 * 7 * (size_t)NE, D->cameras, sizeof(okb_camera) * NC);
  q = cmd_put(S, CMD_SET_FRAMES, 0, (uint32_t)K, (uint32_t)NSB, 8 * (7 * (size_t)K + 9 * (size_t)NSB));
  std::memcpy(q, D->poses, 8 * 7 * (size_t)K);
  if (NSB) std::memcpy(q + 8 * 7 * (size_t)K, D->speed_bias, 8 * 9 * (size_t)NSB);
  q = cmd_put(S, CMD_SET_LANDMARKS, (uint32_t)L, 0, 1, 8 * 4 * (size_t)L);
  std::memcpy(q, D->landmarks, 8 * 4 * (size_t)L);
  if (D->n_obs) {
    q = cmd_put(S, CMD_ADD_OBS, (uint32_t)D->n_obs, 0, 0, sizeof(okb_observation) * (size_t)D->n_obs);
    std::memcpy(q, D->obs, sizeof(okb_observation) * (size_t)D->n_obs);
  }
  q = cmd_put(S, CMD_SET_IMU, 0, (uint32_t)D->n_imu_terms, (uint32_t)D->n_imu_samples,
              sizeof(okb_imu_term) * D->n_imu_terms + sizeof(okb_imu_sample) * (size_t)D->n_imu_samples);
  if (D->n_imu_terms) std::memcpy(q, D->imu_terms, sizeof(okb_imu_term) * D->n_imu_terms);
  if (D->n_imu_samples) std::memcpy(q + sizeof(okb_imu_term) * D->n_imu_terms, D->imu_samples, sizeof(okb_imu_sample) * (size_t)D->n_imu_samples);
  q = cmd_put(S, CMD_SET_POSE_PRIORS, (uint32_t)D->n_pose_priors, 0, 0, sizeof(okb_pose_prior) * D->n_pose_priors);
  if (D->n_pose_priors) std::memcpy(q, D->pose_priors, sizeof(okb_pose_prior) * D->n_pose_priors);
  q = cmd_put(S, CMD_SET_SB_PRIORS, (uint32_t)D->n_sb_priors, 0, 0, sizeof(okb_sb_prior) * D->n_sb_priors);
  if (D->n_sb_priors) std::memcpy(q, D->sb_priors, sizeof(okb_sb_prior) * D->n_sb_priors);
  if (marg_n) {
    const size_t kb = align_up(4 * (size_t)marg_nb, 8);
    q = cmd_put(S, CMD_SET_MARG, 0, (uint32_t)marg_n, (uint32_t)marg_nb, 2 * kb + 8 * ((size_t)marg_xdim + (size_t)marg_n * marg_n + marg_n));
    std::memset(q, 0, 2 * kb);
    std::memcpy(q, D->marg->block_kind, 4 * (size_t)marg_nb);
    std::memcpy(q + kb, D->marg->block_idx, 4 * (size_t)marg_nb);
    double* x = reinterpret_cast<double*>(q + 2 * kb);
    std::memcpy(x, D->marg->x0, 8 * (size_t)marg_xdim);
    std::memcpy(x + marg_xdim, D->marg->J, 8 * (size_t)marg_n * marg_n);
    std::memcpy(x + marg_xdim + (size_t)marg_n * marg_n, D->marg->e0, 8 * (size_t)marg_n);
  }
  if (!store_cmds.empty()) { std::memcpy(S.staging + S.cmd_used, store_cmds.data(), store_cmds.size()); S.cmd_used += store_cmds.size(); }
  // host mirror of the dimensions
  WinDev& W = c->host[win];
  W.K = K; W.NSB = NSB; W.NE = NE; W.L = L; W.NC = NC;
  W.n_imu = D->n_imu_terms; W.n_samples = D->n_imu_samples; W.n_pp = D->n_pose_priors; W.n_sbp = D->n_sb_priors;
  W.marg_n = marg_n; W.marg_nb = marg_nb; W.marg_xdim = marg_xdim;
  W.imu_params = D->imu_params;
  derive_dims(W);
  W.shard_rank = c->shard_rank; W.shard_world = c->shard_world; W.shard_box_cap = c->shard_box_cap; W.shard_marg_cap = c->shard_marg_cap;
  W.shard_lm_cap = c->shard_lm_cap;
  if (c->shard_world > 1) {
    if (shard_box_doubles(K, W.dcp) > (size_t)c->shard_box_cap) { c->set_error("window exceeds the shard mailbox (max_frames of okb_shard_export)"); return OKB_ERR_CAPACITY; }
    for (int r = 0; r < c->shard_world; ++r) {
      if (!c->shard_peer[r]) { c->set_error("landmark sharding: okb_shard_connect has not been called"); return OKB_ERR_INVALID_ARG; }
      W.shard_mail[r] = c->shard_peer[r] + (size_t)win * c->shard_win_bytes;
    }
  }
  S.terms.assign(D->imu_terms, D->imu_terms + D->n_imu_terms);
  S.pp_idx.clear(); S.sbp_idx.clear();
  for (int i = 0; i < D->n_pose_priors; ++i) S.pp_idx.push_back(D->pose_priors[i].pose_idx);
  for (int i = 0; i < D->n_sb_priors; ++i) S.sbp_idx.push_back(D->sb_priors[i].sb_idx);
  S.obs_bound = D->n_obs;
  S.full_pending = true;
  S.K_init = K; S.NSB_init = NSB; S.L_init = L;
  S.cam_model = D->cameras[0].model;      // cameras enter a window only here (CMD_RESET_GRAPH)
  for (int i = 1; i < NC; ++i)
    if (D->cameras[i].model != S.cam_model) S.cam_model = kDistAny;
  if (S.cam_model < OKB_DIST_NONE || S.cam_model > OKB_DIST_RADTAN8) S.cam_model = kDistAny;
  S.uploaded = true;
  return OKB_OK;
}

extern "C" int okb_window_upload(okb_ctx* c, int win, const okb_window_desc* D) {
  int rc = upload_pack(c, win, D);
  if (rc) return rc;
  return commit_range(c, win, 1);
}

extern "C" int okb_window_upload_batch(okb_ctx* c, int first, int count, const okb_window_desc* descs, int host_threads) {
  if (!c || !descs || count < 1 || first < 0 || first + count > c->max_windows) return OKB_ERR_INVALID_ARG;
  const int T = std::max(1, std::min(host_threads > 0 ? host_threads : 8, count));
  std::vector<int> rcs(T, OKB_OK);      // per thread: its first error, after which it packs nothing more
  parallel_for(count, T, [&](int i) {
    int& rc = rcs[i % T];
    if (!rc) rc = upload_pack(c, first + i, descs + i);
  });
  for (int t = 0; t < T; ++t)
    if (rcs[t]) return rcs[t];
  return commit_range(c, first, count);
}

// ---------------------------------------------------------------------------------------------
// incremental graph updates (Estimator::addStates / addLandmark / addObservation / removeObservation / set_*,
// okvis_ceres/src/Estimator.cpp:110-413, implementation/Estimator.hpp:43-90): commands appended to the slot's
// pending stream; nothing touches the device until okb_window_commit / okb_optimize*.
// ---------------------------------------------------------------------------------------------
static int delta_begin(okb_ctx* c, int win, size_t extra, WinStore** S, WinDev** W) {
  if (!c || win < 0 || win >= c->max_windows) return OKB_ERR_INVALID_ARG;
  if (!c->wins[win].uploaded) { c->set_error("window slot not uploaded"); return OKB_ERR_INVALID_ARG; }
  cudaSetDevice(c->device);
  *S = &c->wins[win];
  *W = &c->host[win];
  return cmd_reserve(c, **S, extra + sizeof(CmdHeader) + 64);
}

extern "C" int okb_window_add_frame(okb_ctx* c, int win, const double* pose, const double* speed_bias, const okb_imu_term* term,
                                    const okb_imu_sample* samples, int n_samples) {
  WinStore* S; WinDev* W;
  if (!pose || (term && (!samples || n_samples < 2))) return OKB_ERR_INVALID_ARG;
  int rc = delta_begin(c, win, 16 * 8 + sizeof(okb_imu_term) + sizeof(okb_imu_sample) * (size_t)std::max(n_samples, 0) + sizeof(CmdHeader), &S, &W);
  if (rc) return rc;
  const int K1 = W->K + 1, NSB1 = W->NSB + (speed_bias ? 1 : 0);
  if (K1 > S->caps.K || NSB1 > S->caps.K || 6 * K1 + 9 * NSB1 > kMaxDense) { c->set_error("okb_window_add_frame: frame capacity exceeded (okb_window_reserve)"); return OKB_ERR_CAPACITY; }
  if (smemA2_bytes(K1, 0) > (size_t)c->smem_optin) { c->set_error("window does not fit kernel A shared memory"); return OKB_ERR_CAPACITY; }
  if (term) {
    if ((int)term->pose0 >= K1 || (int)term->pose1 >= K1 || (int)term->sb0 >= NSB1 || (int)term->sb1 >= NSB1 ||
        (uint64_t)term->sample_offset + term->sample_count > (uint64_t)n_samples || term->sample_count < 2) {
      c->set_error("IMU term index out of range");
      return OKB_ERR_INVALID_ARG;
    }
    if (const char* why = imu_term_coverage(*term, samples + term->sample_offset)) {
      c->set_error("IMU term " + std::to_string(W->n_imu) + ": " + why);
      return OKB_ERR_INVALID_ARG;
    }
    if (W->n_imu + 1 > S->caps.T || W->n_samples + n_samples > S->caps.S) { c->set_error("okb_window_add_frame: IMU capacity exceeded (okb_window_reserve)"); return OKB_ERR_CAPACITY; }
  }
  if (c->shard_world > 1 && shard_box_doubles(K1, 4 * ((6 * K1 + 1 + 3) / 4)) > (size_t)c->shard_box_cap) { c->set_error("window exceeds the shard mailbox"); return OKB_ERR_CAPACITY; }
  unsigned char* q = cmd_put(*S, CMD_ADD_FRAME, 0, 0, speed_bias ? 1u : 0u, 8 * 16);
  std::memcpy(q, pose, 56);
  if (speed_bias) std::memcpy(q + 56, speed_bias, 72); else std::memset(q + 56, 0, 72);
  W->K = K1; W->NSB = NSB1;
  if (term) {
    q = cmd_put(*S, CMD_ADD_IMU_TERM, (uint32_t)n_samples, 0, 0, sizeof(okb_imu_term) + sizeof(okb_imu_sample) * (size_t)n_samples);
    std::memcpy(q, term, sizeof(okb_imu_term));
    std::memcpy(q + sizeof(okb_imu_term), samples, sizeof(okb_imu_sample) * (size_t)n_samples);
    okb_imu_term mirror = *term;
    mirror.sample_offset += (uint32_t)W->n_samples;
    S->terms.push_back(mirror);
    W->n_imu += 1; W->n_samples += n_samples;
  }
  derive_dims(*W);
  return OKB_OK;
}

extern "C" int okb_window_remove_frame(okb_ctx* c, int win, uint32_t pose_idx, uint32_t sb_idx) {
  WinStore* S; WinDev* W;
  int rc = delta_begin(c, win, 0, &S, &W);
  if (rc) return rc;
  const bool has_sb = sb_idx != 0xffffffffu;
  if ((int)pose_idx >= W->K || (has_sb && (int)sb_idx >= W->NSB) || W->K < 2) { c->set_error("okb_window_remove_frame: index out of range"); return OKB_ERR_INVALID_ARG; }
  // the host mirror of the IMU term / prior counts needs the terms that touch the frame: it keeps a light copy
  cmd_put(*S, CMD_REMOVE_FRAME, 0, pose_idx, sb_idx, 0);
  int kept = 0, s_lo = 0x7fffffff, s_hi = 0;
  for (auto& T : S->terms) {
    const bool drop = T.pose0 == pose_idx || T.pose1 == pose_idx || (has_sb && (T.sb0 == sb_idx || T.sb1 == sb_idx));
    if (drop) continue;
    if (T.pose0 > pose_idx) T.pose0--;
    if (T.pose1 > pose_idx) T.pose1--;
    if (has_sb && T.sb0 > sb_idx) T.sb0--;
    if (has_sb && T.sb1 > sb_idx) T.sb1--;
    s_lo = std::min(s_lo, (int)T.sample_offset); s_hi = std::max(s_hi, (int)(T.sample_offset + T.sample_count));
    S->terms[kept++] = T;
  }
  S->terms.resize(kept);
  if (!kept) { s_lo = 0; s_hi = 0; }
  for (auto& T : S->terms) T.sample_offset -= (uint32_t)s_lo;
  W->n_imu = kept; W->n_samples = s_hi - s_lo;
  auto drop_priors = [](std::vector<uint32_t>& v, uint32_t idx) {
    size_t o = 0;
    for (size_t i = 0; i < v.size(); ++i) { if (v[i] == idx) continue; v[o++] = v[i] > idx ? v[i] - 1 : v[i]; }
    v.resize(o);
  };
  drop_priors(S->pp_idx, pose_idx);
  if (has_sb) drop_priors(S->sbp_idx, sb_idx);
  W->n_pp = (int)S->pp_idx.size(); W->n_sbp = (int)S->sbp_idx.size();
  W->K -= 1;
  if (has_sb) W->NSB -= 1;
  derive_dims(*W);
  return OKB_OK;
}

extern "C" int okb_window_set_landmarks(okb_ctx* c, int win, int n, const uint32_t* idx, const double* xyzw) {
  WinStore* S; WinDev* W;
  if (n < 1 || !idx || !xyzw) return OKB_ERR_INVALID_ARG;
  int rc = delta_begin(c, win, align_up(4 * (size_t)n, 8) + 32 * (size_t)n, &S, &W);
  if (rc) return rc;
  int L = W->L;
  for (int i = 0; i < n; ++i) {
    if ((int)idx[i] >= S->caps.L) { c->set_error("okb_window_set_landmarks: landmark capacity exceeded (okb_window_reserve)"); return OKB_ERR_CAPACITY; }
    L = std::max(L, (int)idx[i] + 1);
  }
  const size_t ib = align_up(4 * (size_t)n, 8);
  unsigned char* q = cmd_put(*S, CMD_SET_LANDMARKS, (uint32_t)n, 0, 0, ib + 32 * (size_t)n);
  std::memset(q, 0, ib);
  std::memcpy(q, idx, 4 * (size_t)n);
  std::memcpy(q + ib, xyzw, 32 * (size_t)n);
  W->L = L;
  derive_dims(*W);
  return OKB_OK;
}

extern "C" int okb_window_remove_landmarks(okb_ctx* c, int win, int n, const uint32_t* idx) {
  WinStore* S; WinDev* W;
  if (n < 1 || !idx) return OKB_ERR_INVALID_ARG;
  int rc = delta_begin(c, win, 4 * (size_t)n + 8, &S, &W);
  if (rc) return rc;
  for (int i = 0; i < n; ++i)
    if ((int)idx[i] >= W->L) { c->set_error("okb_window_remove_landmarks: index out of range"); return OKB_ERR_INVALID_ARG; }
  unsigned char* q = cmd_put(*S, CMD_REMOVE_LANDMARKS, (uint32_t)n, 0, 0, 4 * (size_t)n);
  std::memcpy(q, idx, 4 * (size_t)n);
  return OKB_OK;
}

extern "C" int okb_window_add_observations(okb_ctx* c, int win, int n, const okb_observation* obs) {
  WinStore* S; WinDev* W;
  if (n < 1 || !obs) return OKB_ERR_INVALID_ARG;
  int rc = delta_begin(c, win, sizeof(okb_observation) * (size_t)n, &S, &W);
  if (rc) return rc;
  for (int i = 0; i < n; ++i) {
    const okb_observation& ob = obs[i];
    if ((int)ob.pose_idx >= W->K || (int)ob.lm_idx >= W->L || (int)ob.ext_idx >= W->NE || (int)ob.cam_idx >= W->NC) { c->set_error("observation index out of range"); return OKB_ERR_INVALID_ARG; }
    if (!(ob.sqrt_info > 0.0)) { c->set_error("observation with non-positive sqrt information"); return OKB_ERR_INVALID_ARG; }
  }
  if (S->obs_bound + n > S->caps.O) { c->set_error("okb_window_add_observations: observation capacity exceeded (okb_window_reserve)"); return OKB_ERR_CAPACITY; }
  unsigned char* q = cmd_put(*S, CMD_ADD_OBS, (uint32_t)n, 0, 0, sizeof(okb_observation) * (size_t)n);
  std::memcpy(q, obs, sizeof(okb_observation) * (size_t)n);
  S->obs_bound += n;
  return OKB_OK;
}

extern "C" int okb_window_remove_observations(okb_ctx* c, int win, int n, const okb_obs_key* keys) {
  WinStore* S; WinDev* W;
  if (n < 1 || !keys) return OKB_ERR_INVALID_ARG;
  int rc = delta_begin(c, win, sizeof(okb_obs_key) * (size_t)n, &S, &W);
  if (rc) return rc;
  for (int i = 0; i < n; ++i)
    if ((int)keys[i].pose_idx >= W->K || (int)keys[i].lm_idx >= W->L || (int)keys[i].cam_idx >= W->NC) { c->set_error("observation key out of range"); return OKB_ERR_INVALID_ARG; }
  unsigned char* q = cmd_put(*S, CMD_REMOVE_OBS, (uint32_t)n, 0, 0, sizeof(okb_obs_key) * (size_t)n);
  std::memcpy(q, keys, sizeof(okb_obs_key) * (size_t)n);
  return OKB_OK;
}

extern "C" int okb_window_set_states(okb_ctx* c, int win, int n_poses, const uint32_t* pose_idx, const double* poses, int n_sb,
                                     const uint32_t* sb_idx, const double* speed_bias) {
  WinStore* S; WinDev* W;
  if (n_poses < 0 || n_sb < 0 || (n_poses && (!pose_idx || !poses)) || (n_sb && (!sb_idx || !speed_bias))) return OKB_ERR_INVALID_ARG;
  int rc = delta_begin(c, win, (sizeof(CmdHeader) + 72) * (size_t)(n_poses + n_sb), &S, &W);
  if (rc) return rc;
  for (int i = 0; i < n_poses; ++i) if ((int)pose_idx[i] >= W->K) { c->set_error("okb_window_set_states: pose index out of range"); return OKB_ERR_INVALID_ARG; }
  for (int i = 0; i < n_sb; ++i) if ((int)sb_idx[i] >= W->NSB) { c->set_error("okb_window_set_states: speed/bias index out of range"); return OKB_ERR_INVALID_ARG; }
  for (int i = 0; i < n_poses; ++i) std::memcpy(cmd_put(*S, CMD_SET_POSE, 0, pose_idx[i], 0, 56), poses + 7 * (size_t)i, 56);
  for (int i = 0; i < n_sb; ++i) std::memcpy(cmd_put(*S, CMD_SET_SB, 0, sb_idx[i], 0, 72), speed_bias + 9 * (size_t)i, 72);
  return OKB_OK;
}

extern "C" int okb_window_set_priors(okb_ctx* c, int win, int n_pose_priors, const okb_pose_prior* pose_priors, int n_sb_priors,
                                     const okb_sb_prior* sb_priors, const okb_marg_prior* marg) {
  WinStore* S; WinDev* W;
  if (n_pose_priors < 0 || n_sb_priors < 0) return OKB_ERR_INVALID_ARG;
  const int mn = marg ? marg->n : 0, mnb = marg ? marg->n_blocks : 0;
  int rc = delta_begin(c, win, sizeof(okb_pose_prior) * (size_t)n_pose_priors + sizeof(okb_sb_prior) * (size_t)n_sb_priors + 3 * sizeof(CmdHeader) +
                                   8 * ((size_t)mn * mn + mn + 11 * (size_t)mnb + 8), &S, &W);
  if (rc) return rc;
  if (n_pose_priors > S->caps.PP || n_sb_priors > S->caps.PP) { c->set_error("okb_window_set_priors: more priors than reserved"); return OKB_ERR_CAPACITY; }
  for (int i = 0; i < n_pose_priors; ++i) if ((int)pose_priors[i].pose_idx >= W->K) { c->set_error("pose prior index out of range"); return OKB_ERR_INVALID_ARG; }
  for (int i = 0; i < n_sb_priors; ++i) if ((int)sb_priors[i].sb_idx >= W->NSB) { c->set_error("speed/bias prior index out of range"); return OKB_ERR_INVALID_ARG; }
  int xdim = 0;
  if (marg) {
    if (mn > S->caps.MN || mn > kMaxMarg || mnb > kMaxMargBlocks || mn < 0) { c->set_error("okb_window_set_priors: marginalisation prior larger than reserved"); return OKB_ERR_CAPACITY; }
    int col = 0;
    for (int b = 0; b < mnb; ++b) {
      const int kind = marg->block_kind[b];
      const int lim = kind == OKB_BLOCK_POSE ? W->K : kind == OKB_BLOCK_SPEED_BIAS ? W->NSB : kind == OKB_BLOCK_EXTRINSICS ? W->NE : -1;
      if (lim < 0 || (int)marg->block_idx[b] >= lim) { c->set_error("marginalisation prior: bad block"); return OKB_ERR_INVALID_ARG; }
      if (kind != OKB_BLOCK_EXTRINSICS) col += (kind == OKB_BLOCK_SPEED_BIAS) ? 9 : 6;
      xdim += (kind == OKB_BLOCK_SPEED_BIAS) ? 9 : 7;
    }
    if (col != mn) { c->set_error("marginalisation prior dimension mismatch"); return OKB_ERR_INVALID_ARG; }
  }
  unsigned char* q = cmd_put(*S, CMD_SET_POSE_PRIORS, (uint32_t)n_pose_priors, 0, 0, sizeof(okb_pose_prior) * (size_t)n_pose_priors);
  if (n_pose_priors) std::memcpy(q, pose_priors, sizeof(okb_pose_prior) * (size_t)n_pose_priors);
  q = cmd_put(*S, CMD_SET_SB_PRIORS, (uint32_t)n_sb_priors, 0, 0, sizeof(okb_sb_prior) * (size_t)n_sb_priors);
  if (n_sb_priors) std::memcpy(q, sb_priors, sizeof(okb_sb_prior) * (size_t)n_sb_priors);
  S->pp_idx.clear(); S->sbp_idx.clear();
  for (int i = 0; i < n_pose_priors; ++i) S->pp_idx.push_back(pose_priors[i].pose_idx);
  for (int i = 0; i < n_sb_priors; ++i) S->sbp_idx.push_back(sb_priors[i].sb_idx);
  W->n_pp = n_pose_priors; W->n_sbp = n_sb_priors;
  if (marg) {
    const size_t kb = align_up(4 * (size_t)mnb, 8);
    q = cmd_put(*S, CMD_SET_MARG, 0, (uint32_t)mn, (uint32_t)mnb, 2 * kb + 8 * ((size_t)xdim + (size_t)mn * mn + mn));
    std::memset(q, 0, 2 * kb);
    if (mnb) { std::memcpy(q, marg->block_kind, 4 * (size_t)mnb); std::memcpy(q + kb, marg->block_idx, 4 * (size_t)mnb); }
    double* x = reinterpret_cast<double*>(q + 2 * kb);
    if (xdim) std::memcpy(x, marg->x0, 8 * (size_t)xdim);
    if (mn) { std::memcpy(x + xdim, marg->J, 8 * (size_t)mn * mn); std::memcpy(x + xdim + (size_t)mn * mn, marg->e0, 8 * (size_t)mn); }
    W->marg_n = mn; W->marg_nb = mnb; W->marg_xdim = xdim;
  }
  return OKB_OK;
}

extern "C" int okb_window_remove_speed_bias(okb_ctx* c, int win, uint32_t sb_idx) {
  WinStore* S; WinDev* W;
  int rc = delta_begin(c, win, 0, &S, &W);
  if (rc) return rc;
  if ((int)sb_idx >= W->NSB) { c->set_error("okb_window_remove_speed_bias: index out of range"); return OKB_ERR_INVALID_ARG; }
  cmd_put(*S, CMD_REMOVE_SB, 0, sb_idx, 0, 0);
  int kept = 0, s_lo = 0x7fffffff, s_hi = 0;
  for (auto& T : S->terms) {
    if (T.sb0 == sb_idx || T.sb1 == sb_idx) continue;
    if (T.sb0 > sb_idx) T.sb0--;
    if (T.sb1 > sb_idx) T.sb1--;
    s_lo = std::min(s_lo, (int)T.sample_offset); s_hi = std::max(s_hi, (int)(T.sample_offset + T.sample_count));
    S->terms[kept++] = T;
  }
  S->terms.resize(kept);
  if (!kept) { s_lo = 0; s_hi = 0; }
  for (auto& T : S->terms) T.sample_offset -= (uint32_t)s_lo;
  W->n_imu = kept; W->n_samples = s_hi - s_lo;
  size_t o = 0;
  for (size_t i = 0; i < S->sbp_idx.size(); ++i) { if (S->sbp_idx[i] == sb_idx) continue; S->sbp_idx[o++] = S->sbp_idx[i] > sb_idx ? S->sbp_idx[i] - 1 : S->sbp_idx[i]; }
  S->sbp_idx.resize(o);
  W->n_sbp = (int)o;
  W->NSB -= 1;
  derive_dims(*W);
  return OKB_OK;
}

// ---------------------------------------------------------------------------------------------
// feature store of okb_track_3d2d_batch (FeatStore, okb_estimator.cuh); edits are graph commands like the others
// ---------------------------------------------------------------------------------------------
extern "C" int okb_window_reserve_features(okb_ctx* c, int win, int max_feature_frames, int max_cameras, int max_keypoints, int desc_bytes) {
  if (!c || win < 0 || win >= c->max_windows || max_feature_frames < 1 || max_cameras < 1 || max_keypoints < 1) return OKB_ERR_INVALID_ARG;
  if (desc_bytes != 32 && desc_bytes != 48 && desc_bytes != 64 && desc_bytes != 128) {
    c->set_error("okb_window_reserve_features: descriptor length must be 32, 48, 64 or 128 bytes");
    return OKB_ERR_INVALID_ARG;
  }
  if (max_keypoints > 65535 || max_cameras > 127) {     // the result records of okb_track_3d2d_batch pack them
    c->set_error("okb_window_reserve_features: at most 65535 keypoints per image and 127 cameras");
    return OKB_ERR_CAPACITY;
  }
  WinStore& S = c->wins[win];
  const int lm_cap = std::max(S.reserve.L, S.caps.L);
  if (lm_cap < 1) { c->set_error("okb_window_reserve_features: reserve or upload the window first"); return OKB_ERR_INVALID_ARG; }
  cudaSetDevice(c->device);
  const FeatStore& o = S.feat;
  if (S.feat_mem && o.F == max_feature_frames && o.C == max_cameras && o.N == max_keypoints && o.D == desc_bytes && o.lm_cap == lm_cap)
    return OKB_OK;
  const size_t pad8 = 7;
  const size_t frame_bytes = (size_t)max_cameras * (sizeof(CmdHeader) + 24 * (size_t)max_keypoints + (4 * (size_t)max_keypoints + pad8) +
                                                    ((size_t)max_keypoints + pad8) + ((size_t)max_keypoints * desc_bytes + pad8)) +
                             sizeof(CmdHeader) + 5 * (size_t)lm_cap + 2 * pad8;
  if (S.arena && S.cmd_cap_dev < align_up(full_upload_bytes(S.caps) + frame_bytes + 65536, 256)) {
    c->set_error("okb_window_reserve_features: the window's command buffer was planned without a feature store: reserve the "
                 "features before the slot's first upload");
    return OKB_ERR_CAPACITY;
  }
  if (S.feat_mem) {                     // replaced: commands already queued for the old store must not reach the new one
    if (S.cmd_used) { const int rc = commit_range(c, win, 1); if (rc) return rc; }
    OKB_CUDA(c, cudaStreamSynchronize(c->stream_xfer));
    if (S.done_idx >= 0) OKB_CUDA(c, cudaEventSynchronize(c->done_ring[S.done_idx]));
    OKB_CUDA(c, cudaFree(S.feat_mem));
    S.feat_mem = nullptr;
  }
  const size_t images = (size_t)max_feature_frames * max_cameras, kps = images * max_keypoints;
  Carve P;
  P.take(sizeof(FeatStore), 256);
  const size_t o_n = P.take(4 * images, 256), o_kp = P.take(16 * kps, 256), o_size = P.take(8 * kps, 256);
  const size_t o_desc = P.take(kps * desc_bytes, 256), o_lm = P.take(4 * kps, 256), o_obs = P.take(kps, 256);
  const size_t o_init = P.take((size_t)lm_cap, 256);
  unsigned char* m = nullptr;
  OKB_CUDA(c, cudaMalloc(&m, P.off));
  FeatStore F{};
  F.F = max_feature_frames; F.C = max_cameras; F.N = max_keypoints; F.D = desc_bytes; F.lm_cap = lm_cap;
  F.n = reinterpret_cast<int*>(m + o_n); F.kp = reinterpret_cast<double*>(m + o_kp); F.size = reinterpret_cast<double*>(m + o_size);
  F.desc = reinterpret_cast<uint32_t*>(m + o_desc); F.lm = reinterpret_cast<int32_t*>(m + o_lm); F.observed = m + o_obs; F.lm_init = m + o_init;
  cudaStream_t xs = c->stream_xfer;
  OKB_CUDA(c, cudaMemsetAsync(m + o_n, 0xff, 4 * images, xs));                 // n = -1: no image
  OKB_CUDA(c, cudaMemsetAsync(m + o_lm, 0xff, 4 * kps, xs));                   // lm = -1
  OKB_CUDA(c, cudaMemsetAsync(m + o_obs, 0, o_init + lm_cap - o_obs, xs));      // observed bits, initialised flags
  S.feat = F;
  S.feat_mem = m;
  S.feat_frame_bytes = frame_bytes;
  OKB_CUDA(c, cudaMemcpyAsync(m, &S.feat, sizeof(FeatStore), cudaMemcpyHostToDevice, xs));
  S.feat_n.assign(images, -1);
  S.feat_n_pending.assign(images, -1);
  FeatStore* dp = reinterpret_cast<FeatStore*>(m);
  c->host[win].feat = dp;
  OKB_CUDA(c, cudaMemcpyAsync(&c->d_wins[win].feat, &c->host[win].feat, sizeof(dp), cudaMemcpyHostToDevice, xs));
  OKB_CUDA(c, cudaStreamSynchronize(xs));
  return OKB_OK;
}

// A landmark-sharded store names global landmark slots: each must lie below the replica's global slot count.
static int store_slots_invalid(okb_ctx* c, const int32_t* lm_slot, int n, const char* who) {
  if (c->shard_world < 2 || !lm_slot) return OKB_OK;
  for (int i = 0; i < n; ++i)
    if (lm_slot[i] >= c->shard_lm_cap) {
      c->set_error(std::string(who) + ": landmark slot beyond the sharded window's global landmark slots (okb_shard_reserve_landmarks)");
      return OKB_ERR_INVALID_ARG;
    }
  return OKB_OK;
}

static int feat_begin(okb_ctx* c, int win, int feat_slot, int cam, size_t extra, WinStore** S, WinDev** W, const char* who) {
  int rc = delta_begin(c, win, extra, S, W);
  if (rc) return rc;
  const FeatStore& F = (*S)->feat;
  if (!(*S)->feat_mem) { c->set_error(std::string(who) + ": no feature store (okb_window_reserve_features)"); return OKB_ERR_INVALID_ARG; }
  if (feat_slot < 0 || feat_slot >= F.F || cam < 0 || cam >= F.C) { c->set_error(std::string(who) + ": feature slot or camera out of range"); return OKB_ERR_INVALID_ARG; }
  return OKB_OK;
}

extern "C" int okb_window_set_features(okb_ctx* c, int win, int feat_slot, int cam, int n, const okb_keypoint* kp, const uint8_t* desc,
                                       const int32_t* lm_slot, const uint8_t* observed) {
  if (!c || n < 0 || (n > 0 && (!kp || !desc))) return OKB_ERR_INVALID_ARG;
  const int D = (win >= 0 && win < c->max_windows) ? c->wins[win].feat.D : 0;
  const size_t bk = 24 * (size_t)n, bl = align_up(4 * (size_t)n, 8), bo = align_up((size_t)n, 8), bd = align_up((size_t)n * D, 8);
  WinStore* S; WinDev* W;
  int rc = feat_begin(c, win, feat_slot, cam, bk + bl + bo + bd, &S, &W, "okb_window_set_features");
  if (rc) return rc;
  if (n > S->feat.N) { c->set_error("okb_window_set_features: more keypoints than reserved"); return OKB_ERR_CAPACITY; }
  for (int i = 0; lm_slot && i < n; ++i)
    if (lm_slot[i] < -1) { c->set_error("okb_window_set_features: landmark slot below -1"); return OKB_ERR_INVALID_ARG; }
  if ((rc = store_slots_invalid(c, lm_slot, n, "okb_window_set_features"))) return rc;
  unsigned char* q = cmd_put(*S, CMD_SET_FEATURES, (uint32_t)n, (uint32_t)feat_slot, (uint32_t)cam, bk + bl + bo + bd);
  double* x = reinterpret_cast<double*>(q);
  for (int i = 0; i < n; ++i) { x[3 * i] = kp[i].x; x[3 * i + 1] = kp[i].y; x[3 * i + 2] = kp[i].size; }
  int32_t* l = reinterpret_cast<int32_t*>(q + bk);
  for (int i = 0; i < n; ++i) l[i] = lm_slot ? lm_slot[i] : -1;
  if (observed) std::memcpy(q + bk + bl, observed, n); else std::memset(q + bk + bl, 0, n);
  if (n) std::memcpy(q + bk + bl + bo, desc, (size_t)n * D);
  S->feat_n_pending[(size_t)feat_slot * S->feat.C + cam] = n;
  return OKB_OK;
}

extern "C" int okb_window_set_feature_landmarks(okb_ctx* c, int win, int feat_slot, int cam, int n, const int32_t* kp_idx,
                                                const int32_t* lm_slot, const uint8_t* observed) {
  if (!c || n < 1 || !kp_idx || !lm_slot || !observed) return OKB_ERR_INVALID_ARG;
  const size_t b4 = align_up(4 * (size_t)n, 8), b1 = align_up((size_t)n, 8);
  WinStore* S; WinDev* W;
  int rc = feat_begin(c, win, feat_slot, cam, 2 * b4 + b1, &S, &W, "okb_window_set_feature_landmarks");
  if (rc) return rc;
  const int nk = S->feat_n_pending[(size_t)feat_slot * S->feat.C + cam];
  for (int i = 0; i < n; ++i)
    if (kp_idx[i] < 0 || kp_idx[i] >= nk || lm_slot[i] < -1) {
      c->set_error("okb_window_set_feature_landmarks: keypoint index or landmark slot out of range");
      return OKB_ERR_INVALID_ARG;
    }
  if ((rc = store_slots_invalid(c, lm_slot, n, "okb_window_set_feature_landmarks"))) return rc;
  unsigned char* q = cmd_put(*S, CMD_SET_FEATURE_LMS, (uint32_t)n, (uint32_t)feat_slot, (uint32_t)cam, 2 * b4 + b1);
  std::memcpy(q, kp_idx, 4 * (size_t)n);
  std::memcpy(q + b4, lm_slot, 4 * (size_t)n);
  std::memcpy(q + 2 * b4, observed, n);
  return OKB_OK;
}

extern "C" int okb_window_clear_features(okb_ctx* c, int win, int feat_slot) {
  WinStore* S; WinDev* W;
  int rc = feat_begin(c, win, feat_slot, 0, 0, &S, &W, "okb_window_clear_features");
  if (rc) return rc;
  cmd_put(*S, CMD_CLEAR_FEATURES, 0, (uint32_t)feat_slot, 0, 0);
  for (int k = 0; k < S->feat.C; ++k) S->feat_n_pending[(size_t)feat_slot * S->feat.C + k] = -1;
  return OKB_OK;
}

extern "C" int okb_window_set_landmark_initialized(okb_ctx* c, int win, int n, const uint32_t* idx, const uint8_t* flags) {
  if (!c || n < 1 || !idx || !flags) return OKB_ERR_INVALID_ARG;
  const size_t b4 = align_up(4 * (size_t)n, 8), b1 = align_up((size_t)n, 8);
  WinStore* S; WinDev* W;
  int rc = feat_begin(c, win, 0, 0, b4 + b1, &S, &W, "okb_window_set_landmark_initialized");
  if (rc) return rc;
  for (int i = 0; i < n; ++i)
    if ((int64_t)idx[i] >= S->feat.lm_cap) { c->set_error("okb_window_set_landmark_initialized: slot beyond the store's landmark capacity"); return OKB_ERR_CAPACITY; }
  unsigned char* q = cmd_put(*S, CMD_SET_LM_INIT, (uint32_t)n, 0, 0, b4 + b1);
  std::memcpy(q, idx, 4 * (size_t)n);
  std::memcpy(q + b4, flags, n);
  return OKB_OK;
}

extern "C" int okb_debug_features(okb_ctx* c, int win, int feat_slot, int cam, int32_t* n, double* kp, double* size, uint8_t* desc,
                                  int32_t* lm_slot, uint8_t* observed) {
  if (!c || win < 0 || win >= c->max_windows || !n) return OKB_ERR_INVALID_ARG;
  const WinStore& S = c->wins[win];
  const FeatStore& F = S.feat;
  if (!S.feat_mem) { c->set_error("okb_debug_features: no feature store (okb_window_reserve_features)"); return OKB_ERR_INVALID_ARG; }
  if (feat_slot < 0 || feat_slot >= F.F || cam < 0 || cam >= F.C) { c->set_error("okb_debug_features: feature slot or camera out of range"); return OKB_ERR_INVALID_ARG; }
  cudaSetDevice(c->device);
  OKB_CUDA(c, cudaStreamSynchronize(c->stream_xfer));     // commits (and the store calls, which block) run there
  const size_t img = (size_t)feat_slot * F.C + cam, base = img * F.N;
  int32_t m = -1;
  OKB_CUDA(c, cudaMemcpy(&m, F.n + img, sizeof m, cudaMemcpyDeviceToHost));
  *n = m;
  if (m <= 0) return OKB_OK;
  if (kp) OKB_CUDA(c, cudaMemcpy(kp, F.kp + 2 * base, 16 * (size_t)m, cudaMemcpyDeviceToHost));
  if (size) OKB_CUDA(c, cudaMemcpy(size, F.size + base, 8 * (size_t)m, cudaMemcpyDeviceToHost));
  if (desc) OKB_CUDA(c, cudaMemcpy(desc, F.desc + base * (F.D / 4), (size_t)m * F.D, cudaMemcpyDeviceToHost));
  if (lm_slot) OKB_CUDA(c, cudaMemcpy(lm_slot, F.lm + base, 4 * (size_t)m, cudaMemcpyDeviceToHost));
  if (observed) OKB_CUDA(c, cudaMemcpy(observed, F.observed + base, (size_t)m, cudaMemcpyDeviceToHost));
  return OKB_OK;
}

// ---------------------------------------------------------------------------------------------
// device-side marginalisation (okb_marg.cuh): MarginalizationError::addResidualBlock / marginalizeOut /
// updateErrorComputation (okvis_ceres/src/MarginalizationError.cpp:127-435, 507-846)
// ---------------------------------------------------------------------------------------------
static int check_range(okb_ctx* c, int first, int count);
namespace {
constexpr int kMargImuCap = 32, kMargSbpCap = 8;
// Work arrays and status word of one slot (WinStore::marg_scratch).
struct MargLayout { size_t H, b, A, Q, T, Hn, bn, xlin, lmrec, lmV, lmvis, lmslot, clist, status, total; };
MargLayout marg_layout(int lm_cap, int K_cap, int L_cap, int O_cap) {
  MargLayout m;
  Carve P;
  const size_t NN = (size_t)kMargWork * kMargWork * 8;
  m.H = P.take(NN); m.b = P.take(8 * kMargWork); m.A = P.take(NN); m.Q = P.take(NN); m.T = P.take(NN); m.Hn = P.take(NN);
  m.bn = P.take(8 * kMargWork); m.xlin = P.take(8 * 9 * kMaxMargBlocks);
  m.lmrec = P.take(8 * (size_t)lm_cap * K_cap * kMargRec); m.lmV = P.take(8 * 16 * (size_t)lm_cap); m.lmvis = P.take(4 * (size_t)lm_cap);
  m.lmslot = P.take(4 * (size_t)std::max(L_cap, 1)); m.clist = P.take(4 * (size_t)std::max(O_cap, 1)); m.status = P.take(16);
  m.total = P.off;
  return m;
}
// One job in the batch buffer of a call: header, then its index lists.
struct MargPayload { size_t kind, idx, prev, marg, imu, sbp, lms, total; };
MargPayload marg_payload(const okb_marg_job* job) {
  MargPayload p;
  Carve P;
  P.take(sizeof(MargJobHeader));
  const size_t nb = (size_t)job->n_blocks;
  p.kind = P.take(4 * nb); p.idx = P.take(4 * nb); p.prev = P.take(4 * nb); p.marg = P.take(nb);
  p.imu = P.take(4 * (size_t)job->n_imu_terms); p.sbp = P.take(4 * (size_t)job->n_sb_priors); p.lms = P.take(4 * (size_t)job->n_landmarks);
  p.total = P.off;
  return p;
}
MargScratch marg_pointers(unsigned char* job, const MargPayload& p, unsigned char* base, const MargLayout& m) {
  MargScratch sc;
  sc.hdr = reinterpret_cast<MargJobHeader*>(job);
  sc.kind = reinterpret_cast<int32_t*>(job + p.kind); sc.idx = reinterpret_cast<uint32_t*>(job + p.idx);
  sc.prev = reinterpret_cast<int32_t*>(job + p.prev); sc.marg = job + p.marg;
  sc.imu_terms = reinterpret_cast<uint32_t*>(job + p.imu); sc.sb_priors = reinterpret_cast<uint32_t*>(job + p.sbp);
  sc.landmarks = reinterpret_cast<uint32_t*>(job + p.lms);
  auto dp = [&](size_t o) { return reinterpret_cast<double*>(base + o); };
  sc.H = dp(m.H); sc.b = dp(m.b); sc.A = dp(m.A); sc.Q = dp(m.Q); sc.T = dp(m.T); sc.Hn = dp(m.Hn); sc.bn = dp(m.bn); sc.xlin = dp(m.xlin);
  sc.lmrec = dp(m.lmrec); sc.lmV = dp(m.lmV); sc.lmvis = reinterpret_cast<uint32_t*>(base + m.lmvis);
  sc.lmslot = reinterpret_cast<int32_t*>(base + m.lmslot); sc.clist = reinterpret_cast<int32_t*>(base + m.clist);
  sc.status = reinterpret_cast<int32_t*>(base + m.status);
  return sc;
}

// Dimensions of a job that passed marg_check.
struct MargDims { int N = 0, n_keep = 0, nb_keep = 0, xdim = 0; };
// Host checks of one job against the slot as the host mirror describes it (pending edits included).  On failure
// returns the status and sets *why.
int marg_check(const okb_ctx* c, int win, const okb_marg_job* job, MargDims& d, const char** why) {
  if (!c->wins[win].uploaded) { *why = "window slot not uploaded"; return OKB_ERR_INVALID_ARG; }
  const WinStore& S = c->wins[win];
  const WinDev& W = c->host[win];
  if (job->n_blocks < 1 || job->n_blocks > kMaxMargBlocks || job->n_imu_terms < 0 || job->n_imu_terms > kMargImuCap || job->n_sb_priors < 0 ||
      job->n_sb_priors > kMargSbpCap || job->n_landmarks < 0 || !job->block_kind || !job->block_idx || !job->block_prev || !job->block_marginalize ||
      (job->n_imu_terms && !job->imu_terms) || (job->n_sb_priors && !job->sb_priors) || (job->n_landmarks && !job->landmarks)) {
    *why = "malformed job";
    return OKB_ERR_INVALID_ARG;
  }
  d = MargDims();
  for (int b = 0; b < job->n_blocks; ++b) {
    const int kind = job->block_kind[b];
    if (kind != OKB_BLOCK_POSE && kind != OKB_BLOCK_SPEED_BIAS) { *why = "block kind must be pose or speed/bias (extrinsics are fixed)"; return OKB_ERR_UNSUPPORTED; }
    const int lim = kind == OKB_BLOCK_POSE ? W.K : W.NSB;
    if ((int)job->block_idx[b] >= lim || job->block_prev[b] < -1 || job->block_prev[b] >= W.marg_nb) { *why = "block index out of range"; return OKB_ERR_INVALID_ARG; }
    const int dim = kind == OKB_BLOCK_SPEED_BIAS ? 9 : 6;
    d.N += dim;
    if (!job->block_marginalize[b]) { d.n_keep += dim; d.nb_keep += 1; d.xdim += (kind == OKB_BLOCK_SPEED_BIAS) ? 9 : 7; }
  }
  for (int i = 0; i < job->n_imu_terms; ++i) if ((int)job->imu_terms[i] >= W.n_imu) { *why = "IMU term index out of range"; return OKB_ERR_INVALID_ARG; }
  for (int i = 0; i < job->n_sb_priors; ++i) if ((int)job->sb_priors[i] >= W.n_sbp) { *why = "prior index out of range"; return OKB_ERR_INVALID_ARG; }
  for (int i = 0; i < job->n_landmarks; ++i) if ((int)job->landmarks[i] >= W.L) { *why = "landmark index out of range"; return OKB_ERR_INVALID_ARG; }
  if (d.N > kMargWork) { *why = "linear system larger than the compiled-in limit"; return OKB_ERR_CAPACITY; }
  if (d.n_keep > kMaxMarg || d.n_keep > S.caps.MN) { *why = "resulting prior larger than reserved (okb_window_reserve max_marg_dim)"; return OKB_ERR_CAPACITY; }
  return OKB_OK;
}

// FNV-1a over the part of a job every rank of a landmark-sharded window must share: N, n_keep, the block lists, the
// IMU-term and speed/bias-prior lists (each with its length).  The landmark list is the rank's own and is left out.
uint64_t marg_job_fingerprint(const okb_marg_job* job) {
  uint64_t h = 1469598103934665603ull;
  auto mix = [&](const void* p, size_t bytes) {
    const unsigned char* b = static_cast<const unsigned char*>(p);
    for (size_t i = 0; i < bytes; ++i) { h ^= b[i]; h *= 1099511628211ull; }
  };
  const size_t nb = (size_t)std::max(job->n_blocks, 0);
  int32_t dims[3] = {0, 0, job->n_blocks};
  for (size_t b = 0; b < nb; ++b) {
    const int dim = job->block_kind[b] == OKB_BLOCK_SPEED_BIAS ? 9 : 6;
    dims[0] += dim;
    if (!job->block_marginalize[b]) dims[1] += dim;
  }
  mix(dims, sizeof dims);
  mix(job->block_kind, 4 * nb); mix(job->block_idx, 4 * nb); mix(job->block_prev, 4 * nb); mix(job->block_marginalize, nb);
  mix(&job->n_imu_terms, 4);
  if (job->n_imu_terms > 0) mix(job->imu_terms, 4 * (size_t)job->n_imu_terms);
  mix(&job->n_sb_priors, 4);
  if (job->n_sb_priors > 0) mix(job->sb_priors, 4 * (size_t)job->n_sb_priors);
  return h;
}

// The one path behind okb_window_marginalize (n = 1) and okb_window_marginalize_batch: jobs[t] runs on slot slots[t]
// (ascending, distinct).  Every job is checked before any device work.  Then, on the transfer stream: the pending
// edits of the job slots are committed, the task table and the job payloads go over in one H2D copy, each run of
// consecutive job slots gets one WinDev copy, and one k_marginalize launch runs one CTA per job after the solver
// work already launched on those slots.  Other slots are not touched.
int marg_run(okb_ctx* c, const int* slots, const okb_marg_job* const* jobs, int n, bool batch) {
  cudaSetDevice(c->device);
  std::vector<MargDims> dims(n);
  for (int t = 0; t < n; ++t) {
    const char* why = "";
    const int rc = marg_check(c, slots[t], jobs[t], dims[t], &why);
    if (rc) {
      c->set_error(batch ? "okb_window_marginalize_batch: slot " + std::to_string(slots[t]) + ": " + why : std::string("okb_window_marginalize: ") + why);
      return rc;
    }
  }
  cudaStream_t xs = c->stream_xfer;
  // Landmark-sharded context: all ranks' calls may come from one host thread in rank order, so nothing below may wait
  // on the host for this rank's earlier launches (they may be spinning until a peer's launch arrives).  Outgrown
  // buffers are retired rather than freed; the launch runs the sharded instantiation.
  const bool sharded = c->shard_world > 1;
  // scratch of the job slots and the call's device buffer: growing frees the old ones, which waits for the transfer
  // stream once
  size_t bytes = align_up(sizeof(MargTask) * (size_t)n, 256);
  std::vector<MargPayload> pay(n);
  std::vector<size_t> off(n);
  for (int t = 0; t < n; ++t) { pay[t] = marg_payload(jobs[t]); off[t] = bytes; bytes += pay[t].total; }
  std::vector<char> grow(n, 0);
  bool wait = c->marg_dev && bytes > c->marg_dev_bytes;
  for (int t = 0; t < n; ++t) {
    const WinStore& S = c->wins[slots[t]];
    grow[t] = !S.marg_scratch || S.marg_lm_cap < jobs[t]->n_landmarks || S.marg_K_cap < S.caps.K || S.marg_L_cap < S.caps.L || S.marg_O_cap < S.caps.O;
    wait = wait || (grow[t] && S.marg_scratch);
  }
  if (wait && !sharded) OKB_CUDA(c, cudaStreamSynchronize(xs));
  for (int t = 0; t < n; ++t) {
    if (!grow[t]) continue;
    WinStore& S = c->wins[slots[t]];
    if (S.marg_scratch) {
      if (sharded) c->marg_retired_dev.push_back(S.marg_scratch); else cudaFree(S.marg_scratch);
      S.marg_scratch = nullptr;
    }
    S.marg_lm_cap = std::max(256, 2 * jobs[t]->n_landmarks); S.marg_K_cap = S.caps.K; S.marg_L_cap = S.caps.L; S.marg_O_cap = S.caps.O;
    const MargLayout m = marg_layout(S.marg_lm_cap, S.marg_K_cap, S.marg_L_cap, S.marg_O_cap);
    OKB_CUDA(c, cudaMalloc(&S.marg_scratch, m.total));
    S.marg_scratch_bytes = m.total;
    OKB_CUDA(c, cudaMemsetAsync(S.marg_scratch, 0, m.total, xs));
  }
  if (bytes > c->marg_dev_bytes) {
    const size_t cap = align_up(std::max(bytes, std::max((size_t)64 << 10, 2 * c->marg_dev_bytes)), 4096);
    if (c->marg_dev) { if (sharded) c->marg_retired_dev.push_back(c->marg_dev); else cudaFree(c->marg_dev); }
    c->marg_dev = nullptr; c->marg_dev_bytes = 0;
    OKB_CUDA(c, cudaMalloc(&c->marg_dev, cap));
    c->marg_dev_bytes = cap;
  }
  // pending graph edits first: the jobs index the windows as they are now
  int rc = for_runs(slots, n, [&](int f, int m) { return commit_range(c, f, m); });
  if (rc) return rc;
  // pack: the previous call's copy reads the pinned buffer until marg_copied
  if (!c->marg_copied) OKB_CUDA(c, cudaEventCreateWithFlags(&c->marg_copied, cudaEventDisableTiming));
  if (c->marg_busy) {
    // sharded: that copy may queue behind this rank's previous k_marginalize, still waiting for its peers; pack into a
    // fresh buffer instead
    const cudaError_t q = sharded ? cudaEventQuery(c->marg_copied) : cudaSuccess;
    if (q == cudaErrorNotReady) {
      cudaGetLastError();
      // park the buffer with an event after its copy; take a parked buffer whose copy has completed, if any
      okb_ctx::MargPinned park{c->marg_host, c->marg_host_bytes, nullptr};
      OKB_CUDA(c, cudaEventCreateWithFlags(&park.done, cudaEventDisableTiming));
      OKB_CUDA(c, cudaEventRecord(park.done, xs));
      c->marg_host = nullptr; c->marg_host_bytes = 0;
      for (size_t i = 0; i < c->marg_pool.size(); ++i) {
        okb_ctx::MargPinned& e = c->marg_pool[i];
        if (e.bytes < bytes) continue;
        const cudaError_t d = cudaEventQuery(e.done);
        if (d == cudaErrorNotReady) { cudaGetLastError(); continue; }
        OKB_CUDA(c, d);
        cudaEventDestroy(e.done);
        c->marg_host = e.p; c->marg_host_bytes = e.bytes;
        c->marg_pool.erase(c->marg_pool.begin() + i);
        break;
      }
      c->marg_pool.push_back(park);
    } else {
      OKB_CUDA(c, cudaEventSynchronize(c->marg_copied));
    }
    c->marg_busy = false;
  }
  if (bytes > c->marg_host_bytes) {
    if (c->marg_host) { if (sharded) c->marg_retired_host.push_back(c->marg_host); else cudaFreeHost(c->marg_host); }
    c->marg_host = nullptr; c->marg_host_bytes = 0;
    const size_t cap = c->marg_dev_bytes;
    OKB_CUDA(c, cudaMallocHost(&c->marg_host, cap));
    c->marg_host_bytes = cap;
  }
  MargTask* tasks = reinterpret_cast<MargTask*>(c->marg_host);
  for (int t = 0; t < n; ++t) {
    const okb_marg_job* job = jobs[t];
    const WinStore& S = c->wins[slots[t]];
    const MargPayload& p = pay[t];
    unsigned char* q = c->marg_host + off[t];
    std::memset(q, 0, p.total);
    const MargJobHeader h{job->n_blocks, job->n_imu_terms, job->n_sb_priors, job->n_landmarks, dims[t].N, dims[t].n_keep, S.marg_lm_cap, 0};
    std::memcpy(q, &h, sizeof h);
    std::memcpy(q + p.kind, job->block_kind, 4 * (size_t)job->n_blocks);
    std::memcpy(q + p.idx, job->block_idx, 4 * (size_t)job->n_blocks);
    std::memcpy(q + p.prev, job->block_prev, 4 * (size_t)job->n_blocks);
    std::memcpy(q + p.marg, job->block_marginalize, (size_t)job->n_blocks);
    if (job->n_imu_terms) std::memcpy(q + p.imu, job->imu_terms, 4 * (size_t)job->n_imu_terms);
    if (job->n_sb_priors) std::memcpy(q + p.sbp, job->sb_priors, 4 * (size_t)job->n_sb_priors);
    if (job->n_landmarks) std::memcpy(q + p.lms, job->landmarks, 4 * (size_t)job->n_landmarks);
    MargTask task{};
    task.win = slots[t];
    if (sharded) task.fingerprint = marg_job_fingerprint(job);
    task.sc = marg_pointers(c->marg_dev + off[t], p, S.marg_scratch, marg_layout(S.marg_lm_cap, S.marg_K_cap, S.marg_L_cap, S.marg_O_cap));
    tasks[t] = task;
  }
  // after the solver work already launched on the job slots
  if ((rc = wait_solver_work(c, xs, slots, n))) return rc;
  OKB_CUDA(c, cudaMemcpyAsync(c->marg_dev, c->marg_host, bytes, cudaMemcpyHostToDevice, xs));
  OKB_CUDA(c, cudaEventRecord(c->marg_copied, xs));
  c->marg_busy = true;
  rc = for_runs(slots, n, [&](int f, int m) {
    OKB_CUDA(c, cudaMemcpyAsync(c->d_wins + f, &c->host[f], sizeof(WinDev) * m, cudaMemcpyHostToDevice, xs));
    return OKB_OK;
  });
  if (rc) return rc;
  if (sharded) k_marginalize<true><<<n, M_THREADS, 0, xs>>>(c->d_wins, reinterpret_cast<const MargTask*>(c->marg_dev));
  else k_marginalize<false><<<n, M_THREADS, 0, xs>>>(c->d_wins, reinterpret_cast<const MargTask*>(c->marg_dev));
  c->launches += 1;
  OKB_CUDA(c, cudaGetLastError());
  for (int t = 0; t < n; ++t) {
    WinDev& W = c->host[slots[t]];
    W.marg_n = dims[t].n_keep; W.marg_nb = dims[t].nb_keep; W.marg_xdim = dims[t].xdim;
  }
  return OKB_OK;
}
}  // namespace

extern "C" int okb_window_marginalize(okb_ctx* c, int win, const okb_marg_job* job) {
  if (!c || !job || win < 0 || win >= c->max_windows) return OKB_ERR_INVALID_ARG;
  return marg_run(c, &win, &job, 1, false);
}

extern "C" int okb_window_marginalize_batch(okb_ctx* c, int win_first, int count, const okb_marg_job* const* jobs) {
  if (!c || !jobs || win_first < 0 || count < 1 || count > c->max_windows - win_first) return OKB_ERR_INVALID_ARG;
  std::vector<int> slots;
  std::vector<const okb_marg_job*> js;
  for (int i = 0; i < count; ++i)
    if (jobs[i]) { slots.push_back(win_first + i); js.push_back(jobs[i]); }
  if (slots.empty()) return OKB_OK;
  return marg_run(c, slots.data(), js.data(), (int)slots.size(), true);
}

extern "C" int okb_marg_job_fingerprint(const okb_marg_job* job, uint64_t* out) {
  if (!job || !out || job->n_blocks < 0 || (job->n_blocks && (!job->block_kind || !job->block_idx || !job->block_prev || !job->block_marginalize)) ||
      job->n_imu_terms < 0 || job->n_sb_priors < 0 || (job->n_imu_terms && !job->imu_terms) || (job->n_sb_priors && !job->sb_priors))
    return OKB_ERR_INVALID_ARG;
  *out = marg_job_fingerprint(job);
  return OKB_OK;
}

extern "C" int okb_window_download_marg(okb_ctx* c, int win, int32_t* n, int32_t* n_blocks, int32_t* block_kind, uint32_t* block_idx, double* x0,
                                        double* J, double* e0, double* H, double* b0, int32_t* status) {
  int rc = check_range(c, win, 1);
  if (rc) return rc;
  cudaSetDevice(c->device);
  rc = commit_range(c, win, 1);
  if (rc) return rc;
  const int cap = 8 + 2 * kMaxMargBlocks + 9 * kMaxMargBlocks + 2 * kMaxMarg * kMaxMarg + 2 * kMaxMarg;
  rc = grow(c, &c->hook_buf, &c->hook_bytes, sizeof(double) * cap);
  if (rc) return rc;
  WinStore& S = c->wins[win];
  cudaStream_t xs = c->stream_xfer;
  if (S.done_idx >= 0) OKB_CUDA(c, cudaStreamWaitEvent(xs, c->done_ring[S.done_idx], 0));
  k_marg_export<<<1, 256, 0, xs>>>(c->d_wins, win, reinterpret_cast<double*>(c->hook_buf), cap);
  c->launches += 1;
  std::vector<double> host(cap);
  OKB_CUDA(c, cudaMemcpyAsync(host.data(), c->hook_buf, sizeof(double) * cap, cudaMemcpyDeviceToHost, xs));
  int32_t st[4] = {0, 0, 0, 0};
  if (S.marg_scratch) {
    const MargLayout m = marg_layout(S.marg_lm_cap, S.marg_K_cap, S.marg_L_cap, S.marg_O_cap);
    OKB_CUDA(c, cudaMemcpyAsync(st, S.marg_scratch + m.status, 16, cudaMemcpyDeviceToHost, xs));
  }
  OKB_CUDA(c, cudaStreamSynchronize(xs));
  const int nn = (int)host[0], nb = (int)host[1], xd = (int)host[2];
  if (n) *n = nn;
  if (n_blocks) *n_blocks = nb;
  if (status) std::memcpy(status, st, 16);
  if ((int)host[3] > cap) { c->set_error("okb_window_download_marg: prior larger than the export buffer"); return OKB_ERR_CAPACITY; }
  const double* o = host.data() + 8;
  for (int i = 0; i < nb; ++i) { if (block_kind) block_kind[i] = (int32_t)o[i]; if (block_idx) block_idx[i] = (uint32_t)o[nb + i]; }
  o += 2 * nb;
  if (x0) std::memcpy(x0, o, sizeof(double) * xd);
  o += xd;
  if (J) std::memcpy(J, o, sizeof(double) * (size_t)nn * nn);
  if (e0) std::memcpy(e0, o + (size_t)nn * nn, sizeof(double) * nn);
  if (H) std::memcpy(H, o + (size_t)nn * nn + nn, sizeof(double) * (size_t)nn * nn);
  if (b0) std::memcpy(b0, o + 2 * (size_t)nn * nn + nn, sizeof(double) * nn);
  return OKB_OK;
}

// ---------------------------------------------------------------------------------------------
// landmark-sharded single window: mailbox set-up (SURVEY 8e row 2)
// ---------------------------------------------------------------------------------------------
static int shard_alloc(okb_ctx* c, int rank, int world, int max_frames) {
  if (!c || world < 2 || world > kMaxShard || rank < 0 || rank >= world || max_frames < 1 || max_frames > kMaxFrames) return OKB_ERR_INVALID_ARG;
  if (c->shard_local) { c->set_error("landmark sharding is already set up on this context"); return OKB_ERR_INVALID_ARG; }
  cudaSetDevice(c->device);
  const int dcp = 4 * ((6 * max_frames + 1 + 3) / 4);
  c->shard_box_cap = (int)shard_box_doubles(max_frames, dcp);
  c->shard_marg_cap = (int)shard_marg_box_doubles(max_frames);
  c->shard_win_bytes = shard_win_bytes(world, (size_t)c->shard_box_cap, (size_t)c->shard_marg_cap, (size_t)c->shard_lm_cap);
  const size_t total = c->shard_win_bytes * (size_t)c->max_windows;
  OKB_CUDA(c, cudaMalloc(&c->shard_local, total));
  OKB_CUDA(c, cudaMemset(c->shard_local, 0, total));
  OKB_CUDA(c, cudaDeviceSynchronize());
  c->shard_rank = rank;
  c->shard_world = world;
  c->shard_peer[rank] = c->shard_local;
  return OKB_OK;
}

extern "C" int okb_shard_mailbox_layout(int world, int max_frames, int max_landmarks, uint64_t out[3]) {
  if (world < 2 || world > kMaxShard || max_frames < 1 || max_frames > kMaxFrames || max_landmarks < 0 || !out) return OKB_ERR_INVALID_ARG;
  const size_t box = shard_box_doubles(max_frames, 4 * ((6 * max_frames + 1 + 3) / 4)), marg = shard_marg_box_doubles(max_frames);
  out[0] = shard_lm_offset(world, box, marg);
  out[1] = 2 * shard_lm_half_bytes((size_t)max_landmarks);
  out[2] = shard_win_bytes(world, box, marg, (size_t)max_landmarks);
  return OKB_OK;
}

extern "C" int okb_shard_reserve_landmarks(okb_ctx* c, int max_landmarks) {
  if (!c || max_landmarks < 0) return OKB_ERR_INVALID_ARG;
  if (c->shard_local) { c->set_error("okb_shard_reserve_landmarks: call it before okb_shard_export / okb_shard_connect_local"); return OKB_ERR_INVALID_ARG; }
  c->shard_lm_cap = max_landmarks;
  return OKB_OK;
}

extern "C" int okb_shard_export(okb_ctx* c, int rank, int world, int max_frames, void* handle_out) {
  if (!handle_out) return OKB_ERR_INVALID_ARG;
  int rc = shard_alloc(c, rank, world, max_frames);
  if (rc) return rc;
  static_assert(sizeof(cudaIpcMemHandle_t) == OKB_SHARD_HANDLE_BYTES, "handle size");
  cudaIpcMemHandle_t h;
  OKB_CUDA(c, cudaIpcGetMemHandle(&h, c->shard_local));
  std::memcpy(handle_out, &h, sizeof h);
  return OKB_OK;
}

extern "C" int okb_shard_connect(okb_ctx* c, const void* handles) {
  if (!c || !handles || c->shard_world < 2 || !c->shard_local) return OKB_ERR_INVALID_ARG;
  cudaSetDevice(c->device);
  for (int r = 0; r < c->shard_world; ++r) {
    if (r == c->shard_rank) continue;
    cudaIpcMemHandle_t h;
    std::memcpy(&h, static_cast<const unsigned char*>(handles) + (size_t)r * sizeof h, sizeof h);
    void* p = nullptr;
    OKB_CUDA(c, cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    c->shard_peer[r] = static_cast<unsigned char*>(p);
    c->shard_peer_ipc[r] = true;
  }
  return OKB_OK;
}

extern "C" int okb_shard_connect_local(okb_ctx* const* ctxs, int world, int max_frames) {
  if (!ctxs || world < 2 || world > kMaxShard) return OKB_ERR_INVALID_ARG;
  for (int r = 0; r < world; ++r) {
    if (!ctxs[r]) return OKB_ERR_INVALID_ARG;
    if (ctxs[r]->max_windows != ctxs[0]->max_windows) { ctxs[r]->set_error("sharded contexts must have the same number of window slots"); return OKB_ERR_INVALID_ARG; }
    const int rc = shard_alloc(ctxs[r], r, world, max_frames);
    if (rc) return rc;
  }
  for (int r = 0; r < world; ++r) {
    okb_ctx* c = ctxs[r];
    cudaSetDevice(c->device);
    for (int q = 0; q < world; ++q) {
      if (q == r) continue;
      if (ctxs[q]->device != c->device) {
        const cudaError_t e = cudaDeviceEnablePeerAccess(ctxs[q]->device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { c->set_error(std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e)); return OKB_ERR_CUDA; }
        cudaGetLastError();
      }
      c->shard_peer[q] = ctxs[q]->shard_local;
    }
  }
  return OKB_OK;
}

extern "C" int okb_shard_stats(okb_ctx* c, int win, double out[4]) {
  if (!c || win < 0 || win >= c->max_windows || !out) return OKB_ERR_INVALID_ARG;
  const SolverState& s = c->h_states[win];
  out[0] = (double)s.shard_rounds; out[1] = 1e-3 * (double)s.shard_wait_ns; out[2] = (double)s.shard_fault; out[3] = (double)s.shard_epoch;
  return OKB_OK;
}

// ---- optional event timing around solver kernels.  Returns the pair's index; `join` >= 0 is the index of the pair
// whose span this one widens: the groups of a grouped solve each time a round's phase on their own stream, and the
// phase's span over the whole batch runs from the earliest group's begin to the latest group's end.
static int prof_begin(okb_ctx* c, int kind, cudaStream_t s, int join = -1) {
  if (!c->profile) return -1;
  if (c->prof_used + 2 > c->prof_events.size()) {
    cudaEvent_t a, b;
    cudaEventCreate(&a); cudaEventCreate(&b);
    c->prof_events.push_back(a); c->prof_events.push_back(b);
  }
  const int i = (int)c->prof_kind.size();
  c->prof_kind.push_back(kind);
  c->prof_join.push_back(join < 0 ? i : join);
  cudaEventRecord(c->prof_events[c->prof_used], s);
  return i;
}
static void prof_end(okb_ctx* c, cudaStream_t s) {
  if (!c->profile) return;
  cudaEventRecord(c->prof_events[c->prof_used + 1], s);
  c->prof_used += 2;
}
extern "C" int okb_profile_enable(okb_ctx* c, int on) {
  if (!c) return OKB_ERR_INVALID_ARG;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  c->profile = on != 0;
  c->prof_used = 0;
  c->prof_kind.clear();
  c->prof_join.clear();
  return OKB_OK;
}
extern "C" int okb_set_solve_groups(okb_ctx* c, int n) {
  if (!c || n < 0 || n > okb_ctx::kMaxSolveGroups) return OKB_ERR_INVALID_ARG;
  c->solve_groups = n;
  return OKB_OK;
}
extern "C" int okb_profile_read(okb_ctx* c, double out[6]) {
  if (!c || !out) return OKB_ERR_INVALID_ARG;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  for (int i = 0; i < 6; ++i) out[i] = 0.0;
  const size_t n = c->prof_kind.size();
  std::vector<float> lo(n, 0.f), hi(n, 0.f);     // per span: earliest begin, latest end, from the span's first begin
  for (size_t i = 0; i < n; ++i) {
    const size_t j = (size_t)c->prof_join[i];      // j <= i
    float b = 0.f, e = 0.f;
    cudaEventElapsedTime(&b, c->prof_events[2 * j], c->prof_events[2 * i]);
    cudaEventElapsedTime(&e, c->prof_events[2 * j], c->prof_events[2 * i + 1]);
    lo[j] = j == i ? b : std::min(lo[j], b);
    hi[j] = j == i ? e : std::max(hi[j], e);
  }
  for (size_t i = 0; i < n; ++i)
    if ((size_t)c->prof_join[i] == i) {
      out[2 * c->prof_kind[i]] += hi[i] - lo[i];
      out[2 * c->prof_kind[i] + 1] += 1.0;
    }
  c->prof_used = 0;
  c->prof_kind.clear();
  c->prof_join.clear();
  return OKB_OK;
}

static int check_range(okb_ctx* c, int first, int count) {
  if (!c || first < 0 || count < 1 || first + count > c->max_windows) return OKB_ERR_INVALID_ARG;
  for (int i = first; i < first + count; ++i)
    if (!c->wins[i].uploaded) { c->set_error("window slot not uploaded"); return OKB_ERR_INVALID_ARG; }
  return OKB_OK;
}

extern "C" int64_t okb_window_h2d_bytes(const okb_ctx* c, int win) {
  if (!c || win < 0 || win >= c->max_windows || !c->wins[win].uploaded) return 0;
  return (int64_t)(c->wins[win].h2d_bytes + sizeof(WinDev));     // the last commit's command stream + the window descriptor
}

extern "C" int okb_window_reset(okb_ctx* c, int first, int count) {
  int rc = check_range(c, first, count);
  if (rc) return rc;
  cudaSetDevice(c->device);
  for (int i = first; i < first + count; ++i) {
    const WinStore& S = c->wins[i];
    const WinDev& W = c->host[i];
    if (W.K != S.K_init || W.NSB != S.NSB_init || W.L != S.L_init) { c->set_error("okb_window_reset: the window changed shape since its last full upload"); return OKB_ERR_INVALID_ARG; }
  }
  rc = commit_range(c, first, count);
  if (rc) return rc;
  // Runs on the TRANSFER stream (after the solver work already launched on these slots): restoring a slot is part of
  // preparing it, so it overlaps a solve that is running on other slots; the next okb_optimize* of the slot joins the
  // transfer stream as it does for uploads.
  cudaStream_t xs = c->stream_xfer;
  if ((rc = wait_solver_work(c, xs, c->ident.data() + first, count))) return rc;
  k_reset<<<count, 128, 0, xs>>>(c->d_wins, c->d_ident + first, 1);
  c->launches += 1;
  OKB_CUDA(c, cudaGetLastError());
  return OKB_OK;
}

// ---------------------------------------------------------------------------------------------
// optimize
// ---------------------------------------------------------------------------------------------
// Launch geometry of one optimize of the listed windows: everything a captured CUDA graph depends on
// besides the kernel arguments.
struct RoundPlan {
  int max_chunks = 1, max_imu = 0, max_cx = 1, lm_wide = 0, acc_smem = 1, chol_smem = 1, solve_threads = S_THREADS, gxQ = 1, shard = 0, push_gx = 1;
  int lm_model = kDistAny, schur_wide = 0;      // (no padding bytes: the plan is compared bytewise as a graph key)
  int groups = 1, unused = 0;                   // window groups of launch_rounds (the second int keeps the ints 8-byte aligned)
  size_t smA = 0, smS = 0, smQ = 0;
};
static int plan_rounds(okb_ctx* c, const int32_t* slots, int count, RoundPlan& P) {
  P = RoundPlan();
  int chol_smem = 1;       // solve_mode of k_solve: 1 system in shared memory, 2 pose system + chain band, 0 chain band only
  // k_schur: the block-pair and right-hand-side accumulators live in shared memory whenever they fit one CTA per SM
  // (K <= 22), else in the chunk's global partial; 256-thread CTAs where two fit an SM (K <= 12), else one 512-thread
  // CTA per SM
  int acc_smem = 1;
  for (int t = 0; t < count; ++t)
    if (smemA2_bytes(c->host[slots[t]].K, 1) > (size_t)c->smem_optin) acc_smem = 0;
  int maxL = 1;
  for (int t = 0; t < count; ++t) {
    const WinDev& W = c->host[slots[t]];
    P.max_chunks = std::max(P.max_chunks, W.n_chunks);
    P.max_imu = std::max(P.max_imu, W.n_imu);
    P.smA = std::max(P.smA, smemA2_bytes(W.K, acc_smem));
    P.max_cx = std::max(P.max_cx, (W.L + L1_THREADS - 1) / L1_THREADS);
    {      // the roomiest mode this window fits; the range runs in the most modest one (1 > 2 > 0)
      const int wm = smemS_bytes(W.d, W.dc, W.K, W.marg_n, W.n_imu, 1) <= (size_t)c->smem_optin ? 1
                   : smemS_bytes(W.d, W.dc, W.K, W.marg_n, W.n_imu, 2) <= (size_t)c->smem_optin ? 2 : 0;
      if (wm == 0 || chol_smem == 0) chol_smem = 0;
      else if (wm == 2) chol_smem = 2;
    }
    P.smQ = std::max(P.smQ, (size_t)W.NS * sizeof(SlotCtx));
    maxL = std::max(maxL, W.L);
  }
  for (int t = 0; t < count; ++t) {
    const WinDev& W = c->host[slots[t]];
    P.smS = std::max(P.smS, smemS_bytes(W.d, W.dc, W.K, W.marg_n, W.n_imu, chol_smem));
  }
  if (P.smS > (size_t)c->smem_optin) { c->set_error("window does not fit kernel S shared memory"); return OKB_ERR_CAPACITY; }
  if (const char* force = getenv("OKB_SOLVE_MODE")) {      // diagnostics / tests: a more modest solve_mode than the windows need (2 or 0)
    const int m = atoi(force);
    if ((m == 0 || m == 2) && chol_smem != 0 && !(chol_smem == 2 && m == 2)) {
      chol_smem = m;
      P.smS = 0;
      for (int t = 0; t < count; ++t) {
        const WinDev& W = c->host[slots[t]];
        P.smS = std::max(P.smS, smemS_bytes(W.d, W.dc, W.K, W.marg_n, W.n_imu, chol_smem));
      }
      if (P.smS > (size_t)c->smem_optin) { c->set_error("window does not fit kernel S shared memory"); return OKB_ERR_CAPACITY; }
    }
  }
  P.acc_smem = acc_smem; P.chol_smem = chol_smem;
  P.schur_wide = P.smA > ((size_t)c->smem_per_sm - 2048) / 2 ? 1 : 0;
  // k_landmarks: launches whose landmark tiles would fill less than half the SMs (few windows, the cfg-5 window) split
  // every tile's frame walk over a cluster of two 512-thread CTAs; the sums keep their order in either shape
  P.lm_wide = (2 * count * P.max_cx <= c->sm_count) ? 1 : 0;
  // k_landmarks is instantiated per distortion model: the one every camera of the launch shares, else the run-time switch
  P.lm_model = c->wins[slots[0]].cam_model;
  for (int t = 1; t < count; ++t)
    if (c->wins[slots[t]].cam_model != P.lm_model) P.lm_model = kDistAny;
  P.solve_threads = (2 * count <= c->sm_count) ? 512 : S_THREADS;      // few windows: one wide CTA per SM (all ranks of a sharded window choose alike)
  P.gxQ = std::max(1, std::min((maxL + 127) / 128, (4 * c->sm_count + count - 1) / count));
  P.shard = c->shard_world > 1 ? 1 : 0;
  P.push_gx = std::max(1, std::min(16, c->sm_count / std::max(1, count)));
  // Window groups: a batch of at least one window per SM runs as kMaxSolveGroups groups, each on its own stream and
  // started behind the previous one, so that one group's k_solve (barrier / latency bound) and each kernel's drain share
  // the SMs with another group's k_landmarks / k_schur.  Four groups were the fastest or within 1 % of it at 132, 264,
  // 528 and 1056 windows (DESIGN §5); smaller batches were not measured and keep one group.  Every field above is the
  // full batch's: each group launches the same kernel shapes over its share of the slot table.  Landmark-sharded windows
  // spin on their peers inside their kernels and stay in one group.
  int G = c->solve_groups;
  if (G == 0) G = count >= c->sm_count ? okb_ctx::kMaxSolveGroups : 1;
  P.groups = P.shard ? 1 : std::max(1, std::min({G, okb_ctx::kMaxSolveGroups, count}));
  return OKB_OK;
}

template <int MODEL>
static void launch_landmarks(okb_ctx* c, int count, const int32_t* tab, cudaStream_t s, const RoundPlan& P) {
  if (P.lm_wide) {     // one cluster of two CTAs per landmark tile
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3(2 * P.max_cx, count); cfg.blockDim = dim3(4 * L1_THREADS); cfg.dynamicSmemBytes = smemL_bytes(4);
    cfg.stream = s; cfg.attrs = attr; cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, k_landmarks<4, 2, MODEL>, (const WinDev*)c->d_wins, tab);
  } else {
    k_landmarks<2, 1, MODEL><<<dim3(P.max_cx, count), 2 * L1_THREADS, smemL_bytes(2), s>>>(c->d_wins, tab);
  }
}

// The rounds of one optimize, group by group (RoundPlan::groups): group g owns slot-table entries [count*g/G,
// count*(g+1)/G) and runs its chain on group_stream[g], which starts behind group g-1's first k_landmarks; the groups
// join `stream` at the end.  Group 0 is `stream` itself, so one group is the plain chain.
static int launch_rounds(okb_ctx* c, int count, const okb_solve_options& opt, int rounds, const RoundPlan& P) {
  static const bool imu_serial = getenv("OKB_IMU_SERIAL") != nullptr;     // diagnostics: k_imu on the main stream, ahead of the landmark kernels
  const int G = P.groups;
  int span[2] = {-1, -1};      // this round's profiled pairs of group 0, which the other groups' pairs widen
  for (int r = 0; r < rounds; ++r)
    for (int g = 0; g < G; ++g) {
      const int first = (int)((int64_t)count * g / G), n = (int)((int64_t)count * (g + 1) / G) - first;
      const int32_t* tab = c->d_slot_tab + first;
      cudaStream_t s = c->group_stream[g];
      if (r == 0 && g > 0) cudaStreamWaitEvent(s, c->group_stagger[g - 1], 0);
      const dim3 gridA(P.max_chunks, n);
      if (P.max_imu > 0 && imu_serial) {
        k_imu<<<dim3((P.max_imu + 32 / IMU_G - 1) / (32 / IMU_G), n), 32, smemI_bytes(), s>>>(c->d_wins, tab);
        c->launches += 1;
      } else if (P.max_imu > 0) {   // IMU terms only depend on the previous round's candidate: run beside the landmark kernels
        cudaEventRecord(c->group_round[g], s);
        cudaStreamWaitEvent(c->group_imu[g], c->group_round[g], 0);
        k_imu<<<dim3((P.max_imu + 32 / IMU_G - 1) / (32 / IMU_G), n), 32, smemI_bytes(), c->group_imu[g]>>>(c->d_wins, tab);
        cudaEventRecord(c->group_imu_done[g], c->group_imu[g]);
        c->launches += 1;
      }
      const int p0 = prof_begin(c, 0, s, g ? span[0] : -1);
      if (g == 0) span[0] = p0;
      switch (P.lm_model) {
        case OKB_DIST_NONE: launch_landmarks<OKB_DIST_NONE>(c, n, tab, s, P); break;
        case OKB_DIST_RADTAN: launch_landmarks<OKB_DIST_RADTAN>(c, n, tab, s, P); break;
        case OKB_DIST_EQUIDISTANT: launch_landmarks<OKB_DIST_EQUIDISTANT>(c, n, tab, s, P); break;
        case OKB_DIST_RADTAN8: launch_landmarks<OKB_DIST_RADTAN8>(c, n, tab, s, P); break;
        default: launch_landmarks<kDistAny>(c, n, tab, s, P); break;
      }
      if (r == 0 && g + 1 < G) cudaEventRecord(c->group_stagger[g], s);
      if (P.schur_wide) k_schur<512><<<gridA, 512, P.smA, s>>>(c->d_wins, tab, P.acc_smem, opt.max_iterations);
      else k_schur<256><<<gridA, 256, P.smA, s>>>(c->d_wins, tab, P.acc_smem, opt.max_iterations);
      if (P.shard) {    // chunk reduction fused with the push half of the all-reduce over peer memory
        k_shard_push<<<dim3(P.push_gx, n), 256, 0, s>>>(c->d_wins, tab);
        c->launches += 1;
      } else if (P.max_chunks > 1) { k_reduce_partials<<<dim3(8, n), 256, 0, s>>>(c->d_wins, tab); c->launches += 1; }
      prof_end(c, s);
      c->launches += 2;
      if (P.max_imu > 0 && !imu_serial) cudaStreamWaitEvent(s, c->group_imu_done[g], 0);
      const int p1 = prof_begin(c, 1, s, g ? span[1] : -1);
      if (g == 0) span[1] = p1;
      if (P.solve_threads == 512) k_solve<512><<<n, 512, P.smS, s>>>(c->d_wins, tab, opt, P.chol_smem);
      else k_solve<S_THREADS><<<n, S_THREADS, P.smS, s>>>(c->d_wins, tab, opt, P.chol_smem);
      prof_end(c, s);
      c->launches += 1;
    }
  for (int g = 1; g < G; ++g) {
    cudaEventRecord(c->group_done[g], c->group_stream[g]);
    cudaStreamWaitEvent(c->stream, c->group_done[g], 0);
  }
  OKB_CUDA(c, cudaGetLastError());
  return OKB_OK;
}

// post-solve landmark quality (Estimator.cpp:880-894)
static int launch_quality(okb_ctx* c, int count, const RoundPlan& P) {
  prof_begin(c, 2, c->stream);
  k_quality<<<dim3(P.gxQ, count), 128, P.smQ, c->stream>>>(c->d_wins, c->d_slot_tab);
  prof_end(c, c->stream);
  c->launches += 1;
  OKB_CUDA(c, cudaGetLastError());
  return OKB_OK;
}

// The fixed launch sequence of one optimize (rounds + quality pass) as a CUDA graph: captured once per launch
// geometry / option set and replayed -- one host call instead of ~70 launches and ~40 event operations, which is
// what bounds the latency of a single window (SURVEY 8d "B = 1").  OKB_NO_GRAPH=1 disables it (diagnostics).
static int run_rounds(okb_ctx* c, const int32_t* slots, int count, const okb_solve_options& opt, int rounds, bool with_quality) {
  RoundPlan P;
  int rc = plan_rounds(c, slots, count, P);
  if (rc) return rc;
  static const bool no_graph = getenv("OKB_NO_GRAPH") != nullptr;
  // landmark-sharded windows spin on their peers inside k_solve: their kernels must reach the device in stream order,
  // not behind whatever hardware queue a graph's internal branches were mapped to
  if (c->profile || no_graph || c->shard_world > 1) {
    rc = launch_rounds(c, count, opt, rounds, P);
    if (!rc && with_quality) rc = launch_quality(c, count, P);
    return rc;
  }
  okb_ctx::GraphEntry key;
  std::memset(&key, 0, sizeof key);
  key.count = count; key.rounds = rounds; key.with_quality = with_quality ? 1 : 0;
  key.opt_iter = opt.max_iterations; key.opt_min = opt.min_iterations; key.opt_cauchy = opt.use_cauchy_loss; key.opt_time = opt.time_limit_s;
  static_assert(sizeof(RoundPlan) <= sizeof(key.plan), "plan blob");
  std::memcpy(key.plan, &P, sizeof P);
  for (auto& e : c->graphs)
    if (e.exec && !std::memcmp(&e, &key, offsetof(okb_ctx::GraphEntry, exec))) {
      e.stamp = ++c->graph_clock;
      OKB_CUDA(c, cudaGraphLaunch(e.exec, c->stream));
      c->launches += e.launches;
      return OKB_OK;
    }
  const int64_t l0 = c->launches;
  cudaGraph_t graph = nullptr;
  OKB_CUDA(c, cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
  rc = launch_rounds(c, count, opt, rounds, P);
  if (!rc && with_quality) rc = launch_quality(c, count, P);
  const cudaError_t ce = cudaStreamEndCapture(c->stream, &graph);
  if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
  OKB_CUDA(c, ce);
  key.launches = c->launches - l0;
  c->launches = l0;
  OKB_CUDA(c, cudaGraphInstantiate(&key.exec, graph, 0));
  cudaGraphDestroy(graph);
  okb_ctx::GraphEntry* slot = nullptr;
  for (auto& e : c->graphs) if (!e.exec) { slot = &e; break; }
  if (!slot && c->graphs.size() < 16) { c->graphs.emplace_back(); slot = &c->graphs.back(); }
  if (!slot) {     // evict the least recently used
    slot = &c->graphs[0];
    for (auto& e : c->graphs) if (e.stamp < slot->stamp) slot = &e;
    cudaGraphExecDestroy(slot->exec);
  }
  key.stamp = ++c->graph_clock;
  *slot = key;
  OKB_CUDA(c, cudaGraphLaunch(slot->exec, c->stream));
  c->launches += slot->launches;
  return OKB_OK;
}

// Checks a slot list of okb_optimize_slots*: n >= 1 distinct, uploaded slots, on a context without landmark sharding.
static int check_slots(okb_ctx* c, int n, const int32_t* slots) {
  if (!c) return OKB_ERR_INVALID_ARG;
  if (n < 1 || !slots) { c->set_error(n < 1 ? "empty slot list" : "NULL slot list"); return OKB_ERR_INVALID_ARG; }
  std::vector<char> seen(c->max_windows, 0);
  for (int t = 0; t < n; ++t) {
    const int s = slots[t];
    const std::string at = "slots[" + std::to_string(t) + "] = " + std::to_string(s);
    if (s < 0 || s >= c->max_windows) { c->set_error(at + ": out of range"); return OKB_ERR_INVALID_ARG; }
    if (!c->wins[s].uploaded) { c->set_error(at + ": window slot not uploaded"); return OKB_ERR_INVALID_ARG; }
    if (seen[s]) { c->set_error(at + ": listed twice"); return OKB_ERR_INVALID_ARG; }
    seen[s] = 1;
  }
  if (c->shard_world > 1) { c->set_error("landmark-sharded windows are optimized with okb_optimize (a range)"); return OKB_ERR_UNSUPPORTED; }
  return OKB_OK;
}

// Writes the slot table of the launch about to be issued on `stream` into d_slot_tab, from ring entry done_next: the
// done_ring entry that mark_work records after this launch, so the entry's previous copy has completed when
// done_ring[done_next] has.  Every caller calls mark_work after it, also when this or a later step fails.  With more
// than kDoneRing launches in flight this waits on the host for the oldest one (documented in okvis_b200.h).
static int stage_slots(okb_ctx* c, const int32_t* slots, int n) {
  const int k = c->done_next;
  OKB_CUDA(c, cudaEventSynchronize(c->done_ring[k]));
  int32_t* h = c->h_slot_ring + (size_t)k * c->max_windows;
  std::memcpy(h, slots, sizeof(int32_t) * n);
  OKB_CUDA(c, cudaMemcpyAsync(c->d_slot_tab, h, sizeof(int32_t) * n, cudaMemcpyHostToDevice, c->stream));
  return OKB_OK;
}

static int read_states(okb_ctx* c, const int32_t* slots, int n) {
  return for_runs(slots, n, [&](int f, int m) {
    OKB_CUDA(c, cudaMemcpyAsync(c->h_states + f, c->d_states + f, sizeof(SolverState) * m, cudaMemcpyDeviceToHost, c->stream));
    return OKB_OK;
  });
}

// The optimize of the n listed windows (checked): a range call passes c->ident.data() + first.
static int optimize_async(okb_ctx* c, const int32_t* slots, int count, const okb_solve_options* opt) {
  cudaSetDevice(c->device);
  // pending graph commands of these slots (no-op when there are none), one commit per run of consecutive slots
  int rc = for_runs(slots, count, [&](int f, int m) { return commit_range(c, f, m); });
  if (rc) return rc;
  // chunking: enough CTAs for ~2 waves when the batch is small
  for (int t = 0; t < count; ++t) {
    WinDev& W = c->host[slots[t]];
    int chunks = (2 * c->sm_count + count - 1) / count;
    chunks = std::max(1, std::min(chunks, c->chunk_cap));
    chunks = std::min(chunks, std::max(1, W.L / (2 * A2_TILE)));
    W.lm_per_chunk = (((W.L + chunks - 1) / chunks) + A2_TILE - 1) / A2_TILE * A2_TILE;   // whole tiles per chunk
    W.n_chunks = (W.L + W.lm_per_chunk - 1) / W.lm_per_chunk;
    W.use_cauchy = opt->use_cauchy_loss ? 1 : 0;
  }
  if (join_transfers(c)) { c->set_error("stream ordering failed"); return OKB_ERR_CUDA; }
  rc = for_runs(slots, count, [&](int f, int m) {
    OKB_CUDA(c, cudaMemcpyAsync(c->d_wins + f, &c->host[f], sizeof(WinDev) * m, cudaMemcpyHostToDevice, c->stream));
    return OKB_OK;
  });
  if (rc) return rc;
  for (int t = 0; t < count; ++t) c->wins[slots[t]].opt = *opt;     // optimize_finish relaunches with the call's own options
  rc = stage_slots(c, slots, count);
  if (!rc) {
    k_reset<<<count, 128, 0, c->stream>>>(c->d_wins, c->d_slot_tab, 0);
    c->launches += 1;
    // round 0 linearises at the initial state; each later round judges one step and proposes the next
    rc = run_rounds(c, slots, count, *opt, opt->max_iterations + 1, true);
  }
  if (!rc) rc = read_states(c, slots, count);
  mark_work(c, slots, count);
  return rc;
}

static int optimize_finish(okb_ctx* c, const int32_t* slots, int count, okb_summary* out) {
  cudaSetDevice(c->device);
  // optimize_async already queued the landmark-quality pass and the copy of the solver states.  Rebuild
  // rounds (linear-solver failures) consume rounds without advancing the iteration count: keep launching
  // until every window reports done (bounded).
  for (int guard = 0; guard < 64; ++guard) {
    OKB_CUDA(c, cudaStreamSynchronize(c->stream));
    bool all_done = true;
    for (int t = 0; t < count; ++t) all_done = all_done && c->h_states[slots[t]].done;
    if (all_done) break;
    int rc = stage_slots(c, slots, count);
    if (!rc) rc = run_rounds(c, slots, count, c->wins[slots[0]].opt, 2, true);
    if (!rc) rc = read_states(c, slots, count);
    mark_work(c, slots, count);
    if (rc) return rc;
  }
  for (int t = 0; t < count; ++t) {
    const SolverState& s = c->h_states[slots[t]];
    if (s.g.err) { c->set_error(graph_error_text(s.g.err)); return graph_error_status(s.g.err); }
    WinStore& S = c->wins[slots[t]];
    if (!S.cmd_used) S.obs_bound = s.g.n_obs;      // exact length of the compacted observation list
  }
  if (out) {
    for (int t = 0; t < count; ++t) {
      const SolverState& s = c->h_states[slots[t]];
      okb_summary& o = out[t];
      o.initial_cost = s.initial_cost; o.final_cost = s.cost; o.iterations = s.iteration;
      o.num_successful_steps = s.num_successful; o.termination = s.done ? s.termination : OKB_TERM_FAILURE;
      o.imu_redo_count = s.imu_redo_final; o.final_radius = s.radius; o.solve_time_s = s.solve_time_s;
    }
  }
  return OKB_OK;
}

extern "C" int okb_optimize_async(okb_ctx* c, int first, int count, const okb_solve_options* opt) {
  int rc = check_range(c, first, count);
  if (rc) return rc;
  if (!opt || opt->max_iterations < 0) return OKB_ERR_INVALID_ARG;
  return optimize_async(c, c->ident.data() + first, count, opt);
}

extern "C" int okb_optimize_finish(okb_ctx* c, int first, int count, okb_summary* out) {
  int rc = check_range(c, first, count);
  if (rc) return rc;
  return optimize_finish(c, c->ident.data() + first, count, out);
}

extern "C" int okb_optimize_slots_async(okb_ctx* c, int n, const int32_t* slots, const okb_solve_options* opt) {
  int rc = check_slots(c, n, slots);
  if (rc) return rc;
  if (!opt || opt->max_iterations < 0) return OKB_ERR_INVALID_ARG;
  return optimize_async(c, slots, n, opt);
}

extern "C" int okb_optimize_slots_finish(okb_ctx* c, int n, const int32_t* slots, okb_summary* summaries) {
  int rc = check_slots(c, n, slots);
  if (rc) return rc;
  return optimize_finish(c, slots, n, summaries);
}

extern "C" int okb_optimize_slots(okb_ctx* c, int n, const int32_t* slots, const okb_solve_options* opt, okb_summary* summaries) {
  int rc = okb_optimize_slots_async(c, n, slots, opt);
  if (rc) return rc;
  return okb_optimize_slots_finish(c, n, slots, summaries);
}

// diagnostics: the ImuError cache of term `term` (reference bias of the preintegration, valid flag, redo counter)
extern "C" int okb_debug_imu_cache(okb_ctx* c, int win, int term, double sb_ref[9], int32_t* valid, int32_t* redo_count) {
  int rc = check_range(c, win, 1);
  if (rc) return rc;
  cudaSetDevice(c->device);
  rc = commit_range(c, win, 1);
  if (rc) return rc;
  const WinDev& W = c->host[win];
  if (term < 0 || term >= W.n_imu) return OKB_ERR_INVALID_ARG;
  OKB_CUDA(c, cudaStreamSynchronize(c->stream));
  OKB_CUDA(c, cudaStreamSynchronize(c->stream_xfer));
  ImuCache h;
  OKB_CUDA(c, cudaMemcpy(&h, W.imu_cache + term, sizeof(ImuCache), cudaMemcpyDeviceToHost));
  if (sb_ref) std::memcpy(sb_ref, h.sb_ref, sizeof(double) * 9);
  if (valid) *valid = h.valid;
  if (redo_count) *redo_count = h.redo_count;
  return OKB_OK;
}

// diagnostics: what the window's last k_imu launch wrote for terms [first_term, first_term + n_terms): H30 (row-major) |
// g30 | cost per term.  Read-only: commits nothing and launches nothing, so after an edit the terms are renumbered and
// the output is stale until the next optimize.
extern "C" int okb_debug_imu_terms(okb_ctx* c, int win, int first_term, int n_terms, double* out) {
  int rc = check_range(c, win, 1);
  if (rc) return rc;
  const WinDev& W = c->host[win];
  if (!out || first_term < 0 || n_terms < 0 || first_term + n_terms > W.n_imu) return OKB_ERR_INVALID_ARG;
  if (n_terms == 0) return OKB_OK;
  cudaSetDevice(c->device);
  OKB_CUDA(c, cudaStreamSynchronize(c->stream));
  OKB_CUDA(c, cudaStreamSynchronize(c->stream_imu));
  OKB_CUDA(c, cudaMemcpy2D(out, sizeof(double) * OKB_IMU_TERM_OUT, W.imu_out + (size_t)first_term * kImuOut, sizeof(double) * kImuOut,
                           sizeof(double) * OKB_IMU_TERM_OUT, (size_t)n_terms, cudaMemcpyDeviceToHost));
  return OKB_OK;
}

// diagnostics: accumulated k_solve phase times (ns) of the last optimize of `win`
extern "C" int okb_debug_schur_plan(okb_ctx* c, int first, int count, int32_t out[3]) {
  int rc = check_range(c, first, count);
  if (rc) return rc;
  if (!out) return OKB_ERR_INVALID_ARG;
  cudaSetDevice(c->device);
  rc = commit_range(c, first, count);
  if (rc) return rc;
  RoundPlan P;
  rc = plan_rounds(c, c->ident.data() + first, count, P);
  if (rc) return rc;
  out[0] = P.acc_smem;
  out[1] = P.schur_wide ? 512 : 256;
  out[2] = (int32_t)P.smA;
  return OKB_OK;
}

extern "C" int okb_debug_phase_ns(okb_ctx* c, int win, double out[16]) {
  if (!c || win < 0 || win >= c->max_windows || !out) return OKB_ERR_INVALID_ARG;
  for (int i = 0; i < 16; ++i) out[i] = (double)c->h_states[win].phase_ns[i];
  return OKB_OK;
}

extern "C" int okb_optimize(okb_ctx* c, int first, int count, const okb_solve_options* opt, okb_summary* out) {
  int rc = okb_optimize_async(c, first, count, opt);
  if (rc) return rc;
  return okb_optimize_finish(c, first, count, out);
}

// The estimates come back from the packed output block (pose | speed/bias | landmarks | quality, caller's order) that
// k_quality / k_prepare / k_reset keep current: one D2H copy per window, plain memcpy on the host.
static size_t out_doubles(const WinDev& W) { return out_lm_offset(W.K, W.NSB) + 5 * (size_t)W.L; }
static void copy_out_window(const WinDev& W, const WinStore& S, double* poses, double* speed_bias, double* landmarks, double* quality) {
  const double* o = reinterpret_cast<const double*>(S.out_staging);
  if (poses) std::memcpy(poses, o, sizeof(double) * 7 * W.K);
  if (speed_bias && W.NSB) std::memcpy(speed_bias, o + 7 * W.K, sizeof(double) * 9 * W.NSB);
  if (landmarks) std::memcpy(landmarks, o + out_lm_offset(W.K, W.NSB), sizeof(double) * 4 * (size_t)W.L);
  if (quality) std::memcpy(quality, o + out_lm_offset(W.K, W.NSB) + 4 * (size_t)W.L, sizeof(double) * (size_t)W.L);
}

// The one path behind okb_window_download_batch (a range passes c->ident.data() + first) and okb_window_download_slots
// (checked list): pending edits committed once per run of consecutive listed slots, a wait on each distinct solver
// event of the listed slots, one D2H copy per slot, one synchronisation.  Output tables are in list order.
static int download_list(okb_ctx* c, const int32_t* slots, int count, double* const* poses, double* const* speed_bias,
                         double* const* landmarks, double* const* quality) {
  cudaSetDevice(c->device);
  int rc = for_runs(slots, count, [&](int f, int m) { return commit_range(c, f, m); });
  if (rc) return rc;
  cudaStream_t xs = c->stream_xfer;
  if ((rc = wait_solver_work(c, xs, slots, count))) return rc;
  for (int t = 0; t < count; ++t) {
    const int i = slots[t];
    OKB_CUDA(c, cudaMemcpyAsync(c->wins[i].out_staging, c->host[i].out, sizeof(double) * out_doubles(c->host[i]), cudaMemcpyDeviceToHost, xs));
  }
  WinStore& S0 = c->wins[slots[0]];
  OKB_CUDA(c, cudaEventRecord(S0.down, xs));
  OKB_CUDA(c, cudaEventSynchronize(S0.down));
  parallel_for(count, std::max(1, std::min(8, count / 32)), [&](int k) {
    const int i = slots[k];
    copy_out_window(c->host[i], c->wins[i], poses ? poses[k] : nullptr, speed_bias ? speed_bias[k] : nullptr,
                    landmarks ? landmarks[k] : nullptr, quality ? quality[k] : nullptr);
  });
  return OKB_OK;
}

extern "C" int okb_window_download(okb_ctx* c, int win, double* poses, double* speed_bias, double* landmarks, double* quality) {
  const int rc = check_range(c, win, 1);
  if (rc) return rc;
  return download_list(c, c->ident.data() + win, 1, &poses, &speed_bias, &landmarks, &quality);
}

extern "C" int okb_window_download_batch(okb_ctx* c, int first, int count, double* const* poses, double* const* speed_bias,
                                         double* const* landmarks, double* const* quality) {
  int rc = check_range(c, first, count);
  if (rc) return rc;
  return download_list(c, c->ident.data() + first, count, poses, speed_bias, landmarks, quality);
}

extern "C" int okb_window_download_slots(okb_ctx* c, int n, const int32_t* slots, double* const* poses, double* const* speed_bias,
                                         double* const* landmarks, double* const* quality) {
  int rc = check_slots(c, n, slots);
  if (rc) return rc;
  return download_list(c, slots, n, poses, speed_bias, landmarks, quality);
}

// ---------------------------------------------------------------------------------------------
// single-block test hooks (ErrorInterface::EvaluateWithMinimalJacobians mirrors)
// ---------------------------------------------------------------------------------------------
namespace {
__global__ void k_hook_reproj(int n, okb_camera cam, const double* pose, const double* lm, const double* ext, const double* z,
                              const double* sq, double* r, double* J0, double* J1, double* J2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  reproj_full(cam, pose + 7 * i, lm + 4 * i, ext + 7 * i, z + 2 * i, sq[i], r + 2 * i, J0 + 12 * i, J1 + 6 * i, J2 + 12 * i);
}
// one warp
__global__ void k_hook_imu(okb_imu_params prm, const okb_imu_sample* s, int n, int64_t t0, int64_t t1, const double* in /*32*/,
                           const double* sb_ref, int have_ref, ImuCache* cache, double* out /* r15 | SF 450 | sqrt 225 | redo */) {
  __shared__ double buf[kImuScratch];
  WarpCtx cx;
  const ImuScratch sc = imu_scratch(buf);
  double* SF = sc.SF; double* r15 = sc.r15;
  if (threadIdx.x == 0) { cache->valid = 0; cache->redo_count = 0; for (int k = 0; k < 9; ++k) cache->sb_ref[k] = 0; }
  __syncwarp();
  if (have_ref) imu_preintegrate(cx, s, n, prm, t0, t1, sb_ref, cache, sc.wk);
  const int before = cache->redo_count;
  __syncwarp();
  imu_evaluate(cx, s, n, prm, t0, t1, in, in + 7, in + 16, in + 23, cache, sc.wk, sc.F01, (double*)nullptr, r15, SF);
  for (int e = threadIdx.x; e < 15; e += 32) out[e] = r15[e];
  for (int e = threadIdx.x; e < 450; e += 32) out[15 + e] = SF[e];
  for (int e = threadIdx.x; e < 225; e += 32) out[465 + e] = cache->sqrt_info[e];
  if (threadIdx.x == 0) out[690] = (double)(cache->redo_count - before);
}
// One job of k_propagate.  `samples` is a byte offset into the input region (job table | samples), `out` one into the
// output region, where the job's record is pose 7 | speed/bias 9 | n_used (int32 in a double slot) | covariance 225
// if want_cov | Jacobian 225 if want_jac.
struct PropEntry {
  okb_imu_params prm;
  int64_t t0, t1;
  uint64_t samples, out;
  int32_t n, want_cov, want_jac, _pad;
  double state[16];     // pose | speed/bias before the propagation
};
constexpr int kPropRecord = 17;   // doubles of an output record without covariance and Jacobian

// One warp per job: ImuError::propagation with the job's scratch in shared memory.  The state is propagated in place in
// the job's output record; imu_propagate leaves it unchanged when the samples end before t1 (n_used = -1).
__global__ void __launch_bounds__(32) k_propagate(const unsigned char* __restrict__ in, unsigned char* __restrict__ out) {
  __shared__ double buf[kImuScratch];
  const PropEntry& e = reinterpret_cast<const PropEntry*>(in)[blockIdx.x];
  double* o = reinterpret_cast<double*>(out + e.out);
  if (threadIdx.x < 16) o[threadIdx.x] = e.state[threadIdx.x];
  __syncwarp();
  double* cov = e.want_cov ? o + kPropRecord : nullptr;
  double* jac = e.want_jac ? o + kPropRecord + (e.want_cov ? 225 : 0) : nullptr;
  WarpCtx cx;
  const int steps = imu_propagate(cx, reinterpret_cast<const okb_imu_sample*>(in + e.samples), e.n, e.prm, e.t0, e.t1, o, o + 7,
                                  cov, jac, imu_scratch(buf).wk);
  if (threadIdx.x == 0) *reinterpret_cast<int32_t*>(o + 16) = steps;
}
__global__ void k_hook_pose(const double* in /* meas7 S36 pose7 */, double* out /* r6 J36 */) {
  if (threadIdx.x == 0) pose_error(in, in + 7, in + 43, out, out + 6);
}
__global__ void k_hook_relpose(const double* in /* S36 p0 p1 */, double* out /* r6 J0 J1 */) {
  if (threadIdx.x == 0) relative_pose_error(in, in + 36, in + 43, out, out + 6, out + 42);
}
}  // namespace

extern "C" int okb_eval_reprojection(okb_ctx* c, int n, const okb_camera* cam, const double* pose, const double* landmark,
                                     const double* extrinsics, const double* z, const double* sqrt_info, double* r,
                                     double* J_pose, double* J_lm, double* J_ext) {
  if (!c || n < 1 || !cam) return OKB_ERR_INVALID_ARG;
  cudaSetDevice(c->device);
  const size_t nin = (size_t)n * (7 + 4 + 7 + 2 + 1), nout = (size_t)n * (2 + 12 + 6 + 12);
  int rc = grow(c, &c->hook_buf, &c->hook_bytes, (nin + nout) * sizeof(double));
  if (rc) return rc;
  double* d = reinterpret_cast<double*>(c->hook_buf);
  double *dp = d, *dl = dp + 7 * (size_t)n, *de = dl + 4 * (size_t)n, *dz = de + 7 * (size_t)n, *dq = dz + 2 * (size_t)n;
  double *dr = dq + n, *d0 = dr + 2 * (size_t)n, *d1 = d0 + 12 * (size_t)n, *d2 = d1 + 6 * (size_t)n;
  OKB_CUDA(c, cudaMemcpyAsync(dp, pose, sizeof(double) * 7 * n, cudaMemcpyHostToDevice, c->stream));
  OKB_CUDA(c, cudaMemcpyAsync(dl, landmark, sizeof(double) * 4 * n, cudaMemcpyHostToDevice, c->stream));
  OKB_CUDA(c, cudaMemcpyAsync(de, extrinsics, sizeof(double) * 7 * n, cudaMemcpyHostToDevice, c->stream));
  OKB_CUDA(c, cudaMemcpyAsync(dz, z, sizeof(double) * 2 * n, cudaMemcpyHostToDevice, c->stream));
  OKB_CUDA(c, cudaMemcpyAsync(dq, sqrt_info, sizeof(double) * n, cudaMemcpyHostToDevice, c->stream));
  k_hook_reproj<<<(n + 127) / 128, 128, 0, c->stream>>>(n, *cam, dp, dl, de, dz, dq, dr, d0, d1, d2);
  c->launches += 1;
  OKB_CUDA(c, cudaGetLastError());
  if (r) OKB_CUDA(c, cudaMemcpyAsync(r, dr, sizeof(double) * 2 * n, cudaMemcpyDeviceToHost, c->stream));
  if (J_pose) OKB_CUDA(c, cudaMemcpyAsync(J_pose, d0, sizeof(double) * 12 * n, cudaMemcpyDeviceToHost, c->stream));
  if (J_lm) OKB_CUDA(c, cudaMemcpyAsync(J_lm, d1, sizeof(double) * 6 * n, cudaMemcpyDeviceToHost, c->stream));
  if (J_ext) OKB_CUDA(c, cudaMemcpyAsync(J_ext, d2, sizeof(double) * 12 * n, cudaMemcpyDeviceToHost, c->stream));
  OKB_CUDA(c, cudaStreamSynchronize(c->stream));
  return OKB_OK;
}

extern "C" int okb_eval_imu(okb_ctx* c, const okb_imu_params* prm, const okb_imu_sample* samples, int n_samples, int64_t t0_ns,
                            int64_t t1_ns, const double* pose0, const double* sb0, const double* pose1, const double* sb1,
                            const double* sb_ref, double* r, double* J0, double* J1, double* J2, double* J3,
                            double* sqrt_info_out) {
  if (!c || !prm || !samples || n_samples < 2) return OKB_ERR_INVALID_ARG;
  cudaSetDevice(c->device);
  const size_t sbytes = align_up(sizeof(okb_imu_sample) * n_samples, 256);
  const size_t total = sbytes + align_up(sizeof(ImuCache), 256) + sizeof(double) * (32 + 9 + 7 + 700);
  int rc = grow(c, &c->hook_buf, &c->hook_bytes, total);
  if (rc) return rc;
  unsigned char* base = c->hook_buf;
  okb_imu_sample* ds = reinterpret_cast<okb_imu_sample*>(base);
  ImuCache* dc = reinterpret_cast<ImuCache*>(base + sbytes);
  double* din = reinterpret_cast<double*>(base + sbytes + align_up(sizeof(ImuCache), 256));
  double* dref = din + 32;
  double* dout = dref + 16;
  double hin[32];
  std::memcpy(hin, pose0, 56); std::memcpy(hin + 7, sb0, 72); std::memcpy(hin + 16, pose1, 56); std::memcpy(hin + 23, sb1, 72);
  OKB_CUDA(c, cudaMemcpyAsync(ds, samples, sizeof(okb_imu_sample) * n_samples, cudaMemcpyHostToDevice, c->stream));
  OKB_CUDA(c, cudaMemcpyAsync(din, hin, sizeof(hin), cudaMemcpyHostToDevice, c->stream));
  if (sb_ref) OKB_CUDA(c, cudaMemcpyAsync(dref, sb_ref, 72, cudaMemcpyHostToDevice, c->stream));
  OKB_CUDA(c, cudaStreamSynchronize(c->stream));
  k_hook_imu<<<1, 32, 0, c->stream>>>(*prm, ds, n_samples, t0_ns, t1_ns, din, dref, sb_ref ? 1 : 0, dc, dout);
  c->launches += 1;
  OKB_CUDA(c, cudaGetLastError());
  std::vector<double> h(691);
  OKB_CUDA(c, cudaMemcpyAsync(h.data(), dout, sizeof(double) * 691, cudaMemcpyDeviceToHost, c->stream));
  OKB_CUDA(c, cudaStreamSynchronize(c->stream));
  if (r) std::memcpy(r, h.data(), 15 * 8);
  const double* SF = h.data() + 15;
  for (int rr = 0; rr < 15; ++rr) {
    for (int cc = 0; cc < 6; ++cc) { if (J0) J0[rr * 6 + cc] = SF[rr * 30 + cc]; if (J2) J2[rr * 6 + cc] = SF[rr * 30 + 15 + cc]; }
    for (int cc = 0; cc < 9; ++cc) { if (J1) J1[rr * 9 + cc] = SF[rr * 30 + 6 + cc]; if (J3) J3[rr * 9 + cc] = SF[rr * 30 + 21 + cc]; }
  }
  if (sqrt_info_out) std::memcpy(sqrt_info_out, h.data() + 465, 225 * 8);
  return (int)h[690] > 0 ? 1 : 0;   // 1 = the evaluation re-preintegrated (not an error)
}

// The argument checks of okb_imu_propagate, per job: the reason a job is rejected, or nullptr.
static const char* prop_invalid(const okb_propagate_job& j) {
  if (!j.params) return "params is NULL";
  if (!j.samples) return "samples is NULL";
  if (j.n_samples < 2) return "n_samples < 2";
  if (!j.pose) return "pose is NULL";
  if (!j.speed_bias) return "speed_bias is NULL";
  return nullptr;
}

// Propagates n checked jobs on stream st through buffers B (the caller holds B.mtx): one H2D copy of the job table and
// all samples, one k_propagate launch (one warp per job), one D2H copy of the output records, one synchronisation.
static int prop_run(okb_ctx* c, cudaStream_t st, CallBuffers& B, int n, const okb_propagate_job* jobs) {
  std::vector<size_t> s_off(n), o_off(n);
  Carve in, out;
  in.take(sizeof(PropEntry) * n, 256);
  for (int i = 0; i < n; ++i) {
    s_off[i] = in.take(sizeof(okb_imu_sample) * (size_t)jobs[i].n_samples);
    o_off[i] = out.take(sizeof(double) * (kPropRecord + (jobs[i].covariance ? 225 : 0) + (jobs[i].jacobian ? 225 : 0)), 8);
  }
  const size_t in_bytes = in.off, out_bytes = out.off, out_at = align_up(in_bytes, 256);
  const int rc = B.reserve(c, align_up(std::max(out_at + out_bytes, (size_t)64 << 10), 4096), 0);
  if (rc) return rc;
  unsigned char *host = B.h_stage, *dev = B.d_stage;
  PropEntry* tab = reinterpret_cast<PropEntry*>(host);
  for (int i = 0; i < n; ++i) {
    const okb_propagate_job& j = jobs[i];
    PropEntry& e = tab[i];
    std::memset(&e, 0, sizeof e);
    e.prm = *j.params;
    e.t0 = j.t0_ns; e.t1 = j.t1_ns;
    e.samples = s_off[i]; e.out = o_off[i];
    e.n = j.n_samples; e.want_cov = j.covariance ? 1 : 0; e.want_jac = j.jacobian ? 1 : 0;
    std::memcpy(e.state, j.pose, 7 * sizeof(double));
    std::memcpy(e.state + 7, j.speed_bias, 9 * sizeof(double));
    std::memcpy(host + s_off[i], j.samples, sizeof(okb_imu_sample) * (size_t)j.n_samples);
  }
  OKB_CUDA(c, cudaMemcpyAsync(dev, host, in_bytes, cudaMemcpyHostToDevice, st));
  k_propagate<<<n, 32, 0, st>>>(dev, dev + out_at);
  c->prop_launches += 1;
  OKB_CUDA(c, cudaGetLastError());
  OKB_CUDA(c, cudaMemcpyAsync(host + out_at, dev + out_at, out_bytes, cudaMemcpyDeviceToHost, st));
  OKB_CUDA(c, cudaStreamSynchronize(st));
  for (int i = 0; i < n; ++i) {
    const okb_propagate_job& j = jobs[i];
    const double* o = reinterpret_cast<const double*>(host + out_at + o_off[i]);
    int32_t used;
    std::memcpy(&used, o + 16, sizeof used);
    if (used >= 0) {
      std::memcpy(j.pose, o, 7 * sizeof(double));
      std::memcpy(j.speed_bias, o + 7, 9 * sizeof(double));
      if (j.covariance) std::memcpy(j.covariance, o + kPropRecord, 225 * sizeof(double));
      if (j.jacobian) std::memcpy(j.jacobian, o + kPropRecord + (j.covariance ? 225 : 0), 225 * sizeof(double));
    }
    if (j.n_used) *j.n_used = used;
  }
  return OKB_OK;
}

// A batch of one on the solver stream, so that it stays ordered after the solver work already launched.
extern "C" int okb_imu_propagate(okb_ctx* c, const okb_imu_params* prm, const okb_imu_sample* samples, int n_samples,
                                 int64_t t0_ns, int64_t t1_ns, double* pose, double* sb, double* covariance, double* jacobian,
                                 int* n_used) {
  const okb_propagate_job j{prm, samples, n_samples, 0, t0_ns, t1_ns, pose, sb, covariance, jacobian, n_used};
  if (!c || prop_invalid(j)) return OKB_ERR_INVALID_ARG;
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> lk(c->prop_one.mtx);
  return prop_run(c, c->stream, c->prop_one, 1, &j);
}

extern "C" int okb_imu_propagate_batch(okb_ctx* c, int n_jobs, const okb_propagate_job* jobs) {
  if (!c) return OKB_ERR_INVALID_ARG;
  if (n_jobs < 0 || (n_jobs > 0 && !jobs)) {
    c->set_error("okb_imu_propagate_batch: n_jobs < 0, or jobs is NULL");
    return OKB_ERR_INVALID_ARG;
  }
  if (n_jobs == 0) return OKB_OK;
  for (int i = 0; i < n_jobs; ++i)
    if (const char* why = prop_invalid(jobs[i])) {
      c->set_error("okb_imu_propagate_batch: job " + std::to_string(i) + ": " + why);
      return OKB_ERR_INVALID_ARG;
    }
  cudaSetDevice(c->device);
  std::lock_guard<std::mutex> lk(c->prop_batch.mtx);
  if (!c->stream_prop) OKB_CUDA(c, create_high_priority_stream(&c->stream_prop));
  return prop_run(c, c->stream_prop, c->prop_batch, n_jobs, jobs);
}

// One single-CTA hook on the solver stream: nin packed input doubles in one H2D copy, a synchronisation, one launch of
// kernel(in, out) with `threads` threads, nout output doubles in one D2H copy, a synchronisation.
static int run_hook(okb_ctx* c, void (*kernel)(const double*, double*), int threads, const double* in, int nin, double* out, int nout) {
  cudaSetDevice(c->device);
  const int rc = grow(c, &c->hook_buf, &c->hook_bytes, sizeof(double) * (nin + nout));
  if (rc) return rc;
  double* d = reinterpret_cast<double*>(c->hook_buf);
  OKB_CUDA(c, cudaMemcpyAsync(d, in, sizeof(double) * nin, cudaMemcpyHostToDevice, c->stream));
  OKB_CUDA(c, cudaStreamSynchronize(c->stream));
  kernel<<<1, threads, 0, c->stream>>>(d, d + nin);
  c->launches += 1;
  OKB_CUDA(c, cudaMemcpyAsync(out, d + nin, sizeof(double) * nout, cudaMemcpyDeviceToHost, c->stream));
  OKB_CUDA(c, cudaStreamSynchronize(c->stream));
  return OKB_OK;
}

extern "C" int okb_eval_pose_error(okb_ctx* c, const double* meas, const double* sqrt_info, const double* pose, double* r, double* J) {
  if (!c) return OKB_ERR_INVALID_ARG;
  double h[50], o[42];
  std::memcpy(h, meas, 56); std::memcpy(h + 7, sqrt_info, 288); std::memcpy(h + 43, pose, 56);
  const int rc = run_hook(c, k_hook_pose, 32, h, 50, o, 42);
  if (rc) return rc;
  if (r) std::memcpy(r, o, 48);
  if (J) std::memcpy(J, o + 6, 288);
  return OKB_OK;
}

namespace {
__global__ void k_hook_sb(const double* in /* meas9 S81 sb9 */, double* out /* r9 J81 */) {
  const int t = threadIdx.x;
  if (t < 9) {
    double s = 0;
    for (int k = 0; k < 9; ++k) s += in[9 + t * 9 + k] * (in[k] - in[90 + k]);
    out[t] = s;
  }
  for (int e = t; e < 81; e += blockDim.x) out[9 + e] = -in[9 + e];
}
}  // namespace

extern "C" int okb_eval_speed_bias_error(okb_ctx* c, const double* meas, const double* sqrt_info, const double* sb, double* r, double* J) {
  if (!c || !meas || !sqrt_info || !sb) return OKB_ERR_INVALID_ARG;
  double h[99], o[90];
  std::memcpy(h, meas, 72); std::memcpy(h + 9, sqrt_info, 648); std::memcpy(h + 90, sb, 72);
  const int rc = run_hook(c, k_hook_sb, 96, h, 99, o, 90);
  if (rc) return rc;
  if (r) std::memcpy(r, o, 72);
  if (J) std::memcpy(J, o + 9, 648);
  return OKB_OK;
}

extern "C" int okb_eval_relative_pose(okb_ctx* c, const double* sqrt_info, const double* pose0, const double* pose1, double* r,
                                      double* J0, double* J1) {
  if (!c) return OKB_ERR_INVALID_ARG;
  double h[50], o[78];
  std::memcpy(h, sqrt_info, 288); std::memcpy(h + 36, pose0, 56); std::memcpy(h + 43, pose1, 56);
  const int rc = run_hook(c, k_hook_relpose, 32, h, 50, o, 78);
  if (rc) return rc;
  if (r) std::memcpy(r, o, 48);
  if (J0) std::memcpy(J0, o + 6, 288);
  if (J1) std::memcpy(J1, o + 42, 288);
  return OKB_OK;
}

namespace {
__global__ void k_hook_marg(int n, int nb, const int32_t* kind, const int32_t* col, const int32_t* off, const double* x0,
                            const double* x, const double* J, const double* e0, double* r, double* Jeff) {
  extern __shared__ double dchi[];
  const int tid = threadIdx.x;
  for (int b = tid; b < nb; b += blockDim.x) {
    if (kind[b] == OKB_BLOCK_SPEED_BIAS) for (int k = 0; k < 9; ++k) dchi[col[b] + k] = x[off[b] + k] - x0[off[b] + k];
    else pose_minus(x0 + off[b], x + off[b], dchi + col[b]);
  }
  __syncthreads();
  for (int i = tid; i < n; i += blockDim.x) {
    double s = e0[i];
    for (int k = 0; k < n; ++k) s += J[(size_t)i * n + k] * dchi[k];
    r[i] = s;
  }
  for (int b = 0; b < nb; ++b) {
    const int m = (kind[b] == OKB_BLOCK_SPEED_BIAS) ? 9 : 6;
    double B[9];
    if (m == 6) marg_pose_rot_block(x0 + off[b], x + off[b], B);
    for (int e = tid; e < n * m; e += blockDim.x) {
      const int i = e / m, a = e % m;
      double s;
      if (m == 9 || a < 3) s = J[(size_t)i * n + col[b] + a];
      else { s = 0; for (int k = 0; k < 3; ++k) s += J[(size_t)i * n + col[b] + 3 + k] * B[k * 3 + (a - 3)]; }
      Jeff[(size_t)i * n + col[b] + a] = s;
    }
  }
}
}  // namespace

extern "C" int okb_eval_marginalization(okb_ctx* c, const okb_marg_prior* m, const double* x, double* r, double* J_eff) {
  if (!c || !m || m->n < 1 || m->n > kMaxMarg) return OKB_ERR_INVALID_ARG;
  cudaSetDevice(c->device);
  const int n = m->n, nb = m->n_blocks;
  std::vector<int32_t> kind(nb), col(nb), off(nb);
  int cc = 0, xo = 0;
  for (int b = 0; b < nb; ++b) {
    kind[b] = m->block_kind[b]; col[b] = cc; off[b] = xo;
    cc += (kind[b] == OKB_BLOCK_SPEED_BIAS) ? 9 : 6;
    xo += (kind[b] == OKB_BLOCK_SPEED_BIAS) ? 9 : 7;
  }
  if (cc != n) return OKB_ERR_INVALID_ARG;
  const size_t ints = align_up(sizeof(int32_t) * 3 * nb, 256);
  const size_t total = ints + sizeof(double) * (2 * xo + (size_t)2 * n * n + 2 * n);
  int rc = grow(c, &c->hook_buf, &c->hook_bytes, total);
  if (rc) return rc;
  unsigned char* base = c->hook_buf;
  int32_t* dk = reinterpret_cast<int32_t*>(base);
  double* dx0 = reinterpret_cast<double*>(base + ints);
  double *dx = dx0 + xo, *dJ = dx + xo, *de0 = dJ + (size_t)n * n, *dr = de0 + n, *dJe = dr + n;
  OKB_CUDA(c, cudaMemcpyAsync(dk, kind.data(), 4 * nb, cudaMemcpyHostToDevice, c->stream));
  OKB_CUDA(c, cudaMemcpyAsync(dk + nb, col.data(), 4 * nb, cudaMemcpyHostToDevice, c->stream));
  OKB_CUDA(c, cudaMemcpyAsync(dk + 2 * nb, off.data(), 4 * nb, cudaMemcpyHostToDevice, c->stream));
  OKB_CUDA(c, cudaMemcpyAsync(dx0, m->x0, 8 * xo, cudaMemcpyHostToDevice, c->stream));
  OKB_CUDA(c, cudaMemcpyAsync(dx, x, 8 * xo, cudaMemcpyHostToDevice, c->stream));
  OKB_CUDA(c, cudaMemcpyAsync(dJ, m->J, 8 * (size_t)n * n, cudaMemcpyHostToDevice, c->stream));
  OKB_CUDA(c, cudaMemcpyAsync(de0, m->e0, 8 * n, cudaMemcpyHostToDevice, c->stream));
  OKB_CUDA(c, cudaStreamSynchronize(c->stream));
  k_hook_marg<<<1, 256, sizeof(double) * n, c->stream>>>(n, nb, dk, dk + nb, dk + 2 * nb, dx0, dx, dJ, de0, dr, dJe);
  c->launches += 1;
  OKB_CUDA(c, cudaGetLastError());
  if (r) OKB_CUDA(c, cudaMemcpyAsync(r, dr, 8 * n, cudaMemcpyDeviceToHost, c->stream));
  if (J_eff) OKB_CUDA(c, cudaMemcpyAsync(J_eff, dJe, 8 * (size_t)n * n, cudaMemcpyDeviceToHost, c->stream));
  OKB_CUDA(c, cudaStreamSynchronize(c->stream));
  return OKB_OK;
}
