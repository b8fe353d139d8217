// Opaque context behind the C-ABI handle (host side).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/okvis_b200.h"
#include "okb_estimator.cuh"

// Capacities an arena is planned for: frames, landmarks, observations, IMU samples / terms, extrinsics, cameras,
// priors per kind, marginalisation prior dimension.
struct WinCaps { int K = 0, L = 0, O = 0, S = 0, T = 0, NE = 0, NC = 0, PP = 0, MN = 0; };

struct WinStore {
  unsigned char* arena = nullptr;     // device
  size_t arena_bytes = 0;
  WinCaps caps, reserve;              // what the arena holds / the minimum asked for by okb_window_reserve
  unsigned char* staging = nullptr;   // pinned: the pending command stream of the slot (okb_graph.cuh)
  size_t staging_bytes = 0;
  size_t cmd_used = 0;                // bytes of commands not yet committed
  size_t cmd_cap_dev = 0;             // size of the device-side command buffer
  bool staging_busy = false;          // an H2D copy of `staging` may still be in flight (wait on `copied` before rewriting)
  bool full_pending = false;          // the pending stream is a full upload
  bool committed = false;
  int obs_bound = 0;                  // upper bound of the device-side observation list length
  int K_init = 0, NSB_init = 0, L_init = 0;   // shape at the last full upload (okb_window_reset)
  int cam_model = okb::kDistAny;      // distortion model shared by all cameras of the last full upload, else kDistAny
  std::vector<okb_imu_term> terms;    // host mirror of the IMU terms / prior indices (dimension bookkeeping of remove_frame)
  std::vector<uint32_t> pp_idx, sbp_idx;
  size_t h2d_bytes = 0;
  bool uploaded = false;
  cudaEvent_t copied = nullptr;       // recorded after the H2D copy of `staging`
  unsigned char* out_staging = nullptr;  // pinned host buffer the estimates are downloaded into
  size_t out_bytes = 0;
  cudaEvent_t down = nullptr;         // recorded after the D2H copies of a download
  okb_solve_options opt{};            // options of the last okb_optimize_async on this slot
  int done_idx = -1;                  // index into okb_ctx::done_ring of the last solver work launched on this slot
  unsigned char* marg_scratch = nullptr;   // device scratch of okb_window_marginalize (okb_marg.cuh), allocated on first use
  size_t marg_scratch_bytes = 0;
  int marg_lm_cap = 0, marg_K_cap = 0, marg_L_cap = 0, marg_O_cap = 0;
  // feature store (okb_window_reserve_features): one device allocation headed by the FeatStore struct, a host copy of
  // that struct, and the keypoint count per (feature slot, camera) as committed / including pending commands (-1: none)
  unsigned char* feat_mem = nullptr;
  okb::FeatStore feat{};
  std::vector<int> feat_n, feat_n_pending;
  size_t feat_frame_bytes = 0;        // commands of one frame's features + every initialised flag: the device command
                                      // buffer (plan_arena) holds them on top of a full upload
};

// Commits the pending commands of the n listed slots on the transfer stream, once per run of consecutive slots after
// sorting, then makes the transfer stream wait once on each distinct solver event of those slots (okb_estimator.cu).
int okb_commit_windows(okb_ctx* c, const int32_t* wins, int n);

// Buffers of one kind of table-driven call: a pinned staging buffer and its device mirror (tables in, results out, one
// copy each way), device-only scratch, and the mutex that serialises the calls using them.  They grow with the largest
// call and are kept.  The Hamming matcher's sets are held under match_mtx / batch_mtx, which guard other buffers too.
struct CallBuffers {
  uint8_t* h_stage = nullptr;      // pinned
  uint8_t* d_stage = nullptr;
  uint8_t* d_scratch = nullptr;
  size_t h_stage_cap = 0, d_stage_cap = 0, d_scratch_cap = 0;
  std::mutex mtx;
  // Grows the buffers to `stage` bytes of staging (pinned and its device mirror) and `scratch` bytes of device scratch.
  int reserve(okb_ctx* c, size_t stage, size_t scratch);
  void release() {
    if (h_stage) cudaFreeHost(h_stage);
    cudaFree(d_stage);
    cudaFree(d_scratch);
  }
};

struct okb_frontend_state;

struct okb_ctx {
  int device = 0;
  int max_windows = 0;
  int sm_count = 132;
  int smem_optin = 0;
  int smem_per_sm = 0;
  int chunk_cap = 1;
  cudaStream_t stream = nullptr;
  cudaStream_t stream_imu = nullptr;     // k_imu runs beside the landmark kernels
  cudaEvent_t ev_round = nullptr, ev_imu = nullptr;
  // Window groups of a batched solve (launch_rounds): group g runs its round chain on group_stream[g] with k_imu on
  // group_imu[g].  Group 0 is the context's own chain: entry 0 aliases stream / stream_imu / ev_round / ev_imu and is
  // not destroyed separately.  group_stagger[g] is recorded on group g's stream after its first k_landmarks, and group
  // g+1 starts behind it; group_done[g] (g >= 1) joins group g back into `stream`.
  static constexpr int kMaxSolveGroups = 4;
  cudaStream_t group_stream[kMaxSolveGroups] = {}, group_imu[kMaxSolveGroups] = {};
  cudaEvent_t group_round[kMaxSolveGroups] = {}, group_imu_done[kMaxSolveGroups] = {};
  cudaEvent_t group_stagger[kMaxSolveGroups] = {}, group_done[kMaxSolveGroups] = {};
  int solve_groups = 0;                  // okb_set_solve_groups: 0 = automatic (plan_rounds)
  // Transfers (window uploads / estimate downloads) run on their own stream so that they overlap solver
  // kernels of other windows.  ev_join orders the solver stream after all uploads issued so far;
  // done_ring[k] is recorded on the solver stream after each optimize / reset and transfers of the
  // windows it touched wait on it.
  cudaStream_t stream_xfer = nullptr;
  cudaEvent_t ev_join = nullptr;
  static constexpr int kDoneRing = 8;
  cudaEvent_t done_ring[kDoneRing] = {};
  int done_next = 0;
  // Slot tables: the solver kernels find their windows as wins[win_slots[blockIdx]].  d_slot_tab holds the table of the
  // optimize being launched on `stream` (a captured graph reads it, so any set of one size replays one graph); it is
  // written by an H2D copy on `stream` from entry k of the pinned ring h_slot_ring, where k is the done_ring index
  // the launch will mark, so an entry is rewritten only after done_ring[k] -- the last work that copied it -- is
  // complete.  d_ident = 0, 1, 2, ...: the table of range calls on other streams (okb_window_reset).
  int32_t* d_slot_tab = nullptr;
  int32_t* d_ident = nullptr;
  int32_t* h_slot_ring = nullptr;       // pinned, [kDoneRing][max_windows]
  std::vector<int32_t> ident;           // host 0, 1, 2, ...: the slot list of a range call
  std::vector<WinStore> wins;
  std::vector<okb::WinDev> host;      // host mirror of d_wins
  okb::WinDev* d_wins = nullptr;
  okb::SolverState* d_states = nullptr;
  okb::SolverState* h_states = nullptr;  // pinned
  unsigned char* hook_buf = nullptr;
  size_t hook_bytes = 0;
  // okb_window_marginalize*: task table + job payloads of a call, packed in pinned memory and copied in one piece
  unsigned char* marg_host = nullptr;    // pinned
  unsigned char* marg_dev = nullptr;
  size_t marg_host_bytes = 0, marg_dev_bytes = 0;
  cudaEvent_t marg_copied = nullptr;     // recorded after the H2D copy of marg_host
  bool marg_busy = false;                // that copy may still be in flight (wait on marg_copied before rewriting)
  // Buffers a landmark-sharded context outgrew, freed with the context: cudaFree / cudaFreeHost wait for the whole
  // device, and a peer rank on the same device may be spinning in k_marginalize until this rank's launch arrives.
  // Growth doubles, so these stay bounded.
  std::vector<unsigned char*> marg_retired_dev, marg_retired_host;
  // Sharded contexts: pinned pack buffers whose H2D copy was still queued when the next call came; reused once `done`
  // (recorded after that copy) has completed, so a pipelining host needs at most one buffer per call in flight.
  struct MargPinned { unsigned char* p; size_t bytes; cudaEvent_t done; };
  std::vector<MargPinned> marg_pool;
  // okb_imu_propagate (on `stream`) and okb_imu_propagate_batch (on stream_prop, created on first use) each own a set
  // of staging buffers ([job table | samples] in, [per-job outputs] out; no scratch)
  CallBuffers prop_one, prop_batch;
  cudaStream_t stream_prop = nullptr;
  std::atomic<int64_t> prop_launches{0};   // counted apart from `launches`: a batch may run beside a solve's launches
  okb_frontend_state* frontend = nullptr;
  // landmark-sharded windows (okb_shard_*): this rank's mailbox and the peers' mailboxes as mapped on this device
  int shard_rank = 0, shard_world = 1, shard_box_cap = 0, shard_marg_cap = 0;
  int shard_lm_cap = 0;                                       // global landmark slots of the frontend's replica
  size_t shard_win_bytes = 0;
  unsigned char* shard_local = nullptr;                       // cudaMalloc'ed, exported through cudaIpc
  unsigned char* shard_peer[okb::kMaxShard] = {};             // [rank]; own entry = shard_local
  bool shard_peer_ipc[okb::kMaxShard] = {};                   // opened with cudaIpcOpenMemHandle (closed at destroy)
  int64_t launches = 0;
  // captured launch sequences of okb_optimize* (run_rounds): key fields up to `exec`, compared bytewise; the windows
  // come from d_slot_tab, so the key holds the batch size, not which slots
  struct GraphEntry {
    int count, rounds, with_quality, opt_iter, opt_min, opt_cauchy;
    double opt_time;
    unsigned char plan[96];
    cudaGraphExec_t exec;
    int64_t launches;
    uint64_t stamp;
  };
  std::vector<GraphEntry> graphs;
  uint64_t graph_clock = 0;
  bool profile = false;
  std::vector<cudaEvent_t> prof_events;   // pairs (start, stop)
  std::vector<int> prof_kind;             // kernel id per pair
  std::vector<int> prof_join;             // per pair: index of the first pair of its span (itself, unless grouped)
  size_t prof_used = 0;
  std::string error;
  std::mutex error_mu;                    // uploads of different slots may run on several host threads
  void set_error(const std::string& e) { std::lock_guard<std::mutex> g(error_mu); error = e; }
};

// Returns OKB_ERR_CUDA with the failing call and the CUDA error as the context's error text unless `call` succeeds.
#define OKB_CUDA(ctx, call)                                                     \
  do {                                                                          \
    cudaError_t e_ = (call);                                                    \
    if (e_ != cudaSuccess) {                                                    \
      (ctx)->set_error(std::string(#call) + ": " + cudaGetErrorString(e_));     \
      return OKB_ERR_CUDA;                                                      \
    }                                                                           \
  } while (0)

// Grows the device allocation *p to at least `need` elements: frees it and allocates exactly `need`; contents are lost.
template <typename T>
int grow(okb_ctx* c, T** p, size_t* cap, size_t need) {
  if (*cap >= need) return OKB_OK;
  cudaFree(*p);
  *p = nullptr; *cap = 0;
  OKB_CUDA(c, cudaMalloc(p, need * sizeof(T)));
  *cap = need;
  return OKB_OK;
}

// grow for pinned host memory.
template <typename T>
int grow_pinned(okb_ctx* c, T** p, size_t* cap, size_t need) {
  if (*cap >= need) return OKB_OK;
  if (*p) cudaFreeHost(*p);
  *p = nullptr; *cap = 0;
  OKB_CUDA(c, cudaMallocHost(p, need * sizeof(T)));
  *cap = need;
  return OKB_OK;
}

inline int CallBuffers::reserve(okb_ctx* c, size_t stage, size_t scratch) {
  int rc;
  if ((rc = grow_pinned(c, &h_stage, &h_stage_cap, stage)) || (rc = grow(c, &d_stage, &d_stage_cap, stage)) ||
      (rc = grow(c, &d_scratch, &d_scratch_cap, scratch)))
    return rc;
  return OKB_OK;
}

// Makes `stream` wait once on each distinct solver event (done_ring entry) of the n listed slots, so that what is
// queued on it next runs after the solver work already launched on them.
inline int wait_solver_work(okb_ctx* c, cudaStream_t stream, const int32_t* slots, int n) {
  bool waited[okb_ctx::kDoneRing] = {};
  for (int i = 0; i < n; ++i) {
    const int k = c->wins[slots[i]].done_idx;
    if (k >= 0 && !waited[k]) { OKB_CUDA(c, cudaStreamWaitEvent(stream, c->done_ring[k], 0)); waited[k] = true; }
  }
  return OKB_OK;
}

void okb_frontend_release(okb_ctx* c);
int64_t okb_frontend_launches(const okb_ctx* c);   // kernel launches of the frontend calls (counted atomically)
