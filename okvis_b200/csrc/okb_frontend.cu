// Frontend path of libokvis_b200.so (sm_90a): Harris detect -> uniformity -> gravity-aligned
// 48/64-byte binary descriptor, and the DenseMatcher Hamming brute force.
//   okb_detect_describe   <- Frontend::detectAndDescribe (okvis_frontend/src/Frontend.cpp:92-114)
//   okb_hamming_match     <- DenseMatcher::match          (okvis_matcher/include/okvis/implementation/DenseMatcher.hpp:48-225,
//                                                          okvis_matcher/src/DenseMatcher.cpp:69-110)
//   okb_hamming_candidates<- VioKeyframeWindowMatchingAlgorithm::specificDescriptorDistance (…hpp:246-254)
// The detector / descriptor follow this project's own specification (DESIGN.md "Frontend spec"):
// brisk 2.0.5 is not part of the reference tree.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include "okb_ctx.h"
#include "okb_math.cuh"

using namespace okb;

#define FE_CUDA(ctx, call)                                                      \
  do {                                                                          \
    cudaError_t e_ = (call);                                                    \
    if (e_ != cudaSuccess) {                                                    \
      (ctx)->set_error(std::string(#call) + ": " + cudaGetErrorString(e_));     \
      return OKB_ERR_CUDA;                                                      \
    }                                                                           \
  } while (0)

namespace {
constexpr int kBorder = 16;
constexpr int kRotBins = 1024;
constexpr int kPts = 60;
constexpr int kMaxSlots = 8;          // concurrent camera slots
constexpr int kMaxCand = 1 << 17;     // NMS candidates per image

struct Pattern {
  int half[kPts];
  std::vector<uint8_t> pi, pj;
  std::vector<int16_t> lut;
};

Pattern make_pattern(int desc_bytes) {
  Pattern P;
  double px[kPts], py[kPts];
  const double rList[5] = {0.0, 2.9 * 0.85, 4.9 * 0.85, 7.4 * 0.85, 10.8 * 0.85};
  const int nList[5] = {1, 10, 14, 15, 20};
  int idx = 0;
  for (int ring = 0; ring < 5; ++ring) {
    const double sigma = 1.3 * (ring == 0 ? rList[1] * std::sin(M_PI / nList[1]) : rList[ring] * std::sin(M_PI / nList[ring]));
    for (int a = 0; a < nList[ring]; ++a) {
      const double alpha = 2.0 * M_PI * a / nList[ring];
      px[idx] = rList[ring] * std::cos(alpha);
      py[idx] = rList[ring] * std::sin(alpha);
      P.half[idx] = std::max(1, (int)std::lround(sigma));
      ++idx;
    }
  }
  // squared distances are quantised to 1e-6 so that the ordering of (mathematically) equal
  // distances does not depend on the compiler's floating-point contraction
  struct Pr { long long d; int i, j; };
  std::vector<Pr> all;
  for (int i = 0; i < kPts; ++i)
    for (int j = i + 1; j < kPts; ++j) {
      const double dx = px[i] - px[j], dy = py[i] - py[j];
      all.push_back({std::llround((dx * dx + dy * dy) * 1e6), i, j});
    }
  std::stable_sort(all.begin(), all.end(), [](const Pr& a, const Pr& b) {
    if (a.d != b.d) return a.d < b.d;
    if (a.i != b.i) return a.i < b.i;
    return a.j < b.j;
  });
  for (int k = 0; k < 8 * desc_bytes; ++k) { P.pi.push_back((uint8_t)all[k].i); P.pj.push_back((uint8_t)all[k].j); }
  P.lut.resize((size_t)kRotBins * kPts * 2);
  for (int r = 0; r < kRotBins; ++r) {
    const double ang = 2.0 * M_PI * r / kRotBins, c = std::cos(ang), s = std::sin(ang);
    for (int p = 0; p < kPts; ++p) {
      P.lut[((size_t)r * kPts + p) * 2 + 0] = (int16_t)std::lround(px[p] * c - py[p] * s);
      P.lut[((size_t)r * kPts + p) * 2 + 1] = (int16_t)std::lround(px[p] * s + py[p] * c);
    }
  }
  return P;
}

struct SlotBuffers {
  cudaStream_t stream = nullptr;
  int W = 0, H = 0;
  uint8_t* d_img = nullptr;
  int32_t* d_score = nullptr;
  uint32_t* d_integral = nullptr;
  unsigned long long* d_keys = nullptr;
  int* d_count = nullptr;          // [0] candidates, [1] accepted
  uint32_t *d_cell_start = nullptr, *d_cell_cur = nullptr, *d_order = nullptr, *d_acc = nullptr;   // uniformity scratch
  uint32_t* d_rounds = nullptr;      // [4][kMaxCand]: blocker | alive list 0 | alive list 1 | pending
  uint8_t* d_state = nullptr;
  int max_cells = 0;
  okb_keypoint* d_kp = nullptr;
  uint8_t* d_desc = nullptr;
  int kp_cap = 0, desc_cap = 0;
  uint8_t* h_img = nullptr;        // pinned
  okb_keypoint* h_kp = nullptr;    // pinned
  uint8_t* h_desc = nullptr;       // pinned
  int* h_count = nullptr;          // pinned
  std::mutex mtx;
};
}  // namespace

struct okb_frontend_state {
  SlotBuffers slots[kMaxSlots];
  // pattern (device), per descriptor length
  int pat_bytes = 0;
  int* d_half = nullptr;
  uint8_t *d_pi = nullptr, *d_pj = nullptr;
  int16_t* d_lut = nullptr;
  std::mutex pat_mtx;
  // matcher buffers
  uint8_t *d_A = nullptr, *d_B = nullptr, *d_skipA = nullptr, *d_skipB = nullptr;
  size_t capA = 0, capB = 0;
  okb_pair *d_topk = nullptr, *d_pairs = nullptr;
  size_t cap_topk = 0, cap_pairs = 0;
  uint32_t *d_rowptr = nullptr, *d_col = nullptr;
  uint16_t* d_dist = nullptr;
  size_t cap_rows = 0, cap_cand = 0;
  uint8_t* h_stage = nullptr;      // pinned staging: descriptors in, top-k lists + winners out
  size_t h_stage_cap = 0;
  uint8_t* d_io = nullptr;         // device mirror of the staging buffer
  size_t d_io_cap = 0;
  std::mutex match_mtx;
};

void okb_frontend_release(okb_ctx* c) {
  if (!c->frontend) return;
  okb_frontend_state* F = c->frontend;
  if (F->h_stage) cudaFreeHost(F->h_stage);
  cudaFree(F->d_io);
  for (auto& s : F->slots) {
    if (s.stream) cudaStreamDestroy(s.stream);
    cudaFree(s.d_img); cudaFree(s.d_score); cudaFree(s.d_integral); cudaFree(s.d_keys);
    cudaFree(s.d_cell_start); cudaFree(s.d_cell_cur); cudaFree(s.d_order); cudaFree(s.d_acc); cudaFree(s.d_state); cudaFree(s.d_rounds);
    cudaFree(s.d_count); cudaFree(s.d_kp); cudaFree(s.d_desc);
    if (s.h_img) cudaFreeHost(s.h_img);
    if (s.h_kp) cudaFreeHost(s.h_kp);
    if (s.h_desc) cudaFreeHost(s.h_desc);
    if (s.h_count) cudaFreeHost(s.h_count);
  }
  cudaFree(F->d_half); cudaFree(F->d_pi); cudaFree(F->d_pj); cudaFree(F->d_lut);
  cudaFree(F->d_A); cudaFree(F->d_B); cudaFree(F->d_skipA); cudaFree(F->d_skipB); cudaFree(F->d_topk); cudaFree(F->d_pairs);
  cudaFree(F->d_rowptr); cudaFree(F->d_col); cudaFree(F->d_dist);
  delete F;
  c->frontend = nullptr;
}

static okb_frontend_state* fe(okb_ctx* c) {
  static std::mutex m;
  std::lock_guard<std::mutex> lk(m);
  if (!c->frontend) c->frontend = new okb_frontend_state();
  return c->frontend;
}

// =================================================================================================
// detector kernels
// =================================================================================================
namespace {
constexpr int HT_X = 32, HT_Y = 8;

// Integer Harris score: Scharr gradients, 5x5 binomial window.  One thread per pixel; the tile's
// gradient products live in shared memory.
__global__ void __launch_bounds__(HT_X* HT_Y) k_harris(const uint8_t* __restrict__ img, int W, int H, int32_t* __restrict__ score) {
  __shared__ uint8_t tile[HT_Y + 6][HT_X + 6 + 2];
  __shared__ int32_t sxx[HT_Y + 4][HT_X + 4], syy[HT_Y + 4][HT_X + 4], sxy[HT_Y + 4][HT_X + 4];
  const int bx = blockIdx.x * HT_X, by = blockIdx.y * HT_Y;
  const int tid = threadIdx.y * HT_X + threadIdx.x;
  for (int i = tid; i < (HT_Y + 6) * (HT_X + 6); i += HT_X * HT_Y) {
    const int ty = i / (HT_X + 6), tx = i % (HT_X + 6);
    const int gx = min(max(bx + tx - 3, 0), W - 1), gy = min(max(by + ty - 3, 0), H - 1);
    tile[ty][tx] = img[(size_t)gy * W + gx];
  }
  __syncthreads();
  for (int i = tid; i < (HT_Y + 4) * (HT_X + 4); i += HT_X * HT_Y) {
    const int ty = i / (HT_X + 4), tx = i % (HT_X + 4);
    const int gxp = bx + tx - 2, gyp = by + ty - 2;          // pixel whose gradient this is
    int vxx = 0, vyy = 0, vxy = 0;
    if (gxp >= 1 && gxp < W - 1 && gyp >= 1 && gyp < H - 1) {
      const int cy = ty + 1, cx = tx + 1;                     // tile coordinates of that pixel
      const int gx = 3 * ((int)tile[cy - 1][cx + 1] - (int)tile[cy - 1][cx - 1]) + 10 * ((int)tile[cy][cx + 1] - (int)tile[cy][cx - 1]) +
                     3 * ((int)tile[cy + 1][cx + 1] - (int)tile[cy + 1][cx - 1]);
      const int gy = 3 * ((int)tile[cy + 1][cx - 1] - (int)tile[cy - 1][cx - 1]) + 10 * ((int)tile[cy + 1][cx] - (int)tile[cy - 1][cx]) +
                     3 * ((int)tile[cy + 1][cx + 1] - (int)tile[cy - 1][cx + 1]);
      vxx = gx * gx; vyy = gy * gy; vxy = gx * gy;
    }
    sxx[ty][tx] = vxx; syy[ty][tx] = vyy; sxy[ty][tx] = vxy;
  }
  __syncthreads();
  const int x = bx + threadIdx.x, y = by + threadIdx.y;
  if (x >= W || y >= H) return;
  int32_t out = 0;
  if (x >= 3 && x < W - 3 && y >= 3 && y < H - 3) {
    const int w5[5] = {1, 4, 6, 4, 1};
    long long a = 0, b = 0, c = 0;
#pragma unroll
    for (int dy = 0; dy < 5; ++dy)
#pragma unroll
      for (int dx = 0; dx < 5; ++dx) {
        const long long wgt = w5[dy] * w5[dx];
        a += wgt * sxx[threadIdx.y + dy][threadIdx.x + dx];
        b += wgt * syy[threadIdx.y + dy][threadIdx.x + dx];
        c += wgt * sxy[threadIdx.y + dy][threadIdx.x + dx];
      }
    a >>= 8; b >>= 8; c >>= 8;
    long long s = (a * b - c * c) - (((a + b) * (a + b)) >> 4);
    s >>= 12;
    if (s > 2147483647LL) s = 2147483647LL;
    if (s < -2147483647LL) s = -2147483647LL;
    out = (int32_t)s;
  }
  score[(size_t)y * W + x] = out;
}

// 3x3 strict NMS + threshold + border -> sortable 64-bit keys (score desc, raster index asc)
__global__ void k_nms(const int32_t* __restrict__ score, int W, int H, int32_t thr, unsigned long long* keys, int* count, int cap) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x < kBorder || x >= W - kBorder || y < kBorder || y >= H - kBorder) return;
  const int32_t s = score[(size_t)y * W + x];
  if (s < thr) return;
  bool mx = true;
#pragma unroll
  for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
    for (int dx = -1; dx <= 1; ++dx) {
      if (dy == 0 && dx == 0) continue;
      mx = mx && (s > score[(size_t)(y + dy) * W + x + dx]);
    }
  if (!mx) return;
  const int slot = atomicAdd(count, 1);
  if (slot < cap) keys[slot] = ((unsigned long long)(uint32_t)s << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)(y * W + x));
}

// Uniformity.  Specification (DESIGN.md "Frontend spec"): walk the NMS candidates in descending (score, raster) order and
// accept a candidate iff no accepted one lies closer than `radius`; stop after max_kp.  That greedy pass is the
// lexicographically-first maximal independent set of the "closer than radius" graph, and it is computed here WITHOUT
// a sort and without a serial walk: in every round a candidate that has no live neighbour of higher priority is
// accepted, accepted candidates kill their live neighbours (Blelloch et al.'s deterministic parallel MIS -- the result
// is identical to the sequential greedy order, not merely equivalent).  Neighbours are found through a bucket grid
// (cell size >= radius: 3x3 cells).  The accepted set is then ranked by counting (score order) and cut at max_kp.
// One CTA of 1024 threads per image; all scratch lives in global memory.
constexpr int UT = 1024;
constexpr int UNI_SN = 6144, UNI_SC = UNI_SN / 2;      // candidates / cells the shared-memory kernel holds
__host__ __device__ inline bool uni_fits_smem(int n, int n_cells) { return n <= UNI_SN && n_cells <= UNI_SC; }
struct UniScratch {
  uint32_t* cell_start;   // [n_cells + 1]
  uint32_t* cell_cur;     // [n_cells]
  uint32_t* order;        // [cap] candidate indices grouped by cell
  uint8_t* state;         // [cap] 0 alive, 1 pending, 2 accepted, 3 dead
  uint32_t* acc;          // [cap] accepted candidates
  uint32_t *blocker, *list0, *list1, *pend;   // [cap] each: rounds scratch
  int max_cells;
};
__device__ __forceinline__ int uni_block_scan(int v, int* s_warp, int* total) {     // exclusive scan over the CTA
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
__global__ void __launch_bounds__(UT) k_uniformity(const unsigned long long* __restrict__ keys, const int* __restrict__ count, int cap,
                                                   int W, int H, double radius, int max_kp, UniScratch sc, okb_keypoint* kps, int* n_out) {
  __shared__ int s_warp[32];
  __shared__ int s_n;
  const int tid = threadIdx.x;
  const int n = min(*count, cap);
  const int cs = max(4, (int)ceil(radius));
  const int gw = (W + cs - 1) / cs, gh = (H + cs - 1) / cs, n_cells = gw * gh;
  if (uni_fits_smem(n, n_cells)) return;       // k_uniformity_smem (launched next) does this image
  const long long r2i = (long long)ceil(radius * radius - 1e-9);     // integer test: dx^2 + dy^2 < radius^2
  auto px = [&](int i, int& x, int& y) { const uint32_t idx = 0xFFFFFFFFu - (uint32_t)(keys[i] & 0xFFFFFFFFull); x = (int)(idx % (uint32_t)W); y = (int)(idx / (uint32_t)W); };
  // ---- bucket grid (counting sort by cell)
  for (int c = tid; c < n_cells; c += UT) sc.cell_cur[c] = 0u;
  __syncthreads();
  for (int i = tid; i < n; i += UT) { int x, y; px(i, x, y); atomicAdd(&sc.cell_cur[(y / cs) * gw + x / cs], 1u); sc.state[i] = 0; }
  __syncthreads();
  int run = 0;
  for (int base = 0; base < n_cells; base += UT) {
    const int c = base + tid;
    const int v = (c < n_cells) ? (int)sc.cell_cur[c] : 0;
    int total;
    const int ex = uni_block_scan(v, s_warp, &total);
    if (c < n_cells) sc.cell_start[c] = (uint32_t)(run + ex);
    run += total;
    __syncthreads();
  }
  if (tid == 0) sc.cell_start[n_cells] = (uint32_t)run;
  for (int c = tid; c < n_cells; c += UT) sc.cell_cur[c] = sc.cell_start[c];
  __syncthreads();
  for (int i = tid; i < n; i += UT) { int x, y; px(i, x, y); const uint32_t pos = atomicAdd(&sc.cell_cur[(y / cs) * gw + x / cs], 1u); sc.order[pos] = (uint32_t)i; }
  __syncthreads();
  // ---- rounds over a shrinking list of live candidates (lists A / B alternate; appended with a shared-memory
  // counter: the ORDER inside a list is arbitrary, the SET is not, and only the set matters).  blocker[i] remembers the
  // live higher-priority neighbour that blocked i: while it lives, i stays blocked without another neighbourhood scan.
  uint32_t* blocker = sc.blocker;
  uint32_t* listA = sc.list0;
  uint32_t* listB = sc.list1;
  uint32_t* pend = sc.pend;
  __shared__ int s_alive, s_pend;
  for (int i = tid; i < n; i += UT) listA[i] = (uint32_t)i;
  int alive = n, rounds = 0;
  bool first_round = true;
  __syncthreads();
  while (alive > 0) {
    ++rounds;
    if (tid == 0) { s_alive = 0; s_pend = 0; }
    __syncthreads();
    // accept: no live (alive or pending) neighbour with a larger key
    for (int t = tid; t < alive; t += UT) {
      const int i = (int)listA[t];
      if (!first_round && sc.state[blocker[i]] <= 1) continue;
      int x, y; px(i, x, y);
      const unsigned long long ki = keys[i];
      bool blocked = false;
      const int cx = x / cs, cy = y / cs;
      for (int yy = max(cy - 1, 0); yy <= min(cy + 1, gh - 1) && !blocked; ++yy)
        for (int xx = max(cx - 1, 0); xx <= min(cx + 1, gw - 1) && !blocked; ++xx) {
          const uint32_t e = sc.cell_start[yy * gw + xx + 1];
          for (uint32_t q = sc.cell_start[yy * gw + xx]; q < e; ++q) {
            const int j = (int)sc.order[q];
            if (keys[j] <= ki || sc.state[j] > 1) continue;
            int xj, yj; px(j, xj, yj);
            const long long dx = xj - x, dy = yj - y;
            if (dx * dx + dy * dy < r2i) { blocked = true; blocker[i] = (uint32_t)j; break; }
          }
        }
      if (!blocked) { sc.state[i] = 1; pend[atomicAdd(&s_pend, 1)] = (uint32_t)i; }
    }
    __syncthreads();
    // kill: every pending candidate marks its live neighbours dead (two pending candidates are never neighbours);
    // a warp per pending candidate, lanes over the candidates of the 3x3 cells
    const int n_pend = s_pend;
    for (int t = tid >> 5; t < n_pend; t += UT / 32) {
      const int i = (int)pend[t];
      int x, y; px(i, x, y);
      const int cx = x / cs, cy = y / cs;
      for (int yy = max(cy - 1, 0); yy <= min(cy + 1, gh - 1); ++yy)
        for (int xx = max(cx - 1, 0); xx <= min(cx + 1, gw - 1); ++xx) {
          const uint32_t e = sc.cell_start[yy * gw + xx + 1];
          for (uint32_t q = sc.cell_start[yy * gw + xx] + (tid & 31); q < e; q += 32) {
            const int j = (int)sc.order[q];
            if (sc.state[j] != 0) continue;
            int xj, yj; px(j, xj, yj);
            const long long dx = xj - x, dy = yj - y;
            if (dx * dx + dy * dy < r2i) sc.state[j] = 3;
          }
        }
    }
    __syncthreads();
    for (int t = tid; t < alive; t += UT) {
      const int i = (int)listA[t];
      const uint8_t st = sc.state[i];
      if (st == 1) sc.state[i] = 2;
      else if (st == 0) listB[atomicAdd(&s_alive, 1)] = (uint32_t)i;
    }
    __syncthreads();
    alive = s_alive;
    uint32_t* tl = listA; listA = listB; listB = tl;
    first_round = false;
    __syncthreads();
  }
  // ---- accepted set -> score order, first max_kp
  if (tid == 0) s_n = 0;
  __syncthreads();
  for (int i = tid; i < n; i += UT) if (sc.state[i] == 2) sc.acc[atomicAdd(&s_n, 1)] = (uint32_t)i;
  __syncthreads();
  const int m = s_n;
  for (int a = tid; a < m; a += UT) {
    const unsigned long long ka = keys[sc.acc[a]];
    int rank = 0;
    for (int b = 0; b < m; ++b) rank += keys[sc.acc[b]] > ka;
    if (rank < max_kp) {
      int x, y; px((int)sc.acc[a], x, y);
      okb_keypoint kp;
      kp.x = (float)x; kp.y = (float)y; kp.size = 12.0f; kp.angle = 0.0f;
      kp.response = (float)(int32_t)(uint32_t)(ka >> 32); kp.octave = 0;
      kps[rank] = kp;
    }
  }
  if (tid == 0) { *n_out = min(m, max_kp); n_out[1] = rounds; }
}

// The same algorithm with every hot array in shared memory (the common case: a few thousand NMS candidates, a few
// thousand cells): one CTA walks dependent chains of loads, so the latency of each load is what the kernel costs.
// The candidates are re-indexed by their position q in the bucket grid and kept as 16-byte records {key, x, y} in
// that order: visiting a neighbour is ONE 16-byte load plus the independent state byte (the global-memory kernel
// chases order -> key -> state -> xy).  The scan starts with the candidate's own cell (where a blocker is most likely),
// suppression runs one thread per (accepted candidate, neighbouring cell), and the final ranking walks the accepted
// records with loads that do not depend on each other.
// Images with more candidates / cells than fit take the global-memory kernel above (both are launched, one returns).
struct __align__(16) UniRec { unsigned long long key; unsigned short x, y; unsigned int pad; };
struct UniSmem {
  UniRec rec[UNI_SN];
  unsigned short blocker[UNI_SN], listA[UNI_SN], listB[UNI_SN], pend[UNI_SN];
  unsigned short cell_start[UNI_SC + 1];
  unsigned int killed[UNI_SN / 32];     // suppressed this round (atomicOr: several accepted neighbours may hit the same candidate)
  unsigned char state[UNI_SN];          // 0 candidate, 2 accepted, 3 suppressed; only written between the phases
};
#ifdef OKB_UNI_PROF
__device__ unsigned long long g_uni_prof[8];     // cycles of thread 0 per phase (diagnostics build)
#define UNI_MARK(i) do { if (tid == 0) { const unsigned long long n_ = clock64(); g_uni_prof[i] += n_ - t_up; t_up = n_; } } while (0)
#else
#define UNI_MARK(i) do { } while (0)
#endif
__global__ void __launch_bounds__(UT) k_uniformity_smem(const unsigned long long* __restrict__ keys, const int* __restrict__ count, int cap,
                                                        int W, int H, double radius, int max_kp, okb_keypoint* kps, int* n_out) {
  extern __shared__ __align__(16) unsigned char uni_raw[];
  UniSmem& S = *reinterpret_cast<UniSmem*>(uni_raw);
  __shared__ int s_warp[32];
  __shared__ int s_n, s_alive, s_pend;
  const int tid = threadIdx.x;
  const int n = min(*count, cap);
  const int cs = max(4, (int)ceil(radius));
  const int gw = (W + cs - 1) / cs, gh = (H + cs - 1) / cs, n_cells = gw * gh;
  if (!uni_fits_smem(n, n_cells)) return;
  const int r2i = (int)ceil(radius * radius - 1e-9);
#ifdef OKB_UNI_PROF
  unsigned long long t_up = clock64();
  if (tid < 8) g_uni_prof[tid] = 0;
#endif
  // bucket grid: 32-bit counters alias the (still unused) second live list -- UNI_SC cells fit its 2 * UNI_SN bytes
  unsigned int* cnt32 = reinterpret_cast<unsigned int*>(S.listB);
  for (int c = tid; c < n_cells; c += UT) cnt32[c] = 0u;
  for (int i = tid; i < UNI_SN / 32; i += UT) S.killed[i] = 0u;
  for (int i = tid; i < n; i += UT) { S.state[i] = 0; S.listA[i] = (unsigned short)i; }
  __syncthreads();
  for (int i = tid; i < n; i += UT) {
    const uint32_t idx = 0xFFFFFFFFu - (uint32_t)(keys[i] & 0xFFFFFFFFull);
    atomicAdd(&cnt32[((idx / (uint32_t)W) / cs) * gw + (idx % (uint32_t)W) / cs], 1u);
  }
  __syncthreads();
  UNI_MARK(0);
  {
    int run = 0;
    for (int base = 0; base < n_cells; base += UT) {
      const int c = base + tid;
      const int v = (c < n_cells) ? (int)cnt32[c] : 0;
      int total;
      const int ex = uni_block_scan(v, s_warp, &total);
      if (c < n_cells) S.cell_start[c] = (unsigned short)(run + ex);
      run += total;
      __syncthreads();
    }
    if (tid == 0) S.cell_start[n_cells] = (unsigned short)run;
    __syncthreads();
    for (int c = tid; c < n_cells; c += UT) cnt32[c] = S.cell_start[c];
    __syncthreads();
    for (int i = tid; i < n; i += UT) {       // the order inside a cell is whatever the atomics give; the result does not depend on it
      const unsigned long long k = keys[i];
      const uint32_t idx = 0xFFFFFFFFu - (uint32_t)(k & 0xFFFFFFFFull);
      const uint32_t x = idx % (uint32_t)W, y = idx / (uint32_t)W;
      const unsigned int pos = atomicAdd(&cnt32[(y / cs) * gw + x / cs], 1u);
      UniRec r; r.key = k; r.x = (unsigned short)x; r.y = (unsigned short)y; r.pad = 0u;
      S.rec[pos] = r;
    }
    __syncthreads();
  }
  UNI_MARK(1);
  int alive = n, rounds = 0;
  bool first_round = true;
  unsigned short* listA = S.listA;
  unsigned short* listB = S.listB;
  while (alive > 0) {
    ++rounds;
    if (tid == 0) { s_alive = 0; s_pend = 0; }
    __syncthreads();
    // accept: a candidate with no undecided neighbour of higher priority (accepted neighbours cannot exist: their
    // neighbourhood was suppressed in the round that accepted them)
    for (int t = tid; t < alive; t += UT) {
      const int i = listA[t];
      if (!first_round && S.state[S.blocker[i]] == 0) continue;      // the candidate that blocked it is still undecided
      const UniRec me = S.rec[i];
      const int x = me.x, y = me.y;
      const int cx = x / cs, cy = y / cs;
      bool blocked = false;
#pragma unroll 1
      for (int k = 0; k < 9 && !blocked; ++k) {          // own cell first
        const int kk = (k == 0) ? 4 : (k <= 4 ? k - 1 : k);
        const int yy = cy + kk / 3 - 1, xx = cx + kk % 3 - 1;
        if (yy < 0 || yy >= gh || xx < 0 || xx >= gw) continue;
        const int e = S.cell_start[yy * gw + xx + 1];
        for (int q = S.cell_start[yy * gw + xx]; q < e; ++q) {
          const UniRec o = S.rec[q];
          if (o.key <= me.key || S.state[q] != 0) continue;
          const int dx = (int)o.x - x, dy = (int)o.y - y;
          if (dx * dx + dy * dy < r2i) { blocked = true; S.blocker[i] = (unsigned short)q; break; }
        }
      }
      if (!blocked) S.pend[atomicAdd(&s_pend, 1)] = (unsigned short)i;       // two candidates accepted in one round are never neighbours
    }
    __syncthreads();
    UNI_MARK(2);
    // suppress: one thread per (accepted candidate, neighbouring cell)
    const int n_pend = s_pend;
    for (int t = tid; t < n_pend * 9; t += UT) {
      const int i = S.pend[t / 9], kk = t % 9;
      const UniRec me = S.rec[i];
      const int yy = (int)me.y / cs + kk / 3 - 1, xx = (int)me.x / cs + kk % 3 - 1;
      if (yy < 0 || yy >= gh || xx < 0 || xx >= gw) continue;
      const int e = S.cell_start[yy * gw + xx + 1];
      for (int q = S.cell_start[yy * gw + xx]; q < e; ++q) {
        if (S.state[q] != 0 || q == i) continue;
        const UniRec o = S.rec[q];
        const int dx = (int)o.x - (int)me.x, dy = (int)o.y - (int)me.y;
        if (dx * dx + dy * dy < r2i) atomicOr(&S.killed[q >> 5], 1u << (q & 31));
      }
    }
    __syncthreads();
    UNI_MARK(3);
    for (int t = tid; t < n_pend; t += UT) S.state[S.pend[t]] = 2;
    __syncthreads();
    for (int t = tid; t < alive; t += UT) {
      const int i = listA[t];
      if (S.state[i] != 0) continue;
      if ((S.killed[i >> 5] >> (i & 31)) & 1u) S.state[i] = 3;
      else listB[atomicAdd(&s_alive, 1)] = (unsigned short)i;
    }
    __syncthreads();
    alive = s_alive;
    unsigned short* tl = listA; listA = listB; listB = tl;
    first_round = false;
    __syncthreads();
    UNI_MARK(4);
  }
  if (tid == 0) s_n = 0;
  __syncthreads();
  unsigned short* acc = S.pend;
  for (int i = tid; i < n; i += UT) if (S.state[i] == 2) acc[atomicAdd(&s_n, 1)] = (unsigned short)i;
  __syncthreads();
  UNI_MARK(5);
  const int m = s_n;
  // ranking by key (descending) = the order the greedy walk would have accepted them in.  The accepted keys are first
  // packed into the dead live lists (blocker | listA | listB are contiguous: 3 * UNI_SN u16 = room for 3 * UNI_SN / 4
  // keys) so that the m^2 comparisons read two keys per 16-byte load, nothing dependent; more accepted candidates
  // than fit there take the indirect loop.
  unsigned long long* ck = reinterpret_cast<unsigned long long*>(S.blocker);
  const bool packed = m <= 3 * UNI_SN / 4 - 1;
  if (packed) {
    for (int a = tid; a < m; a += UT) ck[a] = S.rec[acc[a]].key;
    if (tid == 0) ck[m] = 0ull;                         // pad to an even count (key 0 is below every real key)
  }
  __syncthreads();
  for (int a = tid; a < m; a += UT) {
    const UniRec me = S.rec[acc[a]];
    int rank = 0;
    if (packed) {
      const ulonglong2* ck2 = reinterpret_cast<const ulonglong2*>(ck);
#pragma unroll 4
      for (int b = 0; b < (m + 1) / 2; ++b) { const ulonglong2 k2 = ck2[b]; rank += (k2.x > me.key) + (k2.y > me.key); }
    } else {
      for (int b = 0; b < m; ++b) rank += S.rec[acc[b]].key > me.key;
    }
    if (rank < max_kp) {
      okb_keypoint kp;
      kp.x = (float)me.x; kp.y = (float)me.y; kp.size = 12.0f; kp.angle = 0.0f;
      kp.response = (float)(int32_t)(uint32_t)(me.key >> 32); kp.octave = 0;
      kps[rank] = kp;
    }
  }
  UNI_MARK(6);
  if (tid == 0) { *n_out = min(m, max_kp); n_out[1] = rounds; }
}

// integral image (H+1) x (W+1), uint32
// row pass: one warp per image row, 32 pixels per step (warp inclusive scan + running carry): coalesced byte loads
// and 128-byte stores
__global__ void __launch_bounds__(128) k_integral_rows(const uint8_t* __restrict__ img, int W, int H, uint32_t* II) {
  const int y = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (y > H) return;
  uint32_t* row = II + (size_t)y * (W + 1);
  if (y == 0) { for (int x = lane; x <= W; x += 32) row[x] = 0; return; }
  if (lane == 0) row[0] = 0;
  const uint8_t* src = img + (size_t)(y - 1) * W;
  uint32_t carry = 0;
  for (int x0 = 0; x0 < W; x0 += 32) {
    const int x = x0 + lane;
    uint32_t v = (x < W) ? src[x] : 0u;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += t;
    }
    if (x < W) row[x + 1] = carry + v;
    carry += __shfl_sync(0xffffffffu, v, 31);
  }
}
// column pass: a CTA owns 32 columns; its 16 warps split the rows into 16 segments (lanes = columns: every access is a
// 128-byte row).  Pass 1 sums each segment, the segment offsets are combined through shared memory, pass 2 writes the
// running sums.  Integer arithmetic: any summation order gives the same bits.
constexpr int IC_SEG = 16;
__global__ void __launch_bounds__(32 * IC_SEG) k_integral_cols(int W, int H, uint32_t* II) {
  __shared__ uint32_t seg[IC_SEG][33];
  const int lane = threadIdx.x & 31, s_ = threadIdx.x >> 5;
  const int x = blockIdx.x * 32 + lane;
  const int rows = H + 1, per = (rows + IC_SEG - 1) / IC_SEG;
  const int y0 = s_ * per, y1 = min(rows, y0 + per);
  uint32_t sum = 0;
  if (x <= W)
    for (int y = y0; y < y1; ++y) sum += II[(size_t)y * (W + 1) + x];
  seg[s_][lane] = sum;
  __syncthreads();
  uint32_t run = 0;
  for (int k = 0; k < s_; ++k) run += seg[k][lane];
  if (x <= W)
    for (int y = y0; y < y1; ++y) {
      run += II[(size_t)y * (W + 1) + x];
      II[(size_t)y * (W + 1) + x] = run;
    }
}

__device__ void undistort_gn(const CamIntr& cam, double d0, double d1, double* pu) {
  double x0 = d0, x1 = d1;
  for (int i = 0; i < 5; ++i) {
    double xt[2], E[4];
    distort<true>(cam, x0, x1, xt, E);
    const double e0 = d0 - xt[0], e1 = d1 - xt[1];
    const double a = E[0] * E[0] + E[2] * E[2], b = E[0] * E[1] + E[2] * E[3], d = E[1] * E[1] + E[3] * E[3];
    const double r0 = E[0] * e0 + E[2] * e1, r1 = E[1] * e0 + E[3] * e1;
    const double det = a * d - b * b;
    x0 += (d * r0 - b * r1) / det;
    x1 += (-b * r0 + a * r1) / det;
    if (e0 * e0 + e1 * e1 < 1e-15) break;
  }
  pu[0] = x0; pu[1] = x1;
}

// warp per keypoint: gravity angle, 60 box-smoothed samples, 8*desc_bytes comparisons via ballot
__global__ void __launch_bounds__(128) k_describe(const uint32_t* __restrict__ II, int W, int H, okb_camera camera, const double* gC,
                                                  int rot_inv, const int* __restrict__ half, const uint8_t* __restrict__ pi,
                                                  const uint8_t* __restrict__ pj, const int16_t* __restrict__ lut, int desc_bytes,
                                                  okb_keypoint* kps, const int* n_kp, uint8_t* desc) {
  __shared__ uint32_t sS[4][64], sA[4][64];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int k = blockIdx.x * 4 + wib;
  if (k >= *n_kp) return;
  const int x = (int)kps[k].x, y = (int)kps[k].y;
  float ang = 0.0f;
  if (rot_inv) {
    if (lane == 0) {
      CamIntr cam;
      cam_load(camera, cam);
      double pu[2];
      undistort_gn(cam, ((double)x - cam.cu) / cam.fu, ((double)y - cam.cv) / cam.fv, pu);
      const double ep[3] = {pu[0], pu[1], 1.0};
      double ip[2], J[6];
      project<true>(cam, ep, ip, J);
      const double e0 = J[0] * gC[0] + J[1] * gC[1] + J[2] * gC[2];
      const double e1 = J[3] * gC[0] + J[4] * gC[1] + J[5] * gC[2];
      ang = (float)(atan2(e1, e0) / 3.14159265358979323846 * 180.0);
      kps[k].angle = ang;
    }
    ang = __shfl_sync(0xffffffffu, ang, 0);
  }
  const int bin = ((int)lround((double)ang / 360.0 * kRotBins)) & (kRotBins - 1);
  for (int p = lane; p < kPts; p += 32) {
    const int cx = x + lut[((size_t)bin * kPts + p) * 2], cy = y + lut[((size_t)bin * kPts + p) * 2 + 1];
    const int h = half[p];
    const int x0 = max(cx - h, 0), x1 = min(cx + h, W - 1), y0 = max(cy - h, 0), y1 = min(cy + h, H - 1);
    sS[wib][p] = II[(size_t)(y1 + 1) * (W + 1) + x1 + 1] - II[(size_t)y0 * (W + 1) + x1 + 1] - II[(size_t)(y1 + 1) * (W + 1) + x0] +
                 II[(size_t)y0 * (W + 1) + x0];
    sA[wib][p] = (uint32_t)((x1 - x0 + 1) * (y1 - y0 + 1));
  }
  __syncwarp();
  uint32_t* out = reinterpret_cast<uint32_t*>(desc + (size_t)k * desc_bytes);
  for (int w = 0; w < desc_bytes / 4; ++w) {
    const int b = 32 * w + lane;
    const int i = pi[b], j = pj[b];
    const bool bit = (unsigned long long)sS[wib][i] * sA[wib][j] > (unsigned long long)sS[wib][j] * sA[wib][i];
    const uint32_t word = __ballot_sync(0xffffffffu, bit);
    if (lane == 0) out[w] = word;
  }
}
}  // namespace

static int ensure_pattern(okb_ctx* c, okb_frontend_state* F, int desc_bytes) {
  std::lock_guard<std::mutex> lk(F->pat_mtx);
  if (F->pat_bytes == desc_bytes) return OKB_OK;
  Pattern P = make_pattern(desc_bytes);
  cudaFree(F->d_half); cudaFree(F->d_pi); cudaFree(F->d_pj); cudaFree(F->d_lut);
  FE_CUDA(c, cudaMalloc(&F->d_half, sizeof(int) * kPts));
  FE_CUDA(c, cudaMalloc(&F->d_pi, P.pi.size()));
  FE_CUDA(c, cudaMalloc(&F->d_pj, P.pj.size()));
  FE_CUDA(c, cudaMalloc(&F->d_lut, P.lut.size() * sizeof(int16_t)));
  FE_CUDA(c, cudaMemcpy(F->d_half, P.half, sizeof(int) * kPts, cudaMemcpyHostToDevice));
  FE_CUDA(c, cudaMemcpy(F->d_pi, P.pi.data(), P.pi.size(), cudaMemcpyHostToDevice));
  FE_CUDA(c, cudaMemcpy(F->d_pj, P.pj.data(), P.pj.size(), cudaMemcpyHostToDevice));
  FE_CUDA(c, cudaMemcpy(F->d_lut, P.lut.data(), P.lut.size() * sizeof(int16_t), cudaMemcpyHostToDevice));
  F->pat_bytes = desc_bytes;
  return OKB_OK;
}

extern "C" int okb_detect_describe(okb_ctx* c, int cam_slot, const uint8_t* img, int width, int height, int stride,
                                   const okb_camera* cam, const double R_CW[9], const okb_detect_params* prm,
                                   okb_keypoint* out_kp, uint8_t* out_desc, int max_out, int* n_out) {
  if (!c || !img || !cam || !R_CW || !prm || !out_kp || !out_desc || !n_out) return OKB_ERR_INVALID_ARG;
  if (cam_slot < 0 || cam_slot >= kMaxSlots || width < 64 || height < 64 || stride < width) return OKB_ERR_INVALID_ARG;
  if (prm->desc_bytes < 4 || prm->desc_bytes > 128 || (prm->desc_bytes % 4) != 0) return OKB_ERR_INVALID_ARG;
  cudaSetDevice(c->device);
  okb_frontend_state* F = fe(c);
  int rc = ensure_pattern(c, F, prm->desc_bytes);
  if (rc) return rc;
  SlotBuffers& S = F->slots[cam_slot];
  std::lock_guard<std::mutex> lk(S.mtx);   // the reference guards each camera's detector with a mutex (Frontend.cpp:97)
  const int W = width, H = height;
  const int maxk = std::min(prm->max_keypoints, max_out);
  if (maxk < 1) return OKB_ERR_INVALID_ARG;
  if (!S.stream) FE_CUDA(c, cudaStreamCreateWithFlags(&S.stream, cudaStreamNonBlocking));
  if (S.W != W || S.H != H) {
    cudaFree(S.d_img); cudaFree(S.d_score); cudaFree(S.d_integral); cudaFree(S.d_keys); cudaFree(S.d_count);
    cudaFree(S.d_cell_start); cudaFree(S.d_cell_cur); cudaFree(S.d_order); cudaFree(S.d_acc); cudaFree(S.d_state); cudaFree(S.d_rounds);
    if (S.h_img) cudaFreeHost(S.h_img);
    if (S.h_count) cudaFreeHost(S.h_count);
    FE_CUDA(c, cudaMalloc(&S.d_img, (size_t)W * H));
    FE_CUDA(c, cudaMalloc(&S.d_score, sizeof(int32_t) * W * H));
    FE_CUDA(c, cudaMalloc(&S.d_integral, sizeof(uint32_t) * (W + 1) * (H + 1)));
    FE_CUDA(c, cudaMalloc(&S.d_keys, sizeof(unsigned long long) * kMaxCand));
    FE_CUDA(c, cudaMalloc(&S.d_count, sizeof(int) * 4 + sizeof(double) * 4));      // candidates, accepted, rounds, - | gravity direction
    S.max_cells = ((W + 3) / 4) * ((H + 3) / 4);          // smallest cell is 4 px
    FE_CUDA(c, cudaMalloc(&S.d_cell_start, sizeof(uint32_t) * (S.max_cells + 1)));
    FE_CUDA(c, cudaMalloc(&S.d_cell_cur, sizeof(uint32_t) * S.max_cells));
    FE_CUDA(c, cudaMalloc(&S.d_order, sizeof(uint32_t) * kMaxCand));
    FE_CUDA(c, cudaMalloc(&S.d_acc, sizeof(uint32_t) * kMaxCand));
    FE_CUDA(c, cudaMalloc(&S.d_state, kMaxCand));
    FE_CUDA(c, cudaMalloc(&S.d_rounds, sizeof(uint32_t) * 4 * kMaxCand));
    FE_CUDA(c, cudaMallocHost(&S.h_img, (size_t)W * H));
    FE_CUDA(c, cudaMallocHost(&S.h_count, sizeof(int) * 4));
    S.W = W; S.H = H;
  }
  if (S.kp_cap < maxk || S.desc_cap < maxk * prm->desc_bytes) {
    cudaFree(S.d_kp); cudaFree(S.d_desc);
    if (S.h_kp) cudaFreeHost(S.h_kp);
    if (S.h_desc) cudaFreeHost(S.h_desc);
    FE_CUDA(c, cudaMalloc(&S.d_kp, sizeof(okb_keypoint) * maxk));
    FE_CUDA(c, cudaMalloc(&S.d_desc, (size_t)maxk * prm->desc_bytes));
    FE_CUDA(c, cudaMallocHost(&S.h_kp, sizeof(okb_keypoint) * maxk));
    FE_CUDA(c, cudaMallocHost(&S.h_desc, (size_t)maxk * prm->desc_bytes));
    S.kp_cap = maxk; S.desc_cap = maxk * prm->desc_bytes;
  }
  for (int y = 0; y < H; ++y) std::memcpy(S.h_img + (size_t)y * W, img + (size_t)y * stride, W);
  cudaStream_t st = S.stream;
  FE_CUDA(c, cudaMemcpyAsync(S.d_img, S.h_img, (size_t)W * H, cudaMemcpyHostToDevice, st));
  FE_CUDA(c, cudaMemsetAsync(S.d_count, 0, sizeof(int) * 4, st));
  // gravity direction in the camera frame: R_CW * (0,0,-1)
  double gC[3] = {-R_CW[2], -R_CW[5], -R_CW[8]};
  double* d_gC = reinterpret_cast<double*>(S.d_count + 4);
  FE_CUDA(c, cudaMemcpyAsync(d_gC, gC, sizeof gC, cudaMemcpyHostToDevice, st));
  const dim3 hb(HT_X, HT_Y), hg((W + HT_X - 1) / HT_X, (H + HT_Y - 1) / HT_Y);
  k_harris<<<hg, hb, 0, st>>>(S.d_img, W, H, S.d_score);
  const dim3 nb(32, 8), ng((W + 31) / 32, (H + 7) / 8);
  k_nms<<<ng, nb, 0, st>>>(S.d_score, W, H, (int32_t)std::ceil(prm->absolute_threshold), S.d_keys, S.d_count, kMaxCand);
  UniScratch us{S.d_cell_start, S.d_cell_cur, S.d_order, S.d_state, S.d_acc, S.d_rounds, S.d_rounds + kMaxCand, S.d_rounds + 2 * kMaxCand,
                S.d_rounds + 3 * kMaxCand, S.max_cells};
  k_uniformity<<<1, UT, 0, st>>>(S.d_keys, S.d_count, kMaxCand, W, H, prm->uniformity_radius, maxk, us, S.d_kp, S.d_count + 1);
  {
    FE_CUDA(c, cudaFuncSetAttribute(k_uniformity_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(UniSmem)));
    k_uniformity_smem<<<1, UT, sizeof(UniSmem), st>>>(S.d_keys, S.d_count, kMaxCand, W, H, prm->uniformity_radius, maxk, S.d_kp, S.d_count + 1);
  }
  k_integral_rows<<<(H + 1 + 3) / 4, 128, 0, st>>>(S.d_img, W, H, S.d_integral);
  k_integral_cols<<<(W + 1 + 31) / 32, 32 * IC_SEG, 0, st>>>(W, H, S.d_integral);
  k_describe<<<(maxk + 3) / 4, 128, 0, st>>>(S.d_integral, W, H, *cam, d_gC, prm->rotation_invariance, F->d_half, F->d_pi, F->d_pj,
                                             F->d_lut, prm->desc_bytes, S.d_kp, S.d_count + 1, S.d_desc);
  c->launches += 7;
  FE_CUDA(c, cudaGetLastError());
  FE_CUDA(c, cudaMemcpyAsync(S.h_count, S.d_count, sizeof(int) * 4, cudaMemcpyDeviceToHost, st));
  FE_CUDA(c, cudaMemcpyAsync(S.h_kp, S.d_kp, sizeof(okb_keypoint) * maxk, cudaMemcpyDeviceToHost, st));
  FE_CUDA(c, cudaMemcpyAsync(S.h_desc, S.d_desc, (size_t)maxk * prm->desc_bytes, cudaMemcpyDeviceToHost, st));
  FE_CUDA(c, cudaStreamSynchronize(st));
  { static const bool dbg = getenv("OKB_FE_DEBUG") != nullptr; if (dbg) fprintf(stderr, "[okb frontend] candidates %d accepted %d uniformity rounds %d\n", S.h_count[0], S.h_count[1], S.h_count[2]);
#ifdef OKB_UNI_PROF
    if (dbg) { unsigned long long pr[8]; cudaMemcpyFromSymbol(pr, g_uni_prof, sizeof(pr)); fprintf(stderr, "[okb frontend] uniformity cycles: load %llu grid %llu accept %llu kill %llu rebuild %llu compact %llu rank %llu\n", pr[0], pr[1], pr[2], pr[3], pr[4], pr[5], pr[6]); }
#endif
  }
  if (S.h_count[0] > kMaxCand) { c->set_error("too many corner candidates"); return OKB_ERR_CAPACITY; }
  const int n = S.h_count[1];
  std::memcpy(out_kp, S.h_kp, sizeof(okb_keypoint) * n);
  std::memcpy(out_desc, S.h_desc, (size_t)n * prm->desc_bytes);
  *n_out = n;
  return OKB_OK;
}

// =================================================================================================
// matcher kernels
// =================================================================================================
// =================================================================================================
// geometric match gate (VioKeyframeWindowMatchingAlgorithm::verifyMatch, SURVEY 8f row 2) -- evaluated per
// (A, B) pair inside the list kernel for pairs whose Hamming distance is below the threshold
// =================================================================================================
namespace {
struct GateDev {
  int mode;
  const double *kp_b, *kp_size_b, *proj_into_b, *proj_unc, *kp_a, *kp_size_a, *bearing_a, *bearing_b, *ray_sigma_a, *ray_sigma_b;
  CamIntr cam_a, cam_b;
  int wa, ha, wb, hb;
  double R_AB[9], t_AB[3];
};

// PinholeCamera::projectHomogeneous(...) == Successful (PinholeCamera.hpp(impl):147-226, 345-378; CameraBase::isInImage)
__device__ __forceinline__ bool gate_project(const CamIntr& cam, int W, int H, const double* hp, double* y) {
  double head[3] = {hp[0], hp[1], hp[2]};
  if (hp[3] < 0) { head[0] = -head[0]; head[1] = -head[1]; head[2] = -head[2]; }
  double J[6];
  if (!project<false>(cam, head, y, J)) return false;
  if (y[0] < 0.0 || y[1] < 0.0 || y[0] >= (double)W || y[1] >= (double)H) return false;
  return head[2] > 0.0;
}
// ProbabilisticStereoTriangulator::computeReprojectionError4 (ProbabilisticStereoTriangulator.cpp:359-384)
__device__ __forceinline__ bool gate_reproj_err(const CamIntr& cam, int W, int H, const double* kp, double size, const double* hp, double& err) {
  double y[2];
  if (!gate_project(cam, W, H, hp, y)) return false;
  const double sd = 0.8 * size / 12.0;
  const double w = 1.0 / (sd * sd);
  const double d0 = y[0] - kp[0], d1 = y[1] - kp[1];
  err = d0 * (w * d0) + d1 * (w * d1);
  return true;
}
__device__ bool gate_verify(const GateDev& g, int a, int b) {
  if (g.mode == OKB_GATE_2D2D) {
    // stereoTriangulate (ProbabilisticStereoTriangulator.cpp:168-227) -> triangulateFast (stereo_triangulation.cpp:51-125)
    const double* ba = g.bearing_a + 3 * a;
    const double* bb = g.bearing_b + 3 * b;
    double e1[3], e2[3], eb[3];
    const double na = sqrt(ba[0] * ba[0] + ba[1] * ba[1] + ba[2] * ba[2]);
    e1[0] = ba[0] / na; e1[1] = ba[1] / na; e1[2] = ba[2] / na;
    mat3vec(g.R_AB, bb, eb);
    const double nb = sqrt(eb[0] * eb[0] + eb[1] * eb[1] + eb[2] * eb[2]);
    e2[0] = eb[0] / nb; e2[1] = eb[1] / nb; e2[2] = eb[2] / nb;
    const double sigma = fmax(g.ray_sigma_a[a], g.ray_sigma_b[b]);
    const double* t12 = g.t_AB;                    // p1 = 0, p2 = t_AB
    const double b0 = t12[0] * e1[0] + t12[1] * e1[1] + t12[2] * e1[2];
    const double b1 = t12[0] * e2[0] + t12[1] * e2[1] + t12[2] * e2[2];
    const double A00 = e1[0] * e1[0] + e1[1] * e1[1] + e1[2] * e1[2];
    double A10 = e1[0] * e2[0] + e1[1] * e2[1] + e1[2] * e2[2], A01 = -A10;
    const double A11 = -(e2[0] * e2[0] + e2[1] * e2[1] + e2[2] * e2[2]);
    if (A10 < 0.0) { A10 = -A10; A01 = -A01; }
    const double det = A00 * A11 - A01 * A10;
    double hpA[4];
    if (!(fabs(det) > 1.0e-6)) {
      double c[3];
      cross3(e1, e2, c);
      if (!(sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]) < 6 * sigma)) return false;
      const double v[4] = {(e1[0] + e2[0]) / 2.0, (e1[1] + e2[1]) / 2.0, (e1[2] + e2[2]) / 2.0, 1e-3};
      const double n = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3]);
      hpA[0] = v[0] / n; hpA[1] = v[1] / n; hpA[2] = v[2] / n; hpA[3] = v[3] / n;
    } else {
      const double i00 = A11 / det, i01 = -A01 / det, i10 = -A10 / det, i11 = A00 / det;
      const double l0 = i00 * b0 + i01 * b1, l1 = i10 * b0 + i11 * b1;
      double mid[3], err[3], diff[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double xm = l0 * e1[k], xn = l1 * e2[k] + t12[k];
        mid[k] = (xm + xn) / 2.0;
        err[k] = mid[k] - xm;
        diff[k] = mid[k] - (0.5 * t12[k]);
      }
      const double diff_sq = diff[0] * diff[0] + diff[1] * diff[1] + diff[2] * diff[2];
      const double chi2 = (err[0] * err[0] + err[1] * err[1] + err[2] * err[2]) * (1.0 / (diff_sq * sigma * sigma));
      if (chi2 > 9) return false;
      if (diff[0] * e1[0] + diff[1] * e1[1] + diff[2] * e1[2] < 0)
        for (int k = 0; k < 3; ++k) mid[k] = (0.5 * t12[k]) - diff[k];
      const double n = sqrt(mid[0] * mid[0] + mid[1] * mid[1] + mid[2] * mid[2] + 1.0);
      hpA[0] = mid[0] / n; hpA[1] = mid[1] / n; hpA[2] = mid[2] / n; hpA[3] = 1.0 / n;
    }
    double errA, errB;
    if (!gate_reproj_err(g.cam_a, g.wa, g.ha, g.kp_a + 2 * a, g.kp_size_a[a], hpA, errA)) return false;
    double hpB[4];        // T_BA * hpA = [C_AB^T (x - t_AB w), w]
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double tk = -(g.R_AB[k] * g.t_AB[0] + g.R_AB[3 + k] * g.t_AB[1] + g.R_AB[6 + k] * g.t_AB[2]);
      hpB[k] = g.R_AB[k] * hpA[0] + g.R_AB[3 + k] * hpA[1] + g.R_AB[6 + k] * hpA[2] + tk * hpA[3];
    }
    hpB[3] = hpA[3];
    if (!gate_reproj_err(g.cam_b, g.wb, g.hb, g.kp_b + 2 * b, g.kp_size_b[b], hpB, errB)) return false;
    return !(errA > 4.0 || errB > 4.0);
  }
  // 3D-2D (VioKeyframeWindowMatchingAlgorithm.cpp:317-338)
  const double sd = 0.8 * g.kp_size_b[b] / 12.0;
  const double* P = g.proj_unc + 4 * a;
  const double U00 = sd * sd + P[0], U01 = P[1], U10 = P[2], U11 = sd * sd + P[3];
  const double det = U00 * U11 - U01 * U10;
  const double e0 = g.proj_into_b[2 * a] - g.kp_b[2 * b], e1 = g.proj_into_b[2 * a + 1] - g.kp_b[2 * b + 1];
  const double v0 = (U11 * e0 - U01 * e1) / det, v1 = (-U10 * e0 + U00 * e1) / det;
  const int chi2 = (int)(e0 * v0 + e1 * v1);      // the reference truncates to int before comparing with 4.0
  return chi2 < 4.0;
}
}  // namespace

namespace {
constexpr int MW = 8;            // warps per CTA = A rows per CTA (one warp per A descriptor)
constexpr int MT = 32 * MW;
constexpr int MB_TILE = 128;     // B descriptors staged per shared-memory tile
constexpr int MAX_BEST = 8;

// Warp per A descriptor.  Every lane computes the Hamming distance (XOR + __popc over NW words) of A to one of 32
// consecutive B descriptors, staged tile by tile in shared memory for the CTA's 8 warps; the top-`num_best` list of
// DenseMatcher::listBIteration (implementation/DenseMatcher.hpp:137-225) is kept replicated in the warp and updated
// with exactly the reference's sequential rule -- candidates are taken in ascending B order (lowest set bit of the
// ballot first), a candidate enters only if it beats the CURRENT worst entry (re-voted after every insertion, the
// worst only shrinks), std::lower_bound position, i.e. before entries of equal distance.
template <int NW, bool GATED>
__global__ void __launch_bounds__(MT) k_hamming_topk(const uint32_t* __restrict__ A, int nA, const uint32_t* __restrict__ B, int nB,
                                                     const uint8_t* __restrict__ skipA, const uint8_t* __restrict__ skipB, float list_thr,
                                                     int num_best, okb_pair* __restrict__ topk, float gate_thr, const GateDev* __restrict__ gate) {
  __shared__ uint32_t sB[MB_TILE][NW + 1];
  __shared__ uint8_t sSkip[MB_TILE];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int a = blockIdx.x * MW + warp;
  const bool active = a < nA && !(skipA && skipA[a]);
  uint32_t wa[NW];
#pragma unroll
  for (int w = 0; w < NW; ++w) wa[w] = (a < nA) ? A[(size_t)a * NW + w] : 0u;
  int bi[MAX_BEST];
  float bd[MAX_BEST];
#pragma unroll
  for (int k = 0; k < MAX_BEST; ++k) { bi[k] = -1; bd[k] = list_thr; }
  float worst = list_thr;
  for (int b0 = 0; b0 < nB; b0 += MB_TILE) {
    const int nb = min(MB_TILE, nB - b0);
    __syncthreads();
    for (int i = threadIdx.x; i < nb * NW; i += MT) sB[i / NW][i % NW] = B[(size_t)b0 * NW + i];
    for (int i = threadIdx.x; i < nb; i += MT) sSkip[i] = skipB ? skipB[b0 + i] : 0;
    __syncthreads();
    if (!active) continue;
    for (int j0 = 0; j0 < nb; j0 += 32) {
      const int j = j0 + lane;
      float t = 3.402823466e+38f;          // FLT_MAX: lanes without a B (tail, skipped) never beat any list entry
      if (j < nb && !sSkip[j]) {
        int dist = 0;
#pragma unroll
        for (int w = 0; w < NW; ++w) dist += __popc(wa[w] ^ sB[j][w]);
        t = (float)dist;
        // VioKeyframeWindowMatchingAlgorithm::distance: the Hamming distance counts only below the threshold and
        // if the geometric gate passes, else FLT_MAX (which never enters a list)
        if (GATED) t = (t < gate_thr && gate_verify(*gate, a, b0 + j)) ? t : 3.402823466e+38f;
      }
      uint32_t mask = __ballot_sync(0xffffffffu, t < worst);
      while (mask) {
        const int src = __ffs((int)mask) - 1;
        const float tt = __shfl_sync(0xffffffffu, t, src);
        // lower_bound on distance, shift the tail, insert before equal distances (replicated in every lane)
#pragma unroll
        for (int k = MAX_BEST - 1; k > 0; --k) {
          if (k < num_best && bd[k - 1] >= tt) { bd[k] = bd[k - 1]; bi[k] = bi[k - 1]; }
        }
        int pos = 0;
#pragma unroll
        for (int k = 0; k < MAX_BEST; ++k) if (k < num_best && bd[k] < tt) pos = k + 1;
#pragma unroll
        for (int k = 0; k < MAX_BEST; ++k) if (k == pos) { bd[k] = tt; bi[k] = b0 + j0 + src; }
        worst = bd[0];
#pragma unroll
        for (int k = 1; k < MAX_BEST; ++k) if (k == num_best - 1) worst = bd[k];
        // later lanes vote again against the new worst; earlier ones already failed against a larger one
        mask = __ballot_sync(0xffffffffu, t < worst) & ~((2u << src) - 1u);
      }
    }
  }
  if (a < nA && lane == 0) {
    for (int k = 0; k < num_best; ++k) {
      okb_pair p;
      p.index_a = active ? bi[k] : -1;
      p.distance = active ? bd[k] : list_thr;
      topk[(size_t)a * num_best + k] = p;
    }
  }
}

// Sequential greedy assignment, A ascending (assignbest, DenseMatcher.cpp:69-110; tail recursion unrolled).  The order
// dependence is the reference's semantics, so the walk itself stays serial (thread 0); what makes it fast is that
// nothing on its dependent chain touches global memory: the per-B winners live in shared memory and the top-k lists
// are staged 256 A's at a time by the whole CTA.  Displacement chains read the displaced A's list from shared memory
// when it is in the staged chunk, else from global memory (rare).
// Uncontested A's leave the walk before it starts: if A's first choice b is listed by no other A (count[b] == 1 over all
// list entries of all non-skipped A's), then b is free when A's turn comes, A takes it, nobody can displace A and A
// touches no other b -- its outcome is independent of the order.  Those are assigned in parallel; only A's whose first
// choice is contested walk serially (typically a small fraction).
constexpr int AS_T = 256, AS_CHUNK = 256;
__global__ void __launch_bounds__(AS_T) k_assign(const okb_pair* __restrict__ topk, int nA, int nB, int num_best, const uint8_t* __restrict__ skipA,
                                                 okb_pair* pairs, uint8_t* done /* [nA] scratch */, int in_smem) {
  extern __shared__ okb_pair s_dyn[];
  okb_pair* s_top = s_dyn;                                   // [AS_CHUNK][num_best]
  okb_pair* P = in_smem ? s_dyn + (size_t)AS_CHUNK * MAX_BEST : pairs;
  int* cnt = in_smem ? reinterpret_cast<int*>(P + nB) : nullptr;   // [nB] how many A's list this b
  __shared__ uint8_t s_skip[AS_CHUNK];
  __shared__ int s_contested;          // rows that have to take the serial walk
  const int tid = threadIdx.x;
  if (tid == 0) s_contested = 0;
  for (int b = tid; b < nB; b += AS_T) { P[b].index_a = -1; P[b].distance = 3.402823466e+38f; if (cnt) cnt[b] = 0; }
  for (int a = tid; a < nA; a += AS_T) done[a] = 0;
  __syncthreads();
  if (cnt) {
    for (int e = tid; e < nA * num_best; e += AS_T) {
      const int a = e / num_best;
      if (skipA && skipA[a]) continue;
      const int b = topk[e].index_a;
      if (b >= 0) atomicAdd(&cnt[b], 1);
    }
    __syncthreads();
    for (int a = tid; a < nA; a += AS_T) {
      if (skipA && skipA[a]) continue;
      const okb_pair first = topk[(size_t)a * num_best];
      if (first.index_a >= 0 && cnt[first.index_a] == 1) { P[first.index_a].index_a = a; P[first.index_a].distance = first.distance; done[a] = 1; }
      else if (first.index_a >= 0) atomicAdd(&s_contested, 1);
    }
  } else if (tid == 0) s_contested = nA;
  __syncthreads();
  for (int base = 0; base < nA && s_contested > 0; base += AS_CHUNK) {
    const int n_in = min(AS_CHUNK, nA - base);
    __syncthreads();
    for (int e = tid; e < n_in * num_best; e += AS_T) s_top[e] = topk[(size_t)base * num_best + e];
    for (int i = tid; i < n_in; i += AS_T) s_skip[i] = (skipA ? skipA[base + i] : 0) | done[base + i];
    __syncthreads();
    if (tid != 0) continue;
    for (int i = 0; i < n_in; ++i) {
      if (s_skip[i]) continue;
      int a = base + i, start = 0;
      while (a >= 0) {
        int next = -1;
        const okb_pair* lst = (a >= base && a < base + n_in) ? s_top + (size_t)(a - base) * num_best : topk + (size_t)a * num_best;
        for (int idx = start; idx < num_best; ++idx) {
          const okb_pair cand = lst[idx];
          if (cand.index_a == -1) break;
          const int b = cand.index_a;
          const okb_pair cur = P[b];
          if (cur.index_a == -1) { P[b].index_a = a; P[b].distance = cand.distance; break; }
          if (cand.distance < cur.distance) {
            next = cur.index_a;
            P[b].index_a = a; P[b].distance = cand.distance;
            break;
          }
        }
        a = next;
        start = 1;
      }
    }
  }
  __syncthreads();
  if (in_smem) for (int b = tid; b < nB; b += AS_T) pairs[b] = P[b];
}

// Candidate lists (every B with distance < thr, ascending B): warp per A, lanes over 32 consecutive B's; the ballot's
// prefix population count gives each hit its position, so the CSR rows come out in ascending B order.
template <int NW>
__global__ void __launch_bounds__(MT) k_cand_count(const uint32_t* __restrict__ A, int nA, const uint32_t* __restrict__ B, int nB,
                                                   float thr, uint32_t* counts, const uint32_t* row_ptr, uint32_t* col, uint16_t* dist,
                                                   int cap, int fill) {
  __shared__ uint32_t sB[MB_TILE][NW + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int a = blockIdx.x * MW + warp;
  uint32_t wa[NW];
#pragma unroll
  for (int w = 0; w < NW; ++w) wa[w] = (a < nA) ? A[(size_t)a * NW + w] : 0u;
  uint32_t n = 0;
  const uint32_t base = (fill && a < nA) ? row_ptr[a] : 0;
  for (int b0 = 0; b0 < nB; b0 += MB_TILE) {
    const int nb = min(MB_TILE, nB - b0);
    __syncthreads();
    for (int i = threadIdx.x; i < nb * NW; i += MT) sB[i / NW][i % NW] = B[(size_t)b0 * NW + i];
    __syncthreads();
    if (a >= nA) continue;
    for (int j0 = 0; j0 < nb; j0 += 32) {
      const int j = j0 + lane;
      int d = 1 << 30;
      if (j < nb) {
        d = 0;
#pragma unroll
        for (int w = 0; w < NW; ++w) d += __popc(wa[w] ^ sB[j][w]);
      }
      const bool hit = j < nb && (float)d < thr;
      const uint32_t m = __ballot_sync(0xffffffffu, hit);
      if (fill && hit) {
        const uint32_t pos = base + n + (uint32_t)__popc(m & ((1u << lane) - 1u));
        if (pos < (uint32_t)cap) { col[pos] = (uint32_t)(b0 + j); dist[pos] = (uint16_t)d; }
      }
      n += (uint32_t)__popc(m);
    }
  }
  if (!fill && a < nA && lane == 0) counts[a] = n;
}

// exclusive scan of the per-A counts (one CTA, 1024 threads, chunks of 1024 with a running carry)
__global__ void __launch_bounds__(1024) k_exclusive_scan(const uint32_t* counts, int n, uint32_t* row_ptr) {
  __shared__ int s_warp[32];
  int run = 0;
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = (i < n) ? (int)counts[i] : 0;
    int total;
    const int ex = uni_block_scan(v, s_warp, &total);
    if (i < n) row_ptr[i] = (uint32_t)(run + ex);
    run += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) row_ptr[n] = (uint32_t)run;
}
}  // namespace

template <typename T>
static int grow(okb_ctx* c, T** p, size_t* cap, size_t need) {
  if (*cap >= need) return OKB_OK;
  cudaFree(*p);
  *p = nullptr; *cap = 0;
  FE_CUDA(c, cudaMalloc(p, need * sizeof(T)));
  *cap = need;
  return OKB_OK;
}

#define DISPATCH_NW(nw, CALL)                 \
  switch (nw) {                               \
    case 8: { constexpr int NW = 8; CALL; } break;   \
    case 12: { constexpr int NW = 12; CALL; } break; \
    case 16: { constexpr int NW = 16; CALL; } break; \
    case 32: { constexpr int NW = 32; CALL; } break; \
    default: c->set_error("descriptor length must be 32, 48, 64 or 128 bytes"); return OKB_ERR_UNSUPPORTED; \
  }

static int upload_descriptors(okb_ctx* c, okb_frontend_state* F, const uint8_t* A, int nA, const uint8_t* B, int nB, int bytes,
                              const uint8_t* skipA, const uint8_t* skipB) {
  int rc;
  if ((rc = grow(c, &F->d_A, &F->capA, (size_t)nA * bytes + nA))) return rc;
  if ((rc = grow(c, &F->d_B, &F->capB, (size_t)nB * bytes + nB))) return rc;
  FE_CUDA(c, cudaMemcpyAsync(F->d_A, A, (size_t)nA * bytes, cudaMemcpyHostToDevice, c->stream));
  FE_CUDA(c, cudaMemcpyAsync(F->d_B, B, (size_t)nB * bytes, cudaMemcpyHostToDevice, c->stream));
  if (skipA) FE_CUDA(c, cudaMemcpyAsync(F->d_A + (size_t)nA * bytes, skipA, nA, cudaMemcpyHostToDevice, c->stream));
  if (skipB) FE_CUDA(c, cudaMemcpyAsync(F->d_B + (size_t)nB * bytes, skipB, nB, cudaMemcpyHostToDevice, c->stream));
  return OKB_OK;
}

static int ensure_io(okb_ctx* c, okb_frontend_state* F, size_t bytes) {
  if (F->h_stage_cap < bytes) {
    if (F->h_stage) cudaFreeHost(F->h_stage);
    F->h_stage = nullptr; F->h_stage_cap = 0;
    FE_CUDA(c, cudaMallocHost(&F->h_stage, bytes));
    F->h_stage_cap = bytes;
  }
  if (F->d_io_cap < bytes) {
    cudaFree(F->d_io);
    F->d_io = nullptr; F->d_io_cap = 0;
    FE_CUDA(c, cudaMalloc(&F->d_io, bytes));
    F->d_io_cap = bytes;
  }
  return OKB_OK;
}

static int hamming_match_impl(okb_ctx* c, const uint8_t* A, int nA, const uint8_t* B, int nB, int desc_bytes, const uint8_t* skipA,
                              const uint8_t* skipB, float threshold, int num_best, int use_ratio, const okb_match_gate* gate,
                              okb_pair* out_topk, okb_pair* out_pairs) {
  if (!c || nA < 0 || nB < 0 || num_best < 1 || num_best > MAX_BEST || (nB > 0 && !out_pairs)) return OKB_ERR_INVALID_ARG;
  if (nA == 0 || nB == 0) {     // an empty list matches nothing (DenseMatcher::match on an empty MatchingAlgorithm): no device work
    for (int i = 0; i < nB; ++i) { out_pairs[i].index_a = -1; out_pairs[i].distance = threshold; }
    if (out_topk) for (size_t i = 0; i < (size_t)nA * num_best; ++i) { out_topk[i].index_a = -1; out_topk[i].distance = threshold; }
    return OKB_OK;
  }
  if (!A || !B) return OKB_ERR_INVALID_ARG;
  if (desc_bytes % 4) { c->set_error("descriptor length must be a multiple of 4"); return OKB_ERR_UNSUPPORTED; }
  const int mode = gate ? gate->mode : OKB_GATE_NONE;
  if (mode != OKB_GATE_NONE && mode != OKB_GATE_3D2D && mode != OKB_GATE_2D2D) return OKB_ERR_INVALID_ARG;
  if (mode != OKB_GATE_NONE && (!gate->kp_b || !gate->kp_size_b)) return OKB_ERR_INVALID_ARG;
  if (mode == OKB_GATE_3D2D && (!gate->proj_into_b || !gate->proj_uncertainty)) return OKB_ERR_INVALID_ARG;
  if (mode == OKB_GATE_2D2D && (!gate->kp_a || !gate->kp_size_a || !gate->bearing_a || !gate->bearing_b || !gate->ray_sigma_a || !gate->ray_sigma_b))
    return OKB_ERR_INVALID_ARG;
  cudaSetDevice(c->device);
  okb_frontend_state* F = fe(c);
  std::lock_guard<std::mutex> lk(F->match_mtx);
  // one pinned staging buffer, one copy in, one copy out:
  //   [A | B | skipA | skipB | gate arrays | GateDev]  ...  [top-k lists | winners | scratch]
  auto up16 = [](size_t v) { return (v + 15) & ~(size_t)15; };
  const size_t oA = 0, oB = up16((size_t)nA * desc_bytes), oSA = oB + up16((size_t)nB * desc_bytes), oSB = oSA + up16((size_t)nA);
  size_t oG = oSB + up16((size_t)nB);
  // gate arrays (doubles): kp_b 2nB | size_b nB | proj 2nA | unc 4nA | kp_a 2nA | size_a nA | bear_a 3nA | bear_b 3nB | rs_a nA | rs_b nB
  const size_t g_kpb = oG, g_szb = g_kpb + 16 * (size_t)nB, g_proj = g_szb + up16(8 * (size_t)nB), g_unc = g_proj + 16 * (size_t)nA,
               g_kpa = g_unc + 32 * (size_t)nA, g_sza = g_kpa + 16 * (size_t)nA, g_ba = g_sza + up16(8 * (size_t)nA), g_bb = g_ba + up16(24 * (size_t)nA),
               g_rsa = g_bb + up16(24 * (size_t)nB), g_rsb = g_rsa + up16(8 * (size_t)nA), g_dev = g_rsb + up16(8 * (size_t)nB);
  const size_t in_bytes = mode == OKB_GATE_NONE ? oG : g_dev + up16(sizeof(GateDev));
  const size_t oT = in_bytes, oP = oT + sizeof(okb_pair) * (size_t)nA * num_best, oD = oP + sizeof(okb_pair) * (size_t)nB, total = oD + up16((size_t)nA);
  int rc = ensure_io(c, F, total);
  if (rc) return rc;
  std::memcpy(F->h_stage + oA, A, (size_t)nA * desc_bytes);
  std::memcpy(F->h_stage + oB, B, (size_t)nB * desc_bytes);
  if (skipA) std::memcpy(F->h_stage + oSA, skipA, nA);
  if (skipB) std::memcpy(F->h_stage + oSB, skipB, nB);
  if (mode != OKB_GATE_NONE) {
    GateDev gd;
    std::memset(&gd, 0, sizeof gd);
    gd.mode = mode;
    auto put = [&](size_t off, const double* src, size_t n) -> const double* {
      if (src) std::memcpy(F->h_stage + off, src, 8 * n);
      return reinterpret_cast<const double*>(F->d_io + off);
    };
    gd.kp_b = put(g_kpb, gate->kp_b, 2 * (size_t)nB); gd.kp_size_b = put(g_szb, gate->kp_size_b, nB);
    if (mode == OKB_GATE_3D2D) { gd.proj_into_b = put(g_proj, gate->proj_into_b, 2 * (size_t)nA); gd.proj_unc = put(g_unc, gate->proj_uncertainty, 4 * (size_t)nA); }
    else {
      gd.kp_a = put(g_kpa, gate->kp_a, 2 * (size_t)nA); gd.kp_size_a = put(g_sza, gate->kp_size_a, nA);
      gd.bearing_a = put(g_ba, gate->bearing_a, 3 * (size_t)nA); gd.bearing_b = put(g_bb, gate->bearing_b, 3 * (size_t)nB);
      gd.ray_sigma_a = put(g_rsa, gate->ray_sigma_a, nA); gd.ray_sigma_b = put(g_rsb, gate->ray_sigma_b, nB);
      cam_load(gate->cam_a, gd.cam_a); cam_load(gate->cam_b, gd.cam_b);
      gd.wa = gate->cam_a.width; gd.ha = gate->cam_a.height; gd.wb = gate->cam_b.width; gd.hb = gate->cam_b.height;
      double q[4] = {gate->T_AB[3], gate->T_AB[4], gate->T_AB[5], gate->T_AB[6]};
      qnormalize(q);
      q2R(q, gd.R_AB);
      gd.t_AB[0] = gate->T_AB[0]; gd.t_AB[1] = gate->T_AB[1]; gd.t_AB[2] = gate->T_AB[2];
    }
    std::memcpy(F->h_stage + g_dev, &gd, sizeof gd);
  }
  FE_CUDA(c, cudaMemcpyAsync(F->d_io, F->h_stage, in_bytes, cudaMemcpyHostToDevice, c->stream));
  const uint8_t* dSA = skipA ? F->d_io + oSA : nullptr;
  const uint8_t* dSB = skipB ? F->d_io + oSB : nullptr;
  okb_pair* d_topk = reinterpret_cast<okb_pair*>(F->d_io + oT);
  okb_pair* d_pairs = reinterpret_cast<okb_pair*>(F->d_io + oP);
  const GateDev* d_gate = reinterpret_cast<const GateDev*>(F->d_io + g_dev);
  // DenseMatcher.hpp(impl):188-193: with the ratio test the lists are built without a threshold
  const float list_thr = use_ratio ? 3.402823466e+38f : threshold;
  const int nw = desc_bytes / 4;
  if (mode == OKB_GATE_NONE) {
    DISPATCH_NW(nw, (k_hamming_topk<NW, false><<<(nA + MW - 1) / MW, MT, 0, c->stream>>>(
                        reinterpret_cast<const uint32_t*>(F->d_io + oA), nA, reinterpret_cast<const uint32_t*>(F->d_io + oB), nB, dSA, dSB, list_thr,
                        num_best, d_topk, 0.f, nullptr)));
  } else {
    DISPATCH_NW(nw, (k_hamming_topk<NW, true><<<(nA + MW - 1) / MW, MT, 0, c->stream>>>(
                        reinterpret_cast<const uint32_t*>(F->d_io + oA), nA, reinterpret_cast<const uint32_t*>(F->d_io + oB), nB, dSA, dSB, list_thr,
                        num_best, d_topk, threshold, d_gate)));
  }
  {
    const size_t sm_top = sizeof(okb_pair) * (size_t)AS_CHUNK * MAX_BEST;
    const size_t sm_b = (sizeof(okb_pair) + sizeof(int)) * (size_t)nB;        // per-B winners + list counts
    const int in_smem = sm_top + sm_b + 1024 <= (size_t)c->smem_optin ? 1 : 0;
    const size_t sm = sm_top + (in_smem ? sm_b : 0);
    if (sm > 48 * 1024 - 512) FE_CUDA(c, cudaFuncSetAttribute(k_assign, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    k_assign<<<1, AS_T, sm, c->stream>>>(d_topk, nA, nB, num_best, dSA, d_pairs, F->d_io + oD, in_smem);
  }
  c->launches += 2;
  FE_CUDA(c, cudaGetLastError());
  FE_CUDA(c, cudaMemcpyAsync(F->h_stage + oT, F->d_io + oT, oD - oT, cudaMemcpyDeviceToHost, c->stream));
  FE_CUDA(c, cudaStreamSynchronize(c->stream));
  if (out_topk) std::memcpy(out_topk, F->h_stage + oT, sizeof(okb_pair) * (size_t)nA * num_best);
  std::memcpy(out_pairs, F->h_stage + oP, sizeof(okb_pair) * (size_t)nB);
  return OKB_OK;
}

extern "C" int okb_hamming_match(okb_ctx* c, const uint8_t* A, int nA, const uint8_t* B, int nB, int desc_bytes, const uint8_t* skipA,
                                 const uint8_t* skipB, float threshold, int num_best, int use_ratio, float ratio_threshold,
                                 okb_pair* out_topk, okb_pair* out_pairs) {
  (void)ratio_threshold;   // the ratio test itself belongs to the serial epilogue on the caller's side
  return hamming_match_impl(c, A, nA, B, nB, desc_bytes, skipA, skipB, threshold, num_best, use_ratio, nullptr, out_topk, out_pairs);
}

extern "C" int okb_hamming_match_gated(okb_ctx* c, const uint8_t* A, int nA, const uint8_t* B, int nB, int desc_bytes, const uint8_t* skipA,
                                       const uint8_t* skipB, float threshold, int num_best, int use_ratio, float ratio_threshold,
                                       const okb_match_gate* gate, okb_pair* out_topk, okb_pair* out_pairs) {
  (void)ratio_threshold;
  if (!gate) return OKB_ERR_INVALID_ARG;
  return hamming_match_impl(c, A, nA, B, nB, desc_bytes, skipA, skipB, threshold, num_best, use_ratio, gate, out_topk, out_pairs);
}

extern "C" int okb_hamming_candidates(okb_ctx* c, const uint8_t* A, int nA, const uint8_t* B, int nB, int desc_bytes, float threshold,
                                      uint32_t* row_ptr, uint32_t* col_idx, uint16_t* dist, int cap) {
  if (!c || nA < 0 || nB < 0 || !row_ptr || cap < 0) return OKB_ERR_INVALID_ARG;
  if (nA == 0 || nB == 0) {     // empty lists: empty rows, no device work
    for (int i = 0; i <= nA; ++i) row_ptr[i] = 0;
    return OKB_OK;
  }
  if (!A || !B) return OKB_ERR_INVALID_ARG;
  cudaSetDevice(c->device);
  okb_frontend_state* F = fe(c);
  std::lock_guard<std::mutex> lk(F->match_mtx);
  int rc = upload_descriptors(c, F, A, nA, B, nB, desc_bytes, nullptr, nullptr);
  if (rc) return rc;
  if ((rc = grow(c, &F->d_rowptr, &F->cap_rows, (size_t)2 * nA + 2))) return rc;
  if (cap > 0) {
    size_t cc = F->cap_cand;
    if ((rc = grow(c, &F->d_col, &cc, (size_t)cap))) return rc;
    cc = F->cap_cand;
    if ((rc = grow(c, &F->d_dist, &cc, (size_t)cap))) return rc;
    F->cap_cand = std::max(F->cap_cand, (size_t)cap);
  }
  uint32_t* d_counts = F->d_rowptr + nA + 1;
  const int nw = desc_bytes / 4;
  if (desc_bytes % 4) { c->set_error("descriptor length must be a multiple of 4"); return OKB_ERR_UNSUPPORTED; }
  DISPATCH_NW(nw, (k_cand_count<NW><<<(nA + MW - 1) / MW, MT, 0, c->stream>>>(
                      reinterpret_cast<const uint32_t*>(F->d_A), nA, reinterpret_cast<const uint32_t*>(F->d_B), nB, threshold, d_counts,
                      nullptr, nullptr, nullptr, 0, 0)));
  k_exclusive_scan<<<1, 1024, 0, c->stream>>>(d_counts, nA, F->d_rowptr);
  if (cap > 0) {
    DISPATCH_NW(nw, (k_cand_count<NW><<<(nA + MW - 1) / MW, MT, 0, c->stream>>>(
                        reinterpret_cast<const uint32_t*>(F->d_A), nA, reinterpret_cast<const uint32_t*>(F->d_B), nB, threshold, d_counts,
                        F->d_rowptr, F->d_col, F->d_dist, cap, 1)));
  }
  c->launches += 3;
  FE_CUDA(c, cudaGetLastError());
  FE_CUDA(c, cudaMemcpyAsync(row_ptr, F->d_rowptr, sizeof(uint32_t) * (nA + 1), cudaMemcpyDeviceToHost, c->stream));
  FE_CUDA(c, cudaStreamSynchronize(c->stream));
  const uint32_t total = row_ptr[nA];
  const uint32_t ncopy = std::min<uint32_t>(total, (uint32_t)cap);
  if (ncopy && col_idx) FE_CUDA(c, cudaMemcpyAsync(col_idx, F->d_col, sizeof(uint32_t) * ncopy, cudaMemcpyDeviceToHost, c->stream));
  if (ncopy && dist) FE_CUDA(c, cudaMemcpyAsync(dist, F->d_dist, sizeof(uint16_t) * ncopy, cudaMemcpyDeviceToHost, c->stream));
  FE_CUDA(c, cudaStreamSynchronize(c->stream));
  if (total > (uint32_t)cap) { c->set_error("candidate capacity too small"); return OKB_ERR_CAPACITY; }
  return OKB_OK;
}
