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
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <mutex>
#include <vector>

#include "okb_ctx.h"
#include "okb_hostpack.hpp"
#include "okb_math.cuh"

using namespace okb;

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

// One image of a detect launch (device table, one entry per image): its geometry, its gravity direction and where
// its data lie in the launch's buffers.
struct FeImage {
  okb_camera cam;
  double gC[3];                 // gravity direction in the camera frame: R_CW * (0,0,-1)
  unsigned long long img;       // byte offset of the packed image (row stride W) in the input buffer
  unsigned long long px;        // element offset of its score plane (cumulative W * H)
  unsigned long long ii;        // element offset of its integral image (cumulative (W + 1) * (H + 1))
  unsigned long long uni;       // word offset of its global-memory uniformity scratch (sized by its own cell grid)
  int W, H, max_cells;
};

// Buffers of a detect launch over n images; they grow with the launch and are kept across calls.  A camera slot owns
// one set (n = 1), the batch call another.
struct DetectBuffers {
  uint8_t* h_in = nullptr;         // pinned: [FeImage table | packed images], one H2D copy
  uint8_t* d_in = nullptr;
  size_t h_in_cap = 0, d_in_cap = 0;
  int32_t* d_score = nullptr;
  uint32_t* d_integral = nullptr;
  unsigned long long* d_keys = nullptr;    // [n][kMaxCand]
  uint32_t* d_uni = nullptr;       // [n][uni_stride]: global-memory uniformity scratch (UniScratch)
  uint8_t* d_state = nullptr;      // [n][kMaxCand]
  size_t cap_score = 0, cap_integral = 0, cap_keys = 0, cap_uni = 0, cap_state = 0;
  uint8_t* d_out = nullptr;        // [counts n x 4 | keypoints n x maxk | descriptors n x maxk x desc_bytes], one D2H copy
  uint8_t* h_out = nullptr;        // pinned mirror
  size_t d_out_cap = 0, h_out_cap = 0;
  void release() {
    if (h_in) cudaFreeHost(h_in);
    if (h_out) cudaFreeHost(h_out);
    cudaFree(d_in); cudaFree(d_score); cudaFree(d_integral); cudaFree(d_keys); cudaFree(d_uni); cudaFree(d_state); cudaFree(d_out);
  }
};

struct DevPattern {
  int* half = nullptr;
  uint8_t *pi = nullptr, *pj = nullptr;
  int16_t* lut = nullptr;
};

struct SlotBuffers {
  cudaStream_t stream = nullptr;
  DetectBuffers buf;
  std::mutex mtx;
};

// One image's host outputs of a detect launch: [max_out] keypoints, [max_out][desc_bytes] descriptors (nullptr: not
// wanted) and its count.
struct DetectOut {
  okb_keypoint* kp;
  uint8_t* desc;
  int32_t* n;
};

// One image's store entry (okb_detect_describe_store_batch): the device addresses of keypoint 0 of (feat_slot, cam) in
// each array of the window's FeatStore, and of the entry's count.
struct StoreDest {
  double* kp;                   // [N][2]
  double* size;
  uint32_t* desc;               // [N][D/4]
  int32_t* lm;
  uint8_t* observed;
  int* n;
};
}  // namespace

struct okb_frontend_state {
  SlotBuffers slots[kMaxSlots];
  // batch calls: a stream of their own (never c->stream, so a batch does not queue behind a solve) and their buffers
  cudaStream_t batch_stream = nullptr;
  cudaEvent_t store_ready = nullptr;  // okb_detect_describe_store_batch: recorded after its commit on c->stream_xfer
  DetectBuffers batch_det;
  CallBuffers batch_match;
  std::mutex batch_mtx;
  // pattern (device), per descriptor length
  DevPattern pats[128 / 4 + 1];       // indexed by desc_bytes / 4
  std::mutex pat_mtx;
  // matcher buffers
  uint8_t *d_A = nullptr, *d_B = nullptr, *d_skipA = nullptr, *d_skipB = nullptr;
  size_t capA = 0, capB = 0;
  okb_pair *d_topk = nullptr, *d_pairs = nullptr;
  size_t cap_topk = 0, cap_pairs = 0;
  uint32_t *d_rowptr = nullptr, *d_col = nullptr;
  uint16_t* d_dist = nullptr;
  size_t cap_rows = 0, cap_cand = 0;
  CallBuffers match_io;            // okb_hamming_match / _gated (on c->stream, under match_mtx)
  std::atomic<int64_t> launches{0};   // frontend kernel launches (okb_kernel_launches adds them to the solver's)
  std::mutex match_mtx;
  // the calls on a window's feature store, on c->stream_xfer, one set each so that different calls overlap:
  CallBuffers track;               // okb_track_3d2d_batch
  CallBuffers stereo;              // okb_match2d2d_batch / okb_stereo_init_batch
  CallBuffers kf;                  // okb_keyframe_overlap_batch (scratch: images too large for shared memory)
  CallBuffers ransac;              // okb_ransac_3d2d_batch
  CallBuffers ransac2d;            // okb_ransac_2d2d_batch
};

void okb_frontend_release(okb_ctx* c) {
  if (!c->frontend) return;
  okb_frontend_state* F = c->frontend;
  for (CallBuffers* b : {&F->match_io, &F->batch_match, &F->track, &F->stereo, &F->kf, &F->ransac, &F->ransac2d}) b->release();
  F->batch_det.release();
  if (F->batch_stream) cudaStreamDestroy(F->batch_stream);
  if (F->store_ready) cudaEventDestroy(F->store_ready);
  for (auto& s : F->slots) {
    if (s.stream) cudaStreamDestroy(s.stream);
    s.buf.release();
  }
  for (auto& p : F->pats) { cudaFree(p.half); cudaFree(p.pi); cudaFree(p.pj); cudaFree(p.lut); }
  cudaFree(F->d_A); cudaFree(F->d_B); cudaFree(F->d_skipA); cudaFree(F->d_skipB); cudaFree(F->d_topk); cudaFree(F->d_pairs);
  cudaFree(F->d_rowptr); cudaFree(F->d_col); cudaFree(F->d_dist);
  delete F;
  c->frontend = nullptr;
}

int64_t okb_frontend_launches(const okb_ctx* c) { return c->frontend ? c->frontend->launches.load() : 0; }

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
// gradient products live in shared memory.  blockIdx.z is the image; the grid covers the largest image of the launch
// and the tiles outside an image exit (the detector kernels below all index images the same way).
__global__ void __launch_bounds__(HT_X* HT_Y) k_harris(const FeImage* __restrict__ tab, const uint8_t* __restrict__ in,
                                                       int32_t* __restrict__ score_all) {
  __shared__ uint8_t tile[HT_Y + 6][HT_X + 6 + 2];
  __shared__ int32_t sxx[HT_Y + 4][HT_X + 4], syy[HT_Y + 4][HT_X + 4], sxy[HT_Y + 4][HT_X + 4];
  const FeImage& im = tab[blockIdx.z];
  const int W = im.W, H = im.H;
  const int bx = blockIdx.x * HT_X, by = blockIdx.y * HT_Y;
  if (bx >= W || by >= H) return;
  const uint8_t* __restrict__ img = in + im.img;
  int32_t* __restrict__ score = score_all + im.px;
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
// (per image: keys [cap], candidate count at count[0] of its 4-int record)
__global__ void k_nms(const FeImage* __restrict__ tab, const int32_t* __restrict__ score_all, int32_t thr, unsigned long long* keys_all,
                      int* count_all, int cap) {
  const FeImage& im = tab[blockIdx.z];
  const int W = im.W, H = im.H;
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x < kBorder || x >= W - kBorder || y < kBorder || y >= H - kBorder) return;
  const int32_t* __restrict__ score = score_all + im.px;
  unsigned long long* keys = keys_all + (size_t)blockIdx.z * cap;
  int* count = count_all + 4 * blockIdx.z;
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
// One CTA of 1024 threads per image (blockIdx.x); all scratch lives in global memory, one UniScratch per image.
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
};
// u32 words of one image's scratch (offsets in FeImage::uni): cell_start | cell_cur | order | acc | blocker | list0 | list1 | pend (state apart)
__host__ __device__ inline size_t uni_stride(int max_cells, int cap) { return 2 * (size_t)max_cells + 1 + 6 * (size_t)cap; }
__device__ inline UniScratch uni_scratch(uint32_t* base, uint8_t* state, int max_cells, int cap, int img) {
  UniScratch s;
  s.cell_start = base;
  s.cell_cur = s.cell_start + max_cells + 1;
  s.order = s.cell_cur + max_cells;
  s.acc = s.order + cap;
  s.blocker = s.acc + cap; s.list0 = s.blocker + cap; s.list1 = s.list0 + cap; s.pend = s.list1 + cap;
  s.state = state + (size_t)img * cap;
  return s;
}
// exclusive scan of one int per thread over an NT-thread CTA (s_warp: NT / 32 shared ints); *total = sum (all threads)
template <int NT>
__device__ __forceinline__ int block_scan(int v, int* s_warp, int* total) {
  constexpr int NWT = NT / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  __syncthreads();
  if (lane == 31) s_warp[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = lane < NWT ? s_warp[lane] : 0;
#pragma unroll
    for (int o = 1; o < NWT; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
    if (lane < NWT) s_warp[lane] = w;
  }
  __syncthreads();
  *total = s_warp[NWT - 1];
  return (warp ? s_warp[warp - 1] : 0) + x - v;
}
__global__ void __launch_bounds__(UT, 2) k_uniformity(const FeImage* __restrict__ tab, const unsigned long long* __restrict__ keys_all,
                                                   int* count_all, int cap, double radius, int max_kp, uint32_t* uni_base,
                                                   uint8_t* uni_state, okb_keypoint* kps_all) {
  __shared__ int s_warp[32];
  __shared__ int s_n;
  const int tid = threadIdx.x;
  const int W = tab[blockIdx.x].W, H = tab[blockIdx.x].H;
  const unsigned long long* __restrict__ keys = keys_all + (size_t)blockIdx.x * cap;
  int* n_out = count_all + 4 * blockIdx.x + 1;
  okb_keypoint* kps = kps_all + (size_t)blockIdx.x * max_kp;
  const int n = min(n_out[-1], cap);
  const int cs = max(4, (int)ceil(radius));
  const int gw = (W + cs - 1) / cs, gh = (H + cs - 1) / cs, n_cells = gw * gh;
  if (uni_fits_smem(n, n_cells)) return;       // k_uniformity_smem (launched next) does this image
  const UniScratch sc = uni_scratch(uni_base + tab[blockIdx.x].uni, uni_state, tab[blockIdx.x].max_cells, cap, blockIdx.x);
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
    const int ex = block_scan<UT>(v, s_warp, &total);
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
__global__ void __launch_bounds__(UT) k_uniformity_smem(const FeImage* __restrict__ tab, const unsigned long long* __restrict__ keys_all,
                                                        int* count_all, int cap, double radius, int max_kp, okb_keypoint* kps_all) {
  extern __shared__ __align__(16) unsigned char uni_raw[];
  UniSmem& S = *reinterpret_cast<UniSmem*>(uni_raw);
  __shared__ int s_warp[32];
  __shared__ int s_n, s_alive, s_pend;
  const int tid = threadIdx.x;
  const int W = tab[blockIdx.x].W, H = tab[blockIdx.x].H;
  const unsigned long long* __restrict__ keys = keys_all + (size_t)blockIdx.x * cap;
  int* n_out = count_all + 4 * blockIdx.x + 1;
  okb_keypoint* kps = kps_all + (size_t)blockIdx.x * max_kp;
  const int n = min(n_out[-1], cap);
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
      const int ex = block_scan<UT>(v, s_warp, &total);
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
// (blockIdx.y: image)
__global__ void __launch_bounds__(128) k_integral_rows(const FeImage* __restrict__ tab, const uint8_t* __restrict__ in, uint32_t* II_all) {
  const FeImage& im = tab[blockIdx.y];
  const int W = im.W, H = im.H;
  const int y = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (y > H) return;
  const uint8_t* __restrict__ img = in + im.img;
  uint32_t* row = II_all + im.ii + (size_t)y * (W + 1);
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
// running sums.  Integer arithmetic: any summation order gives the same bits.  blockIdx.y: image.
constexpr int IC_SEG = 16;
__global__ void __launch_bounds__(32 * IC_SEG) k_integral_cols(const FeImage* __restrict__ tab, uint32_t* II_all) {
  __shared__ uint32_t seg[IC_SEG][33];
  const FeImage& im = tab[blockIdx.y];
  const int W = im.W, H = im.H;
  if (blockIdx.x * 32 > W) return;
  uint32_t* II = II_all + im.ii;
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

// Orientation exactly as Frame::describe (Frame.hpp(impl):128-151), thread per keypoint: back-project (5 Gauss-Newton
// undistort iterations), project with Jacobian, atan2 of the projected gravity direction, in degrees, into
// keypoint.angle.  blockIdx.y: image (its camera and gravity direction come from its table entry).  Launched only with
// rotation invariance; k_describe reads the angle back.
__global__ void __launch_bounds__(128) k_orient(const FeImage* __restrict__ tab, okb_keypoint* kps_all, int max_kp, const int* count_all) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count_all[4 * blockIdx.y + 1]) return;
  const FeImage& im = tab[blockIdx.y];
  okb_keypoint& kp = kps_all[(size_t)blockIdx.y * max_kp + k];
  const int x = (int)kp.x, y = (int)kp.y;
  CamIntr cam;
  cam_load(im.cam, cam);
  const double* gC = im.gC;
  double pu[2];
  undistort_gn(cam, ((double)x - cam.cu) / cam.fu, ((double)y - cam.cv) / cam.fv, pu);
  const double ep[3] = {pu[0], pu[1], 1.0};
  double ip[2], J[6];
  project<true>(cam, ep, ip, J);
  const double e0 = J[0] * gC[0] + J[1] * gC[1] + J[2] * gC[2];
  const double e1 = J[3] * gC[0] + J[4] * gC[1] + J[5] * gC[2];
  kp.angle = (float)(atan2(e1, e0) / 3.14159265358979323846 * 180.0);
}

// warp per keypoint: 60 box-smoothed samples rotated by the keypoint's angle (k_orient, or 0), 8*desc_bytes
// comparisons via ballot.  blockIdx.y: image.
__global__ void __launch_bounds__(128) k_describe(const FeImage* __restrict__ tab, const uint32_t* __restrict__ II_all,
                                                  const int* __restrict__ half, const uint8_t* __restrict__ pi,
                                                  const uint8_t* __restrict__ pj, const int16_t* __restrict__ lut, int desc_bytes,
                                                  const okb_keypoint* kps_all, int max_kp, const int* count_all, uint8_t* desc_all) {
  __shared__ uint32_t sS[4][64], sA[4][64];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int k = blockIdx.x * 4 + wib;
  if (k >= count_all[4 * blockIdx.y + 1]) return;
  const FeImage& im = tab[blockIdx.y];
  const int W = im.W, H = im.H;
  const uint32_t* __restrict__ II = II_all + im.ii;
  const okb_keypoint& kp = kps_all[(size_t)blockIdx.y * max_kp + k];
  uint8_t* desc = desc_all + (size_t)blockIdx.y * max_kp * desc_bytes;
  const int x = (int)kp.x, y = (int)kp.y;
  const float ang = kp.angle;
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

// CTA per image: its keypoints and descriptors from the launch's output buffer into its store entry, as
// CMD_SET_FEATURES writes them (okb_graph.cuh): x, y, size widened to double, landmark slot -1, observed 0, the
// descriptor words, then the count.  An image over the candidate capacity keeps its entry.
__global__ void __launch_bounds__(256) k_store_features(const StoreDest* __restrict__ dst, const int* __restrict__ count_all, int max_cand,
                                                        const okb_keypoint* __restrict__ kps_all, int max_kp,
                                                        const uint8_t* __restrict__ desc_all, int desc_bytes) {
  const int i = blockIdx.x;
  if (count_all[4 * i] > max_cand) return;
  const int n = count_all[4 * i + 1];
  const StoreDest d = dst[i];
  const okb_keypoint* kp = kps_all + (size_t)i * max_kp;
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    const okb_keypoint p = kp[k];
    d.kp[2 * k] = p.x; d.kp[2 * k + 1] = p.y; d.size[k] = p.size;
    d.lm[k] = -1; d.observed[k] = 0;
  }
  const int words = n * (desc_bytes / 4);
  const uint32_t* src = reinterpret_cast<const uint32_t*>(desc_all + (size_t)i * max_kp * desc_bytes);
  for (int k = threadIdx.x; k < words; k += blockDim.x) d.desc[k] = src[k];
  if (threadIdx.x == 0) *d.n = n;
}
}  // namespace

// The device pattern of one descriptor length.  Each length gets its own, kept until the context is destroyed, so
// concurrent calls with different lengths never see a pattern replaced under them.
static int ensure_pattern(okb_ctx* c, okb_frontend_state* F, int desc_bytes, DevPattern* out) {
  std::lock_guard<std::mutex> lk(F->pat_mtx);
  DevPattern& D = F->pats[desc_bytes / 4];
  if (!D.lut) {
    Pattern P = make_pattern(desc_bytes);
    DevPattern N;
    OKB_CUDA(c, cudaMalloc(&N.half, sizeof(int) * kPts));
    OKB_CUDA(c, cudaMalloc(&N.pi, P.pi.size()));
    OKB_CUDA(c, cudaMalloc(&N.pj, P.pj.size()));
    OKB_CUDA(c, cudaMalloc(&N.lut, P.lut.size() * sizeof(int16_t)));
    OKB_CUDA(c, cudaMemcpy(N.half, P.half, sizeof(int) * kPts, cudaMemcpyHostToDevice));
    OKB_CUDA(c, cudaMemcpy(N.pi, P.pi.data(), P.pi.size(), cudaMemcpyHostToDevice));
    OKB_CUDA(c, cudaMemcpy(N.pj, P.pj.data(), P.pj.size(), cudaMemcpyHostToDevice));
    OKB_CUDA(c, cudaMemcpy(N.lut, P.lut.data(), P.lut.size() * sizeof(int16_t), cudaMemcpyHostToDevice));
    D = N;
  }
  *out = D;
  return OKB_OK;
}

// f(i) for every i in [0, n), spread over up to `threads` host threads (<= 0: 8, as okb_window_upload_batch), but
// no more than one thread per 8 MB of `bytes` to move: below that, starting a thread costs more than it saves
template <typename Fn>
static void host_parallel(int n, int threads, size_t bytes, const Fn& f) {
  const int by_bytes = (int)std::min<size_t>(1 + bytes / (8u << 20), 64);
  parallel_for(n, std::max(1, std::min({threads > 0 ? threads : 8, n, by_bytes})), f);
}

// Detect and describe n images with one parameter set on stream `st`, into buffers B: one H2D copy (image table and
// packed images), 7 launches whatever n is, one D2H copy (counts, keypoints, and descriptors when some outs[i].desc is
// set), one synchronisation.  With `dests`, image i is also written into the store entry dests[i] by one more launch,
// k_store_features, queued after `store_after` (an event the caller recorded).  Arguments are checked by the callers;
// maxk = min(max_keypoints, max_out) >= 1.  *outs[i].n = -1 marks an image with more NMS candidates than kMaxCand
// (OKB_ERR_CAPACITY); the other images' outputs are written all the same.
static int detect_run(okb_ctx* c, okb_frontend_state* F, DetectBuffers& B, cudaStream_t st, int n, const okb_image_desc* ims,
                      const okb_detect_params* prm, const DetectOut* outs, int max_out, const StoreDest* dests, cudaEvent_t store_after,
                      int host_threads) {
  const int maxk = std::min(prm->max_keypoints, max_out), db = prm->desc_bytes;
  DevPattern pat;
  int rc = ensure_pattern(c, F, db, &pat);
  if (rc) return rc;
  std::vector<FeImage> tab(n);
  Carve in;                     // [FeImage table | StoreDest table (with dests) | packed images], each on a 256-byte boundary
  in.take(sizeof(FeImage) * n, 256);
  const size_t o_dest = dests ? in.take(sizeof(StoreDest) * n, 256) : 0;
  size_t px = 0, ii = 0, uni = 0;
  int Wmax = 0, Hmax = 0;
  for (int i = 0; i < n; ++i) {
    const okb_image_desc& d = ims[i];
    FeImage& t = tab[i];
    std::memset(&t, 0, sizeof t);
    t.cam = d.cam;
    t.gC[0] = -d.R_CW[2]; t.gC[1] = -d.R_CW[5]; t.gC[2] = -d.R_CW[8];
    t.W = d.width; t.H = d.height;
    t.img = in.take((size_t)d.width * d.height, 256); t.px = px; t.ii = ii; t.uni = uni;
    t.max_cells = ((d.width + 3) / 4) * ((d.height + 3) / 4);          // smallest cell is 4 px
    uni += uni_stride(t.max_cells, kMaxCand);
    px += (size_t)d.width * d.height;
    ii += (size_t)(d.width + 1) * (d.height + 1);
    Wmax = std::max(Wmax, d.width); Hmax = std::max(Hmax, d.height);
  }
  const size_t in_bytes = in.off;
  Carve out;                    // [counts n x 4 | keypoints n x maxk | descriptors n x maxk x desc_bytes]
  out.take(sizeof(int) * 4 * n, 256);
  const size_t o_kp = out.take(sizeof(okb_keypoint) * n * maxk, 256), o_desc = out.off;
  const size_t out_bytes = o_desc + (size_t)n * maxk * db;
  if ((rc = grow_pinned(c, &B.h_in, &B.h_in_cap, in_bytes)) || (rc = grow(c, &B.d_in, &B.d_in_cap, in_bytes)) ||
      (rc = grow(c, &B.d_score, &B.cap_score, px)) || (rc = grow(c, &B.d_integral, &B.cap_integral, ii)) ||
      (rc = grow(c, &B.d_keys, &B.cap_keys, (size_t)n * kMaxCand)) || (rc = grow(c, &B.d_uni, &B.cap_uni, uni)) ||
      (rc = grow(c, &B.d_state, &B.cap_state, (size_t)n * kMaxCand)) || (rc = grow(c, &B.d_out, &B.d_out_cap, out_bytes)) ||
      (rc = grow_pinned(c, &B.h_out, &B.h_out_cap, out_bytes)))
    return rc;
  std::memcpy(B.h_in, tab.data(), sizeof(FeImage) * n);
  if (dests) std::memcpy(B.h_in + o_dest, dests, sizeof(StoreDest) * n);
  host_parallel(n, host_threads, in_bytes, [&](int i) {
    const okb_image_desc& d = ims[i];
    uint8_t* dst = B.h_in + tab[i].img;
    if (d.stride == d.width) std::memcpy(dst, d.img, (size_t)d.width * d.height);
    else
      for (int y = 0; y < d.height; ++y) std::memcpy(dst + (size_t)y * d.width, d.img + (size_t)y * d.stride, d.width);
  });
  OKB_CUDA(c, cudaMemcpyAsync(B.d_in, B.h_in, in_bytes, cudaMemcpyHostToDevice, st));
  OKB_CUDA(c, cudaMemsetAsync(B.d_out, 0, sizeof(int) * 4 * n, st));      // per image: candidates, accepted, rounds, -
  const FeImage* d_tab = reinterpret_cast<const FeImage*>(B.d_in);
  int* d_count = reinterpret_cast<int*>(B.d_out);
  okb_keypoint* d_kp = reinterpret_cast<okb_keypoint*>(B.d_out + o_kp);
  uint8_t* d_desc = B.d_out + o_desc;
  const dim3 hb(HT_X, HT_Y), hg((Wmax + HT_X - 1) / HT_X, (Hmax + HT_Y - 1) / HT_Y, n);
  k_harris<<<hg, hb, 0, st>>>(d_tab, B.d_in, B.d_score);
  const dim3 nb(32, 8), ng((Wmax + 31) / 32, (Hmax + 7) / 8, n);
  k_nms<<<ng, nb, 0, st>>>(d_tab, B.d_score, (int32_t)std::ceil(prm->absolute_threshold), B.d_keys, d_count, kMaxCand);
  k_uniformity<<<n, UT, 0, st>>>(d_tab, B.d_keys, d_count, kMaxCand, prm->uniformity_radius, maxk, B.d_uni, B.d_state, d_kp);
  OKB_CUDA(c, cudaFuncSetAttribute(k_uniformity_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(UniSmem)));
  k_uniformity_smem<<<n, UT, sizeof(UniSmem), st>>>(d_tab, B.d_keys, d_count, kMaxCand, prm->uniformity_radius, maxk, d_kp);
  k_integral_rows<<<dim3((Hmax + 1 + 3) / 4, n), 128, 0, st>>>(d_tab, B.d_in, B.d_integral);
  k_integral_cols<<<dim3((Wmax + 1 + 31) / 32, n), 32 * IC_SEG, 0, st>>>(d_tab, B.d_integral);
  if (prm->rotation_invariance) k_orient<<<dim3((maxk + 127) / 128, n), 128, 0, st>>>(d_tab, d_kp, maxk, d_count);
  k_describe<<<dim3((maxk + 3) / 4, n), 128, 0, st>>>(d_tab, B.d_integral, pat.half, pat.pi, pat.pj, pat.lut, db, d_kp, maxk, d_count,
                                                      d_desc);
  F->launches += prm->rotation_invariance ? 8 : 7;
  if (dests) {
    OKB_CUDA(c, cudaStreamWaitEvent(st, store_after, 0));
    k_store_features<<<n, 256, 0, st>>>(reinterpret_cast<const StoreDest*>(B.d_in + o_dest), d_count, kMaxCand, d_kp, maxk, d_desc, db);
    F->launches += 1;
  }
  OKB_CUDA(c, cudaGetLastError());
  bool want_desc = false;
  for (int i = 0; i < n && !want_desc; ++i) want_desc = outs[i].desc != nullptr;
  OKB_CUDA(c, cudaMemcpyAsync(B.h_out, B.d_out, want_desc ? out_bytes : o_desc, cudaMemcpyDeviceToHost, st));
  OKB_CUDA(c, cudaStreamSynchronize(st));
  const int* h_count = reinterpret_cast<const int*>(B.h_out);
  { static const bool dbg = getenv("OKB_FE_DEBUG") != nullptr;
    if (dbg)
      for (int i = 0; i < n; ++i)
        fprintf(stderr, "[okb frontend] image %d: candidates %d accepted %d uniformity rounds %d\n", i, h_count[4 * i], h_count[4 * i + 1], h_count[4 * i + 2]);
#ifdef OKB_UNI_PROF
    if (dbg) { unsigned long long pr[8]; cudaMemcpyFromSymbol(pr, g_uni_prof, sizeof(pr)); fprintf(stderr, "[okb frontend] uniformity cycles: load %llu grid %llu accept %llu kill %llu rebuild %llu compact %llu rank %llu\n", pr[0], pr[1], pr[2], pr[3], pr[4], pr[5], pr[6]); }
#endif
  }
  int status = OKB_OK;
  for (int i = 0; i < n; ++i) {
    *outs[i].n = h_count[4 * i] > kMaxCand ? -1 : h_count[4 * i + 1];
    if (*outs[i].n < 0) status = OKB_ERR_CAPACITY;
  }
  host_parallel(n, host_threads, want_desc ? out_bytes : o_desc, [&](int i) {
    const int m = *outs[i].n;
    if (m <= 0) return;
    std::memcpy(outs[i].kp, B.h_out + o_kp + sizeof(okb_keypoint) * i * maxk, sizeof(okb_keypoint) * m);
    if (outs[i].desc) std::memcpy(outs[i].desc, B.h_out + o_desc + (size_t)i * maxk * db, (size_t)m * db);
  });
  if (status) c->set_error("too many corner candidates");
  return status;
}

static bool detect_params_ok(const okb_detect_params* prm, int max_out) {
  return (prm->desc_bytes >= 4 && prm->desc_bytes <= 128 && (prm->desc_bytes % 4) == 0) && std::min(prm->max_keypoints, max_out) >= 1;
}

static bool batch_image_ok(const okb_image_desc& d) { return d.img && d.width >= 64 && d.height >= 64 && d.stride >= d.width; }

extern "C" int okb_detect_describe(okb_ctx* c, int cam_slot, const uint8_t* img, int width, int height, int stride,
                                   const okb_camera* cam, const double R_CW[9], const okb_detect_params* prm,
                                   okb_keypoint* out_kp, uint8_t* out_desc, int max_out, int* n_out) {
  if (!c || !img || !cam || !R_CW || !prm || !out_kp || !out_desc || !n_out) return OKB_ERR_INVALID_ARG;
  if (cam_slot < 0 || cam_slot >= kMaxSlots || width < 64 || height < 64 || stride < width) return OKB_ERR_INVALID_ARG;
  if (!detect_params_ok(prm, max_out)) return OKB_ERR_INVALID_ARG;
  cudaSetDevice(c->device);
  okb_frontend_state* F = fe(c);
  SlotBuffers& S = F->slots[cam_slot];
  std::lock_guard<std::mutex> lk(S.mtx);   // the reference guards each camera's detector with a mutex (Frontend.cpp:97)
  if (!S.stream) OKB_CUDA(c, cudaStreamCreateWithFlags(&S.stream, cudaStreamNonBlocking));
  okb_image_desc d;
  std::memset(&d, 0, sizeof d);
  d.img = img; d.width = width; d.height = height; d.stride = stride;
  d.cam = *cam;
  std::memcpy(d.R_CW, R_CW, sizeof d.R_CW);
  int32_t n = 0;
  const DetectOut out{out_kp, out_desc, &n};
  const int rc = detect_run(c, F, S.buf, S.stream, 1, &d, prm, &out, max_out, nullptr, nullptr, 1);
  if (rc == OKB_OK) *n_out = n;
  return rc;
}

extern "C" int okb_detect_describe_batch(okb_ctx* c, int n_images, const okb_image_desc* images, const okb_detect_params* prm,
                                         okb_keypoint* out_kp, uint8_t* out_desc, int max_out, int32_t* n_out, int host_threads) {
  if (!c || n_images < 0) return OKB_ERR_INVALID_ARG;
  if (n_images == 0) return OKB_OK;
  if (n_images > 65535) return OKB_ERR_INVALID_ARG;           // the image index is a grid dimension
  if (!images || !prm || !out_kp || !out_desc || !n_out) return OKB_ERR_INVALID_ARG;
  if (!detect_params_ok(prm, max_out)) return OKB_ERR_INVALID_ARG;
  for (int i = 0; i < n_images; ++i)
    if (!batch_image_ok(images[i])) return OKB_ERR_INVALID_ARG;
  std::vector<DetectOut> outs(n_images);
  for (int i = 0; i < n_images; ++i)
    outs[i] = DetectOut{out_kp + (size_t)i * max_out, out_desc + (size_t)i * max_out * prm->desc_bytes, n_out + i};
  cudaSetDevice(c->device);
  okb_frontend_state* F = fe(c);
  std::lock_guard<std::mutex> lk(F->batch_mtx);
  if (!F->batch_stream) OKB_CUDA(c, cudaStreamCreateWithFlags(&F->batch_stream, cudaStreamNonBlocking));
  return detect_run(c, F, F->batch_det, F->batch_stream, n_images, images, prm, outs.data(), max_out, nullptr, nullptr, host_threads);
}

// =================================================================================================
// matcher kernels
// =================================================================================================
// =================================================================================================
// geometric match gate (VioKeyframeWindowMatchingAlgorithm::verifyMatch, SURVEY 8f row 2) -- evaluated per
// (A, B) pair inside the list kernel for pairs whose Hamming distance is below the threshold
// =================================================================================================
namespace {
struct __align__(8) GateDev {
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
// stereoTriangulate (ProbabilisticStereoTriangulator.cpp:168-227) -> triangulateFast (stereo_triangulation.cpp:51-125):
// the return value is stereoTriangulate's; hpA and isParallel are set whenever it returns true.  Used by the 2D-2D gate
// and by setBestMatch's re-triangulation in k_stereo_apply.
__device__ __forceinline__ bool stereo_triangulate(const GateDev& g, int a, int b, double* hpA, bool& isParallel) {
  {
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
    if (!(fabs(det) > 1.0e-6)) {
      isParallel = true;
      double c[3];
      cross3(e1, e2, c);
      if (!(sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]) < 6 * sigma)) return false;
      const double v[4] = {(e1[0] + e2[0]) / 2.0, (e1[1] + e2[1]) / 2.0, (e1[2] + e2[2]) / 2.0, 1e-3};
      const double n = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3]);
      hpA[0] = v[0] / n; hpA[1] = v[1] / n; hpA[2] = v[2] / n; hpA[3] = v[3] / n;
    } else {
      isParallel = false;
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
}
__device__ bool gate_verify(const GateDev& g, int a, int b) {
  if (g.mode == OKB_GATE_2D2D) {
    double hpA[4];
    bool isParallel;
    return stereo_triangulate(g, a, b, hpA, isParallel);
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

// One match of a matcher launch (device table, one entry per job); pointers into the launch's staging mirror.  The
// gate sits in the entry itself (last, so that a plain job's kernel copies only the words before it).
struct __align__(8) MatchJobDev {
  const uint32_t *A, *B;
  const uint8_t *skipA, *skipB;    // may be null
  okb_pair *topk, *pairs;
  uint8_t* done;                   // [nA] k_assign scratch
  int nA, nB, num_best, in_smem;   // in_smem: k_assign keeps the per-B winners in shared memory
  float list_thr, gate_thr;
  GateDev gate;                    // gated jobs only
};

// Warp per A descriptor.  Every lane computes the Hamming distance (XOR + __popc over NW words) of A to one of 32
// consecutive B descriptors, staged tile by tile in shared memory for the CTA's 8 warps; the top-`num_best` list of
// DenseMatcher::listBIteration (implementation/DenseMatcher.hpp:137-225) is kept replicated in the warp and updated
// with exactly the reference's sequential rule -- candidates are taken in ascending B order (lowest set bit of the
// ballot first), a candidate enters only if it beats the CURRENT worst entry (re-voted after every insertion, the
// worst only shrinks), std::lower_bound position, i.e. before entries of equal distance.
// blockIdx.y is the job; the grid covers the largest nA of the launch and CTAs past their job's nA exit.
template <int NW, bool GATED>
__global__ void __launch_bounds__(MT, GATED ? (NW == 32 ? 1 : 2) : (NW <= 16 ? 3 : 2)) k_hamming_topk(const MatchJobDev* __restrict__ jobs) {
  __shared__ uint32_t sB[MB_TILE][NW + 1];
  __shared__ uint8_t sSkip[MB_TILE];
  if ((int)blockIdx.x * MW >= jobs[blockIdx.y].nA) return;
  // the job, gate included, is staged in shared memory once: its fields are then read where they are used, from fixed
  // shared addresses, rather than held in registers across the loop
  __shared__ MatchJobDev J;
  constexpr int words = (GATED ? sizeof(MatchJobDev) : offsetof(MatchJobDev, gate)) / 8;
  static_assert(words <= MT, "one word per thread");
  if (threadIdx.x < words)
    reinterpret_cast<unsigned long long*>(&J)[threadIdx.x] = reinterpret_cast<const unsigned long long*>(jobs + blockIdx.y)[threadIdx.x];
  __syncthreads();
  const uint32_t* const& A = J.A;
  const uint32_t* const& B = J.B;
  const uint8_t* const& skipA = J.skipA;
  const uint8_t* const& skipB = J.skipB;
  okb_pair* const& topk = J.topk;

  const int &nA = J.nA, &nB = J.nB, &num_best = J.num_best;
  const float &list_thr = J.list_thr, &gate_thr = J.gate_thr;
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
        if (GATED) t = (t < gate_thr && gate_verify(J.gate, a, b0 + j)) ? t : 3.402823466e+38f;
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
#pragma unroll
    for (int k = 0; k < MAX_BEST; ++k) {
      if (k >= num_best) break;
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
// One CTA per job (blockIdx.x).
constexpr int AS_T = 256, AS_CHUNK = 256;
__global__ void __launch_bounds__(AS_T) k_assign(const MatchJobDev* __restrict__ jobs) {
  const MatchJobDev& J = jobs[blockIdx.x];
  const okb_pair* __restrict__ topk = J.topk;
  const uint8_t* __restrict__ skipA = J.skipA;
  okb_pair* pairs = J.pairs;
  uint8_t* done = J.done;
  const int nA = J.nA, nB = J.nB, num_best = J.num_best, in_smem = J.in_smem;
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
    const int ex = block_scan<1024>(v, s_warp, &total);
    if (i < n) row_ptr[i] = (uint32_t)(run + ex);
    run += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) row_ptr[n] = (uint32_t)run;
}

// k_assign's dynamic shared memory over one call: the staged top-k lists, and the per-B winners and list counts of every
// job whose winners fit beside them (fit() decides the job's in_smem).  set_attribute() runs once per call: it raises
// the kernel's limit to the largest size any launch asks for, so that concurrent calls never lower it under each other.
struct AssignSmem {
  static constexpr size_t kTop = sizeof(okb_pair) * (size_t)AS_CHUNK * MAX_BEST;
  size_t bytes = kTop;
  void fit(const okb_ctx* c, MatchJobDev& jd) {
    const size_t need = kTop + (sizeof(okb_pair) + sizeof(int)) * (size_t)jd.nB;
    jd.in_smem = need + 1024 <= (size_t)c->smem_optin ? 1 : 0;
    if (jd.in_smem) bytes = std::max(bytes, need);
  }
  int set_attribute(okb_ctx* c) const {
    if (bytes > 48 * 1024 - 512) OKB_CUDA(c, cudaFuncSetAttribute(k_assign, cudaFuncAttributeMaxDynamicSharedMemorySize, c->smem_optin - 1024));
    return OKB_OK;
  }
};

// Offsets of a store-backed match's arrays in the call's device scratch (carve_match lays them out).
struct MatchScratch { size_t topk, pairs, skipA, skipB, done; };
}  // namespace

#define DISPATCH_NW(nw, CALL)                 \
  switch (nw) {                               \
    case 8: { constexpr int NW = 8; CALL; } break;   \
    case 12: { constexpr int NW = 12; CALL; } break; \
    case 16: { constexpr int NW = 16; CALL; } break; \
    case 32: { constexpr int NW = 32; CALL; } break; \
    default: c->set_error("descriptor length must be 32, 48, 64 or 128 bytes"); return OKB_ERR_UNSUPPORTED; \
  }

// The matcher over device table d_tab: n[0] plain jobs, then n[1] gated ones.  One k_hamming_topk<NW, GATED> launch per
// kind present, its grid covering the kind's largest nA (max_a), then one k_assign over all of them.
static int launch_matcher(okb_ctx* c, cudaStream_t st, const MatchJobDev* d_tab, int nw, const int n[2], const int max_a[2],
                          const AssignSmem& sm) {
  auto grid = [&](int kind) { return dim3(std::max(1, (max_a[kind] + MW - 1) / MW), n[kind]); };
  if (n[0]) DISPATCH_NW(nw, (k_hamming_topk<NW, false><<<grid(0), MT, 0, st>>>(d_tab)));
  if (n[1]) DISPATCH_NW(nw, (k_hamming_topk<NW, true><<<grid(1), MT, 0, st>>>(d_tab + n[0])));
  k_assign<<<n[0] + n[1], AS_T, sm.bytes, st>>>(d_tab);
  c->frontend->launches += (n[0] > 0) + (n[1] > 0) + 1;
  return OKB_OK;
}

static MatchScratch carve_match(Carve& sc, size_t nA, size_t nB, int num_best) {
  MatchScratch m;
  m.topk = sc.take(sizeof(okb_pair) * nA * num_best);
  m.pairs = sc.take(sizeof(okb_pair) * nB);
  m.skipA = sc.take(nA);
  m.skipB = sc.take(nB);
  m.done = sc.take(nA);
  return m;
}

// The matcher entry of a job on a window's feature store: A and B are store images ia and ib (feature slot * C + camera)
// with nA and nB keypoints, B's keypoints feed the gate, the arrays lie at m in the device scratch sc, and both
// thresholds are `threshold` (the Frontend's matcher makes no ratio test).  The caller sets the gate's mode and the
// rest of its arrays.
static MatchJobDev store_match_job(const okb_ctx* c, const FeatStore& FS, size_t ia, size_t ib, int nA, int nB, int num_best,
                                   float threshold, uint8_t* sc, const MatchScratch& m, AssignSmem& sm) {
  MatchJobDev jd;
  std::memset(&jd, 0, sizeof jd);
  jd.A = FS.desc + ia * FS.N * (FS.D / 4);
  jd.B = FS.desc + ib * FS.N * (FS.D / 4);
  jd.skipA = sc + m.skipA;
  jd.skipB = sc + m.skipB;
  jd.topk = reinterpret_cast<okb_pair*>(sc + m.topk);
  jd.pairs = reinterpret_cast<okb_pair*>(sc + m.pairs);
  jd.done = sc + m.done;
  jd.nA = nA; jd.nB = nB; jd.num_best = num_best;
  jd.list_thr = threshold; jd.gate_thr = threshold;
  jd.gate.kp_b = FS.kp + 2 * ib * FS.N;
  jd.gate.kp_size_b = FS.size + ib * FS.N;
  sm.fit(c, jd);
  return jd;
}

static int upload_descriptors(okb_ctx* c, okb_frontend_state* F, const uint8_t* A, int nA, const uint8_t* B, int nB, int bytes,
                              const uint8_t* skipA, const uint8_t* skipB) {
  int rc;
  if ((rc = grow(c, &F->d_A, &F->capA, (size_t)nA * bytes + nA))) return rc;
  if ((rc = grow(c, &F->d_B, &F->capB, (size_t)nB * bytes + nB))) return rc;
  OKB_CUDA(c, cudaMemcpyAsync(F->d_A, A, (size_t)nA * bytes, cudaMemcpyHostToDevice, c->stream));
  OKB_CUDA(c, cudaMemcpyAsync(F->d_B, B, (size_t)nB * bytes, cudaMemcpyHostToDevice, c->stream));
  if (skipA) OKB_CUDA(c, cudaMemcpyAsync(F->d_A + (size_t)nA * bytes, skipA, nA, cudaMemcpyHostToDevice, c->stream));
  if (skipB) OKB_CUDA(c, cudaMemcpyAsync(F->d_B + (size_t)nB * bytes, skipB, nB, cudaMemcpyHostToDevice, c->stream));
  return OKB_OK;
}

// The single call's argument checks, for one job.
static int match_job_check(okb_ctx* c, const okb_match_job& j, int desc_bytes) {
  if (j.nA < 0 || j.nB < 0 || j.num_best < 1 || j.num_best > MAX_BEST || (j.nB > 0 && !j.out_pairs)) return OKB_ERR_INVALID_ARG;
  if (j.nA == 0 || j.nB == 0) return OKB_OK;
  if (!j.A || !j.B) return OKB_ERR_INVALID_ARG;
  if (desc_bytes % 4) { c->set_error("descriptor length must be a multiple of 4"); return OKB_ERR_UNSUPPORTED; }
  const okb_match_gate* gate = j.gate;
  const int mode = gate ? gate->mode : OKB_GATE_NONE;
  if (mode != OKB_GATE_NONE && mode != OKB_GATE_3D2D && mode != OKB_GATE_2D2D) return OKB_ERR_INVALID_ARG;
  if (mode != OKB_GATE_NONE && (!gate->kp_b || !gate->kp_size_b)) return OKB_ERR_INVALID_ARG;
  if (mode == OKB_GATE_3D2D && (!gate->proj_into_b || !gate->proj_uncertainty)) return OKB_ERR_INVALID_ARG;
  if (mode == OKB_GATE_2D2D && (!gate->kp_a || !gate->kp_size_a || !gate->bearing_a || !gate->bearing_b || !gate->ray_sigma_a || !gate->ray_sigma_b))
    return OKB_ERR_INVALID_ARG;
  return OKB_OK;
}

// n matches on stream `st` through staging buffers io: one pinned staging buffer, one copy in, one copy out:
//   [job table (gates included) | per job: A | B | skipA | skipB | gate arrays]  ...  [per job: top-k lists | winners] [per job: scratch]
// Plain jobs come first in the table, gated ones after them: one k_hamming_topk launch per kind, one k_assign launch.
static int match_run(okb_ctx* c, CallBuffers& io, cudaStream_t st, int n, const okb_match_job* jobs, int desc_bytes) {
  int rc;
  bool any = false;
  for (int i = 0; i < n; ++i) {
    if ((rc = match_job_check(c, jobs[i], desc_bytes))) return rc;
    any = any || (jobs[i].nA > 0 && jobs[i].nB > 0);
  }
  const int nw = desc_bytes / 4;
  if (any && nw != 8 && nw != 12 && nw != 16 && nw != 32) { c->set_error("descriptor length must be 32, 48, 64 or 128 bytes"); return OKB_ERR_UNSUPPORTED; }
  std::vector<int> order;            // jobs with device work: plain, then gated
  for (int pass = 0; pass < 2; ++pass)
    for (int i = 0; i < n; ++i) {
      const okb_match_job& j = jobs[i];
      if (j.nA == 0 || j.nB == 0) {
        if (pass) continue;
        // an empty list matches nothing (DenseMatcher::match on an empty MatchingAlgorithm): no device work
        for (int b = 0; b < j.nB; ++b) { j.out_pairs[b].index_a = -1; j.out_pairs[b].distance = j.threshold; }
        if (j.out_topk) for (size_t k = 0; k < (size_t)j.nA * j.num_best; ++k) { j.out_topk[k].index_a = -1; j.out_topk[k].distance = j.threshold; }
        continue;
      }
      const bool gated = j.gate && j.gate->mode != OKB_GATE_NONE;
      if (gated == (pass == 1)) order.push_back(i);
    }
  const int nd = (int)order.size();
  if (nd == 0) return OKB_OK;
  struct Lay { size_t oA, oB, oSA, oSB, g_kpb, g_szb, g_proj, g_unc, g_kpa, g_sza, g_ba, g_bb, g_rsa, g_rsb, oT, oP, oD; };
  std::vector<Lay> L(nd);
  Carve q;
  q.take(sizeof(MatchJobDev) * nd, 256);
  for (int t = 0; t < nd; ++t) {
    const okb_match_job& j = jobs[order[t]];
    const size_t nA = j.nA, nB = j.nB;
    Lay& l = L[t];
    l.oA = q.take(nA * desc_bytes); l.oB = q.take(nB * desc_bytes); l.oSA = q.take(nA); l.oSB = q.take(nB);
    if (j.gate && j.gate->mode != OKB_GATE_NONE) {      // gate arrays (doubles)
      l.g_kpb = q.take(16 * nB); l.g_szb = q.take(8 * nB); l.g_proj = q.take(16 * nA); l.g_unc = q.take(32 * nA);
      l.g_kpa = q.take(16 * nA); l.g_sza = q.take(8 * nA); l.g_ba = q.take(24 * nA); l.g_bb = q.take(24 * nB);
      l.g_rsa = q.take(8 * nA); l.g_rsb = q.take(8 * nB);
    }
  }
  const size_t in_bytes = q.off;
  for (int t = 0; t < nd; ++t) {
    const okb_match_job& j = jobs[order[t]];
    L[t].oT = q.take(sizeof(okb_pair) * (size_t)j.nA * j.num_best);
    L[t].oP = q.take(sizeof(okb_pair) * (size_t)j.nB);
  }
  const size_t out_end = q.off;
  for (int t = 0; t < nd; ++t) L[t].oD = q.take((size_t)jobs[order[t]].nA);
  if ((rc = io.reserve(c, q.off, 0))) return rc;
  uint8_t* h = io.h_stage;
  uint8_t* d = io.d_stage;
  AssignSmem sm;
  int maxA[2] = {0, 0}, nkind[2] = {0, 0};
  MatchJobDev* tab = reinterpret_cast<MatchJobDev*>(h);
  for (int t = 0; t < nd; ++t) {
    const okb_match_job& j = jobs[order[t]];
    const Lay& l = L[t];
    const int mode = j.gate ? j.gate->mode : OKB_GATE_NONE;
    std::memcpy(h + l.oA, j.A, (size_t)j.nA * desc_bytes);
    std::memcpy(h + l.oB, j.B, (size_t)j.nB * desc_bytes);
    if (j.skipA) std::memcpy(h + l.oSA, j.skipA, j.nA);
    if (j.skipB) std::memcpy(h + l.oSB, j.skipB, j.nB);
    MatchJobDev jd;
    std::memset(&jd, 0, sizeof jd);
    jd.A = reinterpret_cast<const uint32_t*>(d + l.oA);
    jd.B = reinterpret_cast<const uint32_t*>(d + l.oB);
    jd.skipA = j.skipA ? d + l.oSA : nullptr;
    jd.skipB = j.skipB ? d + l.oSB : nullptr;
    jd.topk = reinterpret_cast<okb_pair*>(d + l.oT);
    jd.pairs = reinterpret_cast<okb_pair*>(d + l.oP);
    jd.done = d + l.oD;
    jd.nA = j.nA; jd.nB = j.nB; jd.num_best = j.num_best;
    // DenseMatcher.hpp(impl):188-193: with the ratio test the lists are built without a threshold
    jd.list_thr = j.use_ratio ? 3.402823466e+38f : j.threshold;
    jd.gate_thr = mode == OKB_GATE_NONE ? 0.f : j.threshold;
    sm.fit(c, jd);
    if (mode != OKB_GATE_NONE) {
      const okb_match_gate* gate = j.gate;
      GateDev gd;
      std::memset(&gd, 0, sizeof gd);
      gd.mode = mode;
      auto put = [&](size_t o, const double* src, size_t cnt) -> const double* {
        if (src) std::memcpy(h + o, src, 8 * cnt);
        return reinterpret_cast<const double*>(d + o);
      };
      const size_t nA = j.nA, nB = j.nB;
      gd.kp_b = put(l.g_kpb, gate->kp_b, 2 * nB); gd.kp_size_b = put(l.g_szb, gate->kp_size_b, nB);
      if (mode == OKB_GATE_3D2D) { gd.proj_into_b = put(l.g_proj, gate->proj_into_b, 2 * nA); gd.proj_unc = put(l.g_unc, gate->proj_uncertainty, 4 * nA); }
      else {
        gd.kp_a = put(l.g_kpa, gate->kp_a, 2 * nA); gd.kp_size_a = put(l.g_sza, gate->kp_size_a, nA);
        gd.bearing_a = put(l.g_ba, gate->bearing_a, 3 * nA); gd.bearing_b = put(l.g_bb, gate->bearing_b, 3 * nB);
        gd.ray_sigma_a = put(l.g_rsa, gate->ray_sigma_a, nA); gd.ray_sigma_b = put(l.g_rsb, gate->ray_sigma_b, nB);
        cam_load(gate->cam_a, gd.cam_a); cam_load(gate->cam_b, gd.cam_b);
        gd.wa = gate->cam_a.width; gd.ha = gate->cam_a.height; gd.wb = gate->cam_b.width; gd.hb = gate->cam_b.height;
        double q[4] = {gate->T_AB[3], gate->T_AB[4], gate->T_AB[5], gate->T_AB[6]};
        qnormalize(q);
        q2R(q, gd.R_AB);
        gd.t_AB[0] = gate->T_AB[0]; gd.t_AB[1] = gate->T_AB[1]; gd.t_AB[2] = gate->T_AB[2];
      }
      jd.gate = gd;
    }
    tab[t] = jd;
    const int kind = mode == OKB_GATE_NONE ? 0 : 1;
    maxA[kind] = std::max(maxA[kind], j.nA);
    ++nkind[kind];
  }
  OKB_CUDA(c, cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, st));
  if ((rc = sm.set_attribute(c)) || (rc = launch_matcher(c, st, reinterpret_cast<const MatchJobDev*>(d), nw, nkind, maxA, sm)))
    return rc;
  OKB_CUDA(c, cudaGetLastError());
  OKB_CUDA(c, cudaMemcpyAsync(h + in_bytes, d + in_bytes, out_end - in_bytes, cudaMemcpyDeviceToHost, st));
  OKB_CUDA(c, cudaStreamSynchronize(st));
  for (int t = 0; t < nd; ++t) {
    const okb_match_job& j = jobs[order[t]];
    if (j.out_topk) std::memcpy(j.out_topk, h + L[t].oT, sizeof(okb_pair) * (size_t)j.nA * j.num_best);
    std::memcpy(j.out_pairs, h + L[t].oP, sizeof(okb_pair) * (size_t)j.nB);
  }
  return OKB_OK;
}

static int hamming_match_single(okb_ctx* c, const uint8_t* A, int nA, const uint8_t* B, int nB, int desc_bytes, const uint8_t* skipA,
                                const uint8_t* skipB, float threshold, int num_best, int use_ratio, const okb_match_gate* gate,
                                okb_pair* out_topk, okb_pair* out_pairs) {
  if (!c) return OKB_ERR_INVALID_ARG;
  okb_match_job j;
  std::memset(&j, 0, sizeof j);
  j.A = A; j.B = B; j.skipA = skipA; j.skipB = skipB;
  j.nA = nA; j.nB = nB; j.threshold = threshold; j.num_best = num_best; j.use_ratio = use_ratio;
  j.gate = gate; j.out_topk = out_topk; j.out_pairs = out_pairs;
  const int rc = match_job_check(c, j, desc_bytes);
  if (rc) return rc;
  cudaSetDevice(c->device);
  okb_frontend_state* F = fe(c);
  std::lock_guard<std::mutex> lk(F->match_mtx);
  return match_run(c, F->match_io, c->stream, 1, &j, desc_bytes);
}

extern "C" int okb_hamming_match(okb_ctx* c, const uint8_t* A, int nA, const uint8_t* B, int nB, int desc_bytes, const uint8_t* skipA,
                                 const uint8_t* skipB, float threshold, int num_best, int use_ratio, float ratio_threshold,
                                 okb_pair* out_topk, okb_pair* out_pairs) {
  (void)ratio_threshold;   // the ratio test itself belongs to the serial epilogue on the caller's side
  return hamming_match_single(c, A, nA, B, nB, desc_bytes, skipA, skipB, threshold, num_best, use_ratio, nullptr, out_topk, out_pairs);
}

extern "C" int okb_hamming_match_gated(okb_ctx* c, const uint8_t* A, int nA, const uint8_t* B, int nB, int desc_bytes, const uint8_t* skipA,
                                       const uint8_t* skipB, float threshold, int num_best, int use_ratio, float ratio_threshold,
                                       const okb_match_gate* gate, okb_pair* out_topk, okb_pair* out_pairs) {
  (void)ratio_threshold;
  if (!gate) return OKB_ERR_INVALID_ARG;
  return hamming_match_single(c, A, nA, B, nB, desc_bytes, skipA, skipB, threshold, num_best, use_ratio, gate, out_topk, out_pairs);
}

extern "C" int okb_hamming_match_batch(okb_ctx* c, int n_jobs, const okb_match_job* jobs, int desc_bytes) {
  if (!c || n_jobs < 0) return OKB_ERR_INVALID_ARG;
  if (n_jobs == 0) return OKB_OK;
  if (n_jobs > 65535 || !jobs) return OKB_ERR_INVALID_ARG;        // the job index is a grid dimension
  cudaSetDevice(c->device);
  okb_frontend_state* F = fe(c);
  std::lock_guard<std::mutex> lk(F->batch_mtx);
  if (!F->batch_stream) OKB_CUDA(c, cudaStreamCreateWithFlags(&F->batch_stream, cudaStreamNonBlocking));
  return match_run(c, F->batch_match, F->batch_stream, n_jobs, jobs, desc_bytes);
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
  F->launches += 3;
  OKB_CUDA(c, cudaGetLastError());
  OKB_CUDA(c, cudaMemcpyAsync(row_ptr, F->d_rowptr, sizeof(uint32_t) * (nA + 1), cudaMemcpyDeviceToHost, c->stream));
  OKB_CUDA(c, cudaStreamSynchronize(c->stream));
  const uint32_t total = row_ptr[nA];
  const uint32_t ncopy = std::min<uint32_t>(total, (uint32_t)cap);
  if (ncopy && col_idx) OKB_CUDA(c, cudaMemcpyAsync(col_idx, F->d_col, sizeof(uint32_t) * ncopy, cudaMemcpyDeviceToHost, c->stream));
  if (ncopy && dist) OKB_CUDA(c, cudaMemcpyAsync(dist, F->d_dist, sizeof(uint16_t) * ncopy, cudaMemcpyDeviceToHost, c->stream));
  OKB_CUDA(c, cudaStreamSynchronize(c->stream));
  if (total > (uint32_t)cap) { c->set_error("candidate capacity too small"); return OKB_ERR_CAPACITY; }
  return OKB_OK;
}

// =================================================================================================
// 3D-2D tracking against resident windows (okb_track_3d2d_batch): the 3D-2D rounds of Frontend::matchToKeyframes
// (okvis_frontend/src/Frontend.cpp:389-411) and matchToLastFrame (:484-494) on the window's feature store.  Per round,
// for all jobs of the call at once:
//   k_track_setup   VioKeyframeWindowMatchingAlgorithm::doSetup (VioKeyframeWindowMatchingAlgorithm.cpp:122-215, 238-255)
//   k_hamming_topk<NW, true> + k_assign   DenseMatcher::match over verifyMatch's gate (the matcher kernels above, unchanged)
//   k_track_apply   setBestMatch, 3D-2D branch (:483-526)
// The setup of round r+1 reads what the apply of round r wrote -- B's landmark references and observed bits, the raised
// observation counts, the cleared initialised flags, and, in a same-frame stereo round, A's own entries -- so the rounds
// are launched in sequence on one stream with no host synchronisation between them.  Setup and apply run one CTA per
// job: a round's work per A keypoint is one projection, and the flag clearing and the result list need the
// reference's order within the job.
// =================================================================================================
namespace {
// One job of a launch (device table, in the order of decreasing round count, so that the jobs of round r are a prefix).
struct TrackJobDev {
  const WinDev* W;
  int pose_b, sb_b, feat_b, n_rounds;
  float threshold;
  int cnt_cap;
  int* cnt;                 // [cnt_cap] observations per landmark slot, raised by every accepted match
  int* hdr;                 // [2 n_rounds + 2] numMatches / numUncertainMatches per round, associations, cleared flags
  uint2* assoc;             // {kp_b | round << 16 | cam_b << 24 | uncertain << 31, landmark slot}
  uint32_t* uninit;
};
struct TrackRoundDev { int feat_a, cam_a, cam_b, _pad; };

// Landmark replica of a sharded window (ShardLmAux, okb_estimator.cuh): one half of rank `rank`'s replica, points
// [lm_cap][4] then ShardLmAux [lm_cap].
struct ShardLmHalf { double* x; ShardLmAux* aux; };
__device__ __forceinline__ ShardLmHalf shard_lm_half(const WinDev& W, int rank, int par) {
  unsigned char* h = W.shard_mail[rank] + shard_lm_offset(W.shard_world, W.shard_box_cap, W.shard_marg_cap) +
                     (size_t)par * shard_lm_half_bytes(W.shard_lm_cap);
  return ShardLmHalf{reinterpret_cast<double*>(h), reinterpret_cast<ShardLmAux*>(h + 32 * (size_t)W.shard_lm_cap)};
}
__device__ __forceinline__ unsigned long long shard_lm_epoch(const WinDev& W) {
  return *reinterpret_cast<const unsigned long long*>(W.shard_mail[W.shard_rank] + kShardLmEpoch);
}
// the half of this rank's replica the current call reads (the last exchange's)
__device__ __forceinline__ ShardLmHalf shard_lm_replica(const WinDev& W) { return shard_lm_half(W, W.shard_rank, (int)(shard_lm_epoch(W) & 1ull)); }

// Per-landmark state the store kernels read, through one indexed read selected by the window: its own graph, or on a
// landmark-sharded window the replica all-gathered at the start of the call (k_shard_lm_* below), indexed by the global
// slots the replicated store names.
__device__ __forceinline__ bool lm_sharded(const WinDev& W) { return W.shard_world > 1; }
// landmark slots the call may name: the graph's, or the replica's global slots
__device__ __forceinline__ int lm_slots(const WinDev& W) { return lm_sharded(W) ? W.shard_lm_cap : W.st->g.L; }
// homogeneous point of slot l < lm_slots(W) (32-byte aligned)
__device__ __forceinline__ const double* lm_point(const WinDev& W, int l) {
  return (lm_sharded(W) ? shard_lm_replica(W).x : W.m_lm) + 4 * (size_t)l;
}
// Estimator::isLandmarkInitialized of slot l
__device__ __forceinline__ bool lm_initialised(const WinDev& W, const FeatStore& F, int l) {
  return lm_sharded(W) ? shard_lm_replica(W).aux[l].init != 0 : (l < F.lm_cap && F.lm_init[l]);
}
// Estimator::setLandmarkInitialized(false) on slot l, initialised before: sharded, in the replica of every rank (each
// clears it in its own) and in the owner's shard at its local slot
__device__ __forceinline__ void lm_clear_initialised(const WinDev& W, const FeatStore& F, int l) {
  if (!lm_sharded(W)) { F.lm_init[l] = 0; return; }
  shard_lm_replica(W).aux[l].init = 0;
  if (l % W.shard_world == W.shard_rank && l / W.shard_world < F.lm_cap) F.lm_init[l / W.shard_world] &= 2;
}
// observations per landmark slot into cnt[0, L) (cnt zeroed by the caller, all threads of the CTA take part)
template <int NT>
__device__ __forceinline__ void lm_count_obs(const WinDev& W, int* cnt, int L) {
  if (lm_sharded(W)) {
    const ShardLmAux* aux = shard_lm_replica(W).aux;
    for (int i = threadIdx.x; i < L; i += NT) cnt[i] = aux[i].n_obs;
    return;
  }
  const int n_obs = W.st->g.n_obs;
  for (int i = threadIdx.x; i < n_obs; i += NT) {
    const okb_observation& ob = W.m_obs[i];
    if (ob.sqrt_info != 0.0 && (int)ob.lm_idx < L) atomicAdd(&cnt[ob.lm_idx], 1);
  }
}

// ---- landmark exchange of a sharded window, at the start of a call that reads landmark state (track, 2D-2D, stereo
// initialisation, RANSAC 3D-2D).  Every rank writes the records of the global slots it owns (g = rank + i * world,
// local slot i) into its own replica half of the new epoch's parity and counts their observations there, then pushes
// those records with plain stores into the same half of every peer's replica and releases its flag in every peer's
// mailbox header (st.release.sys), as k_shard_push does for the solver.  k_shard_lm_wait acquires the `world` flags of
// the epoch, or reports status 7 after kShardTimeoutNs; on success k_shard_lm_forget clears, on every rank alike, the
// store references to slots the owners removed since the last exchange.
__device__ __forceinline__ int shard_lm_owned(const WinDev& W) {
  return W.shard_lm_cap > W.shard_rank ? (W.shard_lm_cap - W.shard_rank + W.shard_world - 1) / W.shard_world : 0;
}

__global__ void __launch_bounds__(256) k_shard_lm_own(const WinDev* __restrict__ Wp) {
  const WinDev& W = *Wp;
  const FeatStore& F = *W.feat;
  const ShardLmHalf rep = shard_lm_half(W, W.shard_rank, (int)((shard_lm_epoch(W) + 1ull) & 1ull));
  const int n = shard_lm_owned(W), L = W.st->g.L;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const size_t g = W.shard_rank + (size_t)i * W.shard_world;
    *reinterpret_cast<double4*>(rep.x + 4 * g) = i < L ? *reinterpret_cast<const double4*>(W.m_lm + 4 * (size_t)i) : make_double4(0, 0, 0, 0);
    const uint8_t v = i < F.lm_cap ? F.lm_init[i] : 0;
    ShardLmAux a;
    a.n_obs = 0; a.init = v & 1; a.removed = v >> 1; a._pad[0] = a._pad[1] = 0;
    rep.aux[g] = a;
    if (v & 2) F.lm_init[i] = v & 1;             // the mark is taken: every rank forgets the slot's references
  }
}

__global__ void __launch_bounds__(256) k_shard_lm_count(const WinDev* __restrict__ Wp) {
  const WinDev& W = *Wp;
  ShardLmAux* aux = shard_lm_half(W, W.shard_rank, (int)((shard_lm_epoch(W) + 1ull) & 1ull)).aux;
  const int n_obs = W.st->g.n_obs, L = min(W.st->g.L, shard_lm_owned(W));
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_obs; i += gridDim.x * blockDim.x) {
    const okb_observation& ob = W.m_obs[i];
    if (ob.sqrt_info != 0.0 && (int)ob.lm_idx < L) atomicAdd(&aux[W.shard_rank + (size_t)ob.lm_idx * W.shard_world].n_obs, 1);
  }
}

__global__ void __launch_bounds__(256) k_shard_lm_push(const WinDev* __restrict__ Wp) {
  const WinDev& W = *Wp;
  const int world = W.shard_world, me = W.shard_rank;
  const unsigned long long epoch = shard_lm_epoch(W) + 1ull;
  const int par = (int)(epoch & 1ull), n = shard_lm_owned(W);
  const ShardLmHalf own = shard_lm_half(W, me, par);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const size_t g = me + (size_t)i * world;
    const double4 x = *reinterpret_cast<const double4*>(own.x + 4 * g);
    const ShardLmAux a = own.aux[g];
    for (int q = 0; q < world; ++q)
      if (q != me) {
        const ShardLmHalf dst = shard_lm_half(W, q, par);
        *reinterpret_cast<double4*>(dst.x + 4 * g) = x;
        dst.aux[g] = a;
      }
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int* counter = reinterpret_cast<unsigned int*>(W.shard_mail[me] + kShardLmCounter);
    if (atomicAdd(counter, 1u) == gridDim.x - 1) {
      *counter = 0u;
      __threadfence_system();
      for (int q = 0; q < world; ++q)
        st_release_sys_u64(reinterpret_cast<unsigned long long*>(W.shard_mail[q] + kShardFlagsL) + par * kMaxShard + me, epoch);
    }
  }
}

__global__ void __launch_bounds__(32) k_shard_lm_wait(const WinDev* __restrict__ Wp) {
  const WinDev& W = *Wp;
  unsigned char* box = W.shard_mail[W.shard_rank];
  const unsigned long long epoch = shard_lm_epoch(W) + 1ull;
  const int par = (int)(epoch & 1ull);
  int late = 0;
  if ((int)threadIdx.x < W.shard_world) {
    const unsigned long long* fl = reinterpret_cast<const unsigned long long*>(box + kShardFlagsL) + par * kMaxShard + threadIdx.x;
    const unsigned long long t0 = globaltimer_ns();
    while (ld_acquire_sys_u64(fl) < epoch)
      if (globaltimer_ns() - t0 > kShardTimeoutNs) { late = 1; break; }
  }
  late = __any_sync(0xffffffffu, late);
  if (threadIdx.x == 0) {
    *reinterpret_cast<int*>(box + kShardLmStatus) = late ? 7 : 0;
    *reinterpret_cast<unsigned long long*>(box + kShardLmEpoch) = epoch;
  }
}

__global__ void __launch_bounds__(256) k_shard_lm_forget(const WinDev* __restrict__ Wp) {
  const WinDev& W = *Wp;
  const FeatStore& F = *W.feat;
  const ShardLmAux* aux = shard_lm_replica(W).aux;
  const int n_ent = F.F * F.C * F.N;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n_ent; e += gridDim.x * blockDim.x) {
    const int l = F.lm[e];
    if (l >= 0 && l < W.shard_lm_cap && aux[l].removed) { F.lm[e] = -1; F.observed[e] = 0; }
  }
}

__device__ __forceinline__ bool track_live(const WinDev& W, int L, int l) {
  // a landmark slot is in the graph iff it is below L and its estimate is not the all-zero vector the graph leaves in
  // removed and unused slots (Estimator::isLandmarkAdded)
  if (l < 0 || l >= L) return false;
  const double4 x = *reinterpret_cast<const double4*>(lm_point(W, l));
  return x.x != 0.0 || x.y != 0.0 || x.z != 0.0 || x.w != 0.0;
}

constexpr int TK_T = 256;     // threads of the setup / apply CTAs (the projection chain needs more than 64 registers)

__global__ void __launch_bounds__(TK_T, 1) k_track_setup(const TrackJobDev* __restrict__ jobs, const MatchJobDev* __restrict__ tab,
                                                      const TrackRoundDev* __restrict__ rinfo, int round) {
  __shared__ int s_warp[TK_T / 32];
  __shared__ int s_cand[TK_T];
  const TrackJobDev& J = jobs[blockIdx.x];
  const MatchJobDev& M = tab[blockIdx.x];
  const TrackRoundDev R = rinfo[blockIdx.x];
  const WinDev& W = *J.W;
  const FeatStore& F = *W.feat;
  const int tid = threadIdx.x;
  const int L = min(lm_slots(W), J.cnt_cap);
  if (round == 0) {
    // observation counts of the window (landmark.observations.size()); later rounds see them raised by the matches
    for (int i = tid; i < J.cnt_cap; i += TK_T) J.cnt[i] = 0;
    for (int i = tid; i < 2 * J.n_rounds + 2; i += TK_T) J.hdr[i] = 0;
    __syncthreads();
    lm_count_obs<TK_T>(W, J.cnt, L);
    __syncthreads();
  }
  // skipB (:238-250): B keypoint k refers to a landmark of the graph that already holds this keypoint's observation
  const size_t base_b = ((size_t)J.feat_b * F.C + R.cam_b) * F.N;
  uint8_t* skipB = const_cast<uint8_t*>(M.skipB);
  for (int b = tid; b < M.nB; b += TK_T) skipB[b] = (F.observed[base_b + b] && track_live(W, L, F.lm[base_b + b])) ? 1 : 0;
  // UOplus (:127-142): velocity-scaled position variance when B is in the IMU window and A is another frame, else 4e-8
  // (also the same-frame stereo 3D-2D match of matchStereo, Frontend.cpp:547-553)
  double s = 4e-8;
  if (J.sb_b >= 0 && R.feat_a != J.feat_b) {
    const double* v = W.sb + 9 * (size_t)J.sb_b;
    const double scale = fmax(1.0, sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]));
    s = (scale * scale) * 1.0e-2;
  }
  SlotXf xf;       // T_CbW = (T_WSb T_SbCb)^-1
  make_slot_xf(W.pose + 7 * (size_t)J.pose_b, W.ext + 7 * (size_t)R.cam_b, xf);
  const okb_camera& camB = W.cams[R.cam_b];
  CamIntr cam;
  cam_load(camB, cam);
  const size_t base_a = ((size_t)R.feat_a * F.C + R.cam_a) * F.N;
  uint8_t* skipA = const_cast<uint8_t*>(M.skipA);
  double* proj = const_cast<double*>(M.gate.proj_into_b);
  double* unc = const_cast<double*>(M.gate.proj_unc);
  for (int k0 = 0; k0 < M.nA; k0 += TK_T) {
    const int k = k0 + tid;
    int clear = 0;
    if (k < M.nA) {
      // doSetup for A keypoint k, in the reference's order (:165-215)
      const int l = F.lm[base_a + k];
      bool skip = true;
      if (!track_live(W, L, l)) {                                       // 1. no landmark, or not in the graph
      } else if (!lm_initialised(W, F, l)) {                             // 2. not initialised
      } else {
        const double* X = lm_point(W, l);
        const double w = X[3];
        double pc[3];
        pc[0] = xf.R[0] * X[0] + xf.R[1] * X[1] + xf.R[2] * X[2] + xf.t[0] * w;
        pc[1] = xf.R[3] * X[0] + xf.R[4] * X[1] + xf.R[5] * X[2] + xf.t[1] * w;
        pc[2] = xf.R[6] * X[0] + xf.R[7] * X[1] + xf.R[8] * X[2] + xf.t[2] * w;
        // 3. projectHomogeneous (PinholeCamera.hpp(impl):358-378): w < 0 projects -xyz; Successful = distortion valid,
        //    inside the image, in front of the camera
        if (w < 0) { pc[0] = -pc[0]; pc[1] = -pc[1]; pc[2] = -pc[2]; }
        double ip[2], Jp[6];
        const bool ok = project<true>(cam, pc, ip, Jp) && !(ip[0] < 0.0 || ip[1] < 0.0 || ip[0] >= (double)camB.width ||
                                                           ip[1] >= (double)camB.height) && pc[2] > 0.0;
        if (!ok) {
        } else if (J.cnt[l] < 2) {                                       // 4. after the projection: fewer than 2 observations
          clear = 1;
        } else {                                                         // 5. projectionsIntoB_, J P_C J^T with P_C = s I3
          skip = false;
          proj[2 * k] = ip[0]; proj[2 * k + 1] = ip[1];
          const double a0 = s * Jp[0], a1 = s * Jp[1], a2 = s * Jp[2], b0 = s * Jp[3], b1 = s * Jp[4], b2 = s * Jp[5];
          unc[4 * k] = a0 * Jp[0] + a1 * Jp[1] + a2 * Jp[2];
          unc[4 * k + 1] = a0 * Jp[3] + a1 * Jp[4] + a2 * Jp[5];
          unc[4 * k + 2] = b0 * Jp[0] + b1 * Jp[1] + b2 * Jp[2];
          unc[4 * k + 3] = b0 * Jp[3] + b1 * Jp[4] + b2 * Jp[5];
        }
      }
      skipA[k] = skip ? 1 : 0;
    }
    // setLandmarkInitialized(false) in ascending k: a landmark two keypoints share is cleared (and listed) once
    int total;
    const int pos = block_scan<TK_T>(clear, s_warp, &total);
    if (clear) s_cand[pos] = k;
    __syncthreads();
    if (tid == 0) {
      const int h = 2 * J.n_rounds + 1;
      int n_u = J.hdr[h];
      for (int i = 0; i < total; ++i) {
        const int l = F.lm[base_a + s_cand[i]];
        if (lm_initialised(W, F, l)) { lm_clear_initialised(W, F, l); J.uninit[n_u++] = (uint32_t)l; }
      }
      J.hdr[h] = n_u;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(TK_T) k_track_apply(const TrackJobDev* __restrict__ jobs, const MatchJobDev* __restrict__ tab,
                                                      const TrackRoundDev* __restrict__ rinfo, int round) {
  __shared__ int s_warp[TK_T / 32];
  const TrackJobDev& J = jobs[blockIdx.x];
  const MatchJobDev& M = tab[blockIdx.x];
  const TrackRoundDev R = rinfo[blockIdx.x];
  const FeatStore& F = *J.W->feat;
  const int tid = threadIdx.x;
  const size_t base_a = ((size_t)R.feat_a * F.C + R.cam_a) * F.N;
  const size_t base_b = ((size_t)J.feat_b * F.C + R.cam_b) * F.N;
  const double* proj = M.gate.proj_into_b;
  const double* unc = M.gate.proj_unc;
  int n_assoc = J.hdr[2 * J.n_rounds], n_match = 0, n_unc = 0;
  for (int b0 = 0; b0 < M.nB; b0 += TK_T) {
    const int b = b0 + tid;
    int acc = 0, uncertain = 0, l = -1;
    if (b < M.nB) {
      const okb_pair p = M.pairs[b];
      // DenseMatcher::match calls setBestMatch for every B whose winner is below the threshold, B ascending
      if (p.index_a >= 0 && p.distance < J.threshold) {
        const int a = p.index_a;
        l = F.lm[base_a + a];
        // setBestMatch 3D-2D (:483-526): chi-square again, in double this time (Eigen's 2x2 inverse), > 4 rejects
        const double sd = 0.8 * F.size[base_b + b] / 12.0;
        const double U00 = sd * sd + unc[4 * a], U01 = unc[4 * a + 1], U10 = unc[4 * a + 2], U11 = sd * sd + unc[4 * a + 3];
        const double e0 = proj[2 * a] - F.kp[2 * (base_b + b)], e1 = proj[2 * a + 1] - F.kp[2 * (base_b + b) + 1];
        const double invdet = 1.0 / (U00 * U11 - U10 * U01);
        const double i00 = U11 * invdet, i10 = -U10 * invdet, i01 = -U01 * invdet, i11 = U00 * invdet;
        const double r0 = e0 * i00 + e1 * i10, r1 = e0 * i01 + e1 * i11;
        const double chi2 = r0 * e0 + r1 * e1;
        if (!(chi2 > 4.0)) {
          acc = 1;
          // saturated image uncertainty: counted, not rejected
          const double nrm = sqrt(U00 * U00 + U10 * U10 + U01 * U01 + U11 * U11);
          uncertain = nrm > 25.0 / (sd * sd * sqrt(2.0)) ? 1 : 0;
        }
      }
    }
    int total, total_u;
    const int pos = block_scan<TK_T>(acc, s_warp, &total);
    block_scan<TK_T>(acc & uncertain, s_warp, &total_u);
    if (acc) {
      // B's keypoint takes A's landmark and its observation; the count of the landmark rises for the later rounds
      F.lm[base_b + b] = l;
      F.observed[base_b + b] = 1;
      if (l < J.cnt_cap) atomicAdd(&J.cnt[l], 1);
      J.assoc[n_assoc + pos] = make_uint2((uint32_t)b | ((uint32_t)round << 16) | ((uint32_t)R.cam_b << 24) | ((uint32_t)uncertain << 31),
                                          (uint32_t)l);
    }
    n_assoc += total; n_match += total; n_unc += total_u;
  }
  if (tid == 0) {
    J.hdr[2 * round] = n_match;
    J.hdr[2 * round + 1] = n_unc;
    J.hdr[2 * J.n_rounds] = n_assoc;
  }
}
}  // namespace

// The host checks every job of a call on the feature store makes of its window; "" = valid.
static std::string store_window_invalid(okb_ctx* c, int win, std::vector<char>& seen) {
  if (win < 0 || win >= c->max_windows) return "window slot out of range";
  const WinStore& S = c->wins[win];
  if (!S.uploaded) return "window slot not uploaded";
  if (!S.feat_mem) return "window has no feature store (okb_window_reserve_features)";
  if (seen[win]) return "window listed twice";
  seen[win] = 1;
  return "";
}

// The argument checks of a call `fn` on the feature store, before any device work: an empty call is a no-op (OKB_OK, and
// the caller returns), more than max_jobs jobs and a landmark-sharded context connected without a landmark replica are
// refused, and invalid(i, seen) checks
// job i against the store as the pending commands leave it ("" = valid; the first failure is reported as
// "fn: jobs[i]: why").
template <typename Job, typename Invalid>
static int store_call_checks(okb_ctx* c, const char* fn, int n_jobs, const Job* jobs, int max_jobs, const Invalid& invalid) {
  if (!c || n_jobs < 0 || (n_jobs > 0 && !jobs)) return OKB_ERR_INVALID_ARG;
  if (n_jobs == 0) return OKB_OK;
  if (n_jobs > max_jobs) { c->set_error(std::string(fn) + ": more than " + std::to_string(max_jobs) + " jobs"); return OKB_ERR_INVALID_ARG; }
  if (c->shard_world > 1 && c->shard_lm_cap < 1) {
    c->set_error(std::string(fn) + ": a landmark-sharded context needs its global landmark slots (okb_shard_reserve_landmarks)");
    return OKB_ERR_UNSUPPORTED;
  }
  std::vector<char> seen(c->max_windows, 0);
  for (int i = 0; i < n_jobs; ++i) {
    const std::string why = invalid(i, seen);
    if (!why.empty()) { c->set_error(std::string(fn) + ": jobs[" + std::to_string(i) + "]: " + why); return OKB_ERR_INVALID_ARG; }
  }
  return OKB_OK;
}

// Pending edits of the jobs' windows first (they may be the store edits the call reads), then after the solver work on
// those windows.
template <typename Job>
static int commit_job_windows(okb_ctx* c, const Job* jobs, int n_jobs) {
  std::vector<int32_t> wl(n_jobs);
  for (int i = 0; i < n_jobs; ++i) wl[i] = jobs[i].win;
  return okb_commit_windows(c, wl.data(), n_jobs);
}

// Landmark slots a call names on window `win`: the graph's, or on a landmark-sharded context the replica's global slots.
static int lm_slots_host(const okb_ctx* c, int win) { return c->shard_world > 1 ? c->shard_lm_cap : std::max(c->host[win].L, 1); }

// Landmark-sharded context: the landmark exchange (k_shard_lm_*) of every job window on `xs`, after the commit.  Every
// rank must make the same call; a peer that does not arrive within the time-out fails the call with status 7 before
// any of its own device work, and a window whose shard names global slots beyond the replica is refused.
template <typename Job>
static int shard_lm_exchange(okb_ctx* c, const char* fn, const Job* jobs, int n_jobs, cudaStream_t xs) {
  if (c->shard_world < 2) return OKB_OK;
  for (int i = 0; i < n_jobs; ++i)
    if ((int64_t)(c->host[jobs[i].win].L - 1) * c->shard_world + c->shard_rank >= c->shard_lm_cap) {
      c->set_error(std::string(fn) + ": the shard's landmarks exceed the global landmark slots (okb_shard_reserve_landmarks)");
      return OKB_ERR_CAPACITY;
    }
  const int gx = std::max(1, std::min(c->sm_count, (c->shard_lm_cap / c->shard_world + 255) / 256));
  for (int i = 0; i < n_jobs; ++i) {
    const WinDev* W = c->d_wins + jobs[i].win;
    k_shard_lm_own<<<gx, 256, 0, xs>>>(W);
    k_shard_lm_count<<<gx, 256, 0, xs>>>(W);
    k_shard_lm_push<<<gx, 256, 0, xs>>>(W);
    k_shard_lm_wait<<<1, 32, 0, xs>>>(W);
  }
  fe(c)->launches += 4 * (int64_t)n_jobs;
  OKB_CUDA(c, cudaGetLastError());
  std::vector<int> status(n_jobs, 0);
  for (int i = 0; i < n_jobs; ++i)
    OKB_CUDA(c, cudaMemcpyAsync(&status[i], c->shard_local + (size_t)jobs[i].win * c->shard_win_bytes + kShardLmStatus, sizeof(int),
                                cudaMemcpyDeviceToHost, xs));
  OKB_CUDA(c, cudaStreamSynchronize(xs));
  for (int i = 0; i < n_jobs; ++i)
    if (status[i]) {
      c->set_error(std::string(fn) + ": jobs[" + std::to_string(i) + "]: a peer rank did not arrive at the landmark exchange (status 7)");
      return OKB_ERR_SHARD_TIMEOUT;
    }
  for (int i = 0; i < n_jobs; ++i) {
    const FeatStore& F = c->wins[jobs[i].win].feat;
    const int n = F.F * F.C * F.N;
    k_shard_lm_forget<<<std::max(1, std::min(c->sm_count, (n + 255) / 256)), 256, 0, xs>>>(c->d_wins + jobs[i].win);
  }
  fe(c)->launches += n_jobs;
  OKB_CUDA(c, cudaGetLastError());
  return OKB_OK;
}

// Host checks of one job (first_win: the window of the call's first job, already checked); "" = valid.
static std::string track_job_invalid(okb_ctx* c, const okb_track_job& j, int first_win, std::vector<char>& seen) {
  const std::string why = store_window_invalid(c, j.win, seen);
  if (!why.empty()) return why;
  const WinStore& S = c->wins[j.win];
  const WinDev& W = c->host[j.win];
  const FeatStore& F = S.feat;
  if (F.D != c->wins[first_win].feat.D) return "descriptor length differs from the call's first job";
  if (j.pose_b < 0 || j.pose_b >= W.K) return "pose_b out of range";
  if (j.sb_b < -1 || j.sb_b >= W.NSB) return "sb_b out of range";
  if (j.feat_slot_b < 0 || j.feat_slot_b >= F.F) return "feat_slot_b out of range";
  if (j.num_best < 1 || j.num_best > MAX_BEST) return "num_best out of range (1..8)";
  if (j.n_rounds < 0 || (j.n_rounds > 0 && (!j.rounds || !j.num_matches || !j.num_uncertain))) return "round list or per-round outputs missing";
  if (j.n_rounds > 255) return "more than 255 rounds";
  if (!j.n_assoc || !j.n_uninit) return "n_assoc / n_uninit missing";
  size_t sumA = 0, sumB = 0;
  for (int r = 0; r < j.n_rounds; ++r) {
    const okb_track_round& R = j.rounds[r];
    if (R.feat_slot_a < 0 || R.feat_slot_a >= F.F || R.cam_a < 0 || R.cam_a >= F.C) return "round " + std::to_string(r) + ": frame A out of range";
    if (R.cam_b < 0 || R.cam_b >= F.C || R.cam_b >= W.NC || R.cam_b >= W.NE) return "round " + std::to_string(r) + ": cam_b out of range";
    // the apply kernel writes B's image while it reads A's: one image cannot be both
    if (R.feat_slot_a == j.feat_slot_b && R.cam_a == R.cam_b) return "round " + std::to_string(r) + ": frame B against itself in one camera";
    const int nA = S.feat_n_pending[(size_t)R.feat_slot_a * F.C + R.cam_a], nB = S.feat_n_pending[(size_t)j.feat_slot_b * F.C + R.cam_b];
    if (nA < 0 || nB < 0) return "round " + std::to_string(r) + ": feature slot has no keypoints for the camera";
    sumA += nA; sumB += nB;
  }
  if ((size_t)std::max(j.assoc_cap, 0) < sumB || (sumB && !j.assoc)) return "assoc capacity below the B keypoints of all rounds";
  if ((size_t)std::max(j.uninit_cap, 0) < sumA || (sumA && !j.uninit)) return "uninit capacity below the A keypoints of all rounds";
  return "";
}

extern "C" int okb_track_3d2d_batch(okb_ctx* c, int n_jobs, const okb_track_job* jobs) {
  int rc = store_call_checks(c, "okb_track_3d2d_batch", n_jobs, jobs, 65535, [&](int i, std::vector<char>& seen) {   // grid dimension
    return track_job_invalid(c, jobs[i], jobs[0].win, seen);
  });
  if (rc || n_jobs == 0) return rc;
  cudaSetDevice(c->device);
  okb_frontend_state* F = fe(c);
  CallBuffers& B = F->track;
  std::lock_guard<std::mutex> lk(B.mtx);
  if ((rc = commit_job_windows(c, jobs, n_jobs))) return rc;
  if ((rc = shard_lm_exchange(c, "okb_track_3d2d_batch", jobs, n_jobs, c->stream_xfer))) return rc;
  cudaStream_t xs = c->stream_xfer;
  // jobs by decreasing round count: the jobs of round r are the first m[r]
  std::vector<int> order(n_jobs);
  for (int i = 0; i < n_jobs; ++i) order[i] = i;
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return jobs[a].n_rounds > jobs[b].n_rounds; });
  const int R = jobs[order[0]].n_rounds;
  std::vector<int> m(R, 0);
  for (int i = 0; i < n_jobs; ++i)
    for (int r = 0; r < jobs[i].n_rounds; ++r) ++m[r];
  // staging (pinned + device mirror): in  = [job table | per round: match table | round table]
  //                                   out = [per job: header | associations | cleared slots]
  // scratch (device only), per job: counts; per (job, round): proj | unc | the matcher's arrays
  Carve st, sc;
  st.take(sizeof(TrackJobDev) * n_jobs, 256);
  std::vector<size_t> o_tab(R), o_rinfo(R);
  for (int r = 0; r < R; ++r) { o_tab[r] = st.take(sizeof(MatchJobDev) * m[r]); o_rinfo[r] = st.take(sizeof(TrackRoundDev) * m[r]); }
  const size_t in_bytes = st.off;
  struct RoundLay { int nA, nB; size_t proj, unc; MatchScratch ms; };
  std::vector<RoundLay> rl;                 // per (job, round); job i's rounds from rl[r0[i]]
  std::vector<size_t> o_hdr(n_jobs), o_assoc(n_jobs), o_un(n_jobs), o_cnt(n_jobs), r0(n_jobs);
  for (int i = 0; i < n_jobs; ++i) {
    const okb_track_job& j = jobs[i];
    const WinStore& S = c->wins[j.win];
    r0[i] = rl.size();
    o_cnt[i] = sc.take(4 * (size_t)lm_slots_host(c, j.win));
    size_t sumA = 0, sumB = 0;
    for (int r = 0; r < j.n_rounds; ++r) {
      RoundLay x;
      x.nA = S.feat_n_pending[(size_t)j.rounds[r].feat_slot_a * S.feat.C + j.rounds[r].cam_a];
      x.nB = S.feat_n_pending[(size_t)j.feat_slot_b * S.feat.C + j.rounds[r].cam_b];
      x.proj = sc.take(16 * (size_t)x.nA);
      x.unc = sc.take(32 * (size_t)x.nA);
      x.ms = carve_match(sc, x.nA, x.nB, j.num_best);
      rl.push_back(x);
      sumA += x.nA; sumB += x.nB;
    }
    o_hdr[i] = st.take(4 * (2 * (size_t)j.n_rounds + 2));
    o_assoc[i] = st.take(8 * sumB);
    o_un[i] = st.take(4 * sumA);
  }
  const size_t out_end = st.off;
  if ((rc = B.reserve(c, out_end, sc.off))) return rc;
  uint8_t* h = B.h_stage;
  uint8_t* d = B.d_stage;
  AssignSmem sm;
  std::vector<int> maxA(R, 0);
  TrackJobDev* tj = reinterpret_cast<TrackJobDev*>(h);
  for (int t = 0; t < n_jobs; ++t) {
    const int i = order[t];
    const okb_track_job& j = jobs[i];
    const FeatStore& FS = c->wins[j.win].feat;
    TrackJobDev J;
    std::memset(&J, 0, sizeof J);
    J.W = c->d_wins + j.win;
    J.pose_b = j.pose_b; J.sb_b = j.sb_b; J.feat_b = j.feat_slot_b; J.n_rounds = j.n_rounds;
    J.threshold = j.threshold;
    J.cnt_cap = lm_slots_host(c, j.win);
    J.cnt = reinterpret_cast<int*>(B.d_scratch + o_cnt[i]);
    J.hdr = reinterpret_cast<int*>(d + o_hdr[i]);
    J.assoc = reinterpret_cast<uint2*>(d + o_assoc[i]);
    J.uninit = reinterpret_cast<uint32_t*>(d + o_un[i]);
    tj[t] = J;
    for (int r = 0; r < j.n_rounds; ++r) {
      const okb_track_round& Rr = j.rounds[r];
      const RoundLay& x = rl[r0[i] + r];
      const size_t ia = (size_t)Rr.feat_slot_a * FS.C + Rr.cam_a, ib = (size_t)j.feat_slot_b * FS.C + Rr.cam_b;
      MatchJobDev jd = store_match_job(c, FS, ia, ib, x.nA, x.nB, j.num_best, j.threshold, B.d_scratch, x.ms, sm);
      jd.gate.mode = OKB_GATE_3D2D;
      jd.gate.proj_into_b = reinterpret_cast<const double*>(B.d_scratch + x.proj);
      jd.gate.proj_unc = reinterpret_cast<const double*>(B.d_scratch + x.unc);
      reinterpret_cast<MatchJobDev*>(h + o_tab[r])[t] = jd;
      reinterpret_cast<TrackRoundDev*>(h + o_rinfo[r])[t] = TrackRoundDev{Rr.feat_slot_a, Rr.cam_a, Rr.cam_b, 0};
      maxA[r] = std::max(maxA[r], x.nA);
    }
  }
  OKB_CUDA(c, cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, xs));
  const TrackJobDev* d_jobs = reinterpret_cast<const TrackJobDev*>(d);
  if ((rc = sm.set_attribute(c))) return rc;
  const int nw = c->wins[jobs[0].win].feat.D / 4;
  for (int r = 0; r < R; ++r) {
    const MatchJobDev* d_tab = reinterpret_cast<const MatchJobDev*>(d + o_tab[r]);
    const TrackRoundDev* d_ri = reinterpret_cast<const TrackRoundDev*>(d + o_rinfo[r]);
    const int n[2] = {0, m[r]}, max_a[2] = {0, maxA[r]};
    k_track_setup<<<m[r], TK_T, 0, xs>>>(d_jobs, d_tab, d_ri, r);
    if ((rc = launch_matcher(c, xs, d_tab, nw, n, max_a, sm))) return rc;
    k_track_apply<<<m[r], TK_T, 0, xs>>>(d_jobs, d_tab, d_ri, r);
  }
  F->launches += 2 * (int64_t)R;
  OKB_CUDA(c, cudaGetLastError());
  OKB_CUDA(c, cudaMemcpyAsync(h + in_bytes, d + in_bytes, out_end - in_bytes, cudaMemcpyDeviceToHost, xs));
  OKB_CUDA(c, cudaStreamSynchronize(xs));
  for (int i = 0; i < n_jobs; ++i) {
    const okb_track_job& j = jobs[i];
    if (j.n_rounds == 0) { *j.n_assoc = 0; *j.n_uninit = 0; continue; }
    const int32_t* hd = reinterpret_cast<const int32_t*>(h + o_hdr[i]);
    for (int r = 0; r < j.n_rounds; ++r) { j.num_matches[r] = hd[2 * r]; j.num_uncertain[r] = hd[2 * r + 1]; }
    const int na = hd[2 * j.n_rounds], nu = hd[2 * j.n_rounds + 1];
    *j.n_assoc = na; *j.n_uninit = nu;
    const uint2* as = reinterpret_cast<const uint2*>(h + o_assoc[i]);
    for (int k = 0; k < na; ++k) {
      okb_track_assoc& o = j.assoc[k];
      o.kp_b = (int32_t)(as[k].x & 0xffffu); o.round = (int32_t)((as[k].x >> 16) & 0xffu); o.cam_b = (int32_t)((as[k].x >> 24) & 0x7fu);
      o.uncertain = (int32_t)(as[k].x >> 31); o.lm_slot = (int32_t)as[k].y; o._pad = 0;
    }
    if (nu) std::memcpy(j.uninit, h + o_un[i], 4 * (size_t)nu);
  }
  return OKB_OK;
}

// =================================================================================================
// 2D-2D landmark initialisation (okb_match2d2d_batch): the 2D-2D rounds of Frontend::matchToKeyframes and
// matchToLastFrame (okvis_frontend/src/Frontend.cpp:413-452, 499-509) on the window's feature store, frame A an older
// frame and frame B the current one; okb_stereo_init_batch is its A = B case (the 2D-2D match of Frontend::matchStereo,
// :521-546):
//   k_stereo_setup  setFrames (VioKeyframeWindowMatchingAlgorithm.cpp:76-111) and doSetup's 2D-2D branch (:124-146,
//                   216-232, 256-274): backProject, ray sigmas and skip flags per keypoint, in parallel over (job, image,
//                   keypoint); one thread per job also writes the gate's geometry and resetFrames' prior H_
//   k_hamming_topk<NW, true> + k_assign   DenseMatcher::match over verifyMatch's 2D-2D gate (unchanged)
//   k_stereo_apply  setBestMatch's 2D-2D branch (:370-481) up to the landmark bookkeeping: a thread per B winner for
//                   stereoTriangulate and getUncertainty's residuals, a warp per remaining 9x9 rank test, a CTA scan for
//                   the ascending-B record list
// The call writes nothing but its scratch and its results: the caller applies them.
// =================================================================================================
namespace {
constexpr int kGeo = 7 + 9 + 3 + 36;     // per job: T_CaCb [t, q], C_WCa, r_WCa, H_ (6x6 pose block of resetFrames' prior)
constexpr int kUJ = 6 + 12 + 6;          // per B keypoint: J_hpA_min 2x3, J_TB_min 2x6, J_hpB_min 2x3

struct StereoJobDev {
  const WinDev* W;
  int pose_a, feat_a, cam_a, pose_b, feat_b, cam_b;
  int sb;                   // speed/bias block whose speed scales UOplus' translation part, -1: 4e-8 (same frame, or
                            // the current frame outside the IMU window)
  float threshold;
  double* geo;              // [kGeo]
  double* uj;               // [nB][kUJ] Jacobians of the winners that reach the rank test
  int* n_out;
  okb_stereo_match* out;    // [nB]
};

// okvis::kinematics::Transformation: (r, q) with q normalised on construction, C = q.toRotationMatrix()
struct XfQ { double r[3], q[4], C[9]; };
__device__ void xfq_make(const double* r, const double* q, XfQ& o) {
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
#pragma unroll
  for (int k = 0; k < 4; ++k) o.q[k] = q[k] / n;
#pragma unroll
  for (int k = 0; k < 3; ++k) o.r[k] = r[k];
  q2R(o.q, o.C);
}
__device__ void xfq_mul(const XfQ& a, const XfQ& b, XfQ& o) {      // Transformation(C_a r_b + r_a, q_a q_b)
  double r[3], q[4];
  mat3vec(a.C, b.r, r);
  r[0] += a.r[0]; r[1] += a.r[1]; r[2] += a.r[2];
  qmul(a.q, b.q, q);
  xfq_make(r, q, o);
}
__device__ void xfq_inv(const XfQ& a, XfQ& o) {                    // Transformation(-(C^T r), q.inverse())
  double r[3], q[4];
  mat3Tvec(a.C, a.r, r);
  r[0] = -r[0]; r[1] = -r[1]; r[2] = -r[2];
  const double n2 = a.q[0] * a.q[0] + a.q[1] * a.q[1] + a.q[2] * a.q[2] + a.q[3] * a.q[3];
  q[0] = -a.q[0] / n2; q[1] = -a.q[1] / n2; q[2] = -a.q[2] / n2; q[3] = a.q[3] / n2;
  xfq_make(r, q, o);
}

__global__ void __launch_bounds__(TK_T) k_stereo_setup(const StereoJobDev* __restrict__ jobs, MatchJobDev* tab) {
  const StereoJobDev& J = jobs[blockIdx.y];
  MatchJobDev& M = tab[blockIdx.y];
  const WinDev& W = *J.W;
  const FeatStore& F = *W.feat;
  const int side = blockIdx.z;
  if (blockIdx.x == 0 && side == 0 && threadIdx.x == 0) {
    // setFrames: T_WCa = T_WSa T_SCa, T_WCb = T_WSb T_SCb, T_CaCb = T_WCa^-1 T_WCb
    const double* Pa = W.pose + 7 * (size_t)J.pose_a;
    const double* Pb = W.pose + 7 * (size_t)J.pose_b;
    const double* Ea = W.ext + 7 * (size_t)J.cam_a;
    const double* Eb = W.ext + 7 * (size_t)J.cam_b;
    XfQ T_WSa, T_WSb, T_SCa, T_SCb, T_WCa, T_WCb, T_CaW, T_AB;
    xfq_make(Pa, Pa + 3, T_WSa);
    xfq_make(Pb, Pb + 3, T_WSb);
    xfq_make(Ea, Ea + 3, T_SCa);
    xfq_make(Eb, Eb + 3, T_SCb);
    xfq_mul(T_WSa, T_SCa, T_WCa);
    xfq_mul(T_WSb, T_SCb, T_WCb);
    xfq_inv(T_WCa, T_CaW);
    xfq_mul(T_CaW, T_WCb, T_AB);
    GateDev& g = M.gate;
    cam_load(W.cams[J.cam_a], g.cam_a);
    cam_load(W.cams[J.cam_b], g.cam_b);
    g.wa = W.cams[J.cam_a].width; g.ha = W.cams[J.cam_a].height;
    g.wb = W.cams[J.cam_b].width; g.hb = W.cams[J.cam_b].height;
    for (int k = 0; k < 9; ++k) g.R_AB[k] = T_AB.C[k];
    for (int k = 0; k < 3; ++k) g.t_AB[k] = T_AB.r[k];
    double* geo = J.geo;
    for (int k = 0; k < 3; ++k) geo[k] = T_AB.r[k];
    for (int k = 0; k < 4; ++k) geo[3 + k] = T_AB.q[k];
    for (int k = 0; k < 9; ++k) geo[7 + k] = T_WCa.C[k];
    for (int k = 0; k < 3; ++k) geo[16 + k] = T_WCa.r[k];
    // doSetup's UOplus (:127-142): diag(u I3, 1e-8 I3), u velocity-scaled when the current frame is in the IMU window
    // and A is another frame (the host passes sb = -1 otherwise), else 4e-8.  resetFrames
    // (ProbabilisticStereoTriangulator.cpp:117-159): PoseError(T_AB, UOplus^-1) evaluated at T_AB; H_ = J_min^T J_min in
    // the pose block
    double u = 4e-8;
    if (J.sb >= 0) {
      const double* v = W.sb + 9 * (size_t)J.sb;
      const double scale = fmax(1.0, sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]));
      u = (scale * scale) * 1.0e-2;
    }
    double S[36], r6[6], Jp[36];
    for (int k = 0; k < 36; ++k) S[k] = 0.0;
    for (int k = 0; k < 3; ++k) { S[7 * k] = sqrt(1.0 / u); S[7 * (k + 3)] = sqrt(1.0 / 1e-8); }
    pose_error(geo, S, geo, r6, Jp);
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j < 6; ++j) {
        double s = 0.0;
        for (int k = 0; k < 6; ++k) s += Jp[k * 6 + i] * Jp[k * 6 + j];
        geo[19 + i * 6 + j] = s;
      }
  }
  // doSetup, 2D-2D: per keypoint of (frame A, cam_a) / (frame B, cam_b) the ray sigma, the backProject bearing and
  // skip when it names an initialised landmark of the graph
  const int cam = side ? J.cam_b : J.cam_a;
  const int feat = side ? J.feat_b : J.feat_a;
  const int n = side ? M.nB : M.nA;
  const int k = blockIdx.x * TK_T + threadIdx.x;
  if (k >= n) return;
  const size_t e = ((size_t)feat * F.C + cam) * F.N + k;
  const okb_camera& cm = W.cams[cam];
  CamIntr ci;
  cam_load(cm, ci);
  const double sd = 0.8 * F.size[e] / 12.0;
  double* rs = const_cast<double*>(side ? M.gate.ray_sigma_b : M.gate.ray_sigma_a);
  rs[k] = sqrt(sqrt(2.0)) * sd / ci.fu;
  // PinholeCamera::backProject (PinholeCamera.hpp(impl):426-444): (p - c) * (1 / f), the model's undistort
  double pu[2];
  undistort_gn(ci, (F.kp[2 * e] - ci.cu) * (1.0 / ci.fu), (F.kp[2 * e + 1] - ci.cv) * (1.0 / ci.fv), pu);
  double* br = const_cast<double*>(side ? M.gate.bearing_b : M.gate.bearing_a) + 3 * (size_t)k;
  br[0] = pu[0]; br[1] = pu[1]; br[2] = 1.0;
  const int l = F.lm[e];
  const bool skip = track_live(W, lm_slots(W), l) && lm_initialised(W, F, l);
  const_cast<uint8_t*>(side ? M.skipB : M.skipA)[k] = skip ? 1 : 0;
}

// Rank test of getUncertainty (:349): H.colPivHouseholderQr().rank() < 9, by Eigen's ColPivHouseholderQR (column
// pivoting on the downdated column norms, Householder reflectors) and its rank rule |R_ii| > 9 eps |max pivot| over the
// nonzero pivots.  One warp; H column-major in shared memory, lane j < 9 owns column j.  Returns rank == 9.
__device__ bool qr_full_rank9(double* H, double* s_tau, int lane) {
  constexpr double eps = 2.220446049250313e-16;
  double nu = 0.0, nd = 0.0;
  if (lane < 9) {
    double s = 0.0;
    for (int i = 0; i < 9; ++i) s += H[lane * 9 + i] * H[lane * 9 + i];
    nd = nu = sqrt(s);
  }
  double maxn = nd;
  for (int o = 16; o > 0; o >>= 1) maxn = fmax(maxn, __shfl_xor_sync(0xffffffffu, maxn, o));
  const double thr_helper = (maxn * eps) * (maxn * eps) / 9.0;
  const double downdate_thr = sqrt(eps);
  int nonzero = 9;
  double maxpivot = 0.0;
  for (int k = 0; k < 9; ++k) {
    // biggest remaining updated norm, the first on ties (maxCoeff)
    double bv = (lane >= k && lane < 9) ? nu : -1.0;
    int bi = lane;
    for (int o = 16; o > 0; o >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (nonzero == 9 && bv * bv < thr_helper * (double)(9 - k)) nonzero = k;
    if (bi != k) {
      const double nu_k = __shfl_sync(0xffffffffu, nu, k), nd_k = __shfl_sync(0xffffffffu, nd, k);
      const double nu_p = __shfl_sync(0xffffffffu, nu, bi), nd_p = __shfl_sync(0xffffffffu, nd, bi);
      if (lane == k) { nu = nu_p; nd = nd_p; }
      if (lane == bi) { nu = nu_k; nd = nd_k; }
      if (lane < 9) {
        const double x = H[k * 9 + lane];
        H[k * 9 + lane] = H[bi * 9 + lane];
        H[bi * 9 + lane] = x;
      }
    }
    __syncwarp();
    if (lane == 0) {
      // makeHouseholderInPlace on rows k..8 of column k; R(k,k) = beta
      double* v = H + k * 9;
      const double c0 = v[k];
      double tail = 0.0;
      for (int i = k + 1; i < 9; ++i) tail += v[i] * v[i];
      double tau, beta;
      if (tail <= 2.2250738585072014e-308) {                   // numeric_limits<double>::min()
        tau = 0.0; beta = c0;
        for (int i = k + 1; i < 9; ++i) v[i] = 0.0;
      } else {
        beta = sqrt(c0 * c0 + tail);
        if (c0 >= 0.0) beta = -beta;
        for (int i = k + 1; i < 9; ++i) v[i] = v[i] / (c0 - beta);
        tau = (beta - c0) / beta;
      }
      v[k] = beta;
      *s_tau = tau;
    }
    __syncwarp();
    maxpivot = fmax(maxpivot, fabs(H[k * 9 + k]));
    if (lane > k && lane < 9) {
      // applyHouseholderOnTheLeft to column `lane`, then downdate its norm (LAPACK xGEQP3)
      const double tau = *s_tau;
      const double* v = H + k * 9;
      double* c = H + lane * 9;
      double w = 0.0;
      for (int i = k + 1; i < 9; ++i) w += v[i] * c[i];
      w += c[k];
      c[k] -= tau * w;
      for (int i = k + 1; i < 9; ++i) c[i] -= tau * v[i] * w;
      if (nu != 0.0) {
        double t = fabs(c[k]) / nu;
        t = (1.0 + t) * (1.0 - t);
        t = t < 0.0 ? 0.0 : t;
        const double t2 = t * (nu / nd) * (nu / nd);
        if (t2 <= downdate_thr) {
          double s = 0.0;
          for (int i = k + 1; i < 9; ++i) s += c[i] * c[i];
          nd = nu = sqrt(s);
        } else {
          nu *= sqrt(t);
        }
      }
    }
    __syncwarp();
  }
  const double thr = maxpivot * (eps * 9.0);
  int rank = 0;
  for (int i = 0; i < nonzero; ++i) rank += fabs(H[i * 9 + i]) > thr ? 1 : 0;
  __syncwarp();
  return rank == 9;
}

__global__ void __launch_bounds__(TK_T, 1) k_stereo_apply(const StereoJobDev* __restrict__ jobs, const MatchJobDev* __restrict__ tab) {
  constexpr int NWT = TK_T / 32;
  __shared__ int s_warp[NWT];
  __shared__ int s_list[TK_T];
  __shared__ uint8_t s_ok[TK_T];
  __shared__ double s_H[NWT][81];
  __shared__ double s_tau[NWT];
  const StereoJobDev& J = jobs[blockIdx.x];
  const MatchJobDev& M = tab[blockIdx.x];
  const GateDev& g = M.gate;
  const WinDev& W = *J.W;
  const FeatStore& F = *W.feat;
  const int L = lm_slots(W);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const size_t base_a = ((size_t)J.feat_a * F.C + J.cam_a) * F.N;
  const size_t base_b = ((size_t)J.feat_b * F.C + J.cam_b) * F.N;
  const double* geo = J.geo;
  int n_out = 0;
  for (int b0 = 0; b0 < M.nB; b0 += TK_T) {
    const int b = b0 + tid;
    int rec = 0, need_qr = 0, cbi = 0, a = -1, la = -1, lb = -1;
    double hpW[4] = {0.0, 0.0, 0.0, 0.0};
    if (b < M.nB) {
      const okb_pair p = M.pairs[b];
      // DenseMatcher::match calls setBestMatch for every B whose winner is below the threshold, B ascending
      if (p.index_a >= 0 && p.distance < J.threshold) {
        a = p.index_a;
        la = F.lm[base_a + a]; la = track_live(W, L, la) ? la : -1;
        lb = F.lm[base_b + b]; lb = track_live(W, L, lb) ? lb : -1;
        double hpA[4];
        bool parallel;
        if (!(la >= 0 && lb >= 0) && stereo_triangulate(g, a, b, hpA, parallel)) {
          rec = 1;
          cbi = parallel ? 0 : 1;
          if (cbi) {
            // getUncertainty (:253-355): A's residual Jacobian at the triangulated point; then the point moved 20 %
            // towards the baseline centre, where B's residual and both its Jacobians are evaluated (parametersB[1]
            // aliases hPA)
            const double I7[7] = {0, 0, 0, 0, 0, 0, 1};
            double* uj = J.uj + (size_t)kUJ * b;
            const double sdA = 0.8 * F.size[base_a + a] / 12.0, sdB = 0.8 * F.size[base_b + b] / 12.0;
            double rA[2], rB[2];
            reproj_full(W.cams[J.cam_a], I7, hpA, I7, F.kp + 2 * (base_a + a), sqrt(1.0 / (sdA * sdA)), rA, nullptr, uj, nullptr);
            double hm[4];
#pragma unroll
            for (int k = 0; k < 3; ++k) hm[k] = 0.8 * (hpA[k] - geo[k] / 2.0 * hpA[3]) + geo[k] / 2.0 * hpA[3];
            hm[3] = hpA[3];
            reproj_full(W.cams[J.cam_b], geo, hm, I7, F.kp + 2 * (base_b + b), sqrt(1.0 / (sdB * sdB)), rB, uj + 6, uj + 18, nullptr);
            if (rB[0] * rB[0] + rB[1] * rB[1] < 4.0) cbi = 0;
            else need_qr = 1;          // the rank of H decides
          }
          // T_WCa * hP_Ca
          const double* C = geo + 7;
          const double* r = geo + 16;
#pragma unroll
          for (int k = 0; k < 3; ++k) hpW[k] = C[3 * k] * hpA[0] + C[3 * k + 1] * hpA[1] + C[3 * k + 2] * hpA[2] + r[k] * hpA[3];
          hpW[3] = hpA[3];
        }
      }
    }
    int total_q;
    const int pos_q = block_scan<TK_T>(need_qr, s_warp, &total_q);
    if (need_qr) s_list[pos_q] = b;
    __syncthreads();
    for (int i = warp; i < total_q; i += NWT) {
      // H = H_ + J_hpA^T J_hpA (point block) + [J_TB J_hpB]^T [J_TB J_hpB], in the reference's order of additions
      const double* uj = J.uj + (size_t)kUJ * s_list[i];
      const double *JA = uj, *JT = uj + 6, *JH = uj + 18;
      double* H = s_H[warp];
      for (int e = lane; e < 81; e += 32) {
        const int r = e % 9, c = e / 9;
        double h;
        if (r < 6 && c < 6) h = geo[19 + r * 6 + c] + (JT[r] * JT[c] + JT[6 + r] * JT[6 + c]);
        else if (r < 6) h = JT[r] * JH[c - 6] + JT[6 + r] * JH[3 + c - 6];
        else if (c < 6) h = JH[r - 6] * JT[c] + JH[3 + r - 6] * JT[6 + c];
        else h = (JA[r - 6] * JA[c - 6] + JA[3 + r - 6] * JA[3 + c - 6]) + (JH[r - 6] * JH[c - 6] + JH[3 + r - 6] * JH[3 + c - 6]);
        H[c * 9 + r] = h;
      }
      __syncwarp();
      const bool ok = qr_full_rank9(H, &s_tau[warp], lane);
      if (lane == 0) s_ok[i] = ok ? 1 : 0;
    }
    __syncthreads();
    if (need_qr) cbi = s_ok[pos_q];
    int total;
    const int pos = block_scan<TK_T>(rec, s_warp, &total);
    if (rec) {
      okb_stereo_match& o = J.out[n_out + pos];
      o.kp_a = a; o.kp_b = b; o.lm_slot_a = la; o.lm_slot_b = lb; o.can_be_initialized = cbi; o._pad = 0;
      o.hp_W[0] = hpW[0]; o.hp_W[1] = hpW[1]; o.hp_W[2] = hpW[2]; o.hp_W[3] = hpW[3];
    }
    n_out += total;
  }
  if (tid == 0) *J.n_out = n_out;
}
}  // namespace

// Host checks of one job (first_win: the window of the call's first job, already checked); "" = valid.
static std::string match2d2d_job_invalid(okb_ctx* c, const okb_match2d2d_job& j, int first_win, std::vector<char>& seen) {
  const std::string why = store_window_invalid(c, j.win, seen);
  if (!why.empty()) return why;
  const WinStore& S = c->wins[j.win];
  const WinDev& W = c->host[j.win];
  const FeatStore& F = S.feat;
  if (F.D != c->wins[first_win].feat.D) return "descriptor length differs from the call's first job";
  if (j.pose_a < 0 || j.pose_a >= W.K) return "pose_a out of range";
  if (j.pose_b < 0 || j.pose_b >= W.K) return "pose_b out of range";
  if (j.sb_current < -1 || j.sb_current >= W.NSB) return "sb_current out of range";
  if (j.feat_slot_a < 0 || j.feat_slot_a >= F.F) return "feat_slot_a out of range";
  if (j.feat_slot_b < 0 || j.feat_slot_b >= F.F) return "feat_slot_b out of range";
  // one frame is one (position, feature slot) pair: the prior's velocity branch tests the slots, setFrames the poses
  if ((j.feat_slot_a == j.feat_slot_b) != (j.pose_a == j.pose_b)) return "feat_slot_a == feat_slot_b but pose_a != pose_b, or the reverse";
  for (int cam : {j.cam_a, j.cam_b})
    if (cam < 0 || cam >= F.C || cam >= W.NC || cam >= W.NE) return "camera " + std::to_string(cam) + " out of range";
  if (j.feat_slot_a == j.feat_slot_b && j.cam_a == j.cam_b) return "frame matched against itself in one camera";
  if (S.feat_n_pending[(size_t)j.feat_slot_a * F.C + j.cam_a] < 0) return "feature slot A has no keypoints for camera " + std::to_string(j.cam_a);
  if (S.feat_n_pending[(size_t)j.feat_slot_b * F.C + j.cam_b] < 0) return "feature slot B has no keypoints for camera " + std::to_string(j.cam_b);
  if (j.num_best < 1 || j.num_best > MAX_BEST) return "num_best out of range (1..8)";
  if (!j.n_out) return "n_out missing";
  const int nB = S.feat_n_pending[(size_t)j.feat_slot_b * F.C + j.cam_b];
  if (j.out_cap < nB || (nB && !j.out)) return "out capacity below the keypoints of (feat_slot_b, cam_b)";
  return "";
}

// okb_match2d2d_batch and okb_stereo_init_batch (which passes its jobs with frame A = frame B); `fn` names the entry
// point in the errors.
static int match2d2d_batch(okb_ctx* c, int n_jobs, const okb_match2d2d_job* jobs, const char* fn) {
  int rc = store_call_checks(c, fn, n_jobs, jobs, 65535, [&](int i, std::vector<char>& seen) {      // grid dimension
    return match2d2d_job_invalid(c, jobs[i], jobs[0].win, seen);
  });
  if (rc || n_jobs == 0) return rc;
  cudaSetDevice(c->device);
  okb_frontend_state* F = fe(c);
  CallBuffers& B = F->stereo;
  std::lock_guard<std::mutex> lk(B.mtx);
  if ((rc = commit_job_windows(c, jobs, n_jobs))) return rc;
  if ((rc = shard_lm_exchange(c, fn, jobs, n_jobs, c->stream_xfer))) return rc;
  cudaStream_t xs = c->stream_xfer;
  // staging (pinned + device mirror): in  = [job table | match table]
  //                                   out = [per job: count | records]
  // scratch (device only), per job: geometry | bearings A, B | ray sigmas A, B | the matcher's arrays | rank-test Jacobians
  struct JobLay { int nA, nB; size_t out, geo, ba, bb, rsa, rsb, uj; MatchScratch ms; };
  std::vector<JobLay> L(n_jobs);
  Carve st, sc;
  st.take(sizeof(StereoJobDev) * n_jobs, 256);
  const size_t o_tab = st.take(sizeof(MatchJobDev) * n_jobs, 256);
  const size_t in_bytes = st.off;
  for (int i = 0; i < n_jobs; ++i) {
    const okb_match2d2d_job& j = jobs[i];
    const WinStore& S = c->wins[j.win];
    JobLay& l = L[i];
    l.nA = S.feat_n_pending[(size_t)j.feat_slot_a * S.feat.C + j.cam_a];
    l.nB = S.feat_n_pending[(size_t)j.feat_slot_b * S.feat.C + j.cam_b];
    const size_t a = l.nA, b = l.nB;
    l.out = st.take(16 + sizeof(okb_stereo_match) * b);
    l.geo = sc.take(8 * kGeo);
    l.ba = sc.take(24 * a); l.bb = sc.take(24 * b);
    l.rsa = sc.take(8 * a); l.rsb = sc.take(8 * b);
    l.ms = carve_match(sc, a, b, j.num_best);
    l.uj = sc.take(8 * kUJ * b);
  }
  const size_t out_end = st.off;
  if ((rc = B.reserve(c, out_end, sc.off))) return rc;
  uint8_t* h = B.h_stage;
  uint8_t* d = B.d_stage;
  uint8_t* s = B.d_scratch;
  AssignSmem sm;
  int maxA = 0, maxN = 0;
  StereoJobDev* tj = reinterpret_cast<StereoJobDev*>(h);
  MatchJobDev* tm = reinterpret_cast<MatchJobDev*>(h + o_tab);
  for (int i = 0; i < n_jobs; ++i) {
    const okb_match2d2d_job& j = jobs[i];
    const FeatStore& FS = c->wins[j.win].feat;
    const JobLay& l = L[i];
    StereoJobDev J;
    std::memset(&J, 0, sizeof J);
    J.W = c->d_wins + j.win;
    J.pose_a = j.pose_a; J.feat_a = j.feat_slot_a; J.cam_a = j.cam_a;
    J.pose_b = j.pose_b; J.feat_b = j.feat_slot_b; J.cam_b = j.cam_b;
    J.sb = j.feat_slot_a != j.feat_slot_b ? j.sb_current : -1;
    J.threshold = j.threshold;
    J.geo = reinterpret_cast<double*>(s + l.geo);
    J.uj = reinterpret_cast<double*>(s + l.uj);
    J.n_out = reinterpret_cast<int*>(d + l.out);
    J.out = reinterpret_cast<okb_stereo_match*>(d + l.out + 16);
    const size_t ia = (size_t)j.feat_slot_a * FS.C + j.cam_a, ib = (size_t)j.feat_slot_b * FS.C + j.cam_b;
    MatchJobDev jd = store_match_job(c, FS, ia, ib, l.nA, l.nB, j.num_best, j.threshold, s, l.ms, sm);
    GateDev& g = jd.gate;                     // geometry and cameras: k_stereo_setup
    g.mode = OKB_GATE_2D2D;
    g.kp_a = FS.kp + 2 * ia * FS.N; g.kp_size_a = FS.size + ia * FS.N;
    g.bearing_a = reinterpret_cast<const double*>(s + l.ba);
    g.bearing_b = reinterpret_cast<const double*>(s + l.bb);
    g.ray_sigma_a = reinterpret_cast<const double*>(s + l.rsa);
    g.ray_sigma_b = reinterpret_cast<const double*>(s + l.rsb);
    tj[i] = J;
    tm[i] = jd;
    maxA = std::max(maxA, l.nA);
    maxN = std::max(maxN, std::max(l.nA, l.nB));
  }
  OKB_CUDA(c, cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, xs));
  const StereoJobDev* d_jobs = reinterpret_cast<const StereoJobDev*>(d);
  MatchJobDev* d_tab = reinterpret_cast<MatchJobDev*>(d + o_tab);
  if ((rc = sm.set_attribute(c))) return rc;
  const int n[2] = {0, n_jobs}, max_a[2] = {0, maxA};
  k_stereo_setup<<<dim3(std::max(1, (maxN + TK_T - 1) / TK_T), n_jobs, 2), TK_T, 0, xs>>>(d_jobs, d_tab);
  if ((rc = launch_matcher(c, xs, d_tab, c->wins[jobs[0].win].feat.D / 4, n, max_a, sm))) return rc;
  k_stereo_apply<<<n_jobs, TK_T, 0, xs>>>(d_jobs, d_tab);
  F->launches += 2;
  OKB_CUDA(c, cudaGetLastError());
  OKB_CUDA(c, cudaMemcpyAsync(h + in_bytes, d + in_bytes, out_end - in_bytes, cudaMemcpyDeviceToHost, xs));
  OKB_CUDA(c, cudaStreamSynchronize(xs));
  for (int i = 0; i < n_jobs; ++i) {
    const int n_rec = *reinterpret_cast<const int32_t*>(h + L[i].out);
    *jobs[i].n_out = n_rec;
    if (n_rec) std::memcpy(jobs[i].out, h + L[i].out + 16, sizeof(okb_stereo_match) * (size_t)n_rec);
  }
  return OKB_OK;
}

extern "C" int okb_match2d2d_batch(okb_ctx* c, int n_jobs, const okb_match2d2d_job* jobs) {
  return match2d2d_batch(c, n_jobs, jobs, "okb_match2d2d_batch");
}

extern "C" int okb_stereo_init_batch(okb_ctx* c, int n_jobs, const okb_stereo_job* jobs) {
  if (n_jobs > 0 && !jobs) return OKB_ERR_INVALID_ARG;      // read here; match2d2d_batch checks the rest
  std::vector<okb_match2d2d_job> mj(std::max(n_jobs, 0));
  for (int i = 0; i < n_jobs; ++i) {
    const okb_stereo_job& j = jobs[i];
    mj[i] = okb_match2d2d_job{j.win, j.pose, j.feat_slot, j.cam_a, j.pose, j.feat_slot, j.cam_b, -1, j.threshold, j.num_best,
                              j.out, j.out_cap, j.n_out};
  }
  return match2d2d_batch(c, n_jobs, mj.data(), "okb_stereo_init_batch");
}

// =================================================================================================
// Keyframe decision (okb_keyframe_overlap_batch): Frontend::doWeNeedANewKeyframe (okvis_frontend/src/Frontend.cpp:
// 295-369) on the window's feature store, one CTA per (job, camera) in one launch.  Per camera and per hull (all points,
// then the matched ones), block-wide:
//   1. the eight extreme points in x, y, x+y and x-y, and a stable compaction of the points not inside their octagon
//      by more than 2^-12 of the bounding box (Akl-Toussaint; those points cannot be hull vertices under any rounding
//      of the scan below, tests/keyframe_reference.py checks it), each with its index in cv::convexHull's input;
//   2. a bitonic sort of the survivors by (x, y, index) in shared memory (or in global scratch for an image with more
//      keypoints than the launch's shared-memory capacity);
//   3. cv::convexHull's Sklansky scan, one thread per quarter chain, differences in float and the convexity in double;
//      one thread assembles the hull in OpenCV's order (clockwise = false, the cyclic shift by input index) and sums
//      contourArea in that order;
// then a block-wide cv::pointPolygonTest of every point against the matched hull.  The last CTA of a job takes the
// maxima and the decision.  The call writes nothing but its scratch and its results.
// =================================================================================================
namespace {
constexpr int KF_T = TK_T;               // threads per CTA
constexpr int KF_SMEM_PTS = 2048;        // largest image kept in shared memory (buffers of 24 B per point)

struct KfCtaDev {                        // one (job, camera)
  const WinDev* W;
  int feat, cam, job, n_cams;
  float thr_o, thr_r;
  okb_keyframe_cam* cams;                // the job's [n_cams] records (device staging)
  okb_keyframe_result* res;
  int* done;                             // CTAs of the job finished (zeroed by the H2D copy)
  uint8_t* buf;                          // point buffers in global scratch, nullptr: shared memory
  int cap;                               // power of two >= the points the buffers hold
  int _pad;
};

__host__ __device__ inline size_t kf_buf_bytes(int cap) { return 24 * (size_t)cap + 64; }

// sortable image of a float (x + 0: -0 sorts as +0, as CHullCmpPoints compares) and back
__device__ __forceinline__ uint32_t kf_f2s(float f) {
  const uint32_t u = __float_as_uint(__fadd_rn(f, 0.0f));
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float kf_s2f(uint32_t s) { return __uint_as_float((s & 0x80000000u) ? (s & 0x7fffffffu) : ~s); }
__device__ __forceinline__ int kf_sign_f(float v) { return (v > 0.f) - (v < 0.f); }
__device__ __forceinline__ int kf_sign_d(double v) { return (v > 0.0) - (v < 0.0); }

struct KfBuf {                           // [cap] sort keys (x, y) | [cap] input index | [cap] hull | 2 x [cap + 8] stacks
  unsigned long long* key;
  uint32_t* idx;
  int* hull;
  int* sa;
  int* sb;
  __device__ KfBuf(uint8_t* p, int cap) {
    key = reinterpret_cast<unsigned long long*>(p);
    idx = reinterpret_cast<uint32_t*>(p + 8 * (size_t)cap);
    hull = reinterpret_cast<int*>(p + 12 * (size_t)cap);
    sa = reinterpret_cast<int*>(p + 16 * (size_t)cap);
    sb = sa + cap + 8;
  }
  __device__ float x(int i) const { return kf_s2f((uint32_t)(key[i] >> 32)); }
  __device__ float y(int i) const { return kf_s2f((uint32_t)key[i]); }
};

// Sklansky_ (OpenCV imgproc/src/convhull.cpp) over the sorted points; returns the stack size
__device__ int kf_sklansky(const KfBuf& B, int start, int end, int* stack, int nsign, int sign2) {
  const int incr = end > start ? 1 : -1;
  int pprev = start, pcur = pprev + incr, pnext = pcur + incr;
  int stacksize = 3;
  if (start == end || (B.x(start) == B.x(end) && B.y(start) == B.y(end))) { stack[0] = start; return 1; }
  stack[0] = pprev; stack[1] = pcur; stack[2] = pnext;
  end += incr;
  while (pnext != end) {
    const float cury = B.y(pcur), nexty = B.y(pnext);
    const float by = __fsub_rn(nexty, cury);
    if (kf_sign_f(by) != nsign) {
      const float ax = __fsub_rn(B.x(pcur), B.x(pprev));
      const float bx = __fsub_rn(B.x(pnext), B.x(pcur));
      const float ay = __fsub_rn(cury, B.y(pprev));
      const double convexity = (double)ay * bx - (double)ax * by;       // products exact: a contraction changes nothing
      if (kf_sign_d(convexity) == sign2 && (ax != 0.f || ay != 0.f)) {
        pprev = pcur; pcur = pnext; pnext += incr;
        stack[stacksize++] = pnext;
      } else if (pprev == start) {
        pcur = pnext; stack[1] = pcur; pnext += incr; stack[2] = pnext;
      } else {
        stack[stacksize - 2] = pnext; pcur = pprev; pprev = stack[stacksize - 4]; --stacksize;
      }
    } else {
      pnext += incr;
      stack[stacksize - 1] = pnext;
    }
  }
  return --stacksize;
}

template <typename T, typename Op>
__device__ __forceinline__ T kf_reduce(T v, T* s, Op op) {     // block-wide; s: [KF_T / 32]; result in every thread
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) s[warp] = v;
  __syncthreads();
  T r = s[0];
  for (int w = 1; w < KF_T / 32; ++w) r = op(r, s[w]);
  return r;
}

struct KfShared {
  int warp_i[KF_T / 32];
  double warp_d[KF_T / 32];
  double ext[8];                        // extreme values
  int ext_k[8];                         // first keypoint attaining them
  unsigned long long ymin, ymax;        // (sortable y, sorted position) of the first minimum / maximum
  int m, nout, cnt[4];
  double area;
};

// cv::convexHull of the points of the image (matched_only: those with a store slot >= 0; n_in of them), then contourArea.  Leaves the
// hull (sorted positions, OpenCV's order) in B.hull[0..nout), the sorted points in B.key, and returns nout; *area in
// every thread.
__device__ int kf_hull(const FeatStore& F, size_t base, int n, int n_in, bool matched_only, const KfBuf& B, int cap, KfShared& S,
                       double* area) {
  const int tid = threadIdx.x;
  auto in = [&](int k) { return !matched_only || F.lm[base + k] >= 0; };
  auto px = [&](int k) { return (double)(float)F.kp[2 * (base + k)]; };
  auto py = [&](int k) { return (double)(float)F.kp[2 * (base + k) + 1]; };
  // 1. extremes: E, NE, N, NW, W, SW, S, SE (counter-clockwise, y up); first keypoint index of each maximum
  double e[8];
#pragma unroll
  for (int d = 0; d < 8; ++d) e[d] = -INFINITY;
  for (int k = tid; k < n; k += KF_T) {
    if (!in(k)) continue;
    const double x = px(k), y = py(k);
    const double v[8] = {x, x + y, y, y - x, -x, -x - y, -y, x - y};
#pragma unroll
    for (int d = 0; d < 8; ++d) e[d] = fmax(e[d], v[d]);
  }
#pragma unroll
  for (int d = 0; d < 8; ++d) {
    const double r = kf_reduce(e[d], S.warp_d, [](double a, double b) { return fmax(a, b); });
    if (tid == 0) { S.ext[d] = r; S.ext_k[d] = INT_MAX; }
  }
  __syncthreads();
  for (int k = tid; k < n; k += KF_T) {
    if (!in(k)) continue;
    const double x = px(k), y = py(k);
    const double v[8] = {x, x + y, y, y - x, -x, -x - y, -y, x - y};
#pragma unroll
    for (int d = 0; d < 8; ++d)
      if (v[d] == S.ext[d]) atomicMin(&S.ext_k[d], k);
  }
  __syncthreads();
  double vx[8], vy[8];
#pragma unroll
  for (int d = 0; d < 8; ++d) { vx[d] = px(S.ext_k[d]); vy[d] = py(S.ext_k[d]); }
  const double D = fmax(S.ext[0] + S.ext[4], S.ext[2] + S.ext[6]);
  int edges = 0;
#pragma unroll
  for (int d = 0; d < 8; ++d) edges += (vx[(d + 1) & 7] != vx[d] || vy[(d + 1) & 7] != vy[d]) ? 1 : 0;
  // stable compaction of the survivors, each with its index among the hull's input points
  int run_in = 0, run_out = 0;
  for (int k0 = 0; k0 < n; k0 += KF_T) {
    const int k = k0 + tid;
    const int inc = k < n && in(k) ? 1 : 0;
    int keep = 0;
    if (inc) {
      keep = 1;
      if (edges > 0 && n_in >= 4) {          // a set of 4 points at least, as tests/keyframe_reference.py:extreme_filter
        const double x = px(k), y = py(k);
        bool inside = true;
#pragma unroll
        for (int d = 0; d < 8; ++d) {
          const double ex = vx[(d + 1) & 7] - vx[d], ey = vy[(d + 1) & 7] - vy[d];
          if (ex == 0.0 && ey == 0.0) continue;
          inside = inside && (ex * (y - vy[d]) - ey * (x - vx[d]) > 0x1p-12 * D * fmax(fabs(ex), fabs(ey)));
        }
        keep = inside ? 0 : 1;
      }
    }
    int t_in, t_out;
    const int r_in = block_scan<KF_T>(inc, S.warp_i, &t_in);
    const int r_out = block_scan<KF_T>(keep, S.warp_i, &t_out);
    if (keep) {
      const int o = run_out + r_out;
      B.key[o] = ((unsigned long long)kf_f2s((float)F.kp[2 * (base + k)]) << 32) | kf_f2s((float)F.kp[2 * (base + k) + 1]);
      B.idx[o] = (uint32_t)(run_in + r_in);
    }
    run_in += t_in; run_out += t_out;
  }
  const int m = run_out;
  int P = 1;
  while (P < m) P <<= 1;
  for (int i = m + tid; i < P; i += KF_T) { B.key[i] = ~0ull; B.idx[i] = ~0u; }
  __syncthreads();
  // 2. bitonic sort by (x, y, index)
  for (int k = 2; k <= P; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < P; i += KF_T) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long ka = B.key[i], kb = B.key[l];
          const uint32_t ia = B.idx[i], ib = B.idx[l];
          const bool gt = ka > kb || (ka == kb && ia > ib);
          if (gt == ((i & k) == 0)) { B.key[i] = kb; B.key[l] = ka; B.idx[i] = ib; B.idx[l] = ia; }
        }
      }
      __syncthreads();
    }
  // the first minimum and maximum of y in sorted order
  if (tid == 0) { S.ymin = ~0ull; S.ymax = ~0ull; }
  __syncthreads();
  unsigned long long lmin = ~0ull, lmax = ~0ull;
  for (int i = tid; i < m; i += KF_T) {
    const uint32_t sy = (uint32_t)B.key[i];
    lmin = min(lmin, ((unsigned long long)sy << 32) | (uint32_t)i);
    lmax = min(lmax, ((unsigned long long)(~sy) << 32) | (uint32_t)i);
  }
  atomicMin(&S.ymin, lmin);
  atomicMin(&S.ymax, lmax);
  __syncthreads();
  const int miny = (int)(uint32_t)S.ymin, maxy = (int)(uint32_t)S.ymax;
  const bool single = B.x(0) == B.x(m - 1) && B.y(0) == B.y(m - 1);
  // 3. the four quarter chains, one thread each: tl | tr in stack A, bl | br in stack B
  if (!single && tid < 4) {
    int* st = tid < 2 ? B.sa + (tid == 1 ? maxy + 3 : 0) : B.sb + (tid == 3 ? miny + 3 : 0);
    if (tid == 0) S.cnt[0] = kf_sklansky(B, 0, maxy, st, -1, 1);
    else if (tid == 1) S.cnt[1] = kf_sklansky(B, m - 1, maxy, st, -1, -1);
    else if (tid == 2) S.cnt[2] = kf_sklansky(B, 0, miny, st, 1, -1);
    else S.cnt[3] = kf_sklansky(B, m - 1, miny, st, 1, 1);
  }
  __syncthreads();
  if (tid == 0) {
    int nout = 0;
    if (single) {
      B.hull[nout++] = 0;
    } else {
      // clockwise = false: the upper chains swap roles
      const int* tl = B.sa + maxy + 3; int tl_count = S.cnt[1];
      const int* tr = B.sa; int tr_count = S.cnt[0];
      for (int i = 0; i < tl_count - 1; ++i) B.hull[nout++] = tl[i];
      for (int i = tr_count - 1; i > 0; --i) B.hull[nout++] = tr[i];
      const int stop_idx = tr_count > 2 ? tr[1] : tl_count > 2 ? tl[tl_count - 2] : -1;
      const int* bl = B.sb; int bl_count = S.cnt[2];
      const int* br = B.sb + miny + 3; int br_count = S.cnt[3];
      if (stop_idx >= 0) {
        const int check_idx = bl_count > 2 ? bl[1] : bl_count + br_count > 2 ? br[2 - bl_count] : -1;
        if (check_idx == stop_idx || (check_idx >= 0 && B.x(check_idx) == B.x(stop_idx) && B.y(check_idx) == B.y(stop_idx))) {
          bl_count = min(bl_count, 2);         // all points on one line
          br_count = min(br_count, 2);
        }
      }
      for (int i = 0; i < bl_count - 1; ++i) B.hull[nout++] = bl[i];
      for (int i = br_count - 1; i > 0; --i) B.hull[nout++] = br[i];
      // the cyclic shift that makes the input indices ascend or descend, where one does
      if (nout >= 3) {
        int min_idx = 0, max_idx = 0, lt = 0;
        for (int i = 1; i < nout; ++i) {
          const uint32_t v = B.idx[B.hull[i]];
          lt += B.idx[B.hull[i - 1]] < v;
          if (lt > 1 && lt <= i - 2) break;
          if (v < B.idx[B.hull[min_idx]]) min_idx = i;
          if (v > B.idx[B.hull[max_idx]]) max_idx = i;
        }
        const int mmdist = abs(max_idx - min_idx);
        if ((mmdist == 1 || mmdist == nout - 1) && (lt <= 1 || lt >= nout - 2)) {
          const bool ascending = (max_idx + 1) % nout == min_idx;
          const int i0 = ascending ? min_idx : max_idx;
          int j = i0, i;
          if (i0 > 0) {
            int* tmp = B.sa;                   // the chains are copied out
            for (i = 0; i < nout; ++i) {
              const int cur = tmp[i] = B.hull[j];
              const int nj = j + 1 < nout ? j + 1 : 0;
              if (i < nout - 1 && (ascending != (B.idx[cur] < B.idx[B.hull[nj]]))) break;
              j = nj;
            }
            if (i == nout)
              for (int q = 0; q < nout; ++q) B.hull[q] = tmp[q];
          }
        }
      }
    }
    // contourArea, in hull order from the last vertex
    double a00 = 0.0;
    float prevx = B.x(B.hull[nout - 1]), prevy = B.y(B.hull[nout - 1]);
    for (int i = 0; i < nout; ++i) {
      const float qx = B.x(B.hull[i]), qy = B.y(B.hull[i]);
      a00 += (double)prevx * qy - (double)prevy * qx;
      prevx = qx; prevy = qy;
    }
    S.area = fabs(a00 * 0.5);
    S.nout = nout;
    S.m = m;
  }
  __syncthreads();
  *area = S.area;
  const int nout = S.nout;
  __syncthreads();
  return nout;
}

__global__ void __launch_bounds__(KF_T) k_keyframe_overlap(const KfCtaDev* __restrict__ ctas) {
  extern __shared__ __align__(16) uint8_t kf_smem[];
  __shared__ KfShared S;
  const KfCtaDev& J = ctas[blockIdx.x];
  const FeatStore& F = *J.W->feat;
  const int tid = threadIdx.x;
  const KfBuf B(J.buf ? J.buf : kf_smem, J.cap);
  const size_t base = ((size_t)J.feat * F.C + J.cam) * F.N;
  const int n = F.n[(size_t)J.feat * F.C + J.cam];
  int nm_local = 0;
  for (int k = tid; k < n; k += KF_T) nm_local += F.lm[base + k] >= 0 ? 1 : 0;
  const int nm = kf_reduce(nm_local, S.warp_i, [](int a, int b) { return a + b; });
  okb_keyframe_cam rec;
  memset(&rec, 0, sizeof rec);
  rec.n_points = n; rec.n_matched = nm; rec.skipped = 1;
  if (n >= 3 && nm >= 3) {
    double area_all, area_m;
    const int h_all = kf_hull(F, base, n, n, false, B, J.cap, S, &area_all);
    const int h_m = kf_hull(F, base, n, nm, true, B, J.cap, S, &area_m);
    // the matched hull's vertices, in order, into the stacks (float2 per vertex)
    float2* poly = reinterpret_cast<float2*>(B.sa);
    for (int i = tid; i < h_m; i += KF_T) poly[i] = make_float2(B.x(B.hull[i]), B.y(B.hull[i]));
    __syncthreads();
    int inside = 0;
    if (h_m > 2) {
      // cv::pointPolygonTest(matchesHull, p, false) > 0 for every point
      for (int k = tid; k < n; k += KF_T) {
        const float ptx = (float)F.kp[2 * (base + k)], pty = (float)F.kp[2 * (base + k) + 1];
        float2 v = poly[h_m - 1];
        int counter = 0, res = 1;
        for (int i = 0; i < h_m; ++i) {
          const float2 v0 = v;
          v = poly[i];
          if ((v0.y <= pty && v.y <= pty) || (v0.y > pty && v.y > pty) || (v0.x < ptx && v.x < ptx)) {
            if (pty == v.y && (ptx == v.x || (pty == v0.y && ((v0.x <= ptx && ptx <= v.x) || (v.x <= ptx && ptx <= v0.x))))) { res = 0; break; }
            continue;
          }
          double dist = (double)__fsub_rn(pty, v0.y) * __fsub_rn(v.x, v0.x) - (double)__fsub_rn(ptx, v0.x) * __fsub_rn(v.y, v0.y);
          if (dist == 0.0) { res = 0; break; }
          if (v.y < v0.y) dist = -dist;
          counter += dist > 0.0;
        }
        if (res != 0 && (counter & 1)) ++inside;
      }
      inside = kf_reduce(inside, S.warp_i, [](int a, int b) { return a + b; });
    }
    rec.skipped = 0;
    rec.hull_all = h_all; rec.hull_matched = h_m; rec.inside = inside;
    rec.area_all = area_all; rec.area_matched = area_m;
    rec.overlap = area_m / area_all;
    rec.ratio = (double)nm / (double)inside;
  }
  if (tid == 0) {
    J.cams[J.cam] = rec;
    __threadfence();
    if (atomicAdd(J.done, 1) == J.n_cams - 1) {
      __threadfence();
      // the maxima in camera order, std::max(value, running) = (value < running) ? running : value
      double overlap = 0.0, ratio = 0.0;
      for (int c = 0; c < J.n_cams; ++c) {
        const volatile okb_keyframe_cam& r = J.cams[c];
        if (r.skipped) continue;
        const double o = r.overlap, q = r.ratio;
        overlap = (o < overlap) ? overlap : o;
        ratio = (q < ratio) ? ratio : q;
      }
      okb_keyframe_result out;
      out.overlap = overlap; out.ratio = ratio;
      out.need_keyframe = (overlap > (double)J.thr_o && ratio > (double)J.thr_r) ? 0 : 1;
      out._pad = 0;
      *J.res = out;
    }
  }
}
}  // namespace

// Host checks of one job; "" = valid.
static std::string keyframe_job_invalid(okb_ctx* c, const okb_keyframe_job& j, std::vector<char>& seen) {
  const std::string why = store_window_invalid(c, j.win, seen);
  if (!why.empty()) return why;
  const WinStore& S = c->wins[j.win];
  const FeatStore& F = S.feat;
  if (j.feat_slot < 0 || j.feat_slot >= F.F) return "feat_slot out of range";
  if (j.n_cams < 1 || j.n_cams > F.C) return "n_cams out of range (1..the store's cameras)";
  for (int cam = 0; cam < j.n_cams; ++cam)
    if (S.feat_n_pending[(size_t)j.feat_slot * F.C + cam] < 0) return "feature slot has no keypoints for camera " + std::to_string(cam);
  if (!j.cams || !j.out) return "cams / out missing";
  return "";
}

extern "C" int okb_keyframe_overlap_batch(okb_ctx* c, int n_jobs, const okb_keyframe_job* jobs) {
  int rc = store_call_checks(c, "okb_keyframe_overlap_batch", n_jobs, jobs, INT_MAX,
                             [&](int i, std::vector<char>& seen) { return keyframe_job_invalid(c, jobs[i], seen); });
  if (rc || n_jobs == 0) return rc;
  cudaSetDevice(c->device);
  okb_frontend_state* F = fe(c);
  CallBuffers& B = F->kf;
  std::lock_guard<std::mutex> lk(B.mtx);
  if ((rc = commit_job_windows(c, jobs, n_jobs))) return rc;
  cudaStream_t xs = c->stream_xfer;
  // staging (pinned + device mirror): in  = [per job: done counter | CTA table]
  //                                   out = [per job: result | camera records]
  // scratch (device only): the point buffers of the images above the shared-memory capacity
  int n_cta = 0;
  for (int i = 0; i < n_jobs; ++i) n_cta += jobs[i].n_cams;
  Carve st, sc;
  st.take(sizeof(int) * (size_t)n_jobs, 256);
  const size_t o_tab = st.take(sizeof(KfCtaDev) * (size_t)n_cta, 256);
  const size_t in_bytes = st.off;
  std::vector<size_t> o_out(n_jobs);
  for (int i = 0; i < n_jobs; ++i) o_out[i] = st.take(sizeof(okb_keyframe_result) + sizeof(okb_keyframe_cam) * (size_t)jobs[i].n_cams, 256);
  const size_t out_end = st.off;
  auto pow2 = [](int v) { int p = 32; while (p < v) p <<= 1; return p; };
  int smem_cap = 32;
  std::vector<size_t> o_sc(n_cta, SIZE_MAX);
  std::vector<int> caps(n_cta);
  for (int i = 0, t = 0; i < n_jobs; ++i) {
    const WinStore& S = c->wins[jobs[i].win];
    for (int cam = 0; cam < jobs[i].n_cams; ++cam, ++t) {
      const int n = S.feat_n_pending[(size_t)jobs[i].feat_slot * S.feat.C + cam];
      caps[t] = pow2(n);
      if (n <= KF_SMEM_PTS) smem_cap = std::max(smem_cap, caps[t]);
      else o_sc[t] = sc.take(kf_buf_bytes(caps[t]), 256);
    }
  }
  if ((rc = B.reserve(c, out_end, sc.off))) return rc;
  uint8_t* h = B.h_stage;
  uint8_t* d = B.d_stage;
  std::memset(h, 0, o_tab);
  KfCtaDev* tc = reinterpret_cast<KfCtaDev*>(h + o_tab);
  for (int i = 0, t = 0; i < n_jobs; ++i) {
    const okb_keyframe_job& j = jobs[i];
    for (int cam = 0; cam < j.n_cams; ++cam, ++t) {
      KfCtaDev J;
      std::memset(&J, 0, sizeof J);
      J.W = c->d_wins + j.win;
      J.feat = j.feat_slot; J.cam = cam; J.job = i; J.n_cams = j.n_cams;
      J.thr_o = j.overlap_threshold; J.thr_r = j.matching_ratio_threshold;
      J.res = reinterpret_cast<okb_keyframe_result*>(d + o_out[i]);
      J.cams = reinterpret_cast<okb_keyframe_cam*>(d + o_out[i] + sizeof(okb_keyframe_result));
      J.done = reinterpret_cast<int*>(d) + i;
      J.buf = o_sc[t] == SIZE_MAX ? nullptr : B.d_scratch + o_sc[t];
      J.cap = o_sc[t] == SIZE_MAX ? smem_cap : caps[t];
      tc[t] = J;
    }
  }
  const size_t smem = kf_buf_bytes(smem_cap);
  OKB_CUDA(c, cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, xs));
  if (smem > 48 * 1024) OKB_CUDA(c, cudaFuncSetAttribute(k_keyframe_overlap, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_keyframe_overlap<<<n_cta, KF_T, smem, xs>>>(reinterpret_cast<const KfCtaDev*>(d + o_tab));
  F->launches += 1;
  OKB_CUDA(c, cudaGetLastError());
  OKB_CUDA(c, cudaMemcpyAsync(h + in_bytes, d + in_bytes, out_end - in_bytes, cudaMemcpyDeviceToHost, xs));
  OKB_CUDA(c, cudaStreamSynchronize(xs));
  for (int i = 0; i < n_jobs; ++i) {
    *jobs[i].out = *reinterpret_cast<const okb_keyframe_result*>(h + o_out[i]);
    std::memcpy(jobs[i].cams, h + o_out[i] + sizeof(okb_keyframe_result), sizeof(okb_keyframe_cam) * (size_t)jobs[i].n_cams);
  }
  return OKB_OK;
}

// =================================================================================================
// 3D-2D outlier rejection (okb_ransac_3d2d_batch): Frontend::runRansac3d2d (okvis_frontend/src/Frontend.cpp:575-642) on
// the window's feature store, one CTA per job in one launch (DESIGN.md 6f; tests/ransac_reference.py restates it):
//   1. the observation counts of the window's landmarks, then FrameNoncentralAbsoluteAdapter's correspondences
//      (FrameNoncentralAbsoluteAdapter.cpp:65-160) compacted in (camera, keypoint) order by a block scan;
//   2. one thread per hypothesis: 4 distinct correspondences from a counter-based SplitMix64 draw, a generalised P3P on
//      the first 3 (an octic in the first depth whose positive roots are bracketed by the roots of its derivatives),
//      the 4th picking the solution of lowest score;
//   3. the whole CTA scores hypotheses x correspondences (FrameAbsolutePoseSacProblem.hpp:134-160), a warp per
//      hypothesis; thread 0 takes the winner (most inliers, the lowest index on ties);
//   4. with at least 10 inliers, the other correspondences as outlier records in correspondence order (block scan).
// The call writes nothing but its scratch and its results.
// =================================================================================================
namespace {
constexpr int RS_T = 256;
constexpr int RS_MAX_HYP = 64;
constexpr int RS_MAX_CAMS = 16;
constexpr int RS_CD = 10;          // doubles per correspondence: point X_W (3), bearing (3), ray C_SC bearing (3), sigmaAngle
constexpr int RS_BISECT = 60;      // bisection steps per bracketed root, every derivative level
constexpr int RS_POLISH = 2;       // Gauss-Newton steps on the three distance equations

struct RansacJobDev {
  const WinDev* W;
  int feat, n_cams, n_hyp, cnt_cap;
  double threshold;
  unsigned long long seed;
  int* cnt;                        // [cnt_cap] observations per landmark slot (scratch)
  double* cd;                      // [n_kp][RS_CD] correspondences (scratch)
  int* ci;                         // [n_kp][3] camera, keypoint, landmark slot (scratch)
  okb_ransac_result* res;
  int* hyp;                        // [n_hyp] inliers per hypothesis
  okb_ransac_outlier* outl;
};

// SplitMix64's output for the counter (hypothesis h, draw c) of a seed: the state after h * 2^32 + c + 1 steps
__device__ __forceinline__ unsigned long long rs_draw(unsigned long long seed, int h, int c) {
  unsigned long long z = seed + 0x9E3779B97F4A7C15ull * ((((unsigned long long)h) << 32) + (unsigned long long)c + 1ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// K distinct indices in [0, n) (multiply-shift of the draw's high word); a duplicate is redrawn with the next counter,
// at most 64 draws (false: no sample)
template <int K>
__device__ bool rs_sample(unsigned long long seed, int h, int n, int* idx) {
  int m = 0;
  for (int c = 0; c < 64 && m < K; ++c) {
    const int v = (int)(((rs_draw(seed, h, c) >> 32) * (unsigned long long)n) >> 32);
    bool dup = false;
    for (int i = 0; i < m; ++i) dup = dup || idx[i] == v;
    if (!dup) idx[m++] = v;
  }
  return m == K;
}

__device__ __forceinline__ double rs_dot(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
__device__ __forceinline__ double rs_horner(const double* c, int m, double x) {
  double v = c[m];
  for (int i = m - 1; i >= 0; --i) v = v * x + c[i];
  return v;
}
// r = p q (degrees np, nq)
__device__ void rs_umul(const double* p, int np, const double* q, int nq, double* r) {
  for (int k = 0; k <= np + nq; ++k) r[k] = 0.0;
  for (int i = 0; i <= np; ++i)
    for (int j = 0; j <= nq; ++j) r[i + j] += p[i] * q[j];
}
// C = A B for polynomials in (x, y) of total degree <= 4, M[i][j] = coefficient of x^i y^j
__device__ void rs_bmul(const double (*A)[5], const double (*B)[5], double (*Cm)[5]) {
  for (int i = 0; i < 5; ++i)
    for (int j = 0; j < 5; ++j) Cm[i][j] = 0.0;
  for (int i1 = 0; i1 < 5; ++i1)
    for (int j1 = 0; i1 + j1 < 5; ++j1) {
      if (A[i1][j1] == 0.0) continue;
      for (int i2 = 0; i1 + i2 < 5; ++i2)
        for (int j2 = 0; i1 + i2 + j1 + j2 < 5; ++j2) Cm[i1 + i2][j1 + j2] += A[i1][j1] * B[i2][j2];
    }
}

// The roots of p (degree <= D) in (0, B] (SIGNED: in (-B, B]), B = Cauchy's bound of p made monic after dropping
// leading coefficients below 1e-14 of the largest, ascending.  Level m = 1..n takes the (n-m)-th derivative: between
// consecutive roots of the level below (and the interval's ends) it is monotone, and each sign change is bisected
// RS_BISECT times.
template <int D, bool SIGNED>
__device__ int rs_real_roots(const double* p, double* roots) {
  double mx = 0.0;
  for (int i = 0; i <= D; ++i) {
    if (!isfinite(p[i])) return 0;
    mx = fmax(mx, fabs(p[i]));
  }
  int n = D;
  while (n > 0 && !(fabs(p[n]) > 1e-14 * mx)) --n;
  if (n == 0) return 0;
  double q[D + 1];
  for (int i = 0; i <= n; ++i) q[i] = p[i] / p[n];
  double bound = 0.0;
  for (int i = 0; i < n; ++i) bound = fmax(bound, fabs(q[i]));
  bound += 1.0;
  int nr = 0;
  for (int m = 1; m <= n; ++m) {
    double c[D + 1];
    for (int i = 0; i <= m; ++i) {
      double f = q[i + n - m];
      for (int t = i + 1; t <= i + n - m; ++t) f *= (double)t;
      c[i] = f;
    }
    double nxt[D];
    int k = 0;
    double lo = SIGNED ? -bound : 0.0, flo = rs_horner(c, m, lo);
    for (int e = 0; e <= nr; ++e) {
      const double hi = e < nr ? roots[e] : bound;
      const double fhi = rs_horner(c, m, hi);
      if ((flo < 0.0 && fhi >= 0.0) || (flo > 0.0 && fhi <= 0.0)) {
        const bool neg = flo < 0.0;
        double a = lo, b = hi;
        for (int it = 0; it < RS_BISECT; ++it) {
          const double mid = 0.5 * (a + b);
          if ((rs_horner(c, m, mid) < 0.0) == neg) a = mid; else b = mid;
        }
        nxt[k++] = 0.5 * (a + b);
      }
      lo = hi; flo = fhi;
    }
    for (int i = 0; i < k; ++i) roots[i] = nxt[i];
    nr = k;
  }
  return nr;
}

// The triad of an edge u1 and a normal nn: rows e1 = u1 / |u1|, e2 = n x e1, n = nn / |nn|
__device__ __forceinline__ void rs_triad(const double* u1, const double* nn, double (*Fr)[3]) {
  const double i1 = 1.0 / sqrt(rs_dot(u1, u1)), in = 1.0 / sqrt(rs_dot(nn, nn));
  for (int k = 0; k < 3; ++k) { Fr[0][k] = u1[k] * i1; Fr[2][k] = nn[k] * in; }
  Fr[1][0] = Fr[2][1] * Fr[0][2] - Fr[2][2] * Fr[0][1];
  Fr[1][1] = Fr[2][2] * Fr[0][0] - Fr[2][0] * Fr[0][2];
  Fr[1][2] = Fr[2][0] * Fr[0][1] - Fr[2][1] * Fr[0][0];
}

// Generalised P3P: rays c_i + l_i f_i (body frame, |f_i| = 1) through world points X_i, i = 0..2.  Depths solve
// Q_ij = |c_i + l_i f_i - c_j - l_j f_j|^2 - |X_i - X_j|^2 = 0 (DESIGN.md 6f): the problem scaled to unit size, the
// resultant of Q02 and Q12 in l_2 reduced modulo Q01 in l_1 to alpha l_1 + beta, the octic alpha^2 b - alpha beta a + beta^2
// in l_0, its positive roots, l_1 = -beta / alpha, l_2 = -D_q / D_p, RS_POLISH Gauss-Newton steps; admissible when every
// depth is positive and every equation holds to 1e-10 of |X_i - X_j|^2.  emit(R, t) (X = R p + t) per admissible
// solution, ascending l_0; (R, t) from the two triangles by the triad of their first edge and normal, about the
// centroids.
template <typename Emit>
__device__ void rs_gp3p(const double (*c)[3], const double (*f)[3], const double (*X)[3], Emit&& emit) {
  double dX[3][3];
  for (int k = 0; k < 3; ++k) { dX[0][k] = X[0][k] - X[1][k]; dX[1][k] = X[0][k] - X[2][k]; dX[2][k] = X[1][k] - X[2][k]; }
  const double D01 = rs_dot(dX[0], dX[0]), D02 = rs_dot(dX[1], dX[1]), D12 = rs_dot(dX[2], dX[2]);
  const double s = sqrt(fmax(D01, fmax(D02, D12)));
  if (!(s > 0.0) || !isfinite(s)) return;
  const double is = 1.0 / s;
  double c01[3], c02[3], c12[3];
  for (int k = 0; k < 3; ++k) {
    c01[k] = (c[0][k] - c[1][k]) * is; c02[k] = (c[0][k] - c[2][k]) * is; c12[k] = (c[1][k] - c[2][k]) * is;
  }
  const double d01 = D01 * is * is, d02 = D02 * is * is, d12 = D12 * is * is;
  const double f01 = rs_dot(f[0], f[1]), f02 = rs_dot(f[0], f[2]), f12 = rs_dot(f[1], f[2]);
  const double k01 = rs_dot(c01, c01) - d01, k02 = rs_dot(c02, c02) - d02, k12 = rs_dot(c12, c12) - d12;
  const double g0_01 = rs_dot(f[0], c01), g1_01 = rs_dot(f[1], c01), g0_02 = rs_dot(f[0], c02), g2_02 = rs_dot(f[2], c02);
  const double g1_12 = rs_dot(f[1], c12), g2_12 = rs_dot(f[2], c12), g2_01 = rs_dot(f[2], c01);
  double Dp[5][5] = {}, Dq[5][5] = {}, R1[5][5] = {}, P1[5][5] = {}, T1[5][5], T2[5][5], S[5][5];
  Dp[1][0] = 2.0 * f02; Dp[0][1] = -2.0 * f12; Dp[0][0] = 2.0 * g2_01;
  Dq[0][2] = 1.0; Dq[0][1] = 2.0 * g1_12; Dq[0][0] = k12 - k02; Dq[1][0] = -2.0 * g0_02; Dq[2][0] = -1.0;
  R1[2][0] = 1.0; R1[1][0] = 2.0 * g0_02; R1[0][0] = k02;
  P1[1][0] = -2.0 * f02; P1[0][0] = -2.0 * g2_02;
  rs_bmul(Dp, R1, T1);
  rs_bmul(Dq, P1, T2);
  for (int i = 0; i < 5; ++i)
    for (int j = 0; j < 5; ++j) T1[i][j] -= T2[i][j];
  rs_bmul(Dp, T1, S);
  rs_bmul(Dq, Dq, T2);
  for (int i = 0; i < 5; ++i)
    for (int j = 0; j < 5; ++j) S[i][j] += T2[i][j];
  // S modulo Q01 = l_1^2 + a l_1 + b: l_1^2 = -a l_1 - b, l_1^3 = (a^2 - b) l_1 + a b, l_1^4 = (2 a b - a^3) l_1 + b^2 - a^2 b
  const double a[2] = {-2.0 * g1_01, -2.0 * f01};
  const double b[3] = {k01, 2.0 * g0_01, 1.0};
  double A2[3], AB[4], A3[4], A2B[5], B2[5], r3y[3], r4y[4], r4c[5];
  rs_umul(a, 1, a, 1, A2);
  rs_umul(a, 1, b, 2, AB);
  rs_umul(A2, 2, a, 1, A3);
  rs_umul(A2, 2, b, 2, A2B);
  rs_umul(b, 2, b, 2, B2);
  for (int i = 0; i < 3; ++i) r3y[i] = A2[i] - b[i];
  for (int i = 0; i < 4; ++i) r4y[i] = 2.0 * AB[i] - A3[i];
  for (int i = 0; i < 5; ++i) r4c[i] = B2[i] - A2B[i];
  double sk[5][5];                                  // sk[k] = coefficient of l_1^k, a polynomial in l_0 of degree 4 - k
  for (int k = 0; k < 5; ++k)
    for (int i = 0; i < 5; ++i) sk[k][i] = S[i][k];
  double al[9] = {}, be[9] = {}, t[9];
  for (int i = 0; i < 4; ++i) al[i] = sk[1][i];
  rs_umul(a, 1, sk[2], 2, t);  for (int i = 0; i < 4; ++i) al[i] -= t[i];
  rs_umul(r3y, 2, sk[3], 1, t); for (int i = 0; i < 4; ++i) al[i] += t[i];
  rs_umul(r4y, 3, sk[4], 0, t); for (int i = 0; i < 4; ++i) al[i] += t[i];
  for (int i = 0; i < 5; ++i) be[i] = sk[0][i];
  rs_umul(b, 2, sk[2], 2, t);  for (int i = 0; i < 5; ++i) be[i] -= t[i];
  rs_umul(AB, 3, sk[3], 1, t); for (int i = 0; i < 5; ++i) be[i] += t[i];
  rs_umul(r4c, 4, sk[4], 0, t); for (int i = 0; i < 5; ++i) be[i] += t[i];
  double oct[9], u[9];
  rs_umul(al, 3, al, 3, u);   rs_umul(u, 6, b, 2, oct);
  rs_umul(al, 3, be, 4, u);   rs_umul(u, 7, a, 1, t);  for (int i = 0; i < 9; ++i) oct[i] -= t[i];
  rs_umul(be, 4, be, 4, u);   for (int i = 0; i < 9; ++i) oct[i] += u[i];
  double roots[8];
  const int nr = rs_real_roots<8, false>(oct, roots);
  for (int r = 0; r < nr; ++r) {
    double x = roots[r];
    const double alx = rs_horner(al, 3, x), bex = rs_horner(be, 4, x);
    if (alx == 0.0) continue;
    double y = -bex / alx;
    const double dp = 2.0 * f02 * x - 2.0 * f12 * y + 2.0 * g2_01;
    if (dp == 0.0) continue;
    const double dq = y * y + 2.0 * g1_12 * y + (k12 - k02) - x * x - 2.0 * g0_02 * x;
    double z = -dq / dp;
    for (int it = 0; it < RS_POLISH; ++it) {
      const double F0 = x * x + y * y - 2.0 * f01 * x * y + 2.0 * g0_01 * x - 2.0 * g1_01 * y + k01;
      const double F1 = x * x + z * z - 2.0 * f02 * x * z + 2.0 * g0_02 * x - 2.0 * g2_02 * z + k02;
      const double F2 = y * y + z * z - 2.0 * f12 * y * z + 2.0 * g1_12 * y - 2.0 * g2_12 * z + k12;
      const double A = 2.0 * x - 2.0 * f01 * y + 2.0 * g0_01, B = 2.0 * y - 2.0 * f01 * x - 2.0 * g1_01;
      const double C = 2.0 * x - 2.0 * f02 * z + 2.0 * g0_02, D = 2.0 * z - 2.0 * f02 * x - 2.0 * g2_02;
      const double E = 2.0 * y - 2.0 * f12 * z + 2.0 * g1_12, G = 2.0 * z - 2.0 * f12 * y - 2.0 * g2_12;
      const double det = -A * D * E - B * C * G;
      if (!(det != 0.0) || !isfinite(det)) break;
      x += (F0 * D * E + B * F1 * G - B * D * F2) / det;
      y += (-A * F1 * G + A * D * F2 + F0 * C * G) / det;
      z += (A * F1 * E + B * C * F2 - F0 * C * E) / det;
    }
    if (!(x > 0.0 && y > 0.0 && z > 0.0) || !isfinite(x + y + z)) continue;
    const double lam[3] = {x, y, z};
    double pp[3][3];                                  // scaled body points
    for (int i = 0; i < 3; ++i)
      for (int k = 0; k < 3; ++k) pp[i][k] = c[i][k] * is + lam[i] * f[i][k];
    const int pr[3][2] = {{0, 1}, {0, 2}, {1, 2}};
    const double dd[3] = {d01, d02, d12};
    bool ok = true;
    for (int e = 0; e < 3; ++e) {
      double v[3];
      for (int k = 0; k < 3; ++k) v[k] = pp[pr[e][0]][k] - pp[pr[e][1]][k];
      ok = ok && fabs(rs_dot(v, v) - dd[e]) <= 1e-10 * dd[e];
    }
    if (!ok) continue;
    double p[3][3];                                   // body points, metric
    for (int i = 0; i < 3; ++i)
      for (int k = 0; k < 3; ++k) p[i][k] = c[i][k] + (lam[i] * s) * f[i][k];
    double Fp[3][3], Fx[3][3];                        // rows: e1, e2, n
    for (int side = 0; side < 2; ++side) {
      const double (*P)[3] = side ? X : p;
      double u1[3], u2[3], nn[3];
      for (int k = 0; k < 3; ++k) { u1[k] = P[1][k] - P[0][k]; u2[k] = P[2][k] - P[0][k]; }
      nn[0] = u1[1] * u2[2] - u1[2] * u2[1]; nn[1] = u1[2] * u2[0] - u1[0] * u2[2]; nn[2] = u1[0] * u2[1] - u1[1] * u2[0];
      rs_triad(u1, nn, side ? Fx : Fp);
    }
    double R[9], tt[3];
    for (int r0 = 0; r0 < 3; ++r0)
      for (int c0 = 0; c0 < 3; ++c0) R[3 * r0 + c0] = Fx[0][r0] * Fp[0][c0] + Fx[1][r0] * Fp[1][c0] + Fx[2][r0] * Fp[2][c0];
    if (!isfinite(R[0] + R[1] + R[2] + R[3] + R[4] + R[5] + R[6] + R[7] + R[8])) continue;
    double pc[3], xc[3];
    for (int k = 0; k < 3; ++k) { pc[k] = (p[0][k] + p[1][k] + p[2][k]) / 3.0; xc[k] = (X[0][k] + X[1][k] + X[2][k]) / 3.0; }
    for (int k = 0; k < 3; ++k) tt[k] = xc[k] - (R[3 * k] * pc[0] + R[3 * k + 1] * pc[1] + R[3 * k + 2] * pc[2]);
    emit(R, tt);
  }
}

// Eigen's Quaternion(Matrix3d) of M (row-major), q = [x, y, z, w]
__device__ __forceinline__ void rs_quat(const double* M, double* q) {
  const double tr = M[0] + M[4] + M[8];
  if (tr > 0.0) {
    double s = sqrt(tr + 1.0);
    q[3] = 0.5 * s; s = 0.5 / s;
    q[0] = (M[7] - M[5]) * s; q[1] = (M[2] - M[6]) * s; q[2] = (M[3] - M[1]) * s;
  } else {
    int i = 0;
    if (M[4] > M[0]) i = 1;
    if (M[8] > M[4 * i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    double s = sqrt(M[4 * i] - M[4 * j] - M[4 * k] + 1.0);
    q[i] = 0.5 * s; s = 0.5 / s;
    q[3] = (M[3 * k + j] - M[3 * j + k]) * s;
    q[j] = (M[3 * j + i] + M[3 * i + j]) * s;
    q[k] = (M[3 * k + i] + M[3 * i + k]) * s;
  }
}

// FrameAbsolutePoseSacProblem::getSelectedDistancesToModel for one correspondence: model (R, t) = T_WS, the camera's
// (C_SC row-major, r_SC)
__device__ __forceinline__ double rs_score(const double* R, const double* t, const double* cd, const double* ext) {
  double body[3];
  for (int r = 0; r < 3; ++r) {
    const double ti = -(R[r] * t[0] + R[3 + r] * t[1] + R[6 + r] * t[2]);
    body[r] = R[r] * cd[0] + R[3 + r] * cd[1] + R[6 + r] * cd[2] + ti;
  }
  const double v[3] = {body[0] - ext[9], body[1] - ext[10], body[2] - ext[11]};
  double rep[3];
  for (int r = 0; r < 3; ++r) rep[r] = ext[r] * v[0] + ext[3 + r] * v[1] + ext[6 + r] * v[2];
  const double nrm = sqrt(rs_dot(rep, rep));
  const double e[3] = {rep[0] / nrm - cd[3], rep[1] / nrm - cd[4], rep[2] / nrm - cd[5]};
  return rs_dot(e, e) / cd[9];
}

__global__ void __launch_bounds__(RS_T) k_ransac_3d2d(const RansacJobDev* __restrict__ jobs) {
  __shared__ int s_warp[RS_T / 32];
  __shared__ double s_ext[RS_MAX_CAMS][12];         // C_SC (row-major), r_SC
  __shared__ double s_model[RS_MAX_HYP][12];        // R (row-major), t
  __shared__ int s_cnt[RS_MAX_HYP];
  __shared__ int s_ok[RS_MAX_HYP];
  __shared__ int s_best;
  const RansacJobDev& J = jobs[blockIdx.x];
  const WinDev& W = *J.W;
  const FeatStore& F = *W.feat;
  const int tid = threadIdx.x;
  okb_ransac_result res;
  memset(&res, 0, sizeof res);
  res.best = -1;
  if (W.st->g.K < 2) {                              // Frontend.cpp:579-582
    res.ret = 1;
    if (tid == 0) *J.res = res;
    for (int h = tid; h < J.n_hyp; h += RS_T) J.hyp[h] = 0;
    return;
  }
  // observation counts (landmark.observations.size())
  const int L = min(lm_slots(W), J.cnt_cap);
  for (int i = tid; i < J.cnt_cap; i += RS_T) J.cnt[i] = 0;
  if (tid < J.n_cams) {
    XfQ T;
    const double* E = W.ext + 7 * (size_t)tid;
    xfq_make(E, E + 3, T);
    for (int k = 0; k < 9; ++k) s_ext[tid][k] = T.C[k];
    for (int k = 0; k < 3; ++k) s_ext[tid][9 + k] = T.r[k];
  }
  __syncthreads();
  lm_count_obs<RS_T>(W, J.cnt, L);
  __syncthreads();
  // the adapter's correspondences, cameras ascending, keypoints ascending
  int n = 0;
  for (int cam = 0; cam < J.n_cams; ++cam) {
    const int nk = F.n[(size_t)J.feat * F.C + cam];
    const size_t base = ((size_t)J.feat * F.C + cam) * F.N;
    CamIntr ci;
    cam_load(W.cams[cam], ci);
    for (int k0 = 0; k0 < nk; k0 += RS_T) {
      const int k = k0 + tid;
      int take = 0, l = -1;
      if (k < nk) {
        l = F.lm[base + k];
        if (track_live(W, L, l) && J.cnt[l] >= 2 && fabs(lm_point(W, l)[3]) >= 1.0e-8) take = 1;
      }
      int total;
      const int pos = block_scan<RS_T>(take, s_warp, &total);
      if (take) {
        double* cd = J.cd + (size_t)(n + pos) * RS_CD;
        const double* hp = lm_point(W, l);
        for (int r = 0; r < 3; ++r) cd[r] = hp[r] / hp[3];
        // PinholeCamera::backProject (its return value ignored), then bearing.normalize()
        double pu[2];
        undistort_gn(ci, (F.kp[2 * (base + k)] - ci.cu) * (1.0 / ci.fu), (F.kp[2 * (base + k) + 1] - ci.cv) * (1.0 / ci.fv), pu);
        double br[3] = {pu[0], pu[1], 1.0};
        const double n2 = rs_dot(br, br);
        if (n2 > 0.0) { const double in = sqrt(n2); br[0] /= in; br[1] /= in; br[2] /= in; }
        for (int r = 0; r < 3; ++r) cd[3 + r] = br[r];
        for (int r = 0; r < 3; ++r) cd[6 + r] = s_ext[cam][3 * r] * br[0] + s_ext[cam][3 * r + 1] * br[1] + s_ext[cam][3 * r + 2] * br[2];
        const double sd = 0.8 * F.size[base + k] / 12.0;
        cd[9] = sqrt(2.0) * sd * sd / (ci.fu * ci.fu);
        int* cr = J.ci + 3 * (size_t)(n + pos);
        cr[0] = cam; cr[1] = k; cr[2] = l;
      }
      n += total;
    }
  }
  res.n_correspondences = n;
  if (n < 5) {                                      // Frontend.cpp:593-596
    res.ret = n;
    if (tid == 0) *J.res = res;
    for (int h = tid; h < J.n_hyp; h += RS_T) J.hyp[h] = 0;
    return;
  }
  __syncthreads();                                  // the correspondences are in global scratch
  // hypotheses, a thread each
  if (tid < J.n_hyp) {
    int idx[4];
    int ok = 0;
    if (rs_sample<4>(J.seed, tid, n, idx)) {
      const double* q[4];
      bool finite = true;
      for (int i = 0; i < 4; ++i) {
        q[i] = J.cd + (size_t)idx[i] * RS_CD;
        finite = finite && isfinite(q[i][3] + q[i][4] + q[i][5]);
      }
      if (finite) {
        double c[3][3], f[3][3], X[3][3];
        for (int i = 0; i < 3; ++i) {
          const int cam = J.ci[3 * (size_t)idx[i]];
          for (int k = 0; k < 3; ++k) { c[i][k] = s_ext[cam][9 + k]; f[i][k] = q[i][6 + k]; X[i][k] = q[i][k]; }
        }
        const double* ext4 = s_ext[J.ci[3 * (size_t)idx[3]]];
        double best = INFINITY;
        rs_gp3p(c, f, X, [&](const double* R, const double* t) {
          const double sc = rs_score(R, t, q[3], ext4);
          if (sc < best) {
            best = sc;
            for (int k = 0; k < 9; ++k) s_model[tid][k] = R[k];
            for (int k = 0; k < 3; ++k) s_model[tid][9 + k] = t[k];
          }
        });
        ok = best < INFINITY ? 1 : 0;
      }
    }
    s_ok[tid] = ok;
  }
  __syncthreads();
  // inliers of every hypothesis, a warp each
  const int lane = tid & 31, warp = tid >> 5;
  for (int h = warp; h < J.n_hyp; h += RS_T / 32) {
    int cnt = 0;
    if (s_ok[h])
      for (int k = lane; k < n; k += 32) {
        const double* cd = J.cd + (size_t)k * RS_CD;
        cnt += rs_score(s_model[h], s_model[h] + 9, cd, s_ext[J.ci[3 * (size_t)k]]) < J.threshold ? 1 : 0;
      }
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if (lane == 0) s_cnt[h] = cnt;
  }
  __syncthreads();
  if (tid == 0) {
    int best = -1, bc = -1;
    for (int h = 0; h < J.n_hyp; ++h) {
      J.hyp[h] = s_cnt[h];
      if (s_ok[h] && s_cnt[h] > bc) { best = h; bc = s_cnt[h]; }
    }
    s_best = best;
  }
  __syncthreads();
  const int best = s_best;
  res.best = best;
  res.n_inliers = best >= 0 ? s_cnt[best] : 0;
  res.ret = res.n_inliers;
  if (best >= 0) {
    const double* M = s_model[best];
    double q[4];
    rs_quat(M, q);
    for (int r = 0; r < 3; ++r) res.T_WS[r] = M[9 + r];
    for (int r = 0; r < 4; ++r) res.T_WS[3 + r] = q[r];
  }
  // Frontend.cpp:613-640: with at least 10 inliers, every other correspondence is removed
  int n_out = 0;
  if (res.n_inliers >= 10) {
    const double* M = s_model[best];
    for (int k0 = 0; k0 < n; k0 += RS_T) {
      const int k = k0 + tid;
      int o = 0;
      if (k < n) o = rs_score(M, M + 9, J.cd + (size_t)k * RS_CD, s_ext[J.ci[3 * (size_t)k]]) < J.threshold ? 0 : 1;
      int total;
      const int pos = block_scan<RS_T>(o, s_warp, &total);
      if (o) {
        const int* cr = J.ci + 3 * (size_t)k;
        J.outl[n_out + pos] = okb_ransac_outlier{cr[0], cr[1], cr[2]};
      }
      n_out += total;
    }
  }
  res.n_outliers = n_out;
  if (tid == 0) *J.res = res;
}
}  // namespace

// Host checks of one job; "" = valid.
static std::string ransac_job_invalid(okb_ctx* c, const okb_ransac_job& j, std::vector<char>& seen) {
  const std::string why = store_window_invalid(c, j.win, seen);
  if (!why.empty()) return why;
  const WinStore& S = c->wins[j.win];
  const WinDev& W = c->host[j.win];
  const FeatStore& F = S.feat;
  if (j.feat_slot < 0 || j.feat_slot >= F.F) return "feat_slot out of range";
  if (j.n_cams < 1 || j.n_cams > F.C || j.n_cams > W.NE || j.n_cams > W.NC || j.n_cams > RS_MAX_CAMS)
    return "n_cams out of range (1..the store's cameras, the window's extrinsics and cameras, 16)";
  size_t n_kp = 0;
  for (int cam = 0; cam < j.n_cams; ++cam) {
    const int nk = S.feat_n_pending[(size_t)j.feat_slot * F.C + cam];
    if (nk < 0) return "feature slot has no keypoints for camera " + std::to_string(cam);
    n_kp += nk;
  }
  if (j.max_iterations < 1 || j.max_iterations > RS_MAX_HYP) return "max_iterations out of range (1..64)";
  if (!(j.threshold > 0.0) || !std::isfinite(j.threshold)) return "threshold not finite and positive";
  if (!j.out) return "out missing";
  if ((size_t)std::max(j.outlier_cap, 0) < n_kp || (n_kp && !j.outliers)) return "outlier capacity below the frame's keypoints";
  return "";
}

extern "C" int okb_ransac_3d2d_batch(okb_ctx* c, int n_jobs, const okb_ransac_job* jobs) {
  int rc = store_call_checks(c, "okb_ransac_3d2d_batch", n_jobs, jobs, INT_MAX,
                             [&](int i, std::vector<char>& seen) { return ransac_job_invalid(c, jobs[i], seen); });
  if (rc || n_jobs == 0) return rc;
  cudaSetDevice(c->device);
  okb_frontend_state* F = fe(c);
  CallBuffers& B = F->ransac;
  std::lock_guard<std::mutex> lk(B.mtx);
  if ((rc = commit_job_windows(c, jobs, n_jobs))) return rc;
  if ((rc = shard_lm_exchange(c, "okb_ransac_3d2d_batch", jobs, n_jobs, c->stream_xfer))) return rc;
  cudaStream_t xs = c->stream_xfer;
  // staging (pinned + device mirror): in  = [job table]
  //                                   out = [per job: result | hypothesis inliers | outlier records]
  // scratch (device only), per job: observation counts | correspondences | their indices
  Carve st, sc;
  st.take(sizeof(RansacJobDev) * (size_t)n_jobs, 256);
  const size_t in_bytes = st.off;
  std::vector<size_t> o_res(n_jobs), o_hyp(n_jobs), o_out(n_jobs), o_cnt(n_jobs), o_cd(n_jobs), o_ci(n_jobs);
  std::vector<int> n_kp(n_jobs, 0);
  for (int i = 0; i < n_jobs; ++i) {
    const okb_ransac_job& j = jobs[i];
    const WinStore& S = c->wins[j.win];
    for (int cam = 0; cam < j.n_cams; ++cam) n_kp[i] += S.feat_n_pending[(size_t)j.feat_slot * S.feat.C + cam];
    o_res[i] = st.take(sizeof(okb_ransac_result));
    o_hyp[i] = st.take(4 * (size_t)j.max_iterations);
    o_out[i] = st.take(sizeof(okb_ransac_outlier) * (size_t)n_kp[i]);
    o_cnt[i] = sc.take(4 * (size_t)lm_slots_host(c, j.win));
    o_cd[i] = sc.take(8 * RS_CD * (size_t)n_kp[i]);
    o_ci[i] = sc.take(12 * (size_t)n_kp[i]);
  }
  const size_t out_end = st.off;
  if ((rc = B.reserve(c, out_end, sc.off))) return rc;
  uint8_t* h = B.h_stage;
  uint8_t* d = B.d_stage;
  RansacJobDev* tj = reinterpret_cast<RansacJobDev*>(h);
  for (int i = 0; i < n_jobs; ++i) {
    const okb_ransac_job& j = jobs[i];
    RansacJobDev J;
    std::memset(&J, 0, sizeof J);
    J.W = c->d_wins + j.win;
    J.feat = j.feat_slot; J.n_cams = j.n_cams; J.n_hyp = j.max_iterations;
    J.cnt_cap = lm_slots_host(c, j.win);
    J.threshold = j.threshold;
    J.seed = (unsigned long long)j.seed;
    J.cnt = reinterpret_cast<int*>(B.d_scratch + o_cnt[i]);
    J.cd = reinterpret_cast<double*>(B.d_scratch + o_cd[i]);
    J.ci = reinterpret_cast<int*>(B.d_scratch + o_ci[i]);
    J.res = reinterpret_cast<okb_ransac_result*>(d + o_res[i]);
    J.hyp = reinterpret_cast<int*>(d + o_hyp[i]);
    J.outl = reinterpret_cast<okb_ransac_outlier*>(d + o_out[i]);
    tj[i] = J;
  }
  OKB_CUDA(c, cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, xs));
  k_ransac_3d2d<<<n_jobs, RS_T, 0, xs>>>(reinterpret_cast<const RansacJobDev*>(d));
  F->launches += 1;
  OKB_CUDA(c, cudaGetLastError());
  OKB_CUDA(c, cudaMemcpyAsync(h + in_bytes, d + in_bytes, out_end - in_bytes, cudaMemcpyDeviceToHost, xs));
  OKB_CUDA(c, cudaStreamSynchronize(xs));
  for (int i = 0; i < n_jobs; ++i) {
    const okb_ransac_job& j = jobs[i];
    *j.out = *reinterpret_cast<const okb_ransac_result*>(h + o_res[i]);
    if (j.hyp_inliers) std::memcpy(j.hyp_inliers, h + o_hyp[i], 4 * (size_t)j.max_iterations);
    if (j.out->n_outliers) std::memcpy(j.outliers, h + o_out[i], sizeof(okb_ransac_outlier) * (size_t)j.out->n_outliers);
  }
  return OKB_OK;
}

// =================================================================================================
// 2D-2D outlier rejection and pose initialisation (okb_ransac_2d2d_batch): Frontend::runRansac2d2d
// (okvis_frontend/src/Frontend.cpp:645-810) on the window's feature store, one CTA per job in one launch (DESIGN.md 6i;
// tests/ransac2d2d_reference.py restates it):
//   1. per camera, FrameRelativeAdapter's correspondences (FrameRelativeAdapter.cpp:139-244): B's first keypoint per
//      landmark of the graph by an atomicMin over the landmark slots, then A's keypoints compacted in order by a block
//      scan;
//   2. one thread per (camera, problem, hypothesis): the two-point rotation or the five-point relative pose, the 6th
//      correspondence choosing among the five-point solutions;
//   3. a warp per (camera, problem, hypothesis) counts its inliers; thread 0 takes the winners, the reference's decision
//      and the pose initialisation camera by camera;
//   4. the outlier records of the applied cameras in correspondence order (block scan).
// The call writes nothing but its scratch and its results.
// =================================================================================================
namespace {
constexpr int R2_CD = 8;           // doubles per correspondence: bearing A (3), bearing B (3), sigmaAngle A, sigmaAngle B
constexpr int R2_TASKS = RS_MAX_CAMS * 2 * RS_MAX_HYP;
constexpr double R2_CONS_TOL = 1e-10;  // an essential matrix is kept when its constraints hold to this, relative to |E|^3

struct Ransac2JobDev {
  const WinDev* W;
  int feat_a, feat_b, pose_a, pose_b, n_cams, n_hyp, init_pose, L;
  double threshold;
  unsigned long long seed;
  int* first;                      // [L] B's first keypoint per landmark slot (scratch)
  double* cd;                      // [sum of A's keypoints][R2_CD] correspondences (scratch)
  int* ci;                         // [sum of A's keypoints][3] kp_a, kp_b, landmark slot (scratch)
  double* model;                   // [n_cams][2][n_hyp][12] R (row-major), t (scratch)
  okb_ransac2d_result* res;
  okb_ransac2d_cam* cams;          // [n_cams]
  int* hyp;                        // [n_cams][2][n_hyp]
  okb_ransac2d_outlier* outl;
};

// Monomial tables of the five-point constraints.  Linear: x, y, z, 1.  Quadratic: x^2, y^2, z^2, xy, xz, yz, x, y, z, 1.
// Cubic (Nister's order): x^3, y^3, x^2y, xy^2, x^2z, x^2, y^2z, y^2, xyz, xy | xz^2, xz, x, yz^2, yz, y, z^3, z^2, z, 1.
__constant__ int8_t c_r2_ll[4][4] = {{0, 3, 4, 6}, {3, 1, 5, 7}, {4, 5, 2, 8}, {6, 7, 8, 9}};
__constant__ int8_t c_r2_ql[10][4] = {{0, 2, 4, 5}, {3, 1, 6, 7}, {10, 13, 16, 17}, {2, 3, 8, 9}, {4, 8, 10, 11},
                                      {8, 6, 13, 14}, {5, 9, 11, 12}, {9, 7, 14, 15}, {11, 14, 17, 18}, {12, 15, 18, 19}};
__constant__ int8_t c_r2_exp[20][3] = {{3, 0, 0}, {0, 3, 0}, {2, 1, 0}, {1, 2, 0}, {2, 0, 1}, {2, 0, 0}, {0, 2, 1},
                                       {0, 2, 0}, {1, 1, 1}, {1, 1, 0}, {1, 0, 2}, {1, 0, 1}, {1, 0, 0}, {0, 1, 2},
                                       {0, 1, 1}, {0, 1, 0}, {0, 0, 3}, {0, 0, 2}, {0, 0, 1}, {0, 0, 0}};

__device__ __forceinline__ void r2_cross(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1]; c[1] = a[2] * b[0] - a[0] * b[2]; c[2] = a[0] * b[1] - a[1] * b[0];
}

// triangulate2 as specified (DESIGN.md 6i): the midpoint of the common perpendicular of l1 f1 and t + l2 R f2, the 2x2
// normal equations solved in closed form; l = (l1, l2)
__device__ __forceinline__ void r2_triangulate(const double* R, const double* t, const double* f1, const double* f2, double* p, double* l) {
  double g[3];
  for (int r = 0; r < 3; ++r) g[r] = R[3 * r] * f2[0] + R[3 * r + 1] * f2[1] + R[3 * r + 2] * f2[2];
  const double a = rs_dot(f1, f1), b = rs_dot(f1, g), c = rs_dot(g, g), d1 = rs_dot(f1, t), d2 = rs_dot(g, t);
  const double det = a * c - b * b;
  l[0] = (c * d1 - b * d2) / det;
  l[1] = (b * d1 - a * d2) / det;
  for (int k = 0; k < 3; ++k) p[k] = 0.5 * (l[0] * f1[k] + (t[k] + l[1] * g[k]));
}

// FrameRotationOnlySacProblem::getSelectedDistancesToModel for one correspondence.  Not inlined: the inlier count and
// the outlier scan call one compiled body, so a score within rounding of the threshold decides both alike.
__device__ __noinline__ double r2_score_rot(const double* R, const double* cd) {
  double e1[3], e2[3];
  for (int r = 0; r < 3; ++r) {
    e1[r] = R[3 * r] * cd[3] + R[3 * r + 1] * cd[4] + R[3 * r + 2] * cd[5] - cd[r];
    e2[r] = R[r] * cd[0] + R[3 + r] * cd[1] + R[6 + r] * cd[2] - cd[3 + r];
  }
  return rs_dot(e1, e1) * 0.5 / cd[6] + rs_dot(e2, e2) * 0.5 / cd[7];
}

// FrameRelativePoseSacProblem::getSelectedDistancesToModel for one correspondence (not inlined, as r2_score_rot)
__device__ __noinline__ double r2_score_rel(const double* R, const double* t, const double* cd) {
  double p[3], l[2], q[3];
  r2_triangulate(R, t, cd, cd + 3, p, l);
  for (int r = 0; r < 3; ++r) {
    const double ti = -(R[r] * t[0] + R[3 + r] * t[1] + R[6 + r] * t[2]);
    q[r] = R[r] * p[0] + R[3 + r] * p[1] + R[6 + r] * p[2] + ti;
  }
  const double n1 = sqrt(rs_dot(p, p)), n2 = sqrt(rs_dot(q, q));
  const double e1[3] = {p[0] / n1 - cd[0], p[1] / n1 - cd[1], p[2] / n1 - cd[2]};
  const double e2[3] = {q[0] / n2 - cd[3], q[1] / n2 - cd[4], q[2] / n2 - cd[5]};
  return rs_dot(e1, e1) * 0.5 / cd[6] + rs_dot(e2, e2) * 0.5 / cd[7];
}

// Two-point rotation: R maps B's triad of (f_a + f_b, f_a x f_b) onto A's (R f2 = f1 for both points when noise-free)
__device__ bool r2_rotation(const double* a0, const double* b0, const double* a1, const double* b1, double* R) {
  double FA[3][3], FB[3][3];
  for (int side = 0; side < 2; ++side) {
    const double* u = side ? b0 : a0;
    const double* v = side ? b1 : a1;
    const double s[3] = {u[0] + v[0], u[1] + v[1], u[2] + v[2]};
    double nn[3];
    r2_cross(u, v, nn);
    rs_triad(s, nn, side ? FB : FA);
  }
  double sum = 0.0;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      R[3 * r + c] = FA[0][r] * FB[0][c] + FA[1][r] * FB[1][c] + FA[2][r] * FB[2][c];
      sum += R[3 * r + c];
    }
  return isfinite(sum);
}

__device__ __forceinline__ double r2_det3(const double (*A)[3]) {
  return A[0][0] * (A[1][1] * A[2][2] - A[1][2] * A[2][1]) - A[0][1] * (A[1][0] * A[2][2] - A[1][2] * A[2][0]) +
         A[0][2] * (A[1][0] * A[2][1] - A[1][1] * A[2][0]);
}

// RS_POLISH Gauss-Newton steps of (x, y, z) on the 10 cubic constraints G0 (before elimination), the 3x3 normal
// equations solved by Cramer's rule; stops at a singular or non-finite system
__device__ void r2_polish(const double (*G0)[20], double& x, double& y, double& z) {
  if (!isfinite(x + y + z)) return;
  for (int it = 0; it < RS_POLISH; ++it) {
    const double px[4] = {1.0, x, x * x, x * x * x}, py[4] = {1.0, y, y * y, y * y * y}, pz[4] = {1.0, z, z * z, z * z * z};
    double g[10], Jm[10][3];
    for (int i = 0; i < 10; ++i) { g[i] = 0.0; Jm[i][0] = Jm[i][1] = Jm[i][2] = 0.0; }
    for (int m = 0; m < 20; ++m) {
      const int a = c_r2_exp[m][0], b = c_r2_exp[m][1], c = c_r2_exp[m][2];
      const double mon = px[a] * py[b] * pz[c];
      const double dx = a * px[max(a - 1, 0)] * py[b] * pz[c];
      const double dy = b * px[a] * py[max(b - 1, 0)] * pz[c];
      const double dw = c * px[a] * py[b] * pz[max(c - 1, 0)];
      for (int i = 0; i < 10; ++i) {
        g[i] += G0[i][m] * mon;
        Jm[i][0] += G0[i][m] * dx; Jm[i][1] += G0[i][m] * dy; Jm[i][2] += G0[i][m] * dw;
      }
    }
    double A[3][3], bb[3];
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) {
        double s = 0.0;
        for (int k = 0; k < 10; ++k) s += Jm[k][r] * Jm[k][c];
        A[r][c] = s;
      }
      double s = 0.0;
      for (int k = 0; k < 10; ++k) s += Jm[k][r] * g[k];
      bb[r] = s;
    }
    const double det = r2_det3(A);
    if (!(det != 0.0) || !isfinite(det)) return;
    double d[3];
    for (int v = 0; v < 3; ++v) {
      double Av[3][3];
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) Av[r][c] = c == v ? bb[r] : A[r][c];
      d[v] = r2_det3(Av) / det;
    }
    x -= d[0]; y -= d[1]; z -= d[2];
  }
}

// Five-point relative pose (Nister's formulation, DESIGN.md 6i) on correspondences (f1[i], f2[i]), i = 0..4, with
// f1^T E f2 = 0, E = [t]x R: the null space of the 5x9 epipolar system by Householder QR, E = x X + y Y + z Z + W, the
// 10 cubic constraints Gauss-Jordan eliminated (partial pivoting), the degree-10 polynomial in z, its real roots, (x, y)
// from the first two rows of the 3x3 polynomial system, RS_POLISH Gauss-Newton steps of (x, y, z) on the 10 cubic
// constraints, E kept when det E and 2 E E^T E - tr(E E^T) E vanish to R2_CONS_TOL |E|^3, and per root the 4 (R, t)
// candidates of E.  emit(R, t) per
// candidate whose 5 points triangulate in front of both cameras (l1 > 0, l2 > 0), roots ascending, candidates in the
// order (R1, t), (R1, -t), (R2, t), (R2, -t).
template <typename Emit>
__device__ void r2_fivept(const double (*f1)[3], const double (*f2)[3], Emit&& emit) {
  double M[9][5];                                   // the epipolar system, transposed
  for (int i = 0; i < 5; ++i)
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) M[3 * r + c][i] = f1[i][r] * f2[i][c];
  double V[5][9], beta[5];
  for (int j = 0; j < 5; ++j) {
    double nx = 0.0;
    for (int i = j; i < 9; ++i) nx += M[i][j] * M[i][j];
    nx = sqrt(nx);
    const double alpha = M[j][j] < 0.0 ? nx : -nx;
    for (int i = 0; i < 9; ++i) V[j][i] = i < j ? 0.0 : M[i][j];
    V[j][j] -= alpha;
    double b = 0.0;
    for (int i = j; i < 9; ++i) b += V[j][i] * V[j][i];
    beta[j] = b;
    if (!(b > 0.0)) continue;
    for (int k = j; k < 5; ++k) {
      double s = 0.0;
      for (int i = j; i < 9; ++i) s += V[j][i] * M[i][k];
      s = 2.0 * s / b;
      for (int i = j; i < 9; ++i) M[i][k] -= s * V[j][i];
    }
  }
  double N[4][9];                                   // X, Y, Z, W = Q e_5 .. Q e_8
  for (int b4 = 0; b4 < 4; ++b4) {
    for (int i = 0; i < 9; ++i) N[b4][i] = i == 5 + b4 ? 1.0 : 0.0;
    for (int j = 4; j >= 0; --j) {
      if (!(beta[j] > 0.0)) continue;
      double s = 0.0;
      for (int i = j; i < 9; ++i) s += V[j][i] * N[b4][i];
      s = 2.0 * s / beta[j];
      for (int i = j; i < 9; ++i) N[b4][i] -= s * V[j][i];
    }
  }
  double G[10][20];                                 // row 0: det E; rows 1..9: 2 E E^T E - tr(E E^T) E, row-major
  {
    double EE[3][3][10];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        for (int q = 0; q < 10; ++q) EE[r][c][q] = 0.0;
        for (int k = 0; k < 3; ++k)
          for (int i = 0; i < 4; ++i)
            for (int j = 0; j < 4; ++j) EE[r][c][c_r2_ll[i][j]] += N[i][3 * r + k] * N[j][3 * c + k];
      }
    double tr[10];
    for (int q = 0; q < 10; ++q) tr[q] = EE[0][0][q] + EE[1][1][q] + EE[2][2][q];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        double S[20], T[20];
        for (int m = 0; m < 20; ++m) S[m] = T[m] = 0.0;
        for (int k = 0; k < 3; ++k)
          for (int q = 0; q < 10; ++q)
            for (int i = 0; i < 4; ++i) S[c_r2_ql[q][i]] += EE[r][k][q] * N[i][3 * k + c];
        for (int q = 0; q < 10; ++q)
          for (int i = 0; i < 4; ++i) T[c_r2_ql[q][i]] += tr[q] * N[i][3 * r + c];
        for (int m = 0; m < 20; ++m) G[1 + 3 * r + c][m] = 2.0 * S[m] - T[m];
      }
    // det E = E00 (E11 E22 - E12 E21) - E01 (E10 E22 - E12 E20) + E02 (E10 E21 - E11 E20)
    for (int m = 0; m < 20; ++m) G[0][m] = 0.0;
    const int cof[3][4] = {{4, 8, 5, 7}, {3, 8, 5, 6}, {3, 7, 4, 6}};
    const double sg[3] = {1.0, -1.0, 1.0};
    for (int e = 0; e < 3; ++e) {
      double mq[10];
      for (int q = 0; q < 10; ++q) mq[q] = 0.0;
      for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
          mq[c_r2_ll[i][j]] += N[i][cof[e][0]] * N[j][cof[e][1]] - N[i][cof[e][2]] * N[j][cof[e][3]];
      for (int q = 0; q < 10; ++q)
        for (int i = 0; i < 4; ++i) G[0][c_r2_ql[q][i]] += sg[e] * (N[i][e] * mq[q]);
    }
  }
  double G0[10][20];
  for (int i = 0; i < 10; ++i)
    for (int m = 0; m < 20; ++m) G0[i][m] = G[i][m];
  for (int j = 0; j < 10; ++j) {                    // Gauss-Jordan, partial pivoting (first largest)
    int p = j;
    for (int i = j + 1; i < 10; ++i)
      if (fabs(G[i][j]) > fabs(G[p][j])) p = i;
    if (!(G[p][j] != 0.0) || !isfinite(G[p][j])) return;
    if (p != j)
      for (int m = j; m < 20; ++m) { const double tmp = G[j][m]; G[j][m] = G[p][m]; G[p][m] = tmp; }
    const double piv = G[j][j];
    for (int m = j; m < 20; ++m) G[j][m] /= piv;
    for (int i = 0; i < 10; ++i) {
      if (i == j) continue;
      const double f = G[i][j];
      for (int m = j; m < 20; ++m) G[i][m] -= f * G[j][m];
    }
  }
  // k = <e> - z <f>, l = <g> - z <h>, m = <i> - z <j>: rows (4, 5), (6, 7), (8, 9); P[row][0: x, 1: y, 2: 1][power of z]
  double P[3][3][5];
  for (int r = 0; r < 3; ++r) {
    const double* a = G[4 + 2 * r];
    const double* b = G[5 + 2 * r];
    P[r][0][0] = a[12]; P[r][0][1] = a[11] - b[12]; P[r][0][2] = a[10] - b[11]; P[r][0][3] = -b[10]; P[r][0][4] = 0.0;
    P[r][1][0] = a[15]; P[r][1][1] = a[14] - b[15]; P[r][1][2] = a[13] - b[14]; P[r][1][3] = -b[13]; P[r][1][4] = 0.0;
    P[r][2][0] = a[19]; P[r][2][1] = a[18] - b[19]; P[r][2][2] = a[17] - b[18]; P[r][2][3] = a[16] - b[17]; P[r][2][4] = -b[16];
  }
  double dz[11];
  {
    double t1[8], t2[8], t3[7], u[11];
    rs_umul(P[1][1], 3, P[2][2], 4, t1); rs_umul(P[1][2], 4, P[2][1], 3, u);  for (int i = 0; i < 8; ++i) t1[i] -= u[i];
    rs_umul(P[1][0], 3, P[2][2], 4, t2); rs_umul(P[1][2], 4, P[2][0], 3, u);  for (int i = 0; i < 8; ++i) t2[i] -= u[i];
    rs_umul(P[1][0], 3, P[2][1], 3, t3); rs_umul(P[1][1], 3, P[2][0], 3, u);  for (int i = 0; i < 7; ++i) t3[i] -= u[i];
    rs_umul(P[0][0], 3, t1, 7, dz);
    rs_umul(P[0][1], 3, t2, 7, u);  for (int i = 0; i < 11; ++i) dz[i] -= u[i];
    rs_umul(P[0][2], 4, t3, 6, u);  for (int i = 0; i < 11; ++i) dz[i] += u[i];
  }
  double roots[10];
  const int nr = rs_real_roots<10, true>(dz, roots);
  for (int ir = 0; ir < nr; ++ir) {
    double row[2][3];
    for (int r = 0; r < 2; ++r)
      for (int v = 0; v < 3; ++v) row[r][v] = rs_horner(P[r][v], 4, roots[ir]);
    double u[3];
    r2_cross(row[0], row[1], u);
    if (!(u[2] != 0.0) || !isfinite(u[0] + u[1] + u[2])) continue;
    double x = u[0] / u[2], y = u[1] / u[2], z = roots[ir];
    r2_polish(G0, x, y, z);
    double E[9], ss = 0.0;
    for (int e = 0; e < 9; ++e) {
      E[e] = x * N[0][e] + y * N[1][e] + z * N[2][e] + N[3][e];
      ss += E[e] * E[e];
    }
    if (!(ss > 0.0) || !isfinite(ss)) continue;
    const double sc = sqrt(2.0) / sqrt(ss);
    for (int e = 0; e < 9; ++e) E[e] *= sc;
    {                                               // det E = 0, 2 E E^T E - tr(E E^T) E = 0 to R2_CONS_TOL |E|^3
      double EEt[9], worst = 0.0;
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) EEt[3 * i + j] = E[3 * i] * E[3 * j] + E[3 * i + 1] * E[3 * j + 1] + E[3 * i + 2] * E[3 * j + 2];
      const double tr = EEt[0] + EEt[4] + EEt[8];
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
          worst = fmax(worst, fabs(2.0 * (EEt[3 * i] * E[j] + EEt[3 * i + 1] * E[3 + j] + EEt[3 * i + 2] * E[6 + j]) - tr * E[3 * i + j]));
      const double Em[3][3] = {{E[0], E[1], E[2]}, {E[3], E[4], E[5]}, {E[6], E[7], E[8]}};
      worst = fmax(worst, fabs(r2_det3(Em)));
      if (!(worst <= R2_CONS_TOL * 2.0 * sqrt(2.0))) continue;
    }
    // t: the left null vector of E, the largest cross product of two of its columns
    double col[3][3], t[3], tn = -1.0;
    for (int c = 0; c < 3; ++c)
      for (int r = 0; r < 3; ++r) col[c][r] = E[3 * r + c];
    const int pr[3][2] = {{0, 1}, {0, 2}, {1, 2}};
    for (int e = 0; e < 3; ++e) {
      double w[3];
      r2_cross(col[pr[e][0]], col[pr[e][1]], w);
      const double wn = sqrt(rs_dot(w, w));
      if (wn > tn) { tn = wn; for (int k = 0; k < 3; ++k) t[k] = w[k]; }
    }
    if (!(tn > 0.0)) continue;
    for (int k = 0; k < 3; ++k) t[k] /= tn;
    // E = +-[t]x R: R1 = cof(E) - [t]x E, R2 = cof(E) + [t]x E
    double Rs[2][9];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        const double cf = E[3 * i1 + j1] * E[3 * i2 + j2] - E[3 * i1 + j2] * E[3 * i2 + j1];
        const double tx = t[i1] * E[3 * i2 + j] - t[i2] * E[3 * i1 + j];
        Rs[0][3 * i + j] = cf - tx;
        Rs[1][3 * i + j] = cf + tx;
      }
    for (int cand = 0; cand < 4; ++cand) {
      const double* R = Rs[cand >> 1];
      const double sgn = (cand & 1) ? -1.0 : 1.0;
      const double tc[3] = {sgn * t[0], sgn * t[1], sgn * t[2]};
      bool ok = true;
      for (int i = 0; i < 5 && ok; ++i) {
        double p[3], l[2];
        r2_triangulate(R, tc, f1[i], f2[i], p, l);
        ok = l[0] > 0.0 && l[1] > 0.0;
      }
      if (ok) emit(R, tc);
    }
  }
}

__global__ void __launch_bounds__(RS_T) k_ransac_2d2d(const Ransac2JobDev* __restrict__ jobs) {
  __shared__ int s_warp[RS_T / 32];
  __shared__ int s_off[RS_MAX_CAMS + 1];            // correspondences of camera c: [s_off[c], s_off[c + 1])
  __shared__ int s_cnt[R2_TASKS];
  __shared__ unsigned char s_ok[R2_TASKS];
  __shared__ int s_pick[RS_MAX_CAMS];               // the applied camera's chosen task, -1: not applied
  const Ransac2JobDev& J = jobs[blockIdx.x];
  const WinDev& W = *J.W;
  const FeatStore& F = *W.feat;
  const int tid = threadIdx.x, H = J.n_hyp;
  for (int i = tid; i < J.L; i += RS_T) J.first[i] = INT_MAX;
  __syncthreads();
  // the adapter's correspondences, per camera
  int n = 0;
  for (int cam = 0; cam < J.n_cams; ++cam) {
    if (tid == 0) s_off[cam] = n;
    const int nA = F.n[(size_t)J.feat_a * F.C + cam], nB = F.n[(size_t)J.feat_b * F.C + cam];
    const size_t bA = ((size_t)J.feat_a * F.C + cam) * F.N, bB = ((size_t)J.feat_b * F.C + cam) * F.N;
    for (int k = tid; k < nB; k += RS_T) {
      const int l = F.lm[bB + k];
      if (track_live(W, J.L, l)) atomicMin(&J.first[l], k);
    }
    __syncthreads();
    CamIntr ci;
    cam_load(W.cams[cam], ci);
    for (int k0 = 0; k0 < nA; k0 += RS_T) {
      const int k = k0 + tid;
      int take = 0, l = -1, kb = -1;
      if (k < nA) {
        l = F.lm[bA + k];
        if (l >= 0 && l < J.L) kb = J.first[l];
        take = kb != INT_MAX && kb >= 0 ? 1 : 0;
      }
      int total;
      const int pos = block_scan<RS_T>(take, s_warp, &total);
      if (take) {
        double* cd = J.cd + (size_t)(n + pos) * R2_CD;
        for (int side = 0; side < 2; ++side) {
          const size_t e = side ? bB + kb : bA + k;
          // PinholeCamera::backProject (its return value ignored), then bearing.normalize()
          double pu[2];
          undistort_gn(ci, (F.kp[2 * e] - ci.cu) * (1.0 / ci.fu), (F.kp[2 * e + 1] - ci.cv) * (1.0 / ci.fv), pu);
          double br[3] = {pu[0], pu[1], 1.0};
          const double n2 = rs_dot(br, br);
          if (n2 > 0.0) { const double in = sqrt(n2); br[0] /= in; br[1] /= in; br[2] /= in; }
          for (int r = 0; r < 3; ++r) cd[3 * side + r] = br[r];
          const double sd = 0.8 * F.size[e] / 12.0;
          cd[6 + side] = sqrt(2.0) * sd * sd / (ci.fu * ci.fu);
        }
        int* cr = J.ci + 3 * (size_t)(n + pos);
        cr[0] = k; cr[1] = kb; cr[2] = l;
      }
      n += total;
    }
    __syncthreads();
    for (int k = tid; k < nB; k += RS_T) {
      const int l = F.lm[bB + k];
      if (l >= 0 && l < J.L) J.first[l] = INT_MAX;
    }
    __syncthreads();
  }
  if (tid == 0) s_off[J.n_cams] = n;
  __syncthreads();                                  // the correspondences are in global scratch
  // hypotheses, a thread each: task = (2 cam + problem) H + h
  const int n_tasks = J.n_cams * 2 * H;
  for (int task = tid; task < n_tasks; task += RS_T) {
    const int cam = task / (2 * H), prob = (task / H) & 1, h = task % H;
    const int o = s_off[cam], nc = s_off[cam + 1] - o;
    const int key = (2 * cam + prob) * RS_MAX_HYP + h;
    double* Mo = J.model + (size_t)task * 12;
    int ok = 0;
    if (nc >= 10) {
      int idx[6];
      const int k = prob ? 6 : 2;
      if (prob ? rs_sample<6>(J.seed, key, nc, idx) : rs_sample<2>(J.seed, key, nc, idx)) {
        bool finite = true;
        for (int i = 0; i < k; ++i) {
          const double* q = J.cd + (size_t)(o + idx[i]) * R2_CD;
          finite = finite && isfinite(q[0] + q[1] + q[2] + q[3] + q[4] + q[5]);
        }
        if (finite && !prob) {
          const double* q0 = J.cd + (size_t)(o + idx[0]) * R2_CD;
          const double* q1 = J.cd + (size_t)(o + idx[1]) * R2_CD;
          double R[9];
          if (r2_rotation(q0, q0 + 3, q1, q1 + 3, R)) {
            for (int e = 0; e < 9; ++e) Mo[e] = R[e];
            for (int e = 9; e < 12; ++e) Mo[e] = 0.0;
            ok = 1;
          }
        } else if (finite) {
          double a[5][3], b[5][3];
          for (int i = 0; i < 5; ++i) {
            const double* q = J.cd + (size_t)(o + idx[i]) * R2_CD;
            for (int r = 0; r < 3; ++r) { a[i][r] = q[r]; b[i][r] = q[3 + r]; }
          }
          const double* q6 = J.cd + (size_t)(o + idx[5]) * R2_CD;
          double best = INFINITY;
          r2_fivept(a, b, [&](const double* R, const double* t) {
            const double sc = r2_score_rel(R, t, q6);
            if (sc < best) {
              best = sc;
              for (int e = 0; e < 9; ++e) Mo[e] = R[e];
              for (int e = 0; e < 3; ++e) Mo[9 + e] = t[e];
            }
          });
          ok = best < INFINITY ? 1 : 0;
        }
      }
    }
    s_ok[task] = (unsigned char)ok;
  }
  __syncthreads();
  // inliers of every hypothesis, a warp each
  const int lane = tid & 31, warp = tid >> 5;
  for (int task = warp; task < n_tasks; task += RS_T / 32) {
    const int cam = task / (2 * H), prob = (task / H) & 1;
    const int o = s_off[cam], nc = s_off[cam + 1] - o;
    int cnt = 0;
    if (s_ok[task]) {
      const double* Mo = J.model + (size_t)task * 12;
      for (int k = lane; k < nc; k += 32) {
        const double* cd = J.cd + (size_t)(o + k) * R2_CD;
        cnt += (prob ? r2_score_rel(Mo, Mo + 9, cd) : r2_score_rot(Mo, cd)) < J.threshold ? 1 : 0;
      }
    }
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if (lane == 0) s_cnt[task] = cnt;
  }
  __syncthreads();
  if (tid == 0) {
    for (int task = 0; task < n_tasks; ++task) J.hyp[task] = s_cnt[task];
    okb_ransac2d_result res;
    memset(&res, 0, sizeof res);
    bool rot_success = false, rel_success = false;
    int total = 0;
    XfQ T_WSA, T_SCA, T_WS0, T_SC0;
    const double* Pa = W.pose + 7 * (size_t)J.pose_a;
    const double* Pb = W.pose + 7 * (size_t)J.pose_b;
    xfq_make(Pa, Pa + 3, T_WSA);
    xfq_make(Pb, Pb + 3, T_WS0);
    for (int cam = 0; cam < J.n_cams; ++cam) {
      okb_ransac2d_cam cr;
      memset(&cr, 0, sizeof cr);
      cr.n_correspondences = s_off[cam + 1] - s_off[cam];
      cr.rot_best = cr.rel_best = -1;
      for (int k = 0; k < 9; k += 4) cr.R_rot[k] = cr.R_rel[k] = 1.0;
      s_pick[cam] = -1;
      if (cr.n_correspondences >= 10) {             // Frontend.cpp:670-671
        int best[2] = {-1, -1}, bc[2] = {-1, -1};
        for (int prob = 0; prob < 2; ++prob)
          for (int h = 0; h < H; ++h) {
            const int task = (2 * cam + prob) * H + h;
            if (s_ok[task] && s_cnt[task] > bc[prob]) { best[prob] = h; bc[prob] = s_cnt[task]; }
          }
        cr.rot_best = best[0]; cr.rel_best = best[1];
        cr.rot_inliers = best[0] >= 0 ? bc[0] : 0;
        cr.rel_inliers = best[1] >= 0 ? bc[1] : 0;
        if (best[0] >= 0) {
          const double* Mo = J.model + (size_t)((2 * cam) * H + best[0]) * 12;
          for (int k = 0; k < 9; ++k) cr.R_rot[k] = Mo[k];
        }
        if (best[1] >= 0) {
          const double* Mo = J.model + (size_t)((2 * cam + 1) * H + best[1]) * 12;
          for (int k = 0; k < 9; ++k) cr.R_rel[k] = Mo[k];
          for (int k = 0; k < 3; ++k) cr.t_rel[k] = Mo[9 + k];
        }
        // Frontend.cpp:709-733
        const float rot_ratio = float(cr.rot_inliers) / float(cr.n_correspondences);
        const float rel_ratio = float(cr.rel_inliers) / float(cr.n_correspondences);
        if (rot_ratio > rel_ratio || rot_ratio > 0.8f) {
          if (cr.rot_inliers > 10) rot_success = true;
          res.rotation_only = 1;
          cr.rotation_only = 1;
          total += cr.rot_inliers;
        } else {
          if (cr.rel_inliers > 10) rel_success = true;
          total += cr.rel_inliers;
        }
        if (rot_success || rel_success) {
          cr.applied = 1;
          const int prob = cr.rotation_only ? 0 : 1;
          const int b = prob ? best[1] : best[0];
          s_pick[cam] = b >= 0 ? (2 * cam + prob) * H + b : -2;      // -2: no model, every correspondence an outlier
          if (J.init_pose) {                        // Frontend.cpp:756-798
            const double* E = W.ext + 7 * (size_t)cam;
            xfq_make(E, E + 3, T_SCA);
            xfq_make(E, E + 3, T_SC0);
            double Rm[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, tm[3] = {0, 0, 0};
            if (rel_success) {
              if (cr.rel_best >= 0) {
                for (int k = 0; k < 9; ++k) Rm[k] = cr.R_rel[k];
                XfQ a, b2, c2, d, prior;
                xfq_inv(T_SCA, a);
                xfq_inv(T_WSA, b2);
                xfq_mul(a, b2, c2);
                xfq_mul(c2, T_WS0, d);
                xfq_mul(d, T_SC0, prior);
                const double s = fmax(0.0, cr.t_rel[0] * prior.r[0] + cr.t_rel[1] * prior.r[1] + cr.t_rel[2] * prior.r[2]);
                for (int k = 0; k < 3; ++k) tm[k] = cr.t_rel[k] * s;
              }
            } else if (cr.rot_best >= 0) {
              for (int k = 0; k < 9; ++k) Rm[k] = cr.R_rot[k];
            }
            double qm[4];
            rs_quat(Rm, qm);
            XfQ T12, a, b2, c2, inv0;
            xfq_make(tm, qm, T12);
            xfq_mul(T_WSA, T_SCA, a);
            xfq_mul(a, T12, b2);
            xfq_inv(T_SC0, inv0);
            xfq_mul(b2, inv0, c2);
            T_WS0 = c2;
            res.pose_set = 1;
          }
        }
      }
      J.cams[cam] = cr;
    }
    if (rot_success || rel_success) res.ret = total;
    else { res.ret = -1; res.rotation_only = 1; }                   // Frontend.cpp:802-808
    if (res.pose_set) {
      for (int k = 0; k < 3; ++k) res.T_WS[k] = T_WS0.r[k];
      for (int k = 0; k < 4; ++k) res.T_WS[3 + k] = T_WS0.q[k];
    }
    *J.res = res;
  }
  __syncthreads();
  // the outlier records of the applied cameras (Frontend.cpp:735-753, with the B keypoint of the correspondence)
  int n_out = 0;
  for (int cam = 0; cam < J.n_cams; ++cam) {
    const int pick = s_pick[cam];
    if (pick == -1) continue;
    const int o = s_off[cam], nc = s_off[cam + 1] - o;
    const bool rel = pick >= 0 && ((pick / H) & 1);
    const double* Mo = J.model + (size_t)max(pick, 0) * 12;
    int cam_out = 0;
    for (int k0 = 0; k0 < nc; k0 += RS_T) {
      const int k = k0 + tid;
      int bad = 0;
      if (k < nc) {
        const double* cd = J.cd + (size_t)(o + k) * R2_CD;
        bad = pick >= 0 && (rel ? r2_score_rel(Mo, Mo + 9, cd) : r2_score_rot(Mo, cd)) < J.threshold ? 0 : 1;
      }
      int total;
      const int pos = block_scan<RS_T>(bad, s_warp, &total);
      if (bad) {
        const int* cr = J.ci + 3 * (size_t)(o + k);
        J.outl[n_out + pos] = okb_ransac2d_outlier{cam, cr[0], cr[1], cr[2]};
      }
      n_out += total;
      cam_out += total;
    }
    if (tid == 0) J.cams[cam].n_outliers = cam_out;
  }
  if (tid == 0) J.res->n_outliers = n_out;
}
}  // namespace

// Host checks of one job; "" = valid.  *n_kp_a: frame A's keypoints in the job's cameras.
static std::string ransac2d_job_invalid(okb_ctx* c, const okb_ransac2d_job& j, std::vector<char>& seen, size_t* n_kp_a) {
  const std::string why = store_window_invalid(c, j.win, seen);
  if (!why.empty()) return why;
  const WinStore& S = c->wins[j.win];
  const WinDev& W = c->host[j.win];
  const FeatStore& F = S.feat;
  if (j.feat_slot_a < 0 || j.feat_slot_a >= F.F || j.feat_slot_b < 0 || j.feat_slot_b >= F.F) return "feat_slot_a / feat_slot_b out of range";
  if (j.pose_a < 0 || j.pose_a >= W.K || j.pose_b < 0 || j.pose_b >= W.K) return "pose_a / pose_b out of range";
  if (j.n_cams < 1 || j.n_cams > F.C || j.n_cams > W.NE || j.n_cams > W.NC || j.n_cams > RS_MAX_CAMS)
    return "n_cams out of range (1..the store's cameras, the window's extrinsics and cameras, 16)";
  size_t n_kp = 0;
  for (int cam = 0; cam < j.n_cams; ++cam) {
    const int na = S.feat_n_pending[(size_t)j.feat_slot_a * F.C + cam], nb = S.feat_n_pending[(size_t)j.feat_slot_b * F.C + cam];
    if (na < 0 || nb < 0) return "feature slot has no keypoints for camera " + std::to_string(cam);
    n_kp += na;
  }
  if (j.max_iterations < 1 || j.max_iterations > RS_MAX_HYP) return "max_iterations out of range (1..64)";
  if (!(j.threshold > 0.0) || !std::isfinite(j.threshold)) return "threshold not finite and positive";
  if (!j.out) return "out missing";
  if ((size_t)std::max(j.outlier_cap, 0) < n_kp || (n_kp && !j.outliers)) return "outlier capacity below frame A's keypoints";
  *n_kp_a = n_kp;
  return "";
}

extern "C" int okb_ransac_2d2d_batch(okb_ctx* c, int n_jobs, const okb_ransac2d_job* jobs) {
  const char* fn = "okb_ransac_2d2d_batch";
  std::vector<size_t> n_kp(std::max(n_jobs, 0), 0);
  int rc = store_call_checks(c, fn, n_jobs, jobs, INT_MAX,
                             [&](int i, std::vector<char>& seen) { return ransac2d_job_invalid(c, jobs[i], seen, &n_kp[i]); });
  if (rc || n_jobs == 0) return rc;
  cudaSetDevice(c->device);
  okb_frontend_state* F = fe(c);
  CallBuffers& B = F->ransac2d;
  std::lock_guard<std::mutex> lk(B.mtx);
  if ((rc = commit_job_windows(c, jobs, n_jobs))) return rc;
  if ((rc = shard_lm_exchange(c, fn, jobs, n_jobs, c->stream_xfer))) return rc;
  cudaStream_t xs = c->stream_xfer;
  // staging (pinned + device mirror): in  = [job table]
  //                                   out = [per job: result | cameras | hypothesis inliers | outlier records]
  // scratch (device only), per job: first keypoint per landmark slot | correspondences | their indices | models
  Carve st, sc;
  st.take(sizeof(Ransac2JobDev) * (size_t)n_jobs, 256);
  const size_t in_bytes = st.off;
  std::vector<size_t> o_res(n_jobs), o_cam(n_jobs), o_hyp(n_jobs), o_out(n_jobs), o_first(n_jobs), o_cd(n_jobs), o_ci(n_jobs), o_mod(n_jobs);
  for (int i = 0; i < n_jobs; ++i) {
    const okb_ransac2d_job& j = jobs[i];
    const size_t tasks = (size_t)j.n_cams * 2 * j.max_iterations;
    o_res[i] = st.take(sizeof(okb_ransac2d_result));
    o_cam[i] = st.take(sizeof(okb_ransac2d_cam) * (size_t)j.n_cams);
    o_hyp[i] = st.take(4 * tasks);
    o_out[i] = st.take(sizeof(okb_ransac2d_outlier) * n_kp[i]);
    o_first[i] = sc.take(4 * (size_t)lm_slots_host(c, j.win));
    o_cd[i] = sc.take(8 * R2_CD * n_kp[i]);
    o_ci[i] = sc.take(12 * n_kp[i]);
    o_mod[i] = sc.take(8 * 12 * tasks);
  }
  const size_t out_end = st.off;
  if ((rc = B.reserve(c, out_end, sc.off))) return rc;
  uint8_t* h = B.h_stage;
  uint8_t* d = B.d_stage;
  Ransac2JobDev* tj = reinterpret_cast<Ransac2JobDev*>(h);
  for (int i = 0; i < n_jobs; ++i) {
    const okb_ransac2d_job& j = jobs[i];
    Ransac2JobDev J;
    std::memset(&J, 0, sizeof J);
    J.W = c->d_wins + j.win;
    J.feat_a = j.feat_slot_a; J.feat_b = j.feat_slot_b; J.pose_a = j.pose_a; J.pose_b = j.pose_b;
    J.n_cams = j.n_cams; J.n_hyp = j.max_iterations; J.init_pose = j.initialize_pose ? 1 : 0;
    J.L = lm_slots_host(c, j.win);
    J.threshold = j.threshold;
    J.seed = (unsigned long long)j.seed;
    J.first = reinterpret_cast<int*>(B.d_scratch + o_first[i]);
    J.cd = reinterpret_cast<double*>(B.d_scratch + o_cd[i]);
    J.ci = reinterpret_cast<int*>(B.d_scratch + o_ci[i]);
    J.model = reinterpret_cast<double*>(B.d_scratch + o_mod[i]);
    J.res = reinterpret_cast<okb_ransac2d_result*>(d + o_res[i]);
    J.cams = reinterpret_cast<okb_ransac2d_cam*>(d + o_cam[i]);
    J.hyp = reinterpret_cast<int*>(d + o_hyp[i]);
    J.outl = reinterpret_cast<okb_ransac2d_outlier*>(d + o_out[i]);
    tj[i] = J;
  }
  OKB_CUDA(c, cudaMemcpyAsync(d, h, in_bytes, cudaMemcpyHostToDevice, xs));
  k_ransac_2d2d<<<n_jobs, RS_T, 0, xs>>>(reinterpret_cast<const Ransac2JobDev*>(d));
  F->launches += 1;
  OKB_CUDA(c, cudaGetLastError());
  OKB_CUDA(c, cudaMemcpyAsync(h + in_bytes, d + in_bytes, out_end - in_bytes, cudaMemcpyDeviceToHost, xs));
  OKB_CUDA(c, cudaStreamSynchronize(xs));
  for (int i = 0; i < n_jobs; ++i) {
    const okb_ransac2d_job& j = jobs[i];
    *j.out = *reinterpret_cast<const okb_ransac2d_result*>(h + o_res[i]);
    if (j.cams) std::memcpy(j.cams, h + o_cam[i], sizeof(okb_ransac2d_cam) * (size_t)j.n_cams);
    if (j.hyp_inliers) std::memcpy(j.hyp_inliers, h + o_hyp[i], 4 * (size_t)j.n_cams * 2 * j.max_iterations);
    if (j.out->n_outliers) std::memcpy(j.outliers, h + o_out[i], sizeof(okb_ransac2d_outlier) * (size_t)j.out->n_outliers);
  }
  return OKB_OK;
}

// =================================================================================================
// detection straight into the feature store (okb_detect_describe_store_batch): detect_run over every image of the call
// on the batch stream, with one store destination per image; k_store_features waits for the commit of the job windows
// =================================================================================================
// Host checks of one job; "" = valid.  *images counts the images of the call so far.
static std::string detect_store_job_invalid(okb_ctx* c, const okb_detect_store_job& j, const okb_detect_params& prm, int max_out,
                                            int* images, std::vector<char>& seen) {
  const std::string why = store_window_invalid(c, j.win, seen);
  if (!why.empty()) return why;
  const FeatStore& F = c->wins[j.win].feat;
  if (j.feat_slot < 0 || j.feat_slot >= F.F) return "feat_slot out of range";
  if (j.n_cams < 1 || j.n_cams > F.C) return "n_cams out of range (1..the store's cameras)";
  if (prm.desc_bytes != F.D) return "params->desc_bytes differs from the store's descriptor length";
  if (F.N < std::min(prm.max_keypoints, max_out)) return "the store holds fewer keypoints per image than min(max_keypoints, max_out)";
  if (!j.images || !j.out_kp || !j.n_out) return "images / out_kp / n_out missing";
  for (int cam = 0; cam < j.n_cams; ++cam)
    if (!batch_image_ok(j.images[cam])) return "images[" + std::to_string(cam) + "]: no pixels, smaller than 64 x 64 or stride < width";
  if ((*images += j.n_cams) > 65535) return "more than 65535 images in the call";     // the image index is a grid dimension
  return "";
}

extern "C" int okb_detect_describe_store_batch(okb_ctx* c, int n_jobs, const okb_detect_store_job* jobs, const okb_detect_params* prm,
                                               int max_out, int host_threads) {
  const char* fn = "okb_detect_describe_store_batch";
  if (c && n_jobs > 0 && (!prm || !detect_params_ok(prm, max_out))) {
    c->set_error(std::string(fn) + ": params missing, or a descriptor length / min(max_keypoints, max_out) out of range");
    return OKB_ERR_INVALID_ARG;
  }
  int n = 0;
  int rc = store_call_checks(c, fn, n_jobs, jobs, 65535,
                             [&](int i, std::vector<char>& seen) { return detect_store_job_invalid(c, jobs[i], *prm, max_out, &n, seen); });
  if (rc || n_jobs == 0) return rc;
  const int db = prm->desc_bytes;
  std::vector<okb_image_desc> ims;
  std::vector<DetectOut> outs;
  std::vector<StoreDest> dests;
  ims.reserve(n); outs.reserve(n); dests.reserve(n);
  for (int i = 0; i < n_jobs; ++i) {
    const okb_detect_store_job& j = jobs[i];
    const FeatStore& FS = c->wins[j.win].feat;
    for (int cam = 0; cam < j.n_cams; ++cam) {
      const size_t img = (size_t)j.feat_slot * FS.C + cam, base = img * FS.N;
      ims.push_back(j.images[cam]);
      outs.push_back(DetectOut{j.out_kp + (size_t)cam * max_out, j.out_desc ? j.out_desc + (size_t)cam * max_out * db : nullptr, j.n_out + cam});
      dests.push_back(StoreDest{FS.kp + 2 * base, FS.size + base, FS.desc + base * (FS.D / 4), FS.lm + base, FS.observed + base, FS.n + img});
    }
  }
  cudaSetDevice(c->device);
  okb_frontend_state* F = fe(c);
  std::lock_guard<std::mutex> lk(F->batch_mtx);
  if (!F->batch_stream) OKB_CUDA(c, cudaStreamCreateWithFlags(&F->batch_stream, cudaStreamNonBlocking));
  if (!F->store_ready) OKB_CUDA(c, cudaEventCreateWithFlags(&F->store_ready, cudaEventDisableTiming));
  if ((rc = commit_job_windows(c, jobs, n_jobs))) return rc;
  OKB_CUDA(c, cudaEventRecord(F->store_ready, c->stream_xfer));
  rc = detect_run(c, F, F->batch_det, F->batch_stream, n, ims.data(), prm, outs.data(), max_out, dests.data(), F->store_ready, host_threads);
  if (rc != OKB_OK && rc != OKB_ERR_CAPACITY) return rc;
  for (int i = 0; i < n_jobs; ++i) {       // the host's counts follow the entries written (an image over capacity kept its own)
    WinStore& S = c->wins[jobs[i].win];
    for (int cam = 0; cam < jobs[i].n_cams; ++cam) {
      const int m = jobs[i].n_out[cam];
      if (m < 0) continue;
      const size_t img = (size_t)jobs[i].feat_slot * S.feat.C + cam;
      S.feat_n[img] = S.feat_n_pending[img] = m;
    }
  }
  return rc;
}
