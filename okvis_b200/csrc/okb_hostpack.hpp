// Host-side helpers of the library's calls (plain C++, no CUDA): buffer layout, runs of consecutive slots, host-thread
// spreading and the internal landmark order of okb_window_upload.
// Kept in a header so that tests/hostcheck can exercise them without a GPU.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <algorithm>
#include <thread>
#include <vector>

namespace okb {

// Lays arrays out one after another in a buffer: take() returns the offset of the next `bytes` and pads their end to
// `align`, so the array after them starts aligned; `off` is the size so far.  Callers lay a buffer out once, keep the
// offsets and fill from them.
struct Carve {
  size_t off = 0;
  size_t take(size_t bytes, size_t align = 16) {
    const size_t o = off;
    off = (off + bytes + align - 1) / align * align;
    return o;
  }
};

// Calls f(first, count) for each run of consecutive slots of a list, in list order (a range is one run); stops at and
// returns the first nonzero result.
template <class F>
int for_runs(const int32_t* slots, int n, F&& f) {
  for (int i = 0; i < n;) {
    int j = i + 1;
    while (j < n && slots[j] == slots[j - 1] + 1) ++j;
    const int rc = f(slots[i], j - i);
    if (rc) return rc;
    i = j;
  }
  return 0;
}

// f(i) for every i in [0, n): thread t of T runs i = t, t + T, ... in that order; T == 1 runs inline.
template <class F>
void parallel_for(int n, int T, const F& f) {
  if (T <= 1) {
    for (int i = 0; i < n; ++i) f(i);
    return;
  }
  std::vector<std::thread> th;
  th.reserve(T);
  for (int t = 0; t < T; ++t)
    th.emplace_back([=, &f]() {
      for (int i = t; i < n; i += T) f(i);
    });
  for (auto& x : th) x.join();
}

// Sort key of a landmark with frame-visibility mask m: first observing frame * 32 + last observing frame;
// landmarks without observations sort last.
inline uint32_t frame_range_key(uint32_t m) {
  if (!m) return 32u * 32u;
  return (uint32_t)__builtin_ctz(m) * 32u + (31u - (uint32_t)__builtin_clz(m));
}

// Internal landmark order: stable counting sort by frame_range_key.  vis[l] = frame-visibility mask of the caller's
// landmark l.  Outputs perm[j] = caller's index of internal landmark j, inv[l] = internal index of caller's l, and
// tile_range[t] = first | last << 8 over the observed landmarks of internal tile t (32 landmarks); first > last
// (value 1) marks a tile without observations.
inline void sort_landmarks_by_frame_range(const uint32_t* vis, int L, uint32_t* perm, uint32_t* inv, uint32_t* tile_range) {
  std::vector<uint32_t> count(32 * 32 + 2, 0u);
  for (int l = 0; l < L; ++l) ++count[frame_range_key(vis[l]) + 1];
  for (size_t k = 1; k < count.size(); ++k) count[k] += count[k - 1];
  for (int l = 0; l < L; ++l) {
    const uint32_t j = count[frame_range_key(vis[l])]++;
    perm[j] = (uint32_t)l;
    inv[l] = j;
  }
  const int n_tiles = (L + 31) / 32;
  for (int t = 0; t < n_tiles; ++t) tile_range[t] = 1u;
  for (int j = 0; j < L; ++j) {
    const uint32_t m = vis[perm[j]];
    if (!m) continue;
    const uint32_t fi = (uint32_t)__builtin_ctz(m), la = 31u - (uint32_t)__builtin_clz(m);
    uint32_t& tr = tile_range[j >> 5];
    const uint32_t a = tr & 0xffu, b = tr >> 8;
    tr = (a > b) ? (fi | (la << 8)) : (std::min(a, fi) | (std::max(b, la) << 8));
  }
}

}  // namespace okb
