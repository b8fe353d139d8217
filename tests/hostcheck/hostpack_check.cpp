// TEST INFRASTRUCTURE ONLY -- exposes the host-side call helpers of okb_hostpack.hpp (buffer layout, runs of
// consecutive slots, host-thread spreading) through a C interface so that tests/test_hostpack.py checks them without a
// GPU.  This library is never loaded by the product.
#include <functional>
#include <thread>

#include "../../okvis_b200/csrc/okb_hostpack.hpp"

extern "C" {
// offs[k] = offset of array k of bytes[k] bytes; returns the total
uint64_t hp_carve(const uint64_t* bytes, int n, uint64_t align, uint64_t* offs) {
  okb::Carve P;
  for (int k = 0; k < n; ++k) offs[k] = P.take(bytes[k], align);
  return P.off;
}
// the runs for_runs visits, in order; the callback fails with 7 on run number stop_at
int hp_for_runs(const int32_t* slots, int n, int stop_at, int32_t* first, int32_t* count, int* n_runs) {
  int k = 0;
  const int rc = okb::for_runs(slots, n, [&](int f, int m) {
    first[k] = f; count[k] = m;
    return k++ == stop_at ? 7 : 0;
  });
  *n_runs = k;
  return rc;
}
// visits[i] counts the calls f(i); owner[i] identifies the thread that made them; returns the calling thread's id
uint64_t hp_parallel_for(int n, int T, int32_t* visits, uint64_t* owner) {
  auto id = [] { return (uint64_t)std::hash<std::thread::id>{}(std::this_thread::get_id()); };
  okb::parallel_for(n, T, [&](int i) {
    __atomic_fetch_add(&visits[i], 1, __ATOMIC_RELAXED);
    owner[i] = id();
  });
  return id();
}
}
