// Host-emulation build of libsrcv_b200's C ABI — TEST INFRASTRUCTURE (see emu_cuda.h).
//
// tests/emu/__init__.py compiles the product's own sources (every csrc/*.cu) as host C++ with
// -DSRCV_HOST_EMU and links them with this file into tests/emu/_build/libsrcv_emu.so, which
// therefore exports the SAME entry points as include/srcv_b200.h, taking HOST pointers.  The
// wgmma kernel runs against the functional wgmma / mbarrier model of emu_tc.h.
#define SRCV_HOST_EMU 1
#include "../../simplerecon_b200/csrc/srcv_kernels.h"

extern "C" {
// "SM count" seen by the launch heuristics (plane-loop split of the dot sweep, persistent
// grid of the MLP backward): lets a test drive those code paths with tiny inputs.
void emu_set_sms(int n) { ::emu::g_sms = n > 0 ? n : 1; }

// 1 if this process may run n threads at once (the largest CTA here has 640): lets the tests
// skip instead of aborting under a restrictive pids / thread limit.
int emu_can_spawn(int n) {
  std::vector<std::thread> pool;
  std::atomic<int> go{0};
  bool ok = true;
  try {
    for (int i = 0; i < n; ++i) pool.emplace_back([&] { while (!go.load()) std::this_thread::yield(); });
  } catch (...) {
    ok = false;
  }
  go.store(1);
  for (auto& t : pool) t.join();
  return ok ? 1 : 0;
}
}
