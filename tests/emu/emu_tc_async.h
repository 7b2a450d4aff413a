// Host emulation of csrc/srcv_tc.cuh with ASYNCHRONOUS warpgroup MMAs — TEST INFRASTRUCTURE.
//
// emu_tc.h models wgmma as executing at issue, with commit / wait as no-ops.  A kernel that hands a
// shared-memory operand buffer back to its producer before the wgmma.wait_group that retires the
// MMAs reading it would still pass there.  This header keeps everything of emu_tc.h (mbarriers,
// bulk copies, descriptors, the fragment arithmetic, the fp16 split) and replaces the four MMA entry
// points with the asynchronous semantics:
//
//   * wgmma_ss_* / wgmma_rs_* queue the MMA in the issuing thread; a register A operand is captured
//     at issue (the hardware reads it then too), the shared-memory operands and the accumulator
//     are NOT touched yet;
//   * wgmma_commit closes the open group;
//   * wgmma_wait<N> performs every committed group but the N newest, oldest first, in issue order —
//     only then are the shared-memory operands read and the accumulator written.
//
// A buffer released early is therefore read after its producer may have overwritten it: wrong
// results in the emulated wgmma tests, and a data race under ThreadSanitizer (the mbarrier
// hand-off no longer orders the read).  Kernels that wait right after each commit (the self-test,
// the earlier single-tile sweep) behave exactly as under emulation at issue.
// Not modelled: an accumulator read before its wait (undefined on the hardware; here it holds the
// value of the last performed group).
//
// srcv_tc.cuh includes this header under SRCV_HOST_EMU.  tests/emu's incremental build tracks
// emu_tc.h and the csrc sources, not this file: rebuild with build(force=True) after editing it.
#pragma once

// emu_tc.h's at-issue MMA entry points are compiled under other names and left unused.
#define wgmma_commit wgmma_commit_at_issue
#define wgmma_wait wgmma_wait_at_issue
#define wgmma_ss_n128 wgmma_ss_n128_at_issue
#define wgmma_rs_n64 wgmma_rs_n64_at_issue
#include "emu_tc.h"
#undef wgmma_commit
#undef wgmma_wait
#undef wgmma_ss_n128
#undef wgmma_rs_n64

#include <utility>
#include <vector>

namespace srcv {
namespace tc {

namespace detail {
// One issued MMA of this thread.
struct Mma {
  float* d;
  int n;                    // 128: ss m64n128k16;  64: rs m64n64k16
  uint64_t a_desc, b_desc;
  uint32_t acc;
  float rows[2][16];        // register A operand (rs), captured at issue
};
struct MmaQueue {
  std::vector<Mma> open;                 // issued since the last commit
  std::vector<std::vector<Mma>> groups;  // committed, oldest first
};
inline thread_local MmaQueue t_mma;
inline void perform(Mma& m) {
  if (m.n == 128) {
    const int r0 = 16 * warp_in_group() + (int)((threadIdx.x & 31u) >> 2);
    for (int h = 0; h < 2; ++h)
      for (int k = 0; k < 16; ++k) m.rows[h][k] = operand_value(m.a_desc, r0 + 8 * h, k);
    mma_fragment<128>(m.d, m.rows, m.b_desc, m.acc);
  } else {
    mma_fragment<64>(m.d, m.rows, m.b_desc, m.acc);
  }
}
}  // namespace detail

inline void wgmma_commit() {
  detail::t_mma.groups.push_back(std::move(detail::t_mma.open));
  detail::t_mma.open.clear();
}
template <int N> inline void wgmma_wait() {
  auto& gs = detail::t_mma.groups;
  while (gs.size() > (size_t)N) {
    for (detail::Mma& m : gs.front()) detail::perform(m);
    gs.erase(gs.begin());
  }
}

inline void wgmma_ss_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  detail::t_mma.open.push_back(detail::Mma{d, 128, a_desc, b_desc, accumulate, {}});
}
inline void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
  // a0: row g, k 2q, 2q+1;  a1: row g+8;  a2: row g, k 8+2q, 9+2q;  a3: row g+8  (q = the source lane of the quad)
  const int g = (int)((threadIdx.x & 31u) >> 2);
  detail::Mma m{d, 64, 0, b_desc, accumulate, {}};
  for (int src = 0; src < 4; ++src)
    for (int i = 0; i < 4; ++i) {
      const uint32_t w = (uint32_t)__shfl_sync(0xffffffffu, (int)a[i], 4 * g + src);
      const int h = i & 1, k = 2 * src + 8 * (i >> 1);
      m.rows[h][k] = detail::half_bits((uint16_t)w);
      m.rows[h][k + 1] = detail::half_bits((uint16_t)(w >> 16));
    }
  detail::t_mma.open.push_back(m);
}

}  // namespace tc
}  // namespace srcv
