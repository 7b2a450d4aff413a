// Host emulation of the wgmma / mbarrier / bulk-copy layer of csrc/srcv_tc.cuh —
// TEST INFRASTRUCTURE (see emu_cuda.h).  Same function names and argument meaning as the
// inline-PTX wrappers, with the FUNCTIONAL semantics the GPU kernel relies on:
//
//   * wgmma m64nNk16 f16 -> f32: each thread computes its own accumulator fragment (layout in
//     srcv_tc.cuh); A from a K-major no-swizzle smem descriptor or from the quad's registers (via
//     __shfl_sync), B from smem; exact products, fp32 accumulation in k order;
//   * MMAs execute at issue; commit / wait / fences are no-ops (the kernels wait right after each commit);
//   * mbarrier: phase bit | pending arrivals | arrival count | pending transaction bytes packed
//     in the 64-bit word, updated with CAS; waits block on the word (std::atomic_ref::wait).
//     Acquire/release on the word gives ThreadSanitizer the happens-before edges of the real
//     protocol: a shared-memory hand-off that is not ordered by a barrier is a data race.
// Not modelled: the asynchrony of wgmma, swizzled layouts, clusters, setmaxnreg.
#pragma once
#include "emu_cuda.h"

#include <atomic>
#include <cstdio>
#include <vector>

struct __half { _Float16 v; };
struct __half2 { __half x, y; };
inline __half __float2half_rn(float f) { return __half{(_Float16)f}; }
inline float __half2float(__half h) { return (float)h.v; }
inline float2 __half22float2(__half2 h) { return make_float2((float)h.x.v, (float)h.y.v); }
inline __half2 __floats2half2_rn(float a, float b) { return __half2{__half{(_Float16)a}, __half{(_Float16)b}}; }

namespace srcv {
namespace tc {

inline uint32_t smem_u32(const void* p) {
  return (uint32_t)(reinterpret_cast<const char*>(p) - reinterpret_cast<const char*>(::emu::dynamic_smem()));
}

// ---- mbarrier ---------------------------------------------------------------------------
namespace detail {
struct Word { uint32_t phase, pending, init; int32_t tx; };
inline Word unpack(uint64_t w) {
  return Word{(uint32_t)(w >> 63), (uint32_t)((w >> 32) & 0x7FFF), (uint32_t)((w >> 47) & 0x7FFF), (int32_t)(uint32_t)w};
}
inline uint64_t pack(const Word& s) {
  return ((uint64_t)s.phase << 63) | ((uint64_t)s.init << 47) | ((uint64_t)s.pending << 32) | (uint32_t)s.tx;
}
inline void update(uint64_t* bar, uint32_t arrivals, int32_t dtx) {
  std::atomic_ref<uint64_t> a(*bar);
  uint64_t old = a.load(std::memory_order_relaxed), nw;
  bool flipped;
  do {
    Word s = unpack(old);
    if (s.pending < arrivals) { std::fprintf(stderr, "emu: mbarrier over-arrival\n"); std::abort(); }
    s.pending -= arrivals;
    s.tx += dtx;
    flipped = (s.pending == 0 && s.tx == 0);
    if (flipped) { s.phase ^= 1u; s.pending = s.init; }
    nw = pack(s);
  } while (!a.compare_exchange_weak(old, nw, std::memory_order_acq_rel, std::memory_order_relaxed));
  if (flipped) a.notify_all();
}
}  // namespace detail

inline void mbar_init(uint64_t* bar, uint32_t count) {
  std::atomic_ref<uint64_t>(*bar).store(detail::pack(detail::Word{0, count, count, 0}), std::memory_order_release);
}
inline void mbar_fence_init() {}
inline void mbar_arrive(uint64_t* bar) { detail::update(bar, 1, 0); }
inline void mbar_expect_tx(uint64_t* bar, uint32_t bytes) { detail::update(bar, 1, (int32_t)bytes); }
inline void mbar_wait(uint64_t* bar, uint32_t parity) {
  std::atomic_ref<uint64_t> a(*bar);
  for (;;) {
    const uint64_t w = a.load(std::memory_order_acquire);
    if ((uint32_t)(w >> 63) != (parity & 1u)) return;
    a.wait(w, std::memory_order_acquire);      // blocks until the word changes
  }
}
inline void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  std::memcpy(smem_dst, gmem_src, bytes);
  detail::update(bar, 0, -(int32_t)bytes);
}
inline void fence_proxy_async_smem() {}

// ---- descriptors (bit-identical to the device versions) -------------------------------------
inline uint64_t smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;
}

// ---- warpgroup MMA ---------------------------------------------------------------------------
inline void wgmma_fence() {}
inline void wgmma_commit() {}
template <int N> inline void wgmma_wait() {}
template <int N> inline void fence_regs(float (&)[N]) {}

namespace detail {
inline float half_bits(uint16_t h) { _Float16 f; std::memcpy(&f, &h, 2); return (float)f; }
inline const char* operand(uint64_t desc, int row, int k) {       // K-major, no swizzle, 8 x 16-byte core matrices
  const uint32_t start = (uint32_t)(desc & 0x3FFFu) << 4, lbo = (uint32_t)((desc >> 16) & 0x3FFFu) << 4,
                 sbo = (uint32_t)((desc >> 32) & 0x3FFFu) << 4;
  return reinterpret_cast<const char*>(::emu::dynamic_smem()) + start + (uint32_t)(k >> 3) * lbo +
         (uint32_t)(row >> 3) * sbo + (uint32_t)(row & 7) * 16u + (uint32_t)(k & 7) * 2u;
}
inline float operand_value(uint64_t desc, int row, int k) {
  uint16_t h;
  std::memcpy(&h, operand(desc, row, k), 2);
  return half_bits(h);
}
inline int warp_in_group() { return (int)(((threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z)) / 32) & 3u); }
// the N / 2 fragment elements of this thread: rows[0] = A row 16 w + g, rows[1] = A row 16 w + g + 8
template <int N>
inline void mma_fragment(float* d, const float (&rows)[2][16], uint64_t b_desc, uint32_t acc) {
  const int q = (int)(threadIdx.x & 3u);
  for (int j = 0; j < N / 8; ++j)
    for (int e = 0; e < 4; ++e) {
      const int n = 8 * j + 2 * q + (e & 1);
      float s = acc ? d[4 * j + e] : 0.f;
      for (int k = 0; k < 16; ++k) s += rows[e >> 1][k] * operand_value(b_desc, n, k);
      d[4 * j + e] = s;
    }
}
}  // namespace detail

inline void wgmma_ss_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  const int r0 = 16 * detail::warp_in_group() + (int)((threadIdx.x & 31u) >> 2);
  float rows[2][16];
  for (int h = 0; h < 2; ++h)
    for (int k = 0; k < 16; ++k) rows[h][k] = detail::operand_value(a_desc, r0 + 8 * h, k);
  detail::mma_fragment<128>(d, rows, b_desc, accumulate);
}
inline void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc, uint32_t accumulate) {
  // a0: row g, k 2q, 2q+1;  a1: row g+8;  a2: row g, k 8+2q, 9+2q;  a3: row g+8  (q = the source lane of the quad)
  const int g = (int)((threadIdx.x & 31u) >> 2);
  float rows[2][16];
  for (int src = 0; src < 4; ++src)
    for (int i = 0; i < 4; ++i) {
      const uint32_t w = (uint32_t)__shfl_sync(0xffffffffu, (int)a[i], 4 * g + src);
      const int h = i & 1, k = 2 * src + 8 * (i >> 1);
      rows[h][k] = detail::half_bits((uint16_t)w);
      rows[h][k + 1] = detail::half_bits((uint16_t)(w >> 16));
    }
  detail::mma_fragment<64>(d, rows, b_desc, accumulate);
}

template <int N> inline void reg_inc() {}
template <int N> inline void reg_dec() {}

// ---- fp32 -> (hi, lo) fp16 pair split (cvt.rn.satfinite.f16x2.f32) ------------------------------
inline uint16_t f16_sat_bits(float x) {
  if (x != x) return 0x7FFFu;
  const _Float16 h = (_Float16)fminf(fmaxf(x, -65504.f), 65504.f);
  uint16_t b;
  std::memcpy(&b, &h, 2);
  return b;
}
inline uint32_t pack_f16x2_sat(float even, float odd) {
  return (uint32_t)f16_sat_bits(even) | ((uint32_t)f16_sat_bits(odd) << 16);
}
inline void split_pack(float even, float odd, uint32_t& hi, uint32_t& lo) {
  hi = pack_f16x2_sat(even, odd);
  const float be = detail::half_bits((uint16_t)hi), bo = detail::half_bits((uint16_t)(hi >> 16));
  lo = pack_f16x2_sat(even - be, odd - bo);
}

}  // namespace tc
}  // namespace srcv
