// The integer-cell hash shared by the voxel-block TSDF volume (srcv_tsdf_sparse.cuh: 8^3-voxel blocks) and the
// nearest-neighbour grid of the mesh evaluation (srcv_mesh_eval.cuh: uniform cells over a point set): a cell
// coordinate in [-2^20, 2^20)^3 packs into 63 bits, and a 64-bit finaliser spreads the key over a power-of-two
// open-addressing table (linear probing, kEmptyKey marks a free slot).
#pragma once
#include "srcv_kernels.h"

namespace srcv {

namespace {

#ifdef SRCV_HOST_EMU
// tests/emu provides 32-bit atomics only
inline unsigned long long atomicCAS(unsigned long long* p, unsigned long long cmp, unsigned long long v) {
  __atomic_compare_exchange_n(p, &cmp, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED);
  return cmp;
}
inline unsigned long long load_key(const unsigned long long* p) { return __atomic_load_n(p, __ATOMIC_RELAXED); }
#else
__device__ __forceinline__ unsigned long long load_key(const unsigned long long* p) {
  return *reinterpret_cast<const volatile unsigned long long*>(p);
}
#endif

constexpr unsigned long long kEmptyKey = ~0ull;
constexpr int kKeyBias = 1 << 20;                      // cell coordinates in [-2^20, 2^20) pack into 21 bits

__device__ __forceinline__ bool block_in_range(int bx, int by, int bz) {
  return bx >= -kKeyBias && bx < kKeyBias && by >= -kKeyBias && by < kKeyBias && bz >= -kKeyBias && bz < kKeyBias;
}

__device__ __forceinline__ unsigned long long block_key(int bx, int by, int bz) {
  return ((unsigned long long)(unsigned)(bx + kKeyBias) << 42) | ((unsigned long long)(unsigned)(by + kKeyBias) << 21) |
         (unsigned long long)(unsigned)(bz + kKeyBias);
}

__device__ __forceinline__ unsigned block_hash(unsigned long long k, unsigned mask) {
  k ^= k >> 31; k *= 0x7fb5d329728ea185ull;           // a 64-bit finaliser (murmur3 style)
  k ^= k >> 27; k *= 0x81dadef4bc2dd44dull;
  k ^= k >> 33;
  return (unsigned)k & mask;
}

}  // namespace

}  // namespace srcv
