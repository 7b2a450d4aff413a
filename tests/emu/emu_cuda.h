// Host emulation of the slice of the CUDA execution model the SIMT kernels in
// simplerecon_b200/csrc use — TEST INFRASTRUCTURE (tests/emu), never part of the product.
//
// With -DSRCV_HOST_EMU the kernel sources include this header instead of <cuda_runtime.h>
// and compile as plain C++20: a launch runs the CTAs one after another, each CUDA thread of
// a CTA as one std::thread, __syncthreads() as a std::barrier, shared memory as a per-CTA
// heap block (poisoned with NaNs so that reads of never-written shared memory show up),
// atomics as real host atomics.  It exists so that indexing, barrier placement and the
// arithmetic of a kernel can be checked against the oracle in the CPU test tier, before any
// GPU time is spent; it says nothing about launch limits, registers or speed.
// Warp-level intrinsics: __shfl_sync / __shfl_xor_sync / __all_sync over full, converged warps.
// The wgmma / mbarrier / bulk-copy layer is modelled in emu_tc.h.
#pragma once
#include <atomic>
#include <barrier>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <thread>
#include <vector>

#define __host__
#define __device__
#define __global__
#define __forceinline__ inline __attribute__((always_inline))
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))
#define __shared__ static   /* CTAs run one at a time: a static is CTA-shared */

// ---- the handful of runtime-API names the launchers and srcv_api.cu use ----------------
typedef int cudaError_t;
typedef void* cudaStream_t;
typedef void* cudaEvent_t;
constexpr cudaError_t cudaSuccess = 0;
constexpr cudaError_t cudaErrorInvalidValue = 1;
enum cudaDeviceAttr { cudaDevAttrComputeCapabilityMajor, cudaDevAttrMultiProcessorCount };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize };
namespace emu { inline int g_sms = 4; }   // "SM count" the launch heuristics see (emu_set_sms)
inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr a, int) {
  *v = (a == cudaDevAttrComputeCapabilityMajor) ? 9 : ::emu::g_sms;
  return cudaSuccess;
}
template <class K> inline cudaError_t cudaFuncSetAttribute(K, cudaFuncAttribute, int bytes) {
  return bytes <= 227 * 1024 ? cudaSuccess : cudaErrorInvalidValue;   // the sm_90 opt-in limit
}
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline const char* cudaGetErrorName(cudaError_t) { return "emuError"; }
inline const char* cudaGetErrorString(cudaError_t) { return "host emulation error"; }
inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { std::memset(p, v, n); return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = nullptr; return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }

struct alignas(16) float4 { float x, y, z, w; };
struct alignas(8) float2 { float x, y; };
inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
inline float2 make_float2(float x, float y) { return float2{x, y}; }
struct uint3 { unsigned x, y, z; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};

namespace emu {
inline thread_local uint3 t_thread{0, 0, 0}, t_block{0, 0, 0};
inline thread_local dim3 t_bdim, t_gdim;
inline thread_local void* t_smem = nullptr;
inline thread_local std::barrier<>* t_bar = nullptr;
inline void* dynamic_smem() { return t_smem; }
struct WarpVote {
  std::barrier<>* bar = nullptr;
  std::atomic<int> acc[3];
};
inline thread_local WarpVote* t_votes = nullptr;
inline thread_local uint32_t* t_shfl = nullptr;        // per-warp exchange slots for __shfl_sync
inline thread_local unsigned t_vote_round = 0;

// Runs body() once per CUDA thread of a (grid x block) launch.
template <class F>
void launch(dim3 grid, dim3 block, size_t smem_bytes, F&& body) {
  const unsigned nthreads = block.x * block.y * block.z;
  const size_t bytes = ((smem_bytes + 127) / 128 + 1) * 128;
  for (unsigned bz = 0; bz < grid.z; ++bz)
    for (unsigned by = 0; by < grid.y; ++by)
      for (unsigned bx = 0; bx < grid.x; ++bx) {
        void* sm = std::aligned_alloc(1024, ((bytes + 1023) / 1024) * 1024);
        std::memset(sm, 0xFF, bytes);
        std::vector<uint32_t> shfl(((nthreads + 31) / 32) * 32, 0u);
        std::barrier<> bar((std::ptrdiff_t)nthreads);
        const unsigned nwarps = (nthreads + 31) / 32;
        std::vector<WarpVote> votes(nwarps);
        std::vector<std::barrier<>*> wbars;
        for (unsigned w = 0; w < nwarps; ++w) {
          wbars.push_back(new std::barrier<>((std::ptrdiff_t)std::min(32u, nthreads - 32 * w)));
          votes[w].bar = wbars.back();
          for (auto& a : votes[w].acc) a.store(1);
        }
        std::vector<std::thread> pool;
        pool.reserve(nthreads);
        for (unsigned t = 0; t < nthreads; ++t)
          pool.emplace_back([&, t] {
            t_thread = uint3{t % block.x, (t / block.x) % block.y, t / (block.x * block.y)};
            t_block = uint3{bx, by, bz};
            t_bdim = block;
            t_gdim = grid;
            t_smem = sm;
            t_bar = &bar;
            t_votes = votes.data();
            t_shfl = shfl.data();
            t_vote_round = 0;
            body();
            bar.arrive_and_drop();   // a CUDA thread that has exited no longer takes part in barriers
            votes[t / 32].bar->arrive_and_drop();
          });
        for (auto& th : pool) th.join();
        for (auto* wb : wbars) delete wb;
        std::free(sm);
      }
}
}  // namespace emu

#define threadIdx (::emu::t_thread)
#define blockIdx (::emu::t_block)
#define blockDim (::emu::t_bdim)
#define gridDim (::emu::t_gdim)

inline void __syncthreads() { ::emu::t_bar->arrive_and_wait(); }
inline void __syncwarp(unsigned = 0xffffffffu) {
  ::emu::t_votes[(threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z)) / 32].bar->arrive_and_wait();
}
inline float __uint_as_float(unsigned u) { float f; std::memcpy(&f, &u, 4); return f; }
inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }
inline void __threadfence() { std::atomic_thread_fence(std::memory_order_seq_cst); }

template <class T> inline T __ldg(const T* p) { return *p; }
template <class T> inline T __ldcg(const T* p) { return *p; }

inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
inline float __fadd_rn(float a, float b) { return a + b; }   // built with -ffp-contract=off
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fdiv_rn(float a, float b) { return a / b; }
inline float __frcp_rn(float a) { return 1.0f / a; }
inline float __fmaf_rn(float a, float b, float c) { return std::fmaf(a, b, c); }
using std::max;
using std::min;

inline float atomicAdd(float* p, float v) {
  uint32_t* ip = reinterpret_cast<uint32_t*>(p);
  uint32_t old = __atomic_load_n(ip, __ATOMIC_RELAXED), nw;
  float f;
  do {
    std::memcpy(&f, &old, 4);
    const float g = f + v;
    std::memcpy(&nw, &g, 4);
  } while (!__atomic_compare_exchange_n(ip, &old, nw, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED));
  return f;
}
inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline int atomicOr(int* p, int v) { return __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }

// __shfl_sync over a full, converged warp (32-bit payloads)
inline int __shfl_sync(unsigned, int v, int src_lane) {
  const unsigned lin = threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z);
  ::emu::WarpVote& w = ::emu::t_votes[lin / 32];
  uint32_t* slots = ::emu::t_shfl + (lin / 32) * 32;
  slots[lin & 31] = (uint32_t)v;
  w.bar->arrive_and_wait();
  const int r = (int)slots[src_lane & 31];
  w.bar->arrive_and_wait();                 // nobody overwrites a slot before everybody has read
  return r;
}
inline float __shfl_xor_sync(unsigned m, float v, int lane_mask) {
  const int lane = (int)((threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z)) & 31u);
  return __uint_as_float((unsigned)__shfl_sync(m, (int)__float_as_uint(v), lane ^ lane_mask));
}

// __all_sync over a full, converged warp (the only warp-level intrinsic the SIMT kernels use):
// the 32 std::threads of the warp meet at a per-warp barrier; three rotating slots so that a
// slot is re-armed while nobody can still be reading it.
inline int __all_sync(unsigned, int pred) {
  ::emu::WarpVote& w = ::emu::t_votes[(threadIdx.x + blockDim.x * (threadIdx.y + blockDim.y * threadIdx.z)) / 32];
  const unsigned n = ::emu::t_vote_round++;
  std::atomic<int>& slot = w.acc[n % 3];
  if (!pred) slot.store(0, std::memory_order_relaxed);
  w.bar->arrive_and_wait();
  const int r = slot.load(std::memory_order_relaxed);
  w.acc[(n + 2) % 3].store(1, std::memory_order_relaxed);   // == slot (n-1): every lane left it before this barrier
  return r;
}
