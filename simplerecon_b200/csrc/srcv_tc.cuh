// Thin inline-PTX layer over the Hopper tensor-core path used by the metadata-MLP sweep:
// warpgroup MMAs (wgmma.mma_async, fp16 operands, fp32 accumulators in registers) with the
// B operand (weights) and optionally the A operand in shared memory, mbarrier hand-offs
// between warp roles, and the bulk-copy (TMA) engine for the weight image.  sm_90a.
//
// Layout conventions used here
//   * shared-memory operands: K-major, no swizzle ("interleave") canonical layout — 8 rows x 16
//     bytes core matrices; row r, K chunk c (8 halves) lives at
//         c * LBO + (r / 8) * SBO + (r % 8) * 16   bytes from the start address.
//   * accumulator fragment of an m64nN wgmma (warp w of the warpgroup, lane = 4 g + q):
//         d[4 j + e] = D[16 w + g + 8 (e / 2)][8 j + 2 q + (e % 2)]
//   * register A fragment of one k16 step (same g, q):  a0 = row g, k 2q..2q+1;  a1 = row g + 8;
//     a2 = row g, k 8 + 2q..;  a3 = row g + 8, k 8 + 2q..  (even k in the low half), i.e. exactly
//     the packed accumulator words d[8 s .. 8 s + 7] of columns 16 s .. 16 s + 15 of an earlier layer.
#pragma once
#ifdef SRCV_HOST_EMU
#include "emu_tc_async.h"   // tests/emu: functional host model of this layer (same names, same semantics)
#else
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace srcv {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier -----------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  } while (!done);
}
// ---- bulk asynchronous copy global -> shared (TMA engine), completion on an mbarrier
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(smem_dst)),
      "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// generic-proxy writes to shared memory -> visible to the tensor core (async proxy)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- descriptors --------------------------------------------------------------------
// shared-memory operand descriptor, K-major, no swizzle (see header comment); bits [62,64) = 0
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);               // start address  [0,14)
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;      // leading offset [16,30)
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;      // stride offset  [32,46)
  return d;
}

// ---- warpgroup MMA (all 128 threads of an aligned warpgroup) --------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator registers across the asynchronous MMAs
template <int N> __device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 128] (+)= A[smem, 64 x 16] B[smem, 128 x 16]^T
__device__ __forceinline__ void wgmma_ss_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, "
      "%22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, "
      "%43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc), "r"(accumulate)
      : "memory");
}

// D[64 x 64] (+)= A[registers, 64 x 16] B[smem, 64 x 16]^T
__device__ __forceinline__ void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc,
                                             uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, "
      "%22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(accumulate)
      : "memory");
}

// ---- per-warpgroup register re-balancing (all 128 threads of an aligned warpgroup) ---------
template <int N> __device__ __forceinline__ void reg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N> __device__ __forceinline__ void reg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}

// ---- fp32 -> (hi, lo) fp16 pair split -------------------------------------------------------
// x = hi + lo with hi = rn16(x), lo = rn16(x - hi): 22 significand bits survive, so
//   A*W ~= A_hi*W_hi + A_hi*W_lo + A_lo*W_hi   (three fp16 MMAs, fp32 accumulate)
// is accurate to ~2^-22 per product — the fp32 noise level of the reference's own GEMMs.
// Magnitudes beyond the fp16 range saturate (65504) instead of becoming inf.
__device__ __forceinline__ uint32_t pack_f16x2_sat(float even, float odd) {
  uint32_t d;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(odd), "f"(even));  // {upper, lower}
  return d;
}
// The residual x - hi is one mixed-precision FMA per value (fma.rn.f32.f16: hi * (-1) + x).
__device__ __forceinline__ void split_pack(float even, float odd, uint32_t& hi, uint32_t& lo) {
  hi = pack_f16x2_sat(even, odd);
  const float2 h = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  lo = pack_f16x2_sat(even - h.x, odd - h.y);
}

}  // namespace tc
}  // namespace srcv
#endif  // SRCV_HOST_EMU
