// Shared device-side geometry for the plane-sweep kernels (sm_90a).
//
// The arithmetic restated here is the reference's
//   BackprojectDepth.forward   utils/geometry_utils.py:51-59  (+0.5 pixel centres :34-44)
//   Project3D.forward          utils/geometry_utils.py:72-89  (eps 1e-8)
//   uv normalisation           modules/cost_volume.py:199, :587
//   F.grid_sample(bilinear, zeros, align_corners=False)  modules/cost_volume.py:201-212
// re-associated for the GPU.  The depth-invariant part of the projection,
//   Hm = (K E)[:3,:3] invK[:3,:3]   and   t = (K E)[:3,3],
// is folded once per (frame, view) by the prep kernel in fp64, so a plane hypothesis d
// at pixel centre p projects with three FMAs,  c = d (Hm p) + t  — the plane-induced
// homography of the sweep.
//
// Precision: everything is evaluated in *centred* pixel coordinates.  The input
// pixel is taken relative to the image centre (exact in fp32) and the projected
// coordinate relative to (floor(W/2)+0.5, floor(H/2)+0.5), i.e. the prep kernel
// folds   c'_x = c_x - cxo c_z   into Hm and t.  In exact arithmetic the sample
// index of grid_sample (align_corners=False, after the reference's 2 p / W - 1
// normalisation) is  i_x = p_x - 0.5 = p'_x + floor(W/2), so floor() and the
// bilinear fraction are taken on p' (|p'| <= W/2: half the ulp of the reference's
// un-centred chain, and no normalise/unnormalise round trip).  Measured against the
// fp64 evaluation of the reference this is closer than the reference's own fp32
// result (DESIGN.md, "numerics").
#pragma once
#ifdef SRCV_HOST_EMU
#include "emu_cuda.h"   // tests/emu: host emulation of the CUDA execution model
#else
#include <cuda_runtime.h>
#endif
#include <stdint.h>

// Dynamic shared memory of a kernel (one definition so the host emulation can map it).
#ifdef SRCV_HOST_EMU
#define SRCV_DYNAMIC_SMEM(type, name) type* name = reinterpret_cast<type*>(::emu::dynamic_smem())
#define SRCV_DYNAMIC_SMEM_ALIGNED(type, name, n) SRCV_DYNAMIC_SMEM(type, name)
#else
#define SRCV_DYNAMIC_SMEM(type, name) extern __shared__ type name[]
#define SRCV_DYNAMIC_SMEM_ALIGNED(type, name, n) extern __shared__ __align__(n) type name[]
#endif

namespace srcv {

constexpr float kEpsProj = 1e-8f;   // utils/geometry_utils.py:66
constexpr float kEpsNorm = 1e-12f;  // F.normalize default
constexpr float kEpsCos = 1e-5f;    // modules/cost_volume.py:687
constexpr float kLeaky = 0.01f;     // nn.LeakyReLU default slope

// ---- fp32 pairs: two independent IEEE FMAs / multiplies on (even, odd) channel pairs -----------
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

// Per (frame b, view k) constants, written by prep_kernel.  32 floats = 128 B.
struct __align__(16) ViewParams {
  float a0[3];     // centred homography applied to the image centre
  float hx[3];     // d a'/d dx  (column 0 of the centred Hm)
  float hy[3];     // d a'/d dy  (column 1)
  float t[3];      // centred translation
  float centre[3]; // src_poses[:3,3]: source camera centre in the reference frame
  float comb;      // pose_distance: sqrt(t_meas^2 + r_meas^2)
  float rmeas;     // sqrt(2 (1 - min(3, tr R)/3))
  float tmeas;     // |src_poses[:3,3]|
  uint32_t rt_hi;  // (rmeas, tmeas) as fp16 (hi, lo) operand words
  uint32_t rt_lo;  //   (csrc/srcv_tc.cuh split_pack)
  float pad[12];
};
static_assert(sizeof(ViewParams) == 128, "ViewParams must be 128 bytes");
constexpr int kViewFloats = 12;  // a0, hx, hy, t: what the sweep kernels stage in smem

// Per frame constants: invK[:3,:3] (row-major) for the ray r = invK3 p.
struct __align__(16) FrameParams {
  float invK[9];
  float pad[7];
};
static_assert(sizeof(FrameParams) == 64, "FrameParams must be 64 bytes");

// Image-size constants of the centred frame.
struct Centre {
  float half_w, half_h;  // W/2, H/2: input centre (pixel centres are u+0.5)
  int nx, ny;            // floor(W/2), floor(H/2): integer part of the output offset
  __host__ __device__ Centre(int W, int H)
      : half_w(0.5f * (float)W), half_h(0.5f * (float)H), nx(W / 2), ny(H / 2) {}
};

// a' = a0 + hx dx + hy dy  for pixel (u, v)
__device__ __forceinline__ void homography_point(const float* __restrict__ vp, float dx, float dy,
                                                 float& ax, float& ay, float& az) {
  ax = fmaf(vp[3], dx, fmaf(vp[6], dy, vp[0]));
  ay = fmaf(vp[4], dx, fmaf(vp[7], dy, vp[1]));
  az = fmaf(vp[5], dx, fmaf(vp[8], dy, vp[2]));
}

// c' = d a' + t', guarded divide (geometry_utils.py:83-89).  px, py are CENTRED.
__device__ __forceinline__ void project_point(float d, float ax, float ay, float az,
                                              float tx, float ty, float tz,
                                              float& px, float& py, float& zp) {
  const float cx = fmaf(d, ax, tx);
  const float cy = fmaf(d, ay, ty);
  const float z = fmaf(d, az, tz);
  zp = __fadd_rn(z, kEpsProj);
  // 1/z': hardware reciprocal + one Newton step (branch-free, <= 1 ulp) instead of the
  // IEEE-rounded division's slow path; the residual is far below the pixel-coordinate
  // rounding that follows.
  float r;
#ifdef SRCV_HOST_EMU
  r = 1.0f / zp;
#else
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(zp));
#endif
  r = fmaf(r, fmaf(-zp, r, 1.0f), r);
  const float s = (fabsf(z) > kEpsProj) ? r : 1.0f;
  px = cx * s;
  py = cy * s;
}

// Bilinear footprint of one projected sample (centred coordinates in).
struct Taps {
  int x0, y0;      // top-left texel (may be out of range by one)
  float fx, fy;    // fractions: weights are (1-fx|fx) x (1-fy|fy)
  unsigned valid;  // bit0 nw, bit1 ne, bit2 sw, bit3 se in-bounds (zeros padding otherwise)
};

__device__ __forceinline__ void bilinear_taps(float px, float py, int W, int H, const Centre& c,
                                              Taps& tp) {
  const float x0f = floorf(px), y0f = floorf(py);
  tp.fx = px - x0f;
  tp.fy = py - y0f;
  // NaN / inf / absurd coordinates sample nothing (all four taps are padding)
  const bool finite = (fabsf(px) < 1.0e6f) && (fabsf(py) < 1.0e6f);
  const int x0 = finite ? (int)x0f + c.nx : -2;
  const int y0 = finite ? (int)y0f + c.ny : -2;
  const bool xa = (unsigned)x0 < (unsigned)W, xb = (unsigned)(x0 + 1) < (unsigned)W;
  const bool ya = (unsigned)y0 < (unsigned)H, yb = (unsigned)(y0 + 1) < (unsigned)H;
  tp.valid = (unsigned)(xa && ya) | ((unsigned)(xb && ya) << 1) | ((unsigned)(xa && yb) << 2) |
             ((unsigned)(xb && yb) << 3);
  const bool any = tp.valid != 0u;
  tp.x0 = any ? x0 : 0;
  tp.y0 = any ? y0 : 0;
}

// Bounds test of CostVolumeManager.get_mask (modules/cost_volume.py:90-95) on
// centred coordinates: 2 < p < size - 2.
__device__ __forceinline__ bool in_mask_bounds(float px, float py, int W, int H, const Centre& c) {
  const float ox = (float)c.nx + 0.5f, oy = (float)c.ny + 0.5f;
  return px > 2.0f - ox && px < (float)(W - 2) - ox && py > 2.0f - oy && py < (float)(H - 2) - oy;
}

__device__ __forceinline__ float leaky(float x) { return fmaxf(x, kLeaky * x); }

// 1 / max(sqrt(s), eps) for s >= 0: hardware rsqrt + one Newton step (< 1 ulp), no
// division and no IEEE-sqrt slow path.  Used for F.normalize / cosine_similarity.
__device__ __forceinline__ float inv_norm(float s, float eps) {
  float y;
#ifdef SRCV_HOST_EMU
  y = 1.0f / sqrtf(s);
#else
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(s));
#endif
  y = y * fmaf(-0.5f * s, y * y, 1.5f);
  return (s > eps * eps) ? y : (1.0f / eps);   // eps is a literal at every call site: folds to a constant
}

// argmax update with torch.argmax semantics: first index wins ties, NaN is max.
__device__ __forceinline__ void argmax_update(float v, float dval, float& best, float& best_d,
                                              bool first) {
  const bool take = first || (v > best) || ((v != v) && (best == best));
  if (take) { best = v; best_d = dval; }
}

}  // namespace srcv
