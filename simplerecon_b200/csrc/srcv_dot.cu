// Dot-product plane-sweep volume — replaces CostVolumeManager.build_cost_volume
// (+ the argmax of CostVolumeManager.forward), reference
// modules/cost_volume.py:237-335, :345-380.
//
//   cost[b,d,p] = sum_k [z'_k > 0] * sum_c cur[b,c,p] * bilinear(src[b,k,c], proj_k(d, p))
//
// The (B,K,D,C,H,W) warped tensor of the reference is never formed: every
// (plane, view, pixel) sample is projected, gathered and reduced in registers.
//
// Two variants:
//  * generic — any K, C; one thread per pixel, planar (NCHW) scalar gathers.
//  * fast    — C == 16; one thread per pixel, a warp owns a 16x2 block of pixels
//    (2-D so the bilinear footprints overlap in both directions).  It gathers
//    from the chunk-planar copy made by the prep pass, laid out (B,K,C/4,H,W,4):
//    the 4-channel chunk of a texel is one 16-byte vector and horizontally
//    adjacent texels are adjacent in memory, so the warp-wide LDG.128 of a tap
//    reads two 256-byte row segments: the full-width 128 B/clk L1 access shape
//    with every lane keeping its own sample (no cross-lane traffic at all, where
//    a channel-last texel layout needs shuffles to re-partition the warp).  Loop
//    order is plane-chunk -> view -> plane-in-chunk, so consecutive samples walk
//    along one epipolar line of one view and re-hit the lines just pulled into L1.
#include <cstdlib>

#include "srcv_kernels.h"

namespace srcv {

namespace {

// --------------------------------------------------------------------------- //
// generic                                                                     //
// --------------------------------------------------------------------------- //
template <bool PER_PIXEL>
__global__ void __launch_bounds__(128)
dot_generic_kernel(srcv_shape s, const float* __restrict__ cur, const float* __restrict__ src,
                   const ViewParams* __restrict__ views, const float* __restrict__ planes,
                   float* __restrict__ cost, float* __restrict__ lowest) {
  SRCV_DYNAMIC_SMEM(float, sview);  // K * 12: a0, hx, hy, t
  const int b = blockIdx.y;
  const int HW = s.H * s.W;
  for (int i = threadIdx.x; i < s.K * kViewFloats; i += blockDim.x)
    sview[i] = reinterpret_cast<const float*>(views + b * s.K + i / kViewFloats)[i % kViewFloats];
  __syncthreads();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const Centre ctr(s.W, s.H);
  const float dx = ((float)(p % s.W) + 0.5f) - ctr.half_w, dy = ((float)(p / s.W) + 0.5f) - ctr.half_h;
  const float* curp = cur + (size_t)b * s.C * HW + p;
  float best = 0.f, best_d = 0.f;
  for (int d = 0; d < s.D; ++d) {
    const float dval = PER_PIXEL ? __ldg(planes + ((size_t)b * s.D + d) * HW + p)
                                 : __ldg(planes + b * s.D + d);
    float acc = 0.f;
    for (int k = 0; k < s.K; ++k) {
      const float* vp = sview + k * kViewFloats;
      float ax, ay, az, px, py, zp;
      homography_point(vp, dx, dy, ax, ay, az);
      project_point(dval, ax, ay, az, vp[9], vp[10], vp[11], px, py, zp);
      Taps tp;
      bilinear_taps(px, py, s.W, s.H, ctr, tp);
      if (!(zp > 0.0f) || tp.valid == 0u) continue;  // mask == 0 or all taps padded
      const float w00 = (1.0f - tp.fx) * (1.0f - tp.fy), w01 = tp.fx * (1.0f - tp.fy);
      const float w10 = (1.0f - tp.fx) * tp.fy, w11 = tp.fx * tp.fy;
      const float* sp = src + ((size_t)(b * s.K + k) * s.C) * HW + (tp.y0 * s.W + tp.x0);
      float dot = 0.f;
      for (int c = 0; c < s.C; ++c) {
        const float* q = sp + (size_t)c * HW;
        float v = 0.f;
        if (tp.valid & 1u) v = w00 * __ldg(q);
        if (tp.valid & 2u) v = fmaf(w01, __ldg(q + 1), v);
        if (tp.valid & 4u) v = fmaf(w10, __ldg(q + s.W), v);
        if (tp.valid & 8u) v = fmaf(w11, __ldg(q + s.W + 1), v);
        dot = fmaf(v, __ldg(curp + (size_t)c * HW), dot);
      }
      acc += dot;
    }
    cost[((size_t)b * s.D + d) * HW + p] = acc;
    argmax_update(acc, dval, best, best_d, d == 0);
  }
  if (lowest) lowest[(size_t)b * HW + p] = best_d;
}

// --------------------------------------------------------------------------- //
// fast: one thread per pixel, gathers from the chunk-planar (B,K,C/4,H,W,4) copy //
// --------------------------------------------------------------------------- //
constexpr int kFastC = 16;
constexpr int kNChunk = kFastC / 4;
constexpr int kFastWarps = 2;           // CTA = 16 x 4 pixels
constexpr int kDC = 4;                  // planes per inner chunk

// One bilinear tap: C/4 vector loads at compile-time-constant distances from the sample's base
// pointer, reduced against the reference features as two packed chains (even / odd channels: FFMA2,
// two IEEE FMAs per issue slot — the sweep shares its issue slots between 16 loads and 64 FMAs per
// sample).
template <bool PRED, int HWC>
__device__ __forceinline__ float tap_dot(const float4* __restrict__ q, int hw, bool on,
                                         const float4 (&cur4)[kNChunk]) {
  const int stride = HWC ? HWC : hw;
  float4 v[kNChunk];
#pragma unroll
  for (int j = 0; j < kNChunk; ++j) {
    if (PRED) v[j] = on ? __ldg(q + (size_t)j * stride) : make_float4(0.f, 0.f, 0.f, 0.f);
    else v[j] = __ldg(q + (size_t)j * stride);
  }
  float2 ta = make_float2(0.f, 0.f), tb = make_float2(0.f, 0.f);
#pragma unroll
  for (int j = 0; j < kNChunk; ++j) {
    ta = fma2(make_float2(v[j].x, v[j].y), make_float2(cur4[j].x, cur4[j].y), ta);
    tb = fma2(make_float2(v[j].z, v[j].w), make_float2(cur4[j].z, cur4[j].w), tb);
  }
  return (ta.x + ta.y) + (tb.x + tb.y);
}

// TW, TH: compile-time feature-map size (0 = take it from the shape at run time).
// With a known size every one of the 16 vector loads of a sample is the sample's
// base pointer plus an immediate, which removes ~45 integer instructions per sample.
template <bool PER_PIXEL, int TW, int TH, int kTileW>
// 68 registers / 28 warps per SM: capping at 64 (32 warps) spills 36 bytes and measures 0.8 % slower (call R)
__global__ void __launch_bounds__(kFastWarps * 32)
dot_fast_kernel(srcv_shape s, const float* __restrict__ cur, const float4* __restrict__ src4,
                const ViewParams* __restrict__ views, const float* __restrict__ planes,
                float* __restrict__ cost, float* __restrict__ lowest, unsigned* __restrict__ tile_done) {
  SRCV_DYNAMIC_SMEM(float, sview);  // K * 12
  const int b = blockIdx.y;
  const int W = TW ? TW : s.W, H = TH ? TH : s.H, HW = W * H, K = s.K;
  constexpr int HWC = TW * TH;
  constexpr int kTileH = 32 / kTileW;  // pixels per warp: lane -> (lane % kTileW, lane / kTileW)
  for (int i = threadIdx.x; i < K * kViewFloats; i += blockDim.x)
    sview[i] = reinterpret_cast<const float*>(views + b * K + i / kViewFloats)[i % kViewFloats];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int tiles_x = (W + kTileW - 1) / kTileW;
  const int ox_raw = (blockIdx.x % tiles_x) * kTileW + (lane & (kTileW - 1));
  const int oy_raw = ((blockIdx.x / tiles_x) * kFastWarps + (threadIdx.x >> 5)) * kTileH + lane / kTileW;
  const bool active = ox_raw < W && oy_raw < H;   // idle lanes / warps shadow a real pixel
  const int ox = min(ox_raw, W - 1), oy = min(oy_raw, H - 1);  // idle lanes shadow a real pixel
  // planes handled by this CTA: [d_begin, d_end)
  const int dper = (s.D + gridDim.z - 1) / gridDim.z;
  const int d_begin = blockIdx.z * dper;
  const int d_end = min(s.D, d_begin + dper);
  const bool fuse_argmax = (gridDim.z == 1) && (lowest != nullptr);
  const Centre ctr(W, H);
  const int p = oy * W + ox;
  const float dx = ((float)ox + 0.5f) - ctr.half_w, dy = ((float)oy + 0.5f) - ctr.half_h;

  float4 cur4[kNChunk];
  if (s.layout == SRCV_LAYOUT_CHUNK_PLANAR) {     // producer already wrote (B,C/4,H,W,4)
#pragma unroll
    for (int j = 0; j < kNChunk; ++j)
      cur4[j] = __ldg(reinterpret_cast<const float4*>(cur) + ((size_t)b * kNChunk + j) * HW + p);
  } else {
#pragma unroll
    for (int j = 0; j < kNChunk; ++j) {
      const float* cp = cur + ((size_t)b * kFastC + 4 * j) * HW + p;
      cur4[j] = make_float4(__ldg(cp), __ldg(cp + HW), __ldg(cp + 2 * (size_t)HW), __ldg(cp + 3 * (size_t)HW));
    }
  }
  float best = 0.f, best_d = 0.f;

  for (int d0 = d_begin; d0 < d_end; d0 += kDC) {
    float dval[kDC], acc[kDC];
#pragma unroll
    for (int dd = 0; dd < kDC; ++dd) {
      const int d = min(d0 + dd, d_end - 1);
      dval[dd] = PER_PIXEL ? __ldg(planes + ((size_t)b * s.D + d) * HW + p)
                           : __ldg(planes + b * s.D + d);
      acc[dd] = 0.f;
    }
#pragma unroll 1
    for (int k = 0; k < K; ++k) {
      const float* vp = sview + k * kViewFloats;
      float ax, ay, az;
      homography_point(vp, dx, dy, ax, ay, az);
      const float tx = vp[9], ty = vp[10], tz = vp[11];
      const float4* view4 = src4 + (size_t)(b * K + k) * kNChunk * HW;
#pragma unroll
      for (int dd = 0; dd < kDC; ++dd) {
        float px, py, zp;
        project_point(dval[dd], ax, ay, az, tx, ty, tz, px, py, zp);
        Taps tp;
        bilinear_taps(px, py, W, H, ctr, tp);
        const unsigned valid = (zp > 0.0f) ? tp.valid : 0u;  // depth mask folded into the footprint
        const float gx = 1.0f - tp.fx, gy = 1.0f - tp.fy;
        const float4* q = view4 + (tp.y0 * W + tp.x0);
        float t0, t1, t2, t3;
        if (__all_sync(0xffffffffu, valid == 15u)) {
          // interior sample for the whole warp: 16 unconditional vector loads
          t0 = tap_dot<false, HWC>(q, HW, true, cur4);
          t1 = tap_dot<false, HWC>(q + 1, HW, true, cur4);
          t2 = tap_dot<false, HWC>(q + W, HW, true, cur4);
          t3 = tap_dot<false, HWC>(q + W + 1, HW, true, cur4);
        } else {
          // border / behind-camera lanes: padding taps are not loaded (zeros)
          t0 = tap_dot<true, HWC>(q, HW, valid & 1u, cur4);
          t1 = tap_dot<true, HWC>(q + 1, HW, valid & 2u, cur4);
          t2 = tap_dot<true, HWC>(q + W, HW, valid & 4u, cur4);
          t3 = tap_dot<true, HWC>(q + W + 1, HW, valid & 8u, cur4);
        }
        acc[dd] = fmaf(gx * gy, t0, fmaf(tp.fx * gy, t1, fmaf(gx * tp.fy, t2,
                       fmaf(tp.fx * tp.fy, t3, acc[dd]))));
      }
    }
#pragma unroll
    for (int dd = 0; dd < kDC; ++dd) {
      const int d = d0 + dd;
      if (d < d_end) {
        if (active) cost[((size_t)b * s.D + d) * HW + p] = acc[dd];
        argmax_update(acc[dd], dval[dd], best, best_d, d == d_begin);
      }
    }
  }
  if (fuse_argmax && active) lowest[(size_t)b * HW + p] = best_d;
  if (gridDim.z > 1 && lowest != nullptr) {
    // Plane loop split over gridDim.z CTAs: the LAST CTA of this pixel tile to finish
    // (counter zeroed by the prep pass) reduces the whole plane column it finds in L2 — the
    // argmax stays fused without a second launch.
    __shared__ unsigned s_last;
    __threadfence();                       // this CTA's cost values are visible device-wide
    __syncthreads();
    if (threadIdx.x == 0)
      s_last = (atomicAdd(tile_done + (size_t)b * gridDim.x + blockIdx.x, 1u) == gridDim.z - 1) ? 1u : 0u;
    __syncthreads();
    if (s_last && active) {
      __threadfence();
      const float* c = cost + (size_t)b * s.D * HW + p;
      float bv = 0.f, bd = 0.f;
#pragma unroll 8
      for (int d = 0; d < s.D; ++d) {
        const float v = __ldcg(c + (size_t)d * HW);   // L2, never a stale L1 line
        const float dv = PER_PIXEL ? __ldg(planes + ((size_t)b * s.D + d) * HW + p) : __ldg(planes + b * s.D + d);
        argmax_update(v, dv, bv, bd, d == 0);
      }
      lowest[(size_t)b * HW + p] = bd;
    }
  }
}

template <bool PER_PIXEL, int kTileW>
void launch_fast_sized(const srcv_shape& s, dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                       const float* cur, const float4* src4, const ViewParams* views,
                       const float* planes, float* cost, float* lowest, unsigned* tile_done) {
#define SRCV_SIZED(TW_, TH_)                                                                   \
  if (s.W == TW_ && s.H == TH_) {                                                              \
    SRCV_LAUNCH((dot_fast_kernel<PER_PIXEL, TW_, TH_, kTileW>), grid, block, smem, stream,       \
                s, cur, src4, views, planes, cost, lowest, tile_done);                         \
    return;                                                                                    \
  }
  SRCV_SIZED(160, 120)  // 640x480 frames (BASELINE configs)
  SRCV_SIZED(128, 96)   // 512x384 frames (the reference's default, options.py:70-71)
  SRCV_SIZED(64, 48)    // 256x192 frames (BASELINE config 0)
#undef SRCV_SIZED
  SRCV_LAUNCH((dot_fast_kernel<PER_PIXEL, 0, 0, kTileW>), grid, block, smem, stream, s, cur, src4, views, planes,
              cost, lowest, tile_done);
}

// --------------------------------------------------------------------------- //
// warp only: the materialising helper the reference exposes as warp_features()  //
// --------------------------------------------------------------------------- //
// One thread per (frame, view, plane, pixel): grid.z walks the planes, so D = 1 is the reference's
// single-plane CostVolumeManager.warp_features (modules/cost_volume.py:139-234) and D > 1 the
// all-planes FastFeatureVolumeManager.warp_features (:812-964) — output layouts (B,K,D,C,H,W),
// (B,K,D,H,W), and the un-centred pixel coordinates (B,K,D,2,H,W) the fast manager also returns.
template <bool PER_PIXEL>
__global__ void __launch_bounds__(128)
warp_planes_kernel(srcv_shape s, const float* __restrict__ src, const ViewParams* __restrict__ views,
                   const float* __restrict__ planes, float* __restrict__ warped,
                   float* __restrict__ depths, float* __restrict__ mask, float* __restrict__ pix) {
  const int HW = s.H * s.W;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int bk = blockIdx.y, b = bk / s.K, d = blockIdx.z;
  if (p >= HW) return;
  const Centre ctr(s.W, s.H);
  const float dx = ((float)(p % s.W) + 0.5f) - ctr.half_w, dy = ((float)(p / s.W) + 0.5f) - ctr.half_h;
  const float dval = PER_PIXEL ? __ldg(planes + ((size_t)b * s.D + d) * HW + p) : __ldg(planes + b * s.D + d);
  const ViewParams& vp = views[bk];
  float ax, ay, az, px, py, zp;
  homography_point(vp.a0, dx, dy, ax, ay, az);
  project_point(dval, ax, ay, az, vp.t[0], vp.t[1], vp.t[2], px, py, zp);
  Taps tp;
  bilinear_taps(px, py, s.W, s.H, ctr, tp);
  const float w00 = (1.0f - tp.fx) * (1.0f - tp.fy), w01 = tp.fx * (1.0f - tp.fy);
  const float w10 = (1.0f - tp.fx) * tp.fy, w11 = tp.fx * tp.fy;
  const float* sp = src + (size_t)bk * s.C * HW + (tp.y0 * s.W + tp.x0);
  const size_t o = (size_t)bk * s.D + d;
  for (int c = 0; c < s.C; ++c) {
    const float* q = sp + (size_t)c * HW;
    float v = 0.f;
    if (tp.valid & 1u) v = w00 * __ldg(q);
    if (tp.valid & 2u) v = fmaf(w01, __ldg(q + 1), v);
    if (tp.valid & 4u) v = fmaf(w10, __ldg(q + s.W), v);
    if (tp.valid & 8u) v = fmaf(w11, __ldg(q + s.W + 1), v);
    warped[(o * s.C + c) * HW + p] = v;
  }
  depths[o * HW + p] = zp;
  mask[o * HW + p] = zp > 0.0f ? 1.0f : 0.0f;
  if (pix != nullptr) {
    // the projector's pixel coordinates (utils/geometry_utils.py:88-89): ours are centred
    pix[(o * 2 + 0) * HW + p] = px + ((float)ctr.nx + 0.5f);
    pix[(o * 2 + 1) * HW + p] = py + ((float)ctr.ny + 0.5f);
  }
}

}  // namespace

cudaError_t launch_warp_planes(const srcv_shape& s, const float* src, const Workspace& ws,
                               const float* planes, bool per_pixel, float* warped, float* depths,
                               float* mask, float* pix, cudaStream_t stream) {
  dim3 grid((s.H * s.W + 127) / 128, s.B * s.K, s.D), block(128);
  if (per_pixel) SRCV_LAUNCH(warp_planes_kernel<true>, grid, block, 0, stream, s, src, ws.views, planes, warped, depths, mask, pix);
  else SRCV_LAUNCH(warp_planes_kernel<false>, grid, block, 0, stream, s, src, ws.views, planes, warped, depths, mask, pix);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_dot_generic(const srcv_shape& s, const float* cur, const float* src,
                               const Workspace& ws, const float* planes, bool per_pixel,
                               float* cost, float* lowest, cudaStream_t stream) {
  const int HW = s.H * s.W;
  dim3 grid((HW + 127) / 128, s.B), block(128);
  const size_t smem = sizeof(float) * kViewFloats * s.K;
  if (per_pixel)
    SRCV_LAUNCH(dot_generic_kernel<true>, grid, block, smem, stream, s, cur, src, ws.views, planes, cost, lowest);
  else
    SRCV_LAUNCH(dot_generic_kernel<false>, grid, block, smem, stream, s, cur, src, ws.views, planes, cost, lowest);
  note_launch();
  return cudaGetLastError();
}

bool dot_fast_supported(const srcv_shape& s) {
  // (texel index * 16) must fit an int; 16-byte texel chunks need C == 16
  return s.C == kFastC && (long long)s.H * s.W < (1ll << 26) && s.K <= 512;
}

cudaError_t launch_dot_fast(const srcv_shape& s, const float* cur, const Workspace& ws,
                            const float* planes, bool per_pixel, float* cost, float* lowest,
                            cudaStream_t stream) {
  // Split the plane loop across CTAs until there are ~64 warps per SM to schedule (the
  // sweep is latency-bound at low occupancy and smaller CTAs balance better: measured
  // 428 -> 370 us at B = 4); the argmax of a split sweep is done by the last CTA of each
  // pixel tile to finish (see the kernel).
  int dev = 0, sms = 1;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  static const int tile_w = [] {
    const char* e = getenv("SRCV_DOT_TILE_W");  // tuning knob: 16 (16x2 warp tile) or 32 (32x1)
    return (e && atoi(e) == 32) ? 32 : 16;
  }();
  const int kTileW = tile_w, kTileH = 32 / tile_w;
  const int tiles_x = (s.W + kTileW - 1) / kTileW;
  const int tiles_y = (s.H + kTileH * kFastWarps - 1) / (kTileH * kFastWarps);
  const long long warps = (long long)s.B * tiles_x * tiles_y * kFastWarps;
  static const long long want = [] {
    const char* e = getenv("SRCV_DOT_WARPS_PER_SM");  // tuning knob, default 128
    return (long long)(e ? atoi(e) : 128);  // 128: ~4 CTA waves at cfg1, 3 % less tail than 64
  }();
  int d_split = 1;
  while (d_split < 8 && warps * d_split < want * sms && s.D / (d_split * 2) >= 2 * kDC) d_split *= 2;
  dim3 grid(tiles_x * tiles_y, s.B, d_split), block(kFastWarps * 32);
  const size_t smem = sizeof(float) * kViewFloats * s.K;
  const float4* src4 = reinterpret_cast<const float4*>(ws.src_c4);
  unsigned* done = ws.tile_done;
  if (d_split > 1 && lowest && (done == nullptr || (size_t)grid.x * s.B > ws.tile_done_count))
    return cudaErrorInvalidValue;
  if (tile_w == 32) {
    if (per_pixel) launch_fast_sized<true, 32>(s, grid, block, smem, stream, cur, src4, ws.views, planes, cost, lowest, done);
    else launch_fast_sized<false, 32>(s, grid, block, smem, stream, cur, src4, ws.views, planes, cost, lowest, done);
  } else {
    if (per_pixel) launch_fast_sized<true, 16>(s, grid, block, smem, stream, cur, src4, ws.views, planes, cost, lowest, done);
    else launch_fast_sized<false, 16>(s, grid, block, smem, stream, cur, src4, ws.views, planes, cost, lowest, done);
  }
  note_launch();
  return cudaGetLastError();
}

size_t dot_fast_tile_counters(const srcv_shape& s) {
  // upper bound over both warp-tile shapes (16x4- and 32x2-pixel CTAs)
  const size_t a = (size_t)((s.W + 15) / 16) * ((s.H + 3) / 4), b = (size_t)((s.W + 31) / 32) * ((s.H + 1) / 2);
  return (size_t)s.B * (a > b ? a : b);
}

}  // namespace srcv
