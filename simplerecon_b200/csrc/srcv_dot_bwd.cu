// Backward of the dot-product plane-sweep volume (SURVEY.md §8f-1: "fused backward").
//
//   cost[b,d,p] = sum_k m_k(d,p) * sum_c cur[b,c,p] * sum_t w_t(d,k,p) * src[b,k,c,tap_t(d,k,p)]
//
// The sampling positions, weights and masks depend on the cameras and the plane depths
// only, never on the features, so with g = dL/dcost
//   dL/dcur[b,c,p]        = sum_{d,k}   g[b,d,p] m_k sum_t w_t src[b,k,c,tap_t]
//   dL/dsrc[b,k,c,texel] += sum_{d,p,t: tap_t = texel} g[b,d,p] m_k w_t cur[b,c,p]
// are exact (this is what autograd of the reference's grid_sample / mul / sum composite
// computes for its feature inputs, modules/cost_volume.py:305-333).  Cameras and plane
// depths receive no gradient — the training loop never asks for one.
//
// One thread per pixel re-projects every (plane, view) sample like the forward sweep,
// accumulates dL/dcur in registers and scatters dL/dsrc with float atomics (RED.ADD.F32 into
// the L2-resident gradient tensor).  Atomic accumulation order varies run to run, so
// dL/dsrc is reproducible only to fp32 rounding.
#include "srcv_kernels.h"

namespace srcv {

namespace {

template <int C, bool PER_PIXEL>
__global__ void __launch_bounds__(128)
dot_backward_kernel(srcv_shape s, const float* __restrict__ cur, const float* __restrict__ src,
                    const ViewParams* __restrict__ views, const float* __restrict__ planes,
                    const float* __restrict__ gcost, float* __restrict__ gcur, float* __restrict__ gsrc,
                    int d_begin, int d_end, bool accumulate_gcur) {
  SRCV_DYNAMIC_SMEM(float, sview);  // K * 12
  const int b = blockIdx.y;
  const int W = s.W, H = s.H, HW = W * H, K = s.K;
  for (int i = threadIdx.x; i < K * kViewFloats; i += blockDim.x)
    sview[i] = reinterpret_cast<const float*>(views + b * K + i / kViewFloats)[i % kViewFloats];
  __syncthreads();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const Centre ctr(W, H);
  const float dx = ((float)(p % W) + 0.5f) - ctr.half_w, dy = ((float)(p / W) + 0.5f) - ctr.half_h;
  float curv[C], acc[C];
#pragma unroll
  for (int c = 0; c < C; ++c) {
    curv[c] = __ldg(cur + ((size_t)b * C + c) * HW + p);
    acc[c] = 0.f;
  }
  for (int d = d_begin; d < d_end; ++d) {
    const float g = __ldg(gcost + ((size_t)b * s.D + d) * HW + p);
    if (g == 0.0f) continue;
    const float dval = plane_depth<PER_PIXEL>(planes, b, s.D, d, HW, p);
    for (int k = 0; k < K; ++k) {
      const Sample sm = project_sample(sview + k * kViewFloats, ctr, W, H, dx, dy, dval);
      const Taps& tp = sm.tp;
      if (!(sm.zp > 0.0f) || tp.valid == 0u) continue;
      // own weights: g * gx * gy rounds differently from g * sm.w00 = g * (gx * gy)
      const float gx = 1.0f - tp.fx, gy = 1.0f - tp.fy;
      const float wgt[4] = {g * gx * gy, g * tp.fx * gy, g * gx * tp.fy, g * tp.fx * tp.fy};
      const int off[4] = {0, 1, W, W + 1};
      const size_t base = ((size_t)(b * K + k) * C) * HW + (tp.y0 * W + tp.x0);
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        if (!((tp.valid >> t) & 1u)) continue;
        const float* sp = src + base + off[t];
        float* gp = gsrc + base + off[t];
#pragma unroll
        for (int c = 0; c < C; ++c) {
          acc[c] = fmaf(wgt[t], __ldg(sp + (size_t)c * HW), acc[c]);
          atomicAdd(gp + (size_t)c * HW, wgt[t] * curv[c]);
        }
      }
    }
  }
#pragma unroll
  for (int c = 0; c < C; ++c) {
    float* o = gcur + ((size_t)b * C + c) * HW + p;
    *o = accumulate_gcur ? *o + acc[c] : acc[c];
  }
}

}  // namespace

bool dot_backward_supported(const srcv_shape& s) { return s.C == 8 || s.C == 16 || s.C == 32; }

// gsrc must be zero-filled by the caller (it is accumulated into); gcur is overwritten.
cudaError_t launch_dot_backward(const srcv_shape& s, const float* cur, const float* src,
                                const Workspace& ws, const float* planes, bool per_pixel,
                                const float* gcost, float* gcur, float* gsrc, cudaStream_t stream) {
  const int HW = s.H * s.W;
  dim3 grid((HW + 127) / 128, s.B), block(128);
  const size_t smem = sizeof(float) * kViewFloats * s.K;
#define SRCV_BWD(CC)                                                                                  \
  if (s.C == CC) {                                                                                    \
    if (per_pixel)                                                                                    \
      SRCV_LAUNCH((dot_backward_kernel<CC, true>), grid, block, smem, stream, s, cur, src, ws.views,     \
                  planes, gcost, gcur, gsrc, 0, s.D, false);                                          \
    else                                                                                              \
      SRCV_LAUNCH((dot_backward_kernel<CC, false>), grid, block, smem, stream, s, cur, src, ws.views,    \
                  planes, gcost, gcur, gsrc, 0, s.D, false);                                          \
    note_launch();                                                                                    \
    return cudaGetLastError();                                                                        \
  }
  SRCV_BWD(8) SRCV_BWD(16) SRCV_BWD(32)
#undef SRCV_BWD
  return cudaErrorInvalidValue;
}

}  // namespace srcv
