// Producer-side fusion (SURVEY.md §8f-2): the last op of the reference's matching encoder,
// nn.InstanceNorm2d(16) without affine (reference modules/networks.py:201, eps 1e-5, biased
// variance), fused with the layout pass the sweeps need — the normalised features are written
// straight into the chunk-planar (…, C/4, H, W, 4) layout the gather kernels read, split into the
// reference-frame block and the source-view block (the encoder runs on the (B, 1+K) image stack
// and depth_model.py:242-243 slices it), so that neither the (B,1+K,C,H,W) NCHW tensor nor the
// prep pass's re-layout copy ever touches HBM.
#include "srcv_kernels.h"

namespace srcv {

namespace {

constexpr int kThreads = 256;

// One CTA per (image n, chunk of 4 channels).  Pass 1: sums in fp64 (19 200 pixels per channel:
// exact enough that mean / variance carry no visible summation-order noise).  Pass 2: re-read (L2),
// normalise, write one 16-byte vector per pixel.
__global__ void __launch_bounds__(kThreads)
instnorm_c4_kernel(const float* __restrict__ x, int V, int C, int HW, float eps,
                   float4* __restrict__ cur_c4, float4* __restrict__ src_c4) {
  const int chunks = C / 4;
  const int n = blockIdx.x / chunks, j = blockIdx.x % chunks;
  const float* xp = x + ((size_t)n * C + 4 * j) * HW;
  double s[4] = {0, 0, 0, 0}, ss[4] = {0, 0, 0, 0};
  for (int p = threadIdx.x; p < HW; p += kThreads) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const double v = (double)__ldg(xp + (size_t)c * HW + p);
      s[c] += v;
      ss[c] += v * v;
    }
  }
  __shared__ double red[8][kThreads];
#pragma unroll
  for (int c = 0; c < 4; ++c) { red[c][threadIdx.x] = s[c]; red[4 + c][threadIdx.x] = ss[c]; }
  block_tree<kThreads>([&](int i, int j) {
#pragma unroll
    for (int c = 0; c < 8; ++c) red[c][i] += red[c][j];
  });
  float mean[4], invstd[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const double m = red[c][0] / (double)HW;
    const double var = red[4 + c][0] / (double)HW - m * m;      // biased, as InstanceNorm uses
    mean[c] = (float)m;
    invstd[c] = 1.0f / sqrtf((float)(var > 0.0 ? var : 0.0) + eps);
  }
  // image n = b * V + v: v == 0 is the reference frame, v >= 1 source view v - 1
  const int b = n / V, v = n % V;
  float4* out = (v == 0) ? cur_c4 + ((size_t)b * chunks + j) * HW
                         : src_c4 + (((size_t)b * (V - 1) + (v - 1)) * chunks + j) * HW;
  for (int p = threadIdx.x; p < HW; p += kThreads) {
    out[p] = make_float4((__ldg(xp + p) - mean[0]) * invstd[0],
                         (__ldg(xp + (size_t)HW + p) - mean[1]) * invstd[1],
                         (__ldg(xp + 2 * (size_t)HW + p) - mean[2]) * invstd[2],
                         (__ldg(xp + 3 * (size_t)HW + p) - mean[3]) * invstd[3]);
  }
}

}  // namespace

cudaError_t launch_instnorm_c4(const float* x, int B, int V, int C, int H, int W, float eps, float* cur_c4,
                               float* src_c4, cudaStream_t stream) {
  const int blocks = B * V * (C / 4);
  SRCV_LAUNCH(instnorm_c4_kernel, blocks, kThreads, 0, stream, x, V, C, H * W, eps,
              reinterpret_cast<float4*>(cur_c4), reinterpret_cast<float4*>(src_c4));
  note_launch();
  return cudaGetLastError();
}

}  // namespace srcv
