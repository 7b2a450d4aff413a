// Multi-scale gradient loss and scale-invariant loss — MSGradientLoss (losses.py:11-37, Equation 3 of the
// paper; experiment_modules/depth_model.py:466, :487) and ScaleInvariantLoss (losses.py:39-54, :468) of the
// reference.  DESIGN §4.14.
//
//   level 0 = the input; level l = blur_pool2d(level l-1, 3): the [1,2,1] x [1,2,1] / 16 kernel at stride 2
//             with ZERO padding 1 (taps outside the map are dropped, so border outputs are darkened), size
//             ceil(h / 2)
//   Gx, Gy  = Sobel / 8 with replicate padding, per level, of the ground truth and of the prediction
//   mask    = per gradient component: every one of the nine clamped window values of the ground truth at that
//             level is finite (the reference's convolution multiplies the zero taps too).  A non-finite value
//             spreads down the pyramid through the blur's arithmetic.
//   loss    = sum_l mean over the masked components of |G(pred_l) - G(gt_l)|; a level without a masked
//             component contributes 0 / 0 = NaN, and no gradient.
//
//   forward : (1) the pyramids, one launch: a CTA stages a 64x64 level-0 tile of one tensor with the halo
//             three blur-pools need (71x71), reduces it in shared memory to 32x32, 16x16 and 8x8 and writes
//             levels 1..3 to the workspace; (2) one launch over the pixels of all levels, each CTA inside one
//             level: fp64 partial sums of |delta| and integer counts; (3) a one-CTA fixed-order finalize that
//             leaves the per-level counts in the workspace.
//   backward: one launch per level, coarsest first, gather form (no atomics): the Sobel adjoint of
//             sign(delta) mask / count on a tile with a two-pixel halo, plus the blur-pool adjoint of the
//             level below's total gradient.  Level 0 writes grad_pred.
//   ScaleInvariantLoss: fp64 partial sums of d and d^2 (d = gt - pred in fp32), a fixed-order finalize that
//             keeps the mean and the loss on the device, and one elementwise backward launch.
// No host synchronisation anywhere; bit-identical run to run.
//
// Limits (checked by the C ABI, SRCV_ERR_SHAPE): 1 <= num_scales <= 4; H, W >= 1 (odd sizes and levels one pixel
// wide are fine); 1 <= B <= 65535 (grid.z); B H W < 2^30 (32-bit element indices into the two pyramids);
// ScaleInvariantLoss 0 <= n < 2^31.
//
// Compiled as part of the multi-view loss unit (srcv_mvloss.cu) after srcv_normals.cuh, whose index and Sobel
// adjoint helpers it shares.
#pragma once
#include "srcv_normals.cuh"

namespace srcv {

namespace gradloss_detail {
namespace {

using normals_detail::clamp_idx;
using normals_detail::finite;
using normals_detail::sobel_adjoint_1d;

constexpr int kThreads = 256, kPerThread = 4;
constexpr int kT0 = 64;                                       // level-0 tile edge of the pyramid kernel
constexpr int kS0 = kT0 + 7, kS1 = kT0 / 2 + 3, kS2 = kT0 / 4 + 1, kS3 = kT0 / 8;   // staged edges per level
constexpr int kTW = 32, kTH = 8;                              // backward tile

struct Levels {
  int n;                          // num_scales
  int h[kMsGradMaxScales], w[kMsGradMaxScales];
  long long off[kMsGradMaxScales];   // element offset of level l >= 1 inside one tensor's pyramid
  long long per_tensor;           // elements of one pyramid (levels 1..n-1)
  unsigned cta0[kMsGradMaxScales + 1];   // first CTA of each level in the loss launch
};

inline Levels make_levels(int B, int H, int W, int n) {
  Levels L{};
  L.n = n;
  long long off = 0;
  unsigned cta = 0;
  for (int l = 0; l < kMsGradMaxScales; ++l) {
    L.h[l] = l == 0 ? H : (L.h[l - 1] + 1) / 2;
    L.w[l] = l == 0 ? W : (L.w[l - 1] + 1) / 2;
    L.off[l] = off;
    L.cta0[l] = cta;
    if (l < n) {
      const long long pix = (long long)B * L.h[l] * L.w[l];
      if (l > 0) off += pix;
      cta += (unsigned)((pix + kThreads * kPerThread - 1) / (kThreads * kPerThread));
    }
  }
  L.per_tensor = off;
  L.cta0[kMsGradMaxScales] = cta;
  return L;
}

// one blur-pool step in shared memory: dst (dn x dn, global origin d0y, d0x, map dh x dw) from src (row stride
// ss), whose local (2i, 2j) is the top-left tap of dst local (i, j).  Positions outside the map are zero: they
// are the next level's padding.
__device__ __forceinline__ void pool_step(const float* src, int ss, float* dst, int dn, int d0y, int d0x, int dh,
                                          int dw, int tid) {
  for (int i = tid; i < dn * dn; i += kThreads) {
    const int y = i / dn, x = i - y * dn, gy = d0y + y, gx = d0x + x;
    float v = 0.f;
    if (gy >= 0 && gy < dh && gx >= 0 && gx < dw) {
      const float* r0 = src + (2 * y) * ss + 2 * x;
      const float* r1 = r0 + ss;
      const float* r2 = r1 + ss;
      v = 0.0625f * ((r0[0] + 2.f * r0[1] + r0[2]) + 2.f * (r1[0] + 2.f * r1[1] + r1[2]) + (r2[0] + 2.f * r2[1] + r2[2]));
    }
    dst[i] = v;
  }
}

__device__ __forceinline__ void store_level(const float* s, int sn, int skip, int tn, int g0y, int g0x, int h, int w,
                                            float* out, int tid) {
  for (int i = tid; i < tn * tn; i += kThreads) {
    const int y = i / tn, x = i - y * tn, gy = g0y + y, gx = g0x + x;
    if (gy < h && gx < w) out[(size_t)gy * w + gx] = s[(y + skip) * sn + x + skip];
  }
}

// grid (2 ceil(W/64), ceil(H/64), B); blockIdx.x & 1 selects the tensor (0 = ground truth, 1 = prediction)
__global__ void __launch_bounds__(kThreads)
msgrad_pyramid_kernel(const float* __restrict__ gt, const float* __restrict__ pred, Levels L, float* __restrict__ pyr) {
  __shared__ float s0[kS0 * kS0], s1[kS1 * kS1], s2[kS2 * kS2], s3[kS3 * kS3];
  const int which = blockIdx.x & 1, tx = blockIdx.x >> 1, ty = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
  const int H = L.h[0], W = L.w[0];
  const float* in = (which ? pred : gt) + (size_t)b * H * W;
  const int y0 = kT0 * ty - 7, x0 = kT0 * tx - 7;
  for (int i = tid; i < kS0 * kS0; i += kThreads) {
    const int y = i / kS0, x = i - y * kS0, gy = y0 + y, gx = x0 + x;
    s0[i] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? __ldg(in + (size_t)gy * W + gx) : 0.f;
  }
  __syncthreads();
  float* out = pyr + (size_t)which * L.per_tensor;
  pool_step(s0, kS0, s1, kS1, kT0 / 2 * ty - 3, kT0 / 2 * tx - 3, L.h[1], L.w[1], tid);
  __syncthreads();
  store_level(s1, kS1, 3, kT0 / 2, kT0 / 2 * ty, kT0 / 2 * tx, L.h[1], L.w[1],
              out + L.off[1] + (size_t)b * L.h[1] * L.w[1], tid);
  if (L.n < 3) return;
  pool_step(s1, kS1, s2, kS2, kT0 / 4 * ty - 1, kT0 / 4 * tx - 1, L.h[2], L.w[2], tid);
  __syncthreads();
  store_level(s2, kS2, 1, kT0 / 4, kT0 / 4 * ty, kT0 / 4 * tx, L.h[2], L.w[2],
              out + L.off[2] + (size_t)b * L.h[2] * L.w[2], tid);
  if (L.n < 4) return;
  pool_step(s2, kS2, s3, kS3, kT0 / 8 * ty, kT0 / 8 * tx, L.h[3], L.w[3], tid);
  __syncthreads();
  store_level(s3, kS3, 0, kT0 / 8, kT0 / 8 * ty, kT0 / 8 * tx, L.h[3], L.w[3],
              out + L.off[3] + (size_t)b * L.h[3] * L.w[3], tid);
}

// (1/8) [[-1,0,1],[-2,0,2],[-1,0,1]] and its transpose, as cross-correlations
__device__ __forceinline__ void sobel(const float v[3][3], float& gx, float& gy) {
  gx = 0.125f * ((v[0][2] - v[0][0]) + 2.0f * (v[1][2] - v[1][0]) + (v[2][2] - v[2][0]));
  gy = 0.125f * ((v[2][0] - v[0][0]) + 2.0f * (v[2][1] - v[0][1]) + (v[2][2] - v[0][2]));
}

// grid L.cta0[4]: CTA c works inside the level l with cta0[l] <= c < cta0[l+1]; per-CTA fp64 sum of
// |dGx| + |dGy| over the masked pixels and the count of masked COMPONENTS (two per pixel)
__global__ void __launch_bounds__(kThreads)
msgrad_loss_kernel(const float* __restrict__ gt, const float* __restrict__ pred, int B, Levels L,
                   const float* __restrict__ pyr, double* __restrict__ psum, long long* __restrict__ pcnt) {
  __shared__ double s_sum[kThreads];
  __shared__ long long s_cnt[kThreads];
  int l = 0, h = L.h[0], w = L.w[0];
  long long off = 0;
  unsigned cta0 = 0;
#pragma unroll   // constant indices: the by-value Levels stays in the parameter space
  for (int k = 1; k < kMsGradMaxScales; ++k)
    if (k < L.n && blockIdx.x >= L.cta0[k]) { l = k; h = L.h[k]; w = L.w[k]; off = L.off[k]; cta0 = L.cta0[k]; }
  const float* G = l ? pyr + off : gt;
  const float* P = l ? pyr + L.per_tensor + off : pred;
  const long long n_pix = (long long)B * h * w;
  double sum = 0.0;
  long long cnt = 0;
  for (int j = 0; j < kPerThread; ++j) {
    const long long i = ((long long)(blockIdx.x - cta0) * kPerThread + j) * kThreads + threadIdx.x;
    if (i >= n_pix) break;
    const int x = (int)(i % w), y = (int)((i / w) % h);
    const size_t base = (size_t)(i / ((long long)h * w)) * h * w;
    float g[3][3], p[3][3];
    bool ok = true;
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        const size_t at = base + (size_t)clamp_idx(y + dy - 1, h) * w + clamp_idx(x + dx - 1, w);
        g[dy][dx] = __ldg(G + at);
        p[dy][dx] = __ldg(P + at);
        ok = ok && finite(g[dy][dx]);
      }
    if (ok) {
      float ggx, ggy, pgx, pgy;
      sobel(g, ggx, ggy);
      sobel(p, pgx, pgy);
      sum += (double)fabsf(pgx - ggx) + (double)fabsf(pgy - ggy);
      cnt += 2;
    }
  }
  s_sum[threadIdx.x] = sum;
  s_cnt[threadIdx.x] = cnt;
  block_tree<kThreads>([&](int t, int u) {
    s_sum[t] += s_sum[u];
    s_cnt[t] += s_cnt[u];
  });
  if (threadIdx.x == 0) {
    psum[blockIdx.x] = s_sum[0];
    pcnt[blockIdx.x] = s_cnt[0];
  }
}

// one CTA: loss = sum_l sum_l / count_l (NaN when a level has no masked component); counts[4] stay in the
// workspace for the backward (0 for the levels past num_scales)
__global__ void __launch_bounds__(kThreads)
msgrad_finalize_kernel(const double* __restrict__ psum, const long long* __restrict__ pcnt, Levels L,
                       float* __restrict__ loss, long long* __restrict__ counts) {
  __shared__ double s_sum[kThreads];
  __shared__ long long s_cnt[kThreads];
  double total = 0.0;
  for (int l = 0; l < kMsGradMaxScales; ++l) {
    if (l >= L.n) {
      if (threadIdx.x == 0) counts[l] = 0;
      continue;
    }
    reduce_partials<kThreads>(psum, pcnt, L.cta0[l], L.cta0[l + 1], s_sum, s_cnt);
    total += s_sum[0] / (double)s_cnt[0];
    if (threadIdx.x == 0) counts[l] = s_cnt[0];
  }
  if (threadIdx.x == 0) *loss = (float)total;
}

// grid (ceil(w/32), ceil(h/8), B) at level l: out(q) = g_loss / count_l / 8 * SobelT(sign(delta) mask)(q)
//                                                     + BlurPoolT(below)(q), below = the total gradient of level l+1
__global__ void __launch_bounds__(kThreads)
msgrad_backward_kernel(const float* __restrict__ G, const float* __restrict__ P, int h, int w,
                       const long long* __restrict__ count, const float* __restrict__ grad_loss,
                       const float* __restrict__ below, int bh, int bw, float* __restrict__ out) {
  __shared__ float s_g[kTH + 4][kTW + 4], s_p[kTH + 4][kTW + 4];   // clamped coordinates, two-pixel halo
  __shared__ float s_sx[kTH + 2][kTW + 2], s_sy[kTH + 2][kTW + 2]; // sign(delta) mask on the one-pixel ring
  const int b = blockIdx.z, tid = threadIdx.x, x0 = blockIdx.x * kTW, y0 = blockIdx.y * kTH;
  const size_t base = (size_t)b * h * w;
  for (int i = tid; i < (kTH + 4) * (kTW + 4); i += kThreads) {
    const int ty = i / (kTW + 4), tx = i - ty * (kTW + 4);
    const size_t at = base + (size_t)clamp_idx(y0 - 2 + ty, h) * w + clamp_idx(x0 - 2 + tx, w);
    s_g[ty][tx] = __ldg(G + at);
    s_p[ty][tx] = __ldg(P + at);
  }
  __syncthreads();
  for (int i = tid; i < (kTH + 2) * (kTW + 2); i += kThreads) {
    const int ry = i / (kTW + 2), rx = i - ry * (kTW + 2), py = y0 - 1 + ry, px = x0 - 1 + rx;
    float sx = 0.f, sy = 0.f;
    if (py >= 0 && py < h && px >= 0 && px < w) {
      float g[3][3], p[3][3];
      bool ok = true;
#pragma unroll
      for (int dy = 0; dy < 3; ++dy)
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
          g[dy][dx] = s_g[ry + dy][rx + dx];
          p[dy][dx] = s_p[ry + dy][rx + dx];
          ok = ok && finite(g[dy][dx]);
        }
      if (ok) {
        float ggx, ggy, pgx, pgy;
        sobel(g, ggx, ggy);
        sobel(p, pgx, pgy);
        const float dx = pgx - ggx, dy = pgy - ggy;
        sx = (float)((dx > 0.f) - (dx < 0.f));
        sy = (float)((dy > 0.f) - (dy < 0.f));
      }
    }
    s_sx[ry][rx] = sx;
    s_sy[ry][rx] = sy;
  }
  __syncthreads();
  const int ty = tid / kTW, tx = tid - ty * kTW, y = y0 + ty, x = x0 + tx;
  if (y >= h || x >= w) return;
  float wsy[3], wdy[3], wsx[3], wdx[3];
  sobel_adjoint_1d(y, h, wsy, wdy);
  sobel_adjoint_1d(x, w, wsx, wdx);
  float acc = 0.f;   // small integers: exact
#pragma unroll
  for (int oy = 0; oy < 3; ++oy)
#pragma unroll
    for (int ox = 0; ox < 3; ++ox)
      acc += wsy[oy] * wdx[ox] * s_sx[ty + oy][tx + ox] + wdy[oy] * wsx[ox] * s_sy[ty + oy][tx + ox];
  const long long n = *count;
  float v = n > 0 ? acc * (0.125f * __fdiv_rn(__ldg(grad_loss), (float)n)) : 0.f;
  if (below) {
    // the level-(l+1) outputs Y with a tap on row y: 2Y + d = y, d in {-1, 0, 1}, weights [1,2,1] / 4
    const int ny = (y & 1) ? 2 : 1, nx = (x & 1) ? 2 : 1;
    const float* bl = below + (size_t)b * bh * bw;
    float up = 0.f;
    for (int iy = 0; iy < ny; ++iy) {
      const int Y = (y >> 1) + iy;
      if (Y >= bh) continue;
      for (int ix = 0; ix < nx; ++ix) {
        const int X = (x >> 1) + ix;
        if (X >= bw) continue;
        up += ((y & 1) ? 1.f : 2.f) * ((x & 1) ? 1.f : 2.f) * __ldg(bl + (size_t)Y * bw + X);
      }
    }
    v = fmaf(0.0625f, up, v);
  }
  out[base + (size_t)y * w + x] = v;
}

// ---- ScaleInvariantLoss ---------------------------------------------------------------------
struct SiStats {
  double mean, loss;   // mean(d), sqrt(mean(d^2) - lambda mean(d)^2)
  long long n;
};

__global__ void __launch_bounds__(kThreads)
si_loss_kernel(const float* __restrict__ gt, const float* __restrict__ pred, long long n, double* __restrict__ psum,
               double* __restrict__ psq) {
  __shared__ double s_a[kThreads], s_b[kThreads];
  double a = 0.0, q = 0.0;
  for (int j = 0; j < kPerThread; ++j) {
    const long long i = ((long long)blockIdx.x * kPerThread + j) * kThreads + threadIdx.x;
    if (i >= n) break;
    const double d = (double)(__ldg(gt + i) - __ldg(pred + i));
    a += d;
    q += d * d;
  }
  s_a[threadIdx.x] = a;
  s_b[threadIdx.x] = q;
  block_tree<kThreads>([&](int t, int u) {
    s_a[t] += s_a[u];
    s_b[t] += s_b[u];
  });
  if (threadIdx.x == 0) {
    psum[blockIdx.x] = s_a[0];
    psq[blockIdx.x] = s_b[0];
  }
}

// one CTA; n == 0 gives 0 / 0 = NaN and a negative radicand gives NaN, as torch.sqrt does
__global__ void __launch_bounds__(kThreads)
si_loss_finalize_kernel(const double* __restrict__ psum, const double* __restrict__ psq, unsigned n_partials,
                        long long n, double lambda, float* __restrict__ loss, SiStats* __restrict__ stats) {
  __shared__ double s_sum[kThreads];
  __shared__ long long s_unused[kThreads];
  reduce_partials<kThreads>(psum, nullptr, 0, n_partials, s_sum, s_unused);
  const double sum = s_sum[0];
  reduce_partials<kThreads>(psq, nullptr, 0, n_partials, s_sum, s_unused);
  if (threadIdx.x == 0) {
    const double mean = sum / (double)n, r = sqrt(s_sum[0] / (double)n - lambda * mean * mean);
    *loss = (float)r;
    *stats = SiStats{mean, r, n};
  }
}

// d loss / d d_i = (d_i - lambda mean) / (n loss);  grad_gt = + that, grad_pred = - that (either may be null)
__global__ void __launch_bounds__(kThreads)
si_loss_backward_kernel(const float* __restrict__ gt, const float* __restrict__ pred, long long n, double lambda,
                        const SiStats* __restrict__ stats, const float* __restrict__ grad_loss,
                        float* __restrict__ grad_gt, float* __restrict__ grad_pred) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const double d = (double)(__ldg(gt + i) - __ldg(pred + i));
  const float g = (float)((double)__ldg(grad_loss) * (d - lambda * stats->mean) / ((double)n * stats->loss));
  if (grad_gt) grad_gt[i] = g;
  if (grad_pred) grad_pred[i] = -g;
}

inline unsigned si_partials(long long n) {
  const long long per = kThreads * kPerThread;
  return n > 0 ? (unsigned)((n + per - 1) / per) : 1u;
}

}  // namespace
}  // namespace gradloss_detail

namespace gd = gradloss_detail;

// workspace: [counts: 4 x int64, padded to 256 B | partial sums: double per loss CTA | partial counts: int64 per
// loss CTA | ground-truth pyramid, levels 1..n-1, each (B,h_l,w_l) fp32 | prediction pyramid | gradient pyramid
// (backward scratch)]
size_t msgrad_workspace_bytes(int B, int H, int W, int num_scales) {
  const gd::Levels L = gd::make_levels(B, H, W, num_scales);
  return 256 + align256((size_t)L.cta0[kMsGradMaxScales] * (sizeof(double) + sizeof(long long))) +
         align256(3 * (size_t)L.per_tensor * sizeof(float));
}

namespace gradloss_detail {
namespace {
struct MsGradWorkspace {
  long long* counts;
  double* psum;
  long long* pcnt;
  float *pyr, *grad;   // pyr = ground truth then prediction
};
inline MsGradWorkspace carve(const Levels& L, void* workspace) {
  MsGradWorkspace ws;
  uint8_t* p = reinterpret_cast<uint8_t*>(workspace);
  ws.counts = reinterpret_cast<long long*>(p);
  ws.psum = reinterpret_cast<double*>(p + 256);
  ws.pcnt = reinterpret_cast<long long*>(ws.psum + L.cta0[kMsGradMaxScales]);
  ws.pyr = reinterpret_cast<float*>(p + 256 + align256((size_t)L.cta0[kMsGradMaxScales] * (sizeof(double) + sizeof(long long))));
  ws.grad = ws.pyr + 2 * L.per_tensor;
  return ws;
}
}  // namespace
}  // namespace gradloss_detail

cudaError_t launch_msgrad_forward(const float* gt, const float* pred, int B, int H, int W, int num_scales, float* loss,
                                  void* workspace, cudaStream_t stream) {
  const gd::Levels L = gd::make_levels(B, H, W, num_scales);
  const gd::MsGradWorkspace ws = gd::carve(L, workspace);
  if (num_scales > 1) {
    const dim3 grid(2u * (unsigned)((W + gd::kT0 - 1) / gd::kT0), (unsigned)((H + gd::kT0 - 1) / gd::kT0), (unsigned)B);
    SRCV_LAUNCH(gd::msgrad_pyramid_kernel, grid, gd::kThreads, 0, stream, gt, pred, L, ws.pyr);
    note_launch();
  }
  SRCV_LAUNCH(gd::msgrad_loss_kernel, L.cta0[kMsGradMaxScales], gd::kThreads, 0, stream, gt, pred, B, L,
              (const float*)ws.pyr, ws.psum, ws.pcnt);
  note_launch();
  SRCV_LAUNCH(gd::msgrad_finalize_kernel, 1, gd::kThreads, 0, stream, (const double*)ws.psum,
              (const long long*)ws.pcnt, L, loss, ws.counts);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_msgrad_backward(const float* gt, const float* pred, int B, int H, int W, int num_scales,
                                   const float* grad_loss, float* grad_pred, void* workspace, cudaStream_t stream) {
  const gd::Levels L = gd::make_levels(B, H, W, num_scales);
  const gd::MsGradWorkspace ws = gd::carve(L, workspace);
  for (int l = num_scales - 1; l >= 0; --l) {
    const float* G = l ? ws.pyr + L.off[l] : gt;
    const float* P = l ? ws.pyr + L.per_tensor + L.off[l] : pred;
    const float* below = l + 1 < num_scales ? ws.grad + L.off[l + 1] : nullptr;
    const dim3 grid((unsigned)((L.w[l] + gd::kTW - 1) / gd::kTW), (unsigned)((L.h[l] + gd::kTH - 1) / gd::kTH), (unsigned)B);
    SRCV_LAUNCH(gd::msgrad_backward_kernel, grid, gd::kThreads, 0, stream, G, P, L.h[l], L.w[l],
                (const long long*)(ws.counts + l), grad_loss, below, l + 1 < num_scales ? L.h[l + 1] : 0,
                l + 1 < num_scales ? L.w[l + 1] : 0, l ? ws.grad + L.off[l] : grad_pred);
    note_launch();
  }
  return cudaGetLastError();
}

// workspace: [mean: double, loss: double, n: int64, padded to 256 B | partial sums of d | partial sums of d^2]
size_t si_loss_workspace_bytes(long long n) {
  return 256 + align256((size_t)gd::si_partials(n) * 2 * sizeof(double));
}

cudaError_t launch_si_loss_forward(const float* gt, const float* pred, long long n, double lambda, float* loss,
                                   void* workspace, cudaStream_t stream) {
  const unsigned nb = gd::si_partials(n);
  gd::SiStats* stats = reinterpret_cast<gd::SiStats*>(workspace);
  double* psum = reinterpret_cast<double*>(reinterpret_cast<uint8_t*>(workspace) + 256);
  double* psq = psum + nb;
  SRCV_LAUNCH(gd::si_loss_kernel, nb, gd::kThreads, 0, stream, gt, pred, n, psum, psq);
  note_launch();
  SRCV_LAUNCH(gd::si_loss_finalize_kernel, 1, gd::kThreads, 0, stream, (const double*)psum, (const double*)psq, nb, n,
              lambda, loss, stats);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_si_loss_backward(const float* gt, const float* pred, long long n, double lambda,
                                    const float* grad_loss, float* grad_gt, float* grad_pred, const void* workspace,
                                    cudaStream_t stream) {
  if (n == 0) return cudaSuccess;
  const unsigned blocks = (unsigned)((n + gd::kThreads - 1) / gd::kThreads);
  SRCV_LAUNCH(gd::si_loss_backward_kernel, blocks, gd::kThreads, 0, stream, gt, pred, n, lambda,
              reinterpret_cast<const gd::SiStats*>(workspace), grad_loss, grad_gt, grad_pred);
  note_launch();
  return cudaGetLastError();
}

}  // namespace srcv
