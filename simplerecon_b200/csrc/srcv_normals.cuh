// Surface normals from depth and the normals loss — NormalGenerator (utils/geometry_utils.py:92-133)
// and NormalsLoss (losses.py:57-77) of the reference; a training step calls the first twice
// (experiment_modules/depth_model.py:526, :530) and feeds both results to the second (:475, Equation 4
// of the paper).  DESIGN §4.13.
//
//   S = gaussian_blur2d(depth, k, sigma)   separable, x pass then y pass, reflect padding
//   P(p) = S(p) invK3 (x + .5, y + .5, 1)   the back-projected point
//   Gx, Gy = Sobel(P) / 8                   replicate padding: a tap outside the map reads P of the
//                                           clamped pixel (its smoothed depth AND its ray)
//   n = c / max(|c|, 1e-12),  c = Gx x Gy
// A normal depends on the 7x7 (k = 5) window of depths under the reflect and clamp index maps; the
// reference multiplies every tap, zero weights included, so one non-finite depth in that window
// makes the normal non-finite: here all three components are written as NaN.
//
//   forward : one launch.  A 32x8 tile stages its depths with a radius k/2 + 1 halo through the
//             reflect map, runs the x and y passes in shared memory on the tile plus its clamped
//             one-pixel ring, forms P there, then Sobel, cross and normalise per pixel.
//   backward: two launches, gather form (no atomics, bit-identical run to run).  (a) is the forward
//             tile again, which turns g_n into g_Gx = Gy x g_c and g_Gy = g_c x Gx (24 B/pixel of
//             workspace); (b) forms g_S = ray . (Sobel adjoint of g_G) on a tile plus a radius k/2
//             halo, then the adjoints of the y and x passes, each a gather over the source pixels a
//             reflected tap maps onto the output.
//   loss    : per-CTA fp64 partial sums and integer counts, a fixed-order finalize; the backward is
//             one elementwise launch that reads the count the forward left in the workspace.
//
// Compiled as part of the multi-view loss unit (srcv_mvloss.cu, which includes this header last), with the
// depth metrics: the consumers of the predicted depth that a training step runs share one translation
// unit.  The internals live in their own namespace.
#pragma once
#include "srcv_kernels.h"

namespace srcv {

namespace normals_detail {
namespace {

constexpr int kTW = 32, kTH = 8, kThreads = kTW * kTH;
constexpr int kMaxR = kNormalsMaxKernel / 2;
constexpr int kDH = kTH + 2 * kMaxR + 2, kDW = kTW + 2 * kMaxR + 2;   // depth tile with a radius R + 1 halo
constexpr int kRH = kTH + 2, kRW = kTW + 2;                           // the tile and its one-pixel ring
constexpr int kSH = kTH + 2 * kMaxR, kSW = kTW + 2 * kMaxR;           // g_S with a radius R halo
constexpr float kNormEps = 1e-12f;                                    // F.normalize

__device__ __forceinline__ int clamp_idx(int i, int n) { return i < 0 ? 0 : (i > n - 1 ? n - 1 : i); }
// PyTorch's 'reflect' (the edge pixel is not repeated), valid for -n < i < 2n - 1
__device__ __forceinline__ int reflect_idx(int i, int n) { return i < 0 ? -i : (i > n - 1 ? 2 * (n - 1) - i : i); }
__device__ __forceinline__ bool finite(float v) { return fabsf(v) <= 3.402823466e38f; }

// the ray invK3 (x + .5, y + .5, 1) of a pixel (BackprojectDepth, geometry_utils.py:56)
__device__ __forceinline__ void pixel_ray(const float* ik, int px, int py, float r[3]) {
  const float x = (float)px + 0.5f, y = (float)py + 0.5f;
#pragma unroll
  for (int c = 0; c < 3; ++c) r[c] = __fmaf_rn(ik[3 * c + 2], 1.0f, __fmaf_rn(ik[3 * c + 1], y, __fmul_rn(ik[3 * c], x)));
}

__device__ __forceinline__ void cross3(const float a[3], const float b[3], float o[3]) {
  o[0] = __fadd_rn(__fmul_rn(a[1], b[2]), -__fmul_rn(a[2], b[1]));
  o[1] = __fadd_rn(__fmul_rn(a[2], b[0]), -__fmul_rn(a[0], b[2]));
  o[2] = __fadd_rn(__fmul_rn(a[0], b[1]), -__fmul_rn(a[1], b[0]));
}

// grid (ceil(W/32), ceil(H/8), B).  FORWARD: out = normals (B,3,H,W).  BACKWARD: reads grad_n (B,3,H,W),
// out = (B,6,H,W) = g_Gx, g_Gy (zero where the window holds a non-finite depth, so that a hole in the
// ground truth does not spread NaN into the gradient of its neighbours).
template <bool BACKWARD>
__global__ void __launch_bounds__(kThreads)
normals_tile_kernel(srcv_normals_args a, const float* __restrict__ grad_n, float* __restrict__ out) {
  __shared__ float s_d[kDH][kDW];        // depth, rows y0-1-R.., columns x0-1-R.. through the reflect map
  __shared__ float s_x[kDH][kRW];        // x pass at the ring columns (clamped pixels)
  __shared__ float s_p[3][kRH][kRW];     // P on the tile and its clamped ring
  __shared__ float s_tap[kNormalsMaxKernel];
  __shared__ float s_ik[9];
  const int H = a.H, W = a.W, K = a.k, R = a.k >> 1, b = blockIdx.z, tid = threadIdx.x;
  const int x0 = blockIdx.x * kTW, y0 = blockIdx.y * kTH;
  const int DH = kTH + 2 * R + 2, DW = kTW + 2 * R + 2;
  if (tid < K) s_tap[tid] = __ldg(a.taps + tid);
  if (tid < 9) s_ik[tid] = __ldg(a.invK + (size_t)b * 16 + (tid / 3) * 4 + tid % 3);
  const float* dep = a.depth + (size_t)b * H * W;
  // rows / columns the passes never read (beyond the reflect range) are clamped only to stay in bounds
  for (int i = tid; i < DH * DW; i += kThreads) {
    const int ty = i / DW, tx = i - ty * DW;
    const int gy = clamp_idx(reflect_idx(y0 - 1 - R + ty, H), H), gx = clamp_idx(reflect_idx(x0 - 1 - R + tx, W), W);
    s_d[ty][tx] = __ldg(dep + (size_t)gy * W + gx);
  }
  __syncthreads();
  // x pass for ring column j: the clamped pixel cx = clamp(x0 - 1 + j) reads s_d columns cx - x0 + 1 + t
  for (int i = tid; i < DH * kRW; i += kThreads) {
    const int ty = i / kRW, j = i - ty * kRW;
    const float* row = &s_d[ty][clamp_idx(x0 - 1 + j, W) - x0 + 1];
    float acc = 0.f;
    for (int t = 0; t < K; ++t) acc = fmaf(s_tap[t], row[t], acc);
    s_x[ty][j] = acc;
  }
  __syncthreads();
  // y pass and back-projection on the ring
  for (int i = tid; i < kRH * kRW; i += kThreads) {
    const int ry = i / kRW, j = i - ry * kRW;
    const int cy = clamp_idx(y0 - 1 + ry, H), cx = clamp_idx(x0 - 1 + j, W);
    const int r0 = cy - y0 + 1;
    float s = 0.f;
    for (int t = 0; t < K; ++t) s = fmaf(s_tap[t], s_x[r0 + t][j], s);
    float ray[3];
    pixel_ray(s_ik, cx, cy, ray);
#pragma unroll
    for (int c = 0; c < 3; ++c) s_p[c][ry][j] = __fmul_rn(s, ray[c]);
  }
  __syncthreads();
  const int ty = tid / kTW, tx = tid - ty * kTW, y = y0 + ty, x = x0 + tx;
  if (y >= H || x >= W) return;
  float gx[3], gy[3];
  bool ok = true;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v[3][3];
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        v[dy][dx] = s_p[c][ty + dy][tx + dx];
        ok = ok && finite(v[dy][dx]);
      }
    // (1/8) [[-1,0,1],[-2,0,2],[-1,0,1]] and its transpose, as cross-correlations
    gx[c] = 0.125f * ((v[0][2] - v[0][0]) + 2.0f * (v[1][2] - v[1][0]) + (v[2][2] - v[2][0]));
    gy[c] = 0.125f * ((v[2][0] - v[0][0]) + 2.0f * (v[2][1] - v[0][1]) + (v[2][2] - v[0][2]));
  }
  float cr[3];
  cross3(gx, gy, cr);
  const float nrm = sqrtf(fmaf(cr[2], cr[2], fmaf(cr[1], cr[1], cr[0] * cr[0])));
  const size_t HW = (size_t)H * W, pix = (size_t)y * W + x;
  if (!BACKWARD) {
    const float den = fmaxf(nrm, kNormEps), nan = __uint_as_float(0x7fc00000u);
#pragma unroll
    for (int c = 0; c < 3; ++c) out[((size_t)b * 3 + c) * HW + pix] = ok ? __fdiv_rn(cr[c], den) : nan;
  } else {
    float gn[3], gc[3], ggx[3], ggy[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) gn[c] = __ldg(grad_n + ((size_t)b * 3 + c) * HW + pix);
    if (nrm > kNormEps) {   // d(c/|c|) = g/|c| - c (c.g)/|c|^3 = (g - n (n.g)) / |c|
      const float inv = __fdiv_rn(1.0f, nrm);
      float n[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) n[c] = cr[c] * inv;
      const float ng = fmaf(n[2], gn[2], fmaf(n[1], gn[1], n[0] * gn[0]));
#pragma unroll
      for (int c = 0; c < 3; ++c) gc[c] = fmaf(-n[c], ng, gn[c]) * inv;
    } else {                // clamp_min passes no gradient to the norm
#pragma unroll
      for (int c = 0; c < 3; ++c) gc[c] = __fdiv_rn(gn[c], kNormEps);
    }
    cross3(gy, gc, ggx);
    cross3(gc, gx, ggy);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      out[((size_t)b * 6 + c) * HW + pix] = ok ? ggx[c] : 0.f;
      out[((size_t)b * 6 + 3 + c) * HW + pix] = ok ? ggy[c] : 0.f;
    }
  }
}

// Sobel adjoint weights along one dimension for output q: for the three sources p = q - 1, q, q + 1,
// the sums of the smoothing [1,2,1] and difference [-1,0,1] taps t with clamp(p + t) == q
// (replicate padding: the edge pixel collects the taps that clamped onto it).
__device__ __forceinline__ void sobel_adjoint_1d(int q, int n, float ws[3], float wd[3]) {
#pragma unroll
  for (int o = 0; o < 3; ++o) {
    const int p = q + o - 1;
    float s = 0.f, d = 0.f;
    if (p >= 0 && p < n) {
#pragma unroll
      for (int t = -1; t <= 1; ++t)
        if (clamp_idx(p + t, n) == q) { s += (t == 0 ? 2.f : 1.f); d += (float)t; }
    }
    ws[o] = s;
    wd[o] = d;
  }
}

// the adjoint of one reflect-padded blur pass at output q along a dimension of size n:
//   sum_t tap[t] g(src) over the sources src whose tap t lands on q: src + t - R == q directly, or
//   through the reflection at either border.  `g(i)` reads source i (always within q +- R).
template <class G>
__device__ __forceinline__ float blur_adjoint_1d(const float* tap, int K, int q, int n, G g) {
  const int R = K >> 1;
  float acc = 0.f;
  for (int t = 0; t < K; ++t) {
    const int d = t - R;
    float v = 0.f;
    const int direct = q - d, left = -q - d, right = 2 * (n - 1) - q - d;
    if (direct >= 0 && direct < n) v = g(direct);
    if (q > 0 && left >= 0 && left < n) v += g(left);
    if (q < n - 1 && right >= 0 && right < n) v += g(right);
    acc = fmaf(tap[t], v, acc);
  }
  return acc;
}

// grid (ceil(W/32), ceil(H/8), B): grad_depth from g_Gx, g_Gy (B,6,H,W)
__global__ void __launch_bounds__(kThreads)
normals_depth_grad_kernel(srcv_normals_args a, const float* __restrict__ gG, float* __restrict__ grad_depth) {
  __shared__ float s_g[6][kDH][kDW];     // g_Gx, g_Gy on the tile with a radius R + 1 halo, 0 outside the map
  __shared__ float s_s[kSH][kSW];        // g_S on the tile with a radius R halo, 0 outside the map
  __shared__ float s_y[kTH][kSW];        // after the adjoint of the y pass
  __shared__ float s_tap[kNormalsMaxKernel];
  __shared__ float s_ik[9];
  const int H = a.H, W = a.W, K = a.k, R = a.k >> 1, b = blockIdx.z, tid = threadIdx.x;
  const int x0 = blockIdx.x * kTW, y0 = blockIdx.y * kTH;
  const int GH = kTH + 2 * R + 2, GW = kTW + 2 * R + 2, SH = kTH + 2 * R, SW = kTW + 2 * R;
  const size_t HW = (size_t)H * W;
  if (tid < K) s_tap[tid] = __ldg(a.taps + tid);
  if (tid < 9) s_ik[tid] = __ldg(a.invK + (size_t)b * 16 + (tid / 3) * 4 + tid % 3);
  for (int i = tid; i < 6 * GH * GW; i += kThreads) {
    const int c = i / (GH * GW), rem = i - c * GH * GW, ty = rem / GW, tx = rem - ty * GW;
    const int gy = y0 - 1 - R + ty, gx = x0 - 1 - R + tx;
    s_g[c][ty][tx] = (gy >= 0 && gy < H && gx >= 0 && gx < W) ? __ldg(gG + ((size_t)b * 6 + c) * HW + (size_t)gy * W + gx) : 0.f;
  }
  __syncthreads();
  // g_S(q) = ray(q) . g_P(q),  g_P = (1/8) sum_p (s_y d_x) g_Gx(p) + (d_y s_x) g_Gy(p)
  for (int i = tid; i < SH * SW; i += kThreads) {
    const int sy = i / SW, sx = i - sy * SW, qy = y0 - R + sy, qx = x0 - R + sx;
    float v = 0.f;
    if (qy >= 0 && qy < H && qx >= 0 && qx < W) {
      float wsy[3], wdy[3], wsx[3], wdx[3];
      sobel_adjoint_1d(qy, H, wsy, wdy);
      sobel_adjoint_1d(qx, W, wsx, wdx);
      float gp[3] = {0.f, 0.f, 0.f};
#pragma unroll
      for (int oy = 0; oy < 3; ++oy)
#pragma unroll
        for (int ox = 0; ox < 3; ++ox) {
          const float wx = wsy[oy] * wdx[ox], wy = wdy[oy] * wsx[ox];   // small integers: exact
#pragma unroll
          for (int c = 0; c < 3; ++c)
            gp[c] = fmaf(wx, s_g[c][sy + oy][sx + ox], fmaf(wy, s_g[3 + c][sy + oy][sx + ox], gp[c]));
        }
      float ray[3];
      pixel_ray(s_ik, qx, qy, ray);
      v = 0.125f * fmaf(ray[2], gp[2], fmaf(ray[1], gp[1], ray[0] * gp[0]));
    }
    s_s[sy][sx] = v;
  }
  __syncthreads();
  // adjoint of the y pass: output rows of the tile, every column of the halo
  for (int i = tid; i < kTH * SW; i += kThreads) {
    const int ty = i / SW, sx = i - ty * SW, y = y0 + ty;
    s_y[ty][sx] = y < H ? blur_adjoint_1d(s_tap, K, y, H, [&](int src) { return s_s[src - y0 + R][sx]; }) : 0.f;
  }
  __syncthreads();
  // adjoint of the x pass
  const int ty = tid / kTW, tx = tid - ty * kTW, y = y0 + ty, x = x0 + tx;
  if (y >= H || x >= W) return;
  grad_depth[(size_t)b * HW + (size_t)y * W + x] =
      blur_adjoint_1d(s_tap, K, x, W, [&](int src) { return s_y[ty][src - x0 + R]; });
}

// ---- NormalsLoss ----------------------------------------------------------------------------
constexpr int kLossThreads = 256, kLossPerThread = 4;

// mask = every component of both normals finite; term = 0.5 (1 - pred . gt) in fp32
__device__ __forceinline__ bool loss_pixel(const float* gt, const float* pred, size_t base, size_t HW, float g[3],
                                           float p[3]) {
  bool ok = true;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    g[c] = __ldg(gt + base + c * HW);
    p[c] = __ldg(pred + base + c * HW);
    ok = ok && finite(g[c]) && finite(p[c]);
  }
  return ok;
}

// grid ceil(B*H*W / (256*4)); partial sums (fp64) and counts per CTA
__global__ void __launch_bounds__(kLossThreads)
normals_loss_kernel(const float* __restrict__ gt, const float* __restrict__ pred, int HW, long long n_pix,
                    double* __restrict__ psum, long long* __restrict__ pcnt) {
  __shared__ double s_sum[kLossThreads];
  __shared__ long long s_cnt[kLossThreads];
  double sum = 0.0;
  long long cnt = 0;
  for (int j = 0; j < kLossPerThread; ++j) {
    const long long i = ((long long)blockIdx.x * kLossPerThread + j) * kLossThreads + threadIdx.x;
    if (i >= n_pix) break;
    const long long b = i / HW, p = i - b * HW;
    float g[3], q[3];
    if (loss_pixel(gt, pred, (size_t)b * 3 * HW + p, HW, g, q)) {
      const float dot = __fadd_rn(__fadd_rn(__fmul_rn(q[0], g[0]), __fmul_rn(q[1], g[1])), __fmul_rn(q[2], g[2]));
      sum += (double)__fmul_rn(0.5f, __fadd_rn(1.0f, -dot));
      ++cnt;
    }
  }
  s_sum[threadIdx.x] = sum;
  s_cnt[threadIdx.x] = cnt;
  block_tree<kLossThreads>([&](int t, int u) {
    s_sum[t] += s_sum[u];
    s_cnt[t] += s_cnt[u];
  });
  if (threadIdx.x == 0) {
    psum[blockIdx.x] = s_sum[0];
    pcnt[blockIdx.x] = s_cnt[0];
  }
}

// one CTA: the partials in a fixed order -> loss = sum / count (NaN without a masked pixel), count
__global__ void __launch_bounds__(kLossThreads)
normals_loss_finalize_kernel(const double* __restrict__ psum, const long long* __restrict__ pcnt, int n_partials,
                             float* __restrict__ loss, long long* __restrict__ count) {
  __shared__ double s_sum[kLossThreads];
  __shared__ long long s_cnt[kLossThreads];
  reduce_partials<kLossThreads>(psum, pcnt, 0, n_partials, s_sum, s_cnt);
  if (threadIdx.x == 0) {
    *loss = (float)(s_sum[0] / (double)s_cnt[0]);
    *count = s_cnt[0];
  }
}

// d loss / d pred_c = -0.5 gt_c (g / count) at masked pixels, 0 elsewhere (and to gt with pred_c)
__global__ void __launch_bounds__(kLossThreads)
normals_loss_backward_kernel(const float* __restrict__ gt, const float* __restrict__ pred, int HW, long long n_pix,
                             const long long* __restrict__ count, const float* __restrict__ grad_loss,
                             float* __restrict__ grad_pred, float* __restrict__ grad_gt) {
  const long long i = (long long)blockIdx.x * kLossThreads + threadIdx.x;
  if (i >= n_pix) return;
  const long long b = i / HW, p = i - b * HW;
  const size_t base = (size_t)b * 3 * HW + p;
  float g[3], q[3];
  const long long n = *count;
  const bool ok = loss_pixel(gt, pred, base, HW, g, q) && n > 0;
  const float scale = ok ? -0.5f * __fdiv_rn(__ldg(grad_loss), (float)n) : 0.f;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    grad_pred[base + c * HW] = ok ? __fmul_rn(g[c], scale) : 0.f;
    if (grad_gt) grad_gt[base + c * HW] = ok ? __fmul_rn(q[c], scale) : 0.f;
  }
}

inline dim3 tile_grid(const srcv_normals_args& a) {
  return dim3((unsigned)((a.W + kTW - 1) / kTW), (unsigned)((a.H + kTH - 1) / kTH), (unsigned)a.B);
}
inline long long loss_pixels(int B, int H, int W) { return (long long)B * H * W; }
inline unsigned loss_partials(long long n) {
  return (unsigned)((n + kLossThreads * kLossPerThread - 1) / (kLossThreads * kLossPerThread));
}

}  // namespace
}  // namespace normals_detail

namespace nd = normals_detail;

// workspace: g_Gx, g_Gy as (B,6,H,W) fp32
size_t normals_workspace_bytes(const srcv_normals_args& a) {
  return align256((size_t)a.B * 6 * a.H * a.W * sizeof(float));
}

cudaError_t launch_normals_forward(const srcv_normals_args& a, float* normals, cudaStream_t stream) {
  SRCV_LAUNCH((nd::normals_tile_kernel<false>), nd::tile_grid(a), nd::kThreads, 0, stream, a, (const float*)nullptr,
              normals);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_normals_backward(const srcv_normals_args& a, const float* grad_normals, float* grad_depth,
                                    void* workspace, cudaStream_t stream) {
  float* gG = reinterpret_cast<float*>(workspace);
  SRCV_LAUNCH((nd::normals_tile_kernel<true>), nd::tile_grid(a), nd::kThreads, 0, stream, a, grad_normals, gG);
  note_launch();
  SRCV_LAUNCH(nd::normals_depth_grad_kernel, nd::tile_grid(a), nd::kThreads, 0, stream, a, (const float*)gG,
              grad_depth);
  note_launch();
  return cudaGetLastError();
}

// workspace: [count int64 | loss copy, padded to 256 B | partial sums: double | partial counts: int64]
size_t normals_loss_workspace_bytes(int B, int H, int W) {
  const size_t n = nd::loss_partials(nd::loss_pixels(B, H, W));
  return 256 + align256(n * (sizeof(double) + sizeof(long long)));
}

cudaError_t launch_normals_loss_forward(const float* gt, const float* pred, int B, int H, int W, float* loss,
                                        void* workspace, cudaStream_t stream) {
  const long long n = nd::loss_pixels(B, H, W);
  const unsigned nb = nd::loss_partials(n);
  long long* count = reinterpret_cast<long long*>(workspace);
  double* psum = reinterpret_cast<double*>(reinterpret_cast<uint8_t*>(workspace) + 256);
  long long* pcnt = reinterpret_cast<long long*>(psum + nb);
  SRCV_LAUNCH(nd::normals_loss_kernel, nb, nd::kLossThreads, 0, stream, gt, pred, H * W, n, psum, pcnt);
  note_launch();
  SRCV_LAUNCH(nd::normals_loss_finalize_kernel, 1, nd::kLossThreads, 0, stream, (const double*)psum,
              (const long long*)pcnt, (int)nb, loss, count);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_normals_loss_backward(const float* gt, const float* pred, int B, int H, int W,
                                         const float* grad_loss, float* grad_pred, float* grad_gt,
                                         const void* workspace, cudaStream_t stream) {
  const long long n = nd::loss_pixels(B, H, W);
  const long long* count = reinterpret_cast<const long long*>(workspace);
  const unsigned blocks = (unsigned)((n + nd::kLossThreads - 1) / nd::kLossThreads);
  SRCV_LAUNCH(nd::normals_loss_backward_kernel, blocks, nd::kLossThreads, 0, stream, gt, pred, H * W, n, count,
              grad_loss, grad_pred, grad_gt);
  note_launch();
  return cudaGetLastError();
}

}  // namespace srcv
