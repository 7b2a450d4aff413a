// The regression terms of the training loss — DepthModel.compute_losses of the reference
// (experiment_modules/depth_model.py:447-474): the multi-scale log-L1 loss (Equation 2 of the paper, weight 1.0 in
// `loss`) and the logged abs, scale-invariant, inverse-abs and log-L1 terms.  DESIGN §4.15.
//
//   lg      = log(gt) per pixel; n = the pixels of mask_b over the whole batch (x[mask_b] flattens the batch)
//   ms      = sum over the present scales i of mean_{mask_b} |lg - lp_i(nearest(p))| / 2^i, lp_i at any h_i x w_i,
//             sampled with PyTorch's nearest rule (the source index of nearest_src_index, srcv_metrics.cuh)
//   abs     = mean_{mask_b} |gt - depth_pred|            log_l1 = mean_{mask_b} |lg - lp_0|
//   si      = sqrt(mean(d^2) - lambda mean(d)^2), d = lg - lp_0 over mask_b
//   inv_abs = mean |1/gt - 1/depth_pred| over mask_b and depth_pred > 0.1 (its own count m)
// An empty mask gives 0 / 0 = NaN, as the mean of an empty tensor does.
//
//   forward : (1) one pass over the ground-truth grid: per pixel the mask, lg, one nearest sample of each present
//             scale and every term; fp64 per-CTA partial sums and integer counts; (2) a one-CTA fixed-order finalize
//             that writes the five losses and keeps n, m, mean(d) and si in the workspace.
//   backward: one launch, gather form (no atomics), each CTA inside one scale.  At scale i >= 1 a thread owns one
//             coarse pixel and sums sign(lp_i - lg) mask over its preimage, a rectangle whose ends are found with the
//             forward index map itself (it is monotone); scale 0 adds the log_l1 and si terms; depth_pred gets the
//             abs and inv_abs terms.  An upstream gradient of zero (an output autograd did not reach) adds nothing.
// No host synchronisation anywhere; bit-identical run to run.
//
// Limits (checked by the C ABI, SRCV_ERR_SHAPE): 1 <= B <= 65535; B H W < 2^30 and B h_i w_i < 2^30 (32-bit
// element indices); every present scale at least 1 x 1; scale 0 is required and is H x W.
//
// Compiled as part of the multi-view loss unit (srcv_mvloss.cu) after srcv_metrics.cuh, whose nearest source index
// it shares.
#pragma once
#include "srcv_metrics.cuh"

namespace srcv {

namespace regloss_detail {
namespace {

constexpr int kThreads = 256, kPerThread = 4;

// the per-CTA partial sums, series-major (series k of CTA c at k * n_cta + c)
enum { kMs, kAbs, kL1, kD, kD2, kInv, kSums };
enum { kCntN, kCntM, kCounts };

struct Scales {
  const float* lp[kRegLossMaxScales];   // NULL = absent (scale 0 is always present)
  int h[kRegLossMaxScales], w[kRegLossMaxScales];
  float sy[kRegLossMaxScales], sx[kRegLossMaxScales];   // in / out in fp32, as PyTorch computes the scale
  unsigned cta0[kRegLossMaxScales + 1];  // first CTA of each scale in the backward launch
};

struct Stats {        // the workspace's head, kept for the backward
  long long n, m;
  double mean_d, si;
};

inline Scales make_scales(const srcv_regloss_args& a) {
  Scales S{};
  unsigned cta = 0;
  for (int i = 0; i < kRegLossMaxScales; ++i) {
    S.lp[i] = a.log_pred[i];
    S.cta0[i] = cta;
    if (!a.log_pred[i]) continue;
    S.h[i] = a.h[i];
    S.w[i] = a.w[i];
    S.sy[i] = (float)a.h[i] / (float)a.H;
    S.sx[i] = (float)a.w[i] / (float)a.W;
    cta += (unsigned)(((long long)a.B * a.h[i] * a.w[i] + kThreads - 1) / kThreads);
  }
  S.cta0[kRegLossMaxScales] = cta;
  return S;
}

inline unsigned forward_ctas(const srcv_regloss_args& a) {
  const long long per = kThreads * kPerThread;
  return (unsigned)(((long long)a.B * a.H * a.W + per - 1) / per);
}

__device__ __forceinline__ float sign_of(float x) { return (float)((x > 0.f) - (x < 0.f)); }   // torch.sign: 0 at 0, NaN

// grid forward_ctas: a thread takes kPerThread pixels of the flattened (B, H, W) grid
__global__ void __launch_bounds__(kThreads)
regloss_kernel(const float* __restrict__ gt, const uint8_t* __restrict__ mask, const float* __restrict__ dp, int B,
               int H, int W, Scales S, double* __restrict__ psum, long long* __restrict__ pcnt) {
  __shared__ double s_sum[kSums][kThreads];
  __shared__ long long s_cnt[kCounts][kThreads];
  const int total = B * H * W, t = threadIdx.x;
  double sum[kSums] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  int cn = 0, cm = 0;
  for (int j = 0; j < kPerThread; ++j) {
    const int i = ((int)blockIdx.x * kPerThread + j) * kThreads + t;
    if (i >= total) break;
    if (!__ldg(mask + i)) continue;
    const int x = i % W, y = (i / W) % H, b = i / (H * W);
    const float g = __ldg(gt + i), lg = logf(g), v = __ldg(dp + i);
    const float d = __fadd_rn(lg, -__ldg(S.lp[0] + i));
    double ms = (double)fabsf(d);
#pragma unroll
    for (int k = 1; k < kRegLossMaxScales; ++k) {
      if (!S.lp[k]) continue;
      const int iy = nearest_src_index(y, S.sy[k], S.h[k]), ix = nearest_src_index(x, S.sx[k], S.w[k]);
      const float e = __fadd_rn(lg, -__ldg(S.lp[k] + ((size_t)b * S.h[k] + iy) * S.w[k] + ix));
      ms += (double)fabsf(e) * (1.0 / (double)(1 << k));
    }
    sum[kMs] += ms;
    sum[kAbs] += (double)fabsf(__fadd_rn(g, -v));
    sum[kL1] += (double)fabsf(d);
    sum[kD] += (double)d;
    sum[kD2] += (double)d * (double)d;
    ++cn;
    if (v > 0.1f) {                       // depth_pred > 0.1 compares in fp32
      sum[kInv] += (double)fabsf(__fadd_rn(__fdiv_rn(1.0f, g), -__fdiv_rn(1.0f, v)));
      ++cm;
    }
  }
#pragma unroll
  for (int k = 0; k < kSums; ++k) s_sum[k][t] = sum[k];
  s_cnt[kCntN][t] = cn;
  s_cnt[kCntM][t] = cm;
  block_tree<kThreads>([&](int i, int j) {
#pragma unroll
    for (int k = 0; k < kSums; ++k) s_sum[k][i] += s_sum[k][j];
#pragma unroll
    for (int k = 0; k < kCounts; ++k) s_cnt[k][i] += s_cnt[k][j];
  });
  if (t < kSums) psum[(size_t)t * gridDim.x + blockIdx.x] = s_sum[t][0];
  if (t < kCounts) pcnt[(size_t)t * gridDim.x + blockIdx.x] = s_cnt[t][0];
}

// one CTA: losses = (ms, abs, si, inv_abs, log_l1); n, m, mean(d) and si stay in the workspace
__global__ void __launch_bounds__(kThreads)
regloss_finalize_kernel(const double* __restrict__ psum, const long long* __restrict__ pcnt, unsigned n_partials,
                        double lambda, float* __restrict__ losses, Stats* __restrict__ stats) {
  __shared__ double s_sum[kThreads];
  __shared__ long long s_cnt[kThreads];
  double total[kSums];
  long long cnt[kCounts] = {0, 0};
  for (int k = 0; k < kSums; ++k) {
    const bool with_count = k < kCounts;
    reduce_partials<kThreads>(psum + (size_t)k * n_partials, with_count ? pcnt + (size_t)k * n_partials : nullptr,
                              0, n_partials, s_sum, s_cnt);
    total[k] = s_sum[0];
    if (with_count) cnt[k] = s_cnt[0];
  }
  if (threadIdx.x != 0) return;
  const double n = (double)cnt[kCntN], m = (double)cnt[kCntM];
  const double mean = total[kD] / n, si = sqrt(total[kD2] / n - lambda * mean * mean);
  losses[0] = (float)(total[kMs] / n);
  losses[1] = (float)(total[kAbs] / n);
  losses[2] = (float)si;
  losses[3] = (float)(total[kInv] / m);
  losses[4] = (float)(total[kL1] / n);
  *stats = Stats{cnt[kCntN], cnt[kCntM], mean, si};
}

// the first destination index whose nearest source index is >= c (n_out if none): the preimage of source row c is
// [first_dst(c), first_dst(c + 1)).  The forward map itself is searched, so the ends agree with the forward.
__device__ __forceinline__ int first_dst(int c, int n_out, float scale, int n_in) {
  int lo = 0, hi = n_out;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (nearest_src_index(mid, scale, n_in) >= c) hi = mid;
    else lo = mid + 1;
  }
  return lo;
}

struct Grads {
  const float* up[5];                      // upstream gradients of (ms, abs, si, inv_abs, log_l1); NULL = zero
  float* lp[kRegLossMaxScales];            // NULL = not wanted
  float* dp;
};

__device__ __forceinline__ float upstream(const float* g) { return g ? __ldg(g) : 0.f; }

// grid S.cta0[4]: CTA c works inside the scale k with cta0[k] <= c < cta0[k+1], one (coarse) pixel per thread
__global__ void __launch_bounds__(kThreads)
regloss_backward_kernel(const float* __restrict__ gt, const uint8_t* __restrict__ mask, const float* __restrict__ dp,
                        int B, int H, int W, Scales S, double lambda, const Stats* __restrict__ stats, Grads G) {
  int h = H, w = W;
  unsigned cta0 = 0;
  const float* lp = S.lp[0];
  float* out = G.lp[0];
  float sy = 1.f, sx = 1.f, inv_pow = 1.f;   // inv_pow = 1 / 2^k
#pragma unroll   // constant indices: the by-value Scales and Grads stay in the parameter space
  for (int s = 1; s < kRegLossMaxScales; ++s)
    if (S.lp[s] && blockIdx.x >= S.cta0[s]) {
      h = S.h[s]; w = S.w[s]; cta0 = S.cta0[s]; lp = S.lp[s]; out = G.lp[s]; sy = S.sy[s]; sx = S.sx[s];
      inv_pow = 1.0f / (float)(1 << s);
    }
  const int i = (int)(blockIdx.x - cta0) * kThreads + threadIdx.x;
  if (i >= B * h * w) return;
  const long long n = stats->n;
  const float g_ms = upstream(G.up[0]);
  if (cta0 > 0) {                                         // a scale k >= 1
    if (!out) return;
    const int cx = i % w, cy = (i / w) % h, b = i / (h * w);
    const int y0 = first_dst(cy, H, sy, h), y1 = first_dst(cy + 1, H, sy, h);
    const int x0 = first_dst(cx, W, sx, w), x1 = first_dst(cx + 1, W, sx, w);
    const float v = __ldg(lp + i);
    int acc = 0;                                          // sum of sign(lp - lg) over the masked preimage
    for (int y = y0; y < y1; ++y) {
      const size_t row = ((size_t)b * H + y) * W;
      for (int x = x0; x < x1; ++x) {
        if (!__ldg(mask + row + x)) continue;
        const float lg = logf(__ldg(gt + row + x));
        acc += (v > lg) - (v < lg);
      }
    }
    out[i] = acc != 0 ? (float)acc * __fdiv_rn(g_ms * inv_pow, (float)n) : 0.f;
    return;
  }
  float g_lp = 0.f, g_dp = 0.f;
  if (__ldg(mask + i)) {                                  // n > 0 here
    const float fn = (float)n;
    const float g = __ldg(gt + i), lg = logf(g), v0 = __ldg(S.lp[0] + i), v = __ldg(dp + i);
    const float d = __fadd_rn(lg, -v0);
    g_lp = sign_of(-d) * (__fdiv_rn(g_ms, fn) + __fdiv_rn(upstream(G.up[4]), fn));
    const float g_si = upstream(G.up[2]);
    if (g_si != 0.f) {
      const Stats st = *stats;
      g_lp -= (float)((double)g_si * ((double)d - lambda * st.mean_d) / ((double)n * st.si));
    }
    g_dp = sign_of(__fadd_rn(v, -g)) * __fdiv_rn(upstream(G.up[1]), fn);
    if (v > 0.1f) {
      const float r = __fdiv_rn(1.0f, v);
      g_dp += sign_of(__fadd_rn(__fdiv_rn(1.0f, g), -r)) * __fdiv_rn(upstream(G.up[3]), (float)stats->m) * (r * r);
    }
  }
  if (G.lp[0]) G.lp[0][i] = g_lp;
  if (G.dp) G.dp[i] = g_dp;
}

inline size_t partials_bytes(const srcv_regloss_args& a) {
  return align256((size_t)forward_ctas(a) * (kSums * sizeof(double) + kCounts * sizeof(long long)));
}

}  // namespace
}  // namespace regloss_detail

namespace rd = regloss_detail;

// workspace: [Stats: n, m (int64), mean(d), si (double), padded to 256 B | partial sums: 6 series of one double per
// forward CTA | partial counts: 2 series of one int64 per forward CTA]
size_t regloss_workspace_bytes(const srcv_regloss_args& a) { return 256 + rd::partials_bytes(a); }

cudaError_t launch_regloss_forward(const srcv_regloss_args& a, float* losses, void* workspace, cudaStream_t stream) {
  const rd::Scales S = rd::make_scales(a);
  const unsigned nb = rd::forward_ctas(a);
  rd::Stats* stats = reinterpret_cast<rd::Stats*>(workspace);
  double* psum = reinterpret_cast<double*>(reinterpret_cast<uint8_t*>(workspace) + 256);
  long long* pcnt = reinterpret_cast<long long*>(psum + (size_t)rd::kSums * nb);
  SRCV_LAUNCH(rd::regloss_kernel, nb, rd::kThreads, 0, stream, a.gt, a.mask, a.depth_pred, a.B, a.H, a.W, S, psum,
              pcnt);
  note_launch();
  SRCV_LAUNCH(rd::regloss_finalize_kernel, 1, rd::kThreads, 0, stream, (const double*)psum, (const long long*)pcnt, nb,
              a.si_lambda, losses, stats);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_regloss_backward(const srcv_regloss_args& a, const float* const grad_losses[5],
                                    float* const grad_log_pred[kRegLossMaxScales], float* grad_depth_pred,
                                    const void* workspace, cudaStream_t stream) {
  const rd::Scales S = rd::make_scales(a);
  rd::Grads G{};
  for (int k = 0; k < 5; ++k) G.up[k] = grad_losses[k];
  for (int k = 0; k < kRegLossMaxScales; ++k) G.lp[k] = a.log_pred[k] ? grad_log_pred[k] : nullptr;
  G.dp = grad_depth_pred;
  SRCV_LAUNCH(rd::regloss_backward_kernel, S.cta0[kRegLossMaxScales], rd::kThreads, 0, stream, a.gt, a.mask,
              a.depth_pred, a.B, a.H, a.W, S, a.si_lambda, reinterpret_cast<const rd::Stats*>(workspace), G);
  note_launch();
  return cudaGetLastError();
}

}  // namespace srcv
