// Depth metrics — compute_depth_metrics / compute_depth_metrics_batched of the reference
// (utils/metrics_utils.py:7-120), fused with the resampling test.py:282-299 runs before them
// (F.interpolate of the prediction to the ground-truth grid, then gt > 0.5).  DESIGN §4.12.
//
// One pass over the ground-truth grid: a thread owns kPix pixels of one frame, decides validity
// (explicit mask, gt > min_valid_depth, or every pixel), samples the prediction at the mapped
// source pixel with PyTorch's index rules, forms the reference's fp32 per-pixel terms and
// accumulates them in fp64 plus exact integer counts.  Each CTA reduces its threads in a fixed
// shared-memory tree and writes one partial; a second launch, one CTA per frame, sums the
// partials in a fixed order and writes the 12 metrics.  No atomics: the result is deterministic,
// and the counts stay exact above 2^24 pixels per frame.
//
// Compiled as part of the multi-view loss unit (srcv_mvloss.cu, which includes this header last): the
// two consumers of the predicted depth that the training step runs next to each other share one
// translation unit, as the mesh kernels share the TSDF one.  The internals live in their own namespace.
#pragma once
#include "srcv_kernels.h"

namespace srcv {

namespace metrics_detail {
namespace {

constexpr int kThreads = 256;
constexpr int kPix = 4;                            // pixels per thread
constexpr int kSums = 5;                           // abs_diff, abs_rel, sq_rel, rmse, rmse_log
constexpr int kThresh = 5;                         // 1.05, 1.10, 1.25, 1.25^2, 1.25^3
constexpr int kCounts = 1 + kThresh + kSums;       // valid, a-counts, non-NaN count of each sum
constexpr int kSlots = kSums + kCounts;            // one partial = 16 eight-byte slots
static_assert(kPix < 16, "per-thread counts are kept in 4-bit fields");

union Slot {
  double d;
  unsigned long long u;
};

// The thresholds the reference compares fp32 ratios against, rounded to fp32 as PyTorch does
// with a Python-float scalar (metrics_utils.py:14-21, :67-93).
__device__ __forceinline__ float thresh_at(int i) {
  switch (i) {
    case 0: return 1.05f;
    case 1: return 1.10f;
    case 2: return 1.25f;
    case 3: return 1.5625f;
    default: return 1.953125f;
  }
}

__device__ __forceinline__ bool is_nan(float x) { return x != x; }

// PyTorch's align_corners=False source coordinate of bilinear resampling,
// scale * (dst + 0.5) - 0.5 clamped at 0 (contracted to one FMA, as nvcc builds PyTorch's kernel)
__device__ __forceinline__ float linear_src(float scale, int dst) {
  const float s = __fmaf_rn(scale, __fadd_rn((float)dst, 0.5f), -0.5f);
  return s < 0.f ? 0.f : s;
}

// The prediction at ground-truth pixel (x, y) of frame `pred` (Hp x Wp).
__device__ __forceinline__ float sample_pred(const srcv_metrics_args& a, const float* __restrict__ pred, int x, int y,
                                             int p, float sy, float sx) {
  if (a.resample == SRCV_RESAMPLE_NEAREST) {       // min(floor(dst * in/out), in - 1)
    const int iy = min((int)floorf(__fmul_rn((float)y, sy)), a.Hp - 1);
    const int ix = min((int)floorf(__fmul_rn((float)x, sx)), a.Wp - 1);
    return __ldg(pred + iy * a.Wp + ix);
  }
  if (a.resample == SRCV_RESAMPLE_BILINEAR) {
    const float hr = linear_src(sy, y), wr = linear_src(sx, x);
    const int h1 = (int)hr, w1 = (int)wr;
    const int dy = h1 < a.Hp - 1 ? a.Wp : 0, dx = w1 < a.Wp - 1 ? 1 : 0;   // PyTorch's clamp of the upper neighbour
    const float h1l = __fadd_rn(hr, -(float)h1), w1l = __fadd_rn(wr, -(float)w1);
    const float h0l = __fadd_rn(1.0f, -h1l), w0l = __fadd_rn(1.0f, -w1l);
    const float* r0 = pred + h1 * a.Wp + w1;
    const float* r1 = r0 + dy;
    // h0 (w0 x00 + w1 x01) + h1 (w0 x10 + w1 x11), with the FMAs nvcc forms for that expression
    const float top = __fmaf_rn(w0l, __ldg(r0), __fmul_rn(w1l, __ldg(r0 + dx)));
    const float bot = __fmaf_rn(w0l, __ldg(r1), __fmul_rn(w1l, __ldg(r1 + dx)));
    return __fmaf_rn(h0l, top, __fmul_rn(h1l, bot));
  }
  return __ldg(pred + p);                          // identity
}

// grid (blocks_per_frame, B)
__global__ void __launch_bounds__(kThreads)
metrics_kernel(srcv_metrics_args a, Slot* __restrict__ partial, float* __restrict__ upsampled) {
  __shared__ Slot s_red[kSlots][kThreads];
  const int b = blockIdx.y, HW = a.H * a.W, t = threadIdx.x;
  const size_t frame = (size_t)b * HW;
  const float* gt = a.gt + frame;
  const float* pred = a.pred + (size_t)b * a.Hp * a.Wp;
  const uint8_t* valid = a.valid ? a.valid + frame : nullptr;
  const float sy = __fdiv_rn((float)a.Hp, (float)a.H), sx = __fdiv_rn((float)a.Wp, (float)a.W);
  double sum[kSums] = {0.0, 0.0, 0.0, 0.0, 0.0};
  // the counts of at most kPix pixels, in 4-bit fields (few registers stay live across the
  // division slow-path calls): [valid, a-count of each threshold], [non-NaN count of each term]
  unsigned cnt_a = 0u, cnt_n = 0u;
  const int base = blockIdx.x * (kThreads * kPix) + t;
#pragma unroll
  for (int i = 0; i < kPix; ++i) {
    const int p = base + i * kThreads;
    if (p >= HW) break;
    const int y = p / a.W, x = p - y * a.W;
    const float g = __ldg(gt + p);
    const float v = sample_pred(a, pred, x, y, p, sy, sx);
    if (upsampled) upsampled[frame + p] = v;
    const bool ok = a.valid_source == SRCV_METRICS_VALID_MASK       ? __ldg(valid + p) != 0
                    : a.valid_source == SRCV_METRICS_VALID_MIN_DEPTH ? g > a.min_valid_depth
                                                                     : true;
    if (!ok) continue;
    // thresh = max(gt / pred, pred / gt), NaN-propagating like torch.max
    const float r1 = __fdiv_rn(g, v), r2 = __fdiv_rn(v, g);
    const float th = (is_nan(r1) || r1 > r2) ? r1 : r2;
    unsigned fa = 1u;
#pragma unroll
    for (int k = 0; k < kThresh; ++k) fa |= (th < thresh_at(k) ? 1u : 0u) << (4 * (1 + k));
    cnt_a += fa;
    const float d = __fadd_rn(g, -v);
    const float sq = __fmul_rn(d, d);
    const float lg = __fadd_rn(logf(g), -logf(v));
    const float term[kSums] = {fabsf(d), __fdiv_rn(fabsf(d), g), __fdiv_rn(sq, g), sq, __fmul_rn(lg, lg)};
#pragma unroll
    for (int k = 0; k < kSums; ++k) {
      if (!is_nan(term[k])) {               // batched: nanmean drops the term; flat: NaN if any dropped
        sum[k] += (double)term[k];
        cnt_n += 1u << (4 * k);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < kSums; ++k) s_red[k][t].d = sum[k];
#pragma unroll
  for (int k = 0; k < kCounts; ++k)
    s_red[kSums + k][t].u = ((k <= kThresh ? cnt_a : cnt_n) >> (4 * (k <= kThresh ? k : k - 1 - kThresh))) & 15u;
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {      // fixed-order tree
    if (t < o) {
#pragma unroll
      for (int k = 0; k < kSums; ++k) s_red[k][t].d += s_red[k][t + o].d;
#pragma unroll
      for (int k = kSums; k < kSlots; ++k) s_red[k][t].u += s_red[k][t + o].u;
    }
    __syncthreads();
  }
  if (t < kSlots) partial[((size_t)b * gridDim.x + blockIdx.x) * kSlots + t] = s_red[t][0];
}

// grid (B): the frame's partials summed in a fixed order (thread-strided, then a shared tree)
__global__ void __launch_bounds__(kThreads)
metrics_finalize_kernel(srcv_metrics_args a, const Slot* __restrict__ partial, int n_blocks,
                        float* __restrict__ metrics, long long* __restrict__ valid_counts) {
  __shared__ Slot s_red[kSlots][kThreads];
  const int b = blockIdx.x, t = threadIdx.x;
  double sum[kSums] = {0.0, 0.0, 0.0, 0.0, 0.0};
  unsigned long long cnt[kCounts] = {};
  for (int i = t; i < n_blocks; i += kThreads) {
    const Slot* s = partial + ((size_t)b * n_blocks + i) * kSlots;
#pragma unroll
    for (int k = 0; k < kSums; ++k) sum[k] += s[k].d;
#pragma unroll
    for (int k = 0; k < kCounts; ++k) cnt[k] += s[kSums + k].u;
  }
#pragma unroll
  for (int k = 0; k < kSums; ++k) s_red[k][t].d = sum[k];
#pragma unroll
  for (int k = 0; k < kCounts; ++k) s_red[kSums + k][t].u = cnt[k];
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if (t < o) {
#pragma unroll
      for (int k = 0; k < kSums; ++k) s_red[k][t].d += s_red[k][t + o].d;
#pragma unroll
      for (int k = kSums; k < kSlots; ++k) s_red[k][t].u += s_red[k][t + o].u;
    }
    __syncthreads();
  }
  if (t != 0) return;
  const double n = (double)s_red[kSums][0].u;
  float* m = metrics + (size_t)b * 12;
  // abs_diff, abs_rel, sq_rel, rmse, rmse_log: mean over the non-NaN terms (batched) or over all
  // valid pixels, NaN if any term was NaN (flat); an empty frame gives 0 / 0 = NaN
#pragma unroll
  for (int k = 0; k < kSums; ++k) {
    const double c = (double)s_red[kSums + 1 + kThresh + k][0].u;
    double mean = (a.nan_mode == SRCV_METRICS_FLAT && c != n) ? (double)NAN : s_red[k][0].d / c;
    if (k >= 3) mean = sqrt(mean);
    m[k] = (float)mean;
  }
  // a5, a10, a25, a0 (= a10), a1 (= a25), a2, a3 over the valid pixels
  const int order[7] = {0, 1, 2, 1, 2, 3, 4};
  for (int j = 0; j < 7; ++j) {
    float v = (float)((double)s_red[kSums + 1 + order[j]][0].u / n);
    if (a.mult_a) v = __fmul_rn(v, 100.0f);
    m[kSums + j] = v;
  }
  valid_counts[b] = (long long)s_red[kSums][0].u;
}

inline int blocks_per_frame(const srcv_metrics_args& a) {
  const long long hw = (long long)a.H * a.W;
  const long long n = (hw + kThreads * kPix - 1) / (kThreads * kPix);
  return n > 0 ? (int)n : 1;                       // an empty frame still writes one (zero) partial
}

}  // namespace
}  // namespace metrics_detail

bool metrics_shape_supported(const srcv_metrics_args& a) {
  return (long long)a.H * a.W <= kMetricsMaxPixels && (long long)a.Hp * a.Wp <= kMetricsMaxPixels &&
         a.B <= 65535;
}

size_t metrics_workspace_bytes(const srcv_metrics_args& a) {
  namespace md = metrics_detail;
  return (((size_t)a.B * md::blocks_per_frame(a) * md::kSlots * sizeof(md::Slot)) + 255) & ~(size_t)255;
}

cudaError_t launch_metrics(const srcv_metrics_args& a, float* metrics, long long* valid_counts, float* upsampled,
                           void* workspace, cudaStream_t stream) {
  namespace md = metrics_detail;
  md::Slot* partial = reinterpret_cast<md::Slot*>(workspace);
  const int nb = md::blocks_per_frame(a);
  SRCV_LAUNCH(md::metrics_kernel, dim3((unsigned)nb, (unsigned)a.B), md::kThreads, 0, stream, a, partial, upsampled);
  note_launch();
  SRCV_LAUNCH(md::metrics_finalize_kernel, (unsigned)a.B, md::kThreads, 0, stream, a, (const md::Slot*)partial, nb,
              metrics, valid_counts);
  note_launch();
  return cudaGetLastError();
}

}  // namespace srcv
