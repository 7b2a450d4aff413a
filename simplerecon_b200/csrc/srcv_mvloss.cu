// Multi-view depth regression loss — MVDepthLoss of the reference (losses.py:79-208, Equation 5
// of the paper; experiment_modules/depth_model.py:477-485 adds it to the training loss x 0.2).
//
//   per source view k:  mean over the batch's VALID pixels of | log s_k(p) - log z_k(p; pred) |
//   loss = mean over k
// where, for reference pixel p, the GROUND-TRUTH depth is back-projected and projected into view k to
// nearest-sample that view's depth map (s_k) and to decide validity (in front of the view, not
// occluded: z < 1.05 s, s > 0), and the PREDICTED depth is pushed through the same projection to
// get its depth in view k (z_k).  NaN terms (a prediction behind the source camera) are dropped
// from the mean (nanmean, :173).
//
// The reference runs, per view, two BackprojectDepth + Project3D chains, a grid_sample and four
// masked (B,1,H,W) intermediates: ~40 launches and ~30 full-size tensors per view.  Here one thread
// owns a pixel and walks the views in registers — the same geometry front end as the sweeps
// (un-project -> rigid transform -> project -> sample) in the reference's fp32 operation order —
// so the traffic is the two depth maps, one nearest sample per (pixel, view), and for the backward
// one gradient write: 8 + 4 K bytes read per pixel.
//
//   forward : per-CTA partial (sum, count) per view -> fixed-order fp64 finalize (deterministic)
//   backward: recomputes the geometry (cheaper than storing K terms per pixel); z_k is affine in
//             the predicted depth, so  d loss / d pred(p) = g/K  sum_k [term kept] sign(log z - log s)
//             (dz_k/dd) / z_k / count_k.
#include "srcv_kernels.h"

namespace srcv {

namespace {

constexpr int kThreads = 256;
constexpr int kMaxViews = 16;        // views staged per CTA (the reference trains with 7)

struct MvlFrame {                    // per batch item, in shared memory
  float invK[9];                     // cur_invK[:3,:3]
  float T[12];                       // cur_world_T_cam rows 0..2
  float P[kMaxViews][12];            // (src_K @ src_cam_T_world) rows 0..2, utils/geometry_utils.py:78
};

__device__ __forceinline__ void stage_frame(const srcv_mvloss_args& a, int b, MvlFrame& f) {
  for (int i = threadIdx.x; i < 9; i += blockDim.x) f.invK[i] = a.cur_invK[(size_t)b * 16 + (i / 3) * 4 + i % 3];
  for (int i = threadIdx.x; i < 12; i += blockDim.x) f.T[i] = a.cur_world_T_cam[(size_t)b * 16 + i];
  for (int i = threadIdx.x; i < a.K * 12; i += blockDim.x) {
    const int k = i / 12, r = (i % 12) / 4, c = i % 4;
    const float* Km = a.src_K + ((size_t)b * a.K + k) * 16 + r * 4;
    const float* Tm = a.src_cam_T_world + ((size_t)b * a.K + k) * 16 + c;
    // 4x4 product as the k-ascending FMA chain of a fp32 GEMM
    f.P[k][r * 4 + c] = __fmaf_rn(Km[3], Tm[12], __fmaf_rn(Km[2], Tm[8], __fmaf_rn(Km[1], Tm[4], __fmul_rn(Km[0], Tm[0]))));
  }
}

// the ray r = invK3 (x + .5, y + .5, 1) of a pixel (utils/geometry_utils.py:55)
__device__ __forceinline__ void pixel_ray(const MvlFrame& f, int px, int py, float& rx, float& ry, float& rz) {
  const float x = (float)px + 0.5f, y = (float)py + 0.5f;
  rx = __fmaf_rn(f.invK[2], 1.0f, __fmaf_rn(f.invK[1], y, __fmul_rn(f.invK[0], x)));
  ry = __fmaf_rn(f.invK[5], 1.0f, __fmaf_rn(f.invK[4], y, __fmul_rn(f.invK[3], x)));
  rz = __fmaf_rn(f.invK[8], 1.0f, __fmaf_rn(f.invK[7], y, __fmul_rn(f.invK[6], x)));
}
// world = cur_world_T_cam [d r; 1]   (:56-57, losses.py:103)
__device__ __forceinline__ void to_world(const MvlFrame& f, float d, float rx, float ry, float rz, float& X, float& Y,
                                         float& Z) {
  const float cx = __fmul_rn(d, rx), cy = __fmul_rn(d, ry), cz = __fmul_rn(d, rz);
  X = __fmaf_rn(f.T[3], 1.0f, __fmaf_rn(f.T[2], cz, __fmaf_rn(f.T[1], cy, __fmul_rn(f.T[0], cx))));
  Y = __fmaf_rn(f.T[7], 1.0f, __fmaf_rn(f.T[6], cz, __fmaf_rn(f.T[5], cy, __fmul_rn(f.T[4], cx))));
  Z = __fmaf_rn(f.T[11], 1.0f, __fmaf_rn(f.T[10], cz, __fmaf_rn(f.T[9], cy, __fmul_rn(f.T[8], cx))));
}
__device__ __forceinline__ float row4(const float* __restrict__ P, float X, float Y, float Z) {
  return __fmaf_rn(P[3], 1.0f, __fmaf_rn(P[2], Z, __fmaf_rn(P[1], Y, __fmul_rn(P[0], X))));
}

// One (pixel, view): validity from the ground-truth depth and the sampled source depth
// (losses.py:90-135).  Returns valid; s = the nearest sample (0 outside the map).
__device__ __forceinline__ bool view_valid(const float* __restrict__ P, float X, float Y, float Z,
                                           const float* __restrict__ src_depth, int W, int H, float& s) {
  const float c0 = row4(P, X, Y, Z), c1 = row4(P + 4, X, Y, Z), c2 = row4(P + 8, X, Y, Z);
  const float z = __fadd_rn(c2, kEpsProj);                                  // geometry_utils.py:84
  const float scale = (fabsf(c2) > kEpsProj) ? __fdiv_rn(1.0f, z) : 1.0f;   // :83-85
  const float u = __fmul_rn(c0, scale), v = __fmul_rn(c1, scale);
  // uv = 2 (pix / [W, H]) - 1 (losses.py:112-117); grid_sample(nearest, align_corners=False):
  // index = nearbyint(((uv + 1) size - 1) / 2), zeros outside
  const float gu = __fadd_rn(__fmul_rn(2.0f, __fdiv_rn(u, (float)W)), -1.0f);
  const float gv = __fadd_rn(__fmul_rn(2.0f, __fdiv_rn(v, (float)H)), -1.0f);
  const float ix = rintf(__fdiv_rn(__fadd_rn(__fmul_rn(__fadd_rn(gu, 1.0f), (float)W), -1.0f), 2.0f));
  const float iy = rintf(__fdiv_rn(__fadd_rn(__fmul_rn(__fadd_rn(gv, 1.0f), (float)H), -1.0f), 2.0f));
  s = 0.f;
  if (ix >= 0.f && ix < (float)W && iy >= 0.f && iy < (float)H) s = __ldg(src_depth + (int)iy * W + (int)ix);
  return (z < __fmul_rn(1.05f, s)) && (z > 0.f) && (s > 0.f);              // losses.py:127-131
}

// grid (ceil(HW / 256), B).  FORWARD: partial[(b * gridDim.x + blockIdx.x) * K + k] = (sum, count);
// optional per-view validity / sample outputs (get_valid_mask).  BACKWARD: grad_pred.
template <bool BACKWARD>
__global__ void __launch_bounds__(kThreads)
mvloss_kernel(srcv_mvloss_args a, float2* __restrict__ partial, uint8_t* __restrict__ valid_out,
              float* __restrict__ sampled_out, const float* __restrict__ inv_count,
              const float* __restrict__ grad_loss, float* __restrict__ grad_pred) {
  __shared__ MvlFrame f;
  __shared__ float s_sum[kThreads / 32][kMaxViews], s_cnt[kThreads / 32][kMaxViews];
  const int b = blockIdx.y, HW = a.H * a.W, K = a.K;
  stage_frame(a, b, f);
  __syncthreads();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const bool live = p < HW;
  const int px = live ? p % a.W : 0, py = live ? p / a.W : 0;
  const size_t pix = (size_t)b * HW + (live ? p : 0);
  float rx, ry, rz, Xg, Yg, Zg, Xp, Yp, Zp;
  pixel_ray(f, px, py, rx, ry, rz);
  const float d_gt = __ldg(a.cur_depth + pix), d_pr = __ldg(a.depth_pred + pix);
  to_world(f, d_gt, rx, ry, rz, Xg, Yg, Zg);
  to_world(f, d_pr, rx, ry, rz, Xp, Yp, Zp);
  // dz/dd of the predicted point: P[2,:3] (R_wc r)
  float wx = 0.f, wy = 0.f, wz = 0.f;
  if (BACKWARD) {
    wx = fmaf(f.T[2], rz, fmaf(f.T[1], ry, f.T[0] * rx));
    wy = fmaf(f.T[6], rz, fmaf(f.T[5], ry, f.T[4] * rx));
    wz = fmaf(f.T[10], rz, fmaf(f.T[9], ry, f.T[8] * rx));
  }
  float gacc = 0.f;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int k = 0; k < K; ++k) {
    const float* P = f.P[k];
    float s = 0.f;
    const bool valid = live && view_valid(P, Xg, Yg, Zg, a.src_depth + ((size_t)b * K + k) * HW, a.W, a.H, s);
    const float zp = __fadd_rn(row4(P + 8, Xp, Yp, Zp), kEpsProj);         // depth of the prediction in view k
    const float diff = __fadd_rn(logf(s), -logf(zp));                      // losses.py:168-170
    const float term = fabsf(diff);
    const bool keep = valid && !(term != term);                            // nanmean drops NaN terms, :173
    if (!BACKWARD) {
      if (live && valid_out) valid_out[((size_t)b * K + k) * HW + p] = valid ? 1 : 0;
      if (live && sampled_out) sampled_out[((size_t)b * K + k) * HW + p] = s;
      // CTA reduction: warp tree through shuffles of the bit patterns, then one row per warp
      float vs = keep ? term : 0.f, vc = keep ? 1.f : 0.f;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        vs += __uint_as_float((unsigned)__shfl_sync(0xffffffffu, (int)__float_as_uint(vs), (lane + o) & 31));
        vc += __uint_as_float((unsigned)__shfl_sync(0xffffffffu, (int)__float_as_uint(vc), (lane + o) & 31));
      }
      if (lane == 0) { s_sum[warp][k] = vs; s_cnt[warp][k] = vc; }
    } else if (keep) {
      // d|log s - log z|/dz = sign(log z - log s) / z ;  z = (dz/dd) d + const
      const float sg = diff < 0.f ? 1.0f : (diff > 0.f ? -1.0f : 0.f);
      const float dzdd = fmaf(P[10], wz, fmaf(P[9], wy, P[8] * wx));
      gacc = fmaf(sg * __ldg(inv_count + k), __fdiv_rn(dzdd, zp), gacc);
    }
  }
  if (!BACKWARD) {
    __syncthreads();
    if (threadIdx.x < K) {
      float ts = 0.f, tc = 0.f;
      for (int w = 0; w < kThreads / 32; ++w) { ts += s_sum[w][threadIdx.x]; tc += s_cnt[w][threadIdx.x]; }
      partial[((size_t)b * gridDim.x + blockIdx.x) * K + threadIdx.x] = make_float2(ts, tc);
    }
  } else if (live) {
    grad_pred[pix] = gacc * (__ldg(grad_loss) / (float)K);
  }
}

// loss = (1/K) sum_k sum_k / count_k, fp64, in a fixed order (thread-strided partial sums, then a
// shared-memory tree: the same association on every run); inv_count[k] for the backward
__global__ void __launch_bounds__(kThreads)
mvloss_finalize_kernel(const float2* __restrict__ partial, int n_partials, int K, float* __restrict__ loss,
                       float* __restrict__ inv_count) {
  __shared__ double s_sum[kThreads], s_cnt[kThreads];
  double total = 0.0;
  for (int k = 0; k < K; ++k) {
    double sum = 0.0, cnt = 0.0;
    for (int i = threadIdx.x; i < n_partials; i += kThreads) {
      const float2 v = partial[(size_t)i * K + k];
      sum += (double)v.x;
      cnt += (double)v.y;
    }
    s_sum[threadIdx.x] = sum;
    s_cnt[threadIdx.x] = cnt;
    __syncthreads();
    for (int o = kThreads / 2; o > 0; o >>= 1) {
      if ((int)threadIdx.x < o) {
        s_sum[threadIdx.x] += s_sum[threadIdx.x + o];
        s_cnt[threadIdx.x] += s_cnt[threadIdx.x + o];
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      total += s_sum[0] / s_cnt[0];              // an empty view gives 0/0 = NaN, like nanmean of nothing
      inv_count[k] = s_cnt[0] > 0.0 ? (float)(1.0 / s_cnt[0]) : 0.f;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss = (float)(total / (double)K);
}

inline size_t partial_count(const srcv_mvloss_args& a) { return (size_t)a.B * (((size_t)a.H * a.W + kThreads - 1) / kThreads); }

}  // namespace

int mvloss_max_views() { return kMaxViews; }

// workspace: [inv_count: kMaxViews floats, padded to 256 B | partials: B * ceil(HW/256) * K float2]
size_t mvloss_workspace_bytes(const srcv_mvloss_args& a) {
  return 256 + ((partial_count(a) * (size_t)a.K * sizeof(float2) + 255) & ~(size_t)255);
}

cudaError_t launch_mvloss_forward(const srcv_mvloss_args& a, float* loss, uint8_t* valid, float* sampled,
                                  void* workspace, cudaStream_t stream) {
  float* inv_count = reinterpret_cast<float*>(workspace);
  float2* partial = reinterpret_cast<float2*>(reinterpret_cast<uint8_t*>(workspace) + 256);
  const dim3 grid((unsigned)((a.H * a.W + kThreads - 1) / kThreads), (unsigned)a.B);
  SRCV_LAUNCH((mvloss_kernel<false>), grid, kThreads, 0, stream, a, partial, valid, sampled,
              (const float*)nullptr, (const float*)nullptr, (float*)nullptr);
  note_launch();
  SRCV_LAUNCH(mvloss_finalize_kernel, 1, kThreads, 0, stream, (const float2*)partial, (int)partial_count(a), a.K, loss,
              inv_count);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_mvloss_backward(const srcv_mvloss_args& a, const float* grad_loss, float* grad_pred,
                                   const void* workspace, cudaStream_t stream) {
  const float* inv_count = reinterpret_cast<const float*>(workspace);
  const dim3 grid((unsigned)((a.H * a.W + kThreads - 1) / kThreads), (unsigned)a.B);
  SRCV_LAUNCH((mvloss_kernel<true>), grid, kThreads, 0, stream, a, (float2*)nullptr, (uint8_t*)nullptr,
              (float*)nullptr, inv_count, grad_loss, grad_pred);
  note_launch();
  return cudaGetLastError();
}

}  // namespace srcv

#include "srcv_metrics.cuh"   // depth metrics (DESIGN §4.12), compiled in this unit
