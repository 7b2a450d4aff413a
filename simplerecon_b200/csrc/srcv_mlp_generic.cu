// Metadata-MLP plane-sweep volume, shape-generic fp32 SIMT variant.
//
// Replaces FeatureVolumeManager.build_cost_volume / FastFeatureVolumeManager
// .build_cost_volume (reference modules/cost_volume.py:451-736, :967-1164) for any
// K, C and any two-hidden-layer MLP with widths <= 128.
//
// One CTA = 128 consecutive pixels of one frame at one depth plane.  The CTA
//   A. builds the 128 x F metadata tile in shared memory (feature-major, so a
//      thread's row is a bank-conflict-free column) — the tensor the reference
//      materialises as (B,F,H,W) per plane (15.5 MB) and the fast reference path
//      as (B*D,H,W,F) (993 MB per frame) lives only here;
//   B. runs F->H1->H2->1 as two register-tiled fp32 GEMMs (8x8 outputs per
//      thread, weights streamed through a double-buffered 8-row chunk) with the
//      LeakyReLU(0.01) epilogues in registers and the final H2->1 layer as a dot
//      in the second epilogue.
// This variant is the fp32-exact fallback of the tensor-core kernel and the
// first-round baseline; it is bound by the FP32 FMA pipe (~85 kFLOP per row).
#include "srcv_kernels.h"

namespace srcv {

namespace {

constexpr int TM = 128;       // rows (pixels) per CTA
constexpr int NT = 256;       // threads per CTA
constexpr int KC = 8;         // weight rows per streamed chunk
constexpr int NMAX = 128;     // padded layer width

struct MlpDims {
  int F;      // true input features
  int Fp;     // padded to a multiple of KC
  int H1, H2; // true hidden widths (<= NMAX)
  int H1p;    // H1 padded to KC
  int rows;   // rows of the activation tile = max(Fp, H1p)
};

__host__ __device__ inline MlpDims make_dims(int K, int C, int H1, int H2) {
  MlpDims m;
  m.F = mlp_features(K, C);
  m.Fp = (m.F + KC - 1) / KC * KC;
  m.H1 = H1; m.H2 = H2;
  m.H1p = (H1 + KC - 1) / KC * KC;
  m.rows = m.Fp > m.H1p ? m.Fp : m.H1p;
  return m;
}

// Transposes nn.Linear weights (out,in) into zero-padded (in_p, NMAX) so that the
// GEMM streams rows of NMAX contiguous output weights.
__global__ void __launch_bounds__(256)
mlp_pack_weights_kernel(const float* __restrict__ w1, const float* __restrict__ w2, MlpDims m,
                        float* __restrict__ w1t, float* __restrict__ w2t) {
  const int n1 = m.Fp * NMAX, n2 = m.H1p * NMAX;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n1 + n2; i += gridDim.x * blockDim.x) {
    if (i < n1) {
      const int f = i / NMAX, n = i - f * NMAX;
      w1t[i] = (f < m.F && n < m.H1) ? w1[(size_t)n * m.F + f] : 0.f;
    } else {
      const int q = i - n1;
      const int f = q / NMAX, n = q - f * NMAX;
      w2t[q] = (f < m.H1 && n < m.H2) ? w2[(size_t)n * m.H1 + f] : 0.f;
    }
  }
}

// acc[8][8] += A[f][r0..r0+7] * Wt[f][n0..n0+7] for f in [0, nf), Wt streamed from global.
__device__ __forceinline__ void tile_gemm(float (&acc)[8][8], const float* __restrict__ sA,
                                          float* __restrict__ sW, const float* __restrict__ wt,
                                          int nf, int r0, int n0) {
  const int tid = threadIdx.x;
  // chunk = KC x NMAX floats = 1024 floats = 256 float4: one per thread
  float4 nxt = __ldg(reinterpret_cast<const float4*>(wt) + tid);
  int buf = 0;
  for (int f0 = 0; f0 < nf; f0 += KC) {
    reinterpret_cast<float4*>(sW + buf * KC * NMAX)[tid] = nxt;
    __syncthreads();
    if (f0 + KC < nf)
      nxt = __ldg(reinterpret_cast<const float4*>(wt + (size_t)(f0 + KC) * NMAX) + tid);
    const float* wb = sW + buf * KC * NMAX;
#pragma unroll
    for (int ff = 0; ff < KC; ++ff) {
      const float4 a0 = *reinterpret_cast<const float4*>(sA + (f0 + ff) * TM + r0);
      const float4 a1 = *reinterpret_cast<const float4*>(sA + (f0 + ff) * TM + r0 + 4);
      const float4 w0 = *reinterpret_cast<const float4*>(wb + ff * NMAX + n0);
      const float4 w1 = *reinterpret_cast<const float4*>(wb + ff * NMAX + n0 + 4);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int jn = 0; jn < 8; ++jn) acc[i][jn] = fmaf(a[i], w[jn], acc[i][jn]);
    }
    buf ^= 1;
    // the next iteration writes the other buffer; the sync after that write also
    // orders this iteration's reads before the write after next.
  }
  __syncthreads();
}

template <bool PER_PIXEL>
__global__ void __launch_bounds__(NT, 1)
mlp_generic_kernel(srcv_shape s, MlpDims m, const float* __restrict__ cur,
                   const float* __restrict__ src, const ViewParams* __restrict__ views,
                   const FrameParams* __restrict__ frames, const float* __restrict__ planes,
                   const float* __restrict__ w1t, const float* __restrict__ b1,
                   const float* __restrict__ w2t, const float* __restrict__ b2,
                   const float* __restrict__ w3, const float* __restrict__ b3,
                   float* __restrict__ cost, uint8_t* __restrict__ mask_out) {
  SRCV_DYNAMIC_SMEM_ALIGNED(float, smem, 16);
  float* sA = smem;                         // [rows][TM]
  float* sW = sA + (size_t)m.rows * TM;     // [2][KC][NMAX]  (also the 16 x TM partial buffer)
  int* sFlag = reinterpret_cast<int*>(sW + 2 * KC * NMAX);  // [TM] mask bits
  const int tid = threadIdx.x;
  const int b = blockIdx.z, d = blockIdx.y;
  const int HW = s.H * s.W, K = s.K, C = s.C;
  const int p0 = blockIdx.x * TM;
  const bool want_mask = (mask_out != nullptr) && (d == s.D - 1);

  const MetaLayout o(K, C);
  const Centre ctr(s.W, s.H);
  const FrameParams fp = frames[b];

  if (tid < TM) sFlag[tid] = 0;
  __syncthreads();

  // ---------------- A. metadata tile -------------------------------------------
  for (int it = tid; it < TM * K; it += NT) {
    const int r = it % TM, k = it / TM;
    const int p = min(p0 + r, HW - 1);
    const Sample sm = metadata_row(sA, TM, r, m.F, m.rows, o, s, cur, src, views[b * K + k], fp, b, k, p,
                                   plane_depth<PER_PIXEL>(planes, b, s.D, d, HW, p));
    if (want_mask) {
      int bits = 0;
      if (sm.zp > 0.0f) bits |= 1;
      if (in_mask_bounds(sm.px, sm.py, s.W, s.H, ctr)) bits |= 2;
      if (bits) atomicOr(&sFlag[r], bits);
    }
  }
  __syncthreads();
  if (want_mask && tid < TM && p0 + tid < HW)
    mask_out[(size_t)b * HW + p0 + tid] = (sFlag[tid] == 3) ? 1 : 0;

  // ---------------- B. MLP --------------------------------------------------------
  const int r0 = (tid & 15) * 8, n0 = (tid >> 4) * 8;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int jn = 0; jn < 8; ++jn) acc[i][jn] = 0.f;
  tile_gemm(acc, sA, sW, w1t, m.Fp, r0, n0);   // ends with a block sync: sA free to overwrite
#pragma unroll
  for (int jn = 0; jn < 8; ++jn) {
    const int n = n0 + jn;
    const float bias = n < m.H1 ? __ldg(b1 + n) : 0.f;
    float4 h0, h1;
    h0.x = leaky(acc[0][jn] + bias); h0.y = leaky(acc[1][jn] + bias);
    h0.z = leaky(acc[2][jn] + bias); h0.w = leaky(acc[3][jn] + bias);
    h1.x = leaky(acc[4][jn] + bias); h1.y = leaky(acc[5][jn] + bias);
    h1.z = leaky(acc[6][jn] + bias); h1.w = leaky(acc[7][jn] + bias);
    if (n < m.H1p) {
      *reinterpret_cast<float4*>(sA + n * TM + r0) = h0;
      *reinterpret_cast<float4*>(sA + n * TM + r0 + 4) = h1;
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int jn = 0; jn < 8; ++jn) acc[i][jn] = 0.f;
  __syncthreads();
  tile_gemm(acc, sA, sW, w2t, m.H1p, r0, n0);
  // layer 3 as a dot in the epilogue; reduce the 16 column groups through smem
  float part[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int jn = 0; jn < 8; ++jn) {
    const int n = n0 + jn;
    if (n < m.H2) {
      const float bias = __ldg(b2 + n), w = __ldg(w3 + n);
#pragma unroll
      for (int i = 0; i < 8; ++i) part[i] = fmaf(leaky(acc[i][jn] + bias), w, part[i]);
    }
  }
  float* sP = sW;  // [16][TM]
  *reinterpret_cast<float4*>(sP + (tid >> 4) * TM + r0) = make_float4(part[0], part[1], part[2], part[3]);
  *reinterpret_cast<float4*>(sP + (tid >> 4) * TM + r0 + 4) = make_float4(part[4], part[5], part[6], part[7]);
  __syncthreads();
  if (tid < TM && p0 + tid < HW) {
    float v = 0.f;
#pragma unroll
    for (int g = 0; g < 16; ++g) v += sP[g * TM + tid];
    cost[((size_t)b * s.D + d) * HW + p0 + tid] = v + __ldg(b3);
  }
}

size_t smem_bytes(const MlpDims& m) {
  return sizeof(float) * ((size_t)m.rows * TM + 2 * KC * NMAX) + sizeof(int) * TM;
}

}  // namespace

bool mlp_generic_supported(const srcv_shape& s, const srcv_mlp_weights& w) {
  if (w.hidden1 < 1 || w.hidden1 > NMAX || w.hidden2 < 1 || w.hidden2 > NMAX) return false;
  const MlpDims m = make_dims(s.K, s.C, w.hidden1, w.hidden2);
  return smem_bytes(m) <= 227 * 1024 && s.D <= 65535 && s.B <= 65535;
}

size_t mlp_generic_extra_bytes(const srcv_shape& s, const srcv_mlp_weights& w) {
  const MlpDims m = make_dims(s.K, s.C, w.hidden1, w.hidden2);
  return sizeof(float) * (size_t)(m.Fp + m.H1p) * NMAX;
}

cudaError_t launch_mlp_generic(const srcv_shape& s, const float* cur, const float* src,
                               const Workspace& ws, const float* planes, bool per_pixel,
                               const srcv_mlp_weights& w, float* cost, float* lowest,
                               uint8_t* mask, cudaStream_t stream) {
  const MlpDims m = make_dims(s.K, s.C, w.hidden1, w.hidden2);
  float* w1t = ws.extra;
  float* w2t = ws.extra + (size_t)m.Fp * NMAX;
  SRCV_LAUNCH(mlp_pack_weights_kernel, 64, 256, 0, stream, w.w1, w.w2, m, w1t, w2t);
  note_launch();
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return err;
  const size_t smem = smem_bytes(m);
  const int HW = s.H * s.W;
  dim3 grid((HW + TM - 1) / TM, s.D, s.B), block(NT);
  if (per_pixel) {
    err = cudaFuncSetAttribute(mlp_generic_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (err != cudaSuccess) return err;
    SRCV_LAUNCH(mlp_generic_kernel<true>, grid, block, smem, stream, s, m, cur, src, ws.views, ws.frames, planes,
                w1t, w.b1, w2t, w.b2, w.w3, w.b3, cost, mask);
  } else {
    err = cudaFuncSetAttribute(mlp_generic_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (err != cudaSuccess) return err;
    SRCV_LAUNCH(mlp_generic_kernel<false>, grid, block, smem, stream, s, m, cur, src, ws.views, ws.frames, planes,
                w1t, w.b1, w2t, w.b2, w.w3, w.b3, cost, mask);
  }
  note_launch();
  err = cudaGetLastError();
  if (err != cudaSuccess) return err;
  if (lowest) err = launch_argmax(s, cost, planes, per_pixel, lowest, stream);
  return err;
}

}  // namespace srcv
