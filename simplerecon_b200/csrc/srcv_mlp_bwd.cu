// Backward of the metadata-MLP plane-sweep volume (fp32 SIMT, any K / C with F <= 208,
// hidden widths <= 128).
//
// What autograd of the reference's composite yields for FeatureVolumeManager
// .build_cost_volume (modules/cost_volume.py:451-736; the fast variant :967-1164 has the
// same derivative): given dL/dcost (B,D,H,W) it returns dL/dcur_feats, dL/dsrc_feats and
// the gradients of the six MLP parameters (modules/networks.py:129-147).  Cameras, plane
// depths and the geometric metadata channels (mask, z', depth, rays, angles, pose
// measures) carry no gradient to the features, exactly as in the reference graph: the
// features enter the MLP input only through the warped channels, the reference-feature
// channels and the masked per-view dot products (:691-723).
//
// Nothing of the forward is saved: a persistent CTA walks 64-row tiles (64 consecutive
// pixels of one frame at one depth plane) and for each tile
//   1. rebuilds the 64 x F metadata tile X in shared memory (same arithmetic as the
//      forward kernels, srcv_common.cuh),
//   2. re-runs  A1 = X W1^T + b1, H1 = lrelu(A1),  A2 = H1 W2^T + b2  (register-tiled fp32),
//   3. forms  G2 = g (x) w3 . lrelu'(A2)  in registers,  dW3 += g^T H2,  db3 += sum g,
//      db2 += sum_r G2,  dW2 += G2^T H1,
//   4. G1 = (G2 W2) . lrelu'(A1),  db1 += sum_r G1,  dW1 += G1^T X,
//   5. dX = G1 W1 (over X in place), and scatters it: dL/dwarped = dX_warped + m_k dX_dot cur
//      through the bilinear taps into dL/dsrc (RED.ADD), dL/dcur = dX_cur + sum_k m_k dX_dot
//      warped_k.
// Parameter gradients are flushed per tile with RED.ADD.F32 (42 k addresses, spread).
//
// Layout of every shared tile: [unit][68] floats — unit-major so the forward GEMMs read a
// thread's 4 rows as one 16-byte vector, padded to 68 so those vector reads and the
// 16-lane-strided accesses of the gradient outer products are bank-conflict-free.
#include "srcv_kernels.h"

namespace srcv {

namespace {

constexpr int BT = 64;      // rows (pixels) per tile
constexpr int BTP = 68;     // padded row pitch of the shared tiles
constexpr int BNT = 256;    // threads per CTA: tx = tid & 15, ty = tid >> 4
constexpr int BN = 128;     // padded hidden width
constexpr int BKC = 8;      // streamed weight rows per chunk
constexpr int BFMAX = 208;  // largest padded feature count (13 x 16)

struct BwdDims {
  int F;       // true input features  C (K+1) + 10 K + 4
  int Fp;      // padded: 64, 128 or 208
  int H1, H2;  // true hidden widths
};

__host__ __device__ inline int padded_features(int F) { return F <= 64 ? 64 : (F <= 128 ? 128 : BFMAX); }

// Packs the nn.Linear weights (out, in) into the four zero-padded operand images the
// kernel streams:  w1t [Fp][128] = W1^T,  w2t [128][128] = W2^T,  w2p [128][128] = W2,
// w1p [128][Fp] = W1.
__global__ void __launch_bounds__(256)
mlp_bwd_pack_kernel(const float* __restrict__ w1, const float* __restrict__ w2, BwdDims m,
                    float* __restrict__ w1t, float* __restrict__ w2t, float* __restrict__ w2p,
                    float* __restrict__ w1p) {
  const int n1 = m.Fp * BN, n2 = BN * BN;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 2 * n1 + 2 * n2; i += gridDim.x * blockDim.x) {
    if (i < n1) {                                   // w1t[f][n]
      const int f = i / BN, n = i - f * BN;
      w1t[i] = (f < m.F && n < m.H1) ? w1[(size_t)n * m.F + f] : 0.f;
    } else if (i < n1 + n2) {                       // w2t[n1][n2]
      const int q = i - n1, a = q / BN, n = q - a * BN;
      w2t[q] = (a < m.H1 && n < m.H2) ? w2[(size_t)n * m.H1 + a] : 0.f;
    } else if (i < n1 + 2 * n2) {                   // w2p[n2][n1]
      const int q = i - n1 - n2, n = q / BN, a = q - n * BN;
      w2p[q] = (a < m.H1 && n < m.H2) ? w2[(size_t)n * m.H1 + a] : 0.f;
    } else {                                        // w1p[n1][f]
      const int q = i - n1 - 2 * n2, n = q / m.Fp, f = q - n * m.Fp;
      w1p[q] = (f < m.F && n < m.H1) ? w1[(size_t)n * m.F + f] : 0.f;
    }
  }
}

// Column owned by slot i of thread-column tx in gemm_rows<NI>: NI/4 groups of four adjacent
// columns (one 16-byte shared-memory read per group and k) plus NI%4 single columns.
template <int NI>
__device__ __forceinline__ int gemm_col(int i, int tx) {
  constexpr int NV = NI / 4;
  return i < 4 * NV ? (i >> 2) * 64 + tx * 4 + (i & 3) : NV * 64 + (i - 4 * NV) * 16 + tx;
}

// acc[ii][i] += sum_k A[k][4 ty + ii] * Wg[k][gemm_col<NI>(i, tx)]   for k in [0, nk),
// A a shared tile [k][BTP], Wg a global (nk, 16 NI) image streamed through a double-buffered
// BKC-row chunk (next chunk prefetched into registers while this one is used).  Ends with a
// block sync.
template <int NI>
__device__ __forceinline__ void gemm_rows(float (&acc)[4][NI], const float* __restrict__ sA,
                                          float* __restrict__ sW, const float* __restrict__ wg, int nk) {
  constexpr int ncols = 16 * NI;
  constexpr int NV = NI / 4;
  constexpr int nvec = BKC * ncols / 4;                 // 16-byte vectors per chunk
  constexpr int PER = (nvec + BNT - 1) / BNT;           // per thread: 1 or 2
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  float4 nxt[PER];
#pragma unroll
  for (int v = 0; v < PER; ++v)
    if (tid + v * BNT < nvec) nxt[v] = __ldg(reinterpret_cast<const float4*>(wg) + tid + v * BNT);
  int buf = 0;
  for (int k0 = 0; k0 < nk; k0 += BKC) {
    float* wb = sW + buf * (BKC * BFMAX);
#pragma unroll
    for (int v = 0; v < PER; ++v)
      if (tid + v * BNT < nvec) reinterpret_cast<float4*>(wb)[tid + v * BNT] = nxt[v];
    __syncthreads();   // chunk visible; also: everyone is past the reads of the buffer written next
    if (k0 + BKC < nk) {
#pragma unroll
      for (int v = 0; v < PER; ++v)
        if (tid + v * BNT < nvec)
          nxt[v] = __ldg(reinterpret_cast<const float4*>(wg + (size_t)(k0 + BKC) * ncols) + tid + v * BNT);
    }
#pragma unroll
    for (int kk = 0; kk < BKC; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(sA + (k0 + kk) * BTP + 4 * ty);
      float w[NI];
#pragma unroll
      for (int q = 0; q < NV; ++q) {
        const float4 w4 = *reinterpret_cast<const float4*>(wb + kk * ncols + q * 64 + tx * 4);
        w[4 * q] = w4.x; w[4 * q + 1] = w4.y; w[4 * q + 2] = w4.z; w[4 * q + 3] = w4.w;
      }
#pragma unroll
      for (int i = 4 * NV; i < NI; ++i) w[i] = wb[kk * ncols + NV * 64 + (i - 4 * NV) * 16 + tx];
#pragma unroll
      for (int i = 0; i < NI; ++i) {
        acc[0][i] = fmaf(a.x, w[i], acc[0][i]);
        acc[1][i] = fmaf(a.y, w[i], acc[1][i]);
        acc[2][i] = fmaf(a.z, w[i], acc[2][i]);
        acc[3][i] = fmaf(a.w, w[i], acc[3][i]);
      }
    }
    buf ^= 1;
  }
  __syncthreads();
}

// gout[(ty + 16 j) * ld + (tx + 16 i)] += sum_r A[ty + 16 j][r] * B[tx + 16 i][r]
// (A, B shared tiles [unit][BTP]; the reduction runs over the tile's BT rows).
template <int NI>
__device__ __forceinline__ void grad_outer(const float* __restrict__ sA, const float* __restrict__ sB,
                                           float* __restrict__ gout, int ld, int na, int nb) {
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  float acc[8][NI];
#pragma unroll
  for (int j = 0; j < 8; ++j)
#pragma unroll
    for (int i = 0; i < NI; ++i) acc[j][i] = 0.f;
  for (int r = 0; r < BT; r += 4) {
    float4 a[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = *reinterpret_cast<const float4*>(sA + (ty + 16 * j) * BTP + r);
#pragma unroll
    for (int i = 0; i < NI; ++i) {
      const float4 bv = *reinterpret_cast<const float4*>(sB + (tx + 16 * i) * BTP + r);
#pragma unroll
      for (int j = 0; j < 8; ++j)
        acc[j][i] = fmaf(a[j].x, bv.x, fmaf(a[j].y, bv.y, fmaf(a[j].z, bv.z, fmaf(a[j].w, bv.w, acc[j][i]))));
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int ra = ty + 16 * j;
    if (ra >= na) continue;
#pragma unroll
    for (int i = 0; i < NI; ++i) {
      const int cb = tx + 16 * i;
      if (cb < nb && acc[j][i] != 0.f) atomicAdd(gout + (size_t)ra * ld + cb, acc[j][i]);
    }
  }
}

// Projection of one (row, view) sample: footprint, bilinear weights, z' and the depth mask.
struct Sample {
  Taps tp;
  float w00, w01, w10, w11;
  float px, py, zp, mk;
};

__device__ __forceinline__ void project_sample(const ViewParams& vp, const Centre& ctr, int W, int H,
                                               float pxc, float pyc, float dval, Sample& sm) {
  float ax, ay, az;
  homography_point(vp.a0, pxc - ctr.half_w, pyc - ctr.half_h, ax, ay, az);
  project_point(dval, ax, ay, az, vp.t[0], vp.t[1], vp.t[2], sm.px, sm.py, sm.zp);
  bilinear_taps(sm.px, sm.py, W, H, ctr, sm.tp);
  sm.w00 = (1.0f - sm.tp.fx) * (1.0f - sm.tp.fy);
  sm.w01 = sm.tp.fx * (1.0f - sm.tp.fy);
  sm.w10 = (1.0f - sm.tp.fx) * sm.tp.fy;
  sm.w11 = sm.tp.fx * sm.tp.fy;
  sm.mk = sm.zp > 0.0f ? 1.0f : 0.0f;
}

__device__ __forceinline__ float gather4(const float* __restrict__ q, int W, const Sample& sm) {
  float v = 0.f;
  if (sm.tp.valid & 1u) v = sm.w00 * __ldg(q);
  if (sm.tp.valid & 2u) v = fmaf(sm.w01, __ldg(q + 1), v);
  if (sm.tp.valid & 4u) v = fmaf(sm.w10, __ldg(q + W), v);
  if (sm.tp.valid & 8u) v = fmaf(sm.w11, __ldg(q + W + 1), v);
  return v;
}

template <bool PER_PIXEL, int NIF>
__global__ void __launch_bounds__(BNT, 1)
mlp_backward_kernel(srcv_shape s, BwdDims m, const float* __restrict__ cur,
                    const float* __restrict__ src, const ViewParams* __restrict__ views,
                    const FrameParams* __restrict__ frames, const float* __restrict__ planes,
                    const float* __restrict__ w1t, const float* __restrict__ b1,
                    const float* __restrict__ w2t, const float* __restrict__ b2,
                    const float* __restrict__ w2p, const float* __restrict__ w1p,
                    const float* __restrict__ w3, const float* __restrict__ gcost,
                    float* __restrict__ gcur, float* __restrict__ gsrc, float* __restrict__ gw1,
                    float* __restrict__ gb1, float* __restrict__ gw2, float* __restrict__ gb2,
                    float* __restrict__ gw3, float* __restrict__ gb3) {
  SRCV_DYNAMIC_SMEM_ALIGNED(float, smem, 16);
  constexpr int Fp = 16 * NIF;
  float* sX = smem;               // [Fp][BTP]  metadata tile X, later dL/dX
  float* sH1 = sX + Fp * BTP;     // [BN][BTP]  H1
  float* sG = sH1 + BN * BTP;     // [BN][BTP]  G2, later G1
  float* sW = sG + BN * BTP;      // [2][BKC * BFMAX] streamed weight chunks
  float* sGo = sW + 2 * BKC * BFMAX;  // [BT] upstream gradient of the tile's rows
  float* sRed = sGo + BT;         // [BN + 1] dW3 partials, db3
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int HW = s.H * s.W, K = s.K, C = s.C;
  const int o_cur = K * C, o_mask = o_cur + C, o_z = o_mask + K, o_depth = o_z + K,
            o_dot = o_depth + 1, o_ang = o_dot + K, o_ncur = o_ang + K, o_nsrc = o_ncur + 3,
            o_comb = o_nsrc + 3 * K, o_r = o_comb + K, o_t = o_r + K;
  const Centre ctr(s.W, s.H);
  const int tiles_per_plane = (HW + BT - 1) / BT;
  const long long n_tiles = (long long)s.B * s.D * tiles_per_plane;

  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int tin = (int)(tile % tiles_per_plane);
    const long long bd = tile / tiles_per_plane;
    const int d = (int)(bd % s.D), b = (int)(bd / s.D);
    const int p0 = tin * BT;
    const FrameParams fp = frames[b];

    if (tid < BT) sGo[tid] = (p0 + tid < HW) ? __ldg(gcost + ((size_t)b * s.D + d) * HW + p0 + tid) : 0.f;
    if (tid <= BN) sRed[tid] = 0.f;

    // ---------------- 1. metadata tile (as the forward kernels build it) ---------------
    for (int it = tid; it < BT * K; it += BNT) {
      const int r = it % BT, k = it / BT;
      const int p = min(p0 + r, HW - 1);
      const float pxc = (float)(p % s.W) + 0.5f, pyc = (float)(p / s.W) + 0.5f;
      const float dval = PER_PIXEL ? __ldg(planes + ((size_t)b * s.D + d) * HW + p)
                                   : __ldg(planes + b * s.D + d);
      const ViewParams& vp = views[b * K + k];
      Sample sm;
      project_sample(vp, ctr, s.W, s.H, pxc, pyc, dval, sm);
      const float* sp = src + ((size_t)(b * K + k) * C) * HW + (sm.tp.y0 * s.W + sm.tp.x0);
      const float* cp = cur + (size_t)b * C * HW + p;
      float dot = 0.f;
      for (int c = 0; c < C; ++c) {
        const float v = gather4(sp + (size_t)c * HW, s.W, sm);
        sX[(k * C + c) * BTP + r] = v;
        dot = fmaf(v, __ldg(cp + (size_t)c * HW), dot);
      }
      sX[(o_mask + k) * BTP + r] = sm.mk;
      sX[(o_z + k) * BTP + r] = sm.zp;
      sX[(o_dot + k) * BTP + r] = dot * sm.mk;
      const float rx = fmaf(fp.invK[0], pxc, fmaf(fp.invK[1], pyc, fp.invK[2]));
      const float ry = fmaf(fp.invK[3], pxc, fmaf(fp.invK[4], pyc, fp.invK[5]));
      const float rz = fmaf(fp.invK[6], pxc, fmaf(fp.invK[7], pyc, fp.invK[8]));
      const float X = dval * rx, Y = dval * ry, Z = dval * rz;
      const float nc = fmaxf(sqrtf(fmaf(X, X, fmaf(Y, Y, Z * Z))), kEpsNorm);
      const float cx = X / nc, cy = Y / nc, cz = Z / nc;
      const float sx0 = X - vp.centre[0], sy0 = Y - vp.centre[1], sz0 = Z - vp.centre[2];
      const float ns = fmaxf(sqrtf(fmaf(sx0, sx0, fmaf(sy0, sy0, sz0 * sz0))), kEpsNorm);
      const float sx = sx0 / ns, sy = sy0 / ns, sz = sz0 / ns;
      const float n1 = fmaxf(sqrtf(fmaf(cx, cx, fmaf(cy, cy, cz * cz))), kEpsCos);
      const float n2 = fmaxf(sqrtf(fmaf(sx, sx, fmaf(sy, sy, sz * sz))), kEpsCos);
      sX[(o_ang + k) * BTP + r] = fmaf(cx / n1, sx / n2, fmaf(cy / n1, sy / n2, (cz / n1) * (sz / n2)));
      sX[(o_nsrc + 3 * k + 0) * BTP + r] = sx;
      sX[(o_nsrc + 3 * k + 1) * BTP + r] = sy;
      sX[(o_nsrc + 3 * k + 2) * BTP + r] = sz;
      sX[(o_comb + k) * BTP + r] = vp.comb;
      sX[(o_r + k) * BTP + r] = vp.rmeas;
      sX[(o_t + k) * BTP + r] = vp.tmeas;
      if (k == 0) {
        for (int c = 0; c < C; ++c) sX[(o_cur + c) * BTP + r] = __ldg(cp + (size_t)c * HW);
        sX[o_depth * BTP + r] = dval;
        sX[(o_ncur + 0) * BTP + r] = cx;
        sX[(o_ncur + 1) * BTP + r] = cy;
        sX[(o_ncur + 2) * BTP + r] = cz;
        for (int f = m.F; f < Fp; ++f) sX[f * BTP + r] = 0.f;
      }
    }
    __syncthreads();

    // ---------------- 2. forward recompute -----------------------------------------------
    float acc[4][8];
#pragma unroll
    for (int ii = 0; ii < 4; ++ii)
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[ii][i] = 0.f;
    gemm_rows<8>(acc, sX, sW, w1t, Fp);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int n = gemm_col<8>(i, tx);
      const float bias = n < m.H1 ? __ldg(b1 + n) : 0.f;
      *reinterpret_cast<float4*>(sH1 + n * BTP + 4 * ty) =
          make_float4(leaky(acc[0][i] + bias), leaky(acc[1][i] + bias), leaky(acc[2][i] + bias),
                      leaky(acc[3][i] + bias));
    }
#pragma unroll
    for (int ii = 0; ii < 4; ++ii)
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[ii][i] = 0.f;
    __syncthreads();
    gemm_rows<8>(acc, sH1, sW, w2t, BN);

    // ---------------- 3. G2 = g w3 lrelu'(A2);  dW3, db3 ------------------------------------
    {
      const float4 g = *reinterpret_cast<const float4*>(sGo + 4 * ty);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int n = gemm_col<8>(i, tx);
        const bool live = n < m.H2;
        const float bias = live ? __ldg(b2 + n) : 0.f, w = live ? __ldg(w3 + n) : 0.f;
        const float a0 = acc[0][i] + bias, a1 = acc[1][i] + bias, a2 = acc[2][i] + bias, a3 = acc[3][i] + bias;
        const float part = fmaf(g.x, leaky(a0), fmaf(g.y, leaky(a1), fmaf(g.z, leaky(a2), g.w * leaky(a3))));
        if (live && part != 0.f) atomicAdd(&sRed[n], part);
        *reinterpret_cast<float4*>(sG + n * BTP + 4 * ty) =
            make_float4(g.x * w * (a0 > 0.f ? 1.f : kLeaky), g.y * w * (a1 > 0.f ? 1.f : kLeaky),
                        g.z * w * (a2 > 0.f ? 1.f : kLeaky), g.w * w * (a3 > 0.f ? 1.f : kLeaky));
      }
      if (tid < BT && sGo[tid] != 0.f) atomicAdd(&sRed[BN], sGo[tid]);
    }
    __syncthreads();
    if (tid < m.H2) {
      if (sRed[tid] != 0.f) atomicAdd(gw3 + tid, sRed[tid]);
      float v = 0.f;
      for (int r = 0; r < BT; ++r) v += sG[tid * BTP + r];
      if (v != 0.f) atomicAdd(gb2 + tid, v);
    }
    if (tid == BN && sRed[BN] != 0.f) atomicAdd(gb3, sRed[BN]);
    grad_outer<8>(sG, sH1, gw2, m.H1, m.H2, m.H1);            // dW2[n2][n1] += G2^T H1
    __syncthreads();

    // ---------------- 4. G1 = (G2 W2) lrelu'(A1);  db1, dW1 --------------------------------
#pragma unroll
    for (int ii = 0; ii < 4; ++ii)
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[ii][i] = 0.f;
    gemm_rows<8>(acc, sG, sW, w2p, BN);                         // k = n2, columns = n1
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int n = gemm_col<8>(i, tx);
      const float4 h = *reinterpret_cast<const float4*>(sH1 + n * BTP + 4 * ty);
      *reinterpret_cast<float4*>(sG + n * BTP + 4 * ty) =
          make_float4(acc[0][i] * (h.x > 0.f ? 1.f : kLeaky), acc[1][i] * (h.y > 0.f ? 1.f : kLeaky),
                      acc[2][i] * (h.z > 0.f ? 1.f : kLeaky), acc[3][i] * (h.w > 0.f ? 1.f : kLeaky));
    }
    __syncthreads();
    if (tid < m.H1) {
      float v = 0.f;
      for (int r = 0; r < BT; ++r) v += sG[tid * BTP + r];
      if (v != 0.f) atomicAdd(gb1 + tid, v);
    }
    grad_outer<NIF>(sG, sX, gw1, m.F, m.H1, m.F);              // dW1[n1][f] += G1^T X
    __syncthreads();                                            // X is dead from here on

    // ---------------- 5. dX = G1 W1, then scatter to the features --------------------------
    {
      float ax[4][NIF];
#pragma unroll
      for (int ii = 0; ii < 4; ++ii)
#pragma unroll
        for (int i = 0; i < NIF; ++i) ax[ii][i] = 0.f;
      gemm_rows<NIF>(ax, sG, sW, w1p, BN);                      // k = n1, columns = f
#pragma unroll
      for (int i = 0; i < NIF; ++i)
        *reinterpret_cast<float4*>(sX + gemm_col<NIF>(i, tx) * BTP + 4 * ty) =
            make_float4(ax[0][i], ax[1][i], ax[2][i], ax[3][i]);
    }
    __syncthreads();
    for (int it = tid; it < BT * K; it += BNT) {
      const int r = it % BT, k = it / BT;
      const int p = p0 + r;
      if (p >= HW) continue;
      const float pxc = (float)(p % s.W) + 0.5f, pyc = (float)(p / s.W) + 0.5f;
      const float dval = PER_PIXEL ? __ldg(planes + ((size_t)b * s.D + d) * HW + p)
                                   : __ldg(planes + b * s.D + d);
      Sample sm;
      project_sample(views[b * K + k], ctr, s.W, s.H, pxc, pyc, dval, sm);
      const size_t off = ((size_t)(b * K + k) * C) * HW + (sm.tp.y0 * s.W + sm.tp.x0);
      const float* cp = cur + (size_t)b * C * HW + p;
      const float gdot = sm.mk * sX[(o_dot + k) * BTP + r];     // dL/d(dot_k) through the mask
      for (int c = 0; c < C; ++c) {
        // dL/dwarped_kc = direct channel + via the dot product (:691-695)
        const float gw = fmaf(gdot, __ldg(cp + (size_t)c * HW), sX[(k * C + c) * BTP + r]);
        if (gw != 0.f) {
          float* q = gsrc + off + (size_t)c * HW;
          if (sm.tp.valid & 1u) atomicAdd(q, sm.w00 * gw);
          if (sm.tp.valid & 2u) atomicAdd(q + 1, sm.w01 * gw);
          if (sm.tp.valid & 4u) atomicAdd(q + s.W, sm.w10 * gw);
          if (sm.tp.valid & 8u) atomicAdd(q + s.W + 1, sm.w11 * gw);
        }
        if (gdot != 0.f) {
          const float v = gather4(src + off + (size_t)c * HW, s.W, sm);
          atomicAdd(&sX[(o_cur + c) * BTP + r], gdot * v);      // dL/dcur via the dot product
        }
      }
    }
    __syncthreads();
    for (int it = tid; it < BT * C; it += BNT) {
      const int r = it % BT, c = it / BT;
      const float v = sX[(o_cur + c) * BTP + r];
      if (p0 + r < HW && v != 0.f) atomicAdd(gcur + ((size_t)b * C + c) * HW + p0 + r, v);
    }
    __syncthreads();   // the next tile rewrites every shared buffer
  }
}

size_t bwd_smem_bytes(int Fp) {
  return sizeof(float) * ((size_t)(Fp + 2 * BN) * BTP + 2 * BKC * BFMAX + BT + BN + 1 + 3);
}

BwdDims make_bwd_dims(const srcv_shape& s, const srcv_mlp_weights& w) {
  BwdDims m;
  m.F = s.C * (s.K + 1) + 10 * s.K + 4;
  m.Fp = padded_features(m.F);
  m.H1 = w.hidden1;
  m.H2 = w.hidden2;
  return m;
}

}  // namespace

bool mlp_backward_supported(const srcv_shape& s, const srcv_mlp_weights& w) {
  const int F = s.C * (s.K + 1) + 10 * s.K + 4;
  return F <= BFMAX && w.hidden1 >= 1 && w.hidden1 <= BN && w.hidden2 >= 1 && w.hidden2 <= BN;
}

size_t mlp_backward_extra_bytes(const srcv_shape& s, const srcv_mlp_weights& w) {
  const BwdDims m = make_bwd_dims(s, w);
  return sizeof(float) * (2 * (size_t)m.Fp * BN + 2 * (size_t)BN * BN);
}

template <bool PP, int NIF>
static cudaError_t launch_bwd_sized(const srcv_shape& s, const BwdDims& m, int grid, size_t smem,
                                    cudaStream_t stream, const float* cur, const float* src,
                                    const Workspace& ws, const float* planes, const float* w1t,
                                    const float* w2t, const float* w2p, const float* w1p,
                                    const srcv_mlp_weights& w, const float* gcost, float* gcur,
                                    float* gsrc, const srcv_mlp_grads& g) {
  cudaError_t err = cudaFuncSetAttribute(mlp_backward_kernel<PP, NIF>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (err != cudaSuccess) return err;
  SRCV_LAUNCH((mlp_backward_kernel<PP, NIF>), grid, BNT, smem, stream, s, m, cur, src, ws.views, ws.frames, planes,
              w1t, w.b1, w2t, w.b2, w2p, w1p, w.w3, gcost, gcur, gsrc, g.w1, g.b1, g.w2, g.b2, g.w3, g.b3);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_mlp_backward(const srcv_shape& s, const float* cur, const float* src,
                                const Workspace& ws, const float* planes, bool per_pixel,
                                const srcv_mlp_weights& w, const float* gcost, float* gcur,
                                float* gsrc, const srcv_mlp_grads& g, cudaStream_t stream) {
  const BwdDims m = make_bwd_dims(s, w);
  float* w1t = ws.extra;
  float* w2t = w1t + (size_t)m.Fp * BN;
  float* w2p = w2t + (size_t)BN * BN;
  float* w1p = w2p + (size_t)BN * BN;
  SRCV_LAUNCH(mlp_bwd_pack_kernel, 64, 256, 0, stream, w.w1, w.w2, m, w1t, w2t, w2p, w1p);
  note_launch();
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return err;
  int dev = 0, sms = 1;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long long n_tiles = (long long)s.B * s.D * ((s.H * s.W + BT - 1) / BT);
  const int grid = (int)(n_tiles < sms ? n_tiles : sms);     // one persistent CTA per SM
  const size_t smem = bwd_smem_bytes(m.Fp);
#define SRCV_BWD_CASE(PP, NIF) \
  return launch_bwd_sized<PP, NIF>(s, m, grid, smem, stream, cur, src, ws, planes, w1t, w2t, w2p, w1p, w, \
                                   gcost, gcur, gsrc, g)
  if (per_pixel) {
    if (m.Fp == 64) SRCV_BWD_CASE(true, 4);
    if (m.Fp == 128) SRCV_BWD_CASE(true, 8);
    SRCV_BWD_CASE(true, 13);
  }
  if (m.Fp == 64) SRCV_BWD_CASE(false, 4);
  if (m.Fp == 128) SRCV_BWD_CASE(false, 8);
  SRCV_BWD_CASE(false, 13);
#undef SRCV_BWD_CASE
}
}  // namespace srcv
