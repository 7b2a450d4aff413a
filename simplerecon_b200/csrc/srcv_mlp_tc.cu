// Metadata-MLP plane-sweep volume on the Hopper tensor cores (wgmma).
//
// Replaces FeatureVolumeManager / FastFeatureVolumeManager.build_cost_volume
// (reference modules/cost_volume.py:451-736, :967-1164) for the hero layout
// K = 7 source views, C = 16 channels, MLP 202 -> 128 -> 128 -> 1.
//
// One persistent CTA per SM walks over 64-row tiles (a 16 x 2 pixel patch at two consecutive planes):
//   * 8 BUILDER warps (four threads per row, two K blocks = one 48-wide K chunk each) project, gather,
//     blend, build the metadata channels and write the row's fp16 (hi, lo) layer-1 operand chunk by
//     chunk into a 5-slot ring of 12 KB chunks;
//   * 2 CONSUMER warpgroups take tiles in turn: layer 1 = 4 chunks x 3 x 3 wgmma m64n128k16 (A_hi W_hi
//     + A_hi W_lo + A_lo W_hi), one commit group per chunk, each chunk's ring slot handed back as soon
//     as its group retires; the layer-1 accumulator fragment, biased, LeakyReLU'd and split in
//     registers, IS the register A operand of layer 2 (8 x 3 wgmma m64n64k16 per 64-column half); the
//     128 -> 1 layer is a per-row dot product reduced over a quad.
// Stages are chained by mbarriers; weights (160 KB, K-major no-swizzle core matrices) stay resident in
// shared memory, pulled in once by the bulk-copy engine.
//
// The K order of layer 1 is OURS (the pack kernel permutes W1's columns to match), 8 blocks x 24:
//   per view k:  16 warped | mask | z' | dot | ray angle | n_src (3) | pad
//   tail:        16 reference features | plane depth | n_cur (3) | pad (4)
// The 21 pose measures (comb, r, t per view) are constant per (frame, view) and enter, with b1, as a
// per-frame bias vector instead of 21 K positions.
//
// Scaling: W1 and W2 are stored x16 (exact) so the lo halves of typical |w| ~ 0.05 weights
// stay out of the fp16 subnormals.  Layer 1 therefore yields 16 (W1 x + b1); LeakyReLU
// commutes with the positive scale, so the layer-2 operand is 16 a and its accumulator is
// 256 (W2 a): the single 1/256 is folded into the layer-2 bias FMA.
#include "srcv_kernels.h"
#include "srcv_tc.cuh"

namespace srcv {

namespace {

using namespace tc;

#ifndef SRCV_TC_REGS_BUILD
#define SRCV_TC_REGS_BUILD 104
#endif

constexpr int kC = 16, kViews = 7;
constexpr int kRows = 64;                // rows (M of one wgmma) per tile
// A tile is a 16 x 2 pixel patch at TWO consecutive depth planes (32 pixels x 2 planes = 64 rows):
// the builder warps of both planes gather along the same epipolar lines and share L1 lines.
constexpr int kTileW = 16, kTileH = 2, kTileD = 2;
constexpr int kN = 128;                  // layer widths
constexpr int kBlk = 24;                 // K positions per block (23 per view + 1 pad; tail 20 + 4 pad)
constexpr int kBlkCols = kBlk / 2;       // 12 packed columns per block and half
constexpr int kK1 = 192;                 // 8 blocks x 24  (12 k-steps of 16)
constexpr int kK2 = 128;
constexpr int kF = kC * (kViews + 1) + 10 * kViews + 4;  // 202

constexpr float kWScale = 16.0f;
constexpr float kUnscale2 = 1.0f / (kWScale * kWScale);

// Warps 0-7 build (slot = warp / 2), warps 8-15 are the two consumer warpgroups.  setmaxnreg moves
// registers from the builders to the consumers; it only REDISTRIBUTES the launch-time allocation
// (an .inc blocks until the pool holds enough), so the totals must fit.
constexpr int kBuildWarps = 8, kSlots = 4, kConsumers = 2;
constexpr int kThreads = (kBuildWarps + 4 * kConsumers) * 32;
constexpr int kBuilders = kBuildWarps * 32;
constexpr int kRegsLaunch = 65536 / kThreads, kRegsBuild = SRCV_TC_REGS_BUILD, kRegsCons = 2 * kRegsLaunch - kRegsBuild;
static_assert(kBuilders == kSlots * kRows, "one builder thread per (row, slot)");
static_assert(kBuilders * kRegsBuild + (kThreads - kBuilders) * kRegsCons <= kThreads * kRegsLaunch &&
              kRegsBuild % 8 == 0 && kRegsCons % 8 == 0 && kRegsCons <= 256, "setmaxnreg budget");

// shared memory image (bytes)
constexpr uint32_t kW1Bytes = kN * kK1 * 2, kW2Bytes = kN * kK2 * 2;   // one of (hi, lo)
constexpr uint32_t kOffW1Hi = 0, kOffW1Lo = kW1Bytes, kOffW2Hi = 2 * kW1Bytes,
                   kOffW2Lo = 2 * kW1Bytes + kW2Bytes, kOffVec = 2 * kW1Bytes + 2 * kW2Bytes;
constexpr uint32_t kVecFloats = 3 * kN + 4;   // b2 | 0.505 w3 | 0.495 w3 | b3
// image = [W1hi | W1lo | W2hi | W2lo | vec] exactly as it sits in shared memory
constexpr uint32_t kImageBytes = kOffVec + kVecFloats * 4;
// The layer-1 operand is built and consumed in K chunks: builder slot s writes K chunk s of a tile
// (its two K blocks, 48 K positions = 3 k-steps).  Chunk n of the CTA's chunk sequence (tile n / 4,
// chunk n % 4) lives in ring slot n % kRing: hi | lo, each kRows x 48 halves as K-major core matrices.
constexpr int kChunkSteps = kK1 / 16 / kSlots;                  // 3 k-steps per chunk
constexpr int kRing = 5;                                        // 6 slots do not fit next to the image
constexpr uint32_t kChunkLo = kRows * (kK1 / kSlots) * 2;       // 6 KB: offset of the lo half
constexpr uint32_t kChunkBytes = 2 * kChunkLo;
constexpr uint32_t kOffRing = (kImageBytes + 127) & ~127u;
constexpr uint32_t kOffBar = kOffRing + kRing * kChunkBytes;
constexpr uint32_t kOffFlag = kOffBar + 16 * 8;                 // 16 mbarrier slots (3 kRing + 1 used)
static_assert(3 * kRing + 1 <= 16, "mbarrier slots: full[kRing], free[kRing][2], image");
constexpr uint32_t kSmemBytes = kOffFlag + kRing * kRows;       // mask bits [ring slot][row]
static_assert(kSlots * kChunkSteps * 16 == kK1 && kBlkCols * 2 * 2 == kK1 / kSlots, "one chunk = two K blocks");
static_assert(kSmemBytes <= 227 * 1024, "shared-memory budget of one CTA");
// operand strides: one 8-wide K group of an A chunk / of a 128-row weight matrix
constexpr uint32_t kALbo = kRows * 16, kWLbo = kN * 16, kSbo = 128;

// K-major no-swizzle core-matrix offset (in halves) of element (n, k) of an N x Kp operand
__host__ __device__ inline uint32_t core_offset(int n, int k, int N) {
  return (uint32_t)(k >> 3) * (uint32_t)(N * 8) + (uint32_t)(n >> 3) * 64u + (uint32_t)(n & 7) * 8u + (uint32_t)(k & 7);
}

// reference channel index (modules/cost_volume.py:698-723 order) of OUR layer-1 K position;
// -1 = padding.  The 21 pose measures (comb, r, t per view) are NOT in K: they are constant per
// (frame, view), so their layer-1 contribution is a per-frame bias vector (tc_frame_bias_kernel).
__host__ __device__ inline int ref_channel(int kk) {
  if (kk < kViews * kBlk) {
    const int k = kk / kBlk, j = kk - k * kBlk;
    if (j < kC) return k * kC + j;                       // warped features
    const int base = kC * (kViews + 1);                  // 128
    switch (j - kC) {
      case 0: return base + k;                           // mask
      case 1: return base + kViews + k;                  // z'
      case 2: return base + 2 * kViews + 1 + k;          // dot
      case 3: return base + 3 * kViews + 1 + k;          // ray angle
      case 4: case 5: case 6: return base + 4 * kViews + 4 + 3 * k + (j - kC - 4);  // n_src
      default: return -1;                                // pad
    }
  }
  const int j = kk - kViews * kBlk;
  if (j < kC) return kViews * kC + j;                    // reference-frame features
  if (j == kC) return kC * (kViews + 1) + 2 * kViews;    // plane depth
  if (j < kC + 4) return kC * (kViews + 1) + 4 * kViews + 1 + (j - kC - 1);  // n_cur
  return -1;                                             // pad
}
// reference channels of the pose measures of view k: comb, r, t (:718-720)
__host__ __device__ inline int pose_channel(int which, int k) {
  return kC * (kViews + 1) + (7 + which) * kViews + 4 + k;
}

// Builds the shared-memory image from nn.Linear weights: fp16 (hi, lo) core matrices.
__global__ void __launch_bounds__(256)
tc_pack_kernel(srcv_mlp_weights w, uint8_t* __restrict__ image) {
  __half* w1hi = reinterpret_cast<__half*>(image + kOffW1Hi);
  __half* w1lo = reinterpret_cast<__half*>(image + kOffW1Lo);
  __half* w2hi = reinterpret_cast<__half*>(image + kOffW2Hi);
  __half* w2lo = reinterpret_cast<__half*>(image + kOffW2Lo);
  float* vec = reinterpret_cast<float*>(image + kOffVec);
  const int n1 = kN * kK1, n2 = kN * kK2;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n1 + n2 + (int)kVecFloats;
       i += gridDim.x * blockDim.x) {
    if (i < n1) {
      const int n = i / kK1, kk = i - n * kK1;
      const int f = ref_channel(kk);
      const float v = kWScale * (f >= 0 ? w.w1[(size_t)n * kF + f] : 0.f);
      const __half h = __float2half_rn(v);
      w1hi[core_offset(n, kk, kN)] = h;
      w1lo[core_offset(n, kk, kN)] = __float2half_rn(v - __half2float(h));
    } else if (i < n1 + n2) {
      const int q = i - n1, n = q / kK2, kk = q - n * kK2;
      const float v = kWScale * w.w2[(size_t)n * kK2 + kk];
      const __half h = __float2half_rn(v);
      w2hi[core_offset(n, kk, kN)] = h;
      w2lo[core_offset(n, kk, kN)] = __float2half_rn(v - __half2float(h));
    } else {
      // LeakyReLU(h) w3 = (0.505 w3) h + (0.495 w3) |h|  (slope 0.01): two FMAs per column
      const int q = i - n1 - n2;
      float v = 0.f;
      if (q < kN) v = w.b2[q];
      else if (q < 2 * kN) v = (0.5f * (1.0f + kLeaky)) * w.w3[q - kN];
      else if (q < 3 * kN) v = (0.5f * (1.0f - kLeaky)) * w.w3[q - 2 * kN];
      else if (q == 3 * kN) v = w.b3[0];
      vec[q] = v;
    }
  }
}

// pb[b][n] = 16 * ( b1[n] + sum_k ( W1[n, comb_k] comb(b,k) + W1[n, r_k] r(b,k) + W1[n, t_k] t(b,k) ) ): the
// layer-1 bias of frame b = b1 + the contribution of the 21 pose measures, fp64 accumulation.
__global__ void __launch_bounds__(kN)
tc_frame_bias_kernel(srcv_mlp_weights w, const ViewParams* __restrict__ views, float* __restrict__ pb) {
  const int b = blockIdx.x, n = threadIdx.x;
  double acc = 0.0;
  for (int k = 0; k < kViews; ++k) {
    const ViewParams& vp = views[b * kViews + k];
    acc += (double)w.w1[(size_t)n * kF + pose_channel(0, k)] * (double)vp.comb;
    acc += (double)w.w1[(size_t)n * kF + pose_channel(1, k)] * (double)vp.rmeas;
    acc += (double)w.w1[(size_t)n * kF + pose_channel(2, k)] * (double)vp.tmeas;
  }
  pb[(size_t)b * kN + n] = (float)((double)kWScale * (acc + (double)w.b1[n]));
}

// 12 packed columns of one K block -> its K chunk in the ring (hi and lo halves).  `a_row` points at
// the row's first core-matrix line of the chunk; column c (K 2c, 2c + 1) sits in K group c / 4, so a
// block (12 columns, starting at column 0 or 12 of the chunk) is three 16-byte stores per half.
__device__ __forceinline__ void store_block(uint8_t* a_row, uint32_t col, const uint32_t (&hi)[kBlkCols],
                                            const uint32_t (&lo)[kBlkCols]) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    uint8_t* p = a_row + ((col >> 2) + (uint32_t)i) * kALbo;
    *reinterpret_cast<uint4*>(p) = uint4{hi[4 * i], hi[4 * i + 1], hi[4 * i + 2], hi[4 * i + 3]};
    *reinterpret_cast<uint4*>(p + kChunkLo) = uint4{lo[4 * i], lo[4 * i + 1], lo[4 * i + 2], lo[4 * i + 3]};
  }
}

// What a worker thread keeps about the tile it builds the A operand for.
struct RowCtx {
  float dval, dxc, dyc;      // plane depth, centred pixel
  float X, Y, Z;             // back-projected point
  float cx, cy, cz;          // n_cur
  float4 cur4[4];            // reference-frame features of the pixel
  int b;                     // frame
  long long out;             // offset of the row's cost element, < 0 for rows outside the volume
  bool last_plane;           // the row's plane is D - 1 (the overall mask is taken there)
};

// The depth-invariant part of one (frame, view): four 16-byte loads (ViewParams is 128-byte
// aligned; the struct order a0 hx hy t | centre comb is what they read).
struct ViewRegs {
  float a0[3], hx[3], hy[3], t[3], centre[3];
};
__device__ __forceinline__ void load_view(const ViewParams* __restrict__ vp, ViewRegs& v) {
  const float4* p = reinterpret_cast<const float4*>(vp);
  const float4 a = __ldg(p), b = __ldg(p + 1), c = __ldg(p + 2), d = __ldg(p + 3);
  v.a0[0] = a.x; v.a0[1] = a.y; v.a0[2] = a.z; v.hx[0] = a.w;
  v.hx[1] = b.x; v.hx[2] = b.y; v.hy[0] = b.z; v.hy[1] = b.w;
  v.hy[2] = c.x; v.t[0] = c.y; v.t[1] = c.z; v.t[2] = c.w;
  v.centre[0] = d.x; v.centre[1] = d.y; v.centre[2] = d.z;
}

// One source view of one row: project, gather, metadata -> the 12 (hi, lo) column pairs of
// the K block.  HWC != 0: compile-time map size, every gather address is base + immediate.
// WANT_BITS (warp-uniform): also return the depth-valid / in-bounds bits of the overall mask.
template <int TW, int HWC>
__device__ __forceinline__ unsigned view_block(const RowCtx& rc, const ViewParams* __restrict__ vpp,
                                               const float4* __restrict__ view4, int Wrt, int H, int HWrt,
                                               const Centre& ctr, bool want_bits, uint32_t (&hi)[kBlkCols],
                                               uint32_t (&lo)[kBlkCols]) {
  const int W = TW ? TW : Wrt, HW = HWC ? HWC : HWrt;
  ViewRegs vr;
  load_view(vpp, vr);
  const float ax = fmaf(vr.hx[0], rc.dxc, fmaf(vr.hy[0], rc.dyc, vr.a0[0]));
  const float ay = fmaf(vr.hx[1], rc.dxc, fmaf(vr.hy[1], rc.dyc, vr.a0[1]));
  const float az = fmaf(vr.hx[2], rc.dxc, fmaf(vr.hy[2], rc.dyc, vr.a0[2]));
  float px, py, zp;
  project_point(rc.dval, ax, ay, az, vr.t[0], vr.t[1], vr.t[2], px, py, zp);
  // bilinear footprint.  Warp-uniform fast path: every lane's 2 x 2 footprint lies inside the
  // map (float compares: NaN / inf coordinates fail them and take the general path).
  const float x0f = floorf(px), y0f = floorf(py);
  const float fx = px - x0f, fy = py - y0f;
  const bool inside = x0f >= -(float)ctr.nx && x0f <= (float)(W - 2 - ctr.nx) &&
                      y0f >= -(float)ctr.ny && y0f <= (float)(H - 2 - ctr.ny);
  const bool interior = __all_sync(0xffffffffu, inside);
  const float gx = 1.0f - fx, gy = 1.0f - fy;
  float w00 = gx * gy, w01 = fx * gy, w10 = gx * fy, w11 = fx * fy;
  int o00, o01, o10, o11;
  if (interior) {
    o00 = ((int)y0f + ctr.ny) * W + ((int)x0f + ctr.nx);
    o01 = o00 + 1; o10 = o00 + W; o11 = o00 + W + 1;
  } else {
    // border patches, branch-free: every tap is loaded from an in-range (clamped) texel and
    // padding taps get a zero weight (zeros padding of grid_sample).
    Taps tp;
    bilinear_taps(px, py, W, H, ctr, tp);
    const int cxa = min(max(tp.x0, 0), W - 1), cxb = min(max(tp.x0 + 1, 0), W - 1);
    const int cya = min(max(tp.y0, 0), H - 1) * W, cyb = min(max(tp.y0 + 1, 0), H - 1) * W;
    o00 = cya + cxa; o01 = cya + cxb; o10 = cyb + cxa; o11 = cyb + cxb;
    w00 = (tp.valid & 1u) ? w00 : 0.f; w01 = (tp.valid & 2u) ? w01 : 0.f;
    w10 = (tp.valid & 4u) ? w10 : 0.f; w11 = (tp.valid & 8u) ? w11 : 0.f;
  }
  // features are sampled even for points behind the camera (only the dot is masked,
  // reference modules/cost_volume.py:590-623)
  // blend and dot on (even, odd) channel pairs
  float2 v2[kC / 2];
  {
    const float4 *q0 = view4 + o00, *q1 = view4 + o01, *q2 = view4 + o10, *q3 = view4 + o11;
    float4 f[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      f[0][j] = __ldg(q0 + (size_t)j * HW);
      f[1][j] = __ldg(q1 + (size_t)j * HW);
      f[2][j] = __ldg(q2 + (size_t)j * HW);
      f[3][j] = __ldg(q3 + (size_t)j * HW);
    }
    const float2 p00 = make_float2(w00, w00), p01 = make_float2(w01, w01), p10 = make_float2(w10, w10),
                 p11 = make_float2(w11, w11);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      v2[2 * j] = fma2(p11, make_float2(f[3][j].x, f[3][j].y), fma2(p10, make_float2(f[2][j].x, f[2][j].y),
                  fma2(p01, make_float2(f[1][j].x, f[1][j].y), mul2(p00, make_float2(f[0][j].x, f[0][j].y)))));
      v2[2 * j + 1] = fma2(p11, make_float2(f[3][j].z, f[3][j].w), fma2(p10, make_float2(f[2][j].z, f[2][j].w),
                      fma2(p01, make_float2(f[1][j].z, f[1][j].w), mul2(p00, make_float2(f[0][j].z, f[0][j].w)))));
    }
  }
  float2 d2 = make_float2(0.f, 0.f);       // even / odd channel partial sums
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    d2 = fma2(v2[2 * j], make_float2(rc.cur4[j].x, rc.cur4[j].y), d2);
    d2 = fma2(v2[2 * j + 1], make_float2(rc.cur4[j].z, rc.cur4[j].w), d2);
  }
  const float dot = d2.x + d2.y;
  const float mk = zp > 0.0f ? 1.0f : 0.0f;
  // n_src = (X - centre_k)/max(|.|, 1e-12) ; ray angle = cosine_similarity(n_cur, n_src, eps 1e-5)
  const float sx0 = rc.X - vr.centre[0], sy0 = rc.Y - vr.centre[1], sz0 = rc.Z - vr.centre[2];
  const float is = inv_norm(fmaf(sx0, sx0, fmaf(sy0, sy0, sz0 * sz0)), kEpsNorm);
  const float sx = sx0 * is, sy = sy0 * is, sz = sz0 * is;
  // cosine_similarity divides each operand by max(|.|, 1e-5) again (:683-688): both are unit vectors to
  // an ulp here (or exactly zero, which stays zero), so the plain dot product is the same to ~1e-7
  const float ang = fmaf(rc.cx, sx, fmaf(rc.cy, sy, rc.cz * sz));
#pragma unroll
  for (int i = 0; i < 8; ++i) split_pack(v2[i].x, v2[i].y, hi[i], lo[i]);
  split_pack(mk, zp, hi[8], lo[8]);
  split_pack(dot * mk, ang, hi[9], lo[9]);
  split_pack(sx, sy, hi[10], lo[10]);
  split_pack(sz, 0.0f, hi[11], lo[11]);
  unsigned bits = 0;
  if (want_bits) {
    if (zp > 0.0f) bits |= 1u;
    if (in_mask_bounds(px, py, W, H, ctr)) bits |= 2u;
  }
  return bits;
}

// The view-independent tail block: reference features | plane depth | n_cur | zeros
__device__ __forceinline__ void tail_block(const RowCtx& rc, uint32_t (&hi)[kBlkCols], uint32_t (&lo)[kBlkCols]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    split_pack(rc.cur4[j].x, rc.cur4[j].y, hi[2 * j], lo[2 * j]);
    split_pack(rc.cur4[j].z, rc.cur4[j].w, hi[2 * j + 1], lo[2 * j + 1]);
  }
  split_pack(rc.dval, rc.cx, hi[8], lo[8]);
  split_pack(rc.cy, rc.cz, hi[9], lo[9]);
#pragma unroll
  for (int j = 10; j < kBlkCols; ++j) hi[j] = lo[j] = 0u;
}

// tile id runs plane-chunk fastest, then pixel patch, then frame (32-bit: the launcher
// refuses >= 2^31 tiles); row -> (plane-in-chunk = row / 32, pixel of the 16 x 2 patch = row % 32)
// id / nd for the runtime plane-chunk count nd: multiply-high by ceil(2^32 / nd), exact while
// id * nd < 2^32 (the launcher refuses larger volumes) — 2 instructions instead of the ~20 of a
// generic 32-bit division, in every warp of every tile.
struct DivNd {
  unsigned nd, magic;
  __device__ __forceinline__ explicit DivNd(unsigned n) : nd(n), magic((unsigned)((0x100000000ull + n - 1) / n)) {}
  __device__ __forceinline__ unsigned div(unsigned id) const { return nd == 1u ? id : __umulhi(id, magic); }
};

template <bool PER_PIXEL>
__device__ __forceinline__ void make_row(unsigned id, int row, int W, int H, int HW, int D, const DivNd& nd,
                                         unsigned tiles_x, unsigned tiles_xy, const Centre& ctr,
                                         const float4* __restrict__ cur4g,
                                         const FrameParams* __restrict__ frames,
                                         const float* __restrict__ planes, RowCtx& rc) {
  const unsigned r = nd.div(id);
  const int d0 = (int)(id - r * nd.nd) * kTileD;
  const unsigned txy = r % tiles_xy;
  const int b = (int)(r / tiles_xy);
  const int x0 = (int)(txy % tiles_x) * kTileW, y0 = (int)(txy / tiles_x) * kTileH;
  const int rx = row & (kTileW - 1), ry = (row >> 4) & (kTileH - 1), dd = row >> 5;
  const int d = min(d0 + dd, D - 1);
  const bool active = (x0 + rx < W) && (y0 + ry < H) && (d0 + dd < D);
  const int ox = min(x0 + rx, W - 1), oy = min(y0 + ry, H - 1);
  const int p = oy * W + ox;
  rc.b = b;
  rc.out = active ? ((long long)b * D + d) * HW + p : -1;
  rc.last_plane = (d == D - 1);
  const float pxc = (float)ox + 0.5f, pyc = (float)oy + 0.5f;
  rc.dval = PER_PIXEL ? __ldg(planes + ((size_t)b * D + d) * HW + p) : __ldg(planes + b * D + d);
  rc.dxc = pxc - ctr.half_w;
  rc.dyc = pyc - ctr.half_h;
#pragma unroll
  for (int j = 0; j < 4; ++j) rc.cur4[j] = __ldg(cur4g + ((size_t)b * 4 + j) * HW + p);
  // rays: X = d * (invK3 p); n_cur = X / max(|X|, 1e-12)
  const float4* fp = reinterpret_cast<const float4*>(frames + b);
  const float4 k0 = __ldg(fp), k1 = __ldg(fp + 1);
  const float k8 = __ldg(reinterpret_cast<const float*>(fp + 2));
  const float rxv = fmaf(k0.x, pxc, fmaf(k0.y, pyc, k0.z));
  const float ryv = fmaf(k0.w, pxc, fmaf(k1.x, pyc, k1.y));
  const float rzv = fmaf(k1.z, pxc, fmaf(k1.w, pyc, k8));
  rc.X = rc.dval * rxv; rc.Y = rc.dval * ryv; rc.Z = rc.dval * rzv;
  const float ic = inv_norm(fmaf(rc.X, rc.X, fmaf(rc.Y, rc.Y, rc.Z * rc.Z)), kEpsNorm);
  rc.cx = rc.X * ic; rc.cy = rc.Y * ic; rc.cz = rc.Z * ic;
}

// K block `blk` (0..6: source view, 7: view-independent tail) of a row -> packed (hi, lo)
template <int TW, int HWC>
__device__ __forceinline__ unsigned build_block(const RowCtx& rc, int blk, const float4* __restrict__ src4,
                                                const ViewParams* __restrict__ views, int W, int H, int HW,
                                                const Centre& ctr, bool want_bits, uint32_t (&hi)[kBlkCols],
                                                uint32_t (&lo)[kBlkCols]) {
  if (blk < kViews)
    return view_block<TW, HWC>(rc, views + (rc.b * kViews + blk),
                               src4 + ((size_t)(rc.b * kViews + blk) * 4) * HW, W, H, HW, ctr, want_bits, hi, lo);
  tail_block(rc, hi, lo);
  return 0u;
}

// where the cost of tile row `row` goes: < 0 for rows outside the volume (integer part of make_row)
struct RowOut {
  long long out;
  bool last_plane;
};
__device__ __forceinline__ RowOut row_out(unsigned id, int row, int W, int H, int HW, int D, const DivNd& nd,
                                          unsigned tiles_x, unsigned tiles_xy) {
  const unsigned r = nd.div(id), txy = r % tiles_xy;
  const int d0 = (int)(id - r * nd.nd) * kTileD;
  const int b = (int)(r / tiles_xy);
  const int x0 = (int)(txy % tiles_x) * kTileW, y0 = (int)(txy / tiles_x) * kTileH;
  const int rx = row & (kTileW - 1), ry = (row >> 4) & (kTileH - 1), dd = row >> 5;
  const int d = d0 + dd;
  const bool active = (x0 + rx < W) && (y0 + ry < H) && (d < D);
  return RowOut{active ? ((long long)b * D + d) * HW + ((y0 + ry) * W + (x0 + rx)) : -1, d == D - 1};
}

template <bool PER_PIXEL, int TW, int TH>
__global__ void __launch_bounds__(kThreads, 1)
mlp_tc_kernel(srcv_shape s, const float4* __restrict__ cur4g, const float4* __restrict__ src4,
              const ViewParams* __restrict__ views, const FrameParams* __restrict__ frames,
              const float* __restrict__ planes, const uint8_t* __restrict__ image,
              const float* __restrict__ frame_bias, float* __restrict__ cost, uint8_t* __restrict__ mask_out,
              unsigned num_tiles) {
  SRCV_DYNAMIC_SMEM_ALIGNED(uint8_t, smem, 1024);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBar);
  // Chunk n = kSlots * it + s (tile it, K chunk s) goes to ring slot n % kRing in use u = n / kRing.
  //   full[slot]:       builder slot s has written chunk n (64 arrivals); completes once per use, the
  //                     consumer of chunk n waits with parity u & 1;
  //   free[slot][u & 1]: the MMAs that read chunk n have retired (128 arrivals); completes once every
  //                     OTHER use, the builder of chunk n + kRing waits with parity (u >> 1) & 1.
  // A parity wait is exact only while the barrier is neither two phases ahead of the waiter nor one
  // phase behind it (then the wait would return at once, on an older phase).
  //   * full: the consumer of chunk n has waited for chunk n - 1 (same tile) or finished its previous
  //     tile (s = 0); either way builder slot (n - kRing) % kSlots, which builds in tile order, has
  //     written chunk n - kRing, so full[slot] has completed use u - 1.  It cannot complete use u + 1
  //     before chunk n is released, which follows this wait.
  //   * free: the two consumer warpgroups release chunks out of order across a tile boundary (tile
  //     it's last chunk retires at its wait_group 0, while the other warpgroup may already release
  //     chunk 0 of tile it + 1), so one free barrier per slot could be one phase behind the builder of
  //     chunk n + kRing.  With a barrier per use parity, being behind means chunk n - 2 kRing is not yet
  //     released; but this builder saw chunk n - kRing + 1 released (its own previous chunk's wait),
  //     and every release chain from that chunk passes through the release of chunk n - 2 kRing.
  //     It cannot be two phases ahead: use u + 2 needs chunk n + kRing, which this builder writes.
  uint64_t* bar_full = bars;              // [kRing]     builders -> consumer
  uint64_t* bar_free = bars + kRing;      // [kRing][2]  consumer -> builders
  uint64_t* bar_img = bars + 3 * kRing;   // weight image landed in shared memory (bulk copies)
  uint8_t* sflag = smem + kOffFlag;   // mask bits of the rows of the chunk in ring slot r: [r][row]
  uint8_t* ring = smem + kOffRing;
  const float* svec = reinterpret_cast<const float*>(smem + kOffVec);

  // The warp index goes through a shuffle broadcast so that ptxas knows the role branches are
  // warp-uniform.
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  const int W = TW ? TW : s.W, H = TH ? TH : s.H, HW = W * H, D = s.D;
  constexpr int HWC = TW * TH;
  const unsigned tiles_x = (unsigned)(W + kTileW - 1) / kTileW;
  const unsigned tiles_xy = tiles_x * ((unsigned)(H + kTileH - 1) / kTileH);
  const DivNd nd((unsigned)(D + kTileD - 1) / kTileD);

  // ---- one-time setup ----------------------------------------------------------------
  if (tid == 0) {
    mbar_init(bar_img, 1);
    for (int r = 0; r < kRing; ++r) {
      mbar_init(bar_full + r, kBuilders / kSlots);
      mbar_init(bar_free + 2 * r, 128);
      mbar_init(bar_free + 2 * r + 1, 128);
    }
    mbar_fence_init();
  }
  __syncthreads();
  // The weight image (fp16 core matrices + biases) is pulled in by the bulk-copy (TMA) engine
  // straight into shared memory — written by the async proxy, which is also the proxy the tensor
  // core reads it through — while the threads finish their setup.
  if (tid == 0) {
    mbar_expect_tx(bar_img, kImageBytes);
    constexpr uint32_t kPiece = 32768;
    for (uint32_t off = 0; off < kImageBytes; off += kPiece)
      bulk_g2s(smem + off, image + off, (kImageBytes - off < kPiece) ? (kImageBytes - off) : kPiece, bar_img);
  }
  mbar_wait(bar_img, 0);
  // Work split: CTA c takes tiles c, c + grid, c + 2 grid, ... of the plane-fastest tile order, i.e.
  // at any moment the CTAs sweep a few neighbouring pixel blocks x all planes of ONE frame, whose
  // source features stay L2-resident, and every CTA sees the same mix of interior and border patches.
  const unsigned n_local = (num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x;
  auto tile_id = [&](unsigned j) { return blockIdx.x + j * gridDim.x; };

  if (warp < kBuildWarps) {
    // =============================== builders ============================================
    // Four threads per row (slot = warp / 2): views 2 slot, 2 slot + 1, i.e. K chunk `slot`; slot 3
    // builds view 6 and the view-independent tail.  The first block of a chunk is built before the
    // wait for its ring slot, so its gathers overlap the MMAs that still read the slot.
    reg_dec<kRegsBuild>();
    const int row = (warp & 1) * 32 + lane, slot = warp >> 1;
    const Centre ctr(W, H);
    const int blk_first = 2 * slot;
    const bool masks = mask_out != nullptr;
    uint8_t* a_row = ring + (uint32_t)(row >> 3) * kSbo + (uint32_t)(row & 7) * 16u;
    RowCtx rc;
    uint32_t hi[kBlkCols], lo[kBlkCols];
    for (unsigned it = 0; it < n_local; ++it) {
      make_row<PER_PIXEL>(tile_id(it), row, W, H, HW, D, nd, tiles_x, tiles_xy, ctr, cur4g, frames, planes, rc);
      const bool wb = masks && rc.last_plane;
      unsigned bits = build_block<TW, HWC>(rc, blk_first, src4, views, W, H, HW, ctr, wb, hi, lo);
      const unsigned n = kSlots * it + (unsigned)slot, rs = n % kRing;
      if (n >= (unsigned)kRing) {                  // chunk n - kRing is out of the slot
        const unsigned v = n / kRing - 1u;
        mbar_wait(bar_free + 2 * rs + (v & 1u), (v >> 1) & 1u);
      }
      uint8_t* a_chunk = a_row + rs * kChunkBytes;
      store_block(a_chunk, 0u, hi, lo);
      bits |= build_block<TW, HWC>(rc, blk_first + 1, src4, views, W, H, HW, ctr, wb, hi, lo);
      store_block(a_chunk, (uint32_t)kBlkCols, hi, lo);
      // the consumer reads the chunk's mask bits before it frees the ring slot
      sflag[rs * kRows + row] = (uint8_t)bits;
      fence_proxy_async_smem();                    // generic-proxy stores -> visible to wgmma
      mbar_arrive(bar_full + rs);
    }
  } else {
    // =============================== consumers ===========================================
    reg_inc<kRegsCons>();
    const int c = (warp - kBuildWarps) >> 2, wl = (warp - kBuildWarps) & 3;
    const int g = lane >> 2, q = lane & 3;
    const int r0 = 16 * wl + g, r1 = r0 + 8;       // the two tile rows of this thread's fragments
    const bool masks = mask_out != nullptr;
    // Descriptors differ between k-steps only in the start-address field (address >> 4, far from
    // overflowing into the LBO field), so each one is a base descriptor + an immediate.
    const uint32_t sbase = smem_u32(smem);
    const uint64_t desc_ring = smem_desc(sbase + kOffRing, kALbo, kSbo);
    const uint64_t desc_w1 = smem_desc(sbase + kOffW1Hi, kWLbo, kSbo);
    const uint64_t desc_w2 = smem_desc(sbase + kOffW2Hi, kWLbo, kSbo);
    auto release = [&](unsigned n) { mbar_arrive(bar_free + 2 * (n % kRing) + ((n / kRing) & 1u)); };
    for (unsigned it = (unsigned)c; it < n_local; it += kConsumers) {
      // ---- layer 1: D1 = 16 (W1 x) over 12 k-steps, three products each, one commit group per
      // K chunk; a chunk's ring slot is released as soon as the group that reads it has retired
      float d1[64];
      unsigned bits0 = 0, bits1 = 0;
      wgmma_fence();
#pragma unroll
      for (int ch = 0; ch < kSlots; ++ch) {
        const unsigned n = kSlots * it + (unsigned)ch, rs = n % kRing;
        mbar_wait(bar_full + rs, (n / kRing) & 1u);
        if (masks) {
          bits0 |= sflag[rs * kRows + r0];
          bits1 |= sflag[rs * kRows + r1];
        }
        const uint64_t da = desc_ring + rs * (kChunkBytes >> 4);
#pragma unroll
        for (int i = 0; i < kChunkSteps; ++i) {
          const int ks = kChunkSteps * ch + i;
          const uint64_t ahi = da + ((uint32_t)i * 2 * kALbo >> 4), alo = ahi + (kChunkLo >> 4);
          const uint64_t bhi = desc_w1 + ((uint32_t)ks * 2 * kWLbo >> 4), blo = bhi + (kW1Bytes >> 4);
          wgmma_ss_n128(d1, ahi, bhi, ks > 0 ? 1u : 0u);
          wgmma_ss_n128(d1, ahi, blo, 1u);
          wgmma_ss_n128(d1, alo, bhi, 1u);
        }
        wgmma_commit();
        if (ch > 0) {
          wgmma_wait<1>();                         // the previous chunk's group has retired
          release(n - 1u);
        }
      }
      wgmma_wait<0>();
      fence_regs(d1);
      release(kSlots * it + kSlots - 1u);
      const unsigned id = tile_id(it);
      const int b = (int)(nd.div(id) / tiles_xy);
      // ---- layer-1 epilogue: + frame bias, LeakyReLU, (hi, lo) split into the layer-2 A fragments
      uint32_t a2hi[kK2 / 16][4], a2lo[kK2 / 16][4];
      const float* pb = frame_bias + (size_t)b * kN + 2 * q;
#pragma unroll
      for (int j = 0; j < kN / 8; ++j) {
        const float2 bb = __ldg(reinterpret_cast<const float2*>(pb + 8 * j));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float x0 = leaky(d1[4 * j + 2 * h] + bb.x), x1 = leaky(d1[4 * j + 2 * h + 1] + bb.y);
          split_pack(x0, x1, a2hi[j >> 1][2 * (j & 1) + h], a2lo[j >> 1][2 * (j & 1) + h]);
        }
      }
      // ---- layer 2 in two 64-column halves, each followed by its share of the 128 -> 1 layer
      float acc0 = 0.f, acc1 = 0.f;                // rows r0, r1
#pragma unroll 1
      for (int nh = 0; nh < 2; ++nh) {
        float d2[32];
        wgmma_fence();
#pragma unroll
        const uint64_t dh = desc_w2 + ((uint32_t)nh * (kN / 2) * 16 >> 4);
#pragma unroll
        for (int ks = 0; ks < kK2 / 16; ++ks) {
          const uint64_t bhi = dh + ((uint32_t)ks * 2 * kWLbo >> 4), blo = bhi + (kW2Bytes >> 4);
          wgmma_rs_n64(d2, a2hi[ks], bhi, ks > 0 ? 1u : 0u);
          wgmma_rs_n64(d2, a2hi[ks], blo, 1u);
          wgmma_rs_n64(d2, a2lo[ks], bhi, 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(d2);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int n = nh * (kN / 2) + 8 * j + 2 * q;
          // columns n, n + 1 of b2 | 0.505 w3 | 0.495 w3
          const float2 b2 = *reinterpret_cast<const float2*>(svec + n);
          const float2 wp = *reinterpret_cast<const float2*>(svec + kN + n);
          const float2 wa = *reinterpret_cast<const float2*>(svec + 2 * kN + n);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float hv = fmaf(d2[4 * j + e], kUnscale2, (e & 1) ? b2.y : b2.x);
            const float t = fmaf((e & 1) ? wa.y : wa.x, fabsf(hv), ((e & 1) ? wp.y : wp.x) * hv);
            if (e < 2) acc0 += t; else acc1 += t;
          }
        }
      }
      // the four threads of a quad hold the four column subsets of the same two rows
      acc0 += __shfl_xor_sync(0xffffffffu, acc0, 1);
      acc1 += __shfl_xor_sync(0xffffffffu, acc1, 1);
      acc0 += __shfl_xor_sync(0xffffffffu, acc0, 2);
      acc1 += __shfl_xor_sync(0xffffffffu, acc1, 2);
      if (q == 0) {
        // where the two rows go is recomputed here rather than held in registers across the MMAs
        const RowOut o0 = row_out(id, r0, W, H, HW, D, nd, tiles_x, tiles_xy);
        const RowOut o1 = row_out(id, r1, W, H, HW, D, nd, tiles_x, tiles_xy);
        const float b3 = svec[3 * kN];
        // overall mask of the LAST plane (reference :625-637): any view in front AND any view
        // inside the 2-pixel border, independently
        if (o0.out >= 0) {
          cost[o0.out] = acc0 + b3;
          if (masks && o0.last_plane)
            mask_out[(size_t)b * HW + (o0.out - ((long long)b * D + (D - 1)) * HW)] = (bits0 == 3u) ? 1 : 0;
        }
        if (o1.out >= 0) {
          cost[o1.out] = acc1 + b3;
          if (masks && o1.last_plane)
            mask_out[(size_t)b * HW + (o1.out - ((long long)b * D + (D - 1)) * HW)] = (bits1 == 3u) ? 1 : 0;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// self-test: D[128,128] = A[128,Kp] W[128,Kp]^T through the same descriptors and (hi, lo) split as
// layer 1 of the sweep (A split and written to shared memory by the threads, W packed to core
// matrices), one 64-row half after the other.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
tc_selftest_pack(const float* __restrict__ Wm, int Kp, __half* __restrict__ hi, __half* __restrict__ lo) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kN * Kp; i += gridDim.x * blockDim.x) {
    const int n = i / Kp, k = i - n * Kp;
    const float v = Wm[i];
    const __half h = __float2half_rn(v);
    hi[core_offset(n, k, kN)] = h;
    lo[core_offset(n, k, kN)] = __float2half_rn(v - __half2float(h));
  }
}

__global__ void __launch_bounds__(128, 1)
tc_selftest_kernel(const float* __restrict__ A, const __half* __restrict__ whi,
                   const __half* __restrict__ wlo, int Kp, float* __restrict__ Dout) {
  SRCV_DYNAMIC_SMEM_ALIGNED(uint8_t, smem, 1024);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
  const uint32_t wbytes = (uint32_t)kN * Kp * 2, abytes = (uint32_t)kRows * Kp * 2;
  uint8_t* sa = smem + 2 * wbytes;
  for (uint32_t i = tid; i < wbytes / 16; i += blockDim.x) {
    reinterpret_cast<uint4*>(smem)[i] = __ldg(reinterpret_cast<const uint4*>(whi) + i);
    reinterpret_cast<uint4*>(smem + wbytes)[i] = __ldg(reinterpret_cast<const uint4*>(wlo) + i);
  }
  const uint32_t sb = smem_u32(smem), lbo_w = kN * 16, lbo_a = kRows * 16;
  for (int mh = 0; mh < 2; ++mh) {
    for (int i = tid; i < kRows * Kp / 2; i += blockDim.x) {
      const int r = i / (Kp / 2), cc = i - r * (Kp / 2);
      const float* a = A + (size_t)(kRows * mh + r) * Kp + 2 * cc;
      uint32_t h, l;
      split_pack(a[0], a[1], h, l);
      const uint32_t off = 2 * core_offset(r, 2 * cc, kRows);
      *reinterpret_cast<uint32_t*>(sa + off) = h;
      *reinterpret_cast<uint32_t*>(sa + abytes + off) = l;
    }
    fence_proxy_async_smem();
    __syncthreads();
    float d[64];
    wgmma_fence();
    for (int ks = 0; ks < Kp / 16; ++ks) {
      const uint32_t ahi = sb + 2 * wbytes + ks * 2 * lbo_a, bhi = sb + ks * 2 * lbo_w;
      wgmma_ss_n128(d, smem_desc(ahi, lbo_a, kSbo), smem_desc(bhi, lbo_w, kSbo), ks > 0 ? 1u : 0u);
      wgmma_ss_n128(d, smem_desc(ahi, lbo_a, kSbo), smem_desc(bhi + wbytes, lbo_w, kSbo), 1u);
      wgmma_ss_n128(d, smem_desc(ahi + abytes, lbo_a, kSbo), smem_desc(bhi, lbo_w, kSbo), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs(d);
#pragma unroll
    for (int j = 0; j < kN / 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e)
        Dout[(size_t)(kRows * mh + 16 * warp + g + 8 * (e >> 1)) * kN + 8 * j + 2 * q + (e & 1)] = d[4 * j + e];
    __syncthreads();                               // every MMA has read the A tile before it is rewritten
  }
}

}  // namespace

bool mlp_tc_supported(const srcv_shape& s, const srcv_mlp_weights& w) {
  return s.K == kViews && s.C == kC && w.hidden1 == kN && w.hidden2 == kN &&
         (long long)s.H * s.W < (1ll << 26);
}

static size_t image_bytes_aligned() { return (kImageBytes + 255) & ~(size_t)255; }
// workspace tail of the tensor-core variant: [weight image | per-frame layer-1 bias (B x 128 floats)]
size_t mlp_tc_extra_bytes(const srcv_shape& s) { return image_bytes_aligned() + (((size_t)s.B * kN * 4 + 255) & ~(size_t)255); }
size_t mlp_tc_image_bytes() { return kImageBytes; }

cudaError_t launch_mlp_tc_pack(const srcv_mlp_weights& w, void* image, cudaStream_t stream) {
  SRCV_LAUNCH(tc_pack_kernel, 64, 256, 0, stream, w, reinterpret_cast<uint8_t*>(image));
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_mlp_tc(const srcv_shape& s, const float* cur, const Workspace& ws,
                          const float* planes, bool per_pixel, const srcv_mlp_weights& w, float* cost,
                          float* lowest, uint8_t* mask, cudaStream_t stream) {
  // the caller may hand over an image packed earlier (srcv_mlp_pack_weights): nothing to do per call
  const uint8_t* image = reinterpret_cast<const uint8_t*>(w.packed_image);
  cudaError_t err = cudaSuccess;
  if (image == nullptr) {
    err = launch_mlp_tc_pack(w, ws.extra, stream);
    if (err != cudaSuccess) return err;
    image = reinterpret_cast<const uint8_t*>(ws.extra);
  }
  // b1 and the 21 pose measures enter layer 1 as a per-frame bias (views were written by the prep pass)
  float* frame_bias = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ws.extra) + image_bytes_aligned());
  SRCV_LAUNCH(tc_frame_bias_kernel, s.B, kN, 0, stream, w, ws.views, frame_bias);
  note_launch();
  int dev = 0, sms = 1;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int tiles_x = (s.W + kTileW - 1) / kTileW, tiles_y = (s.H + kTileH - 1) / kTileH;
  const long long num_tiles = (long long)s.B * ((s.D + kTileD - 1) / kTileD) * tiles_x * tiles_y;
  // tile ids are 32-bit, and the kernel's multiply-high division by the plane-chunk count is exact below 2^32 / nd
  if (num_tiles >= (1ll << 31) || num_tiles * ((s.D + kTileD - 1) / kTileD) >= (1ll << 32)) return cudaErrorInvalidValue;
  const int grid = (int)(num_tiles < sms ? num_tiles : sms);
  const float4* src4 = reinterpret_cast<const float4*>(ws.src_c4);
  const float4* cur4 = reinterpret_cast<const float4*>(ws.cur_c4);
  (void)cur;
#define SRCV_TC_LAUNCH(PP, TW_, TH_)                                                                  \
  do {                                                                                                \
    err = cudaFuncSetAttribute(mlp_tc_kernel<PP, TW_, TH_>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                               (int)kSmemBytes);                                                      \
    if (err != cudaSuccess) return err;                                                               \
    SRCV_LAUNCH((mlp_tc_kernel<PP, TW_, TH_>), grid, kThreads, kSmemBytes, stream,                    \
                s, cur4, src4, ws.views, ws.frames, planes, image, frame_bias, cost, mask,            \
                (unsigned)num_tiles);                                                                 \
  } while (0)
#define SRCV_TC_SIZES(PP)                                                   \
  if (s.W == 160 && s.H == 120) SRCV_TC_LAUNCH(PP, 160, 120);               \
  else if (s.W == 128 && s.H == 96) SRCV_TC_LAUNCH(PP, 128, 96);            \
  else SRCV_TC_LAUNCH(PP, 0, 0)
  if (per_pixel) { SRCV_TC_SIZES(true); } else { SRCV_TC_SIZES(false); }
#undef SRCV_TC_SIZES
#undef SRCV_TC_LAUNCH
  note_launch();
  err = cudaGetLastError();
  if (err != cudaSuccess) return err;
  if (lowest) err = launch_argmax(s, cost, planes, per_pixel, lowest, stream);
  return err;
}

// D (128 x 128) = A (128 x Kp) W^T (128 x Kp), Kp a multiple of 16 and <= 256; `scratch`
// needs 2 * 128 * Kp halves.  Device pointers; test hook for tests/test_gpu_tc.py.
cudaError_t launch_tc_selftest(const float* A, const float* Wm, int Kp, float* Dout, void* scratch,
                               cudaStream_t stream) {
  if (Kp % 16 != 0 || Kp <= 0 || Kp > 256) return cudaErrorInvalidValue;
  __half* hi = reinterpret_cast<__half*>(scratch);
  __half* lo = hi + (size_t)kN * Kp;
  SRCV_LAUNCH(tc_selftest_pack, 32, 256, 0, stream, Wm, Kp, hi, lo);
  note_launch();
  const size_t smem = (size_t)2 * (kN + kRows) * Kp * 2;
  cudaError_t err = cudaFuncSetAttribute(tc_selftest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (err != cudaSuccess) return err;
  SRCV_LAUNCH(tc_selftest_kernel, 1, 128, smem, stream, A, hi, lo, Kp, Dout);
  note_launch();
  return cudaGetLastError();
}

}  // namespace srcv
