// Prep pass: everything that is constant over the sweep, in ONE launch.
//
//  * per (frame, view): the plane-induced homography pieces Hm, t (see
//    srcv_common.cuh), the source camera centre, and the DVMVS pose measures
//    (reference utils/geometry_utils.py:178-191);
//  * per frame: invK[:3,:3] for the rays (utils/geometry_utils.py:56);
//  * plane depths  d_i = exp(log(min) + log(max/min) ramp_i)
//    (reference modules/cost_volume.py:124-127) when the caller gives a range;
//  * optionally the chunk-planar (B,K,C/4,H,W,4) copy of the source features that
//    the fast kernels gather from: a bilinear tap is C/4 16-byte vector loads and
//    horizontally adjacent pixels read adjacent vectors.
#include "srcv_kernels.h"
#include "srcv_tc.cuh"

namespace srcv {

namespace {

__device__ void view_params(const float* __restrict__ Kmat, const float* __restrict__ E,
                            const float* __restrict__ invK, const float* __restrict__ pose,
                            int W, int H, ViewParams* out) {
  // P = K @ E (rows 0..2) and Hm = P[:, :3] @ invK[:3, :3], fp64, rounded once at the end.
  double P[3][4], Hm[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      double a = 0.0;
#pragma unroll
      for (int l = 0; l < 4; ++l) a += (double)Kmat[i * 4 + l] * (double)E[l * 4 + j];
      P[i][j] = a;
    }
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      double a = 0.0;
#pragma unroll
      for (int l = 0; l < 3; ++l) a += P[i][l] * (double)invK[l * 4 + j];
      Hm[i][j] = a;
    }
  // centre the OUTPUT: c'_x = c_x - cxo c_z, c'_y = c_y - cyo c_z  (see srcv_common.cuh)
  const double cxo = (double)(W / 2) + 0.5, cyo = (double)(H / 2) + 0.5;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    Hm[0][j] -= cxo * Hm[2][j];
    Hm[1][j] -= cyo * Hm[2][j];
  }
  // The reference divides by z' = z + eps (utils/geometry_utils.py:83-87):
  //   x / z' - cxo = (x - cxo z - cxo eps) / z',
  // so the centred numerator also carries -cxo eps.  Irrelevant at metric depths (3e-6 px at
  // z = 0.25 m) but 5e-5 px at z = 1 mm: found by the fuzzer on the host emulation.
  const double tx = P[0][3] - cxo * P[2][3] - cxo * (double)kEpsProj,
               ty = P[1][3] - cyo * P[2][3] - cyo * (double)kEpsProj, tz = P[2][3];
  // centre the INPUT: p = (W/2 + dx, H/2 + dy, 1)
  const double ux = 0.5 * (double)W, uy = 0.5 * (double)H;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    out->a0[i] = (float)(Hm[i][0] * ux + Hm[i][1] * uy + Hm[i][2]);
    out->hx[i] = (float)Hm[i][0];
    out->hy[i] = (float)Hm[i][1];
  }
  out->t[0] = (float)tx; out->t[1] = (float)ty; out->t[2] = (float)tz;
  if (pose != nullptr) {
    const float t0 = pose[3], t1 = pose[7], t2 = pose[11];
    out->centre[0] = t0; out->centre[1] = t1; out->centre[2] = t2;
    // pose_distance, fp32 like the reference
    const float tr = __fadd_rn(__fadd_rn(pose[0], pose[5]), pose[10]);
    const float rm = sqrtf(__fmul_rn(2.0f, __fadd_rn(1.0f, -__fdiv_rn(fminf(3.0f, tr), 3.0f))));
    const float tm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(t0, t0), __fmul_rn(t1, t1)), __fmul_rn(t2, t2)));
    out->rmeas = rm;
    out->tmeas = tm;
    out->comb = sqrtf(__fadd_rn(__fmul_rn(tm, tm), __fmul_rn(rm, rm)));
    tc::split_pack(rm, tm, out->rt_hi, out->rt_lo);
  } else {
    out->centre[0] = out->centre[1] = out->centre[2] = 0.0f;
    out->rmeas = out->tmeas = out->comb = 0.0f;
    out->rt_hi = out->rt_lo = 0u;
  }
}

__device__ void mat4_product(const float* __restrict__ A, const float* __restrict__ B, float* out) {
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      double a = 0.0;
#pragma unroll
      for (int l = 0; l < 4; ++l) a += (double)A[r * 4 + l] * (double)B[l * 4 + c];
      out[r * 4 + c] = (float)a;
    }
}

__global__ void __launch_bounds__(256)
prep_kernel(srcv_shape s, srcv_cameras cams, srcv_planes pl, bool need_pose_block, const float* __restrict__ src,
            const float* __restrict__ cur, float* __restrict__ planes_ws,
            ViewParams* __restrict__ views, FrameParams* __restrict__ frames,
            float* __restrict__ src_c4, float* __restrict__ cur_c4,
            unsigned* __restrict__ tile_done, long long n_done) {
  const long long nv = (long long)s.B * s.K;
  const long long nf = s.B;
  const long long np = (pl.mode == SRCV_PLANES_FROM_RANGE) ? (long long)s.B * s.D : 0;
  const long long HW = (long long)s.H * s.W;
  const long long nt = src_c4 ? nv * (s.C / 4) * HW : 0;
  const long long nc = cur_c4 ? (long long)s.B * (s.C / 4) * HW : 0;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  // NCHW -> chunk-planar (B,K,C/4,H,W,4) for the sources and (B,C/4,H,W,4) for the reference
  // features.  A thread transposes a 4-pixel x 4-channel block: four 16-byte reads (one per
  // channel plane, coalesced across the warp) and four 16-byte writes (64 contiguous bytes);
  // needs H*W % 4 == 0 for the vector reads, otherwise one pixel per thread.
  const bool vec4 = (HW & 3) == 0;
  const long long ppt = vec4 ? 4 : 1;                      // pixels per thread
  const long long nt_thr = nt / ppt, nc_thr = nc / ppt;
  if (i < nt_thr + nc_thr) {
    const bool is_cur = i >= nt_thr;
    const long long e = (is_cur ? i - nt_thr : i) * ppt;   // first (chunk, pixel) element index
    const long long cj = e / HW, p = e - cj * HW;          // cj = (image * C/4 + chunk)
    const float* in = (is_cur ? cur : src) + cj * 4 * HW + p;
    float4* out = reinterpret_cast<float4*>(is_cur ? cur_c4 : src_c4) + e;
    if (vec4) {
      const float4 c0 = __ldg(reinterpret_cast<const float4*>(in));
      const float4 c1 = __ldg(reinterpret_cast<const float4*>(in + HW));
      const float4 c2 = __ldg(reinterpret_cast<const float4*>(in + 2 * HW));
      const float4 c3 = __ldg(reinterpret_cast<const float4*>(in + 3 * HW));
      out[0] = make_float4(c0.x, c1.x, c2.x, c3.x);
      out[1] = make_float4(c0.y, c1.y, c2.y, c3.y);
      out[2] = make_float4(c0.z, c1.z, c2.z, c3.z);
      out[3] = make_float4(c0.w, c1.w, c2.w, c3.w);
    } else {
      out[0] = make_float4(__ldg(in), __ldg(in + HW), __ldg(in + 2 * HW), __ldg(in + 3 * HW));
    }
    return;
  }
  i -= nt_thr + nc_thr;
  if (i < n_done) { tile_done[i] = 0u; return; }
  i -= n_done;
  if (i < nv) {
    const long long b = i / s.K;
    if (cams.src_extrinsics == nullptr) {
      // raw poses: the two batched 4x4 products of experiment_modules/depth_model.py:324-332,
      // fp64 accumulation, one rounding to fp32 (what the fp32 matmul yields up to its last bit)
      float E[16], P[16];
      mat4_product(cams.src_cam_T_world + i * 16, cams.cur_world_T_cam + b * 16, E);
      mat4_product(cams.cur_cam_T_world + b * 16, cams.src_world_T_cam + i * 16, P);
      view_params(cams.src_Ks + i * 16, E, cams.cur_invK + b * 16, need_pose_block ? P : nullptr, s.W, s.H, views + i);
    } else {
      view_params(cams.src_Ks + i * 16, cams.src_extrinsics + i * 16, cams.cur_invK + b * 16,
                  cams.src_poses ? cams.src_poses + i * 16 : nullptr, s.W, s.H, views + i);
    }
    return;
  }
  i -= nv;
  if (i < nf) {
    const float* invK = cams.cur_invK + i * 16;
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) frames[i].invK[r * 3 + c] = invK[r * 4 + c];
    return;
  }
  i -= nf;
  if (i < np) {
    const int d = (int)(i % s.D);
    const long long fb = pl.range_per_frame ? i / s.D : 0;   // one range for all frames, or one per frame
    const float mn = pl.min_depth[fb], mx = pl.max_depth[fb];
    // exp(log(min) + log(max/min) * ramp): three separate torch ops in the reference
    const float v = expf(__fadd_rn(logf(mn), __fmul_rn(logf(__fdiv_rn(mx, mn)), pl.ramp[d])));
    planes_ws[i] = v;
    if (pl.planes_out) pl.planes_out[i] = v;
  }
}

template <bool PER_PIXEL>
__global__ void __launch_bounds__(256)
argmax_kernel(srcv_shape s, const float* __restrict__ cost, const float* __restrict__ planes,
              float* __restrict__ lowest) {
  const long long HW = (long long)s.H * s.W;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)s.B * HW) return;
  const long long b = i / HW, p = i - b * HW;
  const float* c = cost + b * s.D * HW + p;
  float best = 0.f;
  int best_i = 0;
  for (int d = 0; d < s.D; ++d) {
    const float v = __ldg(c + (long long)d * HW);
    const bool take = (d == 0) || (v > best) || ((v != v) && (best == best));
    if (take) { best = v; best_i = d; }
  }
  lowest[i] = PER_PIXEL ? planes[(b * s.D + best_i) * HW + p] : planes[b * s.D + best_i];
}

}  // namespace

Workspace carve_workspace(const srcv_shape& s, void* base, bool want_c4, size_t extra_bytes) {
  Workspace ws{};
  size_t off = 0;
  char* p = static_cast<char*>(base);
  auto take = [&](size_t bytes) -> char* {
    char* r = p ? p + off : nullptr;
    off += align256(bytes);
    return r;
  };
  ws.planes = reinterpret_cast<float*>(take(sizeof(float) * (size_t)s.B * s.D));
  ws.views = reinterpret_cast<ViewParams*>(take(sizeof(ViewParams) * (size_t)s.B * s.K));
  ws.frames = reinterpret_cast<FrameParams*>(take(sizeof(FrameParams) * (size_t)s.B));
  if (want_c4) {
    ws.src_c4 = reinterpret_cast<float*>(
        take(sizeof(float) * (size_t)s.B * s.K * s.C * s.H * s.W));
    ws.cur_c4 = reinterpret_cast<float*>(take(sizeof(float) * (size_t)s.B * s.C * s.H * s.W));
    ws.tile_done_count = dot_fast_tile_counters(s);
    ws.tile_done = reinterpret_cast<unsigned*>(take(sizeof(unsigned) * ws.tile_done_count));
  }
  if (extra_bytes) ws.extra = reinterpret_cast<float*>(take(extra_bytes));
  ws.bytes = off;
  if (!p) { ws.planes = nullptr; ws.views = nullptr; ws.frames = nullptr; ws.src_c4 = nullptr; ws.cur_c4 = nullptr; ws.tile_done = nullptr; ws.extra = nullptr; }
  return ws;
}

cudaError_t launch_prep(const srcv_shape& s, const srcv_cameras& cams, const srcv_planes& pl,
                        const float* src_feats, const float* cur_feats, const Workspace& ws,
                        bool need_poses, cudaStream_t stream) {
  srcv_cameras c = cams;
  if (!need_poses) c.src_poses = nullptr;
  // chunk-planar inputs are gathered in place: no re-layout copy (the sweeps read the caller's buffers)
  const bool copy_c4 = s.layout != SRCV_LAYOUT_CHUNK_PLANAR;
  const long long nv = (long long)s.B * s.K;
  const long long np = (pl.mode == SRCV_PLANES_FROM_RANGE) ? (long long)s.B * s.D : 0;
  const long long nt = (ws.src_c4 && copy_c4) ? nv * (s.C / 4) * s.H * s.W : 0;
  const long long ncur = (ws.src_c4 && ws.cur_c4 && copy_c4) ? (long long)s.B * (s.C / 4) * s.H * s.W : 0;
  const long long ppt = (((long long)s.H * s.W) & 3) == 0 ? 4 : 1;
  const long long ndone = ws.tile_done ? (long long)ws.tile_done_count : 0;
  const long long total = nt / ppt + ncur / ppt + ndone + nv + s.B + np;
  const int threads = 256;
  const long long blocks = (total + threads - 1) / threads;
  SRCV_LAUNCH(prep_kernel, (unsigned)blocks, threads, 0, stream, s, c, pl, need_poses, src_feats, cur_feats, ws.planes,
              ws.views, ws.frames, nt ? ws.src_c4 : nullptr, ncur ? ws.cur_c4 : nullptr, ws.tile_done, ndone);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_argmax(const srcv_shape& s, const float* cost, const float* planes,
                          bool per_pixel, float* lowest, cudaStream_t stream) {
  const long long n = (long long)s.B * s.H * s.W;
  const int threads = 256;
  const unsigned blocks = (unsigned)((n + threads - 1) / threads);
  if (per_pixel) SRCV_LAUNCH(argmax_kernel<true>, blocks, threads, 0, stream, s, cost, planes, lowest);
  else SRCV_LAUNCH(argmax_kernel<false>, blocks, threads, 0, stream, s, cost, planes, lowest);
  note_launch();
  return cudaGetLastError();
}
}  // namespace srcv
