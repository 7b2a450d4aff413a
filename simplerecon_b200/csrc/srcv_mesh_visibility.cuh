// Visibility culling for mesh evaluation (DESIGN §4.18): how many depth frames observe each point, and the points
// that at least one frame observes, in input order.
//
// The rule is the fuser's validity test (reference tools/tsdf.py:270-296) applied to arbitrary points, with the
// truncation replaced by a margin: point p is observed by frame f when fusing f's depth map would update a voxel
// at p.  Evaluated in fp64 from the fp32 inputs, in this order (E = cam_T_world[f], K = K[f]):
//   x = ((E00 px + E01 py) + E02 pz) + E03, likewise y and z;  U = (K00 x + K01 y) + K02 z, likewise V;
//   u = U / z, v = V / z;  ix = rint(u - 0.5), iy = rint(v - 0.5) (half to even: grid_sample's nearest read);
//   observed <=> 0 < z < max_depth, 0 <= ix < W, 0 <= iy < H, d = depth[f, iy, ix] with 0 < d < max_depth
//   (so d is finite), and d - z > -margin.
// Every step is an explicitly rounded __dmul_rn / __dadd_rn / __ddiv_rn, so nvcc cannot contract it into FMAs and
// the counts equal the numpy oracle's exactly.  This is deliberately not the integration kernel's projection: that
// one reproduces the reference's fp16 arithmetic on the voxel lattice.
//
// Kernel.  One thread per point, CTAs of 256 consecutive points.  The CTA reduces its points' fp64 bounding box,
// then stages the frames' constants (E's 12 entries, K's 6, as doubles) in shared memory kFrameChunk frames at a
// time; while staging, thread j tests frame j against the box and drops it for the whole tile when all 8 corners
// lie in one of the half-spaces z <= 0, z >= max_depth, U + z < 0, U - (W + 1) z > 0, V + z < 0,
// V - (H + 1) z > 0.  The half-spaces are convex, so the box's points lie there too, and each of them puts u or v
// at least a pixel outside the image, or z outside (0, max_depth); the tests carry a tolerance far above the
// rounding of the corner arithmetic, so a dropped frame observes no point of the tile.  Points from the surface
// sampler come out in triangle order, so a tile is a small patch of surface and most frames drop out.
//
// Outputs.  counts[i] += the frames that observe point i (one thread per point: no atomics), so chunks of frames
// can be fed one call after another.  A non-finite point coordinate ORs SRCV_MESH_EVAL_NONFINITE into the flag
// word (whether or not its tile is culled), a non-finite entry of E or K SRCV_MESH_EVAL_BAD_VIEW; neither kind is
// ever observed.  The compaction keeps the points with count > 0 in input order through the sampler's fixed-tile
// prefix sum and writes the survivor count to the device.  Nothing here synchronises with the host.
//
// Compiled in the srcv_tsdf.cu unit: included at the end of srcv_mesh_eval.cuh, whose scan and helpers it uses.
#pragma once
#include "srcv_mesh_eval.cuh"

namespace srcv {
namespace mesh_vis_detail {
namespace {

namespace me = mesh_eval_detail;
constexpr int kThreads = me::kThreads;                 // points per CTA tile, one per thread
constexpr int kFrameChunk = 64;                        // frames staged in shared memory at a time
constexpr double kCullTol = 1e-9;                      // relative tolerance of the tile test (rounding is ~1e-15)

#ifdef SRCV_HOST_EMU
// the host emulation builds with -ffp-contract=off: every operation rounds once, as the _rn intrinsics do
inline double __dmul_rn(double a, double b) { return a * b; }
inline double __dadd_rn(double a, double b) { return a + b; }
inline double __ddiv_rn(double a, double b) { return a / b; }
#endif

struct View {
  double E[12];                                        // cam_T_world rows 0..2
  double K[6];                                         // K rows 0..1, columns 0..2
};

// row r of E applied to p, in the order of the rule
__device__ __forceinline__ double cam_coord(const double* E, int r, double px, double py, double pz) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(E[4 * r], px), __dmul_rn(E[4 * r + 1], py)), __dmul_rn(E[4 * r + 2], pz)),
                   E[4 * r + 3]);
}

// row r of K applied to (x, y, z)
__device__ __forceinline__ double pix_coord(const double* K, int r, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dmul_rn(K[3 * r], x), __dmul_rn(K[3 * r + 1], y)), __dmul_rn(K[3 * r + 2], z));
}

// the observation rule (DESIGN §4.18) for one finite point and one frame; depth is the frame's (H, W) map
__device__ __forceinline__ bool observes(const View& v, double px, double py, double pz, const float* __restrict__ depth,
                                         int H, int W, double margin, double max_depth) {
  const double z = cam_coord(v.E, 2, px, py, pz);
  if (!(z > 0.0 && z < max_depth)) return false;
  const double x = cam_coord(v.E, 0, px, py, pz), y = cam_coord(v.E, 1, px, py, pz);
  const double fx = rint(__dadd_rn(__ddiv_rn(pix_coord(v.K, 0, x, y, z), z), -0.5));
  const double fy = rint(__dadd_rn(__ddiv_rn(pix_coord(v.K, 1, x, y, z), z), -0.5));
  if (!(fx >= 0.0 && fx < (double)W && fy >= 0.0 && fy < (double)H)) return false;   // before any conversion to int
  const double d = depth[(int)fy * W + (int)fx];        // H W < 2^31
  return d > 0.0 && d < max_depth && __dadd_rn(d, -z) > -margin;
}

// Whether the box [lo, hi] lies in one of the frame's six rejecting half-spaces (all 8 corners in the same one).
// Each test must hold by a tolerance kCullTol times a bound on the magnitudes its arithmetic combines, so that the
// rounding of the corners' evaluation (and of the points' own) cannot turn a rejected box into an observed point.
__device__ __forceinline__ bool box_outside(const View& v, const double lo[3], const double hi[3], int H, int W,
                                            double max_depth) {
  double a[3], S[3];
  for (int k = 0; k < 3; ++k) a[k] = fmax(fabs(lo[k]), fabs(hi[k]));
  for (int r = 0; r < 3; ++r)
    S[r] = fabs(v.E[4 * r]) * a[0] + fabs(v.E[4 * r + 1]) * a[1] + fabs(v.E[4 * r + 2]) * a[2] + fabs(v.E[4 * r + 3]);
  const double SU = fabs(v.K[0]) * S[0] + fabs(v.K[1]) * S[1] + fabs(v.K[2]) * S[2];
  const double SV = fabs(v.K[3]) * S[0] + fabs(v.K[4]) * S[1] + fabs(v.K[5]) * S[2];
  const double Wp = (double)W + 1.0, Hp = (double)H + 1.0;
  const double tz = kCullTol * S[2], tu = kCullTol * (SU + Wp * S[2]), tv = kCullTol * (SV + Hp * S[2]);
  unsigned all = 0x3fu;
  for (int c = 0; c < 8; ++c) {
    const double px = (c & 1) ? hi[0] : lo[0], py = (c & 2) ? hi[1] : lo[1], pz = (c & 4) ? hi[2] : lo[2];
    const double x = cam_coord(v.E, 0, px, py, pz), y = cam_coord(v.E, 1, px, py, pz), z = cam_coord(v.E, 2, px, py, pz);
    const double U = pix_coord(v.K, 0, x, y, z), V = pix_coord(v.K, 1, x, y, z);
    unsigned m = 0u;
    if (z <= -tz) m |= 1u;                              // behind the camera
    if (z - max_depth >= tz) m |= 2u;                   // at or beyond max_depth (never for max_depth = inf)
    if (U + z < -tu) m |= 4u;                           // u < -1
    if (U - Wp * z > tu) m |= 8u;                       // u > W + 1
    if (V + z < -tv) m |= 16u;                          // v < -1
    if (V - Hp * z > tv) m |= 32u;                      // v > H + 1
    all &= m;
  }
  return all != 0u;
}

// tested (optional): adds, per CTA, its points times the frames it evaluated for them (a measurement counter)
__global__ void __launch_bounds__(kThreads)
observation_count_kernel(const float* __restrict__ pts, long long n, const float* __restrict__ depths,
                         const float* __restrict__ Ks, int k_stride, const float* __restrict__ Es, int F, int H, int W,
                         double margin, double max_depth, int tile_cull, int* __restrict__ counts, unsigned* flags,
                         unsigned long long* tested) {
  __shared__ View s_view[kFrameChunk];
  __shared__ int s_live[kFrameChunk];
  __shared__ double s_box[6][kThreads];
  const int t = threadIdx.x;
  const long long i = (long long)blockIdx.x * kThreads + t;
  double p[3] = {0.0, 0.0, 0.0};
  bool ok = false;
  if (i < n) {
    for (int k = 0; k < 3; ++k) p[k] = pts[3 * i + k];
    ok = me::finite3(p[0], p[1], p[2]);
    if (!ok) me::raise_flag(flags, SRCV_MESH_EVAL_NONFINITE);
  }
  for (int k = 0; k < 3; ++k) {
    s_box[k][t] = ok ? p[k] : INFINITY;
    s_box[3 + k][t] = ok ? p[k] : -INFINITY;
  }
  block_tree<kThreads>([&](int a, int b) {
    for (int k = 0; k < 3; ++k) { s_box[k][a] = fmin(s_box[k][a], s_box[k][b]); s_box[3 + k][a] = fmax(s_box[3 + k][a], s_box[3 + k][b]); }
  });
  const double lo[3] = {s_box[0][0], s_box[1][0], s_box[2][0]}, hi[3] = {s_box[3][0], s_box[4][0], s_box[5][0]};
  const bool empty = !(lo[0] <= hi[0]);                 // no finite point in the tile: nothing to observe
  const long long HW = (long long)H * W;
  int count = 0;
  long long live_frames = 0;
  for (int f0 = 0; f0 < F; f0 += kFrameChunk) {
    const int m = min(kFrameChunk, F - f0);
    __syncthreads();                                    // every thread is done with the previous chunk
    if (t < m) {
      const long long f = (long long)f0 + t;
      const float* E = Es + 16 * f;
      const float* K = Ks + (long long)k_stride * f;
      View v;
      bool fin = true;
      for (int k = 0; k < 12; ++k) { v.E[k] = E[k]; fin &= me::finite(v.E[k]); }
      for (int r = 0; r < 2; ++r)
        for (int c = 0; c < 3; ++c) { v.K[3 * r + c] = K[4 * r + c]; fin &= me::finite(v.K[3 * r + c]); }
      if (!fin) me::raise_flag(flags, SRCV_MESH_EVAL_BAD_VIEW);
      s_view[t] = v;
      s_live[t] = fin && !empty && !(tile_cull && box_outside(v, lo, hi, H, W, max_depth));
    }
    __syncthreads();
    for (int j = 0; j < m; ++j) {
      if (!s_live[j]) continue;                         // uniform across the CTA
      ++live_frames;
      if (ok && observes(s_view[j], p[0], p[1], p[2], depths + (long long)(f0 + j) * HW, H, W, margin, max_depth)) ++count;
    }
  }
  if (i < n) counts[i] += count;
  if (tested != nullptr && t == 0 && live_frames > 0) {
    const long long pts_in_tile = n - (long long)blockIdx.x * kThreads < kThreads ? n - (long long)blockIdx.x * kThreads : kThreads;
    me::atomic_add_u64(tested, (unsigned long long)(live_frames * pts_in_tile));
  }
}

__global__ void __launch_bounds__(kThreads) keep_kernel(const int* __restrict__ counts, long long n, int* __restrict__ keep) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i < n) keep[i] = counts[i] > 0 ? 1 : 0;
}

// pos: the inclusive prefix sum of keep, so a kept point goes to pos[i] - 1 and pos[n - 1] points are kept
__global__ void __launch_bounds__(kThreads)
compact_kernel(const float* __restrict__ pts, const int* __restrict__ counts, const int* __restrict__ pos, long long n,
               float* __restrict__ out, long long* __restrict__ num_kept) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  if (counts[i] > 0) {
    const long long j = pos[i] - 1;
    for (int k = 0; k < 3; ++k) out[3 * j + k] = pts[3 * i + k];
  }
  if (i == n - 1) *num_kept = pos[i];
}

struct CompactWs {
  int* keep;
  int* pos;
  int* tile;
  size_t bytes;
};

CompactWs carve_compact(long long n, void* base) {
  CompactWs w{};
  char* p = static_cast<char*>(base);
  size_t off = 0;
  w.keep = reinterpret_cast<int*>(p + off); off += align256(4 * (size_t)n);
  w.pos = reinterpret_cast<int*>(p + off);  off += align256(4 * (size_t)n);
  w.tile = reinterpret_cast<int*>(p + off); off += align256(4 * (size_t)me::tiles_of(n));
  w.bytes = off;
  return w;
}

}  // namespace
}  // namespace mesh_vis_detail

size_t observed_compact_workspace_bytes(long long n) { return mesh_vis_detail::carve_compact(n, nullptr).bytes; }

cudaError_t launch_observation_counts(const srcv_mesh_eval_args& a, const srcv_mesh_views& v, const float* points,
                                      int32_t* counts, cudaStream_t stream) {
  namespace mv = mesh_vis_detail;
  const long long n = a.num_points;
  SRCV_LAUNCH(mv::observation_count_kernel, (unsigned)((n + mv::kThreads - 1) / mv::kThreads), mv::kThreads, 0, stream,
              points, n, v.depths, v.K, v.K_shared ? 0 : 16, v.cam_T_world, v.F, v.H, v.W, v.margin, v.max_depth,
              v.tile_cull, counts, a.flags, reinterpret_cast<unsigned long long*>(a.stats));
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_compact_observed(const srcv_mesh_eval_args& a, const float* points, const int32_t* counts,
                                    float* kept, int64_t* num_kept, void* workspace, cudaStream_t stream) {
  namespace mv = mesh_vis_detail;
  const long long n = a.num_points;
  const mv::CompactWs w = mv::carve_compact(n, workspace);
  const unsigned grid = (unsigned)((n + mv::kThreads - 1) / mv::kThreads);
  SRCV_LAUNCH(mv::keep_kernel, grid, mv::kThreads, 0, stream, counts, n, w.keep);
  note_launch();
  mesh_eval_detail::launch_scan<int>(w.keep, n, w.tile, w.pos, stream);
  SRCV_LAUNCH(mv::compact_kernel, grid, mv::kThreads, 0, stream, points, counts, (const int*)w.pos, n, kept,
              reinterpret_cast<long long*>(num_kept));
  note_launch();
  return cudaGetLastError();
}

}  // namespace srcv
