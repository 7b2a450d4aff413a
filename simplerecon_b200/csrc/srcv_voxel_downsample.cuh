// Voxel down-sampling of a point cloud (DESIGN §4.19): Open3D's VoxelDownSample rule, restated from its documented
// behaviour, with a deterministic output order.
//
// Rule, in fp64 from the fp32 points and the voxel size s:
//   b = min_i p_i - 0.5 s per axis (the minimum over fp32 values is exact);
//   voxel of p: v = floor((p - b) / s) per axis, an IEEE subtraction and division (never a reciprocal), so v >= 0;
//   output point of a voxel: the fp64 sum of its points, accumulated in input order from 0.0, divided by their count
//   in fp64 and rounded once to fp32; colours likewise, uint8 taken as c / 255.0 in fp64 and floats as given.
// Voxels come out in ascending (vx, vy, vz) order.  Every fp64 step is an explicitly rounded __dadd_rn / __ddiv_rn,
// so nvcc cannot contract or reassociate it and the outputs equal the numpy oracle's bitwise.
//
// Kernels.  The box partials of the mesh evaluation give the bounding box; one thread turns it into b, the voxel
// extent n_k = vmax_k + 1 per axis (2^21 or more on an axis raises SRCV_VOXEL_EXTENT) and the number of 8-bit digit
// passes the key needs.  The key is the mixed-radix index (vx n_y + vy) n_z + vz < n_x n_y n_z < 2^63, so a room at
// 2 cm needs three passes instead of the eight of a 63-bit key.  A stable LSD radix sort of (key, index): per pass a
// per-tile digit histogram (digit-major, so one scan gives every (digit, tile) its output offset), the fixed-tile
// scan of srcv_mesh_eval.cuh, and a scatter that ranks each tile's items in tile order from the digits of each group
// of 32 threads and per-group digit counts in shared memory: no atomics decide any position.  The
// passes the extent does not need exit at once; the keys start in the buffer that leaves the result in buffer 0.
// Segment heads of the sorted keys, scanned, give each voxel its id and first sorted position; one thread per voxel
// walks its run in sorted order, which is input order because the sort is stable, and writes the means and the
// count.  The cost of a voxel is linear in its point count: a cloud in one voxel is one thread's walk.
//
// Robustness.  A non-finite coordinate (SRCV_MESH_EVAL_NONFINITE) or extent makes every key 0 and no row written;
// a non-finite colour raises SRCV_VOXEL_NONFINITE_COLOR.  Nothing here synchronises with the host.
//
// Compiled in the srcv_tsdf.cu unit: included at the end of srcv_mesh_eval.cuh, whose box partials and scan it uses.
#pragma once
#include "srcv_mesh_eval.cuh"

namespace srcv {
namespace voxel_ds_detail {
namespace {

namespace me = mesh_eval_detail;
constexpr int kThreads = me::kThreads;                 // 256: one digit per thread in the sort's shared tables
constexpr int kPerThread = me::kPerThread;
constexpr int kTile = me::kTile;                       // 2048 items per sort tile, 8 rounds of 256
constexpr int kWarps = kThreads / 32;
constexpr int kDigits = 256;
constexpr int kMaxPasses = 8;
constexpr int kBatch = 8;                              // points a voxel's walk loads ahead of its adds
constexpr double kMaxExtent = (double)(1 << 21);       // voxels per axis, exclusive
constexpr unsigned kBad = SRCV_MESH_EVAL_NONFINITE | SRCV_VOXEL_EXTENT;
static_assert(kThreads == kDigits, "the sort gives each thread one digit");

#ifdef SRCV_HOST_EMU
using mesh_vis_detail::__dadd_rn;
using mesh_vis_detail::__ddiv_rn;
#endif

struct Params {
  double b[3];                 // the voxel grid's corner
  double s;
  unsigned long long ny, nz;   // voxels along y and z
  int passes;                  // 8-bit digit passes the key needs (0: one voxel)
  int bad;                     // a coordinate or extent flag: keys are 0, no row is written
};

// one thread: the box from the partials, the corner, the extent check and the pass count
__global__ void params_kernel(const double* __restrict__ partial, int nparts, double s, Params* P, unsigned* flags) {
  double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int p = 0; p < nparts; ++p)
    for (int k = 0; k < 3; ++k) { lo[k] = fmin(lo[k], partial[6 * p + k]); hi[k] = fmax(hi[k], partial[6 * p + 3 + k]); }
  bool bad = (me::read_flags(flags) & SRCV_MESH_EVAL_NONFINITE) != 0u;
  unsigned long long n[3] = {1ull, 1ull, 1ull};
  for (int k = 0; k < 3; ++k) {
    P->b[k] = __dadd_rn(lo[k], -0.5 * s);
    const double vmax = floor(__ddiv_rn(__dadd_rn(hi[k], -P->b[k]), s));
    if (!bad && !(vmax + 1.0 < kMaxExtent)) {           // also NaN and inf
      me::raise_flag(flags, SRCV_VOXEL_EXTENT);
      bad = true;
    }
    if (!bad) n[k] = (unsigned long long)vmax + 1ull;
  }
  P->s = s;
  P->ny = n[1];
  P->nz = n[2];
  const unsigned long long top = n[0] * n[1] * n[2] - 1ull;   // the largest key, < 2^63
  int bits = 0;
  while (bits < 64 && (top >> bits) != 0ull) ++bits;
  P->passes = bad ? 0 : (bits + 7) / 8;
  P->bad = bad ? 1 : 0;
}

__device__ __forceinline__ unsigned long long voxel_key(const float* __restrict__ p, const Params& P) {
  unsigned long long v[3];
  for (int k = 0; k < 3; ++k) v[k] = (unsigned long long)floor(__ddiv_rn(__dadd_rn((double)p[k], -P.b[k]), P.s));
  return (v[0] * P.ny + v[1]) * P.nz + v[2];
}

// the keys and the identity permutation, in the buffer from which the passes leave the result in buffer 0
__global__ void __launch_bounds__(kThreads)
key_kernel(const float* __restrict__ pts, long long n, const Params* __restrict__ P, unsigned long long* keys0,
           unsigned long long* keys1, int* idx0, int* idx1) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  const Params p = *P;
  const bool one = (p.passes & 1) != 0;
  (one ? keys1 : keys0)[i] = p.bad ? 0ull : voxel_key(pts + 3 * i, p);
  (one ? idx1 : idx0)[i] = (int)i;
}

// pass `pass` reads buffer (passes + pass) & 1 and writes the other
__device__ __forceinline__ bool reads_one(const Params* P, int pass) { return ((P->passes + pass) & 1) != 0; }

// hist[d * ntiles + tile]: the items of the tile with digit d
__global__ void __launch_bounds__(kThreads)
radix_hist_kernel(const unsigned long long* __restrict__ keys0, const unsigned long long* __restrict__ keys1, long long n,
                  int pass, const Params* __restrict__ P, unsigned* __restrict__ hist, int ntiles) {
  __shared__ unsigned s_cnt[kDigits];
  if (pass >= P->passes) return;                          // uniform
  const unsigned long long* keys = reads_one(P, pass) ? keys1 : keys0;
  const int t = threadIdx.x, shift = 8 * pass;
  s_cnt[t] = 0u;
  __syncthreads();
  for (int r = 0; r < kPerThread; ++r) {
    const long long i = (long long)blockIdx.x * kTile + (long long)r * kThreads + t;
    if (i < n) atomicAdd(&s_cnt[(unsigned)(keys[i] >> shift) & 255u], 1u);   // integer counts: order-free
  }
  __syncthreads();
  hist[(long long)t * ntiles + blockIdx.x] = s_cnt[t];
}

// Item (round r, thread t) of a tile is its (r * 256 + t)-th: a round is ranked in group and lane order (groups of
// 32 consecutive threads), the rounds in turn, so equal digits keep their order.  Each thread reads its group's 32
// digits from shared memory (the same address for the whole warp, a broadcast) to count the equal ones before it.
// incl is the inclusive scan of hist; incl - hist is the (digit, tile)'s first output position.
__global__ void __launch_bounds__(kThreads)
radix_scatter_kernel(unsigned long long* keys0, unsigned long long* keys1, int* idx0, int* idx1, long long n, int pass,
                     const Params* __restrict__ P, const unsigned* __restrict__ hist, const unsigned* __restrict__ incl,
                     int ntiles) {
  __shared__ unsigned s_run[kDigits];                     // the next output position of each digit
  __shared__ unsigned s_warp[kWarps][kDigits];            // this round's items per (group, digit)
  __shared__ unsigned s_digit[kThreads];                  // this round's digits, kDigits for no item
  if (pass >= P->passes) return;                          // uniform
  const bool one = reads_one(P, pass);
  const unsigned long long* kin = one ? keys1 : keys0;
  const int* iin = one ? idx1 : idx0;
  unsigned long long* kout = one ? keys0 : keys1;
  int* iout = one ? idx0 : idx1;
  const int t = threadIdx.x, w = t >> 5, lane = t & 31, shift = 8 * pass;
  const long long h = (long long)t * ntiles + blockIdx.x;
  s_run[t] = incl[h] - hist[h];
  for (int v = 0; v < kWarps; ++v) s_warp[v][t] = 0u;
  for (int r = 0; r < kPerThread; ++r) {
    const long long i = (long long)blockIdx.x * kTile + (long long)r * kThreads + t;
    const bool live = i < n;
    const unsigned long long k = live ? kin[i] : 0ull;
    const int id = live ? iin[i] : 0;
    const unsigned d = live ? (unsigned)(k >> shift) & 255u : (unsigned)kDigits;
    s_digit[t] = d;
    __syncthreads();
    unsigned before = 0u;                                 // equal digits earlier in the group
    bool last = true;                                     // no equal digit later in the group
    for (int l = 0; l < 32; ++l) {
      const bool eq = s_digit[32 * w + l] == d;
      before += (eq && l < lane) ? 1u : 0u;
      last &= !(eq && l > lane);
    }
    if (live && last) s_warp[w][d] = before + 1u;
    __syncthreads();
    if (live) {
      unsigned pos = s_run[d] + before;
      for (int v = 0; v < w; ++v) pos += s_warp[v][d];
      kout[pos] = k;
      iout[pos] = id;
    }
    __syncthreads();
    unsigned add = 0u;                                    // thread t advances digit t past this round
    for (int v = 0; v < kWarps; ++v) { add += s_warp[v][t]; s_warp[v][t] = 0u; }
    s_run[t] += add;
  }
}

__global__ void __launch_bounds__(kThreads)
head_kernel(const unsigned long long* __restrict__ keys, long long n, unsigned* __restrict__ head) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i < n) head[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1u : 0u;
}

// pos: the inclusive scan of head, so voxel pos[i] - 1 starts at sorted position i; start[M] = n
__global__ void __launch_bounds__(kThreads)
start_kernel(const unsigned* __restrict__ head, const unsigned* __restrict__ pos, long long n, int* __restrict__ start,
             long long* __restrict__ num_out) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n) return;
  if (head[i]) start[pos[i] - 1u] = (int)i;
  if (i == n - 1) {
    start[pos[i]] = (int)n;
    *num_out = (long long)pos[i];
  }
}

__device__ __forceinline__ double color_of(const void* colors, int type, long long j) {
  if (type == SRCV_COLORS_U8) return __ddiv_rn((double)static_cast<const unsigned char*>(colors)[j], 255.0);
  if (type == SRCV_COLORS_F32) return (double)static_cast<const float*>(colors)[j];
  return static_cast<const double*>(colors)[j];
}

// one thread per voxel: its run of sorted positions start[j] .. start[j + 1], in input order
__global__ void __launch_bounds__(kThreads)
mean_kernel(const float* __restrict__ pts, const void* __restrict__ colors, int color_type, const int* __restrict__ idx,
            const int* __restrict__ start, const long long* __restrict__ num_out, const Params* __restrict__ P,
            float* __restrict__ out_pts, float* __restrict__ out_colors, int* __restrict__ out_counts, unsigned* flags) {
  const long long j = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (j >= *num_out || P->bad) return;
  const int b = start[j], e = start[j + 1];
  double sp[3] = {0.0, 0.0, 0.0}, sc[3] = {0.0, 0.0, 0.0};
  bool fin = true;
  // kBatch points' loads go out before their adds, which stay in input order: a long run is bound by the adds,
  // not by one load latency per point
  for (int i0 = b; i0 < e; i0 += kBatch) {
    const int m = min(kBatch, e - i0);
    float x[kBatch][3];
    double c[kBatch][3];
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      if (u >= m) break;
      const long long q = idx[i0 + u];
      for (int k = 0; k < 3; ++k) x[u][k] = pts[3 * q + k];
      if (color_type != SRCV_COLORS_NONE)
        for (int k = 0; k < 3; ++k) c[u][k] = color_of(colors, color_type, 3 * q + k);
    }
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      if (u >= m) break;
      for (int k = 0; k < 3; ++k) sp[k] = __dadd_rn(sp[k], (double)x[u][k]);
      if (color_type != SRCV_COLORS_NONE)
        for (int k = 0; k < 3; ++k) {
          fin &= me::finite(c[u][k]);
          sc[k] = __dadd_rn(sc[k], c[u][k]);
        }
    }
  }
  if (!fin) me::raise_flag(flags, SRCV_VOXEL_NONFINITE_COLOR);
  const double cnt = (double)(e - b);
  for (int k = 0; k < 3; ++k) out_pts[3 * j + k] = (float)__ddiv_rn(sp[k], cnt);
  if (color_type != SRCV_COLORS_NONE)
    for (int k = 0; k < 3; ++k) out_colors[3 * j + k] = (float)__ddiv_rn(sc[k], cnt);
  out_counts[j] = e - b;
}

struct Ws {
  double* box;
  Params* params;
  unsigned long long* keys[2];
  int* idx[2];
  unsigned* hist;              // [kDigits * ntiles], digit-major
  unsigned* incl;              // its inclusive scan
  unsigned* tile;              // the scan's tile sums
  unsigned* head;
  unsigned* pos;
  int* start;                  // [n + 1]
  size_t bytes;
};

Ws carve(long long n, void* base) {
  Ws w{};
  char* p = static_cast<char*>(base);
  size_t off = 0;
  const long long nh = (long long)kDigits * me::tiles_of(n);
  const long long nscan = nh > n ? nh : n;
  w.box = reinterpret_cast<double*>(p + off);                     off += align256(sizeof(double) * 6 * me::kBoxCtas);
  w.params = reinterpret_cast<Params*>(p + off);                  off += align256(sizeof(Params));
  for (int k = 0; k < 2; ++k) {
    w.keys[k] = reinterpret_cast<unsigned long long*>(p + off);   off += align256(8 * (size_t)n);
    w.idx[k] = reinterpret_cast<int*>(p + off);                   off += align256(4 * (size_t)n);
  }
  w.hist = reinterpret_cast<unsigned*>(p + off);                  off += align256(4 * (size_t)nh);
  w.incl = reinterpret_cast<unsigned*>(p + off);                  off += align256(4 * (size_t)nh);
  w.tile = reinterpret_cast<unsigned*>(p + off);                  off += align256(4 * (size_t)me::tiles_of(nscan));
  w.head = reinterpret_cast<unsigned*>(p + off);                  off += align256(4 * (size_t)n);
  w.pos = reinterpret_cast<unsigned*>(p + off);                   off += align256(4 * (size_t)n);
  w.start = reinterpret_cast<int*>(p + off);                      off += align256(4 * (size_t)(n + 1));
  w.bytes = off;
  return w;
}

}  // namespace
}  // namespace voxel_ds_detail

size_t voxel_down_sample_workspace_bytes(long long n) { return voxel_ds_detail::carve(n, nullptr).bytes; }

cudaError_t launch_voxel_down_sample(const float* points, long long n, double voxel_size, const void* colors,
                                     int color_type, float* out_points, float* out_colors, int32_t* out_counts,
                                     int64_t* num_out, unsigned* flags, void* workspace, cudaStream_t stream) {
  namespace vd = voxel_ds_detail;
  namespace me = mesh_eval_detail;
  const vd::Ws w = vd::carve(n, workspace);
  const long long nt = me::tiles_of(n);
  const unsigned grid = (unsigned)((n + vd::kThreads - 1) / vd::kThreads);
  const int nbox = (int)me::capped(nt, me::kBoxCtas);
  SRCV_LAUNCH(me::bbox_kernel, nbox, me::kThreads, 0, stream, points, n, w.box, flags);
  SRCV_LAUNCH(vd::params_kernel, 1, 1, 0, stream, (const double*)w.box, nbox, voxel_size, w.params, flags);
  SRCV_LAUNCH(vd::key_kernel, grid, vd::kThreads, 0, stream, points, n, (const vd::Params*)w.params, w.keys[0],
              w.keys[1], w.idx[0], w.idx[1]);
  note_launch(3);
  for (int pass = 0; pass < vd::kMaxPasses; ++pass) {
    SRCV_LAUNCH(vd::radix_hist_kernel, (unsigned)nt, vd::kThreads, 0, stream, (const unsigned long long*)w.keys[0],
                (const unsigned long long*)w.keys[1], n, pass, (const vd::Params*)w.params, w.hist, (int)nt);
    note_launch();
    me::launch_scan<unsigned>(w.hist, (long long)vd::kDigits * nt, w.tile, w.incl, stream);
    SRCV_LAUNCH(vd::radix_scatter_kernel, (unsigned)nt, vd::kThreads, 0, stream, w.keys[0], w.keys[1], w.idx[0],
                w.idx[1], n, pass, (const vd::Params*)w.params, (const unsigned*)w.hist, (const unsigned*)w.incl,
                (int)nt);
    note_launch();
  }
  SRCV_LAUNCH(vd::head_kernel, grid, vd::kThreads, 0, stream, (const unsigned long long*)w.keys[0], n, w.head);
  note_launch();
  me::launch_scan<unsigned>(w.head, n, w.tile, w.pos, stream);
  SRCV_LAUNCH(vd::start_kernel, grid, vd::kThreads, 0, stream, (const unsigned*)w.head, (const unsigned*)w.pos, n,
              w.start, reinterpret_cast<long long*>(num_out));
  SRCV_LAUNCH(vd::mean_kernel, grid, vd::kThreads, 0, stream, points, colors, color_type, (const int*)w.idx[0],
              (const int*)w.start, (const long long*)num_out, (const vd::Params*)w.params, out_points, out_colors,
              out_counts, flags);
  note_launch(2);
  return cudaGetLastError();
}

}  // namespace srcv
