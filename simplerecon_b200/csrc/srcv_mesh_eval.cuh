// Mesh evaluation (DESIGN §4.17): accuracy, completeness, Chamfer distance, precision, recall and F-score of a
// predicted surface against the ground truth, each side a point set or a mesh sampled uniformly by area.
//
// Sampler.  Triangle areas in fp64 from the fp32 vertices, a deterministic inclusive prefix sum (fixed tiles,
// fixed trees, no atomics), then per sample i three uniforms u0, u1, u2 from a counter hash of (seed, i, draw):
// the triangle is the first whose CDF value exceeds (i + u0) / N * total (stratified: sample i lies in the i-th
// N-th of the area, so samples come out in triangle order, spatially coherent), and the point is
// (1 - sqrt u1) a + sqrt u1 (1 - u2) b + sqrt u1 u2 c in fp64, rounded to fp32.
//
// Nearest distances.  A uniform grid over the target points, cells hashed with block_key / block_hash
// (srcv_block_hash.cuh), built in three steps: count per cell, scan over the table's slots, scatter into a
// cell-ordered copy.  The cell edge h comes from the device: the target count N and bounding box (sides a, b,
// c), h = sqrt(2 (ab + bc + ca) / N), the point spacing of N points on a surface of the box's area; it is
// widened so that every axis has at most 2^20 cells.  A query visits the shells of cells of Chebyshev radius
// r = 0, 1, ... around its own cell; after shell r, every unvisited point lies outside the visited cube, at
// least m_r away (the distance from the query to the cube's nearest face), so the best distance is final once
// it is <= m_r (or the cube covers the whole grid).  A query still open after kMaxShell shells goes to a
// device queue for the next level, a grid of 8 times the cell edge (four levels: h, 8h, 64h, 512h), which
// starts from the best distance found so far.  What the last level leaves open (a floater far from all
// geometry) a last kernel brute-forces against every target point in shared-memory tiles, with an
// atomicMin on the fp64 bits of the squared distance (non-negative doubles order like their bits): exact, and
// independent of the order of the updates.  Distances are fp64 evaluations from the fp32 coordinates.
//
// Metrics.  Per-CTA fp64 sums and int64 counts in fixed shared-memory trees, then one CTA sums the partials in
// a fixed order: no atomics in the sums, bitwise the same result on every run.
//
// Robustness.  A face index outside [0, V), a non-finite coordinate or a zero total area raises a bit in the
// caller's flag word; the kernels after it read nothing out of bounds, and the outputs are NaN.  Nothing here
// synchronises with the host.
//
// Compiled in the srcv_tsdf.cu unit, after the mesh kernels whose output it scores.
#pragma once
#include "srcv_block_hash.cuh"
#include "srcv_kernels.h"

namespace srcv {
namespace mesh_eval_detail {
namespace {

constexpr int kThreads = 256;
constexpr int kPerThread = 8;
constexpr int kTile = kThreads * kPerThread;          // scan and reduction tile: 2048 elements
constexpr int kMaxShell = 4;                          // grid-search radius before a query moves to the next level
constexpr int kLevels = 4;                            // grids of cell edge h, 8 h, 64 h, 512 h
constexpr double kLevelScale = 8.0;
constexpr int kBoxCtas = 1024;                        // bounding-box partials
constexpr int kBruteChunk = 8192;                     // target points per brute-force work item
constexpr unsigned kBad = SRCV_MESH_EVAL_BAD_FACE | SRCV_MESH_EVAL_NONFINITE | SRCV_MESH_EVAL_ZERO_AREA;
constexpr unsigned long long kNanBits = 0x7ff8000000000000ull;

#ifdef SRCV_HOST_EMU
inline unsigned long long atomic_min_u64(unsigned long long* p, unsigned long long v) {
  unsigned long long old = __atomic_load_n(p, __ATOMIC_RELAXED);
  while (v < old && !__atomic_compare_exchange_n(p, &old, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
  return old;
}
inline void atomic_add_u64(unsigned long long* p, unsigned long long v) { __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline unsigned read_flags(const unsigned* f) { return __atomic_load_n(f, __ATOMIC_RELAXED); }
inline double bits_double(unsigned long long u) { double d; std::memcpy(&d, &u, 8); return d; }
inline unsigned long long double_bits(double d) { unsigned long long u; std::memcpy(&u, &d, 8); return u; }
#else
__device__ __forceinline__ unsigned long long atomic_min_u64(unsigned long long* p, unsigned long long v) {
  return atomicMin(p, v);
}
__device__ __forceinline__ void atomic_add_u64(unsigned long long* p, unsigned long long v) { atomicAdd(p, v); }
// other threads of the same kernel may OR bits in while it is read: any value read is a valid snapshot
__device__ __forceinline__ unsigned read_flags(const unsigned* f) { return *reinterpret_cast<const volatile unsigned*>(f); }
__device__ __forceinline__ double bits_double(unsigned long long u) { return __longlong_as_double((long long)u); }
__device__ __forceinline__ unsigned long long double_bits(double d) { return (unsigned long long)__double_as_longlong(d); }
#endif

__device__ __forceinline__ void raise_flag(unsigned* flags, unsigned bit) {
  atomicOr(reinterpret_cast<int*>(flags), (int)bit);
}

// ---- the counter hash of the sampler (DESIGN §4.17; oracle/mesh_eval_oracle.py restates it) -------------
__device__ __forceinline__ double uniform(unsigned long long seed, unsigned long long i, unsigned draw) {
  unsigned long long x = seed * 0x9e3779b97f4a7c15ull + (3ull * i + draw + 1ull) * 0xd1b54a32d192ed03ull;
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;           // splitmix64's finaliser
  x ^= x >> 27; x *= 0x94d049bb133111ebull;
  x ^= x >> 31;
  return (double)(x >> 11) * 0x1.0p-53;               // [0, 1), 53 bits
}

// ---- a deterministic inclusive scan: tiles of kTile, each thread kPerThread consecutive items -------------

// scan of one value per thread (Hillis-Steele, fixed order): the inclusive prefix, and the exclusive one in *excl
template <class T>
__device__ __forceinline__ T block_scan(T v, T* s, T* excl) {
  const int t = threadIdx.x;
  s[t] = v;
  __syncthreads();
  for (int o = 1; o < kThreads; o <<= 1) {
    const T add = t >= o ? s[t - o] : T(0);
    __syncthreads();
    s[t] += add;
    __syncthreads();
  }
  const T r = s[t];
  if (excl) *excl = t > 0 ? s[t - 1] : T(0);
  __syncthreads();
  return r;
}

template <class T>
__global__ void __launch_bounds__(kThreads) scan_tiles_kernel(const T* __restrict__ in, long long n, T* __restrict__ tile_sum) {
  __shared__ T s[kThreads];
  const long long base = (long long)blockIdx.x * kTile + (long long)threadIdx.x * kPerThread;
  T acc = T(0);
  for (int k = 0; k < kPerThread; ++k)
    if (base + k < n) acc += in[base + k];
  const T inc = block_scan(acc, s, (T*)nullptr);
  if (threadIdx.x == kThreads - 1) tile_sum[blockIdx.x] = inc;
}

// one CTA: tile sums -> exclusive tile offsets, in place
template <class T>
__global__ void __launch_bounds__(kThreads) scan_offsets_kernel(T* __restrict__ tile, int ntiles) {
  __shared__ T s[kThreads];
  const int per = (ntiles + kThreads - 1) / kThreads, b0 = threadIdx.x * per;
  T acc = T(0);
  for (int k = 0; k < per; ++k)
    if (b0 + k < ntiles) acc += tile[b0 + k];
  T run;
  block_scan(acc, s, &run);
  for (int k = 0; k < per; ++k)
    if (b0 + k < ntiles) { const T v = tile[b0 + k]; tile[b0 + k] = run; run += v; }
}

template <class T>
__global__ void __launch_bounds__(kThreads)
scan_apply_kernel(const T* __restrict__ in, long long n, const T* __restrict__ tile_off, T* __restrict__ out) {
  __shared__ T s[kThreads];
  const long long base = (long long)blockIdx.x * kTile + (long long)threadIdx.x * kPerThread;
  T v[kPerThread];
  T acc = T(0);
  for (int k = 0; k < kPerThread; ++k) { v[k] = base + k < n ? in[base + k] : T(0); acc += v[k]; }
  T excl;
  block_scan(acc, s, &excl);
  T run = tile_off[blockIdx.x] + excl;
  for (int k = 0; k < kPerThread; ++k)
    if (base + k < n) { run += v[k]; out[base + k] = run; }
}

long long tiles_of(long long n) { return (n + kTile - 1) / kTile; }

template <class T>
void launch_scan(const T* in, long long n, T* tile, T* out, cudaStream_t stream) {
  const long long nt = tiles_of(n);
  SRCV_LAUNCH(scan_tiles_kernel<T>, (unsigned)nt, kThreads, 0, stream, in, n, tile);
  SRCV_LAUNCH(scan_offsets_kernel<T>, 1, kThreads, 0, stream, tile, (int)nt);
  SRCV_LAUNCH(scan_apply_kernel<T>, (unsigned)nt, kThreads, 0, stream, in, n, (const T*)tile, out);
  note_launch(3);
}

// ---- sampler --------------------------------------------------------------------------------------------

__device__ __forceinline__ bool finite(double x) { return fabs(x) < INFINITY; }   // false for NaN and +-inf
__device__ __forceinline__ bool finite3(double x, double y, double z) { return finite(x) && finite(y) && finite(z); }

__global__ void __launch_bounds__(kThreads)
area_kernel(const float* __restrict__ verts, int V, const int* __restrict__ faces, long long F, double* __restrict__ area,
            unsigned* flags) {
  const long long f = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (f >= F) return;
  const int i0 = faces[3 * f], i1 = faces[3 * f + 1], i2 = faces[3 * f + 2];
  if (i0 < 0 || i0 >= V || i1 < 0 || i1 >= V || i2 < 0 || i2 >= V) {
    raise_flag(flags, SRCV_MESH_EVAL_BAD_FACE);
    area[f] = 0.0;
    return;
  }
  const float* a = verts + 3ll * i0;
  const float* b = verts + 3ll * i1;
  const float* c = verts + 3ll * i2;
  const double ux = (double)b[0] - a[0], uy = (double)b[1] - a[1], uz = (double)b[2] - a[2];
  const double vx = (double)c[0] - a[0], vy = (double)c[1] - a[1], vz = (double)c[2] - a[2];
  const double cx = uy * vz - uz * vy, cy = uz * vx - ux * vz, cz = ux * vy - uy * vx;
  const double A = 0.5 * sqrt(cx * cx + cy * cy + cz * cz);
  if (!finite(A)) {
    raise_flag(flags, SRCV_MESH_EVAL_NONFINITE);
    area[f] = 0.0;
    return;
  }
  area[f] = A;
}

__global__ void __launch_bounds__(kThreads)
sample_kernel(const float* __restrict__ verts, const int* __restrict__ faces, long long F, const double* __restrict__ cdf,
              long long N, unsigned long long seed, float* __restrict__ out, unsigned* flags) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= N) return;
  const double total = cdf[F - 1];
  if ((read_flags(flags) & kBad) != 0u || !(total > 0.0)) {
    if (!(total > 0.0)) raise_flag(flags, SRCV_MESH_EVAL_ZERO_AREA);
    out[3 * i] = out[3 * i + 1] = out[3 * i + 2] = __uint_as_float(0x7fc00000u);
    return;
  }
  const double u0 = uniform(seed, (unsigned long long)i, 0), u1 = uniform(seed, (unsigned long long)i, 1),
               u2 = uniform(seed, (unsigned long long)i, 2);
  double t = ((double)i + u0) / (double)N * total;
  if (!(t < total)) t = total * (1.0 - 0x1.0p-52);       // below total: a face with cdf > t exists
  long long lo = 0, hi = F - 1;                        // first face with cdf > t
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (cdf[mid] > t) hi = mid; else lo = mid + 1;
  }
  const int* fc = faces + 3 * lo;
  const float* a = verts + 3ll * fc[0];
  const float* b = verts + 3ll * fc[1];
  const float* c = verts + 3ll * fc[2];
  const double s = sqrt(u1), wa = 1.0 - s, wb = s * (1.0 - u2), wc = s * u2;
  for (int k = 0; k < 3; ++k) out[3 * i + k] = (float)(wa * a[k] + wb * b[k] + wc * c[k]);
}

// ---- the uniform grid over the target points ------------------------------------------------------------

struct GridParams {
  double lo[3];
  double h, inv_h;
  int n[3];                       // cells per axis
};

struct GridCounters {
  unsigned queued[kLevels];                // queries each level leaves open (the last level's go to the brute force)
  unsigned overflow[kLevels];              // non-zero: a cell did not fit the level's table; the level is skipped
  unsigned long long candidates[kLevels];  // target points each level's search evaluated
};

__global__ void __launch_bounds__(kThreads)
bbox_kernel(const float* __restrict__ pts, long long n, double* __restrict__ partial, unsigned* flags) {
  __shared__ double s[6][kThreads];
  double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  bool bad = false;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
    for (int k = 0; k < 3; ++k) {
      const double v = pts[3 * i + k];
      bad |= !finite(v);
      lo[k] = fmin(lo[k], v);
      hi[k] = fmax(hi[k], v);
    }
  }
  if (bad) raise_flag(flags, SRCV_MESH_EVAL_NONFINITE);
  const int t = threadIdx.x;
  for (int k = 0; k < 3; ++k) { s[k][t] = lo[k]; s[3 + k][t] = hi[k]; }
  block_tree<kThreads>([&](int i, int j) {
    for (int k = 0; k < 3; ++k) { s[k][i] = fmin(s[k][i], s[k][j]); s[3 + k][i] = fmax(s[3 + k][i], s[3 + k][j]); }
  });
  if (t < 6) partial[blockIdx.x * 6 + t] = s[t][0];
}

// one thread: the box, every level's cell edge and cell counts; resets the queues and the statistics
__global__ void grid_params_kernel(const double* __restrict__ partial, int nparts, long long n, GridParams* levels,
                                   GridCounters* cnt) {
  double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int p = 0; p < nparts; ++p)
    for (int k = 0; k < 3; ++k) { lo[k] = fmin(lo[k], partial[6 * p + k]); hi[k] = fmax(hi[k], partial[6 * p + 3 + k]); }
  double e[3], emax = 0.0;
  for (int k = 0; k < 3; ++k) { e[k] = finite(hi[k] - lo[k]) ? hi[k] - lo[k] : 0.0; emax = fmax(emax, e[k]); }
  const double S = 2.0 * (e[0] * e[1] + e[1] * e[2] + e[2] * e[0]);
  double h = S > 0.0 ? sqrt(S / (double)n) : (e[0] + e[1] + e[2]) / (double)n;
  h = fmax(h, emax / (double)(kKeyBias - 2));          // at most 2^20 - 1 cells per axis
  if (!(h > 0.0)) h = 1.0;                              // one point, or all points equal
  for (int l = 0; l < kLevels; ++l, h *= kLevelScale) {
    GridParams* g = levels + l;
    g->h = h;
    g->inv_h = 1.0 / h;
    for (int k = 0; k < 3; ++k) {
      g->lo[k] = finite(lo[k]) ? lo[k] : 0.0;
      g->n[k] = min((int)floor(e[k] * g->inv_h) + 1, kKeyBias - 1);
    }
    cnt->queued[l] = 0u;
    cnt->overflow[l] = 0u;
    cnt->candidates[l] = 0ull;
  }
}

__device__ __forceinline__ int point_cell(double rel, const GridParams& g, int k) {
  return min(max((int)floor(rel * g.inv_h), 0), g.n[k] - 1);
}

// a level is built and searched only if the level before it left queries open
__device__ __forceinline__ bool level_idle(const GridCounters* c, int level) {
  return level > 0 && c->queued[level - 1] == 0u;
}

__global__ void __launch_bounds__(kThreads)
grid_clear_kernel(unsigned long long* __restrict__ keys, int* __restrict__ cnt, long long H, const GridCounters* gc,
                  int level) {
  if (level_idle(gc, level)) return;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < H; i += (long long)gridDim.x * kThreads) {
    keys[i] = kEmptyKey;
    cnt[i] = 0;
  }
}

// Every key sits within kMaxProbe slots of its home slot: an insert that would go farther fails (and the caller
// disables the level), so a lookup can stop after kMaxProbe slots as well.
constexpr unsigned kMaxProbe = 256;

// the table slot of cell (x, y, z), inserting it when `insert`; -1 if absent (or it did not fit)
__device__ __forceinline__ long long cell_slot(unsigned long long* keys, unsigned hmask, int x, int y, int z, bool insert) {
  const unsigned long long key = block_key(x, y, z);
  unsigned h = block_hash(key, hmask);
  const unsigned probes = hmask + 1 < kMaxProbe ? hmask + 1 : kMaxProbe;
  for (unsigned i = 0; i < probes; ++i) {
    unsigned long long k = insert ? load_key(&keys[h]) : keys[h];
    if (insert && k == kEmptyKey) {
      k = atomicCAS(&keys[h], kEmptyKey, key);
      if (k == kEmptyKey) return h;
    }
    if (k == key) return h;
    if (k == kEmptyKey) return -1;
    h = (h + 1) & hmask;
  }
  return -1;
}

// target i: level 0 reads the caller's (N,3) array, a coarser level the cell-ordered copy level 0 made
__device__ __forceinline__ float4 target(const float* __restrict__ pts, const float4* __restrict__ pts4, long long i) {
  return pts4 != nullptr ? pts4[i] : make_float4(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], 0.0f);
}

__device__ __forceinline__ long long target_cell(unsigned long long* keys, unsigned hmask, const GridParams& g, float4 p,
                                                 bool insert) {
  return cell_slot(keys, hmask, point_cell((double)p.x - g.lo[0], g, 0), point_cell((double)p.y - g.lo[1], g, 1),
                   point_cell((double)p.z - g.lo[2], g, 2), insert);
}

__global__ void __launch_bounds__(kThreads)
grid_count_kernel(const float* __restrict__ pts, const float4* __restrict__ pts4, long long n,
                  const GridParams* __restrict__ gp, unsigned long long* __restrict__ keys, int* __restrict__ cnt,
                  unsigned hmask, GridCounters* gc, int level, const unsigned* flags) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n || (read_flags(flags) & kBad) != 0u || level_idle(gc, level)) return;
  const long long s = target_cell(keys, hmask, *gp, target(pts, pts4, i), true);
  if (s >= 0) atomicAdd(reinterpret_cast<unsigned*>(&cnt[s]), 1u);
  else atomicOr(reinterpret_cast<int*>(&gc->overflow[level]), 1);
}

// start[0] = 0 before the scan writes start[1 ..]; each point takes the next free place of its cell (counting
// the cell's count down to 0 again); the order inside a cell does not matter to a minimum.  Level 0 writes the
// points (out4), a coarser level their index in level 0's copy (out_idx).
__global__ void __launch_bounds__(kThreads)
grid_scatter_kernel(const float* __restrict__ pts, const float4* __restrict__ pts4, long long n,
                    const GridParams* __restrict__ gp, unsigned long long* __restrict__ keys, int* __restrict__ cnt,
                    const int* __restrict__ start, unsigned hmask, float4* __restrict__ out4, int* __restrict__ out_idx,
                    const GridCounters* gc, int level, const unsigned* flags) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (i >= n || (read_flags(flags) & kBad) != 0u || level_idle(gc, level)) return;
  const float4 p = target(pts, pts4, i);
  const long long s = target_cell(keys, hmask, *gp, p, false);
  if (s < 0) return;
  const int j = start[s] + (int)atomicAdd(reinterpret_cast<unsigned*>(&cnt[s]), 0xffffffffu) - 1;
  if (out4 != nullptr) out4[j] = p;
  else out_idx[j] = (int)i;
}

__device__ __forceinline__ double sq_dist(double qx, double qy, double qz, float4 p) {
  const double dx = qx - (double)p.x, dy = qy - (double)p.y, dz = qz - (double)p.z;
  return dx * dx + dy * dy + dz * dz;
}

// the gap between coordinate r (relative to the box corner) and cell c's slab [c h, (c + 1) h] along one axis,
// reduced by delta (so rounded down), 0 inside
__device__ __forceinline__ double axis_gap(int c, double r, double h, double delta) {
  const double gap = fmax(c * h - r, r - (c + 1) * h) - delta;
  return gap > 0.0 ? gap * gap : 0.0;
}

// the distance from r to the nearer face of the slab of cells [c - k, c + k] along one axis
__device__ __forceinline__ double face_dist(int c, int k, double r, double h) {
  return fmin(r - (c - k) * h, (c + k + 1) * h - r);
}

// The search of one query at one level over shells of Chebyshev radius 0 .. kMaxShell; best is updated in place.
// Returns whether best is final.
__device__ __forceinline__ bool shell_search(double qx, double qy, double qz, const GridParams& g,
                                          const unsigned long long* __restrict__ keys, const int* __restrict__ start,
                                          unsigned hmask, const float4* __restrict__ pts4, const int* __restrict__ idx,
                                          double& best, unsigned long long& cand) {
  const double rx = qx - g.lo[0], ry = qy - g.lo[1], rz = qz - g.lo[2];
  const double fx = floor(rx * g.inv_h), fy = floor(ry * g.inv_h), fz = floor(rz * g.inv_h);
  const double lo = -(double)(kMaxShell + 1);
  if (!(fx >= lo && fx <= (double)(g.n[0] + kMaxShell) && fy >= lo && fy <= (double)(g.n[1] + kMaxShell) && fz >= lo &&
        fz <= (double)(g.n[2] + kMaxShell)))
    return false;                                               // no cell within kMaxShell shells
  const int cx = (int)fx, cy = (int)fy, cz = (int)fz;
  const double h = g.h, amax = fmax(fabs(rx), fmax(fabs(ry), fabs(rz)));
  for (int r = 0; r <= kMaxShell; ++r) {
    // rounding of the cell arithmetic: far below any distance that matters, far above fp64's error
    const double delta = 1e-12 * (amax + (r + 2) * h);
    for (int dx = -r; dx <= r; ++dx) {
      const int x = cx + dx;
      if (x < 0 || x >= g.n[0]) continue;
      const double gx = axis_gap(x, rx, h, delta);
      const bool ex = dx == -r || dx == r;
      for (int dy = -r; dy <= r; ++dy) {
        const int y = cy + dy;
        if (y < 0 || y >= g.n[1]) continue;
        const double gxy = gx + axis_gap(y, ry, h, delta);
        const int step = (ex || dy == -r || dy == r || r == 0) ? 1 : 2 * r;   // inside the x-y faces: z = +-r only
        for (int dz = -r; dz <= r; dz += step) {
          const int z = cz + dz;
          if (z < 0 || z >= g.n[2]) continue;
          if (gxy + axis_gap(z, rz, h, delta) > best) continue;  // the cell's box is farther than best
          const long long sl = cell_slot(const_cast<unsigned long long*>(keys), hmask, x, y, z, false);
          if (sl < 0) continue;
          const int e = start[sl + 1], b = start[sl];
          for (int j = b; j < e; ++j) best = fmin(best, sq_dist(qx, qy, qz, pts4[idx != nullptr ? idx[j] : j]));
          cand += (unsigned long long)(e - b);
        }
      }
    }
    // every unvisited point lies outside the cube [c - r, c + r]^3: at least m away
    const double m = fmin(face_dist(cx, r, rx, h), fmin(face_dist(cy, r, ry, h), face_dist(cz, r, rz, h))) - delta;
    const bool covers = cx - r <= 0 && cx + r >= g.n[0] - 1 && cy - r <= 0 && cy + r >= g.n[1] - 1 && cz - r <= 0 &&
                        cz + r >= g.n[2] - 1;
    if (covers || (m > 0.0 && best <= m * m)) return true;
  }
  return false;
}

// the grid search at one level, one query per thread: level 0 takes every query, a later level the ones the level
// before left open (queue_in, its length read on the device).  The query's squared distance, or the best so far
// and an entry in queue_out.  A level whose table overflowed passes its queries on unsearched.
// (kThreads, 1): without the minimum ptxas caps the kernel at 48 registers and spills; it needs 72
__global__ void __launch_bounds__(kThreads, 1)
near_kernel(const float* __restrict__ queries, long long nq, int level, const GridParams* __restrict__ gp,
            GridCounters* counters, const unsigned long long* __restrict__ keys, const int* __restrict__ start,
            unsigned hmask, const float4* __restrict__ pts4, const int* __restrict__ idx,
            unsigned long long* __restrict__ d2, const int* __restrict__ queue_in, int* __restrict__ queue_out,
            unsigned* flags) {
  __shared__ unsigned long long s_cand[kThreads];
  const long long t_ = (long long)blockIdx.x * kThreads + threadIdx.x;
  const long long n_in = level == 0 ? nq : (long long)counters->queued[level - 1];
  unsigned long long cand = 0;
  if (t_ < n_in && (read_flags(flags) & kBad) == 0u) {
    const long long i = level == 0 ? t_ : (long long)queue_in[t_];
    const double qx = queries[3 * i], qy = queries[3 * i + 1], qz = queries[3 * i + 2];
    double best = level == 0 ? INFINITY : bits_double(d2[i]);
    if (!finite3(qx, qy, qz)) {
      raise_flag(flags, SRCV_MESH_EVAL_NONFINITE);
    } else {
      const bool settled = counters->overflow[level] == 0u &&
                           shell_search(qx, qy, qz, *gp, keys, start, hmask, pts4, idx, best, cand);
      if (!settled) queue_out[atomicAdd(&counters->queued[level], 1u)] = (int)i;
    }
    d2[i] = double_bits(best);
  }
  const int t = threadIdx.x;
  s_cand[t] = cand;
  block_tree<kThreads>([&](int i, int j) { s_cand[i] += s_cand[j]; });
  if (t == 0 && s_cand[0] != 0ull) atomic_add_u64(&counters->candidates[level], s_cand[0]);
}

// work item = (256 queued queries, kBruteChunk target points), grid-stride; the queue length is read on the device
__global__ void __launch_bounds__(kThreads)
brute_kernel(const float* __restrict__ queries, const GridCounters* __restrict__ counters, const int* __restrict__ queue,
             const float4* __restrict__ sorted, long long np, unsigned long long* __restrict__ d2, const unsigned* flags) {
  __shared__ float4 tile[kThreads];
  if ((read_flags(flags) & kBad) != 0u) return;
  const long long nqueued = counters->queued[kLevels - 1];
  const long long qchunks = (nqueued + kThreads - 1) / kThreads, tchunks = (np + kBruteChunk - 1) / kBruteChunk;
  for (long long w = blockIdx.x; w < qchunks * tchunks; w += gridDim.x) {
    const long long qc = w / tchunks, t0 = (w % tchunks) * kBruteChunk;
    const long long qi = qc * kThreads + threadIdx.x;
    const bool live = qi < nqueued;
    const int qidx = live ? queue[qi] : 0;
    const double qx = queries[3ll * qidx], qy = queries[3ll * qidx + 1], qz = queries[3ll * qidx + 2];
    double best = INFINITY;
    const long long t1 = t0 + kBruteChunk < np ? t0 + kBruteChunk : np;
    for (long long b = t0; b < t1; b += kThreads) {
      const long long j = b + threadIdx.x;
      if (j < t1) tile[threadIdx.x] = sorted[j];
      __syncthreads();
      const int m = (int)(t1 - b < kThreads ? t1 - b : kThreads);
      for (int k = 0; k < m; ++k) best = fmin(best, sq_dist(qx, qy, qz, tile[k]));
      __syncthreads();
    }
    if (live) atomic_min_u64(&d2[qidx], double_bits(best));
  }
}

__global__ void __launch_bounds__(kThreads)
dist_out_kernel(const unsigned long long* __restrict__ d2, long long nq, double* __restrict__ out, const GridCounters* gc,
                long long* stats, const unsigned* flags) {
  const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
  const bool bad = (read_flags(flags) & kBad) != 0u;
  if (i < nq) out[i] = bad ? bits_double(kNanBits) : sqrt(bits_double(d2[i]));
  if (i == 0 && stats != nullptr)                // per level: candidates evaluated, then queries left open
    for (int l = 0; l < kLevels; ++l) {
      stats[l] = bad ? 0ll : (long long)gc->candidates[l];
      stats[kLevels + l] = bad ? 0ll : (long long)gc->queued[l];
    }
}

// ---- metrics --------------------------------------------------------------------------------------------

struct Partial {
  double sum;
  unsigned long long below;
};

__global__ void __launch_bounds__(kThreads)
reduce_kernel(const double* __restrict__ d, long long n, double tau, Partial* __restrict__ partial) {
  __shared__ double s_sum[kThreads];
  __shared__ unsigned long long s_cnt[kThreads];
  const int t = threadIdx.x;
  double sum = 0.0;
  unsigned long long cnt = 0;
  for (int k = 0; k < kPerThread; ++k) {
    const long long i = (long long)blockIdx.x * kTile + (long long)k * kThreads + t;
    if (i < n) { sum += d[i]; cnt += d[i] < tau ? 1ull : 0ull; }
  }
  s_sum[t] = sum;
  s_cnt[t] = cnt;
  block_tree<kThreads>([&](int i, int j) { s_sum[i] += s_sum[j]; s_cnt[i] += s_cnt[j]; });
  if (t == 0) partial[blockIdx.x] = Partial{s_sum[0], s_cnt[0]};
}

// one CTA: both sides' partials in a fixed order, then the six metrics and the flag word
__global__ void __launch_bounds__(kThreads)
metrics_finalize_kernel(const Partial* __restrict__ pp, int np_, long long n_pred, const Partial* __restrict__ pg, int ng_,
                        long long n_gt, double* __restrict__ out, const unsigned* flags) {
  __shared__ double s_sum[kThreads];
  __shared__ unsigned long long s_cnt[kThreads];
  const int t = threadIdx.x;
  double mean[2], share[2];
#pragma unroll
  for (int side = 0; side < 2; ++side) {
    const Partial* p = side ? pg : pp;
    const int m = side ? ng_ : np_;
    double sum = 0.0;
    unsigned long long cnt = 0;
    for (int j = t; j < m; j += kThreads) { sum += p[j].sum; cnt += p[j].below; }
    s_sum[t] = sum;
    s_cnt[t] = cnt;
    block_tree<kThreads>([&](int i, int j) { s_sum[i] += s_sum[j]; s_cnt[i] += s_cnt[j]; });
    const double n = (double)(side ? n_gt : n_pred);
    mean[side] = s_sum[0] / n;
    share[side] = (double)s_cnt[0] / n;
    __syncthreads();
  }
  if (t != 0) return;
  const unsigned f = read_flags(flags);
  const double pr = share[0], rc = share[1], nan = bits_double(kNanBits);
  const bool bad = (f & kBad) != 0u;
  out[0] = bad ? nan : mean[0];
  out[1] = bad ? nan : mean[1];
  out[2] = bad ? nan : 0.5 * (mean[0] + mean[1]);
  out[3] = bad ? nan : pr;
  out[4] = bad ? nan : rc;
  out[5] = bad ? nan : (pr + rc > 0.0 ? 2.0 * pr * rc / (pr + rc) : 0.0);
  out[6] = (double)f;
  out[7] = 0.0;
}

// ---- workspace ------------------------------------------------------------------------------------------

long long hash_slots(long long n) {
  long long h = 1024;
  while (h < 2 * n) h <<= 1;
  return h;
}

struct SampleWs {
  double* area;
  double* cdf;
  double* tile;
  size_t bytes;
};

SampleWs carve_sample(long long F, void* base) {
  SampleWs w{};
  char* p = static_cast<char*>(base);
  size_t off = 0;
  w.area = reinterpret_cast<double*>(p + off); off += align256(8 * (size_t)F);
  w.cdf = reinterpret_cast<double*>(p + off);  off += align256(8 * (size_t)F);
  w.tile = reinterpret_cast<double*>(p + off); off += align256(8 * (size_t)tiles_of(F));
  w.bytes = off;
  return w;
}

struct GridLevel {
  unsigned long long* keys;
  int* cnt;
  int* start;                     // [H + 1]
  float4* pts4;                   // level 0: the targets in cell order
  int* idx;                       // coarser levels: indices into level 0's pts4, in the level's cell order
  long long H;
};

struct GridWs {
  GridParams* g;                  // [kLevels]
  GridCounters* counters;
  double* box;
  int* tile;
  GridLevel level[kLevels];
  unsigned long long* d2;
  int* queue[2];                  // ping-pong between levels
  size_t bytes;
};

// Level l's table: the next power of two >= 2 N / 4^l slots.  Level 0's holds every cell of N points at load <= 1/2;
// a coarser level's cells are 8^l times larger, so on a surface they are about 64^l times fewer.  Should a
// level's cells not fit (points spread through a volume), its inserts fail and the level is skipped.
GridWs carve_grid(long long nq, long long np, void* base) {
  GridWs w{};
  char* p = static_cast<char*>(base);
  size_t off = 0;
  w.g = reinterpret_cast<GridParams*>(p + off);             off += align256(sizeof(GridParams) * kLevels);
  w.counters = reinterpret_cast<GridCounters*>(p + off);    off += align256(sizeof(GridCounters));
  w.box = reinterpret_cast<double*>(p + off);               off += align256(sizeof(double) * 6 * kBoxCtas);
  w.tile = reinterpret_cast<int*>(p + off);                 off += align256(4 * (size_t)tiles_of(hash_slots(np)));
  for (int l = 0; l < kLevels; ++l) {
    GridLevel& v = w.level[l];
    v.H = hash_slots((np >> (2 * l)) > 0 ? (np >> (2 * l)) : 1);
    v.keys = reinterpret_cast<unsigned long long*>(p + off);  off += align256(8 * (size_t)v.H);
    v.cnt = reinterpret_cast<int*>(p + off);                  off += align256(4 * (size_t)v.H);
    v.start = reinterpret_cast<int*>(p + off);                off += align256(4 * (size_t)(v.H + 1));
    if (l == 0) { v.pts4 = reinterpret_cast<float4*>(p + off); off += align256(16 * (size_t)np); }
    else { v.idx = reinterpret_cast<int*>(p + off);           off += align256(4 * (size_t)np); }
  }
  w.d2 = reinterpret_cast<unsigned long long*>(p + off);    off += align256(8 * (size_t)nq);
  w.queue[0] = reinterpret_cast<int*>(p + off);             off += align256(4 * (size_t)nq);
  w.queue[1] = reinterpret_cast<int*>(p + off);             off += align256(4 * (size_t)nq);
  w.bytes = off;
  return w;
}

size_t metrics_ws_bytes(long long n_pred, long long n_gt) {
  return align256(sizeof(Partial) * (size_t)tiles_of(n_pred)) + align256(sizeof(Partial) * (size_t)tiles_of(n_gt));
}

unsigned capped(long long ctas, long long cap) {
  if (ctas < 1) ctas = 1;
  return (unsigned)(ctas < cap ? ctas : cap);
}

long long sm_count() {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    sms = 132;
  return sms;
}

}  // namespace
}  // namespace mesh_eval_detail

size_t mesh_eval_workspace_bytes(const srcv_mesh_eval_args& a) {
  namespace me = mesh_eval_detail;
  size_t n = a.num_faces > 0 ? me::carve_sample(a.num_faces, nullptr).bytes : 0;
  if (a.num_queries > 0 && a.num_points > 0) {
    const size_t g = me::carve_grid(a.num_queries, a.num_points, nullptr).bytes;
    const size_t m = me::metrics_ws_bytes(a.num_queries, a.num_points);
    n = n > g ? n : g;
    n = n > m ? n : m;
  }
  return n > 256 ? n : 256;
}

cudaError_t launch_mesh_sample(const srcv_mesh_eval_args& a, const float* verts, int V, const int32_t* faces,
                               long long num_samples, unsigned long long seed, float* samples, void* workspace,
                               cudaStream_t stream) {
  namespace me = mesh_eval_detail;
  const me::SampleWs w = me::carve_sample(a.num_faces, workspace);
  const long long F = a.num_faces;
  SRCV_LAUNCH(me::area_kernel, (unsigned)((F + me::kThreads - 1) / me::kThreads), me::kThreads, 0, stream, verts, V, faces,
              F, w.area, a.flags);
  note_launch();
  me::launch_scan<double>(w.area, F, w.tile, w.cdf, stream);
  SRCV_LAUNCH(me::sample_kernel, (unsigned)((num_samples + me::kThreads - 1) / me::kThreads), me::kThreads, 0, stream,
              verts, faces, F, (const double*)w.cdf, num_samples, seed, samples, a.flags);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_nearest_distances(const srcv_mesh_eval_args& a, const float* queries, const float* points,
                                     double* dist, void* workspace, cudaStream_t stream) {
  namespace me = mesh_eval_detail;
  const me::GridWs w = me::carve_grid(a.num_queries, a.num_points, workspace);
  const long long nq = a.num_queries, np = a.num_points, sms = me::sm_count();
  const int nbox = (int)me::capped((np + me::kTile - 1) / me::kTile, me::kBoxCtas);
  SRCV_LAUNCH(me::bbox_kernel, nbox, me::kThreads, 0, stream, points, np, w.box, a.flags);
  SRCV_LAUNCH(me::grid_params_kernel, 1, 1, 0, stream, (const double*)w.box, nbox, np, w.g, w.counters);
  note_launch(2);
  const unsigned pc = (unsigned)((np + me::kThreads - 1) / me::kThreads);
  const unsigned qc = (unsigned)((nq + me::kThreads - 1) / me::kThreads);
  const float4* pts4 = w.level[0].pts4;
  for (int l = 0; l < me::kLevels; ++l) {        // each level: count, scan, scatter, then the search
    const me::GridLevel& v = w.level[l];
    const me::GridParams* g = w.g + l;
    const unsigned hmask = (unsigned)(v.H - 1);
    const float* src = l == 0 ? points : nullptr;           // a coarser level reads level 0's copy
    const float4* src4 = l == 0 ? nullptr : pts4;
    SRCV_LAUNCH(me::grid_clear_kernel, me::capped(v.H / me::kThreads, 16 * sms), me::kThreads, 0, stream, v.keys, v.cnt,
                v.H, (const me::GridCounters*)w.counters, l);
    SRCV_LAUNCH(me::grid_count_kernel, pc, me::kThreads, 0, stream, src, src4, np, g, v.keys, v.cnt, hmask, w.counters, l,
                (const unsigned*)a.flags);
    note_launch(2);
    cudaError_t err = cudaMemsetAsync(v.start, 0, sizeof(int), stream);
    if (err != cudaSuccess) return err;
    me::launch_scan<int>(v.cnt, v.H, w.tile, v.start + 1, stream);
    SRCV_LAUNCH(me::grid_scatter_kernel, pc, me::kThreads, 0, stream, src, src4, np, g, v.keys, v.cnt,
                (const int*)v.start, hmask, l == 0 ? v.pts4 : nullptr, v.idx, (const me::GridCounters*)w.counters, l,
                (const unsigned*)a.flags);
    SRCV_LAUNCH(me::near_kernel, qc, me::kThreads, 0, stream, queries, nq, l, g, w.counters,
                (const unsigned long long*)v.keys, (const int*)v.start, hmask, pts4, (const int*)v.idx, w.d2,
                (const int*)w.queue[(l + 1) & 1], w.queue[l & 1], a.flags);
    note_launch(2);
  }
  SRCV_LAUNCH(me::brute_kernel, (unsigned)(8 * sms), me::kThreads, 0, stream, queries, (const me::GridCounters*)w.counters,
              (const int*)w.queue[(me::kLevels - 1) & 1], pts4, np, w.d2, (const unsigned*)a.flags);
  note_launch();
  SRCV_LAUNCH(me::dist_out_kernel, qc, me::kThreads, 0, stream, (const unsigned long long*)w.d2, nq, dist,
              (const me::GridCounters*)w.counters, reinterpret_cast<long long*>(a.stats), (const unsigned*)a.flags);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_mesh_metrics(const srcv_mesh_eval_args& a, const double* dist_pred, const double* dist_gt,
                                double threshold, double* metrics, void* workspace, cudaStream_t stream) {
  namespace me = mesh_eval_detail;
  const long long tp = me::tiles_of(a.num_queries), tg = me::tiles_of(a.num_points);
  me::Partial* pp = static_cast<me::Partial*>(workspace);
  me::Partial* pg = reinterpret_cast<me::Partial*>(static_cast<char*>(workspace) + align256(sizeof(me::Partial) * tp));
  SRCV_LAUNCH(me::reduce_kernel, (unsigned)tp, me::kThreads, 0, stream, dist_pred, a.num_queries, threshold, pp);
  SRCV_LAUNCH(me::reduce_kernel, (unsigned)tg, me::kThreads, 0, stream, dist_gt, a.num_points, threshold, pg);
  SRCV_LAUNCH(me::metrics_finalize_kernel, 1, me::kThreads, 0, stream, (const me::Partial*)pp, (int)tp, a.num_queries,
              (const me::Partial*)pg, (int)tg, a.num_points, metrics, (const unsigned*)a.flags);
  note_launch(3);
  return cudaGetLastError();
}

}  // namespace srcv
