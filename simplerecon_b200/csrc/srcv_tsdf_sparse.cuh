// The voxel-block hashed TSDF volume (SparseTSDF, DESIGN §4.16): the dense volume's voxels and arithmetic,
// stored only where some frame can change a voxel.
//
// Layout.  The lattice is the dense one (voxel i at origin + i * voxel_size, i any int) cut into 8^3-voxel
// blocks.  A fixed pool of max_blocks blocks holds fp16 values / weights (and fp32 colour planes), each
// block z-fastest like the dense volume, and an open-addressing hash table (linear probing, a power of two
// >= 2 max_blocks slots) maps a block coordinate, packed into 63 bits, to its pool slot.  Pool slots come
// from a device counter in the state header; the whole state is initialised by one reset kernel, so a new
// block needs no initialisation (-1 / 0 / 0 like the dense volume's untouched voxels).
//
// Allocation (per launch of <= 16 frames, before the update): every block that holds a voxel that any
// of the frames could update is inserted.  A thread takes one 8x8-pixel tile of one frame and one depth
// slab of one block edge; the tile's depth range is 0 .. min(d + trunc, max_depth) over its valid pixels,
// widened by the dense kernel's cull margins, and its pixel footprint is widened by 2 + 1 % of the image
// size.  The slab's frustum piece is a convex polytope: its world AABB is the AABB of its 8 corners
// (computed in fp64 through the inverse of the fp16 projection), widened by 2^-10 of its largest
// coordinate for the fp16 rounding of the voxel coordinates.  DESIGN §4.16 has the argument.
//
// Update: one thread per z row of 8 voxels of an allocated block, through tsdf_integrate_column — the
// dense kernel's per-voxel arithmetic, so values, weights and colours are bitwise the dense volume's.
//
// Meshing: srcv_mesh.cuh's kernels over the allocated blocks with a view that reads neighbour blocks
// through a per-block table of its 26 neighbours' slots (missing -> -1 / weight 0).  A vertex's owner or a
// cube's anchor can lie in an unallocated block just below an allocated one; those "boundary" blocks are
// inserted for the extraction (mesh_begin) and taken out again afterwards (mesh_end).
//
// Overflow never writes out of bounds and never syncs: the counter keeps counting past the pool (so it
// reads back as the number of blocks needed), a block without a slot is skipped, and a failed hash probe
// or a block outside the packable range raises a header flag.  The Python layer checks the header at
// its next host-visible point.
#pragma once
#include "srcv_block_hash.cuh"
#include "srcv_kernels.h"
#ifdef SRCV_HOST_EMU
#include "emu_tc.h"
#else
#include <cuda_fp16.h>
#endif

namespace srcv {

namespace {

constexpr int kSpTile = 8;                             // pixels per allocation tile edge
constexpr int kSpThreads = 256;
constexpr int kSpMaxCtas = 2112;                       // grid-stride kernels over the pool: 16 CTAs per SM

struct alignas(16) BlockCoord { int x, y, z, pad; };

struct SparseState {
  unsigned* hdr;                 // SRCV_SPARSE_HDR_* words
  unsigned long long* keys;      // [hash_slots]
  int* vals;                     // [hash_slots] pool slot, -1 when the pool was full
  BlockCoord* coords;            // [max_blocks] block coordinate of each slot
  __half* val;                   // [max_blocks][512]
  __half* w;                     // [max_blocks][512]
  float* col;                    // [3][max_blocks * 512] or null
  int max_blocks;
  unsigned hmask;                // hash_slots - 1
};

size_t sparse_hash_slots(int max_blocks) {
  size_t h = 1024;
  while (h < 2 * (size_t)max_blocks) h <<= 1;
  return h;
}

SparseState carve_sparse(const srcv_sparse_tsdf& v, size_t* bytes = nullptr) {
  SparseState s{};
  char* p = static_cast<char*>(v.state);
  const size_t H = sparse_hash_slots(v.max_blocks), nb = (size_t)v.max_blocks, nv = nb * 512;
  size_t off = 0;
  s.hdr = reinterpret_cast<unsigned*>(p + off);            off += 256;
  s.keys = reinterpret_cast<unsigned long long*>(p + off); off += align256(8 * H);
  s.vals = reinterpret_cast<int*>(p + off);                off += align256(4 * H);
  s.coords = reinterpret_cast<BlockCoord*>(p + off);       off += align256(16 * nb);
  s.val = reinterpret_cast<__half*>(p + off);              off += align256(2 * nv);
  s.w = reinterpret_cast<__half*>(p + off);                off += align256(2 * nv);
  s.col = v.color ? reinterpret_cast<float*>(p + off) : nullptr;
  if (v.color) off += align256(12 * nv);
  s.max_blocks = v.max_blocks;
  s.hmask = (unsigned)(H - 1);
  if (bytes) *bytes = off;
  return s;
}

// pool slot of block (bx,by,bz), -1 if it is not allocated
__device__ __forceinline__ int block_lookup(const SparseState& s, int bx, int by, int bz) {
  if (!block_in_range(bx, by, bz)) return -1;
  const unsigned long long key = block_key(bx, by, bz);
  unsigned h = block_hash(key, s.hmask);
  for (unsigned i = 0; i <= s.hmask; ++i) {
    const unsigned long long k = s.keys[h];
    if (k == key) return s.vals[h];
    if (k == kEmptyKey) return -1;
    h = (h + 1) & s.hmask;
  }
  return -1;
}

__device__ void block_insert(const SparseState& s, int bx, int by, int bz) {
  if (!block_in_range(bx, by, bz)) { atomicOr(reinterpret_cast<int*>(&s.hdr[SRCV_SPARSE_HDR_RANGE]), 1); return; }
  const unsigned long long key = block_key(bx, by, bz);
  unsigned h = block_hash(key, s.hmask);
  for (unsigned i = 0; i <= s.hmask; ++i) {
    unsigned long long k = load_key(&s.keys[h]);
    if (k == kEmptyKey) k = atomicCAS(&s.keys[h], kEmptyKey, key);
    if (k == kEmptyKey) {                                 // this thread inserted the key
      const unsigned slot = atomicAdd(&s.hdr[SRCV_SPARSE_HDR_BLOCKS], 1u);
      if (slot < (unsigned)s.max_blocks) {
        s.coords[slot] = BlockCoord{bx, by, bz, 0};
        s.vals[h] = (int)slot;
      }
      return;
    }
    if (k == key) return;
    h = (h + 1) & s.hmask;
  }
  atomicAdd(&s.hdr[SRCV_SPARSE_HDR_LOST], 1u);
}

__device__ __forceinline__ unsigned pool_blocks(const SparseState& s) {
  const unsigned n = s.hdr[SRCV_SPARSE_HDR_BLOCKS];
  return n < (unsigned)s.max_blocks ? n : (unsigned)s.max_blocks;
}

__global__ void __launch_bounds__(kSpThreads) sparse_reset_kernel(SparseState s) {
  const size_t stride = (size_t)gridDim.x * blockDim.x, t0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (size_t i = t0; i <= s.hmask; i += stride) { s.keys[i] = kEmptyKey; s.vals[i] = -1; }
  const size_t nv = (size_t)s.max_blocks * 512;
  const __half m1 = __float2half_rn(-1.0f), z = __float2half_rn(0.0f);
  for (size_t i = t0; i < nv; i += stride) {
    s.val[i] = m1;
    s.w[i] = z;
    if (s.col) { s.col[i] = 0.0f; s.col[nv + i] = 0.0f; s.col[2 * nv + i] = 0.0f; }
  }
  if (t0 < SRCV_SPARSE_HDR_WORDS) s.hdr[t0] = 0u;
}

// per (frame, 8x8 tile): the far end of the depth range any voxel updated through the tile's valid pixels
// can have, min(d + trunc, max_depth) with fp16 trunc / max_depth; -1 if no pixel of the tile is valid
__global__ void __launch_bounds__(kSpThreads)
sparse_tile_depth_kernel(TsdfParams p, const __half* __restrict__ depth, const uint8_t* __restrict__ mask, int tiles_x,
                         int tiles_y, float* __restrict__ tile_far) {
  const int t = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (t >= p.B * tiles_x * tiles_y) return;
  const int b = t / (tiles_x * tiles_y), ty = (t / tiles_x) % tiles_y, tx = t % tiles_x;
  const float trunc_h = -p.neg_trunc_h;
  float far = -1.0f;
  for (int y = ty * kSpTile; y < min(ty * kSpTile + kSpTile, p.H); ++y)
    for (int x = tx * kSpTile; x < min(tx * kSpTile + kSpTile, p.W); ++x) {
      const size_t pix = ((size_t)b * p.H + y) * p.W + x;
      float ds = __half2float(depth[pix]);
      if (mask != nullptr && mask[pix] == 0) ds = -1.0f;
      if (!(ds > 0.0f) || !(tsdf_confidence(p, ds) > 0.0f)) continue;   // the pixel can update no voxel
      far = fmaxf(far, fminf(ds + trunc_h, p.max_depth_h));
    }
  tile_far[t] = far;
}

// per (frame, tile, depth slab): insert every block whose voxels the slab's widened frustum piece can hold
__global__ void __launch_bounds__(kSpThreads)
sparse_alloc_kernel(TsdfParams p, const TsdfFrame* __restrict__ frames, const float* __restrict__ tile_far,
                    int tiles_x, int tiles_y, int slabs, SparseState s) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int ntiles = tiles_x * tiles_y;
  if (t >= (long long)p.B * ntiles * slabs) return;
  const int k = (int)(t % slabs), tile = (int)((t / slabs) % ntiles), b = (int)(t / ((long long)slabs * ntiles));
  const float far_t = tile_far[b * ntiles + tile];
  if (!(far_t > 0.0f)) return;
  const double slab = 8.0 * p.voxel_size;
  const double zfar = (double)far_t * 1.01 + 0.01;       // the dense kernel's cull margin on the far limit
  const double z0 = k * slab;
  if (z0 >= zfar) return;
  const double z1 = fmin((k + 1) * slab, zfar);
  // pixel x covers u = cam_x / cam_z in [x, x + 1] (grid_sample's nearest with align_corners=False)
  const int tx = tile % tiles_x, ty = tile / tiles_x;
  const double mx = 2.0 + 0.01 * p.W, my = 2.0 + 0.01 * p.H;
  const double u0 = tx * kSpTile - mx, u1 = min(tx * kSpTile + kSpTile, p.W) + mx;
  const double v0 = ty * kSpTile - my, v1 = min(ty * kSpTile + kSpTile, p.H) + my;
  // world = M^-1 (cam - t) with M, t the fp16 projection the update uses
  const float* P = frames[b].P;
  // a non-finite entry (an fp16 overflow of K @ E) makes every voxel's pixel or depth non-finite in the update,
  // so the frame changes no voxel: nothing to allocate (and no corner below can come out NaN)
  for (int q = 0; q < 12; ++q)
    if (!(fabsf(P[q]) <= 65504.0f)) return;           // the fp16 maximum: P was rounded to half
  const double a = P[0], bb = P[1], c = P[2], d = P[4], e = P[5], f = P[6], g = P[8], h = P[9], i = P[10];
  const double A = e * i - f * h, B = f * g - d * i, Cc = d * h - e * g;
  const double det = a * A + bb * B + c * Cc;
  if (!(fabs(det) > 0.0)) { atomicOr(reinterpret_cast<int*>(&s.hdr[SRCV_SPARSE_HDR_RANGE]), 2); return; }
  const double inv[9] = {A / det, (c * h - bb * i) / det, (bb * f - c * e) / det,
                         B / det, (a * i - c * g) / det, (c * d - a * f) / det,
                         Cc / det, (bb * g - a * h) / det, (a * e - bb * d) / det};
  double lo[3] = {1e300, 1e300, 1e300}, hi[3] = {-1e300, -1e300, -1e300};
  for (int q = 0; q < 8; ++q) {
    const double z = (q & 4) ? z1 : z0, u = (q & 1) ? u1 : u0, vv = (q & 2) ? v1 : v0;
    const double cam[3] = {u * z - P[3], vv * z - P[7], z - P[11]};
    for (int r = 0; r < 3; ++r) {
      const double w = inv[3 * r] * cam[0] + inv[3 * r + 1] * cam[1] + inv[3 * r + 2] * cam[2];
      lo[r] = fmin(lo[r], w);
      hi[r] = fmax(hi[r], w);
    }
  }
  double amax = 0.0;
  for (int r = 0; r < 3; ++r) amax = fmax(amax, fmax(fabs(lo[r]), fabs(hi[r])));
  const double margin = amax * (1.0 / 1024.0) + 1e-4;  // >= twice the fp16 half-ulp of any coordinate in the box
  const double o[3] = {p.ox, p.oy, p.oz};
  int blo[3], bhi[3];
  for (int r = 0; r < 3; ++r) {
    const double ilo = floor((lo[r] - margin - o[r]) / p.voxel_size), ihi = ceil((hi[r] + margin - o[r]) / p.voxel_size);
    // blocks -2^20 + 1 .. 2^20 - 1: one short of the packable range at the low end, so that meshing can insert
    // the boundary block below every allocated block
    if (!(ilo >= -8.0 * (kKeyBias - 1) && ihi < 8.0 * kKeyBias)) {
      atomicOr(reinterpret_cast<int*>(&s.hdr[SRCV_SPARSE_HDR_RANGE]), 1);
      return;
    }
    blo[r] = (int)floor(ilo / 8.0);
    bhi[r] = (int)floor(ihi / 8.0);
  }
  for (int bx = blo[0]; bx <= bhi[0]; ++bx)
    for (int by = blo[1]; by <= bhi[1]; ++by)
      for (int bz = blo[2]; bz <= bhi[2]; ++bz) block_insert(s, bx, by, bz);
}

// one thread per z row of 8 voxels of an allocated block, grid-stride over the pool
template <bool kColor>
__global__ void __launch_bounds__(kSpThreads)
sparse_integrate_kernel(TsdfParams p, const TsdfFrame* __restrict__ frames, const __half* __restrict__ depth,
                        const uint8_t* __restrict__ mask, SparseState s, TsdfColorParams cp) {
  const long long rows = (long long)pool_blocks(s) * 64;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < rows; t += (long long)gridDim.x * blockDim.x) {
    const int slot = (int)(t >> 6), r = (int)(t & 63);
    const BlockCoord bc = s.coords[slot];
    tsdf_integrate_column<8, kColor>(p, frames, depth, mask, s.val, s.w, cp, bc.x * 8 + (r >> 3), bc.y * 8 + (r & 7),
                                     bc.z * 8, (size_t)slot * 512 + (size_t)r * 8);
  }
}

// the dense (X,Y,Z) read-back of the lattice box starting at voxel lo
__global__ void __launch_bounds__(kSpThreads)
sparse_read_box_kernel(SparseState s, int lx, int ly, int lz, int X, int Y, int Z, __half* __restrict__ values,
                       __half* __restrict__ weights, float* __restrict__ colors) {
  const size_t n = (size_t)X * Y * Z, stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int x = lx + (int)(i / ((size_t)Y * Z)), y = ly + (int)((i / Z) % Y), z = lz + (int)(i % Z);
    const int slot = block_lookup(s, x >> 3, y >> 3, z >> 3);
    const size_t j = (size_t)slot * 512 + (((x & 7) << 6) | ((y & 7) << 3) | (z & 7));
    values[i] = slot >= 0 ? s.val[j] : __float2half_rn(-1.0f);
    weights[i] = slot >= 0 ? s.w[j] : __float2half_rn(0.0f);
    if (colors != nullptr) {
      const size_t nv = (size_t)s.max_blocks * 512;
      for (int ch = 0; ch < 3; ++ch) colors[ch * n + i] = slot >= 0 ? s.col[ch * nv + j] : 0.0f;
    }
  }
}

// ---- meshing -------------------------------------------------------------------------------------------

// the 7 blocks below each allocated block (offsets in {0,-1}^3 \ 0): where a vertex owner or cube anchor
// next to an allocated block can lie
__global__ void __launch_bounds__(kSpThreads) sparse_boundary_kernel(SparseState s, int n) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 7ll * n) return;
  const int slot = (int)(t / 7), d = (int)(t % 7) + 1;
  const BlockCoord c = s.coords[slot];
  block_insert(s, c.x - (d & 1), c.y - ((d >> 1) & 1), c.z - (d >> 2));
}

// take the boundary blocks out again: they were inserted after every allocated block, so no allocated
// block's probe sequence runs through their slots, and emptying them restores the table exactly
__global__ void __launch_bounds__(kSpThreads) sparse_release_kernel(SparseState s, int n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x, t0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (size_t i = t0; i <= s.hmask; i += stride)
    if (s.keys[i] != kEmptyKey && (s.vals[i] < 0 || s.vals[i] >= n)) { s.keys[i] = kEmptyKey; s.vals[i] = -1; }
  if (t0 == 0) { s.hdr[SRCV_SPARSE_HDR_BLOCKS] = (unsigned)n; s.hdr[SRCV_SPARSE_HDR_LOST] = 0u; }
}

// the slots of each block's 3x3x3 neighbourhood (-1: not allocated)
__global__ void __launch_bounds__(kSpThreads) sparse_neighbour_kernel(SparseState s, int n, int* __restrict__ nbr) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 27ll * n) return;
  const int slot = (int)(t / 27), j = (int)(t % 27);
  const BlockCoord c = s.coords[slot];
  nbr[t] = block_lookup(s, c.x + j / 9 - 1, c.y + (j / 3) % 3 - 1, c.z + j % 3 - 1);
}

struct SparseMeshParams {
  const __half* val;
  const __half* w;
  const BlockCoord* coords;
  const int* nbr;
  int nblocks;
  float ox, oy, oz, vs;
  int world, single;
};

struct SparseChunk {
  int x, y, z0;
  bool live;
  int slot;
};

// what srcv_mesh.cuh's helpers see of one block and its neighbours: an unbounded lattice
struct SparseView {
  const __half* val;
  const __half* w;
  const int* nbr;                // the home block's 27 neighbour slots
  int bx, by, bz;                // the home block's first voxel
  float ox, oy, oz, vs;
  int world, single;
};

__device__ __forceinline__ SparseView view_of(const SparseMeshParams& p, const SparseChunk& c) {
  return SparseView{p.val, p.w, p.nbr + (size_t)c.slot * 27, c.x & ~7, c.y & ~7, c.z0 & ~7,
                    p.ox, p.oy, p.oz, p.vs, p.world, p.single};
}

__device__ __forceinline__ int nb_slot(const SparseView& v, int x, int y, int z) {
  return v.nbr[(((x - v.bx) >> 3) + 1) * 9 + (((y - v.by) >> 3) + 1) * 3 + ((z - v.bz) >> 3) + 1];
}

__device__ __forceinline__ int in_block(int x, int y, int z) { return ((x & 7) << 6) | ((y & 7) << 3) | (z & 7); }

__device__ __forceinline__ float ld(const SparseView& v, int x, int y, int z) {
  const int s = nb_slot(v, x, y, z);
  return s < 0 ? -1.0f : clamp1(__half2float(v.val[(size_t)s * 512 + in_block(x, y, z)]));
}
__device__ __forceinline__ float wt(const SparseView& v, int x, int y, int z) {
  const int s = nb_slot(v, x, y, z);
  return s < 0 ? 0.0f : __half2float(v.w[(size_t)s * 512 + in_block(x, y, z)]);
}
// every voxel a vertex or colour is asked of lies in an allocated or boundary block (DESIGN §4.16)
__device__ __forceinline__ size_t vslot(const SparseView& v, int x, int y, int z) {
  return (size_t)nb_slot(v, x, y, z) * 512 + in_block(x, y, z);
}
__device__ __forceinline__ bool cube_exists(const SparseView&, int, int, int) { return true; }
__device__ __forceinline__ bool has_next(const SparseView&, int, int) { return true; }
__device__ __forceinline__ bool at_low(const SparseView&, int, int) { return false; }
__device__ __forceinline__ bool at_high(const SparseView&, int, int) { return false; }

template <int VEC>
__device__ SparseChunk chunk_of(const SparseMeshParams& p) {
  static_assert(VEC == 8, "a chunk is one z row of a block");
  const long long t = (long long)blockIdx.x * kMeshThreads + threadIdx.x;
  SparseChunk c{0, 0, 0, false, 0};
  if (t < (long long)p.nblocks * 64) {
    c.slot = (int)(t >> 6);
    const int r = (int)(t & 63);
    const BlockCoord b = p.coords[c.slot];
    c.x = b.x * 8 + (r >> 3);
    c.y = b.y * 8 + (r & 7);
    c.z0 = b.z * 8;
    const SparseView v = view_of(p, c);
    int n_in = 0;             // the 4 rows (x|x+1, y|y+1) over z0 .. z0+8 share one sign: nothing to mesh
    for (int q = 0; q < 4; ++q)
      for (int i = 0; i <= 8; ++i) n_in += ld(v, c.x + (q & 1), c.y + (q >> 1), c.z0 + i) < 0.0f;
    c.live = !(n_in == 0 || n_in == 36);
  }
  return c;
}

// srcv_mesh.cuh's kernels on the voxel-block volume
constexpr auto sparse_count_kernel = &mesh_count_kernel<kMeshVec, SparseMeshParams>;
constexpr auto sparse_vertex_kernel = &mesh_vertex_kernel<kMeshVec, SparseMeshParams>;
constexpr auto sparse_vertex_color_kernel = &mesh_vertex_color_kernel<kMeshVec, SparseMeshParams>;
constexpr auto sparse_face_kernel = &mesh_face_kernel<kMeshVec, SparseMeshParams>;

struct SparseMeshWs {
  long long* totals;
  int* block_counts;
  long long* block_off;
  int* vbase;
  int* nbr;
  size_t bytes;
};

long long sparse_mesh_ctas(int nblocks) { return ((long long)nblocks * 64 + kMeshThreads - 1) / kMeshThreads; }

SparseMeshWs carve_sparse_mesh(int nblocks, void* base) {
  SparseMeshWs w{};
  char* p = static_cast<char*>(base);
  const long long nc = sparse_mesh_ctas(nblocks);
  size_t off = 0;
  w.totals = reinterpret_cast<long long*>(p + off);  off += 256;
  w.block_counts = reinterpret_cast<int*>(p + off);  off += align256(sizeof(int) * 2 * (size_t)nc);
  w.block_off = reinterpret_cast<long long*>(p + off); off += align256(sizeof(long long) * 2 * (size_t)nc);
  w.vbase = reinterpret_cast<int*>(p + off);         off += align256(sizeof(int) * 512 * (size_t)nblocks);
  w.nbr = reinterpret_cast<int*>(p + off);           off += align256(sizeof(int) * 27 * (size_t)nblocks);
  w.bytes = off;
  return w;
}

SparseMeshParams sparse_mesh_params(const srcv_sparse_tsdf& v, const srcv_sparse_mesh_args& a, const int* nbr) {
  const SparseState s = carve_sparse(v);
  SparseMeshParams p;
  p.val = s.val; p.w = s.w; p.coords = s.coords; p.nbr = nbr; p.nblocks = a.blocks;
  p.ox = a.origin[0]; p.oy = a.origin[1]; p.oz = a.origin[2]; p.vs = v.voxel_size;
  p.world = a.scale_to_world != 0;
  p.single = a.single_mesh != 0;
  return p;
}

unsigned grid_for(long long threads, long long cap) {
  long long g = (threads + kSpThreads - 1) / kSpThreads;
  if (g < 1) g = 1;
  return (unsigned)(g < cap ? g : cap);
}

}  // namespace

size_t sparse_tsdf_state_bytes(const srcv_sparse_tsdf& v) {
  size_t bytes = 0;
  srcv_sparse_tsdf tmp = v;
  tmp.state = nullptr;
  carve_sparse(tmp, &bytes);
  return bytes;
}

size_t sparse_tsdf_workspace_bytes(const srcv_tsdf_frames& f) {
  const int nb = f.B < kMaxFrames ? f.B : kMaxFrames;
  const size_t tiles = (size_t)((f.W + kSpTile - 1) / kSpTile) * ((f.H + kSpTile - 1) / kSpTile);
  return align256(sizeof(TsdfFrame) * kMaxFrames) + align256(sizeof(float) * nb * tiles);
}

cudaError_t launch_sparse_tsdf_reset(const srcv_sparse_tsdf& v, cudaStream_t stream) {
  const SparseState s = carve_sparse(v);
  SRCV_LAUNCH(sparse_reset_kernel, grid_for((long long)v.max_blocks * 512, kSpMaxCtas), kSpThreads, 0, stream, s);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_sparse_tsdf_integrate(const srcv_sparse_tsdf& v, const srcv_tsdf_frames& f, void* workspace,
                                         cudaStream_t stream, const srcv_tsdf_color* color) {
  const SparseState s = carve_sparse(v);
  TsdfFrame* frames = reinterpret_cast<TsdfFrame*>(workspace);
  float* tile_far = reinterpret_cast<float*>(static_cast<char*>(workspace) + align256(sizeof(TsdfFrame) * kMaxFrames));
  const int tiles_x = (f.W + kSpTile - 1) / kSpTile, tiles_y = (f.H + kSpTile - 1) / kSpTile;
  const float max_depth_h = __half2float(__float2half_rn(f.max_depth));
  const int slabs = (int)ceil(((double)max_depth_h * 1.01 + 0.01) / (8.0 * v.voxel_size));
  for (int b0 = 0; b0 < f.B; b0 += kMaxFrames) {
    const int nb = (f.B - b0 < kMaxFrames) ? (f.B - b0) : kMaxFrames;
    const __half* K = reinterpret_cast<const __half*>(f.K) + (size_t)b0 * 16;
    const __half* E = reinterpret_cast<const __half*>(f.cam_T_world) + (size_t)b0 * 16;
    SRCV_LAUNCH(tsdf_prep_kernel, 1, 256, 0, stream, K, E, nb, frames);
    const TsdfParams p = tsdf_params(v.origin, v.voxel_size, v.truncation_voxels, v.max_weight, f, nb);
    const __half* depth = reinterpret_cast<const __half*>(f.depth) + (size_t)b0 * f.H * f.W;
    const uint8_t* mask = f.depth_mask ? f.depth_mask + (size_t)b0 * f.H * f.W : nullptr;
    const long long ntiles = (long long)nb * tiles_x * tiles_y;
    SRCV_LAUNCH(sparse_tile_depth_kernel, grid_for(ntiles, 1ll << 30), kSpThreads, 0, stream, p, depth, mask, tiles_x,
                tiles_y, tile_far);
    SRCV_LAUNCH(sparse_alloc_kernel, grid_for(ntiles * slabs, 1ll << 30), kSpThreads, 0, stream, p, frames, tile_far,
                tiles_x, tiles_y, slabs, s);
    const unsigned grid = grid_for((long long)v.max_blocks * 64, kSpMaxCtas);
    if (color != nullptr) {
      const TsdfColorParams cp = tsdf_color_params(*color, s.col, (size_t)v.max_blocks * 512, f, b0);
      SRCV_LAUNCH(sparse_integrate_kernel<true>, grid, kSpThreads, 0, stream, p, frames, depth, mask, s, cp);
    } else {
      SRCV_LAUNCH(sparse_integrate_kernel<false>, grid, kSpThreads, 0, stream, p, frames, depth, mask, s, TsdfColorParams{});
    }
    note_launch(4);
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) return err;
  }
  return cudaSuccess;
}

cudaError_t launch_sparse_tsdf_read_box(const srcv_sparse_tsdf& v, const int lo[3], const int dims[3], void* values,
                                        void* weights, void* colors, cudaStream_t stream) {
  const SparseState s = carve_sparse(v);
  SRCV_LAUNCH(sparse_read_box_kernel, grid_for((long long)dims[0] * dims[1] * dims[2], kSpMaxCtas), kSpThreads, 0,
              stream, s, lo[0], lo[1], lo[2], dims[0], dims[1], dims[2], reinterpret_cast<__half*>(values),
              reinterpret_cast<__half*>(weights), reinterpret_cast<float*>(colors));
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_sparse_mesh_begin(const srcv_sparse_tsdf& v, int blocks, cudaStream_t stream) {
  if (blocks == 0) return cudaSuccess;
  SRCV_LAUNCH(sparse_boundary_kernel, grid_for(7ll * blocks, 1ll << 30), kSpThreads, 0, stream, carve_sparse(v), blocks);
  note_launch();
  return cudaGetLastError();
}

cudaError_t launch_sparse_mesh_end(const srcv_sparse_tsdf& v, int blocks, cudaStream_t stream) {
  const SparseState s = carve_sparse(v);
  SRCV_LAUNCH(sparse_release_kernel, grid_for((long long)s.hmask + 1, kSpMaxCtas), kSpThreads, 0, stream, s, blocks);
  note_launch();
  return cudaGetLastError();
}

size_t sparse_mesh_workspace_bytes(const srcv_sparse_mesh_args& a) { return carve_sparse_mesh(a.blocks, nullptr).bytes; }

cudaError_t launch_sparse_mesh_count(const srcv_sparse_tsdf& v, const srcv_sparse_mesh_args& a, long long* counts,
                                     void* workspace, cudaStream_t stream) {
  const SparseMeshWs w = carve_sparse_mesh(a.blocks, workspace);
  const SparseMeshParams p = sparse_mesh_params(v, a, w.nbr);
  const unsigned nc = (unsigned)sparse_mesh_ctas(a.blocks);
  if (a.blocks > 0) {
    SRCV_LAUNCH(sparse_neighbour_kernel, grid_for(27ll * a.blocks, 1ll << 30), kSpThreads, 0, stream, carve_sparse(v),
                a.blocks, w.nbr);
    SRCV_LAUNCH(sparse_count_kernel, nc, kMeshThreads, 0, stream, p, w.block_counts);
    note_launch(2);
  }
  SRCV_LAUNCH(mesh_scan_kernel, 1, kMeshScanThreads, 0, stream, w.block_counts, (long long)(a.blocks > 0 ? nc : 0),
              w.block_off, w.totals, counts);
  note_launch();
  return cudaGetLastError();
}

cudaError_t sparse_mesh_read_totals(const srcv_sparse_mesh_args& a, void* workspace, long long totals[2],
                                    cudaStream_t stream) {
  const SparseMeshWs w = carve_sparse_mesh(a.blocks, workspace);
#ifdef SRCV_HOST_EMU
  (void)stream;
  std::memcpy(totals, w.totals, 2 * sizeof(long long));
  return cudaSuccess;
#else
  cudaError_t err = cudaMemcpyAsync(totals, w.totals, 2 * sizeof(long long), cudaMemcpyDeviceToHost, stream);
  if (err != cudaSuccess) return err;
  return cudaStreamSynchronize(stream);
#endif
}

cudaError_t launch_sparse_mesh_extract(const srcv_sparse_tsdf& v, const srcv_sparse_mesh_args& a, float* verts,
                                       float* normals, float* vert_colors, int32_t* faces, void* workspace,
                                       cudaStream_t stream) {
  if (a.blocks == 0) return cudaSuccess;
  const SparseMeshWs w = carve_sparse_mesh(a.blocks, workspace);
  const SparseMeshParams p = sparse_mesh_params(v, a, w.nbr);
  const unsigned nc = (unsigned)sparse_mesh_ctas(a.blocks);
  SRCV_LAUNCH(sparse_vertex_kernel, nc, kMeshThreads, 0, stream, p, w.block_counts,
              w.block_off, w.vbase, verts, normals);
  note_launch();
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return err;
  if (vert_colors != nullptr) {
    SRCV_LAUNCH(sparse_vertex_color_kernel, nc, kMeshThreads, 0, stream, p, w.block_counts,
                w.block_off, carve_sparse(v).col, (size_t)v.max_blocks * 512, vert_colors);
    note_launch();
    err = cudaGetLastError();
    if (err != cudaSuccess) return err;
  }
  SRCV_LAUNCH(sparse_face_kernel, nc, kMeshThreads, 0, stream, p, w.block_counts,
              w.block_off, w.vbase, faces);
  note_launch();
  return cudaGetLastError();
}

}  // namespace srcv
