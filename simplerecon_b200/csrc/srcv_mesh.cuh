// Marching-cubes mesh extraction from the fused TSDF volume (the reference's TSDF.to_mesh,
// tools/tsdf.py:125-157, which copies the fp16 volume to the host and runs scikit-image there).
//
// Semantics (DESIGN §4.10; oracle/mesh_oracle.py restates them in fp64):
//   - values fp16 (X,Y,Z), z fastest, taken to fp32 and clamped to [-1, 1]; level 0; a corner is
//     inside iff its value is < 0; cube (x,y,z) exists for x < X-1, y < Y-1, z < Z-1;
//   - one vertex per crossing edge (two axis neighbours, exactly one inside), owned by the edge's
//     lower endpoint; vertices ordered by owner in linear order, then axis x, y, z; position
//     a + t (b - a), t = (0 - v_a) / (v_b - v_a) in fp32;
//   - normal = central-difference gradient (one-sided at the border) interpolated with t,
//     normalised, pointing toward increasing values; a zero gradient gives a zero normal;
//   - faces cube by cube in linear order, then in the order of the generated table
//     (srcv_mc_table.h); a triangle two of whose vertices have bitwise-equal fp32 index-space
//     coordinates is dropped (its vertices stay);
//   - single_mesh: a cube is processed only if its 8 corners have weight > 0, and a vertex is
//     emitted only if a processed cube contains its edge;
//   - scale_to_world: world = origin + v * voxel_size in fp32 (origin as given, fp16-rounded by
//     the caller as the reference's half origin is).
//
// Four launches, all reading the volume coalesced along z, no atomics on the output order:
//   count  : a thread owns VEC consecutive voxels of a z row; it first loads the 4 rows
//            (x|x+1, y|y+1) of its chunk plus the one-voxel z halo and stops there if all share a
//            sign (nearly all of a scene-sized volume); otherwise it counts the vertices its
//            voxels own and the non-degenerate faces of the cubes they anchor.  One (V, F) total
//            per block;
//   scan   : one CTA turns the block totals into exclusive block offsets and the two grand totals;
//   verts  : a block whose count-pass total is zero returns at once; the others recount, block
//            scan, write vertices / normals and each owner's first vertex index into a dense int32
//            array (only active voxels' entries are touched);
//   faces  : likewise for faces; a vertex index is the owner's first index plus the rank of the
//            edge's axis among the owner's emitted edges.
// Blocks cover contiguous ranges of chunks in linear order and scan in a fixed order, so the
// output is deterministic and canonically ordered.
//
// This file is compiled as part of srcv_tsdf.cu's translation unit (included at its end): the
// TSDF unit holds both operations on the fused volume, integration and mesh extraction.  The helpers
// and kernels are templates over the volume they read (MeshParams here; the voxel-block view of
// srcv_tsdf_sparse.cuh, which instantiates the same kernels on an unbounded lattice).
#pragma once
#include "srcv_kernels.h"
#ifdef SRCV_HOST_EMU
#include "emu_tc.h"      // tests/emu: __half and its conversions on the host
#else
#include <cuda_fp16.h>
#endif
#include "srcv_mc_table.h"

namespace srcv {

namespace {

constexpr int kMeshThreads = 256;        // threads per block of the three voxel passes
constexpr int kMeshScanThreads = 512;    // the one block of the scan pass
constexpr int kMeshVec = 8;              // voxels per thread on the vector path (one 16-byte load per row)

struct MeshParams {
  const __half* val;
  const __half* w;
  int X, Y, Z, zchunks;              // zchunks = Z / VEC
  float ox, oy, oz, vs;
  int world, single;
};

__device__ __forceinline__ size_t vidx(const MeshParams& p, int x, int y, int z) {
  return ((size_t)x * p.Y + y) * p.Z + z;
}

__device__ __forceinline__ float clamp1(float v) { return fminf(fmaxf(v, -1.0f), 1.0f); }

__device__ __forceinline__ float ld(const MeshParams& p, int x, int y, int z) {
  return clamp1(__half2float(p.val[vidx(p, x, y, z)]));
}

__device__ __forceinline__ int dim(const MeshParams& p, int a) { return a == 0 ? p.X : (a == 1 ? p.Y : p.Z); }

// The voxel access the helpers and kernels below are written against, so that the voxel-block volume
// (srcv_tsdf_sparse.cuh) runs the same code with its own overloads: the weight, the bounds of the lattice,
// and the index of a voxel's slot in the per-voxel arrays (vbase, colour planes).
__device__ __forceinline__ float wt(const MeshParams& p, int x, int y, int z) { return __half2float(p.w[vidx(p, x, y, z)]); }
__device__ __forceinline__ bool cube_exists(const MeshParams& p, int x, int y, int z) {
  return !(x < 0 || y < 0 || z < 0 || x >= p.X - 1 || y >= p.Y - 1 || z >= p.Z - 1);
}
__device__ __forceinline__ bool has_next(const MeshParams& p, int a, int c) { return c + 1 < dim(p, a); }
__device__ __forceinline__ bool at_low(const MeshParams&, int, int c) { return c == 0; }
__device__ __forceinline__ bool at_high(const MeshParams& p, int a, int c) { return c == dim(p, a) - 1; }

__device__ __forceinline__ int popc3(unsigned m) { return (int)(m & 1u) + (int)((m >> 1) & 1u) + (int)((m >> 2) & 1u); }

// the cube anchored at (x,y,z) exists and is processed
template <class P>
__device__ __forceinline__ bool cube_ok(const P& p, int x, int y, int z) {
  if (!cube_exists(p, x, y, z)) return false;
  if (!p.single) return true;
#pragma unroll
  for (int c = 0; c < 8; ++c)
    if (!(wt(p, x + (c & 1), y + ((c >> 1) & 1), z + (c >> 2)) > 0.0f)) return false;
  return true;
}

// bit a: the edge along axis a from (x,y,z) crosses the level and is emitted
template <class P>
__device__ __forceinline__ unsigned owned_edges(const P& p, int x, int y, int z) {
  const bool in0 = ld(p, x, y, z) < 0.0f;
  unsigned m = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int c = a == 0 ? x : (a == 1 ? y : z);
    if (!has_next(p, a, c)) continue;
    if ((ld(p, x + (a == 0), y + (a == 1), z + (a == 2)) < 0.0f) == in0) continue;
    if (p.single) {
      // the (up to) four cubes that contain the edge: anchors owner - {0,1} e_b - {0,1} e_c
      bool any = false;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int db = j & 1, dc = j >> 1;
        const int ax = x - (a == 0 ? 0 : db), ay = y - (a == 1 ? 0 : (a == 0 ? db : dc)), az = z - (a == 2 ? 0 : dc);
        any = any || cube_ok(p, ax, ay, az);
      }
      if (!any) continue;
    }
    m |= 1u << a;
  }
  return m;
}

__device__ __forceinline__ float edge_t(float va, float vb) { return __fdiv_rn(-va, __fadd_rn(vb, -va)); }

// inside-mask of the cube anchored at (x,y,z), and its 8 corner values
template <class P>
__device__ __forceinline__ unsigned cube_case(const P& p, int x, int y, int z, float v[8]) {
  unsigned cs = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    v[c] = ld(p, x + (c & 1), y + ((c >> 1) & 1), z + (c >> 2));
    cs |= (v[c] < 0.0f ? 1u : 0u) << c;
  }
  return cs;
}

// lower-corner offset and axis of cube edge e (edge e = 4 axis + j, see srcv_mc_table.h)
__device__ __forceinline__ void edge_geom(int e, int o[3], int& a) {
  a = e >> 2;
  const int j = e & 3;
  o[0] = a == 0 ? 0 : (j & 1);
  o[1] = a == 1 ? 0 : (a == 0 ? (j & 1) : (j >> 1));
  o[2] = a == 2 ? 0 : (j >> 1);
}

// v[i] by compare-and-select: keeps the corner values in registers (a dynamic index would put them in
// local memory)
__device__ __forceinline__ float pick8(const float v[8], int i) {
  float r = v[0];
#pragma unroll
  for (int c = 1; c < 8; ++c) r = (i == c) ? v[c] : r;
  return r;
}

// fp32 index-space position of the vertex on edge e of the cube at (x,y,z)
__device__ __forceinline__ void edge_pos(int x, int y, int z, int e, const float v[8], float out[3]) {
  int o[3], a;
  edge_geom(e, o, a);
  const int lo = o[0] | (o[1] << 1) | (o[2] << 2), hi = lo | (1 << a);
  out[0] = (float)(x + o[0]);
  out[1] = (float)(y + o[1]);
  out[2] = (float)(z + o[2]);
  const float t = edge_t(pick8(v, lo), pick8(v, hi));
  out[a] = __fadd_rn(out[a], t);
}

__device__ __forceinline__ bool same_point(const float a[3], const float b[3]) {
  return __float_as_uint(a[0]) == __float_as_uint(b[0]) && __float_as_uint(a[1]) == __float_as_uint(b[1]) &&
         __float_as_uint(a[2]) == __float_as_uint(b[2]);
}

// bit k: triangle k of the cube's case is kept (not degenerate); 0 if the cube is not processed
template <class P>
__device__ __forceinline__ unsigned kept_tris(const P& p, int x, int y, int z, float v[8], unsigned& cs) {
  if (!cube_exists(p, x, y, z)) return 0u;
  cs = cube_case(p, x, y, z, v);
  if (cs == 0u || cs == 255u || !cube_ok(p, x, y, z)) return 0u;
  unsigned keep = 0;
  const int nt = mc::kTriCount[cs];
  for (int k = 0; k < nt; ++k) {
    float P0[3], P1[3], P2[3];
    edge_pos(x, y, z, mc::kTris[cs][3 * k + 0], v, P0);
    edge_pos(x, y, z, mc::kTris[cs][3 * k + 1], v, P1);
    edge_pos(x, y, z, mc::kTris[cs][3 * k + 2], v, P2);
    if (!(same_point(P0, P1) || same_point(P1, P2) || same_point(P0, P2))) keep |= 1u << k;
  }
  return keep;
}

__device__ __forceinline__ int popc_tris(unsigned m) {
  int n = 0;
#pragma unroll
  for (int k = 0; k < mc::kMaxTris; ++k) n += (int)((m >> k) & 1u);
  return n;
}

// eight halves as one 16-byte vector
union Pack8h {
  uint4 u;
  __half h[8];
  __device__ Pack8h() {}
};

__device__ __forceinline__ bool inside_h(__half h) { return clamp1(__half2float(h)) < 0.0f; }

// the chunk's 4 rows (x|x+1, y|y+1) over z0 .. z0+VEC, clamped at the volume border, share one sign
template <int VEC>
__device__ bool chunk_uniform(const MeshParams& p, int x, int y, int z0) {
  const int x1 = x + 1 < p.X ? x + 1 : x, y1 = y + 1 < p.Y ? y + 1 : y;
  const int zh = z0 + VEC < p.Z ? z0 + VEC : p.Z - 1;
  int n_in = 0;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const size_t row = vidx(p, (r & 1) ? x1 : x, (r & 2) ? y1 : y, 0);
    if (VEC == kMeshVec) {
      Pack8h pk;
      pk.u = *reinterpret_cast<const uint4*>(p.val + row + z0);
#pragma unroll
      for (int i = 0; i < 8; ++i) n_in += inside_h(pk.h[i]);
    } else {
#pragma unroll
      for (int i = 0; i < VEC; ++i) n_in += inside_h(p.val[row + z0 + i]);
    }
    n_in += inside_h(p.val[row + zh]);
  }
  return n_in == 0 || n_in == 4 * (VEC + 1);
}

// ---- block scans: shared memory plus __shfl_sync (no CUB, no ballot) ---------------------------

__device__ __forceinline__ int warp_incl_scan(int v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_sync(0xffffffffu, v, lane >= o ? lane - o : lane);
    if (lane >= o) v += u;
  }
  return v;
}

// exclusive block scan of (a, b) over kMeshThreads threads; tot_* = block totals
__device__ void block_scan2(int& a, int& b, int& tot_a, int& tot_b) {
  __shared__ int sa[kMeshThreads / 32], sb[kMeshThreads / 32];
  const int tid = (int)threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ia = warp_incl_scan(a, lane), ib = warp_incl_scan(b, lane);
  if (lane == 31) { sa[warp] = ia; sb[warp] = ib; }
  __syncthreads();
  int pa = 0, pb = 0;
  tot_a = 0; tot_b = 0;
#pragma unroll
  for (int w = 0; w < kMeshThreads / 32; ++w) {
    if (w < warp) { pa += sa[w]; pb += sb[w]; }
    tot_a += sa[w]; tot_b += sb[w];
  }
  a = pa + ia - a;
  b = pb + ib - b;
  __syncthreads();   // sa / sb are reused by the next call
}

struct Chunk {
  int x, y, z0;
  bool live;     // inside the volume and not sign-uniform
};

template <int VEC>
__device__ Chunk chunk_of(const MeshParams& p) {
  const unsigned t = blockIdx.x * kMeshThreads + threadIdx.x;
  const unsigned plane = (unsigned)p.Y * (unsigned)p.zchunks;
  Chunk c{(int)blockIdx.y, 0, 0, false};
  if (t < plane) {
    c.y = (int)(t / (unsigned)p.zchunks);
    c.z0 = (int)(t % (unsigned)p.zchunks) * VEC;
    c.live = !chunk_uniform<VEC>(p, c.x, c.y, c.z0);
  }
  return c;
}

// the dense volume is its own view; a voxel's slot in the per-voxel arrays is its linear index
__device__ __forceinline__ const MeshParams& view_of(const MeshParams& p, const Chunk&) { return p; }
__device__ __forceinline__ size_t vslot(const MeshParams& p, int x, int y, int z) { return vidx(p, x, y, z); }

template <int VEC, class P, class C>
__device__ void chunk_counts(const P& p, const C& c, int& nv, int& nf) {
  nv = 0;
  nf = 0;
  if (!c.live) return;
  for (int i = 0; i < VEC; ++i) {
    float v[8];
    unsigned cs = 0;
    nv += popc3(owned_edges(p, c.x, c.y, c.z0 + i));
    nf += popc_tris(kept_tris(p, c.x, c.y, c.z0 + i, v, cs));
  }
}

__device__ __forceinline__ unsigned block_linear() { return blockIdx.y * gridDim.x + blockIdx.x; }

template <int VEC, class P = MeshParams>
__global__ void __launch_bounds__(kMeshThreads) mesh_count_kernel(P p, int* __restrict__ block_counts) {
  const auto c = chunk_of<VEC>(p);
  int nv, nf, ta, tb;
  chunk_counts<VEC>(view_of(p, c), c, nv, nf);
  block_scan2(nv, nf, ta, tb);
  if (threadIdx.x == 0) {
    block_counts[2 * block_linear() + 0] = ta;
    block_counts[2 * block_linear() + 1] = tb;
  }
}

// one CTA: exclusive offsets of the block totals, in block order; grand totals to totals[] and counts[]
__global__ void __launch_bounds__(kMeshScanThreads)
mesh_scan_kernel(const int* __restrict__ block_counts, long long nblocks, long long* __restrict__ block_off,
                 long long* __restrict__ totals, long long* __restrict__ counts) {
  __shared__ long long s[2][kMeshScanThreads];
  const int tid = (int)threadIdx.x;
  const long long per = (nblocks + kMeshScanThreads - 1) / kMeshScanThreads;
  const long long b0 = tid * per, b1 = (b0 + per < nblocks) ? b0 + per : nblocks;
  long long sv = 0, sf = 0;
  for (long long b = b0; b < b1; ++b) { sv += block_counts[2 * b]; sf += block_counts[2 * b + 1]; }
  s[0][tid] = sv;
  s[1][tid] = sf;
  __syncthreads();
  // Hillis-Steele inclusive scan of the per-thread segment sums
  for (int o = 1; o < kMeshScanThreads; o <<= 1) {
    const long long av = tid >= o ? s[0][tid - o] : 0, af = tid >= o ? s[1][tid - o] : 0;
    __syncthreads();
    s[0][tid] += av;
    s[1][tid] += af;
    __syncthreads();
  }
  long long ov = s[0][tid] - sv, of = s[1][tid] - sf;
  for (long long b = b0; b < b1; ++b) {
    block_off[2 * b] = ov;
    block_off[2 * b + 1] = of;
    ov += block_counts[2 * b];
    of += block_counts[2 * b + 1];
  }
  if (tid == kMeshScanThreads - 1) {
    totals[0] = s[0][tid];
    totals[1] = s[1][tid];
    counts[0] = s[0][tid];
    counts[1] = s[1][tid];
  }
}

template <class P>
__device__ __forceinline__ float grad1(const P& p, int x, int y, int z, int a) {
  const int c = a == 0 ? x : (a == 1 ? y : z);
  const int dx = a == 0, dy = a == 1, dz = a == 2;
  if (at_low(p, a, c)) return __fadd_rn(ld(p, x + dx, y + dy, z + dz), -ld(p, x, y, z));
  if (at_high(p, a, c)) return __fadd_rn(ld(p, x, y, z), -ld(p, x - dx, y - dy, z - dz));
  return __fmul_rn(__fadd_rn(ld(p, x + dx, y + dy, z + dz), -ld(p, x - dx, y - dy, z - dz)), 0.5f);
}

template <int VEC, class P = MeshParams>
__global__ void __launch_bounds__(kMeshThreads)
mesh_vertex_kernel(P pp, const int* __restrict__ block_counts, const long long* __restrict__ block_off,
                   int* __restrict__ vbase, float* __restrict__ verts, float* __restrict__ normals) {
  if (block_counts[2 * block_linear()] == 0) return;    // the whole block owns no vertex (block-uniform)
  const auto c = chunk_of<VEC>(pp);
  decltype(auto) p = view_of(pp, c);      // the dense volume by reference, a block view by value
  int nv, nf, ta, tb;
  chunk_counts<VEC>(p, c, nv, nf);
  nf = 0;
  block_scan2(nv, nf, ta, tb);
  if (!c.live) return;
  long long off = block_off[2 * block_linear()] + nv;
  for (int i = 0; i < VEC; ++i) {
    const int x = c.x, y = c.y, z = c.z0 + i;
    const unsigned m = owned_edges(p, x, y, z);
    if (m == 0u) continue;
    vbase[vslot(p, x, y, z)] = (int)off;
    const float v0 = ld(p, x, y, z);
    float g0[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) g0[k] = grad1(p, x, y, z, k);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (!((m >> a) & 1u)) continue;
      const int qx = x + (a == 0), qy = y + (a == 1), qz = z + (a == 2);
      const float t = edge_t(v0, ld(p, qx, qy, qz));
      float pos[3] = {(float)x, (float)y, (float)z};
      pos[a] = __fadd_rn(pos[a], t);
      if (p.world) {
        pos[0] = __fadd_rn(p.ox, __fmul_rn(pos[0], p.vs));
        pos[1] = __fadd_rn(p.oy, __fmul_rn(pos[1], p.vs));
        pos[2] = __fadd_rn(p.oz, __fmul_rn(pos[2], p.vs));
      }
      verts[3 * off + 0] = pos[0];
      verts[3 * off + 1] = pos[1];
      verts[3 * off + 2] = pos[2];
      if (normals != nullptr) {
        float n[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) n[k] = __fadd_rn(g0[k], __fmul_rn(t, __fadd_rn(grad1(p, qx, qy, qz, k), -g0[k])));
        const float l2 = __fadd_rn(__fadd_rn(__fmul_rn(n[0], n[0]), __fmul_rn(n[1], n[1])), __fmul_rn(n[2], n[2]));
        const float inv = l2 > 0.0f ? __fdiv_rn(1.0f, sqrtf(l2)) : 0.0f;
        normals[3 * off + 0] = __fmul_rn(n[0], inv);
        normals[3 * off + 1] = __fmul_rn(n[1], inv);
        normals[3 * off + 2] = __fmul_rn(n[2], inv);
      }
      ++off;
    }
  }
}

// Vertex colours (DESIGN §4.11), a pass of its own after the vertex pass (same chunks, same vertex order):
// each vertex takes the colour of its edge (a, b) from the (3,X,Y,Z) planes with the position's t.  Both
// endpoints observed (weight > 0): ca + t (cb - ca); one: its colour; none: grey 0.7.  Separately rounded
// fp32 ops.  (Folded into the vertex pass, the colour state lives across the normals' IEEE-division
// slow-path calls and ptxas spills it.)
template <int VEC, class P = MeshParams>
__global__ void __launch_bounds__(kMeshThreads)
mesh_vertex_color_kernel(P pp, const int* __restrict__ block_counts, const long long* __restrict__ block_off,
                         const float* __restrict__ colors, size_t cplane, float* __restrict__ vert_colors) {
  if (block_counts[2 * block_linear()] == 0) return;    // the whole block owns no vertex (block-uniform)
  const auto c = chunk_of<VEC>(pp);
  decltype(auto) p = view_of(pp, c);      // the dense volume by reference, a block view by value
  int nv, nf, ta, tb;
  chunk_counts<VEC>(p, c, nv, nf);
  nf = 0;
  block_scan2(nv, nf, ta, tb);
  if (!c.live) return;
  long long off = block_off[2 * block_linear()] + nv;
  for (int i = 0; i < VEC; ++i) {
    const int x = c.x, y = c.y, z = c.z0 + i;
    const unsigned m = owned_edges(p, x, y, z);
    if (m == 0u) continue;
    const float v0 = ld(p, x, y, z);
    const bool oa = wt(p, x, y, z) > 0.0f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (!((m >> a) & 1u)) continue;
      const int qx = x + (a == 0), qy = y + (a == 1), qz = z + (a == 2);
      const float t = edge_t(v0, ld(p, qx, qy, qz));           // the position's t (mesh_vertex_kernel)
      const bool ob = wt(p, qx, qy, qz) > 0.0f;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float* cc = colors + ch * cplane;
        float r = 0.7f;
        // (a weighted voxel always has a slot: vslot is only asked for those)
        if (oa && ob) {
          const float ca = cc[vslot(p, x, y, z)];
          r = __fadd_rn(ca, __fmul_rn(t, __fadd_rn(cc[vslot(p, qx, qy, qz)], -ca)));
        } else if (oa) {
          r = cc[vslot(p, x, y, z)];
        } else if (ob) {
          r = cc[vslot(p, qx, qy, qz)];
        }
        vert_colors[3 * off + ch] = r;
      }
      ++off;
    }
  }
}

template <int VEC, class P = MeshParams>
__global__ void __launch_bounds__(kMeshThreads)
mesh_face_kernel(P pp, const int* __restrict__ block_counts, const long long* __restrict__ block_off,
                 const int* __restrict__ vbase, int* __restrict__ faces) {
  if (block_counts[2 * block_linear() + 1] == 0) return;   // the whole block anchors no face (block-uniform)
  const auto c = chunk_of<VEC>(pp);
  decltype(auto) p = view_of(pp, c);      // the dense volume by reference, a block view by value
  int nv, nf, ta, tb;
  chunk_counts<VEC>(p, c, nv, nf);
  nv = 0;
  block_scan2(nv, nf, ta, tb);
  if (!c.live) return;
  long long off = block_off[2 * block_linear() + 1] + nf;
  for (int i = 0; i < VEC; ++i) {
    const int x = c.x, y = c.y, z = c.z0 + i;
    float v[8];
    unsigned cs = 0;
    const unsigned keep = kept_tris(p, x, y, z, v, cs);
    if (keep == 0u) continue;
    const int nt = mc::kTriCount[cs];
    for (int k = 0; k < nt; ++k) {
      if (!((keep >> k) & 1u)) continue;
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        int o[3], a;
        edge_geom(mc::kTris[cs][3 * k + j], o, a);
        const int ox = x + o[0], oy = y + o[1], oz = z + o[2];
        const unsigned m = owned_edges(p, ox, oy, oz);
        faces[3 * off + j] = vbase[vslot(p, ox, oy, oz)] + popc3(m & ((1u << a) - 1u));
      }
      ++off;
    }
  }
}

struct MeshWs {
  long long* totals;     // [2]: V, F of the last count
  int* block_counts;     // [nblocks][2]
  long long* block_off;  // [nblocks][2]
  int* vbase;            // [X*Y*Z] first vertex index of each owner (touched for active voxels only)
  size_t bytes;
};

// blocks of the voxel passes; the workspace is sized for the scalar path (the most blocks)
long long mesh_blocks(const srcv_mesh_args& a, int vec) {
  const long long plane = (long long)a.Y * (a.Z / vec);
  return (long long)a.X * ((plane + kMeshThreads - 1) / kMeshThreads);
}

MeshWs carve(const srcv_mesh_args& a, void* base) {
  MeshWs w{};
  char* p = static_cast<char*>(base);
  const long long nb = mesh_blocks(a, 1);
  size_t off = 0;
  w.totals = reinterpret_cast<long long*>(p + off);
  off += 256;
  w.block_counts = reinterpret_cast<int*>(p + off);
  off += align256(sizeof(int) * 2 * (size_t)nb);
  w.block_off = reinterpret_cast<long long*>(p + off);
  off += align256(sizeof(long long) * 2 * (size_t)nb);
  w.vbase = reinterpret_cast<int*>(p + off);
  off += align256(sizeof(int) * (size_t)a.X * a.Y * a.Z);
  w.bytes = off;
  return w;
}

MeshParams params(const srcv_mesh_args& a, int vec) {
  MeshParams p;
  p.val = reinterpret_cast<const __half*>(a.tsdf_values);
  p.w = reinterpret_cast<const __half*>(a.tsdf_weights);
  p.X = a.X; p.Y = a.Y; p.Z = a.Z; p.zchunks = a.Z / vec;
  p.ox = a.origin[0]; p.oy = a.origin[1]; p.oz = a.origin[2]; p.vs = a.voxel_size;
  p.world = a.scale_to_world != 0;
  p.single = a.single_mesh != 0;
  return p;
}

int vec_of(const srcv_mesh_args& a) {
  return ((a.Z % kMeshVec) == 0 && (reinterpret_cast<uintptr_t>(a.tsdf_values) & 15u) == 0) ? kMeshVec : 1;
}

dim3 grid_of(const srcv_mesh_args& a, int vec) {
  const long long plane = (long long)a.Y * (a.Z / vec);
  return dim3((unsigned)((plane + kMeshThreads - 1) / kMeshThreads), (unsigned)a.X);
}

}  // namespace

size_t mesh_workspace_bytes(const srcv_mesh_args& a) { return carve(a, nullptr).bytes; }

bool mesh_shape_supported(const srcv_mesh_args& a) {
  return a.X <= 65535 && (long long)a.Y * a.Z <= 2147483647ll && (long long)a.X * a.Y * a.Z <= (1ll << 40);
}

cudaError_t launch_mesh_count(const srcv_mesh_args& a, long long* counts, void* workspace, cudaStream_t stream) {
  const MeshWs w = carve(a, workspace);
  const int vec = vec_of(a);
  const MeshParams p = params(a, vec);
  if (vec == kMeshVec) SRCV_LAUNCH(mesh_count_kernel<kMeshVec>, grid_of(a, vec), kMeshThreads, 0, stream, p, w.block_counts);
  else SRCV_LAUNCH(mesh_count_kernel<1>, grid_of(a, vec), kMeshThreads, 0, stream, p, w.block_counts);
  note_launch();
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return err;
  SRCV_LAUNCH(mesh_scan_kernel, 1, kMeshScanThreads, 0, stream, w.block_counts, mesh_blocks(a, vec), w.block_off,
              w.totals, counts);
  note_launch();
  return cudaGetLastError();
}

cudaError_t mesh_read_totals(const srcv_mesh_args& a, void* workspace, long long totals[2], cudaStream_t stream) {
  const MeshWs w = carve(a, workspace);
#ifdef SRCV_HOST_EMU
  (void)stream;
  std::memcpy(totals, w.totals, 2 * sizeof(long long));   // emulated device memory is host memory
  return cudaSuccess;
#else
  cudaError_t err = cudaMemcpyAsync(totals, w.totals, 2 * sizeof(long long), cudaMemcpyDeviceToHost, stream);
  if (err != cudaSuccess) return err;
  return cudaStreamSynchronize(stream);
#endif
}

cudaError_t launch_mesh_extract(const srcv_mesh_args& a, float* verts, float* normals, int32_t* faces,
                                void* workspace, cudaStream_t stream, const float* colors, float* vert_colors) {
  const MeshWs w = carve(a, workspace);
  const int vec = vec_of(a);
  const MeshParams p = params(a, vec);
  if (vec == kMeshVec) SRCV_LAUNCH(mesh_vertex_kernel<kMeshVec>, grid_of(a, vec), kMeshThreads, 0, stream, p, w.block_counts, w.block_off, w.vbase, verts, normals);
  else SRCV_LAUNCH(mesh_vertex_kernel<1>, grid_of(a, vec), kMeshThreads, 0, stream, p, w.block_counts, w.block_off, w.vbase, verts, normals);
  note_launch();
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return err;
  if (colors != nullptr) {
    const size_t cplane = (size_t)a.X * a.Y * a.Z;
    if (vec == kMeshVec) SRCV_LAUNCH(mesh_vertex_color_kernel<kMeshVec>, grid_of(a, vec), kMeshThreads, 0, stream, p, w.block_counts, w.block_off, colors, cplane, vert_colors);
    else SRCV_LAUNCH(mesh_vertex_color_kernel<1>, grid_of(a, vec), kMeshThreads, 0, stream, p, w.block_counts, w.block_off, colors, cplane, vert_colors);
    note_launch();
    err = cudaGetLastError();
    if (err != cudaSuccess) return err;
  }
  if (vec == kMeshVec) SRCV_LAUNCH(mesh_face_kernel<kMeshVec>, grid_of(a, vec), kMeshThreads, 0, stream, p, w.block_counts, w.block_off, w.vbase, faces);
  else SRCV_LAUNCH(mesh_face_kernel<1>, grid_of(a, vec), kMeshThreads, 0, stream, p, w.block_counts, w.block_off, w.vbase, faces);
  note_launch();
  return cudaGetLastError();
}

}  // namespace srcv
