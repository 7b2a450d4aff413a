/*
 * srcv_b200 — C ABI of the H100-native plane-sweep cost-volume library.
 *
 * This is the drop-in boundary for SimpleRecon's cost-volume hot path.  The
 * reference has no native layer (it is pure PyTorch), so each entry point below
 * names the reference *Python* interface it replaces; the Python classes in
 * simplerecon_b200/cost_volume.py bind these symbols through ctypes and keep the
 * reference's class / method signatures (see INTEGRATION.md for the binding a
 * maintainer of the reference would add).
 *
 * Conventions
 *   - plain C types only: device pointers, sizes, an opaque stream handle
 *     (a cudaStream_t passed as void*; NULL = legacy default stream);
 *   - all tensors are fp32, contiguous, row-major in the reference's layouts;
 *   - outputs and the workspace are caller-allocated (the Python side hands
 *     PyTorch caching-allocator memory); nothing is allocated, freed or retained
 *     by the library, and no call synchronises the device: work is enqueued on
 *     `stream` and the call returns;
 *   - every function returns an srcv_status (0 = ok).  Argument errors are
 *     detected on the host before anything is launched; CUDA launch errors are
 *     returned as SRCV_ERR_CUDA with the text available from srcv_last_error().
 */
#ifndef SRCV_B200_H_
#define SRCV_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SRCV_ABI_VERSION 2

typedef enum srcv_status {
  SRCV_OK = 0,
  SRCV_ERR_NULL = 1,        /* a required pointer is NULL                      */
  SRCV_ERR_SHAPE = 2,       /* a dimension is <= 0 or out of the supported set */
  SRCV_ERR_WORKSPACE = 3,   /* workspace too small or misaligned               */
  SRCV_ERR_UNSUPPORTED = 4, /* valid request this build cannot serve           */
  SRCV_ERR_CUDA = 5,        /* CUDA runtime error (see srcv_last_error)        */
  SRCV_ERR_DEVICE = 6       /* current device is not an sm_90 part             */
} srcv_status;

/* Problem shape.  Mirrors the tensor contract of
 * CostVolumeManager.forward (reference modules/cost_volume.py:345-380):
 *   cur_feats (B,C,H,W)  src_feats (B,K,C,H,W)  cost (B,D,H,W).          */
typedef struct srcv_shape {
  int32_t B; /* reference frames in this call (batch)                        */
  int32_t K; /* source views per frame                                       */
  int32_t C; /* matching-feature channels                                    */
  int32_t H; /* matching feature-map height                                  */
  int32_t W; /* matching feature-map width                                   */
  int32_t D; /* depth planes                                                 */
  int32_t layout; /* srcv_feature_layout of cur_feats / src_feats (0 = the reference's NCHW)  */
} srcv_shape;

/* Memory layout of the two feature inputs.  CHUNK_PLANAR is what the gather kernels read
 * internally — cur_feats (B,C/4,H,W,4), src_feats (B,K,C/4,H,W,4): a texel's 4-channel chunk is
 * one 16-byte vector — and what srcv_instnorm_to_chunk_planar_f32 produces: a caller that
 * hands it over skips the re-layout copy of the prep pass (SURVEY.md §8f-2).  Served by the
 * chunk-planar dot sweep (C == 16) and the tensor-core MLP sweep (K == 7, C == 16, 128/128);
 * other shapes return SRCV_ERR_UNSUPPORTED.                                               */
typedef enum srcv_feature_layout {
  SRCV_LAYOUT_NCHW = 0,
  SRCV_LAYOUT_CHUNK_PLANAR = 1
} srcv_feature_layout;

/* How the depth hypotheses are given. */
typedef enum srcv_planes_mode {
  /* planes == NULL on input: the library evaluates
   *   d_i = exp(log(min) + log(max/min) * ramp_i)
   * (reference modules/cost_volume.py:100-136) from the DEVICE scalars
   * min_depth / max_depth and the DEVICE ramp (D floats, the module buffer
   * `linear_ramp_1d11`) and writes the (B,D) result to planes_out.          */
  SRCV_PLANES_FROM_RANGE = 0,
  /* planes is a DEVICE (B,D) array: one depth per plane and frame.         */
  SRCV_PLANES_PER_PLANE = 1,
  /* planes is a DEVICE (B,D,H,W) array: caller-supplied per-pixel
   * hypotheses (the `depth_planes_bdhw` argument, modules/cost_volume.py:247) */
  SRCV_PLANES_PER_PIXEL = 2
} srcv_planes_mode;

typedef struct srcv_planes {
  int32_t mode;            /* srcv_planes_mode                               */
  const float* planes;     /* (B,D) or (B,D,H,W); NULL for FROM_RANGE        */
  const float* min_depth;  /* device scalar, FROM_RANGE only                 */
  const float* max_depth;  /* device scalar, FROM_RANGE only                 */
  const float* ramp;       /* device (D), FROM_RANGE only                    */
  float* planes_out;       /* device (B,D), FROM_RANGE only (may be NULL)    */
  int32_t range_per_frame; /* FROM_RANGE: 0 = min/max_depth are single scalars (the
                            * (1,1,1,1) tensors of depth_model.py:358-359); 1 = B values each,
                            * one range per frame (generate_depth_planes broadcasts a
                            * (B,1,1,1) range, modules/cost_volume.py:124-127)  */
} srcv_planes;

/* Camera block shared by both volumes (all DEVICE pointers). */
typedef struct srcv_cameras {
  const float* src_extrinsics; /* (B,K,4,4) src_cam_T_cur_cam               */
  const float* src_poses;      /* (B,K,4,4) cur_cam_T_src_cam (MLP volume only; may be NULL for dot) */
  const float* src_Ks;         /* (B,K,4,4) source intrinsics at matching scale */
  const float* cur_invK;       /* (B,4,4) inverse intrinsics of the reference frame */
  /* Optional raw poses (SURVEY.md §8f-2).  When src_extrinsics is NULL the prep kernel forms
   *   src_cam_T_cur_cam = src_cam_T_world @ cur_world_T_cam          (-> src_extrinsics)
   *   cur_cam_T_src_cam = cur_cam_T_world @ src_world_T_cam          (-> src_poses)
   * itself — the two batched 4x4 products experiment_modules/depth_model.py:324-332 runs in
   * PyTorch before the call — evaluated in fp64 and rounded to fp32.  All four DEVICE pointers
   * are then required ((B,K,4,4), (B,4,4), (B,4,4), (B,K,4,4)); ignored otherwise.        */
  const float* src_cam_T_world;
  const float* cur_world_T_cam;
  const float* cur_cam_T_world;
  const float* src_world_T_cam;
} srcv_cameras;

/* Weights of the matching MLP — the parameters of the reference's
 * `MLP([F,H1,H2,1], disable_final_activation=True)` (modules/networks.py:129-147),
 * in nn.Linear layout (out_features, in_features), LeakyReLU slope 0.01.    */
typedef struct srcv_mlp_weights {
  const float* w1; const float* b1; /* (H1,F), (H1)  F = C*(K+1)+10*K+4       */
  const float* w2; const float* b2; /* (H2,H1), (H2)                          */
  const float* w3; const float* b3; /* (1,H2), (1)                            */
  int32_t hidden1;                  /* H1                                     */
  int32_t hidden2;                  /* H2                                     */
  /* Optional: DEVICE image written by srcv_mlp_pack_weights for exactly these weights
   * (srcv_mlp_packed_bytes bytes, 256-byte aligned).  NULL = the forward call packs the
   * weights itself, into its workspace, on every call.  A caller whose parameters change
   * rarely (inference; one optimiser step per forward in training) packs once per change.  */
  const void* packed_image;
} srcv_mlp_weights;

/* ---- library / device ------------------------------------------------- */
int32_t srcv_abi_version(void);
/* 0 if the CURRENT CUDA device can run this library (compute capability 10.x),
 * else SRCV_ERR_DEVICE / SRCV_ERR_CUDA.                                      */
int32_t srcv_check_device(void);
const char* srcv_status_string(int32_t status);
/* Thread-local text of the last SRCV_ERR_* raised on this thread.           */
const char* srcv_last_error(void);

/* ---- dot-product volume ----------------------------------------------- *
 * Replaces CostVolumeManager.build_cost_volume + the argmax in
 * CostVolumeManager.forward (reference modules/cost_volume.py:237-335,
 * :345-380): per plane, homography-warp every source feature map into the
 * reference frustum (bilinear, zeros padding, align_corners=False), dot it with
 * the reference features, mask by depth validity, sum over views.
 *   cost   (B,D,H,W) out
 *   lowest (B,H,W)   out, plane depth at argmax_d cost (first index on ties);
 *                    NULL to skip.                                           */
size_t srcv_dot_workspace_bytes(const srcv_shape* shape);
int32_t srcv_dot_forward_f32(const srcv_shape* shape,
                             const float* cur_feats, const float* src_feats,
                             const srcv_cameras* cams, const srcv_planes* planes,
                             float* cost, float* lowest,
                             void* workspace, size_t workspace_bytes,
                             void* stream);

/* ---- backward of the dot-product volume (training) ----------------------- *
 * Gradients of a scalar loss w.r.t. the FEATURE inputs of srcv_dot_forward_f32, given
 * grad_cost = dL/dcost (B,D,H,W) — what autograd of the reference's composite
 * (modules/cost_volume.py:305-333: grid_sample, mul, sum) yields for cur_feats and
 * src_feats.  Cameras and plane depths get no gradient.  C must be 8, 16 or 32.
 *   grad_cur (B,C,H,W) out      grad_src (B,K,C,H,W) out (zeroed here, then accumulated
 *   with float atomics: reproducible to fp32 rounding, not bit-for-bit)           */
size_t srcv_dot_backward_workspace_bytes(const srcv_shape* shape);
/* 1 if srcv_dot_backward_f32 serves this shape (C in {8,16,32}), else 0 — lets the caller
 * refuse an unsupported training shape in forward() instead of at backward() time.          */
int32_t srcv_dot_backward_supported(const srcv_shape* shape);
int32_t srcv_dot_backward_f32(const srcv_shape* shape, const float* cur_feats, const float* src_feats,
                              const srcv_cameras* cams, const srcv_planes* planes,
                              const float* grad_cost, float* grad_cur, float* grad_src,
                              void* workspace, size_t workspace_bytes, void* stream);

/* ---- single-plane warp -------------------------------------------------- *
 * Replaces CostVolumeManager.warp_features (reference modules/cost_volume.py:139-234),
 * the helper that MATERIALISES the warped source features of one depth plane; the
 * sweeps above never call it (they keep the warped values in registers / shared memory), it is
 * exported because the reference exposes it as a method.  shape->D is ignored.
 *   depth_plane  DEVICE (B) one depth per frame, or (B,H,W) when per_pixel != 0
 *   warped (B,K,C,H,W)  depths (B,K,H,W) = z' of the plane point in each source camera
 *   mask   (B,K,H,W)    1.0 where z' > 0                                         */
size_t srcv_warp_workspace_bytes(const srcv_shape* shape);
int32_t srcv_warp_features_f32(const srcv_shape* shape, const float* src_feats,
                               const srcv_cameras* cams, const float* depth_plane,
                               int32_t per_pixel, float* warped, float* depths, float* mask,
                               void* workspace, size_t workspace_bytes, void* stream);

/* All planes at once: replaces FastFeatureVolumeManager.warp_features (reference
 * modules/cost_volume.py:812-964), which materialises the warped features of EVERY plane
 * (550 MB per frame at the hero shape) — exported for callers of that method; the sweeps
 * never call it.  shape->D = number of planes.
 *   depth_planes DEVICE (B,D), or (B,D,H,W) when per_pixel != 0
 *   warped (B,K,D,C,H,W)   depths, mask (B,K,D,H,W)
 *   pix_coords (B,K,D,2,H,W): the projected pixel coordinates (x, y); NULL to skip        */
int32_t srcv_warp_features_planes_f32(const srcv_shape* shape, const float* src_feats,
                                      const srcv_cameras* cams, const float* depth_planes,
                                      int32_t per_pixel, float* warped, float* depths, float* mask,
                                      float* pix_coords, void* workspace, size_t workspace_bytes,
                                      void* stream);

/* ---- metadata-MLP volume ---------------------------------------------- *
 * Replaces FeatureVolumeManager.build_cost_volume /
 * FastFeatureVolumeManager.build_cost_volume + the argmax in forward
 * (reference modules/cost_volume.py:451-736, :967-1164): builds the per
 * (plane,pixel) metadata vector (warped features, reference features, validity,
 * source depths, plane depth, per-view dot, ray angle, rays, pose measures —
 * order of :698-723) and runs the matching MLP on it, without materialising it.
 *   overall_mask (B,H,W) uint8 out (1 = some source view sees the pixel at the
 *   LAST plane, :625-637); NULL when return_mask is False.                   */
size_t srcv_mlp_workspace_bytes(const srcv_shape* shape, const srcv_mlp_weights* w);
/* Size of the packed weight image of the tensor-core variant for this shape / these widths
 * (0 when that variant does not serve them and there is nothing to pack), and the packing
 * itself: `image` DEVICE, 256-byte aligned, srcv_mlp_packed_bytes bytes.                   */
size_t srcv_mlp_packed_bytes(const srcv_shape* shape, const srcv_mlp_weights* w);
int32_t srcv_mlp_pack_weights(const srcv_shape* shape, const srcv_mlp_weights* w, void* image,
                              void* stream);
int32_t srcv_mlp_forward_f32(const srcv_shape* shape,
                             const float* cur_feats, const float* src_feats,
                             const srcv_cameras* cams, const srcv_planes* planes,
                             const srcv_mlp_weights* weights,
                             float* cost, float* lowest, uint8_t* overall_mask,
                             void* workspace, size_t workspace_bytes,
                             void* stream);

/* ---- metadata-MLP volume, backward ------------------------------------ *
 * What autograd of the reference composite (modules/cost_volume.py:451-736 with the
 * MLP of modules/networks.py:129-147; used for training by
 * experiment_modules/depth_model.py:362-372 under train.py) yields for the two feature
 * inputs and the six MLP parameters, given dL/dcost.  Nothing of the forward is saved:
 * the kernel recomputes the metadata tile and the activations per 64-row tile.  Every
 * output is OVERWRITTEN (zeroed, then accumulated with fp32 atomics — the summation
 * order, hence the last bits, may differ between calls).  Cameras and plane depths get
 * no gradient.  Supported: C (K+1) + 10 K + 4 <= 208 features, hidden widths <= 128.
 *   grad_cost (B,D,H,W)   grad_cur (B,C,H,W)   grad_src (B,K,C,H,W)
 *   grads     DEVICE pointers shaped like the parameters in srcv_mlp_weights        */
typedef struct srcv_mlp_grads {
  float* w1; float* b1;
  float* w2; float* b2;
  float* w3; float* b3;
} srcv_mlp_grads;
size_t srcv_mlp_backward_workspace_bytes(const srcv_shape* shape, const srcv_mlp_weights* w);
/* 1 if srcv_mlp_backward_f32 serves this shape and these hidden widths, else 0.             */
int32_t srcv_mlp_backward_supported(const srcv_shape* shape, int32_t hidden1, int32_t hidden2);
int32_t srcv_mlp_backward_f32(const srcv_shape* shape,
                              const float* cur_feats, const float* src_feats,
                              const srcv_cameras* cams, const srcv_planes* planes,
                              const srcv_mlp_weights* weights, const float* grad_cost,
                              float* grad_cur, float* grad_src, const srcv_mlp_grads* grads,
                              void* workspace, size_t workspace_bytes, void* stream);

/* ---- producer-side fusion: encoder tail -> chunk-planar features -------------------- *
 * Replaces the last op of the reference's matching encoder, nn.InstanceNorm2d(C) without
 * affine (modules/networks.py:201; biased variance), AND the re-layout pass of the sweeps:
 *   x        DEVICE (B, V, C, H, W) fp32 — the conv output for the stacked (reference frame,
 *            K = V-1 source views) images, as depth_model.py:220-243 produces it
 *   cur_c4   DEVICE (B, C/4, H, W, 4)        normalised features of view 0
 *   src_c4   DEVICE (B, V-1, C/4, H, W, 4)   normalised features of views 1..V-1
 * Pass both to the forward calls with shape->layout = SRCV_LAYOUT_CHUNK_PLANAR.  C % 4 == 0. */
int32_t srcv_instnorm_to_chunk_planar_f32(const float* x, int32_t B, int32_t V, int32_t C, int32_t H,
                                          int32_t W, float eps, float* cur_c4, float* src_c4, void* stream);

/* ---- TSDF integration of depth maps (the consumer of the predicted depth) ---- *
 * Replaces TSDFFuser.integrate_depth + project_to_camera (reference tools/tsdf.py:221-320,
 * :204-219) as OurFuser.fuse_frames drives them (tools/fusers_helper.py:64-71): a dense
 * (X,Y,Z) fp16 volume of truncated signed distances and running-average weights, z fastest,
 * updated in place with a batch of depth maps applied IN ORDER.  All tensors are fp16, as in
 * the reference (which `.half()`s depth, intrinsics and extrinsics): the arithmetic is the
 * reference's op for op, every operation rounded to fp16.  One launch per <= 16 frames; a
 * voxel's 4 bytes are read and written at most once per launch.
 *   tsdf_values, tsdf_weights  DEVICE (X,Y,Z) fp16, updated in place (16-byte aligned and
 *                              Z % 8 == 0 take the vector path; anything else a scalar path)
 *   origin                     world position of voxel (0,0,0) (fp32, TSDF.from_bounds :85)
 *   depth        DEVICE (B,H,W) fp16     cam_T_world, K  DEVICE (B,4,4) fp16
 *   depth_mask   DEVICE (B,H,W) uint8 (0 = invalid pixel, :251-253) or NULL
 * Limits (SRCV_ERR_SHAPE): B >= 1, 1 <= H, W <= 2048 (pixel coordinates exact in fp16), max_depth > min_depth.
 * srcv_tsdf_workspace_bytes and srcv_sparse_tsdf_workspace_bytes are 0 for frame sizes outside them.      */
typedef struct srcv_tsdf_volume {
  void* tsdf_values;
  void* tsdf_weights;
  int32_t X, Y, Z;
  float origin[3];
  float voxel_size;
  float truncation_voxels; /* TSDFFuser.truncation_size (3.0), :181 */
  float max_weight;        /* TSDFFuser.maxW (100.0), :182          */
} srcv_tsdf_volume;
typedef struct srcv_tsdf_frames {
  const void* depth;
  const void* cam_T_world;
  const void* K;
  const uint8_t* depth_mask;
  int32_t B, H, W;
  float min_depth; /* TSDFFuser(min_depth=0.5)  */
  float max_depth; /* TSDFFuser(max_depth=5.0)  */
} srcv_tsdf_frames;
size_t srcv_tsdf_workspace_bytes(const srcv_tsdf_frames* frames);
int32_t srcv_tsdf_integrate_f16(const srcv_tsdf_volume* volume, const srcv_tsdf_frames* frames,
                                void* workspace, size_t workspace_bytes, void* stream);

/* ---- colour fusion into the TSDF volume (DESIGN §4.11) --------------------------------- *
 * srcv_tsdf_integrate_color_f16 is srcv_tsdf_integrate_f16 (same volume, frames, workspace; values
 * and weights bit-identical) that also averages each frame's colour into an fp32 colour volume:
 *   colors   DEVICE (3,X,Y,Z) f32 R, G, B planes in [0, 1], z fastest, updated in place (0 = unseen)
 *   images   DEVICE (B,3,Hc,Wc) f32, any Hc, Wc >= 1 (normalised with mean / std per channel)
 * For every (voxel, frame) update of the values: the depth pixel (sx, sy) the update sampled maps to
 * colour pixel (min(floor(sx * (Wc/W)), Wc-1), min(floor(sy * (Hc/H)), Hc-1)) (PyTorch's `nearest`,
 * each scale an fp32 in/out), rgb = clamp((x - mean) / std, 0, 1), and
 * c = (c * tw + rgb * nw) / total with the update's own fp16 old weight tw, nw and total, every op a
 * separately rounded fp32 op.  The vector path also needs `colors` 16-byte aligned.              */
typedef struct srcv_tsdf_color {
  void* colors;
  const void* images;
  int32_t Hc, Wc;
  float mean[3], std[3];
} srcv_tsdf_color;
int32_t srcv_tsdf_integrate_color_f16(const srcv_tsdf_volume* volume, const srcv_tsdf_frames* frames,
                                      const srcv_tsdf_color* color, void* workspace, size_t workspace_bytes,
                                      void* stream);

/* ---- marching-cubes mesh extraction from the TSDF volume ------------------------------ *
 * Replaces TSDF.to_mesh (reference tools/tsdf.py:125-157: host copy of the volume, clamp, and
 * scikit-image's marching_cubes at level 0) on the GPU.  The mesh is defined precisely (DESIGN
 * §4.10) rather than byte-matched to scikit-image:
 *   - values are taken to fp32 and clamped to [-1, 1]; a corner is inside iff its value is < 0;
 *   - one vertex per crossing edge, shared between cubes, ordered by owning voxel (the edge's
 *     lower endpoint) in linear order, then axis x, y, z; index-space position a + t (b - a) with
 *     t = (0 - v_a) / (v_b - v_a) in fp32;
 *   - normals: central-difference gradients (one-sided at the border) interpolated with t and
 *     normalised, pointing toward increasing values (free space); zero gradient -> zero normal;
 *   - faces: cube by cube in linear order, then in the order of the generated table
 *     (simplerecon_b200/csrc/srcv_mc_table.h, scripts/gen_mc_table.py); right-hand normals point
 *     toward increasing values; a triangle with two bitwise-equal fp32 index-space vertex
 *     positions is dropped (allow_degenerate=False); the surface is closed away from the border
 *     and from exact zeros;
 *   - single_mesh (this library's reading of the reference's export_single_mesh): a cube is
 *     processed only if all 8 corners have weight > 0, and a vertex is emitted only if a processed
 *     cube contains its edge;
 *   - scale_to_world: world = origin + v * voxel_size in fp32.  The reference's origin is fp16, so
 *     callers pass origin already rounded to fp16.
 * Two calls with the same args and workspace: srcv_mesh_count writes V and F to the DEVICE int64
 * counts[2] (2 launches) and keeps them in the workspace; after reading them the caller allocates
 * verts (V,3) f32, normals (V,3) f32 (or NULL) and faces (F,3) int32 and calls srcv_mesh_extract
 * (2 launches), which first reads the kept totals back (16 bytes, a stream synchronisation) and
 * refuses V / F that differ from them.  V > 2^31 - 1 is refused (faces are int32).
 * Workspace: 4 bytes per voxel plus 24 bytes per 256 voxels.  X, Y, Z >= 2, X <= 65535,
 * Y * Z < 2^31.  Deterministic: no atomics, fixed-order scans.                              */
typedef struct srcv_mesh_args {
  const void* tsdf_values;   /* DEVICE (X,Y,Z) fp16 */
  const void* tsdf_weights;  /* DEVICE (X,Y,Z) fp16, read only when single_mesh */
  int32_t X, Y, Z;
  float origin[3];           /* already fp16-rounded by the caller */
  float voxel_size;
  int32_t scale_to_world, single_mesh;
} srcv_mesh_args;
size_t srcv_mesh_workspace_bytes(const srcv_mesh_args* args);
int32_t srcv_mesh_count(const srcv_mesh_args* args, int64_t* counts, void* workspace, size_t workspace_bytes,
                        void* stream);
int32_t srcv_mesh_extract(const srcv_mesh_args* args, float* verts, float* normals, int32_t* faces, int64_t V,
                          int64_t F, void* workspace, size_t workspace_bytes, void* stream);
/* srcv_mesh_extract with vertex colours (DESIGN §4.11), after the same srcv_mesh_count and with the
 * same workspace; verts, normals and faces are bitwise srcv_mesh_extract's.  colors is the DEVICE
 * (3,X,Y,Z) f32 colour volume, args->tsdf_weights is required, vert_colors is (V,3) f32: each vertex
 * takes the colour of its crossing edge (a, b) with the position's t — both endpoints weighted:
 * ca + t (cb - ca) in fp32; one: that endpoint's colour; none: grey 0.7.                         */
int32_t srcv_mesh_extract_color(const srcv_mesh_args* args, const void* colors, float* verts, float* normals,
                                float* vert_colors, int32_t* faces, int64_t V, int64_t F, void* workspace,
                                size_t workspace_bytes, void* stream);

/* ---- the voxel-block hashed TSDF volume (SparseTSDF, DESIGN §4.16) -------------------- *
 * The dense volume's lattice (voxel i at origin + i * voxel_size, any integer i) stored as 8^3-voxel
 * blocks, allocated where some frame can change a voxel: values, weights and colours read back bitwise
 * equal to a dense volume on the same lattice fed the same frames, wherever that volume lies.
 *   state        DEVICE, srcv_sparse_tsdf_state_bytes() bytes, 256-byte aligned, owned by the caller:
 *                a header of SRCV_SPARSE_HDR_WORDS uint32 words at offset 0, then the hash table (a
 *                power of two >= 2 max_blocks slots), the pool of max_blocks blocks (fp16 values and
 *                weights, 1 KiB each; 6 KiB of fp32 colour planes more when `color`)
 *   max_blocks   pool capacity in blocks, 1 .. 2^26
 * Header words: BLOCKS = blocks requested so far (it keeps counting past max_blocks, so after an overflow
 * it is the capacity needed), LOST = inserts that found the hash table full, RANGE = non-zero if a frame
 * reached outside voxel indices -2^23 + 8 .. 2^23 - 1 (blocks -2^20 + 1 .. 2^20 - 1, so that meshing can
 * insert the block below each one) or had a singular projection.  The state is valid while
 * BLOCKS <= max_blocks and LOST == RANGE == 0; nothing here synchronises to check it.
 * srcv_sparse_tsdf_reset initialises the state (1 launch).  The integrate calls take the dense calls'
 * frames, workspace sizing rule (srcv_sparse_tsdf_workspace_bytes) and colour descriptor (its `colors`
 * is ignored: the colour planes are in the state): 4 launches per <= 16 frames.
 * Mesh extraction is srcv_mesh_*'s mesh (DESIGN §4.10) on the unbounded lattice, in index space
 * relative to `origin`: srcv_sparse_tsdf_mesh_begin(blocks = BLOCKS) adds the unallocated blocks just
 * below allocated ones (re-read BLOCKS: allocated + boundary, which must fit max_blocks), then
 * srcv_sparse_tsdf_mesh_count / _extract with args->blocks = that count, as srcv_mesh_count / _extract
 * (vert_colors NULL: no colours), then srcv_sparse_tsdf_mesh_end(blocks = the first BLOCKS) restores the
 * table.  srcv_sparse_tsdf_read_box writes the (X,Y,Z) = dims box starting at lattice voxel lo as dense
 * fp16 values / weights (and (3,X,Y,Z) f32 colours, or NULL), -1 / 0 / 0 where nothing is allocated. */
#define SRCV_SPARSE_HDR_BLOCKS 0
#define SRCV_SPARSE_HDR_LOST 1
#define SRCV_SPARSE_HDR_RANGE 2
#define SRCV_SPARSE_HDR_WORDS 4
typedef struct srcv_sparse_tsdf {
  void* state;
  int32_t max_blocks;
  int32_t color;            /* 1: the state holds colour planes */
  float origin[3];
  float voxel_size;
  float truncation_voxels;
  float max_weight;
} srcv_sparse_tsdf;
typedef struct srcv_sparse_mesh_args {
  int32_t blocks;           /* allocated + boundary blocks, read back after srcv_sparse_tsdf_mesh_begin */
  float origin[3];          /* already fp16-rounded, as srcv_mesh_args */
  int32_t scale_to_world, single_mesh;
} srcv_sparse_mesh_args;
size_t srcv_sparse_tsdf_state_bytes(const srcv_sparse_tsdf* volume);
int32_t srcv_sparse_tsdf_reset(const srcv_sparse_tsdf* volume, void* stream);
size_t srcv_sparse_tsdf_workspace_bytes(const srcv_tsdf_frames* frames);
int32_t srcv_sparse_tsdf_integrate_f16(const srcv_sparse_tsdf* volume, const srcv_tsdf_frames* frames,
                                       void* workspace, size_t workspace_bytes, void* stream);
int32_t srcv_sparse_tsdf_integrate_color_f16(const srcv_sparse_tsdf* volume, const srcv_tsdf_frames* frames,
                                             const srcv_tsdf_color* color, void* workspace, size_t workspace_bytes,
                                             void* stream);
int32_t srcv_sparse_tsdf_mesh_begin(const srcv_sparse_tsdf* volume, int32_t blocks, void* stream);
int32_t srcv_sparse_tsdf_mesh_end(const srcv_sparse_tsdf* volume, int32_t blocks, void* stream);
size_t srcv_sparse_tsdf_mesh_workspace_bytes(const srcv_sparse_mesh_args* args);
int32_t srcv_sparse_tsdf_mesh_count(const srcv_sparse_tsdf* volume, const srcv_sparse_mesh_args* args, int64_t* counts,
                                    void* workspace, size_t workspace_bytes, void* stream);
int32_t srcv_sparse_tsdf_mesh_extract(const srcv_sparse_tsdf* volume, const srcv_sparse_mesh_args* args, float* verts,
                                      float* normals, float* vert_colors, int32_t* faces, int64_t V, int64_t F,
                                      void* workspace, size_t workspace_bytes, void* stream);
int32_t srcv_sparse_tsdf_read_box(const srcv_sparse_tsdf* volume, const int32_t lo[3], const int32_t dims[3],
                                  void* values, void* weights, void* colors, void* stream);

/* ---- mesh evaluation (DESIGN §4.17) ------------------------------------------------------ *
 * Scores a predicted surface P against a ground truth G (metres, fp32 coordinates).  With
 * d(x, S) = min over s in S of |x - s|, evaluated in fp64 from the fp32 coordinates, and threshold tau:
 *   acc = mean_p d(p, G)   comp = mean_g d(g, P)   chamfer = (acc + comp) / 2
 *   precision = share of p with d(p, G) < tau   recall = share of g with d(g, P) < tau
 *   fscore = 2 precision recall / (precision + recall), 0 when both are 0.
 * srcv_mesh_sample_f32 draws num_samples points (num_samples,3) f32 uniformly by area from the mesh
 *   (verts (V,3) f32, faces (num_faces,3) int32, DEVICE): sample i takes uniforms u_k = U(seed, i, k),
 *   k = 0, 1, 2, with U the counter hash of DESIGN §4.17; its triangle is the first whose inclusive area CDF
 *   exceeds (i + u0) / num_samples * total area; its point is (1 - sqrt u1) a + sqrt u1 (1 - u2) b +
 *   sqrt u1 u2 c in fp64.  Same inputs and seed: bitwise the same samples.  5 launches.
 * srcv_nearest_distances_f32: dist (num_queries) f64 out = d(query, points) for queries (num_queries,3)
 *   and points (num_points,3) f32, DEVICE; exact (four grid levels plus a brute-force queue).  32 launches;
 *   a level no query reaches exits at once.
 * srcv_mesh_metrics_f64: from dist_pred (num_queries = |P|) = d(p, G) and dist_gt (num_points = |G|) =
 *   d(g, P), metrics (8) f64 out: acc, comp, chamfer, precision, recall, fscore, the flag word, 0.
 *   fp64 sums and int64 counts in a fixed order.  3 launches.
 * flags: DEVICE uint32 the caller zeroes; the calls OR into it SRCV_MESH_EVAL_BAD_FACE (a face index outside
 *   [0, V)), _NONFINITE (a non-finite coordinate or area) and _ZERO_AREA (a mesh of zero total area).  Once a
 *   bit is set the later kernels read nothing out of bounds and write NaN.  stats: optional DEVICE int64[8],
 *   written by srcv_nearest_distances_f32: per grid level (cell edge h, 8h, 64h, 512h) the target points its
 *   search evaluated, then per level the queries it left open (the last of these reached the brute force).
 * Nothing synchronises with the host.  Limits (SRCV_ERR_SHAPE): 1 <= num_points, num_queries, num_samples
 * <= 2^28 (the workspace is about 48 bytes per target point and 16 per query, ~25 GB at the limit); 1 <= num_faces, V < 2^31.  The workspace is sized by srcv_mesh_eval_workspace_bytes for the same
 * args, 256-byte aligned.                                                                                   */
#define SRCV_MESH_EVAL_BAD_FACE 1u
#define SRCV_MESH_EVAL_NONFINITE 2u
#define SRCV_MESH_EVAL_ZERO_AREA 4u
typedef struct srcv_mesh_eval_args {
  int64_t num_faces;        /* faces of the mesh sampled (0: no sampling)                  */
  int64_t num_queries;      /* queries of the distances; |P| of the metrics                */
  int64_t num_points;       /* target points of the distances; |G| of the metrics          */
  uint32_t* flags;          /* DEVICE, one word                                            */
  int64_t* stats;           /* DEVICE int64[8] or NULL                                     */
} srcv_mesh_eval_args;
size_t srcv_mesh_eval_workspace_bytes(const srcv_mesh_eval_args* args);
int32_t srcv_mesh_sample_f32(const srcv_mesh_eval_args* args, const float* verts, int32_t V, const int32_t* faces,
                             int64_t num_samples, uint64_t seed, float* samples, void* workspace,
                             size_t workspace_bytes, void* stream);
int32_t srcv_nearest_distances_f32(const srcv_mesh_eval_args* args, const float* queries, const float* points,
                                   double* dist, void* workspace, size_t workspace_bytes, void* stream);
int32_t srcv_mesh_metrics_f64(const srcv_mesh_eval_args* args, const double* dist_pred, const double* dist_gt,
                              double threshold, double* metrics, void* workspace, size_t workspace_bytes,
                              void* stream);

/* ---- visibility culling for mesh evaluation (DESIGN §4.18) ------------------------------- *
 * Point p (fp32, metres) is observed by frame f when fusing f's depth map would update a voxel at p.  In fp64
 * from the fp32 inputs, in this order, with E = cam_T_world[f] (world -> camera) and K = K[f]:
 *   x = ((E00 px + E01 py) + E02 pz) + E03, likewise y, z;  U = (K00 x + K01 y) + K02 z, likewise V;
 *   ix = rint(U / z - 0.5), iy = rint(V / z - 0.5), rounding half to even;
 *   observed <=> 0 < z < max_depth, 0 <= ix < W, 0 <= iy < H, 0 < d < max_depth for d = depths[f, iy, ix],
 *   and d - z > -margin.
 * srcv_observation_counts_f32: counts (num_points) int32 in/out += the frames observing each point of points
 *   (num_points,3) f32, DEVICE.  Integer counts, no other atomics: bitwise deterministic.  Feeding the frames
 *   in chunks over several calls gives the counts of one call.  1 launch.  stats: optional DEVICE int64[1],
 *   += the (point, frame) pairs evaluated after the per-tile frustum test (tile_cull).
 * srcv_compact_observed_f32: kept (num_points,3) f32 out = the points with counts > 0, in input order;
 *   num_kept DEVICE int64 out = their number.  5 launches; workspace from srcv_mesh_eval_workspace_bytes with
 *   the same args.
 * flags (as above): a non-finite point coordinate ORs SRCV_MESH_EVAL_NONFINITE, a non-finite entry of the E rows
 *   0..2 or the K entries used SRCV_MESH_EVAL_BAD_VIEW; such points and frames observe nothing.
 * Limits (SRCV_ERR_SHAPE): 1 <= num_points <= 2^28; F, H, W >= 1, H W < 2^31; margin finite and >= 0;
 * max_depth > 0 (may be +inf).  Nothing synchronises with the host.                                          */
#define SRCV_MESH_EVAL_BAD_VIEW 8u
typedef struct srcv_mesh_views {
  const float* depths;      /* DEVICE (F,H,W) f32, metres                                   */
  const float* K;           /* DEVICE (F,4,4) f32, or one (4,4) when K_shared               */
  const float* cam_T_world; /* DEVICE (F,4,4) f32, world -> camera                          */
  int32_t F, H, W;
  int32_t K_shared;         /* 1: one K for every frame                                     */
  double margin;            /* metres, >= 0                                                 */
  double max_depth;         /* metres, > 0, may be +inf                                     */
  int32_t tile_cull;        /* 1: skip a frame for a tile of 256 points whose bounding box
                               lies outside its frustum (the result is the same); 0: test
                               every frame for every point (for measurement)               */
} srcv_mesh_views;
int32_t srcv_observation_counts_f32(const srcv_mesh_eval_args* args, const srcv_mesh_views* views,
                                    const float* points, int32_t* counts, void* stream);
int32_t srcv_compact_observed_f32(const srcv_mesh_eval_args* args, const float* points, const int32_t* counts,
                                  float* kept, int64_t* num_kept, void* workspace, size_t workspace_bytes,
                                  void* stream);

/* ---- voxel down-sampling (DESIGN §4.19) --------------------------------------------------- *
 * Open3D's VoxelDownSample rule, in fp64 from the fp32 points (metres) and voxel size s:
 *   b = min_i p_i - 0.5 s per axis;  voxel of p: v = floor((p - b) / s), an IEEE subtraction and division;
 *   each occupied voxel's point is the fp64 sum of its points, accumulated in input order from 0.0, divided by
 *   their count and rounded once to fp32; colours likewise (uint8 taken as c / 255.0 in fp64, floats as given).
 * srcv_voxel_down_sample_f32: points (num_points,3) f32 and colors (num_points,3) of color_type (NULL for
 *   SRCV_COLORS_NONE), DEVICE.  out_points (num_points,3) f32, out_colors (num_points,3) f32 (NULL without
 *   colours) and out_counts (num_points) int32 out: the first M rows, one per occupied voxel in ascending
 *   (vx, vy, vz) order; num_out DEVICE int64 out = M.  A stable LSD radix sort of the voxel keys with as many
 *   8-bit passes as the extent needs: bitwise deterministic, independent of thread timing and input order.
 *   49 launches; the sort passes the extent does not need exit at once.
 * flags: DEVICE uint32 the caller zeroes; ORs SRCV_MESH_EVAL_NONFINITE (a non-finite coordinate),
 *   SRCV_VOXEL_NONFINITE_COLOR (a non-finite colour) and SRCV_VOXEL_EXTENT (2^21 or more voxels on an axis).
 *   Once a coordinate or extent bit is set no output row is written.
 * Limits (SRCV_ERR_SHAPE): 1 <= num_points <= 2^28; s finite and > 0.  The workspace (about 40 bytes per point)
 * is sized by srcv_voxel_down_sample_workspace_bytes (0 outside the limits).  Nothing synchronises with the
 * host.                                                                                                      */
#define SRCV_VOXEL_NONFINITE_COLOR 16u
#define SRCV_VOXEL_EXTENT 32u
#define SRCV_COLORS_NONE 0
#define SRCV_COLORS_U8 1
#define SRCV_COLORS_F32 2
#define SRCV_COLORS_F64 3
size_t srcv_voxel_down_sample_workspace_bytes(int64_t num_points);
int32_t srcv_voxel_down_sample_f32(const float* points, int64_t num_points, double voxel_size, const void* colors,
                                   int32_t color_type, float* out_points, float* out_colors, int32_t* out_counts,
                                   int64_t* num_out, uint32_t* flags, void* workspace, size_t workspace_bytes,
                                   void* stream);

/* ---- multi-view depth consistency (point-cloud fusion) ------------------------------ *
 * Replaces process_depth of the reference's 3DVNet-style fuser (tools/torch_point_cloud_fusion.py
 * :12-97), which pc_fusion.py:158 runs for every frame of a scan against all the others: for each
 * pixel of frame `ref_index`, un-project, re-project into every other frame, nearest-sample its
 * depth, count the frames that agree within z_thresh, and average the back-projected consistent
 * samples with the pixel's own point.  fp32, the reference's operation order.
 *   scan: N frames — depths (N,H,W), K and K_inv (N,3,3), cam_T_world and world_T_cam (N,4,4)
 *         (the caller inverts once per scan; the reference inverts per call, :25-27), all DEVICE
 *   pts_avg (H*W,3) out    n_valid (H*W) int32 out    valid (H*W) uint8 out (n_valid >= n_consistent)
 * The workspace keeps the staged per-frame matrices: pass frames_ready != 0 on every call after
 * the first of a scan to skip re-staging them.  Limits (SRCV_ERR_SHAPE): N >= 1, H, W >= 2,
 * H W <= 2^26, N H W <= 2^40; srcv_mvs_workspace_bytes is 0 outside them.                   */
typedef struct srcv_mvs_scan {
  const float* depths;
  const float* K;
  const float* K_inv;
  const float* cam_T_world;
  const float* world_T_cam;
  int32_t N, H, W;
} srcv_mvs_scan;
size_t srcv_mvs_workspace_bytes(const srcv_mvs_scan* scan);
int32_t srcv_mvs_consistency_f32(const srcv_mvs_scan* scan, int32_t ref_index, float z_thresh,
                                 int32_t n_consistent, float* pts_avg, int32_t* n_valid, uint8_t* valid,
                                 void* workspace, size_t workspace_bytes, int32_t frames_ready, void* stream);

/* ---- multi-view depth regression loss (training) ------------------------------------- *
 * Replaces MVDepthLoss.forward of the reference (losses.py:180-208, with get_valid_mask :90-135
 * and get_error_for_pair :138-178; called from experiment_modules/depth_model.py:477-485): for every
 * source view, the whole-batch mean over valid pixels of |log s - log z|, s = the view's depth
 * nearest-sampled where the GROUND-TRUTH depth projects, z = the depth of the PREDICTED point in
 * that view; the loss is the mean over the views.  NaN terms are dropped (nanmean).  fp32, the
 * reference's operation order.  All pointers DEVICE memory, dense:
 *   depth_pred, cur_depth (B,1,H,W)   src_depth (B,K,1,H,W)
 *   cur_invK, cur_world_T_cam (B,4,4)   src_K, src_cam_T_world (B,K,4,4)          K <= 16
 * forward : loss (1 float) out; optional valid_mask (B,K,H,W) uint8 and src_depth_sampled
 *           (B,K,H,W) float outputs = get_valid_mask of every view (NULL: not written).
 * backward: grad_depth_pred (B,1,H,W) out = grad_loss[0] * d loss / d depth_pred; `workspace` must
 *           be the one the forward call of the same arguments filled (it keeps the per-view counts).
 * Deterministic: per-CTA partial sums reduced in a fixed order.
 * Limits: B, K, H, W >= 1, B <= 65535, H W <= 2^26, B K H W <= 2^40 (SRCV_ERR_SHAPE) and K <= 16
 * (SRCV_ERR_UNSUPPORTED); srcv_mvloss_workspace_bytes is 0 outside them.                         */
typedef struct srcv_mvloss_args {
  const float* depth_pred;
  const float* cur_depth;
  const float* src_depth;
  const float* cur_invK;
  const float* src_K;
  const float* cur_world_T_cam;
  const float* src_cam_T_world;
  int32_t B, K, H, W;
} srcv_mvloss_args;
size_t srcv_mvloss_workspace_bytes(const srcv_mvloss_args* args);
int32_t srcv_mvloss_forward_f32(const srcv_mvloss_args* args, float* loss, uint8_t* valid_mask,
                                float* src_depth_sampled, void* workspace, size_t workspace_bytes,
                                void* stream);
int32_t srcv_mvloss_backward_f32(const srcv_mvloss_args* args, const float* grad_loss,
                                 float* grad_depth_pred, const void* workspace, size_t workspace_bytes,
                                 void* stream);

/* ---- depth metrics (evaluation and training logs) ------------------------------------ *
 * Replaces compute_depth_metrics_batched and compute_depth_metrics of the reference
 * (utils/metrics_utils.py:7-120) together with the resampling test.py:282-299 runs before them
 * (F.interpolate of the prediction to the ground-truth size, then gt > 0.5).  DESIGN §4.12.
 *   gt     DEVICE (B,H,W) fp32 ground truth          pred  DEVICE (B,Hp,Wp) fp32 prediction
 *   valid  DEVICE (B,H,W) uint8 (0 = invalid), read when valid_source == SRCV_METRICS_VALID_MASK
 *   (each may be NULL when it holds no element: H*W == 0 gives NaN metrics and zero counts)
 * Per pixel, with the prediction v sampled at the ground-truth pixel (PyTorch's rules,
 * align_corners=False; a same-size nearest or bilinear resampling is the identity):
 *   thresh = max(gt/v, v/gt) (NaN-propagating); a_t counts thresh < t for the fp32 constants
 *   1.05, 1.10, 1.25, 1.25^2, 1.25^3; the terms |gt-v|, |gt-v|/gt, (gt-v)^2/gt, (gt-v)^2 and
 *   (log gt - log v)^2 are fp32 ops in the reference's order.
 * Sums are fp64, counts are integers, and each metric is the fp32 rounding of the fp64 formula:
 *   metrics (B,12) f32 out: abs_diff, abs_rel, sq_rel, rmse, rmse_log, a5, a10, a25, a0 (= a10),
 *                  a1 (= a25), a2, a3 — the a-values are a_count / valid_count, times 100 in
 *                  fp32 when mult_a; rmse and rmse_log are sqrt of the mean;
 *   valid_counts (B) int64 out; upsampled (B,H,W) f32 out = the resampled prediction, or NULL.
 * SRCV_METRICS_BATCHED: each continuous metric is the mean of its non-NaN terms (nanmean);
 * SRCV_METRICS_FLAT: plain means, NaN if any term is NaN.  A frame without valid pixels gives NaN.
 * Two launches (per-CTA partials, then one CTA per frame summing them in a fixed order): no
 * atomics, no host synchronisation, bit-identical on every run.  At most 2^30 pixels per frame
 * (H*W and Hp*Wp), B <= 65535.  Workspace: 128 bytes per 1024 ground-truth pixels per frame.     */
typedef enum srcv_resample_mode {
  SRCV_RESAMPLE_IDENTITY = 0, /* Hp == H, Wp == W                         */
  SRCV_RESAMPLE_NEAREST = 1,  /* src = min(floor(dst * fp32(in/out)), in-1) */
  SRCV_RESAMPLE_BILINEAR = 2  /* src = max(0, fp32(in/out) (dst + 0.5) - 0.5) */
} srcv_resample_mode;
typedef enum srcv_metrics_nan_mode { SRCV_METRICS_BATCHED = 0, SRCV_METRICS_FLAT = 1 } srcv_metrics_nan_mode;
typedef enum srcv_metrics_valid_source {
  SRCV_METRICS_VALID_MASK = 0,      /* valid[p] != 0                 */
  SRCV_METRICS_VALID_MIN_DEPTH = 1, /* gt > min_valid_depth, in fp32 */
  SRCV_METRICS_VALID_ALL = 2        /* every pixel                   */
} srcv_metrics_valid_source;
typedef struct srcv_metrics_args {
  const float* gt;
  const float* pred;
  const uint8_t* valid;
  float min_valid_depth;
  int32_t B, H, W, Hp, Wp;
  int32_t resample;      /* srcv_resample_mode        */
  int32_t nan_mode;      /* srcv_metrics_nan_mode     */
  int32_t valid_source;  /* srcv_metrics_valid_source */
  int32_t mult_a;
} srcv_metrics_args;
size_t srcv_metrics_workspace_bytes(const srcv_metrics_args* args);
int32_t srcv_depth_metrics_f32(const srcv_metrics_args* args, float* metrics, int64_t* valid_counts, float* upsampled,
                               void* workspace, size_t workspace_bytes, void* stream);

/* ---- surface normals from depth (training loss, Equation 4) --------------------------- *
 * Replaces NormalGenerator.forward of the reference (utils/geometry_utils.py:92-133; called twice
 * per training step, experiment_modules/depth_model.py:526, :530).  DESIGN §4.13.  Per pixel:
 *   S = the separable Gaussian blur of depth (x pass, then y pass, cross-correlations with `taps`,
 *       PyTorch 'reflect' padding);  P = S * invK[:3,:3] (x + .5, y + .5, 1);
 *   Gx, Gy = Sobel of P, normalised (1/8), replicate padding (a tap outside the map reads P of the
 *       clamped pixel);  normal = c / max(|c|, 1e-12), c = Gx x Gy.
 * A non-finite depth anywhere in the pixel's (k + 2) x (k + 2) window (after the reflect and clamp
 * maps) makes all three components NaN.  All pointers DEVICE memory, dense fp32:
 *   depth (B,1,H,W)   invK (B,4,4)   taps (k) (the caller computes them, kornia's gaussian(k, sigma))
 *   normals (B,3,H,W) out
 * backward: grad_depth (B,1,H,W) out from grad_normals (B,3,H,W).  Pixels whose window holds a
 *   non-finite depth pass no gradient.  Workspace: srcv_normals_workspace_bytes (24 bytes per pixel),
 *   scratch only (nothing is kept between calls).
 * Limits (SRCV_ERR_SHAPE): k odd in [1, 15]; min(H, W) > k/2 (the reflect padding); 1 <= B <= 65535;
 * 6 B H W < 2^31 (32-bit element indices).  One forward launch, two backward launches; gather form,
 * no atomics: bit-identical on every run.                                                         */
typedef struct srcv_normals_args {
  const float* depth;
  const float* invK;
  const float* taps;
  int32_t B, H, W, k;
} srcv_normals_args;
size_t srcv_normals_workspace_bytes(const srcv_normals_args* args);
int32_t srcv_normals_forward_f32(const srcv_normals_args* args, float* normals, void* stream);
int32_t srcv_normals_backward_f32(const srcv_normals_args* args, const float* grad_normals, float* grad_depth,
                                  void* workspace, size_t workspace_bytes, void* stream);

/* ---- normals loss ----------------------------------------------------------------------- *
 * Replaces NormalsLoss.forward of the reference (losses.py:57-77; depth_model.py:475): the mean over
 * the pixels whose six components (both normals) are finite of 0.5 (1 - pred . gt), fp32 terms, fp64
 * sum, exact count.  No such pixel: the loss is NaN and the gradients are zero.
 *   normals_gt, normals_pred DEVICE (B,3,H,W) fp32     loss DEVICE (1 float) out
 * backward: grad_pred = -0.5 gt (grad_loss[0] / count) at masked pixels and 0 elsewhere; grad_gt the
 *   same with pred (grad_gt may be NULL).  `workspace` must be the one the forward call on the same
 *   inputs filled: it keeps the count, so nothing goes through the host.
 * Limits: B, H, W >= 1, 3 B H W < 2^31.  Two forward launches (per-CTA partials, a fixed-order
 * finalize), one backward launch; bit-identical on every run.                                     */
size_t srcv_normals_loss_workspace_bytes(int32_t B, int32_t H, int32_t W);
int32_t srcv_normals_loss_forward_f32(const float* normals_gt, const float* normals_pred, int32_t B, int32_t H,
                                      int32_t W, float* loss, void* workspace, size_t workspace_bytes, void* stream);
int32_t srcv_normals_loss_backward_f32(const float* normals_gt, const float* normals_pred, int32_t B, int32_t H,
                                       int32_t W, const float* grad_loss, float* grad_pred, float* grad_gt,
                                       const void* workspace, size_t workspace_bytes, void* stream);

/* ---- multi-scale gradient loss (training loss, Equation 3) ------------------------------ *
 * Replaces MSGradientLoss.forward of the reference (losses.py:11-37; depth_model.py:466, :487).
 * DESIGN §4.14.  Level 0 is the input; level l is blur_pool2d of level l-1: the [1,2,1] x [1,2,1] / 16
 * kernel at stride 2 with zero padding 1, size ceil(h / 2).  Per level, Gx and Gy are the Sobel
 * gradients / 8 with replicate padding of both tensors; a gradient component is in the mask when all
 * nine clamped window values of the ground truth at that level are finite; the level's term is the
 * mean of |G(pred) - G(gt)| over the masked components (fp32 terms, fp64 sum, exact count), and the
 * loss is the sum over the levels.  A level without a masked component makes the loss NaN and passes
 * no gradient.  All pointers DEVICE memory, dense fp32:
 *   depth_gt, depth_pred (B,1,H,W)     loss (1 float) out
 * backward: grad_pred (B,1,H,W) out from grad_loss (1 float): per level the Sobel adjoint of
 *   sign(delta) mask grad_loss / count, summed down the pyramid through the blur-pool adjoints.
 *   `workspace` must be the one the forward call on the same inputs filled.
 * Workspace layout (srcv_msgrad_workspace_bytes):
 *   [ counts: 4 x int64 = masked components per level, 0 past num_scales; padded to 256 bytes
 *   | partial sums (double) then partial counts (int64), one per CTA of the loss launch; padded to 256
 *   | ground-truth pyramid: levels 1..num_scales-1, each (B,h_l,w_l) fp32 | prediction pyramid
 *   | gradient pyramid (scratch of the backward) ]
 * Limits (SRCV_ERR_SHAPE): num_scales in [1, 4]; H, W >= 1; 1 <= B <= 65535; B H W < 2^30.  At most three
 * forward launches (pyramids, per-CTA partials, a fixed-order finalize) and num_scales backward
 * launches; gather form, no atomics, no host synchronisation: bit-identical on every run.          */
size_t srcv_msgrad_workspace_bytes(int32_t B, int32_t H, int32_t W, int32_t num_scales);
int32_t srcv_msgrad_forward_f32(const float* depth_gt, const float* depth_pred, int32_t B, int32_t H, int32_t W,
                                int32_t num_scales, float* loss, void* workspace, size_t workspace_bytes,
                                void* stream);
int32_t srcv_msgrad_backward_f32(const float* depth_gt, const float* depth_pred, int32_t B, int32_t H, int32_t W,
                                 int32_t num_scales, const float* grad_loss, float* grad_pred, void* workspace,
                                 size_t workspace_bytes, void* stream);

/* ---- scale-invariant loss --------------------------------------------------------------- *
 * Replaces ScaleInvariantLoss.forward of the reference (losses.py:39-54; depth_model.py:468):
 *   loss = sqrt(mean(d^2) - si_lambda mean(d)^2),  d = log_depth_gt - log_depth_pred (n fp32 elements
 * each, DEVICE), d in fp32, the sums and the formula in fp64.  A negative radicand or n == 0 gives NaN
 * (with n == 0 the two inputs may be NULL).
 * backward: grad_gt = grad_loss[0] (d - si_lambda mean(d)) / (n loss), grad_pred = -grad_gt (either may
 *   be NULL).  `workspace` must be the one the forward call on the same inputs filled:
 *   [ mean(d): double, loss: double, n: int64; padded to 256 bytes | partial sums of d, then of d^2 ]
 * Limits: 0 <= n < 2^31.  Two forward launches, one backward launch (none when n == 0); bit-identical
 * on every run.                                                                                    */
size_t srcv_si_loss_workspace_bytes(int64_t n);
int32_t srcv_si_loss_forward_f32(const float* log_depth_gt, const float* log_depth_pred, int64_t n, double si_lambda,
                                 float* loss, void* workspace, size_t workspace_bytes, void* stream);
int32_t srcv_si_loss_backward_f32(const float* log_depth_gt, const float* log_depth_pred, int64_t n,
                                  double si_lambda, const float* grad_loss, float* grad_gt, float* grad_pred,
                                  const void* workspace, size_t workspace_bytes, void* stream);

/* ---- regression terms of the training loss (Equation 2 and the logged terms) ------------ *
 * Replaces lines 447-474 of DepthModel.compute_losses of the reference (experiment_modules/depth_model.py).
 * DESIGN §4.15.  Over the whole batch, with lg = log(gt) in fp32 and n = the number of pixels whose mask byte is
 * nonzero:
 *   ms_loss      = sum over the present scales i of mean_mask |lg - lp_i(nearest)| / 2^i, lp_i sampled at
 *                  PyTorch's nearest source index min(floor(dst * in/out), in - 1) (fp32 scale)
 *   abs_loss     = mean_mask |gt - depth_pred|            log_l1_loss = mean_mask |lg - lp_0|
 *   si_loss      = sqrt(mean(d^2) - si_lambda mean(d)^2), d = lg - lp_0 over the mask
 *   inv_abs_loss = mean |1/gt - 1/depth_pred| over the mask and depth_pred > 0.1f (its own count m)
 * fp32 terms, fp64 sums, exact counts; an empty mask (n = 0, or m = 0 for inv_abs_loss) gives NaN.  Values
 * outside the mask are never read as terms, so NaN ground truth there is ignored.  All pointers DEVICE memory,
 * dense:
 *   gt, depth_pred (B,1,H,W) fp32   mask (B,1,H,W) uint8   log_pred[i] (B,1,h[i],w[i]) fp32 or NULL (absent)
 *   losses (5 floats) out, in the order ms_loss, abs_loss, si_loss, inv_abs_loss, log_l1_loss
 * backward: grad_losses[5] point to the upstream gradient of each loss in the same order (NULL, or a zero, adds
 *   nothing: an output autograd did not reach); grad_log_pred[i] (B,1,h[i],w[i]) and grad_depth_pred (B,1,H,W)
 *   out, each may be NULL (not wanted).  At scale i >= 1 the gradient is sign(lp_i - lg) mask g_ms / (n 2^i)
 *   summed over the pixel's nearest-resampling preimage (0 for an empty preimage); sign(0) = sign(NaN) = 0.
 *   `workspace` must be the one the forward call on the same inputs filled.
 * Workspace layout (srcv_regloss_workspace_bytes):
 *   [ n, m: int64; mean(d), si_loss: double; padded to 256 bytes
 *   | partial sums: 6 series (ms, abs, log_l1, d, d^2, inv_abs) of one double per forward CTA
 *   | partial counts: 2 series (n, m) of one int64 per forward CTA; padded to 256 ]
 * Limits (SRCV_ERR_SHAPE): 1 <= B <= 65535; H, W >= 1; B H W < 2^30; log_pred[0] required (SRCV_ERR_NULL)
 *   with h[0] = H, w[0] = W; every present scale h[i], w[i] >= 1 with B h[i] w[i] < 2^30.  Two forward
 *   launches (per-CTA partials, a fixed-order finalize), one backward launch; gather form, no atomics, no host
 *   synchronisation: bit-identical on every run.                                                      */
typedef struct srcv_regloss_args {
  const float* gt;
  const uint8_t* mask;
  const float* depth_pred;
  const float* log_pred[4];
  int32_t h[4], w[4];
  int32_t B, H, W;
  double si_lambda;
} srcv_regloss_args;
size_t srcv_regloss_workspace_bytes(const srcv_regloss_args* args);
int32_t srcv_regloss_forward_f32(const srcv_regloss_args* args, float* losses, void* workspace, size_t workspace_bytes,
                                 void* stream);
int32_t srcv_regloss_backward_f32(const srcv_regloss_args* args, const float* const grad_losses[5],
                                  float* const grad_log_pred[4], float* grad_depth_pred, const void* workspace,
                                  size_t workspace_bytes, void* stream);

/* ---- tuning / introspection ------------------------------------------- *
 * Selects the kernel variant used by the two forward calls on this thread's
 * next invocations (process-global).  0 = automatic choice.  Used by the tests
 * to exercise every variant against the oracle and by bench.py to report which
 * one ran.  Unknown values are rejected with SRCV_ERR_UNSUPPORTED.           */
typedef enum srcv_variant {
  SRCV_VARIANT_AUTO = 0,
  SRCV_VARIANT_GENERIC = 1, /* shape-generic SIMT kernels                     */
  SRCV_VARIANT_FAST = 2     /* chunk-planar gather / wgmma kernels            */
} srcv_variant;
int32_t srcv_set_variant(int32_t variant);
/* Name of the kernel variant the last forward call on this process launched. */
const char* srcv_last_variant(void);
/* Number of kernel launches issued by the library since load (monotonic).    */
uint64_t srcv_launch_count(void);


/* ---- tensor-core self-test (test support) -------------------------------- *
 * D (128,128) = A (128,Kp) W^T, W (128,Kp), all DEVICE fp32, Kp a multiple of 16
 * and <= 256, through the same descriptors and (hi, lo) split as the
 * metadata-MLP kernel (fp16 hi/lo split, three MMAs).  `scratch` = 512*Kp bytes.  */
int32_t srcv_tc_selftest_f32(const float* A, const float* W, int32_t Kp, float* D, void* scratch,
                             void* stream);

/* ---- per-kernel timing (benchmark support) ---------------------------- *
 * Between srcv_profile_begin and srcv_profile_end every forward call records
 * CUDA events on ITS stream around the prep pass and around the sweep kernel(s)
 * (at most max_records calls are recorded; later ones run unrecorded).
 * srcv_profile_end waits for the recorded events, returns the summed device
 * times in milliseconds and the number of recorded calls, and releases the
 * events.  Outside a begin/end pair nothing is recorded.                     */
int32_t srcv_profile_begin(int32_t max_records);
int32_t srcv_profile_end(double* prep_ms_total, double* sweep_ms_total, int32_t* n_records);

#ifdef __cplusplus
}
#endif
#endif /* SRCV_B200_H_ */
