// Internal host-side launch interface between srcv_api.cu and the kernel files.
#pragma once
#ifdef SRCV_HOST_EMU
#include "emu_cuda.h"   // tests/emu: the kernels compiled as host C++ (one std::thread per CUDA thread)
#else
#include <cuda_runtime.h>
#endif
#include <stddef.h>
#include <stdint.h>

#include "../../include/srcv_b200.h"
#include "srcv_common.cuh"
#include "srcv_reduce.cuh"

// One spelling for a kernel launch, so that the host emulation (tests/emu) can run the same
// launcher code: a template kernel name with commas goes in parentheses.
#ifdef SRCV_HOST_EMU
#define SRCV_LAUNCH(kernel, grid, block, smem, stream, ...) \
  ::emu::launch(dim3(grid), dim3(block), (size_t)(smem), [&] { kernel(__VA_ARGS__); })
#else
#define SRCV_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<grid, block, smem, stream>>>(__VA_ARGS__)
#endif

namespace srcv {

// the size of a workspace region, rounded up to the 256-byte alignment of every region
inline size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

// Workspace carve-up (all offsets 256-byte aligned).
struct Workspace {
  float* planes;        // (B,D) plane depths (FROM_RANGE / PER_PLANE copy)
  ViewParams* views;    // (B,K)
  FrameParams* frames;  // (B)
  float* src_c4;        // (B,K,C/4,H,W,4) chunk-planar copy of src_feats, or nullptr
  float* cur_c4;        // (B,C/4,H,W,4) chunk-planar copy of cur_feats, or nullptr
  unsigned* tile_done;  // per (frame, pixel tile) completion counters, zeroed by the prep pass
  size_t tile_done_count;
  float* extra;         // variant-specific scratch, or nullptr
  size_t bytes;         // total bytes needed
};

Workspace carve_workspace(const srcv_shape& s, void* base, bool want_c4, size_t extra_bytes);

// counts kernel launches for srcv_launch_count()
void note_launch(int n = 1);

// prep: view/frame params, plane depths, optional chunk-planar copy of src_feats.
cudaError_t launch_prep(const srcv_shape& s, const srcv_cameras& cams, const srcv_planes& pl,
                        const float* src_feats, const float* cur_feats, const Workspace& ws,
                        bool need_poses, cudaStream_t stream);

// dot-product volume
cudaError_t launch_dot_generic(const srcv_shape& s, const float* cur, const float* src,
                               const Workspace& ws, const float* planes, bool per_pixel,
                               float* cost, float* lowest, cudaStream_t stream);
bool dot_fast_supported(const srcv_shape& s);
size_t dot_fast_tile_counters(const srcv_shape& s);
// `cur` is NCHW, or chunk-planar (B,C/4,H,W,4) when s.layout says so
cudaError_t launch_dot_fast(const srcv_shape& s, const float* cur, const Workspace& ws,
                            const float* planes, bool per_pixel, float* cost, float* lowest,
                            cudaStream_t stream);

// backward of the dot-product volume w.r.t. the feature inputs
bool dot_backward_supported(const srcv_shape& s);
cudaError_t launch_dot_backward(const srcv_shape& s, const float* cur, const float* src,
                                const Workspace& ws, const float* planes, bool per_pixel,
                                const float* gcost, float* gcur, float* gsrc, cudaStream_t stream);

// single-plane warp (the reference's warp_features helper)
cudaError_t launch_warp_planes(const srcv_shape& s, const float* src, const Workspace& ws,
                               const float* planes, bool per_pixel, float* warped, float* depths,
                               float* mask, float* pix, cudaStream_t stream);

// metadata-MLP volume
bool mlp_generic_supported(const srcv_shape& s, const srcv_mlp_weights& w);
size_t mlp_generic_extra_bytes(const srcv_shape& s, const srcv_mlp_weights& w);
cudaError_t launch_mlp_generic(const srcv_shape& s, const float* cur, const float* src,
                               const Workspace& ws, const float* planes, bool per_pixel,
                               const srcv_mlp_weights& w, float* cost, float* lowest,
                               uint8_t* mask, cudaStream_t stream);

// backward of the metadata-MLP volume (fp32 SIMT, recompute)
bool mlp_backward_supported(const srcv_shape& s, const srcv_mlp_weights& w);
size_t mlp_backward_extra_bytes(const srcv_shape& s, const srcv_mlp_weights& w);
cudaError_t launch_mlp_backward(const srcv_shape& s, const float* cur, const float* src,
                                const Workspace& ws, const float* planes, bool per_pixel,
                                const srcv_mlp_weights& w, const float* gcost, float* gcur,
                                float* gsrc, const srcv_mlp_grads& g, cudaStream_t stream);

// tensor-core variant (wgmma): K = 7, C = 16, 202 -> 128 -> 128 -> 1
bool mlp_tc_supported(const srcv_shape& s, const srcv_mlp_weights& w);
size_t mlp_tc_extra_bytes(const srcv_shape& s);
size_t mlp_tc_image_bytes();
cudaError_t launch_mlp_tc_pack(const srcv_mlp_weights& w, void* image, cudaStream_t stream);
cudaError_t launch_mlp_tc(const srcv_shape& s, const float* cur, const Workspace& ws,
                          const float* planes, bool per_pixel, const srcv_mlp_weights& w, float* cost,
                          float* lowest, uint8_t* mask, cudaStream_t stream);
cudaError_t launch_tc_selftest(const float* A, const float* Wm, int Kp, float* Dout, void* scratch,
                               cudaStream_t stream);

// producer-side fusion (csrc/srcv_producer.cu): InstanceNorm2d + chunk-planar layout
cudaError_t launch_instnorm_c4(const float* x, int B, int V, int C, int H, int W, float eps, float* cur_c4,
                               float* src_c4, cudaStream_t stream);

// dense-grid TSDF integration (csrc/srcv_tsdf.cu)
size_t tsdf_workspace_bytes(int frames);
// color != nullptr: also fuse the frames' colour into color->colors (DESIGN §4.11)
cudaError_t launch_tsdf_integrate(const srcv_tsdf_volume& v, const srcv_tsdf_frames& f, void* workspace,
                                  cudaStream_t stream, const srcv_tsdf_color* color = nullptr);

// marching-cubes mesh extraction from the TSDF volume (csrc/srcv_mesh.cuh)
size_t mesh_workspace_bytes(const srcv_mesh_args& a);
bool mesh_shape_supported(const srcv_mesh_args& a);
cudaError_t launch_mesh_count(const srcv_mesh_args& a, long long* counts, void* workspace, cudaStream_t stream);
cudaError_t mesh_read_totals(const srcv_mesh_args& a, void* workspace, long long totals[2], cudaStream_t stream);
// colors != nullptr: also vertex colours (V,3) from the (3,X,Y,Z) colour volume (DESIGN §4.11)
cudaError_t launch_mesh_extract(const srcv_mesh_args& a, float* verts, float* normals, int32_t* faces,
                                void* workspace, cudaStream_t stream, const float* colors = nullptr,
                                float* vert_colors = nullptr);

// the voxel-block hashed TSDF volume (csrc/srcv_tsdf_sparse.cuh, in the srcv_tsdf.cu unit)
size_t sparse_tsdf_state_bytes(const srcv_sparse_tsdf& v);
size_t sparse_tsdf_workspace_bytes(const srcv_tsdf_frames& f);
cudaError_t launch_sparse_tsdf_reset(const srcv_sparse_tsdf& v, cudaStream_t stream);
cudaError_t launch_sparse_tsdf_integrate(const srcv_sparse_tsdf& v, const srcv_tsdf_frames& f, void* workspace,
                                         cudaStream_t stream, const srcv_tsdf_color* color = nullptr);
cudaError_t launch_sparse_tsdf_read_box(const srcv_sparse_tsdf& v, const int lo[3], const int dims[3], void* values,
                                        void* weights, void* colors, cudaStream_t stream);
cudaError_t launch_sparse_mesh_begin(const srcv_sparse_tsdf& v, int blocks, cudaStream_t stream);
cudaError_t launch_sparse_mesh_end(const srcv_sparse_tsdf& v, int blocks, cudaStream_t stream);
size_t sparse_mesh_workspace_bytes(const srcv_sparse_mesh_args& a);
cudaError_t launch_sparse_mesh_count(const srcv_sparse_tsdf& v, const srcv_sparse_mesh_args& a, long long* counts,
                                     void* workspace, cudaStream_t stream);
cudaError_t sparse_mesh_read_totals(const srcv_sparse_mesh_args& a, void* workspace, long long totals[2],
                                    cudaStream_t stream);
cudaError_t launch_sparse_mesh_extract(const srcv_sparse_tsdf& v, const srcv_sparse_mesh_args& a, float* verts,
                                       float* normals, float* vert_colors, int32_t* faces, void* workspace,
                                       cudaStream_t stream);

// mesh evaluation: surface sampling, exact nearest distances, metrics (csrc/srcv_mesh_eval.cuh, in the srcv_tsdf.cu unit)
size_t mesh_eval_workspace_bytes(const srcv_mesh_eval_args& a);
cudaError_t launch_mesh_sample(const srcv_mesh_eval_args& a, const float* verts, int V, const int32_t* faces,
                               long long num_samples, unsigned long long seed, float* samples, void* workspace,
                               cudaStream_t stream);
cudaError_t launch_nearest_distances(const srcv_mesh_eval_args& a, const float* queries, const float* points,
                                     double* dist, void* workspace, cudaStream_t stream);
cudaError_t launch_mesh_metrics(const srcv_mesh_eval_args& a, const double* dist_pred, const double* dist_gt,
                                double threshold, double* metrics, void* workspace, cudaStream_t stream);

// multi-view depth consistency (csrc/srcv_mvs.cu)
size_t mvs_workspace_bytes(int n);
cudaError_t launch_mvs_consistency(const srcv_mvs_scan& s, int ref, float z_thresh, int n_consistent,
                                   float* pts_avg, int* n_valid, uint8_t* valid, void* workspace,
                                   bool frames_ready, cudaStream_t stream);

// multi-view depth regression loss (csrc/srcv_mvloss.cu)
int mvloss_max_views();
size_t mvloss_workspace_bytes(const srcv_mvloss_args& a);
cudaError_t launch_mvloss_forward(const srcv_mvloss_args& a, float* loss, uint8_t* valid, float* sampled,
                                  void* workspace, cudaStream_t stream);
cudaError_t launch_mvloss_backward(const srcv_mvloss_args& a, const float* grad_loss, float* grad_pred,
                                   const void* workspace, cudaStream_t stream);

// depth metrics (csrc/srcv_metrics.cuh, compiled in the srcv_mvloss.cu unit)
constexpr long long kMetricsMaxPixels = 1ll << 30;   // per frame, so that 32-bit pixel indices never overflow
bool metrics_shape_supported(const srcv_metrics_args& a);
size_t metrics_workspace_bytes(const srcv_metrics_args& a);
cudaError_t launch_metrics(const srcv_metrics_args& a, float* metrics, long long* valid_counts, float* upsampled,
                           void* workspace, cudaStream_t stream);

// surface normals from depth and the normals loss (csrc/srcv_normals.cuh, compiled in the srcv_mvloss.cu unit)
constexpr int kNormalsMaxKernel = 15;                 // largest (odd) Gaussian kernel size
size_t normals_workspace_bytes(const srcv_normals_args& a);
cudaError_t launch_normals_forward(const srcv_normals_args& a, float* normals, cudaStream_t stream);
cudaError_t launch_normals_backward(const srcv_normals_args& a, const float* grad_normals, float* grad_depth,
                                    void* workspace, cudaStream_t stream);
size_t normals_loss_workspace_bytes(int B, int H, int W);
cudaError_t launch_normals_loss_forward(const float* gt, const float* pred, int B, int H, int W, float* loss,
                                        void* workspace, cudaStream_t stream);
cudaError_t launch_normals_loss_backward(const float* gt, const float* pred, int B, int H, int W,
                                         const float* grad_loss, float* grad_pred, float* grad_gt,
                                         const void* workspace, cudaStream_t stream);

// multi-scale gradient loss and scale-invariant loss (csrc/srcv_gradloss.cuh, compiled in the srcv_mvloss.cu unit)
constexpr int kMsGradMaxScales = 4;                   // pyramid levels, the input included
size_t msgrad_workspace_bytes(int B, int H, int W, int num_scales);
cudaError_t launch_msgrad_forward(const float* gt, const float* pred, int B, int H, int W, int num_scales, float* loss,
                                  void* workspace, cudaStream_t stream);
cudaError_t launch_msgrad_backward(const float* gt, const float* pred, int B, int H, int W, int num_scales,
                                   const float* grad_loss, float* grad_pred, void* workspace, cudaStream_t stream);
size_t si_loss_workspace_bytes(long long n);
cudaError_t launch_si_loss_forward(const float* gt, const float* pred, long long n, double lambda, float* loss,
                                   void* workspace, cudaStream_t stream);
cudaError_t launch_si_loss_backward(const float* gt, const float* pred, long long n, double lambda,
                                    const float* grad_loss, float* grad_gt, float* grad_pred, const void* workspace,
                                    cudaStream_t stream);

// the regression terms of the training loss (csrc/srcv_regloss.cuh, compiled in the srcv_mvloss.cu unit)
constexpr int kRegLossMaxScales = 4;                  // decoder scales s0..s3
size_t regloss_workspace_bytes(const srcv_regloss_args& a);
cudaError_t launch_regloss_forward(const srcv_regloss_args& a, float* losses, void* workspace, cudaStream_t stream);
cudaError_t launch_regloss_backward(const srcv_regloss_args& a, const float* const grad_losses[5],
                                    float* const grad_log_pred[kRegLossMaxScales], float* grad_depth_pred,
                                    const void* workspace, cudaStream_t stream);

// argmax over planes -> plane depth (used by variants that do not fuse it)
cudaError_t launch_argmax(const srcv_shape& s, const float* cost, const float* planes,
                          bool per_pixel, float* lowest, cudaStream_t stream);

}  // namespace srcv
