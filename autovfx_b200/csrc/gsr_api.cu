// gsr_b200 — extern "C" surface declared in include/gsr_b200.h.
#include "gsr_common.cuh"
#include <cstring>
#include <nvtx3/nvToolsExt.h>  // header-only NVTX v3: the ranges cost nothing unless a profiler is attached

namespace {
struct NvtxRange {  // one named range per C-ABI call (SURVEY §5: the reference has no instrumentation; this build adds NVTX)
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};
}  // namespace

namespace gsr {
int forward_impl(const gsr_frame* f, const gsr_workspace* ws, float* out_color, float* out_depth, float* out_alpha,
                 int32_t* radii, const float* extra_colors, float* out_extra, int flags, cudaStream_t st);
int axis_normals_impl(int P, const float* means3D, const float* scales, const float* rotations, const float* campos, int remap01,
                      float* out, cudaStream_t st);
int sugar_normals_impl(int P, const float* positions, const float* scales, const float* quaternions, const float* campos, float* out,
                       cudaStream_t st);
int sugar_normals_backward_impl(int P, const float* positions, const float* scales, const float* quaternions, const float* campos,
                                const float* dL_dnormals, float* dL_dquaternions, cudaStream_t st);
int sugar_colors_impl(int P, int M, int deg, const float* positions, const float* campos, const float* directions, const float* sh_dc,
                      const float* sh_rest, const float* densities, float* out_colors, float* out_opacities, cudaStream_t st);
int sugar_colors_backward_impl(int P, int M, int deg, const float* positions, const float* campos, const float* directions,
                               const float* sh_dc, const float* sh_rest, const float* densities, const float* dL_dcolors,
                               const float* dL_dopacities, float* dL_dsh_dc, float* dL_dsh_rest, float* dL_dpositions, float* dL_ddensities,
                               cudaStream_t st);
int normal_maps_impl(int W, int H, const float* normal_img, const float* depth, const float* c2w, float fx, float fy, float cx, float cy,
                     float* out_normal, float* out_pseudo, cudaStream_t st);
int pack_frame_impl(int W, int H, const float* rgb, const float* alpha, const float* depth, const float* normal_hwc, float depth_scale,
                    uint8_t* rgba8, uint8_t* normal8, uint8_t* depth8, cudaStream_t st);
int backward_impl(const gsr_frame* f, const gsr_workspace* ws, const int32_t* radii, const float* out_alpha, const float* dL_dc,
                  const float* dL_dd, const float* dL_da, const float* extra_colors, const float* dL_de, float* dL_dextra,
                  const gsr_grads* g, bool det, void* scratch, size_t scratch_bytes, cudaStream_t st);
size_t backward_det_bytes(size_t R, int W, int H, bool extra);
int compose_impl(int N, int M, const float* xyz, const float* f_dc, const float* f_rest, const float* opacity_raw, const float* scaling_raw,
                 const float* rotation_raw, const gsr_object_xform* xform, float* means3D, float* shs, float* opacities, float* scales,
                 float* rotations, cudaStream_t st);
int activate_backward_impl(int N, int M, const float* xyz, const float* campos, const float* opacities, const float* scales,
                           const float* rotations, const float* rotation_raw, const float* g_o, const float* g_s, const float* g_r,
                           const float* g_sh, const float* g_e, float* d_opacity, float* d_scaling, float* d_rotation, float* d_fdc,
                           float* d_frest, cudaStream_t st);
int dist2_impl(int P, const float* points, float* out, void* ws, size_t ws_bytes, cudaStream_t st);
size_t dist2_bytes(int P);
int knn_impl(int P1, int P2, int K, const float* queries, const float* points, float* out_d, int64_t* out_i, void* ws, size_t ws_bytes,
             cudaStream_t st);
size_t knn_bytes(int P1, int P2);
size_t sugar_field_bytes(int P);
int sugar_field_impl(int N, int K, int P, int R, const float* x, const int64_t* rows, const int64_t* row_idx, const float* points,
                     const float* scaling, const float* quaternions, const float* strengths, float density_factor,
                     float opacity_min_clamp, float sdf_offset, float* out_density, float* out_opac, float* out_beta, float* out_sdf,
                     void* ws, size_t ws_bytes, cudaStream_t st);
int sugar_field_backward_impl(int N, int K, int P, int R, const float* x, const int64_t* rows, const int64_t* row_idx,
                              const float* points, const float* scaling, const float* quaternions, const float* strengths,
                              float density_factor, float opacity_min_clamp, float sdf_offset, const float* g_density, const float* g_opac,
                              const float* g_beta, const float* g_sdf, float* dx, float* d_points, float* d_scaling, float* d_quaternions,
                              float* d_strengths, void* ws, size_t ws_bytes, bool det, cudaStream_t st);
size_t sugar_field_backward_det_bytes(int N, int K, int P);
size_t sugar_sdf_normal_bytes(int P);
int sugar_sdf_normal_impl(int N, int K, int P, const float* x, const int64_t* gidx, const int64_t* knn, const float* points,
                          const float* scaling, const float* quaternions, const float* opac, float* out_loss, float* out_est, void* ws,
                          size_t ws_bytes, cudaStream_t st);
int sugar_sdf_normal_backward_impl(int N, int K, int P, const float* x, const int64_t* gidx, const int64_t* knn, const float* points,
                                   const float* scaling, const float* quaternions, const float* opac, const float* g_loss,
                                   const float* g_est, float* dx, float* d_points, float* d_quaternions, void* ws, size_t ws_bytes,
                                   bool det, cudaStream_t st);
size_t sugar_sdf_normal_backward_det_bytes(int N, int K, int P, bool with_loss);
int densify_stats_impl(int P, int C, const float* grad, const uint8_t* mask, const int32_t* radii, float* accum, float* denom,
                       float* max_radii, cudaStream_t st);
size_t densify_plan_bytes(int P);
int densify_plan_impl(int P, const float* accum, const float* denom, const float* scaling, const float* opacity, float max_grad,
                      float dense_thr, float min_opacity, int use_screen, float max_screen_size, float big_thr, int32_t* dst,
                      int32_t* totals, void* ws, size_t ws_bytes, cudaStream_t st);
int densify_apply_impl(int P, int S, int n_groups, const gsr_densify_group* groups, const int32_t* dst, const float* xyz,
                       const float* scaling, const float* rotation, const float* eps, int rotation_mode, cudaStream_t st);
int adam_step_impl(int n, const gsr_adam_tensor* tensors, cudaStream_t st);
size_t photometric_loss_bytes(int B, int C, int H, int W, int for_backward);
int photometric_loss_impl(int B, int C, int H, int W, const float* x, const int64_t* xs, const float* y, const int64_t* ys,
                          const float* window, int for_backward, float* out_l1, float* out_ssim, void* ws, size_t ws_bytes,
                          cudaStream_t st);
int photometric_loss_backward_impl(int B, int C, int H, int W, const float* x, const int64_t* xs, const float* y, const int64_t* ys,
                                   const float* window, const float* g_l1, const float* g_ssim, float* dx, const void* ws,
                                   size_t ws_bytes, cudaStream_t st);
int normal_loss_impl(int64_t n, const float* pred, const int64_t* ps, const float* gt, const int64_t* gs, const float* depth,
                     int64_t d_sp, float scene_scale, float* out, void* ws, size_t ws_bytes, cudaStream_t st);
int normal_loss_backward_impl(int64_t n, const float* pred, const int64_t* ps, const float* gt, const int64_t* gs, const float* depth,
                              int64_t d_sp, float scene_scale, const float* g_out, float* d_pred, const void* ws, size_t ws_bytes,
                              cudaStream_t st);
int anisotropic_loss_impl(int64_t P, const float* scales, float r, float* out, void* ws, size_t ws_bytes, cudaStream_t st);
int anisotropic_loss_backward_impl(int64_t P, const float* scales, float r, const float* g_out, float* d_scales, cudaStream_t st);
int percentile_low_impl(int64_t n, const float* x, float* out, void* ws, size_t ws_bytes, cudaStream_t st);
int composite_impl(int32_t W, int32_t H, const uint8_t* frame, const uint8_t* obj, const float* obj_d, const uint8_t* shadow,
                   const float* shadow_d, const uint8_t* all, const uint8_t* gs, const float* gs_d, const uint8_t* smoke,
                   const float* smoke_d, const float* smoke_pct, const uint8_t* fire, uint8_t* out, cudaStream_t st);
size_t sugar_sample_bytes(int P);
int sugar_sample_impl(int N, int P, float f, int volume, const uint8_t* mask, const float* strengths, const double* u, const float* z,
                      const float* points, const float* scaling, const float* quaternions, float* out_points, int64_t* out_idx,
                      double* out_total, void* ws, size_t ws_bytes, cudaStream_t st);
int sugar_sample_backward_impl(int N, int P, float f, const int64_t* idx, const float* z, const float* scaling, const float* quaternions,
                               const double* total, const float* dL_dsamples, float* d_points, float* d_scaling, float* d_quaternions,
                               bool det, void* scratch, size_t scratch_bytes, cudaStream_t st);
size_t sugar_sample_backward_det_bytes(int N, int P);
int profile_begin(int max_frames, int stride);
int set_option(const char* name, int value);
int profile_end(float* ms, int* frames);

// checkFrustum (rasterizer_impl.cu:54-66): in_frustum() only tests view-space z (auxiliary.h:154)
__global__ void k_mark_visible(int P, const float* __restrict__ means3D, const float* __restrict__ view, uint8_t* __restrict__ present) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    const float3 p = {means3D[3 * (size_t)idx], means3D[3 * (size_t)idx + 1], means3D[3 * (size_t)idx + 2]};
    const float3 pv = xform4x3(p, view);
    present[idx] = !(pv.z <= 0.2f);
}
}  // namespace gsr

extern "C" {

int gsr_abi_version(void) { return GSR_ABI_VERSION; }
const char* gsr_last_error(void) { return gsr::last_error(); }

size_t gsr_geom_bytes(int32_t P) { return gsr::GeomLayout((size_t)(P < 0 ? 0 : P)).total; }
size_t gsr_binning_bytes(size_t capacity) { return gsr::BinLayout(capacity < 1 ? 1 : capacity).total; }
size_t gsr_binning_capacity(size_t bytes) { return gsr::BinLayout::capacity_of(bytes); }
size_t gsr_binning_bytes_slab(size_t capacity, int32_t W, int32_t H, int32_t slab_stride) {
    if (slab_stride <= 0) return gsr_binning_bytes(capacity);
    const gsr::ImageLayout il(W < 1 ? 1 : W, H < 1 ? 1 : H);
    return gsr::BinLayout::bytes_with_slab(capacity < 1 ? 1 : capacity, (size_t)il.tiles * (size_t)slab_stride);
}
size_t gsr_binning_capacity_slab(size_t bytes, int32_t W, int32_t H, int32_t slab_stride) {
    if (slab_stride <= 0) return gsr_binning_capacity(bytes);
    const gsr::ImageLayout il(W < 1 ? 1 : W, H < 1 ? 1 : H);
    return gsr::BinLayout::slab_offset(gsr::BinLayout::capacity_of(bytes), (size_t)il.tiles * (size_t)slab_stride) / 8;
}
size_t gsr_image_bytes(int32_t W, int32_t H) { return gsr::ImageLayout(W < 1 ? 1 : W, H < 1 ? 1 : H).total; }

int gsr_forward(const gsr_frame* frame, const gsr_workspace* ws, float* out_color, float* out_depth, float* out_alpha,
                int32_t* radii, int flags, void* stream) {
    NvtxRange nvtx_("gsr_forward");
    return gsr::forward_impl(frame, ws, out_color, out_depth, out_alpha, radii, nullptr, nullptr, flags, (cudaStream_t)stream);
}

int gsr_forward_multi(const gsr_frame* frame, const gsr_workspace* ws, float* out_color, float* out_depth, float* out_alpha,
                      int32_t* radii, const float* extra_colors, float* out_extra, int flags, void* stream) {
    NvtxRange nvtx_("gsr_forward_multi");
    return gsr::forward_impl(frame, ws, out_color, out_depth, out_alpha, radii, extra_colors, out_extra, flags, (cudaStream_t)stream);
}

int gsr_axis_normals(int32_t P, const float* means3D, const float* scales, const float* rotations, const float* campos, int remap01,
                     float* out, void* stream) {
    NvtxRange nvtx_("gsr_axis_normals");
    return gsr::axis_normals_impl(P, means3D, scales, rotations, campos, remap01, out, (cudaStream_t)stream);
}

int gsr_sugar_normals(int32_t P, const float* positions, const float* scales, const float* quaternions, const float* campos, float* out,
                      void* stream) {
    NvtxRange nvtx_("gsr_sugar_normals");
    return gsr::sugar_normals_impl(P, positions, scales, quaternions, campos, out, (cudaStream_t)stream);
}

int gsr_sugar_normals_backward(int32_t P, const float* positions, const float* scales, const float* quaternions, const float* campos,
                               const float* dL_dnormals, float* dL_dquaternions, void* stream) {
    NvtxRange nvtx_("gsr_sugar_normals_backward");
    return gsr::sugar_normals_backward_impl(P, positions, scales, quaternions, campos, dL_dnormals, dL_dquaternions, (cudaStream_t)stream);
}

int gsr_sugar_colors(int32_t P, int32_t M, int32_t deg, const float* positions, const float* campos, const float* directions,
                     const float* sh_dc, const float* sh_rest, const float* densities, float* out_colors, float* out_opacities, void* stream) {
    NvtxRange nvtx_("gsr_sugar_colors");
    return gsr::sugar_colors_impl(P, M, deg, positions, campos, directions, sh_dc, sh_rest, densities, out_colors, out_opacities,
                                  (cudaStream_t)stream);
}

int gsr_sugar_colors_backward(int32_t P, int32_t M, int32_t deg, const float* positions, const float* campos, const float* directions,
                              const float* sh_dc, const float* sh_rest, const float* densities, const float* dL_dcolors,
                              const float* dL_dopacities, float* dL_dsh_dc, float* dL_dsh_rest, float* dL_dpositions, float* dL_ddensities,
                              void* stream) {
    NvtxRange nvtx_("gsr_sugar_colors_backward");
    return gsr::sugar_colors_backward_impl(P, M, deg, positions, campos, directions, sh_dc, sh_rest, densities, dL_dcolors, dL_dopacities,
                                           dL_dsh_dc, dL_dsh_rest, dL_dpositions, dL_ddensities, (cudaStream_t)stream);
}

int gsr_normal_maps(int32_t W, int32_t H, const float* normal_img, const float* depth, const float* c2w, float fx, float fy, float cx,
                    float cy, float* out_normal, float* out_pseudo, void* stream) {
    NvtxRange nvtx_("gsr_normal_maps");
    return gsr::normal_maps_impl(W, H, normal_img, depth, c2w, fx, fy, cx, cy, out_normal, out_pseudo, (cudaStream_t)stream);
}

int gsr_pack_frame(int32_t W, int32_t H, const float* rgb, const float* alpha, const float* depth, const float* normal_hwc,
                   float depth_scale, uint8_t* rgba8, uint8_t* normal8, uint8_t* depth8, void* stream) {
    NvtxRange nvtx_("gsr_pack_frame");
    return gsr::pack_frame_impl(W, H, rgb, alpha, depth, normal_hwc, depth_scale, rgba8, normal8, depth8, (cudaStream_t)stream);
}

int gsr_activate_gaussians(int32_t N, int32_t M, const float* xyz, const float* f_dc, const float* f_rest, const float* opacity_raw,
                           const float* scaling_raw, const float* rotation_raw, const gsr_object_xform* xform, float* means3D, float* shs,
                           float* opacities, float* scales, float* rotations, void* stream) {
    NvtxRange nvtx_("gsr_activate_gaussians");
    return gsr::compose_impl(N, M, xyz, f_dc, f_rest, opacity_raw, scaling_raw, rotation_raw, xform, means3D, shs, opacities, scales, rotations,
                             (cudaStream_t)stream);
}

int gsr_activate_gaussians_backward(int32_t N, int32_t M, const float* xyz, const float* campos, const float* opacities,
                                    const float* scales, const float* rotations, const float* rotation_raw, const float* dL_dopacities,
                                    const float* dL_dscales, const float* dL_drotations, const float* dL_dshs, const float* dL_dnormals,
                                    float* dL_dopacity_raw, float* dL_dscaling_raw, float* dL_drotation_raw, float* dL_df_dc,
                                    float* dL_df_rest, void* stream) {
    NvtxRange nvtx_("gsr_activate_gaussians_backward");
    return gsr::activate_backward_impl(N, M, xyz, campos, opacities, scales, rotations, rotation_raw, dL_dopacities, dL_dscales,
                                       dL_drotations, dL_dshs, dL_dnormals, dL_dopacity_raw, dL_dscaling_raw, dL_drotation_raw, dL_df_dc,
                                       dL_df_rest, (cudaStream_t)stream);
}

int gsr_backward(const gsr_frame* frame, const gsr_workspace* ws, const int32_t* radii, const float* out_alpha,
                 const float* dL_dout_color, const float* dL_dout_depth, const float* dL_dout_alpha, const gsr_grads* grads,
                 void* stream) {
    NvtxRange nvtx_("gsr_backward");
    return gsr::backward_impl(frame, ws, radii, out_alpha, dL_dout_color, dL_dout_depth, dL_dout_alpha, nullptr, nullptr, nullptr, grads,
                              false, nullptr, 0, (cudaStream_t)stream);
}

int gsr_backward_multi(const gsr_frame* frame, const gsr_workspace* ws, const int32_t* radii, const float* out_alpha,
                       const float* dL_dout_color, const float* dL_dout_depth, const float* dL_dout_alpha, const float* extra_colors,
                       const float* dL_dout_extra, float* dL_dextra, const gsr_grads* grads, void* stream) {
    NvtxRange nvtx_("gsr_backward_multi");
    return gsr::backward_impl(frame, ws, radii, out_alpha, dL_dout_color, dL_dout_depth, dL_dout_alpha, extra_colors, dL_dout_extra,
                              dL_dextra, grads, false, nullptr, 0, (cudaStream_t)stream);
}

size_t gsr_backward_det_bytes(size_t num_rendered, int32_t W, int32_t H, int with_extra) {
    return gsr::backward_det_bytes(num_rendered, W, H, with_extra != 0);
}

int gsr_backward_det(const gsr_frame* frame, const gsr_workspace* ws, const int32_t* radii, const float* out_alpha,
                     const float* dL_dout_color, const float* dL_dout_depth, const float* dL_dout_alpha, const float* extra_colors,
                     const float* dL_dout_extra, float* dL_dextra, const gsr_grads* grads, void* scratch, size_t scratch_bytes,
                     void* stream) {
    NvtxRange nvtx_("gsr_backward_det");
    return gsr::backward_impl(frame, ws, radii, out_alpha, dL_dout_color, dL_dout_depth, dL_dout_alpha, extra_colors, dL_dout_extra,
                              dL_dextra, grads, true, scratch, scratch_bytes, (cudaStream_t)stream);
}

int gsr_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix, uint8_t* present,
                     void* stream) {
    (void)projmatrix;
    if (P < 0 || (P > 0 && (!means3D || !viewmatrix || !present))) { gsr::set_error("gsr_mark_visible: bad arguments"); return GSR_ERR_INVALID; }
    if (P == 0) return GSR_OK;
    gsr::k_mark_visible<<<(P + 255) / 256, 256, 0, (cudaStream_t)stream>>>(P, means3D, viewmatrix, present);
    return gsr::check_launch("gsr_mark_visible", false, (cudaStream_t)stream);
}

size_t gsr_dist2_bytes(int32_t P) { return gsr::dist2_bytes(P); }
int gsr_dist2(int32_t P, const float* points, float* mean_dists, void* workspace, size_t workspace_bytes, void* stream) {
    NvtxRange nvtx_("gsr_dist2");
    return gsr::dist2_impl(P, points, mean_dists, workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t gsr_knn_bytes(int32_t P1, int32_t P2, int32_t K) {
    (void)K;  // the workspace does not depend on K
    return gsr::knn_bytes(P1, P2);
}
int gsr_knn(int32_t P1, int32_t P2, int32_t K, const float* queries, const float* points, float* out_dists, int64_t* out_idx,
            void* workspace, size_t workspace_bytes, void* stream) {
    NvtxRange nvtx_("gsr_knn");
    return gsr::knn_impl(P1, P2, K, queries, points, out_dists, out_idx, workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t gsr_sugar_field_bytes(int32_t P) { return gsr::sugar_field_bytes(P); }
int gsr_sugar_field(int32_t N, int32_t K, int32_t P, int32_t R, const float* x, const int64_t* rows, const int64_t* row_idx,
                    const float* points, const float* scaling, const float* quaternions, const float* strengths, float density_factor,
                    float opacity_min_clamp, float sdf_offset, float* out_density, float* out_opacities, float* out_beta, float* out_sdf,
                    void* workspace, size_t workspace_bytes, void* stream) {
    NvtxRange nvtx_("gsr_sugar_field");
    return gsr::sugar_field_impl(N, K, P, R, x, rows, row_idx, points, scaling, quaternions, strengths, density_factor, opacity_min_clamp,
                                 sdf_offset, out_density, out_opacities, out_beta, out_sdf, workspace, workspace_bytes, (cudaStream_t)stream);
}
int gsr_sugar_field_backward(int32_t N, int32_t K, int32_t P, int32_t R, const float* x, const int64_t* rows, const int64_t* row_idx,
                             const float* points, const float* scaling, const float* quaternions, const float* strengths,
                             float density_factor, float opacity_min_clamp, float sdf_offset, const float* dL_ddensity,
                             const float* dL_dopacities, const float* dL_dbeta, const float* dL_dsdf, float* dL_dx, float* dL_dpoints,
                             float* dL_dscaling, float* dL_dquaternions, float* dL_dstrengths, void* workspace, size_t workspace_bytes,
                             void* stream) {
    NvtxRange nvtx_("gsr_sugar_field_backward");
    return gsr::sugar_field_backward_impl(N, K, P, R, x, rows, row_idx, points, scaling, quaternions, strengths, density_factor,
                                          opacity_min_clamp, sdf_offset, dL_ddensity, dL_dopacities, dL_dbeta, dL_dsdf, dL_dx, dL_dpoints,
                                          dL_dscaling, dL_dquaternions, dL_dstrengths, workspace, workspace_bytes, false, (cudaStream_t)stream);
}

size_t gsr_sugar_field_backward_det_bytes(int32_t N, int32_t K, int32_t P) { return gsr::sugar_field_backward_det_bytes(N, K, P); }
int gsr_sugar_field_backward_det(int32_t N, int32_t K, int32_t P, int32_t R, const float* x, const int64_t* rows, const int64_t* row_idx,
                                 const float* points, const float* scaling, const float* quaternions, const float* strengths,
                                 float density_factor, float opacity_min_clamp, float sdf_offset, const float* dL_ddensity,
                                 const float* dL_dopacities, const float* dL_dbeta, const float* dL_dsdf, float* dL_dx, float* dL_dpoints,
                                 float* dL_dscaling, float* dL_dquaternions, float* dL_dstrengths, void* scratch, size_t scratch_bytes,
                                 void* stream) {
    NvtxRange nvtx_("gsr_sugar_field_backward_det");
    return gsr::sugar_field_backward_impl(N, K, P, R, x, rows, row_idx, points, scaling, quaternions, strengths, density_factor,
                                          opacity_min_clamp, sdf_offset, dL_ddensity, dL_dopacities, dL_dbeta, dL_dsdf, dL_dx, dL_dpoints,
                                          dL_dscaling, dL_dquaternions, dL_dstrengths, scratch, scratch_bytes, true, (cudaStream_t)stream);
}

size_t gsr_sugar_sdf_normal_bytes(int32_t P) { return gsr::sugar_sdf_normal_bytes(P); }
int gsr_sugar_sdf_normal(int32_t N, int32_t K, int32_t P, const float* x, const int64_t* gidx, const int64_t* knn_idx,
                         const float* points, const float* scaling, const float* quaternions, const float* opacities, float* out_loss,
                         float* out_estimate, void* workspace, size_t workspace_bytes, void* stream) {
    NvtxRange nvtx_("gsr_sugar_sdf_normal");
    return gsr::sugar_sdf_normal_impl(N, K, P, x, gidx, knn_idx, points, scaling, quaternions, opacities, out_loss, out_estimate,
                                      workspace, workspace_bytes, (cudaStream_t)stream);
}
int gsr_sugar_sdf_normal_backward(int32_t N, int32_t K, int32_t P, const float* x, const int64_t* gidx, const int64_t* knn_idx,
                                  const float* points, const float* scaling, const float* quaternions, const float* opacities,
                                  const float* dL_dloss, const float* dL_destimate, float* dL_dx, float* dL_dpoints,
                                  float* dL_dquaternions, void* workspace, size_t workspace_bytes, void* stream) {
    NvtxRange nvtx_("gsr_sugar_sdf_normal_backward");
    return gsr::sugar_sdf_normal_backward_impl(N, K, P, x, gidx, knn_idx, points, scaling, quaternions, opacities, dL_dloss, dL_destimate,
                                               dL_dx, dL_dpoints, dL_dquaternions, workspace, workspace_bytes, false, (cudaStream_t)stream);
}

size_t gsr_sugar_sdf_normal_backward_det_bytes(int32_t N, int32_t K, int32_t P, int with_loss) {
    return gsr::sugar_sdf_normal_backward_det_bytes(N, K, P, with_loss != 0);
}
int gsr_sugar_sdf_normal_backward_det(int32_t N, int32_t K, int32_t P, const float* x, const int64_t* gidx, const int64_t* knn_idx,
                                      const float* points, const float* scaling, const float* quaternions, const float* opacities,
                                      const float* dL_dloss, const float* dL_destimate, float* dL_dx, float* dL_dpoints,
                                      float* dL_dquaternions, void* scratch, size_t scratch_bytes, void* stream) {
    NvtxRange nvtx_("gsr_sugar_sdf_normal_backward_det");
    return gsr::sugar_sdf_normal_backward_impl(N, K, P, x, gidx, knn_idx, points, scaling, quaternions, opacities, dL_dloss, dL_destimate,
                                               dL_dx, dL_dpoints, dL_dquaternions, scratch, scratch_bytes, true, (cudaStream_t)stream);
}

int gsr_densify_stats(int32_t P, int32_t C, const float* grad, const uint8_t* mask, const int32_t* radii, float* accum, float* denom,
                      float* max_radii2D, void* stream) {
    NvtxRange nvtx_("gsr_densify_stats");
    return gsr::densify_stats_impl(P, C, grad, mask, radii, accum, denom, max_radii2D, (cudaStream_t)stream);
}
size_t gsr_densify_plan_bytes(int32_t P) { return gsr::densify_plan_bytes(P); }
int gsr_densify_plan(int32_t P, const float* accum, const float* denom, const float* scaling, const float* opacity, float max_grad,
                     float dense_thr, float min_opacity, int32_t use_screen, float max_screen_size, float big_thr, int32_t* dst,
                     int32_t* totals, void* workspace, size_t workspace_bytes, void* stream) {
    NvtxRange nvtx_("gsr_densify_plan");
    return gsr::densify_plan_impl(P, accum, denom, scaling, opacity, max_grad, dense_thr, min_opacity, use_screen, max_screen_size,
                                  big_thr, dst, totals, workspace, workspace_bytes, (cudaStream_t)stream);
}
int gsr_densify_apply(int32_t P, int32_t S, int32_t n_groups, const gsr_densify_group* groups, const int32_t* dst, const float* xyz,
                      const float* scaling, const float* rotation, const float* eps, int32_t rotation_mode, void* stream) {
    NvtxRange nvtx_("gsr_densify_apply");
    return gsr::densify_apply_impl(P, S, n_groups, groups, dst, xyz, scaling, rotation, eps, rotation_mode, (cudaStream_t)stream);
}

size_t gsr_sugar_sample_bytes(int32_t P) { return gsr::sugar_sample_bytes(P); }
int gsr_sugar_sample(int32_t N, int32_t P, float sampling_scale_factor, int32_t proportional_to_volume, const uint8_t* mask,
                     const float* strengths, const double* u, const float* z, const float* points, const float* scaling,
                     const float* quaternions, float* out_samples, int64_t* out_idx, double* out_total, void* workspace,
                     size_t workspace_bytes, void* stream) {
    NvtxRange nvtx_("gsr_sugar_sample");
    return gsr::sugar_sample_impl(N, P, sampling_scale_factor, proportional_to_volume, mask, strengths, u, z, points, scaling, quaternions,
                                  out_samples, out_idx, out_total, workspace, workspace_bytes, (cudaStream_t)stream);
}
int gsr_sugar_sample_backward(int32_t N, int32_t P, float sampling_scale_factor, const int64_t* idx, const float* z, const float* scaling,
                              const float* quaternions, const double* total, const float* dL_dsamples, float* dL_dpoints,
                              float* dL_dscaling, float* dL_dquaternions, void* stream) {
    NvtxRange nvtx_("gsr_sugar_sample_backward");
    return gsr::sugar_sample_backward_impl(N, P, sampling_scale_factor, idx, z, scaling, quaternions, total, dL_dsamples, dL_dpoints,
                                           dL_dscaling, dL_dquaternions, false, nullptr, 0, (cudaStream_t)stream);
}

size_t gsr_sugar_sample_backward_det_bytes(int32_t N, int32_t P) { return gsr::sugar_sample_backward_det_bytes(N, P); }
int gsr_sugar_sample_backward_det(int32_t N, int32_t P, float sampling_scale_factor, const int64_t* idx, const float* z,
                                  const float* scaling, const float* quaternions, const double* total, const float* dL_dsamples,
                                  float* dL_dpoints, float* dL_dscaling, float* dL_dquaternions, void* scratch, size_t scratch_bytes,
                                  void* stream) {
    NvtxRange nvtx_("gsr_sugar_sample_backward_det");
    return gsr::sugar_sample_backward_impl(N, P, sampling_scale_factor, idx, z, scaling, quaternions, total, dL_dsamples, dL_dpoints,
                                           dL_dscaling, dL_dquaternions, true, scratch, scratch_bytes, (cudaStream_t)stream);
}

int gsr_adam_step(int32_t n, const gsr_adam_tensor* tensors, void* stream) {
    NvtxRange nvtx_("gsr_adam_step");
    return gsr::adam_step_impl(n, tensors, (cudaStream_t)stream);
}

size_t gsr_photometric_loss_bytes(int32_t B, int32_t C, int32_t H, int32_t W, int32_t for_backward) {
    return gsr::photometric_loss_bytes(B, C, H, W, for_backward);
}

int gsr_photometric_loss(int32_t B, int32_t C, int32_t H, int32_t W, const float* x, const int64_t* x_strides, const float* y,
                         const int64_t* y_strides, const float* window, int32_t for_backward, float* out_l1, float* out_ssim,
                         void* workspace, size_t workspace_bytes, void* stream) {
    NvtxRange nvtx_("gsr_photometric_loss");
    return gsr::photometric_loss_impl(B, C, H, W, x, x_strides, y, y_strides, window, for_backward, out_l1, out_ssim, workspace,
                                      workspace_bytes,
                                      (cudaStream_t)stream);
}

int gsr_photometric_loss_backward(int32_t B, int32_t C, int32_t H, int32_t W, const float* x, const int64_t* x_strides, const float* y,
                                  const int64_t* y_strides, const float* window, const float* g_l1, const float* g_ssim, float* dx,
                                  const void* workspace, size_t workspace_bytes, void* stream) {
    NvtxRange nvtx_("gsr_photometric_loss_backward");
    return gsr::photometric_loss_backward_impl(B, C, H, W, x, x_strides, y, y_strides, window, g_l1, g_ssim, dx, workspace,
                                               workspace_bytes, (cudaStream_t)stream);
}

int gsr_normal_loss(int64_t n, const float* pred, const int64_t* pred_strides, const float* gt, const int64_t* gt_strides,
                    const float* depth, int64_t depth_stride, float scene_scale, float* out, void* workspace, size_t workspace_bytes,
                    void* stream) {
    NvtxRange nvtx_("gsr_normal_loss");
    return gsr::normal_loss_impl(n, pred, pred_strides, gt, gt_strides, depth, depth_stride, scene_scale, out, workspace,
                                 workspace_bytes, (cudaStream_t)stream);
}

int gsr_normal_loss_backward(int64_t n, const float* pred, const int64_t* pred_strides, const float* gt, const int64_t* gt_strides,
                             const float* depth, int64_t depth_stride, float scene_scale, const float* g_out, float* d_pred,
                             const void* workspace, size_t workspace_bytes, void* stream) {
    NvtxRange nvtx_("gsr_normal_loss_backward");
    return gsr::normal_loss_backward_impl(n, pred, pred_strides, gt, gt_strides, depth, depth_stride, scene_scale, g_out, d_pred,
                                          workspace, workspace_bytes, (cudaStream_t)stream);
}

int gsr_anisotropic_loss(int64_t P, const float* scales, float r, float* out, void* workspace, size_t workspace_bytes, void* stream) {
    NvtxRange nvtx_("gsr_anisotropic_loss");
    return gsr::anisotropic_loss_impl(P, scales, r, out, workspace, workspace_bytes, (cudaStream_t)stream);
}

int gsr_anisotropic_loss_backward(int64_t P, const float* scales, float r, const float* g_out, float* d_scales, void* stream) {
    NvtxRange nvtx_("gsr_anisotropic_loss_backward");
    return gsr::anisotropic_loss_backward_impl(P, scales, r, g_out, d_scales, (cudaStream_t)stream);
}

int gsr_percentile_low(int64_t n, const float* x, float* out, void* workspace, size_t workspace_bytes, void* stream) {
    NvtxRange nvtx_("gsr_percentile_low");
    return gsr::percentile_low_impl(n, x, out, workspace, workspace_bytes, (cudaStream_t)stream);
}

int gsr_composite(int32_t W, int32_t H, const uint8_t* frame, const uint8_t* obj, const float* obj_depth, const uint8_t* shadow,
                  const float* shadow_depth, const uint8_t* all, const uint8_t* obj3dgs, const float* obj3dgs_depth, const uint8_t* smoke,
                  const float* smoke_depth, const float* smoke_pct, const uint8_t* fire, uint8_t* out, void* stream) {
    NvtxRange nvtx_("gsr_composite");
    return gsr::composite_impl(W, H, frame, obj, obj_depth, shadow, shadow_depth, all, obj3dgs, obj3dgs_depth, smoke, smoke_depth, smoke_pct,
                               fire, out, (cudaStream_t)stream);
}

int gsr_profile_begin(int max_frames) { return gsr::profile_begin(max_frames, 1); }
int gsr_profile_begin_strided(int max_frames, int stride) { return gsr::profile_begin(max_frames, stride); }
int gsr_profile_end(float* ms_per_kernel, int* frames) { return gsr::profile_end(ms_per_kernel, frames); }

int gsr_set_option(const char* name, int value) {
    if (!name) { gsr::set_error("gsr_set_option: null name"); return GSR_ERR_INVALID; }
    const int rc = gsr::set_option(name, value);
    if (rc != GSR_OK) gsr::set_error("gsr_set_option: unknown option or bad value (%s = %d)", name, value);
    return rc;
}

int gsr_get_views(const gsr_workspace* ws, int32_t P, int32_t W, int32_t H, gsr_views* out) {
    if (!ws || !out) { gsr::set_error("gsr_get_views: null argument"); return GSR_ERR_INVALID; }
    const gsr::GeomLayout gl((size_t)P);
    const gsr::ImageLayout il(W, H);
    const gsr::BinLayout bl(gsr::BinLayout::capacity_of(ws->binning_bytes));
    const char* geo = (const char*)ws->geom; const char* img = (const char*)ws->image; const char* bin = (const char*)ws->binning;
    out->records = (const float*)(geo + gl.records);
    out->cov3D = (const float*)(geo + gl.cov3D);
    out->clamped = (const uint8_t*)(geo + gl.clamped);
    out->point_list = (const uint32_t*)(bin + bl.point_list);
    out->sorted_keys = (const uint64_t*)(bin + bl.pairs);
    out->ranges = (const uint32_t*)(img + il.ranges);
    out->n_contrib = (const uint32_t*)(img + il.n_contrib);
    out->tile_count = (const uint32_t*)(img + il.tile_count);
    out->tile_big = (const uint32_t*)(img + il.tile_big);
    out->counters = (const gsr_counters*)(img + il.counters);
    return GSR_OK;
}

}  // extern "C"
