/* gsr_b200 — C ABI of the H100-native 3D-Gaussian-splatting rasterizer hot path.
 *
 * This is the drop-in boundary for the reference's native entry points ("DGR/" =
 * sugar/gaussian_splatting/submodules/diff-gaussian-rasterization, "KNN/" = .../simple-knn of
 * haoyuhsu/autovfx):
 *
 *   gsr_forward       replaces  _C.rasterize_gaussians           DGR/rasterize_points.cu:35-119
 *                               (CudaRasterizer::Rasterizer::forward, DGR/cuda_rasterizer/rasterizer_impl.cu:197-339)
 *   gsr_backward      replaces  _C.rasterize_gaussians_backward  DGR/rasterize_points.cu:121-209
 *                               (Rasterizer::backward, rasterizer_impl.cu:343-446)
 *   gsr_mark_visible  replaces  _C.mark_visible                  DGR/rasterize_points.cu:211-230
 *   gsr_dist2         replaces  simple_knn._C.distCUDA2          KNN/spatial.cu:15-26 (SimpleKNN::knn, KNN/simple_knn.cu:185-220)
 *   gsr_knn           replaces  pytorch3d.ops.knn_points in SuGaR  sugar_scene/sugar_model.py:47, :233, :899, :914, :1213 (N = 1, D = 3)
 *   gsr_sugar_field   replaces  SuGaR.get_field_values / compute_density  sugar_scene/sugar_model.py:1118-1187, :1216-1239
 *                               (get_covariance :602-608, get_beta 'average' :1063-1066); gsr_sugar_field_backward their autograd
 *   gsr_sugar_sdf_normal replaces the coarse trainers' better-normal loss and projection estimate
 *                               sugar_trainers/coarse_density.py:704-707, :756-780; gsr_sugar_sdf_normal_backward their autograd
 *   gsr_densify_stats, gsr_densify_plan, gsr_densify_apply replace the densification bookkeeping of GaussianModel
 *                               (scene/gaussian_model.py:268-417) and SuGaRDensifier (sugar_scene/sugar_densifier.py:48-246)
 *   gsr_sugar_sample  replaces  SuGaR.sample_points_in_gaussians               sugar_scene/sugar_model.py:757-799;
 *                               gsr_sugar_sample_backward its autograd backward
 *   gsr_sugar_surface_mask replaces coarse_sdf's close-to-surface mask           sugar_trainers/coarse_sdf.py:655-665
 *   gsr_sugar_depth_sdf_loss replaces coarse_sdf's depth-map 'sdf' estimation loss  coarse_sdf.py:689-712 (get_points_depth_in_depth_map
 *                               sugar_model.py:1189-1204); gsr_sugar_depth_sdf_loss_backward its autograd backward
 *   gsr_adam_step     replaces  torch.optim.Adam.step() (foreach) of every trainer  GS/train.py:183-184, scene_representation.py:538-540,
 *                               sugar_trainers/coarse_density.py:822
 *   gsr_photometric_loss replaces l1_loss and ssim of every trainer's objective  GS/utils/loss_utils.py:17-18, :33-62 (train.py:98-99,
 *                               coarse_density.py:550-590, scene_representation.py:513-515); gsr_photometric_loss_backward their autograd
 *   gsr_normal_loss   replaces  normal_loss                                       GS/utils/loss_utils.py:118-132; gsr_normal_loss_backward
 *   gsr_anisotropic_loss replaces anisotropic_loss                                GS/utils/loss_utils.py:159-168; gsr_anisotropic_loss_backward
 *   gsr_depth_loss    replaces  depth_loss (compute_scale_and_shift)              GS/utils/loss_utils.py:65-111; gsr_depth_loss_backward
 *   gsr_opacity_loss, gsr_sparsity_loss replace opacity_loss, sparsity_loss      GS/utils/loss_utils.py:143-157; their _backward
 *   gsr_entropy_loss  replaces  the coarse trainers' opacity entropy term          sugar_trainers/coarse_density.py:598-606; its _backward
 *   gsr_density_estimation_loss replaces coarse_density's 'density' SDF estimation loss  coarse_density.py:735-741; its _backward
 *   gsr_percentile_low replaces np.percentile(smoke_depth, 0.001)                blender/blend_all.py:206-208
 *   gsr_composite     replaces  the per-frame compositing of blend_frames          blender/blend_all.py:236-342
 *   gsr_select_rows   replaces  the deepcopy + boolean indexing of each candidate subset  extract/extract_object.py:196-202, :315-321
 *   gsr_pack_masks, gsr_mask_disagreement replace the host readback and numpy XOR count of each tracked view  :215-221, :334-340
 *   gsr_png_encode    replaces  save_image / cv2.imwrite of the frame loop's PNGs     scene_representation.py:424-438; blend_all's frames
 *
 * and, for the render() wrapper around the two rasterizer passes ("GR/" = sugar/gaussian_splatting/gaussian_renderer/__init__.py):
 *
 *   gsr_forward_multi replaces  both rasterizer(...) calls of one frame           GR/:134-166 (same geometry, second colour set)
 *   gsr_backward_multi replaces both rasterizer backward passes of that frame (training with a loss on the normal image)
 *   gsr_axis_normals  replaces  pc.get_normal(dir_pp_normalized) * 0.5 + 0.5      GR/:131-132,146-147; scene/gaussian_model.py:120-128
 *   gsr_normal_maps   replaces  normal normalisation + depth pseudo normal        GR/:168-191 (depth_pcd2normal GR/:23-38)
 *   gsr_pack_frame    replaces  the per-frame 8-bit conversions before encoding   scene_representation.py:424-438, sugar/render.py:18-22
 *   gsr_activate_gaussians replaces the activations of every render call and the per-frame object edit
 *                               get_scaling/get_rotation/get_opacity/get_features   sugar/gaussian_splatting/scene/gaussian_model.py:95-115
 *                               transform_gaussians + merge_two_gaussians            gaussians_utils.py:71-125, scene_representation.py:357-371
 *   gsr_activate_gaussians_backward replaces the autograd backward of those activations and of get_normal * 0.5 + 0.5
 *   gsr_sugar_normals replaces  SuGaR's shading normal * 0.5 + 0.5               sugar_scene/sugar_model.py:2164-2168 (get_smallest_axis :801-815)
 *   gsr_sugar_normals_backward replaces its autograd backward (gradient with respect to the raw quaternions)
 *   gsr_sugar_colors  replaces  SuGaR.get_points_rgb (eval_sh, degrees 0-4) and   sugar_model.py:711-755, :394-398
 *                               SuGaR.strengths = sigmoid(all_densities)           (sugar_utils/spherical_harmonics.py:117-172)
 *   gsr_sugar_colors_backward replaces their autograd backward
 *
 * Conventions (same as the reference's C++ layer):
 *   - every pointer is a DEVICE pointer to contiguous fp32 / int32 data unless it says "host";
 *   - a NULL pointer means "input absent" (the reference encodes None as an empty tensor whose
 *     data_ptr is null, DGR/diff_gaussian_rasterization/__init__.py:200-210);
 *   - no torch types; the caller owns every buffer, the library never allocates device memory;
 *   - `stream` is a cudaStream_t (the reference uses the legacy default stream; pass 0 for that);
 *   - functions return GSR_OK or a negative error code, gsr_last_error() gives the message;
 *     CUDA errors are only checked synchronously when frame->debug != 0 (reference: CHECK_CUDA,
 *     DGR/cuda_rasterizer/auxiliary.h:166-173).
 */
#ifndef GSR_B200_H_INCLUDED
#define GSR_B200_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSR_ABI_VERSION 4

enum {
    GSR_OK = 0,
    GSR_ERR_INVALID = -1,   /* bad argument combination / sizes                                   */
    GSR_ERR_WORKSPACE = -2, /* a workspace is smaller than the gsr_*_bytes() query                 */
    GSR_ERR_CUDA = -3,      /* CUDA runtime error (launch failure, or any error when debug is set) */
};

/* gsr_forward flags */
enum {
    GSR_FLAG_FOR_BACKWARD = 1, /* also keep cov3D, SH clamp flags and n_contrib for gsr_backward   */
    GSR_FLAG_SORTED_KEYS = 2,  /* also write the sorted 64-bit (tile<<32 | depth bits) keys (parity/debug) */
    GSR_FLAG_TIGHT_TILES = 4,  /* opt-in: emit a (Gaussian, tile) instance only if the splat can reach alpha >= 1/255 at a
                                  pixel of the tile; per-tile lists become a sub-sequence of the reference's, num_rendered and
                                  n_contrib shrink accordingly, color/depth/alpha/radii and all gradients are unchanged */
    GSR_FLAG_REUSE_GEOMETRY = 8, /* second pass of a frame: the workspaces still hold the projection + binning of the previous
                                  gsr_forward on the SAME geometry / camera / image size; only colors_precomp is re-read and the
                                  blend re-run.  `radii` must point to the radii written by that previous call (input). */
    GSR_FLAG_EXACT_IMAGES = 16, /* blend with the reference's own fp32 instruction sequence (expf, separate opacity multiply):
                                  color / depth / alpha are bit-identical to the reference's CUDA.  Default (flag clear): alpha =
                                  ex2.approx(power * log2e + log2(opacity)); every skip / termination decision that falls inside
                                  the approximation's error band is detected and that warp's pixels are re-blended exactly, so
                                  the images differ from the exact ones by ~1e-6 relative (requirement: 1e-4 max abs) and
                                  n_contrib / all integer outputs are unchanged. */
    GSR_FLAG_BINNING_ONLY = 32, /* first half of a frame issued in two calls: projection + tile scan only.  Afterwards the counters
                                  (num_rendered, overflow, max_tile, trapped, num_visible) are final, so a caller that validates the
                                  binning capacity on the host (the reference blocks on the same number, rasterizer_impl.cu:281-282)
                                  can start that copy now and let it overlap the rest of the frame. */
    GSR_FLAG_RESUME = 64,       /* second half: same arguments and workspaces as the GSR_FLAG_BINNING_ONLY call; runs colour +
                                  emission, the tile sort and the blend. */
};
/* Slab emission: flags | ((S / 32) << GSR_SLAB_SHIFT) gives every tile a slab of S sort pairs (S a multiple of 32, 0 = off), so
 * the projection writes each (Gaussian, tile) pair the moment it draws the tile's ticket, and the separate emission pass and its
 * per-Gaussian ranks go away.  The slab takes tiles * S instances at the end of the binning workspace's pair region: size the
 * workspace with gsr_binning_bytes_slab().  A tile with more than S instances sets gsr_counters.overflow (max_tile says how many
 * it had), like a capacity overflow.  Outputs are identical with and without a slab; it is ignored when P > 2^24 and with GSR_FLAG_TIGHT_TILES. */
#define GSR_SLAB_SHIFT 16

/* One rasterizer invocation = the argument list of Rasterizer::forward (DGR/cuda_rasterizer/rasterizer.h:33-58). */
typedef struct gsr_frame {
    int32_t P;              /* number of Gaussians                                                 */
    int32_t D;              /* active SH degree (0..3; larger values are treated as 3, forward.cu:29-59) */
    int32_t M;              /* SH coefficients per channel in `shs` (stride), 0 if shs == NULL      */
    int32_t W, H;           /* image width / height                                               */
    float scale_modifier;
    float tanfovx, tanfovy;
    int32_t prefiltered;    /* !=0: a near-culled point is an error (reference __trap()s, auxiliary.h:156-160) */
    int32_t debug;          /* !=0: synchronise and check for CUDA errors after the call          */
    const float* bg;            /* [3]                                                            */
    const float* means3D;       /* [P,3]                                                          */
    const float* shs;           /* [P,M,3] coefficient-major, or NULL                             */
    const float* colors_precomp;/* [P,3] or NULL  (exactly one of shs / colors_precomp)            */
    const float* opacities;     /* [P]                                                            */
    const float* scales;        /* [P,3] or NULL                                                  */
    const float* rotations;     /* [P,4] (r,x,y,z), NOT normalised here, or NULL                  */
    const float* cov3D_precomp; /* [P,6] or NULL  (exactly one of scales+rotations / cov3D_precomp) */
    const float* viewmatrix;    /* [16] row-major torch buffer of the transposed W2C              */
    const float* projmatrix;    /* [16] view @ proj                                               */
    const float* campos;        /* [3]                                                            */
} gsr_frame;

/* Opaque workspaces, the analogue of the reference's geomBuffer / binningBuffer / imgBuffer
 * (rasterizer_impl.h:30-63).  They must stay untouched between gsr_forward and the matching
 * gsr_backward.  `binning` is sized by a CAPACITY in splat instances, not by the exact count: the
 * pipeline never reads the instance count back to the host (the reference's blocking cudaMemcpy,
 * rasterizer_impl.cu:281-282).  If the frame produces more instances than the capacity the frame is
 * incomplete, gsr_counters.overflow is set, and the caller re-runs with a larger binning workspace. */
typedef struct gsr_workspace {
    void* geom;    size_t geom_bytes;    /* >= gsr_geom_bytes(P)                                   */
    void* binning; size_t binning_bytes; /* >= gsr_binning_bytes(capacity), capacity >= 1          */
    void* image;   size_t image_bytes;   /* >= gsr_image_bytes(W, H)                               */
} gsr_workspace;

/* First bytes of the image workspace; copy them to the host (async) to learn the frame's statistics. */
typedef struct gsr_counters {
    uint32_t num_rendered; /* R = sum over Gaussians of tiles touched (what the reference returns)  */
    uint32_t overflow;     /* 1 if R > binning capacity: outputs are incomplete                    */
    uint32_t max_tile;     /* longest per-tile list                                               */
    uint32_t trapped;      /* 1 if prefiltered was set and a point was near-culled                 */
    uint32_t num_visible;  /* Gaussians with radii > 0                                             */
    uint32_t foot_total;   /* reserved (0)                                                          */
    uint32_t exact_redos;  /* warps whose pixels were re-blended exactly (default image mode)       */
    uint32_t reserved;     /* reserved (0)                                                          */
} gsr_counters;

size_t gsr_geom_bytes(int32_t P);
/* 13 bytes per instance of capacity (8-byte sort pair, 4-byte list entry, 1 byte of the footprint ballot matrix) + a fixed 4 MiB of
 * ballot rows (one 32-byte row per 32 list entries and one extra per tile: enough for 131,072 tiles; an image with more tiles needs
 * capacity >= 32 * (tiles - 131072)). */
size_t gsr_binning_bytes(size_t capacity_instances);
size_t gsr_image_bytes(int32_t W, int32_t H);
/* Largest capacity (in instances) a binning workspace of `bytes` bytes provides. */
size_t gsr_binning_capacity(size_t bytes);
/* The same two queries for a forward with slab stride S (GSR_SLAB_SHIFT) on a W x H image: the workspace holds `capacity`
 * instances besides the slab.  S = 0 gives gsr_binning_bytes / gsr_binning_capacity; 0 from the second means the slab does not fit. */
size_t gsr_binning_bytes_slab(size_t capacity_instances, int32_t W, int32_t H, int32_t slab_stride);
size_t gsr_binning_capacity_slab(size_t bytes, int32_t W, int32_t H, int32_t slab_stride);

/* Forward: projection (+ per-tile histogram) -> tile scan -> colour + key emission (+ footprint masks) -> per-tile depth sort
 * (+ footprint ballot matrix) -> blend (one warp per 8x4-pixel footprint).
 * Outputs: out_color [3,H,W], out_depth [1,H,W], out_alpha [1,H,W], radii [P] (int32).
 * All four are fully written (no pre-zeroing needed).  With P == 0 the images are zero-filled
 * (reference: rasterize_points.cu:68-71,82).  Asynchronous on `stream`. */
int gsr_forward(const gsr_frame* frame, const gsr_workspace* ws, float* out_color, float* out_depth,
                float* out_alpha, int32_t* radii, int flags, void* stream);

/* gsr_forward plus a second colour set blended with the SAME per-pixel weights: out_extra [3,H,W] is what a second
 * gsr_forward with colors_precomp = extra_colors ([P,3]) would write to out_color (bit for bit), at the cost of three
 * more accumulators in the blend instead of a second pass.  extra_colors == NULL && out_extra == NULL is gsr_forward.
 * With GSR_FLAG_REUSE_GEOMETRY, colors_precomp recolours the cached records and extra_colors is blended alongside. */
int gsr_forward_multi(const gsr_frame* frame, const gsr_workspace* ws, float* out_color, float* out_depth, float* out_alpha,
                      int32_t* radii, const float* extra_colors, float* out_extra, int flags, void* stream);

/* Per-Gaussian shading normal of the reference's GaussianModel.get_normal: the rotation-matrix column of the smallest
 * scale (ties: lowest index), flipped so that it faces the camera, normalised; remap01 != 0 stores normal*0.5+0.5.
 * out [P,3]. */
int gsr_axis_normals(int32_t P, const float* means3D, const float* scales, const float* rotations, const float* campos,
                     int remap01, float* out, void* stream);

/* SuGaR's per-Gaussian shading normal (SuGaR.render_image_gaussian_rasterizer): column k = argmin(scales) (ties: lowest
 * index) of quaternion_to_matrix(q) for the RAW quaternion q (2 / |q|^2, no normalisation), flipped so that
 * dot(axis, -normalize(position - campos)) >= 0, divided by its norm (no epsilon); out [P,3] = normal * 0.5 + 0.5.
 * positions [P,3], scales [P,3], quaternions [P,4] (real part first), campos [3].  P = 0 is a no-op. */
int gsr_sugar_normals(int32_t P, const float* positions, const float* scales, const float* quaternions, const float* campos, float* out,
                      void* stream);

/* Backward of gsr_sugar_normals: dL_dnormals [P,3] (the gradient of normal * 0.5 + 0.5) -> dL_dquaternions [P,4].  The axis and the
 * flip are the forward's decisions, recomputed from the same inputs; they are piecewise constant, so positions and scales get no
 * gradient.  Every pointer is required when P > 0. */
int gsr_sugar_normals_backward(int32_t P, const float* positions, const float* scales, const float* quaternions, const float* campos,
                               const float* dL_dnormals, float* dL_dquaternions, void* stream);

/* SuGaR's per-Gaussian colours and opacities (SuGaR.get_points_rgb with its eval_sh, degrees 0..4, and SuGaR.strengths):
 *   out_colors [P,3]  = clamp_min(eval_sh(deg, cat(sh_dc, sh_rest)[:, :(deg+1)^2], dirs) + 0.5, 0)
 *   out_opacities [P] = sigmoid(densities)
 * dirs = F.normalize(positions - campos) (1e-12 clamp) when directions == NULL, otherwise directions [P,3] as given (not
 * normalised).  sh_dc [P,1,3], sh_rest [P,M-1,3] (may be NULL when M == 1), densities [P], positions [P,3], campos [3].  One
 * IEEE rounding per torch op in the order SuGaR's Python writes them.  out_colors == NULL skips the colours (no SH, position or
 * direction is read); out_opacities == NULL skips the opacities (densities is not read).  deg outside 0..4 or
 * M < (deg+1)^2 is GSR_ERR_INVALID.  P = 0 is a no-op. */
int gsr_sugar_colors(int32_t P, int32_t M, int32_t deg, const float* positions, const float* campos, const float* directions,
                     const float* sh_dc, const float* sh_rest, const float* densities, float* out_colors, float* out_opacities, void* stream);

/* Backward of gsr_sugar_colors (same P, M, deg and inputs): dL_dcolors [P,3] and / or dL_dopacities [P] in (either may be NULL).
 * With dL_dcolors: dL_dsh_dc [P,1,3], dL_dsh_rest [P,M-1,3] (coefficients beyond the active degree get zeros) and dL_dpositions
 * [P,3] (the gradient of `directions` when directions != NULL) are written in full.  With dL_dopacities: dL_ddensities [P] =
 * g * o (1 - o).  The clamp decisions (gradient where the pre-clamp colour is >= 0) and the normalisation branch (below 1e-12
 * the denominator is the constant 1e-12) are recomputed from the inputs; nothing is kept between the two calls. */
int gsr_sugar_colors_backward(int32_t P, int32_t M, int32_t deg, const float* positions, const float* campos, const float* directions,
                              const float* sh_dc, const float* sh_rest, const float* densities, const float* dL_dcolors,
                              const float* dL_dopacities, float* dL_dsh_dc, float* dL_dsh_rest, float* dL_dpositions, float* dL_ddensities,
                              void* stream);

/* normal_img [3,H,W] (a rendered normal*0.5+0.5 image) -> out_normal [H,W,3] = normalize((img - 0.5) * 2);
 * depth [H,W] -> out_pseudo [H,W,3] = normalised cross product of central differences of the unprojected depth map,
 * zero on the 1-pixel border.  c2w: DEVICE pointer to >= 12 floats, rows 0..2 of the 4x4 the reference calls c2w
 * (world_view_transform.inverse(), row-major); fx, fy, cx, cy as in GR/:180-184.  Either pair may be NULL. */
int gsr_normal_maps(int32_t W, int32_t H, const float* normal_img, const float* depth, const float* c2w, float fx, float fy,
                    float cx, float cy, float* out_normal, float* out_pseudo, void* stream);

/* 8-bit hand-off of a finished frame (any output may be NULL):
 *   rgba8   [H,W,4] = clamp(v*255+0.5, 0, 255) of rgb [3,H,W] and alpha [H,W] (alpha NULL -> 255)
 *   normal8 [H,W,3] = trunc((n+1)/2*255) of normal_hwc [H,W,3]
 *   depth8  [H,W]   = trunc(clip(depth/depth_scale, 0, 1)*255), the colormap index */
int gsr_pack_frame(int32_t W, int32_t H, const float* rgb, const float* alpha, const float* depth, const float* normal_hwc,
                   float depth_scale, uint8_t* rgba8, uint8_t* normal8, uint8_t* depth8, void* stream);

/* Rigid edit of one inserted object for one frame = the arguments of the reference's transform_gaussians(gaussians, center,
 * rotation, scaling, initial_center) (gaussians_utils.py:88-125), plus the two values its host code derives from them. */
typedef struct gsr_object_xform {
    float rotation[9];       /* R, row-major 3x3                                                       */
    float quat[4];           /* matrix_to_quaternion(R), (w,x,y,z) (rotation_utils.py:24-84)           */
    float center[3];         /* target position of the pivot                                          */
    float initial_center[3]; /* the pivot: centre of the object's mesh                                 */
    float scaling;           /* uniform scale                                                          */
    float log_scaling;       /* (float)log(scaling), added to the log-scales                           */
} gsr_object_xform;

/* RAW parameters (the reference's GaussianModel fields: _xyz [N,3], _features_dc [N,1,3], _features_rest [N,M-1,3],
 * _opacity [N], _scaling [N,3], _rotation [N,4]) -> the ACTIVATED tensors the rasterizer takes: means3D [N,3],
 * shs [N,M,3] = cat(dc, rest), opacities [N] = sigmoid, scales [N,3] = exp, rotations [N,4] = normalize.
 * xform (HOST pointer, may be NULL) applies transform_gaussians first: scale about the pivot, rotate, translate,
 * compose the quaternions, shift the log-scales.  The output pointers may address a sub-range of larger arrays
 * (the tail of a resident scene): this replaces merge_two_gaussians' concatenation.  M >= 1. */
int gsr_activate_gaussians(int32_t N, int32_t M, const float* xyz, const float* f_dc, const float* f_rest, const float* opacity_raw,
                           const float* scaling_raw, const float* rotation_raw, const gsr_object_xform* xform, float* means3D,
                           float* shs, float* opacities, float* scales, float* rotations, void* stream);

/* Backward of gsr_activate_gaussians (xform NULL) together with gsr_axis_normals(xyz, scales, rotations, campos, remap01 = 1) on
 * its outputs: gradients with respect to the activated tensors in, gradients with respect to the raw parameters out.
 * opacities / scales / rotations are the activated values, rotation_raw the raw quaternions [N,4].  dL_dopacities [N],
 * dL_dscales [N,3], dL_drotations [N,4] are required; dL_dshs [N,M,3] may be NULL (then dL_df_dc / dL_df_rest are not written),
 * dL_dnormals [N,3] (the gradient of the remapped normals) may be NULL (then xyz and campos are not read).  Outputs:
 * dL_dopacity_raw [N], dL_dscaling_raw [N,3], dL_drotation_raw [N,4], dL_df_dc [N,1,3], dL_df_rest [N,M-1,3] (unused when M == 1).
 * The smallest axis and the flip towards campos are the forward's decisions, recomputed from the same values. */
int gsr_activate_gaussians_backward(int32_t N, int32_t M, const float* xyz, const float* campos, const float* opacities,
                                    const float* scales, const float* rotations, const float* rotation_raw, const float* dL_dopacities,
                                    const float* dL_dscales, const float* dL_drotations, const float* dL_dshs, const float* dL_dnormals,
                                    float* dL_dopacity_raw, float* dL_dscaling_raw, float* dL_drotation_raw, float* dL_df_dc,
                                    float* dL_df_rest, void* stream);

/* Gradient buffers, all caller-allocated; the library zero-fills what it accumulates into (the
 * reference's torch::zeros, rasterize_points.cu:158-168).  dL_dsh may be NULL when shs is NULL,
 * dL_dscales / dL_drotations may be NULL when scales is NULL. */
typedef struct gsr_grads {
    float* dL_dmeans2D;   /* [P,3]  (x,y in NDC-scaled units, z = 0), returned to Python            */
    float* dL_dconic;     /* [P,4]  scratch (slots 0,1,3)                                          */
    float* dL_dopacity;   /* [P]                                                                   */
    float* dL_dcolors;    /* [P,3]  = grad of colors_precomp, or scratch for the SH backward        */
    float* dL_ddepths;    /* [P]    scratch                                                        */
    float* dL_dmeans3D;   /* [P,3]                                                                 */
    float* dL_dcov3D;     /* [P,6]                                                                 */
    float* dL_dsh;        /* [P,M,3] or NULL                                                       */
    float* dL_dscales;    /* [P,3] or NULL                                                         */
    float* dL_drotations; /* [P,4] or NULL                                                         */
} gsr_grads;

/* Backward of the frame last run through gsr_forward(..., GSR_FLAG_FOR_BACKWARD) on `ws`.
 * out_alpha is the forward's alpha image; dL_dout_* are the three image gradients
 * ([3,H,W], [1,H,W], [1,H,W]); radii is the forward's radii output. */
int gsr_backward(const gsr_frame* frame, const gsr_workspace* ws, const int32_t* radii, const float* out_alpha,
                 const float* dL_dout_color, const float* dL_dout_depth, const float* dL_dout_alpha,
                 const gsr_grads* grads, void* stream);

/* Backward of a frame run through gsr_forward_multi(..., GSR_FLAG_FOR_BACKWARD) with a second colour set: gsr_backward plus
 * the gradient of the second image.  extra_colors [P,3] is the forward's extra_colors, dL_dout_extra [3,H,W] the gradient of
 * its out_extra, and dL_dextra [P,3] receives dL/d(extra_colors) (zero-filled by the library).  The geometry gradients in
 * `grads` are those of the sum of both images' losses: what two gsr_backward calls of two separate passes would add up to,
 * up to summation order.  All three extra pointers NULL is gsr_backward; only some of them NULL is GSR_ERR_INVALID. */
int gsr_backward_multi(const gsr_frame* frame, const gsr_workspace* ws, const int32_t* radii, const float* out_alpha,
                       const float* dL_dout_color, const float* dL_dout_depth, const float* dL_dout_alpha,
                       const float* extra_colors, const float* dL_dout_extra, float* dL_dextra,
                       const gsr_grads* grads, void* stream);

/* Deterministic backward: the arguments of gsr_backward_multi (the three extra pointers all NULL or all given, as there) plus a
 * device scratch (16-byte aligned) of at least gsr_backward_det_bytes(num_rendered, W, H, extra_colors != NULL) bytes, where
 * num_rendered is the forward's gsr_counters.num_rendered.  Every gradient is bit-identical from call to call, whatever the CTA
 * scheduling, the concurrent streams or the blend backward's register budget: each component of dL_dmeans2D, dL_dconic,
 * dL_dopacity, dL_dcolors, dL_ddepths and dL_dextra is a sequential fp32 sum from +0.0 of the per-(footprint, splat) partials in
 * a fixed order (tiles of the Gaussian's tile rectangle row-major, then footprints 0..7; DESIGN.md §4), and the rest of the
 * backward is per Gaussian.  The values agree with gsr_backward's to rounding, not bit for bit.  The library writes every row of
 * the gradient buffers itself (no zero-fill is needed) and never reads a scratch byte it has not written in the same call.
 * A NULL or misaligned scratch is GSR_ERR_INVALID; one smaller than gsr_backward_det_bytes(0, W, H, with_extra) is
 * GSR_ERR_WORKSPACE.  Both are reported before anything is enqueued.  A scratch sized for fewer instances than the frame rendered
 * is never written beyond its end; the Gaussians whose partials did not fit get NaN gradients. */
size_t gsr_backward_det_bytes(size_t num_rendered, int32_t W, int32_t H, int with_extra);
int gsr_backward_det(const gsr_frame* frame, const gsr_workspace* ws, const int32_t* radii, const float* out_alpha,
                     const float* dL_dout_color, const float* dL_dout_depth, const float* dL_dout_alpha,
                     const float* extra_colors, const float* dL_dout_extra, float* dL_dextra,
                     const gsr_grads* grads, void* scratch, size_t scratch_bytes, void* stream);

/* present[i] = (view-space z of means3D[i] > 0.2)  — checkFrustum, rasterizer_impl.cu:54-66. */
int gsr_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                     uint8_t* present, void* stream);

/* Mean squared distance to the 3 nearest neighbours.  `workspace` needs gsr_dist2_bytes(P) bytes. */
size_t gsr_dist2_bytes(int32_t P);
int gsr_dist2(int32_t P, const float* points, float* mean_dists, void* workspace, size_t workspace_bytes,
              void* stream);

/* Exact K nearest neighbours (pytorch3d.ops.knn_points for one cloud pair in 3-D): for each of the P1 queries [P1,3], the K
 * nearest of the P2 points [P2,3], ascending, as squared distances out_dists [P1,K] and indices into points out_idx [P1,K].
 * queries == NULL: the queries are the points themselves (P1 == P2).  d = (dx*dx + dy*dy) + dz*dz, dx = point.x - query.x,
 * each operation rounded once (no FMA).  Ties in d go to the lower index; the query itself is not excluded.
 * 1 <= K <= 32 and K <= P2, otherwise GSR_ERR_INVALID.  P1 = 0 launches nothing.  `workspace` needs gsr_knn_bytes(P1, P2, K)
 * bytes (with queries == NULL, gsr_knn_bytes(0, P2, K) suffices). */
size_t gsr_knn_bytes(int32_t P1, int32_t P2, int32_t K);
int gsr_knn(int32_t P1, int32_t P2, int32_t K, const float* queries, const float* points, float* out_dists, int64_t* out_idx,
            void* workspace, size_t workspace_bytes, void* stream);

/* SuGaR's SDF-regularisation field (SuGaR.get_field_values with beta_mode 'average', SuGaR.compute_density) at N samples x [N,3]
 * over K neighbours each (1 <= K <= 32) among P Gaussians given by SuGaR's getters: points [P,3], scaling [P,3], quaternions [P,4]
 * (as the getter returns them; quaternion_to_matrix divides by |q|^2), strengths [P].  Sample n uses the Gaussians
 * rows[row_idx[n], 0..K-1] of the int64 table rows [R,K] (row_idx NULL: rows[n], R == N).  Per pair, with
 * A = quaternion_to_matrix(q) * (1 / clamp(s, 1e-8)) column-wise and w = A^T (x - centre):
 *   out_opacities [N,K] = (density_factor * strength) * exp(-0.5 * clamp((w0^2 + w1^2) + w2^2, 0, 1e8))
 *   out_density   [N]   = the sum over the K pairs
 *   out_beta      [N]   = the mean over the K pairs of the Gaussian's min scale
 *   out_sdf       [N]   = beta * (sqrt(-2 log(clamp(d_hat, opacity_min_clamp))) - sdf_offset), d_hat = d / (d + 1e-12) where
 *                         d >= 1, else d; sdf_offset = sqrt(-2 log(min(density_threshold, 1))) as float
 * Any output may be NULL (not requested).  N = 0 is a no-op.  Negative sizes, K outside 1..32, row_idx NULL with R != N, or a
 * missing input when N > 0 are GSR_ERR_INVALID; `workspace` (16-byte aligned) needs gsr_sugar_field_bytes(P) bytes for the
 * forward, twice that for the backward, else GSR_ERR_WORKSPACE.  A row or Gaussian index outside its array is never read: the
 * sample's density, beta and sdf are NaN, and so are its opacities at the pairs whose index is outside (all K for a bad row). */
size_t gsr_sugar_field_bytes(int32_t P);
int gsr_sugar_field(int32_t N, int32_t K, int32_t P, int32_t R, const float* x, const int64_t* rows, const int64_t* row_idx,
                    const float* points, const float* scaling, const float* quaternions, const float* strengths, float density_factor,
                    float opacity_min_clamp, float sdf_offset, float* out_density, float* out_opacities, float* out_beta, float* out_sdf,
                    void* workspace, size_t workspace_bytes, void* stream);

/* Backward of gsr_sugar_field (same sizes, inputs and constants; it recomputes the forward): the gradients of the four outputs in
 * (any may be NULL; dL_dsdf and dL_dbeta need no forward output), torch's backward formulas out: dL_dx [N,3] (may be NULL) and
 * dL_dpoints [P,3], dL_dscaling [P,3], dL_dquaternions [P,4], dL_dstrengths [P] (required, written in full).  Where torch's
 * gradient is not finite (d >= 1 with an sdf gradient: sqrt'(0)), this one is not either.  A sample with a row or Gaussian index
 * outside its array adds nothing to any Gaussian, through none of its K pairs; its dL_dx is NaN. */
int gsr_sugar_field_backward(int32_t N, int32_t K, int32_t P, int32_t R, const float* x, const int64_t* rows, const int64_t* row_idx,
                             const float* points, const float* scaling, const float* quaternions, const float* strengths,
                             float density_factor, float opacity_min_clamp, float sdf_offset, const float* dL_ddensity,
                             const float* dL_dopacities, const float* dL_dbeta, const float* dL_dsdf, float* dL_dx, float* dL_dpoints,
                             float* dL_dscaling, float* dL_dquaternions, float* dL_dstrengths, void* workspace, size_t workspace_bytes,
                             void* stream);

/* Deterministic backward of gsr_sugar_field: gsr_sugar_field_backward's arguments, with a device scratch (16-byte aligned) of at
 * least gsr_sugar_field_backward_det_bytes(N, K, P) bytes in place of its workspace (the scratch includes it).  Every output is
 * bit-identical from call to call, whatever the scheduling or the concurrent streams.  Pair (n, k) has the id n*K + k and goes to
 * Gaussian g = rows[row_idx[n], k]; for every g each of the 14 record gradient components (-dL/dshift, dL/d(density_factor *
 * strength), the 9 of dL/dA, dL/d(min scale)) is a sequential fp32 sum from +0.0 of g's pair partials in ascending id, and the
 * per-Gaussian chain to dL_dpoints, dL_dscaling, dL_dquaternions and dL_dstrengths follows as in gsr_sugar_field_backward (DESIGN.md
 * §4).  dL_dx is per sample, as there.  The values agree with gsr_sugar_field_backward's to rounding, not bit for bit.  The exclusion
 * rules are the same: a sample with an index outside its array adds nothing through any pair and its dL_dx is NaN.  Every row of the
 * gradients is written; no scratch byte is read before it is written in the same call.  N*K at or above 2^32, and a NULL or
 * misaligned scratch (when N > 0), are GSR_ERR_INVALID; a scratch smaller than the query is GSR_ERR_WORKSPACE.  All are reported
 * before anything is enqueued.  With A(x) = x rounded up to a multiple of 256 and G(M, P), the grouping of M ids over P Gaussians,
 *   G(M, P) = 4 A(4M) + A(1024 c) + A(4 ceil(max(256 c, P + 1) / 1024)) + A(4 (P + 1)),  c = ceil(M / 2048),
 * the query is A(128 P) + 2 A(4 N) + G(N K, P). */
size_t gsr_sugar_field_backward_det_bytes(int32_t N, int32_t K, int32_t P);
int gsr_sugar_field_backward_det(int32_t N, int32_t K, int32_t P, int32_t R, const float* x, const int64_t* rows, const int64_t* row_idx,
                                 const float* points, const float* scaling, const float* quaternions, const float* strengths,
                                 float density_factor, float opacity_min_clamp, float sdf_offset, const float* dL_ddensity,
                                 const float* dL_dopacities, const float* dL_dbeta, const float* dL_dsdf, float* dL_dx, float* dL_dpoints,
                                 float* dL_dscaling, float* dL_dquaternions, float* dL_dstrengths, void* scratch, size_t scratch_bytes,
                                 void* stream);

/* The coarse trainers' better-normal loss and projection estimate (sugar_trainers/coarse_density.py:704-707, :756-780) at N samples
 * x [N,3], each in the Gaussian gidx[n] of P given by SuGaR's getters (points [P,3], scaling [P,3], quaternions [P,4]), with the K
 * neighbours knn_idx[gidx[n], 0..K-1] of the int64 table knn_idx [P,K] (1 <= K <= 32) and their opacities [N,K].  n_g is column
 * k_g of quaternion_to_matrix(q_g), k_g the lowest index of min(s_g); with i = gidx[n], per neighbour j:
 *   sigma_j = sign(n_j . n_i), w_j = (o_nj * |(x - p_j) . sigma_j n_j|) / clamp(min s_j, 1e-6)^2, w_hat_j = w_j / clamp(sum w, 1e-6)
 *   out_loss     [N] = |n_i - sum_j w_hat_j sigma_j n_j|^2
 *   out_estimate [N] = (x - p_i) . n_i
 * Either output may be NULL (not requested); knn_idx and opacities are read only for the loss.  N = 0 is a no-op.  Negative sizes,
 * K outside 1..32 or a missing input for a requested output are GSR_ERR_INVALID; `workspace` (16-byte aligned) needs
 * gsr_sugar_sdf_normal_bytes(P) bytes for the forward, twice that for the backward, else GSR_ERR_WORKSPACE.  An index outside its
 * array is never read: the outputs that depend on it are NaN. */
size_t gsr_sugar_sdf_normal_bytes(int32_t P);
int gsr_sugar_sdf_normal(int32_t N, int32_t K, int32_t P, const float* x, const int64_t* gidx, const int64_t* knn_idx,
                         const float* points, const float* scaling, const float* quaternions, const float* opacities, float* out_loss,
                         float* out_estimate, void* workspace, size_t workspace_bytes, void* stream);

/* Backward of gsr_sugar_sdf_normal (same sizes and inputs; it recomputes the forward).  sigma, the weights, their sum, the
 * opacities and the scales are constants, as in the trainer, so the loss reaches the quaternions only; the estimate reaches x,
 * the points and the quaternions.  dL_dloss and dL_destimate may be NULL; dL_dx [N,3] may be NULL; dL_dpoints [P,3] and
 * dL_dquaternions [P,4] are required and written in full.  A sample with an index outside its array adds nothing; its dL_dx is NaN. */
int gsr_sugar_sdf_normal_backward(int32_t N, int32_t K, int32_t P, const float* x, const int64_t* gidx, const int64_t* knn_idx,
                                  const float* points, const float* scaling, const float* quaternions, const float* opacities,
                                  const float* dL_dloss, const float* dL_destimate, float* dL_dx, float* dL_dpoints,
                                  float* dL_dquaternions, void* workspace, size_t workspace_bytes, void* stream);

/* Deterministic backward of gsr_sugar_sdf_normal: gsr_sugar_sdf_normal_backward's arguments, with a device scratch (16-byte aligned)
 * of at least gsr_sugar_sdf_normal_backward_det_bytes(N, K, P, dL_dloss != NULL) bytes in place of its workspace.  With the loss,
 * sample n has K + 1 partial ids: slot k < K (id n*(K+1) + k) is the loss's neighbour term, to knn_idx[gidx[n], k]; slot K (id
 * n*(K+1) + K) is the sample's own term, to gidx[n]: its dL/dn and, with dL_destimate, -dL/dx for the centre.  Without the loss,
 * sample n has only its own slot, id n.  For every Gaussian each component of the normal and centre gradients is a sequential fp32
 * sum from +0.0 of its partials in ascending id (the centre's over own terms only, so in ascending n); the chain to
 * dL_dquaternions follows as in gsr_sugar_sdf_normal_backward.  The rules for a bad index, the full writes, the unread scratch and
 * the errors are those of gsr_sugar_field_backward_det, the id limit being N*(K+1) (with the loss).  With A and G as there, the query
 * is A(64 P) + A(16 N) + A(32 N) + G(N (K + 1), P) with the loss and A(64 P) + A(16 N) + A(32 N) + G(N, P) without. */
size_t gsr_sugar_sdf_normal_backward_det_bytes(int32_t N, int32_t K, int32_t P, int with_loss);
int gsr_sugar_sdf_normal_backward_det(int32_t N, int32_t K, int32_t P, const float* x, const int64_t* gidx, const int64_t* knn_idx,
                                      const float* points, const float* scaling, const float* quaternions, const float* opacities,
                                      const float* dL_dloss, const float* dL_destimate, float* dL_dx, float* dL_dpoints,
                                      float* dL_dquaternions, void* scratch, size_t scratch_bytes, void* stream);

/* SuGaR.sample_points_in_gaussians (sugar_model.py:757-799) given its random draws: N samples among P >= 1 Gaussians given by
 * SuGaR's getters, points [P,3], scaling [P,3], quaternions [P,4] (as the getters return them).  A row is selected where mask [P]
 * (bool bytes) is non-zero, every row when mask is NULL.  A selected row's weight is w = |s0 * s1 * s2| (float32, left to right) when
 * proportional_to_volume, else 1, times strengths [P] when strengths is not NULL (proportional to opacity).  As in SuGaR, whose
 * torch.multinomial receives cumsum(w) / sum(w) as the weights, selected row k is drawn with probability proportional to
 * C_k = sum of w over the selected rows up to k.  In float64, with T_i = sum_{j <= i, j selected} C_j and total = T_{P-1}:
 *   out_idx     [N] (int64) = the first row i whose T_i exceeds u[n] * total (capped below the total); a row of zero C or an
 *                             unselected row is never returned.  u [N] (float64) is uniform in [0, 1).
 *   out_samples [N,3]       = points[i] + quaternion_apply(quaternions[i], (sampling_scale_factor * scaling[i]) * z[n]), pytorch3d's
 *                             raw_multiply(raw_multiply(q, (0, v)), conjugate(q)) op for op in float32 (a non-unit q scales by |q|^2).
 *                             z [N,3] (float32) is standard normal.
 *   out_total   [1] (float64) = total, for the backward.
 * No host synchronisation.  When the total is zero (an empty selection), infinite or NaN, every index is 0 and every sample NaN.
 * N = 0 is a no-op.  N < 0, P < 1 or a missing pointer other than mask and strengths is GSR_ERR_INVALID; `workspace` (16-byte
 * aligned) needs gsr_sugar_sample_bytes(P) bytes, else GSR_ERR_WORKSPACE. */
size_t gsr_sugar_sample_bytes(int32_t P);
int gsr_sugar_sample(int32_t N, int32_t P, float sampling_scale_factor, int32_t proportional_to_volume, const uint8_t* mask,
                     const float* strengths, const double* u, const float* z, const float* points, const float* scaling,
                     const float* quaternions, float* out_samples, int64_t* out_idx, double* out_total, void* workspace,
                     size_t workspace_bytes, void* stream);

/* Backward of gsr_sugar_sample (same N, P, factor, z, scaling and quaternions; idx and total as it wrote them): the gradient of the
 * samples dL_dsamples [N,3] in, dL_dpoints [P,3], dL_dscaling [P,3] and dL_dquaternions [P,4] out (required, written in full;
 * gsr_sugar_sample_backward_det below sums the per-sample terms in a fixed order).  The weights get no gradient, as through
 * torch.multinomial.  When the total is zero, infinite or NaN the gradients are zero. */
int gsr_sugar_sample_backward(int32_t N, int32_t P, float sampling_scale_factor, const int64_t* idx, const float* z, const float* scaling,
                              const float* quaternions, const double* total, const float* dL_dsamples, float* dL_dpoints,
                              float* dL_dscaling, float* dL_dquaternions, void* stream);

/* Deterministic backward of gsr_sugar_sample: gsr_sugar_sample_backward's arguments plus a device scratch (16-byte aligned) of at
 * least gsr_sugar_sample_backward_det_bytes(N, P) = G(N, P) bytes (G as for gsr_sugar_field_backward_det).  Sample n (id n) goes to
 * Gaussian idx[n]; for every Gaussian each of its 10 gradient components is a sequential fp32 sum from +0.0 of its samples' terms in
 * ascending n.  A sample whose index is outside [0, P), or every sample when the total is zero or not finite, adds nothing; every
 * row is written (+0.0 where no sample adds).  A NULL or misaligned scratch (when N > 0) is GSR_ERR_INVALID, a smaller one
 * GSR_ERR_WORKSPACE, both before anything is enqueued. */
size_t gsr_sugar_sample_backward_det_bytes(int32_t N, int32_t P);
int gsr_sugar_sample_backward_det(int32_t N, int32_t P, float sampling_scale_factor, const int64_t* idx, const float* z,
                                  const float* scaling, const float* quaternions, const double* total, const float* dL_dsamples,
                                  float* dL_dpoints, float* dL_dscaling, float* dL_dquaternions, void* scratch, size_t scratch_bytes,
                                  void* stream);

/* coarse_sdf's depth-map SDF estimate (sugar_trainers/coarse_sdf.py:650-712, SuGaR.get_points_depth_in_depth_map
 * sugar_model.py:1189-1204).  The depth map is the float32 view depth [H,W] read with element strides (stride_h, stride_w), so a
 * channel of an [H,W,3] render is read in place.  camera [36] (device, float32) = the world-to-view matrix M (16, row-major, row
 * vectors: [p, 1] @ M, as pytorch3d's get_world_to_view_transform().get_matrix()), the projection matrix (16, likewise, as
 * get_projection_transform().get_matrix(): K^T for SuGaR's SfM cameras), znear, the camera centre (3).  sx, sy are SuGaR's
 * -min(H_img, W_img) / W_img and -min(H_img, W_img) / H_img rounded to float32.  The map depth of a world point p is
 *   v = ([p, 1] @ M).xyz / w;  h = [v, 1] @ K^T;  grid = (sx h.x / h.w, sy h.y / h.w)
 *   map_z = torch's CUDA grid_sample(depth, grid, bilinear, border, align_corners=False): same unnormalize, clip, weights, taps.
 * The 4x4 products are fp32 multiply-add chains in row order; the rest is one rounding per torch op, with the multiply-adds
 * torch's grid sampler is compiled to.
 *
 * gsr_sugar_surface_mask: for P Gaussians (points, scaling [P,3], quaternions [P,4] as SuGaR's getters return them), out_mask [P]
 * (bytes 0/1) = |map_z(p) - v.z| < threshold * |scaling * quaternion_apply(quaternion_invert(q), normalize(c - p))| (coarse_sdf.py
 * :655-666; pytorch3d's Hamilton products, one rounding per op); out_map_z [P] (may be NULL) = map_z(p).  No gradient.
 * P = 0 is a no-op; P < 0, H or W < 1, H * W >= 2^31 or a missing pointer other than out_map_z is GSR_ERR_INVALID. */
int gsr_sugar_surface_mask(int32_t P, int32_t H, int32_t W, int64_t depth_stride_h, int64_t depth_stride_w, const float* depth,
                           float sx, float sy, const float* camera, const float* points, const float* scaling, const float* quaternions,
                           float threshold, uint8_t* out_mask, float* out_map_z, void* stream);

/* gsr_sugar_depth_sdf_loss: coarse_sdf's 'sdf' estimation loss (coarse_sdf.py:689-712, not squared, not normalised by the sample
 * std) over N samples [N,3] with their field sdf_values [N]: with v the camera-space sample and masked = v.z > znear,
 *   term = clamp(|sdf - |map_z - v.z|| * inv_std, max=clamp_max)   (inv_std = float32 1 / float32(std), as torch divides a
 *                                                                    CUDA tensor by a Python number)
 *   out_loss [1] = sum of term over the masked samples / their count (NaN when none is masked), out_count [1] (int64) = the count.
 * Both sums run on the device in a fixed order (float64, then one division), so the result does not depend on the launch.
 * N < 0, H or W < 1, H * W >= 2^31, 4 N >= 2^32 or a missing pointer is GSR_ERR_INVALID; `workspace` (16-byte aligned) needs
 * gsr_sugar_depth_sdf_loss_bytes(N) bytes, else GSR_ERR_WORKSPACE.  No host synchronisation. */
size_t gsr_sugar_depth_sdf_loss_bytes(int32_t N);
int gsr_sugar_depth_sdf_loss(int32_t N, int32_t H, int32_t W, int64_t depth_stride_h, int64_t depth_stride_w, const float* depth,
                             float sx, float sy, const float* camera, const float* samples, const float* sdf_values, float inv_std,
                             float clamp_max, float* out_loss, int64_t* out_count, void* workspace, size_t workspace_bytes,
                             void* stream);

/* Backward of gsr_sugar_depth_sdf_loss (same arguments; count as the forward wrote it; dL_dloss [1]): dL_dsamples [N,3] (through
 * v.z, the projection and the bilinear weights), dL_dsdf [N] and dL_ddepth [H,W] (contiguous, the four taps of every masked
 * sample), all written in full.  A gradient is 0 where torch's autograd of the same expression gives 0: an unmasked sample, a
 * clamped term (term > clamp_max), sign(0) of either |.|, and a grid coordinate the border clip moved or left exactly on a limit.
 * dL_ddepth is summed with atomics here; gsr_sugar_depth_sdf_loss_backward_det sums it in a fixed order. */
int gsr_sugar_depth_sdf_loss_backward(int32_t N, int32_t H, int32_t W, int64_t depth_stride_h, int64_t depth_stride_w, const float* depth,
                                      float sx, float sy, const float* camera, const float* samples, const float* sdf_values, float inv_std,
                                      float clamp_max, const int64_t* count, const float* dL_dloss, float* dL_dsamples, float* dL_dsdf,
                                      float* dL_ddepth, void* stream);

/* Deterministic backward of gsr_sugar_depth_sdf_loss: gsr_sugar_depth_sdf_loss_backward's arguments plus a device scratch (16-byte
 * aligned) of at least gsr_sugar_depth_sdf_loss_backward_det_bytes(N, H, W) = G(4 N, H W) bytes (G as for
 * gsr_sugar_field_backward_det).  Tap k of sample n (id 4n + k) goes to its texel; every texel of dL_ddepth is a sequential fp32
 * sum from +0.0 of its partials in ascending id.  dL_dsamples and dL_dsdf are per sample and equal the atomic backward's.  A NULL
 * or misaligned scratch (when N > 0) is GSR_ERR_INVALID, a smaller one GSR_ERR_WORKSPACE, both before anything is enqueued. */
size_t gsr_sugar_depth_sdf_loss_backward_det_bytes(int32_t N, int32_t H, int32_t W);
int gsr_sugar_depth_sdf_loss_backward_det(int32_t N, int32_t H, int32_t W, int64_t depth_stride_h, int64_t depth_stride_w,
                                          const float* depth, float sx, float sy, const float* camera, const float* samples,
                                          const float* sdf_values, float inv_std, float clamp_max, const int64_t* count,
                                          const float* dL_dloss, float* dL_dsamples, float* dL_dsdf, float* dL_ddepth, void* scratch,
                                          size_t scratch_bytes, void* stream);

/* Densification statistics (GaussianModel.add_densification_stats plus the trainers' max-radii line, gaussian_model.py:415-417,
 * train.py:163-164; SuGaRDensifier.update_densification_stats, sugar_densifier.py:156-164).  For every row i < P with mask[i] != 0:
 *   accum[i] += sqrt(grad[i,0]^2 + grad[i,1]^2)   (grad [P,C], C >= 2: the viewspace points' gradient)
 *   denom[i] += 1
 *   max_radii2D[i] = max(max_radii2D[i], float(radii[i]))   (only when both are given; NaN stays)
 * Other rows are not touched.  No host synchronisation.  P = 0 is a no-op. */
int gsr_densify_stats(int32_t P, int32_t C, const float* grad, const uint8_t* mask, const int32_t* radii, float* accum, float* denom,
                      float* max_radii2D, void* stream);

/* The decisions of densify_and_prune (gaussian_model.py:359-413, sugar_densifier.py:186-246) over the P original rows, given
 * accum [P], denom [P], the raw scaling [P,3] (exp activation) and the raw opacity [P] (sigmoid activation).  Thresholds are the
 * caller's Python floats rounded to float: max_grad, dense_thr = percent_dense * extent, min_opacity, max_screen_size (used only when
 * use_screen, the truthiness of the Python value) and big_thr = 0.1 * extent.  With g = accum / denom (NaN -> 0) and m = max(exp(s)):
 *   clone  = sqrt(g^2) >= max_grad and m <= dense_thr;  split = g >= max_grad and m > dense_thr
 *   prune  = sigmoid(o) < min_opacity or (use_screen and (0 > max_screen_size or m' > big_thr)), m' = m of the row as it will be
 *            (split children: scaling log(exp(s) * (1 / 1.6f))); max_radii2D is 0 there, as densification_postfix leaves it.
 * dst [5,P] (int32) receives, per original row, its destination row in each of the four streams of the final order (surviving
 * originals, surviving clones, surviving first split copies, surviving second split copies), -1 where there is none, and in row 4
 * its index among the split-selected rows.  totals [2] (int32, device) receives {S = split-selected rows, P' = rows after}.
 * `workspace` (16-byte aligned) needs gsr_densify_plan_bytes(P) bytes, else GSR_ERR_WORKSPACE. */
size_t gsr_densify_plan_bytes(int32_t P);
int gsr_densify_plan(int32_t P, const float* accum, const float* denom, const float* scaling, const float* opacity, float max_grad,
                     float dense_thr, float min_opacity, int32_t use_screen, float max_screen_size, float big_thr, int32_t* dst,
                     int32_t* totals, void* workspace, size_t workspace_bytes, void* stream);

#define GSR_DENSIFY_MAX_GROUPS 8
enum { GSR_DENSIFY_ROLE_COPY = 0, GSR_DENSIFY_ROLE_XYZ = 1, GSR_DENSIFY_ROLE_SCALING = 2 };
enum { GSR_DENSIFY_ROTATION_3DGS = 0, GSR_DENSIFY_ROTATION_SUGAR = 1 };
/* One optimizer parameter group of gsr_densify_apply: the parameter [P,width] -> [P',width] and, when the group has Adam state, its
 * two moments (both pointers of a moment NULL otherwise). */
typedef struct gsr_densify_group {
    const float* src;
    float* dst;
    const float* m1_src;
    float* m1_dst;
    const float* m2_src;
    float* m2_dst;
    int32_t width; /* floats per row (0 allowed) */
    int32_t role;  /* GSR_DENSIFY_ROLE_*: how split children are written */
} gsr_densify_group;

/* Writes every row of the new parameters and moments from gsr_densify_plan's dst [5,P]: kept rows and their moments are copied,
 * clones copied with zero moments, split children (zero moments) copied except
 *   ROLE_XYZ (width 3):     R(q) (eps * exp(s)) + xyz, eps row k*S + j for copy k of split row j (eps [2S,3] standard normal),
 *                           R = build_rotation(q) (GSR_DENSIFY_ROTATION_3DGS, general_utils.py:78-99) or pytorch3d
 *                           quaternion_to_matrix(F.normalize(q)) (GSR_DENSIFY_ROTATION_SUGAR), from the raw xyz [P,3],
 *                           scaling [P,3] and rotation [P,4]
 *   ROLE_SCALING (width 3): log(exp(s) * (1 / 1.6f))
 * n_groups <= GSR_DENSIFY_MAX_GROUPS (host array).  The outputs must not alias the inputs. */
int gsr_densify_apply(int32_t P, int32_t S, int32_t n_groups, const gsr_densify_group* groups, const int32_t* dst, const float* xyz,
                      const float* scaling, const float* rotation, const float* eps, int32_t rotation_mode, void* stream);

/* One tensor of gsr_adam_step: a parameter, its gradient and its two Adam moments (numel floats each), and the scalars
 * torch.optim.Adam's foreach path computes for it on the host in double (torch/optim/adam.py:_multi_tensor_adam), each rounded to
 * float as the foreach kernels receive it, for the step count after this step's increment: */
typedef struct gsr_adam_tensor {
    float* param;
    const float* grad;
    float* exp_avg;
    float* exp_avg_sq;
    int64_t numel;
    float lerp_weight;           /* 1 - beta1                                  */
    float beta2;                 /* beta2                                      */
    float one_minus_beta2;       /* 1 - beta2                                  */
    float bias_correction2_sqrt; /* (1 - beta2 ** step) ** 0.5                 */
    float eps;                   /* eps                                        */
    float step_size;             /* (lr / (1 - beta1 ** step)) * -1            */
} gsr_adam_tensor;
#define GSR_ADAM_MAX_TENSORS 32

/* torch.optim.Adam.step() with its defaults (no amsgrad, weight_decay 0, not maximize, foreach) over n tensors, in place and
 * bit-identical to torch's seven list ops:
 *   exp_avg    = lerp(exp_avg, grad, lerp_weight)
 *   exp_avg_sq = exp_avg_sq * beta2 + one_minus_beta2 * grad * grad
 *   param      = param + step_size * exp_avg / (sqrt(exp_avg_sq) / bias_correction2_sqrt + eps)
 * with torch's roundings (see gsr_adam.cu).  Descriptors travel in the kernel parameters (host array, no copy); n beyond
 * GSR_ADAM_MAX_TENSORS takes one launch per GSR_ADAM_MAX_TENSORS.  Float4 accesses where all four pointers of a tensor are 16-byte
 * aligned.  No workspace, no host synchronisation.  n = 0 is a no-op. */
int gsr_adam_step(int32_t n, const gsr_adam_tensor* tensors, void* stream);

/* The training objective's terms (gsr_loss.cu).  Every value is a float32 device scalar written by the call; every mean is a
 * fixed-order reduction (per-CTA float partials, one ordered double sum), bit-identical from call to call.  Upstream gradients are
 * device pointers, so nothing synchronises with the host. */
#define GSR_LOSS_REDUCE_BYTES (256 + 16 * 1024) /* the workspace of every reduction term below but gsr_photometric_loss               */

/* Workspace of gsr_photometric_loss for [B,C,H,W] images: the partial sums, and with for_backward != 0 three float maps of
 * B*C*H*W.  0 for an empty or oversized shape (B*C >= 65536). */
size_t gsr_photometric_loss_bytes(int32_t B, int32_t C, int32_t H, int32_t W, int32_t for_backward);
/* out_l1[0] = mean |x - y| (skipped when out_l1 is NULL), out_ssim[0] = mean SSIM of ssim(x, y) with the 11-tap window `window` (host [11], the 1-D
 * float weights of create_window; applied separably), zero padding of 5, C1 = 0.01^2, C2 = 0.03^2.  x and y are [B,C,H,W] float
 * images addressed by element strides x_strides / y_strides (host [4]: b, c, y, x), so a channel-innermost view needs no copy.
 * `workspace` (16-byte aligned) needs gsr_photometric_loss_bytes(B, C, H, W, for_backward), else GSR_ERR_WORKSPACE; with
 * for_backward != 0 it keeps the three per-pixel SSIM maps dS/d(mu_x, E[x^2], E[xy]) for gsr_photometric_loss_backward. */
int gsr_photometric_loss(int32_t B, int32_t C, int32_t H, int32_t W, const float* x, const int64_t* x_strides, const float* y,
                         const int64_t* y_strides, const float* window, int32_t for_backward, float* out_l1, float* out_ssim,
                         void* workspace, size_t workspace_bytes, void* stream);
/* dx (contiguous [B,C,H,W]) = g_ssim * d mean SSIM / dx + g_l1 * d mean |x - y| / dx, the upstream gradients read on the device
 * (NULL = zero); the abs's gradient is 0 where x == y.  `workspace` is the forward's, run with for_backward on the same
 * images.  Each pixel is written by one thread; no atomics. */
int gsr_photometric_loss_backward(int32_t B, int32_t C, int32_t H, int32_t W, const float* x, const int64_t* x_strides, const float* y,
                                  const int64_t* y_strides, const float* window, const float* g_l1, const float* g_ssim, float* dx,
                                  const void* workspace, size_t workspace_bytes, void* stream);
/* normal_loss over n pixels: pred and gt are [n,3] by (pixel, component) element strides (host [2] each).  Each is normalised as
 * F.normalize does (norm clamped at 1e-12); out[0] = mean |n - g| + 0.1 * (-mean n.g) over the selected pixels: all, or with
 * depth != NULL those with depth[i * depth_stride] in (0, scene_scale).  No selected pixel gives NaN, as torch's mean of an empty
 * tensor.  `workspace` (16-byte aligned) needs GSR_LOSS_REDUCE_BYTES; it keeps the selected count for the backward. */
int gsr_normal_loss(int64_t n, const float* pred, const int64_t* pred_strides, const float* gt, const int64_t* gt_strides,
                    const float* depth, int64_t depth_stride, float scene_scale, float* out, void* workspace, size_t workspace_bytes,
                    void* stream);
/* d_pred (contiguous [n,3]) = g_out[0] * d out / d pred, through normalize's Jacobian (divided by 1e-12 below the clamp); zero for
 * pixels outside the selection.  `workspace` is the forward's. */
int gsr_normal_loss_backward(int64_t n, const float* pred, const int64_t* pred_strides, const float* gt, const int64_t* gt_strides,
                             const float* depth, int64_t depth_stride, float scene_scale, const float* g_out, float* d_pred,
                             const void* workspace, size_t workspace_bytes, void* stream);
/* out[0] = mean over P Gaussians of clamp_min(max / (min + 1e-6), r) - r of contiguous scales [P,3].  `workspace` (16-byte aligned)
 * needs GSR_LOSS_REDUCE_BYTES. */
int gsr_anisotropic_loss(int64_t P, const float* scales, float r, float* out, void* workspace, size_t workspace_bytes, void* stream);
/* d_scales [P,3] = g_out[0] * d out / d scales: the max's and the min's gradient go to the first extreme index (NaN first), as
 * torch's max(dim) / min(dim) return it; nothing where the ratio is below r (clamp_min passes ratio == r).  One thread per Gaussian. */
int gsr_anisotropic_loss_backward(int64_t P, const float* scales, float r, const float* g_out, float* d_scales, void* stream);
/* depth_loss over n pixels of pred (the rendered depth) and gt (the monocular depth), each by one element stride.  With
 * d = gt * float32(1 / 25) and the mask d > 0, the five masked sums (p^2, p, count, p d, d) are accumulated in double in a fixed
 * order and rounded to float32; x0 (scale) and x1 (shift) solve the 2x2 system with torch's operation order in one thread and stay
 * in `workspace`.  out[0] = mean over all n of w * exp(-p * scene_scale_inv) * (x0 p + x1 - d)^2, w = 1 on the mask, else 0;
 * scene_scale_inv is float32(1 / float32(scene_scale)), as torch divides by a Python number.  det == 0 (an empty mask included)
 * gives x0 = x1 = NaN, so the value and every gradient are NaN.  `workspace` (16-byte aligned) needs GSR_LOSS_REDUCE_BYTES. */
int gsr_depth_loss(int64_t n, const float* pred, int64_t pred_stride, const float* gt, int64_t gt_stride, float scene_scale_inv,
                   float* out, void* workspace, size_t workspace_bytes, void* stream);
/* d_pred (contiguous [n]) = g_out[0] / n * w exp(-p s^-1) * 2 (x0 p + x1 - d) * x0; the scale, the shift and the exp factor are
 * constants, as the reference detaches them.  `workspace` is the forward's (it holds x0 and x1). */
int gsr_depth_loss_backward(int64_t n, const float* pred, int64_t pred_stride, const float* gt, int64_t gt_stride,
                            float scene_scale_inv, const float* g_out, float* d_pred, const void* workspace, size_t workspace_bytes,
                            void* stream);
/* out[0] = mean of n values x[i * x_stride].  `workspace` (16-byte aligned) needs GSR_LOSS_REDUCE_BYTES. */
int gsr_opacity_loss(int64_t n, const float* x, int64_t x_stride, float* out, void* workspace, size_t workspace_bytes, void* stream);
/* dx (contiguous [n]) = g_out[0] / n. */
int gsr_opacity_loss_backward(int64_t n, const float* g_out, float* dx, void* stream);
/* out[0] = mean of log c + log(1 - c), c = clamp(x, 1e-3, 1 - 1e-3) with the bounds rounded to float32.  `workspace` as above. */
int gsr_sparsity_loss(int64_t n, const float* x, int64_t x_stride, float* out, void* workspace, size_t workspace_bytes, void* stream);
/* dx (contiguous [n]) = g_out[0] / n * (1 / c - 1 / (1 - c)) where 1e-3 <= x <= 1 - 1e-3 (both bounds pass, as torch's clamp
 * backward), else 0. */
int gsr_sparsity_loss_backward(int64_t n, const float* x, int64_t x_stride, const float* g_out, float* dx, void* stream);
/* out[0] = mean over the P Gaussians with radii[i * r_stride] > 0 of -o log(o + 1e-10) - (1 - o) log(1 - o + 1e-10),
 * o = opacities[i * o_stride]; the visible count stays in `workspace` (16-byte aligned, GSR_LOSS_REDUCE_BYTES).  No visible
 * Gaussian gives NaN, as torch's mean of an empty tensor. */
int gsr_entropy_loss(int64_t P, const float* opacities, int64_t o_stride, const int32_t* radii, int64_t r_stride, float* out,
                     void* workspace, size_t workspace_bytes, void* stream);
/* d_opacities (contiguous [P]) = g_out[0] / count * d term / d o on the visible Gaussians, 0 elsewhere.  `workspace` is the
 * forward's. */
int gsr_entropy_loss_backward(int64_t P, const float* opacities, int64_t o_stride, const int32_t* radii, int64_t r_stride,
                              const float* g_out, float* d_opacities, const void* workspace, size_t workspace_bytes, void* stream);
/* out[0] = mean over n samples of |d - exp(-0.5 s^2 / beta^2)| (squared != 0: its square), d = density, s = sdf_estimation, each
 * by one element stride, with one float32 rounding per torch op.  `workspace` (16-byte aligned) needs GSR_LOSS_REDUCE_BYTES. */
int gsr_density_estimation_loss(int64_t n, const float* density, int64_t d_stride, const float* beta, int64_t b_stride,
                                const float* sdf_estimation, int64_t s_stride, int32_t squared, float* out, void* workspace,
                                size_t workspace_bytes, void* stream);
/* The three gradients (contiguous [n] each) = g_out[0] * d out / d (density, beta, sdf_estimation), by torch's backward chain:
 * the abs's gradient is 0 where d equals its target, and then so are the other two. */
int gsr_density_estimation_loss_backward(int64_t n, const float* density, int64_t d_stride, const float* beta, int64_t b_stride,
                                         const float* sdf_estimation, int64_t s_stride, int32_t squared, const float* g_out,
                                         float* d_density, float* d_beta, float* d_sdf_estimation, void* stream);

/* Frame compositing (gsr_composite.cu), bit-identical to blender/blend_all.py:blend_frames on the same decoded arrays. */
#define GSR_PERCENTILE_BYTES 2048 /* the workspace of gsr_percentile_low */
/* out[0] = np.percentile(x, 0.001) of n float32 values (numpy's default 'linear' method, in float32 as NumPy >= 2 computes it
 * for a float32 array); NaN when any value is NaN.  The result stays on the device; nothing synchronises with the host.
 * 1 <= n < 2^31, else GSR_ERR_INVALID; `workspace` (16-byte aligned) needs GSR_PERCENTILE_BYTES, else GSR_ERR_WORKSPACE. */
int gsr_percentile_low(int64_t n, const float* x, float* out, void* workspace, size_t workspace_bytes, void* stream);
/* out [H,W,4] uint8 = the composited frame of blend_frames (:236-342) from:
 *   frame [H,W,4] uint8 (the 3DGS frame: images/*.png, or rgba8 of gsr_pack_frame);
 *   obj, shadow, all [H,W,4] uint8 (rgb_obj, rgb_shadow, rgb_all) and obj_depth, shadow_depth [H,W] float (depth_obj, depth_shadow);
 *   optional pairs obj3dgs + obj3dgs_depth (rgb_obj_3dgs, depth_obj_3dgs) and smoke + smoke_depth (rgb_smoke_fire,
 *   depth_smoke_fire) with smoke_pct, the device scalar gsr_percentile_low wrote for smoke_depth; optional fire [H,W,4] uint8
 *   (rgb_smoke_fire_pre), which needs smoke.
 * The frame's depth, depth_all and depth_smoke_fire_pre never affect the frame and are not arguments.  8-bit layers must be
 * 4-byte aligned.  A missing required layer, an unpaired optional one or fire without smoke is GSR_ERR_INVALID. */
int gsr_composite(int32_t W, int32_t H, const uint8_t* frame, const uint8_t* obj, const float* obj_depth, const uint8_t* shadow,
                  const float* shadow_depth, const uint8_t* all, const uint8_t* obj3dgs, const float* obj3dgs_depth, const uint8_t* smoke,
                  const float* smoke_depth, const float* smoke_pct, const uint8_t* fire, uint8_t* out, void* stream);

/* Candidate-subset scoring of extract_object (gsr_extract.cu).  Nothing here synchronises with the host. */
/* Bytes of gsr_select_rows' workspace for P rows (0 when P is out of range). */
size_t gsr_select_rows_bytes(int64_t P);
/* t_out[:n] = t[keep] for means3D [P,3], opacities [P,1], scales [P,3] and rotations [P,4], with *count = n (device int32): the kept
 * rows in their original order, bit for bit (sort ties resolve by Gaussian index, so the order decides the image).  keep is a
 * bool [P] (one byte per row, nonzero = kept); the outputs hold P rows.  0 <= P < 2^31, else GSR_ERR_INVALID. */
int gsr_select_rows(int64_t P, const uint8_t* keep, const float* means3D, const float* opacities, const float* scales, const float* rotations,
                    float* means3D_out, float* opacities_out, float* scales_out, float* rotations_out, int32_t* count, void* workspace,
                    size_t workspace_bytes, void* stream);
/* bits [V,H,ceil(W/32)] uint32 from masks [V,H,W] uint8: bit x % 32 of word (v, y, x / 32) is masks[v,y,x] == 255; bits past W are 0. */
int gsr_pack_masks(int32_t V, int32_t W, int32_t H, const uint8_t* masks, uint32_t* bits, void* stream);
/* *count += the pixels of one [H,W] frame where (alpha >= thr) differs from the packed mask bit (bits [H,ceil(W/32)] of
 * gsr_pack_masks).  The comparison is float32, and false for a NaN alpha, as numpy's `alpha >= np.float32(thr)` is.  count is an
 * 8-byte aligned device int64; the sum is exact and the same on every run. */
int gsr_mask_disagreement(int32_t W, int32_t H, const float* alpha, const uint32_t* bits, float thr, int64_t* count, void* stream);

/* PNG encoding (gsr_png.cu): standard 8-bit, non-interlaced PNG files (one IHDR, one IDAT holding one zlib stream, IEND) whose
 * pixels decode to the input exactly.  The bytes are this encoder's own, not libpng's or zlib's: they depend only on the pixels
 * and the shape (not on the stream, the batch or the order of atomics).  Nothing synchronises with the host. */
#define GSR_PNG_SWAP_RB 1    /* read channels 0 and 2 swapped: BGR / BGRA input, RGB / RGBA file */
#define GSR_PNG_MAX_BATCH 16 /* images per launch; gsr_png_encode launches 4 kernels per group of this many images */
typedef struct gsr_png_image {
    const uint8_t* data;                 /* byte (y, x, c) at data + y * stride_h + x * stride_w + c * stride_c (device or UVA) */
    int64_t stride_h, stride_w, stride_c; /* byte strides, may be negative */
    int32_t H, W, C;                     /* C in {1, 3, 4}: grey (colour type 0), RGB (2) or RGBA (6) */
    int32_t flags;                       /* GSR_PNG_SWAP_RB */
    const uint8_t* lut;                  /* NULL, or a device [256,3] RGB table for C = 1: the file is RGB lut[data] */
} gsr_png_image;
/* The largest file an H x W image with C channels in the file (3 for a lookup-table image) can take: the filtered stream
 * H (1 + W C), 5 bytes per 32 KiB deflate block, and 63 bytes of signature, chunks and zlib framing.  0 for a bad shape or a
 * stream too long for one IDAT chunk. */
size_t gsr_png_bound(int32_t H, int32_t W, int32_t C);
/* Bytes of gsr_png_encode's workspace for these images (about 5.1 times their filtered streams); 0 for bad arguments. */
size_t gsr_png_workspace_bytes(int32_t n, const gsr_png_image* images);
/* Encode n images: outputs[i] (device or pinned host memory, at least gsr_png_bound bytes) receives the file and sizes[i] (an
 * 8-byte aligned device or pinned int64) its length.  `workspace` is 256-byte aligned device memory of gsr_png_workspace_bytes.
 * An image with no data, H or W < 1, C not in {1, 3, 4}, a lookup table with C != 1, unknown flags or a too-long stream, a NULL
 * output or misaligned sizes is GSR_ERR_INVALID, a smaller workspace GSR_ERR_WORKSPACE, all before anything is enqueued.
 * n = 0 is a no-op. */
int gsr_png_encode(const gsr_png_image* images, int32_t n, uint8_t* const* outputs, int64_t* sizes, void* workspace, size_t workspace_bytes,
                   void* stream);

/* ---- first-hit ray casts and closest triangles on a triangle mesh (gsr_mesh.cu): an LBVH over F triangles, DESIGN.md §4 ---- */
/* Bytes of the BVH buffer of F triangles (float32 boxes, float64 triangles in leaf order), and of gsr_mesh_build's scratch. */
size_t gsr_mesh_bvh_bytes(int32_t F);
size_t gsr_mesh_build_bytes(int32_t F);
/* Build the BVH of F triangles: vertices float64 [V,3], faces int64 [F,3] (device).  A triangle with a vertex index outside
 * [0, V), a non-finite vertex, or (v1 - v0) x (v2 - v0) == 0 in float64 is never hit.  bvh and workspace are 256-byte aligned
 * device memory; the workspace may be reused once the build has run on the stream. */
int gsr_mesh_build(int64_t V, int32_t F, const double* vertices, const int64_t* faces, void* bvh, size_t bvh_bytes, void* workspace,
                   size_t workspace_bytes, void* stream);
/* First hit of N rays (origins, directions [N,3], float32 if f64 == 0, float64 if f64 == 1, widened exactly) on a BVH built for
 * F triangles: tri[i] the original index of the triangle with the smallest t > 0 (ties: the lower index), -1 on a miss;
 * t[i] (may be NULL) its distance in units of the direction as given, +inf on a miss.  The watertight test in float64, every
 * operation rounded on its own, both faces; a zero, NaN or infinite ray misses.  active (may be NULL): rays with
 * active[i] < 0 are not cast and miss.  Identical results on any stream and from run to run. */
int gsr_mesh_first_hit(int32_t F, const void* bvh, int64_t N, const void* origins, const void* directions, int32_t f64, const int64_t* active,
                       int64_t* tri, double* t, void* stream);
/* The inpainting mask of one view (extract_object.py:563-606) from a planar-mesh cast and a combined-mesh cast of the same N rays:
 * mask[i] = 255 where ray i hits the planar mesh and |depth_all - depth_planar| < 0.01, else 0, with location = o + t d per
 * component, depth = ((x w2c[8] + y w2c[9]) + z w2c[10]) + w2c[11] (w2c row-major float64 [4,4]), and depth_all = 0 where the
 * combined mesh is missed.  counts (8-byte aligned int64 [2]) = (planar hits, planar hits that also hit the combined mesh). */
int gsr_mesh_inpaint_mask(int64_t N, const void* origins, const void* directions, int32_t f64, const int64_t* tri_planar, const double* t_planar,
                          const int64_t* tri_all, const double* t_all, const double* w2c, uint8_t* mask, int64_t* counts, void* stream);
/* Bytes of gsr_mesh_closest's workspace for N points (0 when N is out of range). */
size_t gsr_mesh_closest_bytes(int64_t N);
/* Closest triangle of N < 2^31 points ([N,3], float32 if f64 == 0, float64 if f64 == 1, widened exactly) on a BVH built for F
 * triangles, the queries processed along a Morton curve (workspace: 256-byte aligned device memory), the results in caller order:
 * tri[i] the original index of the valid triangle with the smallest squared distance to point i (ties: the lower index); d2[i]
 * (may be NULL) that squared distance.  Ericson's ClosestPtPointTriangle in float64, every operation rounded on its own
 * (DESIGN.md §4).  A point with a non-finite coordinate, F == 0 or a mesh without a valid triangle gives -1 and +inf.
 * Identical results on any stream and from run to run. */
int gsr_mesh_closest(int32_t F, const void* bvh, int64_t N, const void* points, int32_t f64, int64_t* tri, double* d2, void* workspace,
                     size_t workspace_bytes, void* stream);
/* Bytes of gsr_mesh_isin_rows' workspace for N rows and F triangles (0 when out of range). */
size_t gsr_mesh_isin_rows_bytes(int64_t N, int32_t F);
/* np.isin(tri, query_tri) followed by boolean indexing, for the melting-mesh frame: row i (of N) is kept when 0 <= tri[i] < F and
 * tri[i] is one of the Q entries of query_tri (entries outside [0, F) match nothing).  The kept rows of K <= 8 arrays, array k
 * holding words[k] 32-bit words per row (src[k], dst[k]: host arrays of device pointers), are copied in row order to the front
 * of dst[k], bit for bit; count (device int64) receives their number.  workspace: 4-byte aligned device memory. */
int gsr_mesh_isin_rows(int64_t N, const int64_t* tri, int64_t Q, const int64_t* query_tri, int32_t F, int32_t K, const void* const* src,
                       void* const* dst, const int32_t* words, int64_t* count, void* workspace, size_t workspace_bytes, void* stream);

/* Device pointers into the workspaces of the last layout (P, capacity, W, H) — for parity tests that
 * compare per-stage buffers with the reference (SURVEY §4).  Pure pointer arithmetic, no CUDA calls. */
typedef struct gsr_views {
    const float* records;        /* [P,12]: x, y, conic_a, conic_b | conic_c, opacity, depth, radius (int bits) | r, g, b, log2 opacity */
    const float* cov3D;          /* [P,6]  (GSR_FLAG_FOR_BACKWARD only)                             */
    const uint8_t* clamped;      /* [P]    bit c set = channel c clamped (GSR_FLAG_FOR_BACKWARD only) */
    const uint32_t* point_list;  /* [capacity] Gaussian ids, per tile front-to-back                 */
    const uint64_t* sorted_keys; /* [capacity] (GSR_FLAG_SORTED_KEYS only)                          */
    const uint32_t* ranges;      /* [tiles,2]                                                       */
    const uint32_t* n_contrib;   /* [H,W]  (GSR_FLAG_FOR_BACKWARD only)                             */
    const uint32_t* tile_count;  /* [tiles] instances of Gaussians touching <= 8 tiles                   */
    const uint32_t* tile_big;    /* [tiles] instances of Gaussians touching > 8 tiles                    */
    const gsr_counters* counters;
} gsr_views;
int gsr_get_views(const gsr_workspace* ws, int32_t P, int32_t W, int32_t H, gsr_views* out);

/* Per-kernel device timing of gsr_forward (CUDA events on the launching stream), for roofline reports.
 * ms_per_kernel[5] = average ms of {preprocess, tile_scan, emit, sort_tiles, blend} over the profiled frames. */
int gsr_profile_begin(int max_frames);
/* Same, timing only every stride-th gsr_forward call. */
int gsr_profile_begin_strided(int max_frames, int stride);
int gsr_profile_end(float* ms_per_kernel, int* frames);

const char* gsr_last_error(void);
int gsr_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* GSR_B200_H_INCLUDED */
