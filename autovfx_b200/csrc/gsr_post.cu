// gsr_b200 — the per-Gaussian and per-pixel work the reference's render() wrappers do around the two rasterizer passes
// (sugar/gaussian_splatting/gaussian_renderer/__init__.py:83-218 = "GR/", utils/general_utils.py = "GU/"), as three
// HBM-streaming kernels instead of ~25 elementwise torch launches:
//
//   k_axis_normals   per-Gaussian shading normal = shortest axis of the Gaussian, flipped towards the camera
//                    (GaussianModel.get_normal, scene/gaussian_model.py:120-128; GU/:78-99,136-157), optionally remapped
//                    to [0,1] (GR/:147) — the colors_precomp of the reference's second pass
//   k_sugar_normals  the same for SuGaR's wrapper (sugar_scene/sugar_model.py:2164-2168): quaternion_to_matrix of the raw
//                    quaternion, min-scale axis, flip, * 0.5 + 0.5; k_sugar_normals_backward gives its quaternion gradient
//   k_normal_maps    rendered normal image -> unit normals [H,W,3] (GR/:168-176) and the pseudo normal from the depth map
//                    (depth_pcd2normal + get_ray_directions, GR/:23-38,41-80,178-191)
//   k_pack_frame     8-bit hand-off of a finished frame: RGBA (torchvision.utils.save_image rounding), normal map and
//                    depth colormap index (scene_representation.py:424-438, sugar/render.py:18-22)
//
// Each torch op of the reference rounds once, so the arithmetic below uses explicit round-to-nearest intrinsics in the
// reference's operation order (no FMA contraction); reductions over 3-4 elements are summed left to right.
#include "gsr_common.cuh"

namespace gsr {

__global__ void __launch_bounds__(256) k_axis_normals(int P, const float* __restrict__ means3D, const float* __restrict__ scales,
                                                      const float* __restrict__ rotations, const float* __restrict__ campos, int remap01,
                                                      float* __restrict__ out) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    const AxisPick p = axis_pick(scales[3 * (size_t)idx], scales[3 * (size_t)idx + 1], scales[3 * (size_t)idx + 2], rotations[4 * (size_t)idx],
                                 rotations[4 * (size_t)idx + 1], rotations[4 * (size_t)idx + 2], rotations[4 * (size_t)idx + 3],
                                 means3D[3 * (size_t)idx], means3D[3 * (size_t)idx + 1], means3D[3 * (size_t)idx + 2], campos);
    float n0 = p.a0, n1 = p.a1, n2 = p.a2;
    if (p.flip) { n0 = -n0; n1 = -n1; n2 = -n2; }
    const float nn = norm3_rn(n0, n1, n2);
    n0 = __fdiv_rn(n0, nn); n1 = __fdiv_rn(n1, nn); n2 = __fdiv_rn(n2, nn);
    if (remap01) {  // normal * 0.5 + 0.5 (GR/:147)
        n0 = __fadd_rn(__fmul_rn(n0, 0.5f), 0.5f); n1 = __fadd_rn(__fmul_rn(n1, 0.5f), 0.5f); n2 = __fadd_rn(__fmul_rn(n2, 0.5f), 0.5f);
    }
    out[3 * (size_t)idx] = n0; out[3 * (size_t)idx + 1] = n1; out[3 * (size_t)idx + 2] = n2;
}

// SuGaR's per-Gaussian shading normal (sugar_model.py:2164-2168): get_smallest_axis, flip_align_view towards camera_center,
// division by the norm (no epsilon), then normal * 0.5 + 0.5.  positions / scales / quaternions as SuGaR's getters return them.
__global__ void __launch_bounds__(256) k_sugar_normals(int P, const float* __restrict__ positions, const float* __restrict__ scales,
                                                       const float* __restrict__ quaternions, const float* __restrict__ campos,
                                                       float* __restrict__ out) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    const size_t n3 = 3 * (size_t)idx, n4 = 4 * (size_t)idx;
    const SugarAxisPick p = sugar_axis_pick(scales[n3], scales[n3 + 1], scales[n3 + 2], quaternions[n4], quaternions[n4 + 1],
                                            quaternions[n4 + 2], quaternions[n4 + 3], positions[n3], positions[n3 + 1], positions[n3 + 2],
                                            campos);
    float n0 = p.a0, n1 = p.a1, n2 = p.a2;
    if (p.flip) { n0 = -n0; n1 = -n1; n2 = -n2; }
    const float nn = norm3_rn(n0, n1, n2);
    n0 = __fdiv_rn(n0, nn); n1 = __fdiv_rn(n1, nn); n2 = __fdiv_rn(n2, nn);
    out[n3] = __fadd_rn(__fmul_rn(n0, 0.5f), 0.5f);
    out[n3 + 1] = __fadd_rn(__fmul_rn(n1, 0.5f), 0.5f);
    out[n3 + 2] = __fadd_rn(__fmul_rn(n2, 0.5f), 0.5f);
}

// Its backward with respect to the raw quaternion q = (r, i, j, k).  With the column a = base + sigma * t * u(q) (base = 1 and
// sigma = -1 on the diagonal entry, 0 and +1 elsewhere), t = 2 / |q|^2 and dt/dq = -t^2 q:
//   c = dL/da = sign * (e - m (m.e)) / |a|,   e = 0.5 * dL/dout,   m the unit normal,
//   dL/dq = t * sum_l sigma_l c_l du_l/dq - t^2 * (sum_l sigma_l c_l u_l) * q.
// The axis k and the flip are piecewise constant in positions and scales, which therefore get no gradient here;
// sugar_axis_pick recomputes the forward's decisions from the same fp32 inputs.
__global__ void __launch_bounds__(256) k_sugar_normals_backward(int P, const float* __restrict__ positions, const float* __restrict__ scales,
                                                                const float* __restrict__ quaternions, const float* __restrict__ campos,
                                                                const float* __restrict__ dL_dout, float* __restrict__ dL_dq) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    const size_t n3 = 3 * (size_t)idx, n4 = 4 * (size_t)idx;
    const float r = quaternions[n4], i = quaternions[n4 + 1], j = quaternions[n4 + 2], k = quaternions[n4 + 3];
    const SugarAxisPick a = sugar_axis_pick(scales[n3], scales[n3 + 1], scales[n3 + 2], r, i, j, k, positions[n3], positions[n3 + 1],
                                            positions[n3 + 2], campos);
    const float sg = a.flip ? -1.0f : 1.0f;
    const float ia = 1.0f / sqrtf(a.a0 * a.a0 + a.a1 * a.a1 + a.a2 * a.a2);
    const float m0 = sg * a.a0 * ia, m1 = sg * a.a1 * ia, m2 = sg * a.a2 * ia;
    const float e0 = 0.5f * dL_dout[n3], e1 = 0.5f * dL_dout[n3 + 1], e2 = 0.5f * dL_dout[n3 + 2];
    const float me = m0 * e0 + m1 * e1 + m2 * e2;
    const float c0 = sg * (e0 - m0 * me) * ia, c1 = sg * (e1 - m1 * me) * ia, c2 = sg * (e2 - m2 * me) * ia;
    float gr, gi, gj, gk, su;  // sum_l sigma_l c_l du_l/dq and sum_l sigma_l c_l u_l
    if (a.k == 0) {         // u = (jj + kk, ij + kr, ik - jr)
        gr = c1 * k - c2 * j; gi = c1 * j + c2 * k; gj = c1 * i - c2 * r - 2.0f * j * c0; gk = c1 * r + c2 * i - 2.0f * k * c0;
        su = -c0 * (j * j + k * k) + c1 * (i * j + k * r) + c2 * (i * k - j * r);
    } else if (a.k == 1) {  // u = (ij - kr, ii + kk, jk + ir)
        gr = c2 * i - c0 * k; gi = c0 * j + c2 * r - 2.0f * i * c1; gj = c0 * i + c2 * k; gk = c2 * j - c0 * r - 2.0f * k * c1;
        su = c0 * (i * j - k * r) - c1 * (i * i + k * k) + c2 * (j * k + i * r);
    } else {                // u = (ik + jr, jk - ir, ii + jj)
        gr = c0 * j - c1 * i; gi = c0 * k - c1 * r - 2.0f * i * c2; gj = c0 * r + c1 * k - 2.0f * j * c2; gk = c0 * i + c1 * j;
        su = c0 * (i * k + j * r) + c1 * (j * k - i * r) - c2 * (i * i + j * j);
    }
    const float t = a.two_s, tts = t * t * su;
    dL_dq[n4] = t * gr - tts * r; dL_dq[n4 + 1] = t * gi - tts * i; dL_dq[n4 + 2] = t * gj - tts * j; dL_dq[n4 + 3] = t * gk - tts * k;
}

// world-space point of pixel (x, y) at the rendered depth (GR/:41-80,185-190): directions @ c2w[:3,:3].T * depth + c2w[:3,3]
struct PseudoCam {
    float m[12];  // c2w rows 0..2 (row-major 3x4) of the matrix the reference calls c2w = world_view_transform.inverse()
    float fx, fy, cx, cy;
};
__device__ __forceinline__ float3 unproject(const PseudoCam& c, int x, int y, float depth) {
    const float d0 = __fdiv_rn(__fadd_rn(__fsub_rn((float)x, c.cx), 0.5f), c.fx);
    const float d1 = __fdiv_rn(__fadd_rn(__fsub_rn((float)y, c.cy), 0.5f), c.fy);
    float3 p;
    p.x = __fadd_rn(c.m[3], __fmul_rn(__fadd_rn(__fadd_rn(__fmul_rn(d0, c.m[0]), __fmul_rn(d1, c.m[1])), c.m[2]), depth));
    p.y = __fadd_rn(c.m[7], __fmul_rn(__fadd_rn(__fadd_rn(__fmul_rn(d0, c.m[4]), __fmul_rn(d1, c.m[5])), c.m[6]), depth));
    p.z = __fadd_rn(c.m[11], __fmul_rn(__fadd_rn(__fadd_rn(__fmul_rn(d0, c.m[8]), __fmul_rn(d1, c.m[9])), c.m[10]), depth));
    return p;
}

__global__ void __launch_bounds__(256) k_normal_maps(int W, int H, const float* __restrict__ normal_img /*[3,H,W] or null*/,
                                                     const float* __restrict__ depth /*[H,W] or null*/, const float* __restrict__ c2w,
                                                     float fx, float fy, float cx, float cy, float* __restrict__ out_normal /*[H,W,3]*/,
                                                     float* __restrict__ out_pseudo /*[H,W,3]*/) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= W || y >= H) return;
    const size_t pid = (size_t)y * W + x, HW = (size_t)W * H;
    if (normal_img && out_normal) {  // (img - 0.5) * 2, then F.normalize(p=2, dim=-1, eps=1e-12)  (GR/:168-176)
        const float a = __fmul_rn(__fsub_rn(normal_img[pid], 0.5f), 2.0f), b = __fmul_rn(__fsub_rn(normal_img[HW + pid], 0.5f), 2.0f),
                    c = __fmul_rn(__fsub_rn(normal_img[2 * HW + pid], 0.5f), 2.0f);
        const float n = fmaxf(norm3_rn(a, b, c), 1e-12f);
        out_normal[3 * pid] = __fdiv_rn(a, n); out_normal[3 * pid + 1] = __fdiv_rn(b, n); out_normal[3 * pid + 2] = __fdiv_rn(c, n);
    }
    if (depth && out_pseudo) {  // depth_pcd2normal (GR/:23-38): central differences, zero border
        float o0 = 0.f, o1 = 0.f, o2 = 0.f;
        if (x > 0 && y > 0 && x < W - 1 && y < H - 1) {
            PseudoCam c;
#pragma unroll
            for (int i = 0; i < 12; i++) c.m[i] = c2w[i];
            c.fx = fx; c.fy = fy; c.cx = cx; c.cy = cy;
            const float3 pr = unproject(c, x + 1, y, depth[pid + 1]), pl = unproject(c, x - 1, y, depth[pid - 1]);
            const float3 pt = unproject(c, x, y - 1, depth[pid - W]), pb = unproject(c, x, y + 1, depth[pid + W]);
            const float ax = __fsub_rn(pr.x, pl.x), ay = __fsub_rn(pr.y, pl.y), az = __fsub_rn(pr.z, pl.z);  // left_to_right
            const float bx = __fsub_rn(pt.x, pb.x), by = __fsub_rn(pt.y, pb.y), bz = __fsub_rn(pt.z, pb.z);  // bottom_to_top
            const float nx = __fsub_rn(__fmul_rn(ay, bz), __fmul_rn(az, by)), ny = __fsub_rn(__fmul_rn(az, bx), __fmul_rn(ax, bz)),
                        nz = __fsub_rn(__fmul_rn(ax, by), __fmul_rn(ay, bx));
            const float n = fmaxf(norm3_rn(nx, ny, nz), 1e-12f);
            o0 = __fdiv_rn(nx, n); o1 = __fdiv_rn(ny, n); o2 = __fdiv_rn(nz, n);
        }
        out_pseudo[3 * pid] = o0; out_pseudo[3 * pid + 1] = o1; out_pseudo[3 * pid + 2] = o2;
    }
}

// 8-bit hand-off.  rgba8: torchvision.utils.save_image = mul(255).add(0.5).clamp(0,255).to(uint8) on cat(rgb, alpha)
// (scene_representation.py:424-425, GR/:143); normal8: ((n + 1) / 2 * 255).astype(uint8) (scene_representation.py:433-436);
// depth8: (clip(depth / scale, 0, 1) * 255).astype(uint8), the index into the TURBO colormap (sugar/render.py:18-22).
__device__ __forceinline__ uint32_t q_save_image(float v) {
    const float t = fminf(fmaxf(__fadd_rn(__fmul_rn(v, 255.0f), 0.5f), 0.0f), 255.0f);
    return (uint32_t)t;  // NaN -> 0 like the clamp + cast on the GPU path
}
__global__ void __launch_bounds__(256) k_pack_frame(int W, int H, const float* __restrict__ rgb, const float* __restrict__ alpha,
                                                    const float* __restrict__ depth, const float* __restrict__ normal_hwc, float depth_scale,
                                                    uint32_t* __restrict__ rgba8, uint8_t* __restrict__ normal8, uint8_t* __restrict__ depth8) {
    const size_t HW = (size_t)W * H;
    const size_t pid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (pid >= HW) return;
    if (rgba8) {
        const uint32_t a = alpha ? q_save_image(alpha[pid]) : 255u;
        rgba8[pid] = q_save_image(rgb[pid]) | (q_save_image(rgb[HW + pid]) << 8) | (q_save_image(rgb[2 * HW + pid]) << 16) | (a << 24);
    }
    if (normal8) {
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const float v = __fmul_rn(__fdiv_rn(__fadd_rn(normal_hwc[3 * pid + c], 1.0f), 2.0f), 255.0f);
            normal8[3 * pid + c] = (uint8_t)(int)v;  // numpy astype(uint8) truncates; the value is in [0, 255]
        }
    }
    if (depth8) {
        const float v = __fmul_rn(fminf(fmaxf(__fdiv_rn(depth[pid], depth_scale), 0.0f), 1.0f), 255.0f);
        depth8[pid] = (uint8_t)(int)v;
    }
}

int axis_normals_impl(int P, const float* means3D, const float* scales, const float* rotations, const float* campos, int remap01,
                      float* out, cudaStream_t st) {
    if (P < 0 || (P > 0 && (!means3D || !scales || !rotations || !campos || !out))) { set_error("gsr_axis_normals: bad arguments"); return GSR_ERR_INVALID; }
    if (P == 0) return GSR_OK;
    k_axis_normals<<<(P + 255) / 256, 256, 0, st>>>(P, means3D, scales, rotations, campos, remap01, out);
    return check_launch("gsr_axis_normals", false, st);
}

int sugar_normals_impl(int P, const float* positions, const float* scales, const float* quaternions, const float* campos, float* out,
                       cudaStream_t st) {
    if (P < 0 || (P > 0 && (!positions || !scales || !quaternions || !campos || !out))) { set_error("gsr_sugar_normals: bad arguments"); return GSR_ERR_INVALID; }
    if (P == 0) return GSR_OK;
    k_sugar_normals<<<(P + 255) / 256, 256, 0, st>>>(P, positions, scales, quaternions, campos, out);
    return check_launch("gsr_sugar_normals", false, st);
}

int sugar_normals_backward_impl(int P, const float* positions, const float* scales, const float* quaternions, const float* campos,
                                const float* dL_dnormals, float* dL_dquaternions, cudaStream_t st) {
    if (P < 0 || (P > 0 && (!positions || !scales || !quaternions || !campos || !dL_dnormals || !dL_dquaternions))) {
        set_error("gsr_sugar_normals_backward: bad arguments");
        return GSR_ERR_INVALID;
    }
    if (P == 0) return GSR_OK;
    k_sugar_normals_backward<<<(P + 255) / 256, 256, 0, st>>>(P, positions, scales, quaternions, campos, dL_dnormals, dL_dquaternions);
    return check_launch("gsr_sugar_normals_backward", false, st);
}

int normal_maps_impl(int W, int H, const float* normal_img, const float* depth, const float* c2w, float fx, float fy, float cx, float cy,
                     float* out_normal, float* out_pseudo, cudaStream_t st) {
    if (W <= 0 || H <= 0) { set_error("gsr_normal_maps: bad size"); return GSR_ERR_INVALID; }
    if ((normal_img == nullptr) != (out_normal == nullptr) || (depth == nullptr) != (out_pseudo == nullptr) || (depth && !c2w)) {
        set_error("gsr_normal_maps: inputs and outputs must come in pairs");
        return GSR_ERR_INVALID;
    }
    k_normal_maps<<<dim3((W + 31) / 32, (H + 7) / 8), 256, 0, st>>>(W, H, normal_img, depth, c2w, fx, fy, cx, cy, out_normal, out_pseudo);
    return check_launch("gsr_normal_maps", false, st);
}

int pack_frame_impl(int W, int H, const float* rgb, const float* alpha, const float* depth, const float* normal_hwc, float depth_scale,
                    uint8_t* rgba8, uint8_t* normal8, uint8_t* depth8, cudaStream_t st) {
    if (W <= 0 || H <= 0) { set_error("gsr_pack_frame: bad size"); return GSR_ERR_INVALID; }
    if ((rgba8 && !rgb) || (normal8 && !normal_hwc) || (depth8 && (!depth || !(depth_scale > 0.0f)))) { set_error("gsr_pack_frame: missing input for a requested output"); return GSR_ERR_INVALID; }
    if (rgba8 && ((uintptr_t)rgba8 & 3)) { set_error("gsr_pack_frame: rgba8 must be 4-byte aligned"); return GSR_ERR_INVALID; }
    const size_t HW = (size_t)W * H;
    k_pack_frame<<<(unsigned)((HW + 255) / 256), 256, 0, st>>>(W, H, rgb, alpha, depth, normal_hwc, depth_scale, (uint32_t*)rgba8, normal8, depth8);
    return check_launch("gsr_pack_frame", false, st);
}

}  // namespace gsr
