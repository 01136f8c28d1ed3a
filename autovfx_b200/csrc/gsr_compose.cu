// gsr_b200 — Gaussian parameter activation and the per-frame rigid edit of inserted objects, in one streaming pass.
//
// The reference keeps RAW parameters (log-scales, unnormalised quaternions, logit opacities, SH split into dc / rest) and
// activates them with separate torch ops on every render call (scene/gaussian_model.py:95-115 = "GM/": exp, normalize,
// sigmoid, cat).  For edited scenes its frame loop additionally, per frame and per inserted object, re-reads the object
// .ply, applies transform_gaussians (gaussians_utils.py:88-125 = "GUt/": scale about a pivot, rotate, translate, compose
// quaternions, shift log-scales), concatenates everything into a new model (GUt/:71-84) and deep-copies the whole scene
// (scene_representation.py:357-371).  Here the scene is activated once into resident arrays with spare capacity and each
// object's raw parameters stay resident; one launch of k_compose per (frame, object) writes the transformed + activated
// object straight into the tail of the scene arrays the rasterizer reads.
//
// Arithmetic: one IEEE rounding per reference torch op, in the reference's order (explicit _rn intrinsics, no contraction);
// the [N,3]x[3,3] product and the 4-element norm are summed left to right.
#include "gsr_common.cuh"

namespace gsr {

struct ComposeParams {
    int N, M;                    // Gaussians, SH coefficients per channel in the OUTPUT rows (1 + rest coefficients)
    const float* xyz;            // [N,3]
    const float* f_dc;           // [N,1,3]
    const float* f_rest;         // [N,M-1,3] (ignored when M == 1)
    const float* opacity_raw;    // [N]
    const float* scaling_raw;    // [N,3]
    const float* rotation_raw;   // [N,4]
    float *means3D, *shs, *opacities, *scales, *rotations;
    int has_xform;
    gsr_object_xform x;
};

__global__ void __launch_bounds__(256) k_compose(const ComposeParams p) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n < p.N) {
        float a0 = p.xyz[3 * (size_t)n], a1 = p.xyz[3 * (size_t)n + 1], a2 = p.xyz[3 * (size_t)n + 2];
        float s0 = p.scaling_raw[3 * (size_t)n], s1 = p.scaling_raw[3 * (size_t)n + 1], s2 = p.scaling_raw[3 * (size_t)n + 2];
        float q0 = p.rotation_raw[4 * (size_t)n], q1 = p.rotation_raw[4 * (size_t)n + 1], q2 = p.rotation_raw[4 * (size_t)n + 2],
              q3 = p.rotation_raw[4 * (size_t)n + 3];
        if (p.has_xform) {
            const gsr_object_xform& x = p.x;
            const float c0 = x.initial_center[0], c1 = x.initial_center[1], c2 = x.initial_center[2];
            // scale about the pivot (GUt/:99-103): (xyz - c) * s + c, then log-scale += log(s)
            a0 = __fadd_rn(__fmul_rn(__fsub_rn(a0, c0), x.scaling), c0);
            a1 = __fadd_rn(__fmul_rn(__fsub_rn(a1, c1), x.scaling), c1);
            a2 = __fadd_rn(__fmul_rn(__fsub_rn(a2, c2), x.scaling), c2);
            s0 = __fadd_rn(s0, x.log_scaling); s1 = __fadd_rn(s1, x.log_scaling); s2 = __fadd_rn(s2, x.log_scaling);
            // rotate about the pivot (GUt/:105-109): (xyz - c) @ R^T + c
            a0 = __fsub_rn(a0, c0); a1 = __fsub_rn(a1, c1); a2 = __fsub_rn(a2, c2);
            const float* R = x.rotation;
            const float b0 = __fmaf_rn(a2, R[2], __fmaf_rn(a1, R[1], __fmul_rn(a0, R[0])));
            const float b1 = __fmaf_rn(a2, R[5], __fmaf_rn(a1, R[4], __fmul_rn(a0, R[3])));
            const float b2 = __fmaf_rn(a2, R[8], __fmaf_rn(a1, R[7], __fmul_rn(a0, R[6])));
            // translate (GUt/:112-114): + (center - c)
            a0 = __fadd_rn(__fadd_rn(b0, c0), __fsub_rn(x.center[0], c0));
            a1 = __fadd_rn(__fadd_rn(b1, c1), __fsub_rn(x.center[1], c1));
            a2 = __fadd_rn(__fadd_rn(b2, c2), __fsub_rn(x.center[2], c2));
            // quaternion_multiply(matrix_to_quaternion(R), q) + standardize_quaternion (rotation_utils.py:113-150)
            const float aw = x.quat[0], ax = x.quat[1], ay = x.quat[2], az = x.quat[3];
            const float ow = __fsub_rn(__fsub_rn(__fsub_rn(__fmul_rn(aw, q0), __fmul_rn(ax, q1)), __fmul_rn(ay, q2)), __fmul_rn(az, q3));
            const float ox = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(aw, q1), __fmul_rn(ax, q0)), __fmul_rn(ay, q3)), __fmul_rn(az, q2));
            const float oy = __fadd_rn(__fadd_rn(__fsub_rn(__fmul_rn(aw, q2), __fmul_rn(ax, q3)), __fmul_rn(ay, q0)), __fmul_rn(az, q1));
            const float oz = __fadd_rn(__fsub_rn(__fadd_rn(__fmul_rn(aw, q3), __fmul_rn(ax, q2)), __fmul_rn(ay, q1)), __fmul_rn(az, q0));
            const bool neg = ow < 0.0f;
            q0 = neg ? -ow : ow; q1 = neg ? -ox : ox; q2 = neg ? -oy : oy; q3 = neg ? -oz : oz;
        }
        p.means3D[3 * (size_t)n] = a0; p.means3D[3 * (size_t)n + 1] = a1; p.means3D[3 * (size_t)n + 2] = a2;
        // activations (GM/:95-115): exp, F.normalize (x / max(||x||, 1e-12)), sigmoid = 1 / (1 + exp(-x))
        p.scales[3 * (size_t)n] = expf(s0); p.scales[3 * (size_t)n + 1] = expf(s1); p.scales[3 * (size_t)n + 2] = expf(s2);
        const float qn = fmaxf(__fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q0, q0), __fmul_rn(q1, q1)), __fmul_rn(q2, q2)), __fmul_rn(q3, q3))), 1e-12f);
        p.rotations[4 * (size_t)n] = __fdiv_rn(q0, qn); p.rotations[4 * (size_t)n + 1] = __fdiv_rn(q1, qn);
        p.rotations[4 * (size_t)n + 2] = __fdiv_rn(q2, qn); p.rotations[4 * (size_t)n + 3] = __fdiv_rn(q3, qn);
        p.opacities[n] = sigmoid_rn(p.opacity_raw[n]);
    }
    // SH rows: shs[n] = cat(f_dc[n], f_rest[n]) (GM/:107-110).  The block's 256 rows are copied as one flat, coalesced range.
    const size_t row = (size_t)3 * p.M, rest_row = row - 3;
    const size_t first = (size_t)blockIdx.x * blockDim.x;
    const size_t rows_here = min((size_t)blockDim.x, (size_t)p.N - first);
    const size_t total = rows_here * row;
    float* dst = p.shs + first * row;
    for (size_t j = threadIdx.x; j < total; j += blockDim.x) {
        const size_t r = j / row, k = j - r * row;
        dst[j] = k < 3 ? p.f_dc[(first + r) * 3 + k] : p.f_rest[(first + r) * rest_row + (k - 3)];
    }
}

int compose_impl(int N, int M, const float* xyz, const float* f_dc, const float* f_rest, const float* opacity_raw, const float* scaling_raw,
                 const float* rotation_raw, const gsr_object_xform* xform, float* means3D, float* shs, float* opacities, float* scales,
                 float* rotations, cudaStream_t st) {
    if (N < 0 || M < 1) { set_error("gsr_activate_gaussians: bad sizes N=%d M=%d", N, M); return GSR_ERR_INVALID; }
    if (N == 0) return GSR_OK;
    if (!xyz || !f_dc || (M > 1 && !f_rest) || !opacity_raw || !scaling_raw || !rotation_raw || !means3D || !shs || !opacities || !scales || !rotations) {
        set_error("gsr_activate_gaussians: null pointer");
        return GSR_ERR_INVALID;
    }
    ComposeParams p{};
    p.N = N; p.M = M; p.xyz = xyz; p.f_dc = f_dc; p.f_rest = f_rest; p.opacity_raw = opacity_raw; p.scaling_raw = scaling_raw;
    p.rotation_raw = rotation_raw; p.means3D = means3D; p.shs = shs; p.opacities = opacities; p.scales = scales; p.rotations = rotations;
    p.has_xform = xform != nullptr;
    if (xform) p.x = *xform;
    k_compose<<<(N + 255) / 256, 256, 0, st>>>(p);
    return check_launch("gsr_activate_gaussians", false, st);
}

// ---- backward of the activation (xform = NULL) and of the remapped shading normal (gsr_axis_normals(..., remap01 = 1)) ----------
// Gradients with respect to the activated tensors in, gradients with respect to the raw parameters out.  With s = exp(sigma),
// r = rho / max(||rho||, 1e-12), o = sigmoid(omega) and e = n * 0.5 + 0.5 the shading normal of the smallest axis:
//   d sigma = g_s * s,   d omega = g_o * o (1 - o),   d f_dc | d f_rest = split of g_sh (the inverse of k_compose's cat),
//   d rho   = the Jacobian of F.normalize applied to g_r + (the normal's gradient through build_rotation's own normalisation).
// The axis k and the flip are piecewise constant; axis_pick recomputes the forward's decisions from the same fp32 inputs.
struct ActivateBwdParams {
    int N, M;
    const float* xyz;            // [N,3] (only with g_e)
    const float* campos;         // [3]   (only with g_e)
    const float* opacities;      // [N]   activated
    const float* scales;         // [N,3] activated
    const float* rotations;      // [N,4] activated
    const float* rotation_raw;   // [N,4]
    const float *g_o, *g_s, *g_r;
    const float* g_sh;           // [N,M,3] or null (colours precomputed: no SH gradient)
    const float* g_e;            // [N,3]   or null (the normal image has no gradient)
    float *d_opacity, *d_scaling, *d_rotation, *d_fdc, *d_frest;
};

__global__ void __launch_bounds__(256) k_activate_backward(const ActivateBwdParams p) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n < p.N) {
        const size_t n3 = 3 * (size_t)n, n4 = 4 * (size_t)n;
        const float s0 = p.scales[n3], s1 = p.scales[n3 + 1], s2 = p.scales[n3 + 2];
        p.d_scaling[n3] = p.g_s[n3] * s0; p.d_scaling[n3 + 1] = p.g_s[n3 + 1] * s1; p.d_scaling[n3 + 2] = p.g_s[n3 + 2] * s2;
        const float o = p.opacities[n];
        p.d_opacity[n] = p.g_o[n] * ((1.0f - o) * o);
        const float r0 = p.rotations[n4], r1 = p.rotations[n4 + 1], r2 = p.rotations[n4 + 2], r3 = p.rotations[n4 + 3];
        float b0 = p.g_r[n4], b1 = p.g_r[n4 + 1], b2 = p.g_r[n4 + 2], b3 = p.g_r[n4 + 3];  // d r
        if (p.g_e) {
            const AxisPick a = axis_pick(s0, s1, s2, r0, r1, r2, r3, p.xyz[n3], p.xyz[n3 + 1], p.xyz[n3 + 2], p.campos);
            const float sg = a.flip ? -1.0f : 1.0f;
            const float ia = 1.0f / sqrtf(a.a0 * a.a0 + a.a1 * a.a1 + a.a2 * a.a2);
            const float m0 = sg * a.a0 * ia, m1 = sg * a.a1 * ia, m2 = sg * a.a2 * ia;  // the unit normal
            const float e0 = 0.5f * p.g_e[n3], e1 = 0.5f * p.g_e[n3 + 1], e2 = 0.5f * p.g_e[n3 + 2];
            const float me = m0 * e0 + m1 * e1 + m2 * e2;
            const float c0 = sg * (e0 - m0 * me) * ia, c1 = sg * (e1 - m1 * me) * ia, c2 = sg * (e2 - m2 * me) * ia;  // d (column k)
            const float w = a.w, x = a.x, y = a.y, z = a.z;
            float qw, qx, qy, qz;  // d q^ = (d column / d q^)^T d column
            if (a.k == 0) {         // (1 - 2(y^2 + z^2), 2(xy + wz), 2(xz - wy))
                qw = 2.0f * (z * c1 - y * c2); qx = 2.0f * (y * c1 + z * c2);
                qy = 2.0f * (x * c1 - w * c2) - 4.0f * y * c0; qz = 2.0f * (w * c1 + x * c2) - 4.0f * z * c0;
            } else if (a.k == 1) {  // (2(xy - wz), 1 - 2(x^2 + z^2), 2(yz + wx))
                qw = 2.0f * (x * c2 - z * c0); qx = 2.0f * (y * c0 + w * c2) - 4.0f * x * c1;
                qy = 2.0f * (x * c0 + z * c2); qz = 2.0f * (y * c2 - w * c0) - 4.0f * z * c1;
            } else {                // (2(xz + wy), 2(yz - wx), 1 - 2(x^2 + y^2))
                qw = 2.0f * (y * c0 - x * c1); qx = 2.0f * (z * c0 - w * c1) - 4.0f * x * c2;
                qy = 2.0f * (w * c0 + z * c1) - 4.0f * y * c2; qz = 2.0f * (x * c0 + y * c1);
            }
            const float dq = w * qw + x * qx + y * qy + z * qz, iq = 1.0f / a.qn;  // build_rotation's q / ||q||
            b0 += (qw - w * dq) * iq; b1 += (qx - x * dq) * iq; b2 += (qy - y * dq) * iq; b3 += (qz - z * dq) * iq;
        }
        // F.normalize = rho / clamp_min(||rho||, 1e-12): below the clamp the denominator is a constant
        const float p0 = p.rotation_raw[n4], p1 = p.rotation_raw[n4 + 1], p2 = p.rotation_raw[n4 + 2], p3 = p.rotation_raw[n4 + 3];
        const float pn = __fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(p0, p0), __fmul_rn(p1, p1)), __fmul_rn(p2, p2)), __fmul_rn(p3, p3)));
        if (pn >= 1e-12f) {  // the branch k_compose's fmaxf took
            const float rb = r0 * b0 + r1 * b1 + r2 * b2 + r3 * b3, ip = 1.0f / pn;
            b0 = (b0 - r0 * rb) * ip; b1 = (b1 - r1 * rb) * ip; b2 = (b2 - r2 * rb) * ip; b3 = (b3 - r3 * rb) * ip;
        } else {
            b0 = b0 / 1e-12f; b1 = b1 / 1e-12f; b2 = b2 / 1e-12f; b3 = b3 / 1e-12f;
        }
        p.d_rotation[n4] = b0; p.d_rotation[n4 + 1] = b1; p.d_rotation[n4 + 2] = b2; p.d_rotation[n4 + 3] = b3;
    }
    if (!p.g_sh) return;
    // SH rows: g_sh[n] = cat(d f_dc[n], d f_rest[n]).  The block's 256 rows are split as one flat, coalesced range.
    const size_t row = (size_t)3 * p.M, rest_row = row - 3;
    const size_t first = (size_t)blockIdx.x * blockDim.x;
    const size_t total = min((size_t)blockDim.x, (size_t)p.N - first) * row;
    const float* src = p.g_sh + first * row;
    for (size_t j = threadIdx.x; j < total; j += blockDim.x) {
        const size_t r = j / row, k = j - r * row;
        if (k < 3) p.d_fdc[(first + r) * 3 + k] = src[j];
        else p.d_frest[(first + r) * rest_row + (k - 3)] = src[j];
    }
}

int activate_backward_impl(int N, int M, const float* xyz, const float* campos, const float* opacities, const float* scales,
                           const float* rotations, const float* rotation_raw, const float* g_o, const float* g_s, const float* g_r,
                           const float* g_sh, const float* g_e, float* d_opacity, float* d_scaling, float* d_rotation, float* d_fdc,
                           float* d_frest, cudaStream_t st) {
    if (N < 0 || M < 1) { set_error("gsr_activate_gaussians_backward: bad sizes N=%d M=%d", N, M); return GSR_ERR_INVALID; }
    if (N == 0) return GSR_OK;
    if (!opacities || !scales || !rotations || !rotation_raw || !g_o || !g_s || !g_r || !d_opacity || !d_scaling || !d_rotation ||
        (g_e && (!xyz || !campos)) || (g_sh && (!d_fdc || (M > 1 && !d_frest)))) {
        set_error("gsr_activate_gaussians_backward: null pointer");
        return GSR_ERR_INVALID;
    }
    ActivateBwdParams p{};
    p.N = N; p.M = M; p.xyz = xyz; p.campos = campos; p.opacities = opacities; p.scales = scales; p.rotations = rotations;
    p.rotation_raw = rotation_raw; p.g_o = g_o; p.g_s = g_s; p.g_r = g_r; p.g_sh = g_sh; p.g_e = g_e;
    p.d_opacity = d_opacity; p.d_scaling = d_scaling; p.d_rotation = d_rotation; p.d_fdc = d_fdc; p.d_frest = d_frest;
    k_activate_backward<<<(N + 255) / 256, 256, 0, st>>>(p);
    return check_launch("gsr_activate_gaussians_backward", false, st);
}

}  // namespace gsr
