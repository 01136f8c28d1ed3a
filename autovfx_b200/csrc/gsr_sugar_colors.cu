// gsr_b200 — SuGaR's per-Gaussian colours and opacities, forward and backward, one thread per Gaussian:
//
//   colors[P,3]  = clamp_min(eval_sh(deg, cat(sh_dc, sh_rest)[:, :(deg+1)^2], dirs) + 0.5, 0)   SuGaR.get_points_rgb
//                  (sugar_scene/sugar_model.py:711-755 = "SS/"), eval_sh up to degree 4 (sugar_utils/spherical_harmonics.py:
//                  117-172 = "SH/"), dirs = F.normalize(positions - campos) or the caller's directions (sh_rotations branch)
//   opacities[P] = sigmoid(densities)                                                            SuGaR.strengths (SS/:394-398)
//
// Forward arithmetic: one IEEE rounding per torch op, in the order SH/ writes them (explicit _rn intrinsics, no contraction):
// sums left to right (`r - a + b - c` is ((r - a) + b) - c), `C * y * sh` is (C * y) * sh, Python constants and integer literals
// rounded to float once.  The backward recomputes the forward's basis and clamp decisions from the same fp32 inputs (nothing is
// kept between the two launches) and evaluates the closed-form derivative of each polynomial in plain fp32.
//
// SH rows are 12 M bytes (only 4-byte aligned at M = 25), so a block stages the active coefficients of its 128 rows through shared
// memory as one flat, coalesced range (k_compose's pattern); the backward writes its SH gradient rows back the same way.
#include "gsr_common.cuh"

namespace gsr {

constexpr int SC_THREADS = 128;

struct SugarColorArgs {
    int P, M;
    const float* positions;   // [P,3] (camera-centre mode)
    const float* campos;      // [3]
    const float* directions;  // [P,3] or null
    const float* sh_dc;       // [P,1,3]
    const float* sh_rest;     // [P,M-1,3]
    const float* densities;   // [P]
    float *colors, *opacities;                    // forward outputs (either may be null)
    const float *g_colors, *g_opacities;          // backward inputs (either may be null)
    float *d_sh_dc, *d_sh_rest, *d_dirs, *d_densities;
};

template <int DEG>
struct ShDims {
    static constexpr int K = (DEG + 1) * (DEG + 1);  // active coefficients per channel
    static constexpr int S = (3 * K) | 1;            // staged row stride in floats: odd, so a warp's rows hit distinct banks
};

// the active coefficients of rows [first, first + n): row r of the stage holds coefficient k, channel c at s[r * S + 3 k + c]
template <int DEG>
__device__ __forceinline__ void stage_sh(float* s, const SugarColorArgs& a, int first, int n) {
    constexpr int S = ShDims<DEG>::S, KR = 3 * (ShDims<DEG>::K - 1);
    const float* dc = a.sh_dc + 3 * (size_t)first;
    for (int j = threadIdx.x; j < 3 * n; j += SC_THREADS) s[(j / 3) * S + j % 3] = dc[j];
    if (KR > 0) {
        const size_t RS = 3 * (size_t)(a.M - 1);
        const float* rest = a.sh_rest + (size_t)first * RS;
        for (int j = threadIdx.x; j < n * KR; j += SC_THREADS) {
            const int r = j / KR, k = j - r * KR;
            s[r * S + 3 + k] = rest[r * RS + k];
        }
    }
}

// view direction of Gaussian i; `n` receives the unclamped norm of positions - campos (camera-centre mode only)
__device__ __forceinline__ void view_dir(const SugarColorArgs& a, int i, float& x, float& y, float& z, float& dx, float& dy, float& dz,
                                         float& n) {
    const size_t i3 = 3 * (size_t)i;
    if (a.directions) {
        x = a.directions[i3]; y = a.directions[i3 + 1]; z = a.directions[i3 + 2];
        dx = dy = dz = n = 0.0f;
    } else {
        dx = __fsub_rn(a.positions[i3], a.campos[0]);
        dy = __fsub_rn(a.positions[i3 + 1], a.campos[1]);
        dz = __fsub_rn(a.positions[i3 + 2], a.campos[2]);
        n = normalize3_rn(dx, dy, dz, x, y, z);
    }
}

// b[k]: the factor SH/ multiplies coefficient k by, as torch rounds it.  b[1..3] are C1 y, C1 z, C1 x without the signs of
// `result - C1 * y * sh1 + C1 * z * sh2 - C1 * x * sh3`, which sh_eval applies.
template <int DEG>
__device__ __forceinline__ void sh_basis(float x, float y, float z, float (&b)[ShDims<DEG>::K]) {
    b[0] = SH_C0;
    if (DEG > 0) { b[1] = __fmul_rn(SH_C1, y); b[2] = __fmul_rn(SH_C1, z); b[3] = __fmul_rn(SH_C1, x); }
    if (DEG > 1) {
        const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
        const float xy = __fmul_rn(x, y), yz = __fmul_rn(y, z), xz = __fmul_rn(x, z);
        b[4] = __fmul_rn(SH_C2_0, xy);
        b[5] = __fmul_rn(SH_C2_1, yz);
        b[6] = __fmul_rn(SH_C2_2, __fsub_rn(__fsub_rn(__fmul_rn(2.0f, zz), xx), yy));
        b[7] = __fmul_rn(SH_C2_3, xz);
        b[8] = __fmul_rn(SH_C2_4, __fsub_rn(xx, yy));
        if (DEG > 2) {
            const float xx3 = __fmul_rn(3.0f, xx), yy3 = __fmul_rn(3.0f, yy), zz4_xx_yy = __fsub_rn(__fsub_rn(__fmul_rn(4.0f, zz), xx), yy);
            const float xx_yy = __fsub_rn(xx, yy), xx_3yy = __fsub_rn(xx, yy3), _3xx_yy = __fsub_rn(xx3, yy);
            b[9] = __fmul_rn(__fmul_rn(SH_C3_0, y), _3xx_yy);
            b[10] = __fmul_rn(__fmul_rn(SH_C3_1, xy), z);
            b[11] = __fmul_rn(__fmul_rn(SH_C3_2, y), zz4_xx_yy);
            b[12] = __fmul_rn(__fmul_rn(SH_C3_3, z), __fsub_rn(__fsub_rn(__fmul_rn(2.0f, zz), xx3), yy3));
            b[13] = __fmul_rn(__fmul_rn(SH_C3_4, x), zz4_xx_yy);
            b[14] = __fmul_rn(__fmul_rn(SH_C3_5, z), xx_yy);
            b[15] = __fmul_rn(__fmul_rn(SH_C3_6, x), xx_3yy);
            if (DEG > 3) {
                const float zz7_1 = __fsub_rn(__fmul_rn(7.0f, zz), 1.0f), zz7_3 = __fsub_rn(__fmul_rn(7.0f, zz), 3.0f);
                b[16] = __fmul_rn(__fmul_rn(SH_C4_0, xy), xx_yy);
                b[17] = __fmul_rn(__fmul_rn(SH_C4_1, yz), _3xx_yy);
                b[18] = __fmul_rn(__fmul_rn(SH_C4_2, xy), zz7_1);
                b[19] = __fmul_rn(__fmul_rn(SH_C4_3, yz), zz7_3);
                b[20] = __fmul_rn(SH_C4_4, __fadd_rn(__fmul_rn(zz, __fsub_rn(__fmul_rn(35.0f, zz), 30.0f)), 3.0f));
                b[21] = __fmul_rn(__fmul_rn(SH_C4_5, xz), zz7_3);
                b[22] = __fmul_rn(__fmul_rn(SH_C4_6, xx_yy), zz7_1);
                b[23] = __fmul_rn(__fmul_rn(SH_C4_7, xz), xx_3yy);
                b[24] = __fmul_rn(SH_C4_8, __fsub_rn(__fmul_rn(xx, xx_3yy), __fmul_rn(yy, _3xx_yy)));
            }
        }
    }
}

// eval_sh(...)[c] + 0.5, before the clamp; row = the staged row (coefficient k, channel c at row[3 k + c])
template <int DEG>
__device__ __forceinline__ float sh_pre(const float (&b)[ShDims<DEG>::K], const float* row, int c) {
    float r = __fmul_rn(b[0], row[c]);
    if (DEG > 0) {
        r = __fadd_rn(__fsub_rn(r, __fmul_rn(b[1], row[3 + c])), __fmul_rn(b[2], row[6 + c]));
        r = __fsub_rn(r, __fmul_rn(b[3], row[9 + c]));
#pragma unroll
        for (int k = 4; k < ShDims<DEG>::K; k++) r = __fadd_rn(r, __fmul_rn(b[k], row[3 * k + c]));
    }
    return __fadd_rn(r, 0.5f);
}

template <int DEG>
__global__ void __launch_bounds__(SC_THREADS) k_sugar_colors(const SugarColorArgs a) {
    constexpr int K = ShDims<DEG>::K, S = ShDims<DEG>::S;
    __shared__ float s[SC_THREADS * S];
    const int first = blockIdx.x * SC_THREADS, n = min(SC_THREADS, a.P - first), i = first + threadIdx.x;
    if (a.opacities && i < a.P) a.opacities[i] = sigmoid_rn(a.densities[i]);
    if (!a.colors) return;  // uniform over the block
    stage_sh<DEG>(s, a, first, n);
    __syncthreads();
    if (threadIdx.x >= n) return;
    float x, y, z, dx, dy, dz, nrm;
    view_dir(a, i, x, y, z, dx, dy, dz, nrm);
    float b[K];
    sh_basis<DEG>(x, y, z, b);
    const float* row = s + threadIdx.x * S;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float pre = sh_pre<DEG>(b, row, c);
        a.colors[3 * (size_t)i + c] = pre < 0.0f ? 0.0f : pre;  // clamp_min(., 0): NaN stays NaN, as in torch
    }
}

// Backward.  With g' = dL/dcolors where the pre-clamp colour is >= 0 (torch's clamp_min passes equality) and 0 elsewhere:
//   dL/dsh[k][c] = g'_c * (+-b_k)                 (zero for k beyond the active degree: the slice's backward)
//   dL/ddir      = sum_k w_k grad(b_k),  w_k = +-sum_c g'_c sh[k][c]   (signs: - for k = 1 and 3)
//   camera-centre mode, through F.normalize(d) = d / max(|d|, 1e-12):
//     dL/dpositions = (dL/ddir - u (u . dL/ddir)) / |d|  if |d| >= 1e-12 (u = d / |d|),  else dL/ddir / 1e-12
//   dL/ddensities = (g_o * (1 - o)) * o, o = sigmoid(densities) recomputed.
template <int DEG>
__global__ void __launch_bounds__(SC_THREADS) k_sugar_colors_backward(const SugarColorArgs a) {
    constexpr int K = ShDims<DEG>::K, S = ShDims<DEG>::S;
    __shared__ float s[SC_THREADS * S];
    const int first = blockIdx.x * SC_THREADS, n = min(SC_THREADS, a.P - first), i = first + threadIdx.x;
    if (a.g_opacities && i < a.P) {
        const float o = sigmoid_rn(a.densities[i]);
        a.d_densities[i] = a.g_opacities[i] * (1.0f - o) * o;
    }
    if (!a.g_colors) return;  // uniform over the block
    stage_sh<DEG>(s, a, first, n);
    __syncthreads();
    if (threadIdx.x < n) {
        float x, y, z, dx, dy, dz, nrm;
        view_dir(a, i, x, y, z, dx, dy, dz, nrm);
        float b[K];
        sh_basis<DEG>(x, y, z, b);
        float* row = s + threadIdx.x * S;
        float g[3];
#pragma unroll
        for (int c = 0; c < 3; c++) g[c] = sh_pre<DEG>(b, row, c) >= 0.0f ? a.g_colors[3 * (size_t)i + c] : 0.0f;
        float w[K];
#pragma unroll
        for (int k = 0; k < K; k++) {  // the row is consumed and replaced by its gradient
            const float sg = (k == 1 || k == 3) ? -1.0f : 1.0f;
            w[k] = sg * (g[0] * row[3 * k] + g[1] * row[3 * k + 1] + g[2] * row[3 * k + 2]);
            const float bk = sg * b[k];
            row[3 * k] = g[0] * bk; row[3 * k + 1] = g[1] * bk; row[3 * k + 2] = g[2] * bk;
        }
        float gx = 0.0f, gy = 0.0f, gz = 0.0f;
        if (DEG > 0) { gx = w[3] * SH_C1; gy = w[1] * SH_C1; gz = w[2] * SH_C1; }
        if (DEG > 1) {
            const float xx = x * x, yy = y * y, zz = z * z;
            gx += w[4] * SH_C2_0 * y - w[6] * SH_C2_2 * 2.0f * x + w[7] * SH_C2_3 * z + w[8] * SH_C2_4 * 2.0f * x;
            gy += w[4] * SH_C2_0 * x + w[5] * SH_C2_1 * z - w[6] * SH_C2_2 * 2.0f * y - w[8] * SH_C2_4 * 2.0f * y;
            gz += w[5] * SH_C2_1 * y + w[6] * SH_C2_2 * 4.0f * z + w[7] * SH_C2_3 * x;
            if (DEG > 2) {
                const float xy = x * y, yz = y * z, xz = x * z;
                gx += w[9] * SH_C3_0 * 6.0f * xy + w[10] * SH_C3_1 * yz - w[11] * SH_C3_2 * 2.0f * xy - w[12] * SH_C3_3 * 6.0f * xz +
                      w[13] * SH_C3_4 * (4.0f * zz - 3.0f * xx - yy) + w[14] * SH_C3_5 * 2.0f * xz + w[15] * SH_C3_6 * (3.0f * xx - 3.0f * yy);
                gy += w[9] * SH_C3_0 * (3.0f * xx - 3.0f * yy) + w[10] * SH_C3_1 * xz + w[11] * SH_C3_2 * (4.0f * zz - xx - 3.0f * yy) -
                      w[12] * SH_C3_3 * 6.0f * yz - w[13] * SH_C3_4 * 2.0f * xy - w[14] * SH_C3_5 * 2.0f * yz - w[15] * SH_C3_6 * 6.0f * xy;
                gz += w[10] * SH_C3_1 * xy + w[11] * SH_C3_2 * 8.0f * yz + w[12] * SH_C3_3 * (6.0f * zz - 3.0f * xx - 3.0f * yy) +
                      w[13] * SH_C3_4 * 8.0f * xz + w[14] * SH_C3_5 * (xx - yy);
                if (DEG > 3) {
                    const float xyz = xy * z, zz7_1 = 7.0f * zz - 1.0f, zz7_3 = 7.0f * zz - 3.0f, zz21_3 = 21.0f * zz - 3.0f;
                    gx += w[16] * SH_C4_0 * (3.0f * xx * y - yy * y) + w[17] * SH_C4_1 * 6.0f * xyz + w[18] * SH_C4_2 * y * zz7_1 +
                          w[21] * SH_C4_5 * z * zz7_3 + w[22] * SH_C4_6 * 2.0f * x * zz7_1 + w[23] * SH_C4_7 * z * (3.0f * xx - 3.0f * yy) +
                          w[24] * SH_C4_8 * (4.0f * xx * x - 12.0f * x * yy);
                    gy += w[16] * SH_C4_0 * (xx * x - 3.0f * x * yy) + w[17] * SH_C4_1 * (3.0f * xx * z - 3.0f * yy * z) +
                          w[18] * SH_C4_2 * x * zz7_1 + w[19] * SH_C4_3 * z * zz7_3 - w[22] * SH_C4_6 * 2.0f * y * zz7_1 -
                          w[23] * SH_C4_7 * 6.0f * xyz + w[24] * SH_C4_8 * (4.0f * yy * y - 12.0f * xx * y);
                    gz += w[17] * SH_C4_1 * (3.0f * xx * y - yy * y) + w[18] * SH_C4_2 * 14.0f * xyz + w[19] * SH_C4_3 * y * zz21_3 +
                          w[20] * SH_C4_4 * (140.0f * zz * z - 60.0f * z) + w[21] * SH_C4_5 * x * zz21_3 +
                          w[22] * SH_C4_6 * 14.0f * z * (xx - yy) + w[23] * SH_C4_7 * x * (xx - 3.0f * yy);
                }
            }
        }
        if (!a.directions) {
            if (nrm >= 1e-12f) {  // the branch normalize3_rn's clamp did not take
                const float inv = 1.0f / nrm, ux = dx * inv, uy = dy * inv, uz = dz * inv, ug = ux * gx + uy * gy + uz * gz;
                gx = (gx - ux * ug) * inv; gy = (gy - uy * ug) * inv; gz = (gz - uz * ug) * inv;
            } else {
                gx = gx / 1e-12f; gy = gy / 1e-12f; gz = gz / 1e-12f;
            }
        }
        a.d_dirs[3 * (size_t)i] = gx; a.d_dirs[3 * (size_t)i + 1] = gy; a.d_dirs[3 * (size_t)i + 2] = gz;
    }
    __syncthreads();
    // the block's gradient rows, coalesced; coefficients beyond the active degree get zeros
    constexpr int KR = 3 * (K - 1);
    float* ddc = a.d_sh_dc + 3 * (size_t)first;
    for (int j = threadIdx.x; j < 3 * n; j += SC_THREADS) ddc[j] = s[(j / 3) * S + j % 3];
    if (a.M > 1) {
        const int RS = 3 * (a.M - 1);
        float* drest = a.d_sh_rest + (size_t)first * RS;
        for (int j = threadIdx.x; j < n * RS; j += SC_THREADS) {
            const int r = j / RS, k = j - r * RS;
            drest[j] = k < KR ? s[r * S + 3 + k] : 0.0f;
        }
    }
}

static bool sugar_color_args_ok(const char* what, int P, int M, int deg, const SugarColorArgs& a, bool need_sh, bool need_dens) {
    if (P < 0 || deg < 0 || deg > 4 || M < (deg + 1) * (deg + 1)) {
        set_error("%s: bad sizes P=%d M=%d deg=%d (deg must be 0..4 and M >= (deg+1)^2)", what, P, M, deg);
        return false;
    }
    if (P == 0) return true;
    if ((need_sh && (!a.sh_dc || (M > 1 && !a.sh_rest) || (!a.directions && (!a.positions || !a.campos)))) || (need_dens && !a.densities)) {
        set_error("%s: null pointer", what);
        return false;
    }
    return true;
}

#define GSR_SC_LAUNCH(KERNEL)                                                                                     \
    switch (deg) {                                                                                               \
        case 0: KERNEL<0><<<(P + SC_THREADS - 1) / SC_THREADS, SC_THREADS, 0, st>>>(a); break;                   \
        case 1: KERNEL<1><<<(P + SC_THREADS - 1) / SC_THREADS, SC_THREADS, 0, st>>>(a); break;                   \
        case 2: KERNEL<2><<<(P + SC_THREADS - 1) / SC_THREADS, SC_THREADS, 0, st>>>(a); break;                   \
        case 3: KERNEL<3><<<(P + SC_THREADS - 1) / SC_THREADS, SC_THREADS, 0, st>>>(a); break;                   \
        default: KERNEL<4><<<(P + SC_THREADS - 1) / SC_THREADS, SC_THREADS, 0, st>>>(a); break;                  \
    }

int sugar_colors_impl(int P, int M, int deg, const float* positions, const float* campos, const float* directions, const float* sh_dc,
                      const float* sh_rest, const float* densities, float* out_colors, float* out_opacities, cudaStream_t st) {
    SugarColorArgs a{};
    a.P = P; a.M = M; a.positions = positions; a.campos = campos; a.directions = directions; a.sh_dc = sh_dc; a.sh_rest = sh_rest;
    a.densities = densities; a.colors = out_colors; a.opacities = out_opacities;
    if (!sugar_color_args_ok("gsr_sugar_colors", P, M, deg, a, out_colors != nullptr, out_opacities != nullptr)) return GSR_ERR_INVALID;
    if (P == 0 || (!out_colors && !out_opacities)) return GSR_OK;
    GSR_SC_LAUNCH(k_sugar_colors)
    return check_launch("gsr_sugar_colors", false, st);
}

int sugar_colors_backward_impl(int P, int M, int deg, const float* positions, const float* campos, const float* directions,
                               const float* sh_dc, const float* sh_rest, const float* densities, const float* dL_dcolors,
                               const float* dL_dopacities, float* dL_dsh_dc, float* dL_dsh_rest, float* dL_dpositions, float* dL_ddensities,
                               cudaStream_t st) {
    SugarColorArgs a{};
    a.P = P; a.M = M; a.positions = positions; a.campos = campos; a.directions = directions; a.sh_dc = sh_dc; a.sh_rest = sh_rest;
    a.densities = densities; a.g_colors = dL_dcolors; a.g_opacities = dL_dopacities; a.d_sh_dc = dL_dsh_dc; a.d_sh_rest = dL_dsh_rest;
    a.d_dirs = dL_dpositions; a.d_densities = dL_ddensities;
    if (!sugar_color_args_ok("gsr_sugar_colors_backward", P, M, deg, a, dL_dcolors != nullptr, dL_dopacities != nullptr)) return GSR_ERR_INVALID;
    if (P > 0 && ((dL_dcolors && (!dL_dsh_dc || (M > 1 && !dL_dsh_rest) || !dL_dpositions)) || (dL_dopacities && !dL_ddensities))) {
        set_error("gsr_sugar_colors_backward: null output pointer");
        return GSR_ERR_INVALID;
    }
    if (P == 0 || (!dL_dcolors && !dL_dopacities)) return GSR_OK;
    GSR_SC_LAUNCH(k_sugar_colors_backward)
    return check_launch("gsr_sugar_colors_backward", false, st);
}

#undef GSR_SC_LAUNCH

}  // namespace gsr
