// gsr_b200 training objective: the per-step loss terms of every trainer ("LU/" = sugar/gaussian_splatting/utils/loss_utils.py),
// forward and backward.
//
//   k_photo_fwd        l1_loss (LU/:17-18) and ssim (LU/:33-62) of two [B,C,H,W] images given by element strides.  One CTA per
//                      32x32 output tile and channel plane: the tile and its 5-pixel halo of both images are staged in shared
//                      memory, the five moment maps (mu_x, mu_y, E[x^2], E[y^2], E[xy]) come from a horizontal then a vertical
//                      11-tap pass with the separable weights, then the SSIM map in torch's operation order.  Per-CTA partial sums
//                      of |x - y| and SSIM; for a backward also the three per-pixel maps dS/d(mu_x, E[x^2], E[xy]).
//   k_photo_bwd        dL/dx = g_ssim/N * (conv(g_mu) + 2x conv(g_xx) + y conv(g_xy)) + g_l1/N * sign(x - y): the window is
//                      symmetric, so the adjoint of the zero-padded correlation is the same correlation over the stored maps.
//                      One thread writes each pixel; no atomics.
//   k_normal_fwd/bwd   normal_loss (LU/:118-132): F.normalize of both inputs (norm clamped at 1e-12), the optional depth mask
//                      selected on the device, mean |n - g| + 0.1 * (-mean n.g); the backward through normalize's Jacobian.
//   k_aniso_fwd/bwd    anisotropic_loss (LU/:159-168): mean(clamp_min(max / (min + 1e-6), r) - r); the backward sends the max's
//                      and the min's gradient to the first extreme index, as torch's max(dim) / min(dim) return it on ties.
//   k_depth_sums/fwd/bwd  depth_loss (LU/:65-111): the masked sums of compute_scale_and_shift in double, the 2x2 solve in one
//                      thread of the finalize (x0, x1 stay on the device), then mean w exp(-p/s) (x0 p + x1 - d)^2 and its gradient.
//   k_opacity_fwd/bwd  opacity_loss (LU/:143-147) and sparsity_loss (LU/:149-157).
//   k_entropy_fwd/bwd  the coarse trainers' entropy term over the Gaussians with radii > 0, the visible count on the device.
//   k_density_fwd/bwd  coarse_density's 'density' SDF estimation loss, |d - exp(-s^2 / (2 beta^2))| or its square.
//   k_loss_finalize    every mean: per-CTA partials, then one CTA sums them in double in a fixed order, so a value is
//                      bit-identical from call to call.
//
// Elementwise arithmetic uses _rn intrinsics in torch's operation order so nvcc contracts nothing across torch's roundings; the
// window sums are not in cuDNN's order (see INTEGRATION.md).
#include "gsr_common.cuh"

namespace gsr {

namespace {

constexpr int PT = 32;              // output tile edge
constexpr int PR = 5;               // window radius
constexpr int PS = PT + 2 * PR;     // staged edge
constexpr int PB = 256;             // threads per photometric CTA
constexpr int RB = 256;             // threads per reduction CTA
constexpr int RMAX_BLOCKS = 1024;   // reduction CTAs of the normal and anisotropic terms
constexpr float SSIM_C1 = 0.01f * 0.01f;
constexpr float SSIM_C2 = 0.03f * 0.03f;

struct Window { float w[2 * PR + 1]; };
struct Strides { int64_t b, c, y, x; };

size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

// fixed-order block sum of K values per thread (warp butterflies, then warps in order); the result is valid in thread 0
template <int K, typename T>
__device__ __forceinline__ void block_sum(T (&v)[K], T (*red)[PB / 32]) {
#pragma unroll
    for (int k = 0; k < K; ++k)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(GSR_FULL, v[k], o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < K; ++k) red[k][warp] = v[k];
    __syncthreads();
    if (threadIdx.x == 0)
#pragma unroll
        for (int k = 0; k < K; ++k) {
            T s = red[k][0];
            for (int w = 1; w < (int)(blockDim.x >> 5); ++w) s += red[k][w];
            v[k] = s;
        }
}

__device__ __forceinline__ float load_px(const float* p, const Strides& s, int b, int c, int y, int x, int H, int W) {
    if (y < 0 || y >= H || x < 0 || x >= W) return 0.0f;
    return p[(int64_t)b * s.b + (int64_t)c * s.c + (int64_t)y * s.y + (int64_t)x * s.x];
}

struct PhotoArgs {
    int B, C, H, W, l1, store;
    const float* x;
    const float* y;
    Strides sx, sy;
    Window win;
    float* partials;   // [blocks][2]: sum |x - y|, sum SSIM
    float* maps;       // [3][B*C*H*W]: g_mu, g_xx, g_xy
};

__global__ void __launch_bounds__(PB) k_photo_fwd(const __grid_constant__ PhotoArgs a) {
    __shared__ float xs[PS][PS], ys[PS][PS];
    __shared__ float hs[5][PS][PT];
    __shared__ float red[2][PB / 32];
    const int plane = blockIdx.z, b = plane / a.C, c = plane % a.C;
    const int x0 = blockIdx.x * PT - PR, y0 = blockIdx.y * PT - PR;
    for (int i = threadIdx.x; i < PS * PS; i += PB) {
        const int r = i / PS, q = i % PS;
        xs[r][q] = load_px(a.x, a.sx, b, c, y0 + r, x0 + q, a.H, a.W);
        ys[r][q] = load_px(a.y, a.sy, b, c, y0 + r, x0 + q, a.H, a.W);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < PS * PT; i += PB) {
        const int r = i / PT, q = i % PT;
        float m1 = 0.f, m2 = 0.f, e11 = 0.f, e22 = 0.f, e12 = 0.f;
#pragma unroll
        for (int k = 0; k < 2 * PR + 1; ++k) {
            const float w = a.win.w[k], u = xs[r][q + k], v = ys[r][q + k];
            m1 = __fmaf_rn(w, u, m1);
            m2 = __fmaf_rn(w, v, m2);
            e11 = __fmaf_rn(w, __fmul_rn(u, u), e11);
            e22 = __fmaf_rn(w, __fmul_rn(v, v), e22);
            e12 = __fmaf_rn(w, __fmul_rn(u, v), e12);
        }
        hs[0][r][q] = m1; hs[1][r][q] = m2; hs[2][r][q] = e11; hs[3][r][q] = e22; hs[4][r][q] = e12;
    }
    __syncthreads();
    const int64_t HW = (int64_t)a.H * a.W, N = HW * a.B * a.C;
    float acc[2] = {0.f, 0.f};
    for (int i = threadIdx.x; i < PT * PT; i += PB) {
        const int r = i / PT, q = i % PT;
        const int gy = y0 + PR + r, gx = x0 + PR + q;
        if (gy >= a.H || gx >= a.W) continue;
        float m[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int k = 0; k < 2 * PR + 1; ++k)
#pragma unroll
            for (int j = 0; j < 5; ++j) m[j] = __fmaf_rn(a.win.w[k], hs[j][r + k][q], m[j]);
        // ssim's own expressions (LU/:43-58), one rounding per torch op
        const float mu1 = m[0], mu2 = m[1];
        const float mu1_sq = __fmul_rn(mu1, mu1), mu2_sq = __fmul_rn(mu2, mu2), mu1_mu2 = __fmul_rn(mu1, mu2);
        const float s1 = __fsub_rn(m[2], mu1_sq), s2 = __fsub_rn(m[3], mu2_sq), s12 = __fsub_rn(m[4], mu1_mu2);
        const float A = __fadd_rn(__fmul_rn(2.0f, mu1_mu2), SSIM_C1), Bv = __fadd_rn(__fmul_rn(2.0f, s12), SSIM_C2);
        const float Cv = __fadd_rn(__fadd_rn(mu1_sq, mu2_sq), SSIM_C1), D = __fadd_rn(__fadd_rn(s1, s2), SSIM_C2);
        const float CD = __fmul_rn(Cv, D);
        const float S = __fdiv_rn(__fmul_rn(A, Bv), CD);
        acc[1] += S;
        const float u = xs[PR + r][PR + q], v = ys[PR + r][PR + q];
        if (a.l1) acc[0] += fabsf(__fsub_rn(u, v));
        if (a.store) {
            // dS/dmu_x = 2 mu_y (B - A) / (C D) + 2 mu_x S (1/D - 1/C), dS/dE[x^2] = -S / D, dS/dE[xy] = 2 A / (C D)
            const int64_t o = (int64_t)plane * HW + (int64_t)gy * a.W + gx;
            a.maps[o] = 2.0f * mu2 * (Bv - A) / CD + 2.0f * mu1 * S * (1.0f / D - 1.0f / Cv);
            a.maps[N + o] = -S / D;
            a.maps[2 * N + o] = 2.0f * A / CD;
        }
    }
    block_sum<2>(acc, red);
    if (threadIdx.x == 0) {
        const int64_t blk = ((int64_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
        a.partials[2 * blk] = acc[0];
        a.partials[2 * blk + 1] = acc[1];
    }
}

struct PhotoBwdArgs {
    int B, C, H, W;
    const float* x;
    const float* y;
    Strides sx, sy;
    Window win;
    const float* maps;
    const float* g_l1;
    const float* g_ssim;
    float* dx;          // contiguous [B,C,H,W]
};

__global__ void __launch_bounds__(PB) k_photo_bwd(const __grid_constant__ PhotoBwdArgs a) {
    __shared__ float ms[3][PS][PS];
    __shared__ float hs[3][PS][PT];
    const int plane = blockIdx.z, b = plane / a.C, c = plane % a.C;
    const int x0 = blockIdx.x * PT - PR, y0 = blockIdx.y * PT - PR;
    const int64_t HW = (int64_t)a.H * a.W, N = HW * a.B * a.C;
    const float* mp = a.maps + (int64_t)plane * HW;
    for (int i = threadIdx.x; i < PS * PS; i += PB) {
        const int r = i / PS, q = i % PS, gy = y0 + r, gx = x0 + q;
        const bool in = gy >= 0 && gy < a.H && gx >= 0 && gx < a.W;
        const int64_t o = (int64_t)gy * a.W + gx;
#pragma unroll
        for (int j = 0; j < 3; ++j) ms[j][r][q] = in ? mp[j * N + o] : 0.0f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < PS * PT; i += PB) {
        const int r = i / PT, q = i % PT;
        float h[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int k = 0; k < 2 * PR + 1; ++k)
#pragma unroll
            for (int j = 0; j < 3; ++j) h[j] = __fmaf_rn(a.win.w[k], ms[j][r][q + k], h[j]);
#pragma unroll
        for (int j = 0; j < 3; ++j) hs[j][r][q] = h[j];
    }
    __syncthreads();
    const float inv_n = (float)(1.0 / (double)N);
    const float gs = a.g_ssim ? __fmul_rn(*a.g_ssim, inv_n) : 0.0f;
    const float gl = a.g_l1 ? __fmul_rn(*a.g_l1, inv_n) : 0.0f;
    for (int i = threadIdx.x; i < PT * PT; i += PB) {
        const int r = i / PT, q = i % PT;
        const int gy = y0 + PR + r, gx = x0 + PR + q;
        if (gy >= a.H || gx >= a.W) continue;
        float cm[3] = {0.f, 0.f, 0.f};
#pragma unroll
        for (int k = 0; k < 2 * PR + 1; ++k)
#pragma unroll
            for (int j = 0; j < 3; ++j) cm[j] = __fmaf_rn(a.win.w[k], hs[j][r + k][q], cm[j]);
        const float u = load_px(a.x, a.sx, b, c, gy, gx, a.H, a.W), v = load_px(a.y, a.sy, b, c, gy, gx, a.H, a.W);
        float g = gs * (cm[0] + 2.0f * u * cm[1] + v * cm[2]);
        if (a.g_l1) {
            const float d = u - v;  // torch's abs backward: sign(d), 0 at d == 0, NaN stays NaN
            g += gl * (d > 0.f ? 1.0f : d < 0.f ? -1.0f : d == 0.f ? 0.0f : d);
        }
        a.dx[(int64_t)plane * HW + (int64_t)gy * a.W + gx] = g;
    }
}

// F.normalize(v, dim=-1): v / max(|v|, 1e-12), |v| as torch's norm (sqrt of the sum of squares)
__device__ __forceinline__ float norm3(float x, float y, float z) {
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}

struct NormalArgs {
    int64_t n;
    const float* pred;
    int64_t p_sp, p_sc;
    const float* gt;
    int64_t g_sp, g_sc;
    const float* depth;  // NULL: every pixel
    int64_t d_sp;
    float scene_scale;
};

__device__ __forceinline__ bool normal_selected(const NormalArgs& a, int64_t i) {
    if (!a.depth) return true;
    const float d = a.depth[i * a.d_sp];
    return d > 0.0f && d < a.scene_scale;
}

__device__ __forceinline__ void normal_load(const NormalArgs& a, int64_t i, float (&n)[3], float (&g)[3], float& len) {
    float v[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        v[k] = a.pred[i * a.p_sp + k * a.p_sc];
        g[k] = a.gt[i * a.g_sp + k * a.g_sc];
    }
    len = norm3(v[0], v[1], v[2]);
    const float dn = fmaxf(len, 1e-12f), dg = fmaxf(norm3(g[0], g[1], g[2]), 1e-12f);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        n[k] = __fdiv_rn(v[k], dn);
        g[k] = __fdiv_rn(g[k], dg);
    }
}

__global__ void __launch_bounds__(RB) k_normal_fwd(const NormalArgs a, float* partials) {
    __shared__ float red[3][PB / 32];
    float acc[3] = {0.f, 0.f, 0.f};  // sum |n - g|, sum n.g, selected pixels
    for (int64_t i = (int64_t)blockIdx.x * RB + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * RB) {
        if (!normal_selected(a, i)) continue;
        float n[3], g[3], len;
        normal_load(a, i, n, g, len);
        acc[0] += fabsf(__fsub_rn(n[0], g[0])) + fabsf(__fsub_rn(n[1], g[1])) + fabsf(__fsub_rn(n[2], g[2]));
        acc[1] += __fadd_rn(__fadd_rn(__fmul_rn(n[0], g[0]), __fmul_rn(n[1], g[1])), __fmul_rn(n[2], g[2]));
        acc[2] += 1.0f;
    }
    block_sum<3>(acc, red);
    if (threadIdx.x == 0)
        for (int k = 0; k < 3; ++k) partials[4 * blockIdx.x + k] = acc[k];
}

__global__ void __launch_bounds__(RB) k_normal_bwd(const NormalArgs a, const double* totals, const float* g_out, float* d_pred) {
    const double cnt = totals[2];
    const float g = *g_out;
    const float g_l1 = (float)((double)g / (3.0 * cnt)), g_cos = (float)((double)__fmul_rn(0.1f, g) / cnt);
    for (int64_t i = (int64_t)blockIdx.x * RB + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * RB) {
        float d[3] = {0.f, 0.f, 0.f};
        if (normal_selected(a, i)) {
            float v[3], n[3], gt[3], len;
            normal_load(a, i, n, gt, len);
            float dn[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const float e = n[k] - gt[k];
                dn[k] = g_l1 * (e > 0.f ? 1.0f : e < 0.f ? -1.0f : e == 0.f ? 0.0f : e) - g_cos * gt[k];
                v[k] = a.pred[i * a.p_sp + k * a.p_sc];
            }
            // n = v / c with c = max(|v|, 1e-12): dv = dn / c - (dn.v / c^2) * (|v| >= 1e-12 ? v / |v| : 0)
            const float c = fmaxf(len, 1e-12f);
            const float s = (dn[0] * v[0] + dn[1] * v[1] + dn[2] * v[2]) / (c * c);
            const bool pass = len >= 1e-12f;
#pragma unroll
            for (int k = 0; k < 3; ++k) d[k] = dn[k] / c - (pass ? s * (v[k] / len) : 0.0f);
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) d_pred[3 * i + k] = d[k];
    }
}

// the first maximal / minimal index, NaN first (torch's max(dim) / min(dim) on an H100: tests/test_gpu_losses.py pins it)
__device__ __forceinline__ void extremes3(const float* s, int& imax, int& imin) {
    imax = imin = 0;
    for (int k = 1; k < 3; ++k) {
        if (s[imax] == s[imax] && (s[k] > s[imax] || s[k] != s[k])) imax = k;
        if (s[imin] == s[imin] && (s[k] < s[imin] || s[k] != s[k])) imin = k;
    }
}

__global__ void __launch_bounds__(RB) k_aniso_fwd(int64_t P, const float* __restrict__ scales, float r, float* partials) {
    __shared__ float red[1][PB / 32];
    float acc[1] = {0.f};
    for (int64_t i = (int64_t)blockIdx.x * RB + threadIdx.x; i < P; i += (int64_t)gridDim.x * RB) {
        const float s[3] = {scales[3 * i], scales[3 * i + 1], scales[3 * i + 2]};
        int imax, imin;
        extremes3(s, imax, imin);
        const float q = __fdiv_rn(s[imax], __fadd_rn(s[imin], 1e-6f));
        acc[0] += __fsub_rn(q < r ? r : q, r);  // clamp_min keeps NaN
    }
    block_sum<1>(acc, red);
    if (threadIdx.x == 0) partials[4 * blockIdx.x] = acc[0];
}

__global__ void __launch_bounds__(RB) k_aniso_bwd(int64_t P, const float* __restrict__ scales, float r, const float* g_out,
                                                  float* __restrict__ d_scales) {
    const float g = (float)((double)*g_out / (double)P);
    for (int64_t i = (int64_t)blockIdx.x * RB + threadIdx.x; i < P; i += (int64_t)gridDim.x * RB) {
        const float s[3] = {scales[3 * i], scales[3 * i + 1], scales[3 * i + 2]};
        int imax, imin;
        extremes3(s, imax, imin);
        const float den = __fadd_rn(s[imin], 1e-6f);
        const float q = __fdiv_rn(s[imax], den);
        float d[3] = {0.f, 0.f, 0.f};
        if (q >= r) {  // clamp_min passes the gradient where input >= min (equality included)
            d[imax] += g / den;
            d[imin] += -g * s[imax] / (den * den);
        }
        for (int k = 0; k < 3; ++k) d_scales[3 * i + k] = d[k];
    }
}

// torch's abs backward: sign(e), 0 at e == 0, NaN stays NaN
__device__ __forceinline__ float sgn(float e) { return e > 0.f ? 1.0f : e < 0.f ? -1.0f : e == 0.f ? 0.0f : e; }

// ---- depth_loss: d = gt / 25 and -p / scene_scale as torch divides a float32 CUDA tensor by a Python number, x * float32(1 / b)
constexpr float DEPTH_INV_25 = 1.0f / 25.0f;
constexpr int RMAX_BLOCKS64 = 256;  // CTAs of the double-partial reduction: 256 x 8 doubles fill GSR_LOSS_REDUCE_BYTES - 256

struct DepthArgs {
    int64_t n;
    const float* p;
    int64_t p_s;
    const float* gt;
    int64_t g_s;
    float inv_scale;
};

__global__ void __launch_bounds__(RB) k_depth_sums(const DepthArgs a, double* partials) {
    __shared__ double red[5][PB / 32];
    double acc[5] = {0.0, 0.0, 0.0, 0.0, 0.0};  // sum p^2, sum p, count, sum p d, sum d over d > 0
    for (int64_t i = (int64_t)blockIdx.x * RB + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * RB) {
        const float d = __fmul_rn(a.gt[i * a.g_s], DEPTH_INV_25);
        if (!(d > 0.0f)) continue;
        const float p = a.p[i * a.p_s];
        acc[0] += (double)__fmul_rn(p, p);
        acc[1] += (double)p;
        acc[2] += 1.0;
        acc[3] += (double)__fmul_rn(p, d);
        acc[4] += (double)d;
    }
    block_sum<5>(acc, red);
    if (threadIdx.x == 0)
        for (int k = 0; k < 5; ++k) partials[8 * blockIdx.x + k] = acc[k];
}

// r = x0 p + x1 - d and we = weight * exp(-p / scene_scale), in the reference's operation order
__device__ __forceinline__ float depth_residual(const DepthArgs& a, int64_t i, float x0, float x1, float& we) {
    const float p = a.p[i * a.p_s], d = __fmul_rn(a.gt[i * a.g_s], DEPTH_INV_25);
    we = __fmul_rn(d > 0.0f ? 1.0f : 0.0f, expf(__fmul_rn(-p, a.inv_scale)));
    return __fsub_rn(__fadd_rn(__fmul_rn(x0, p), x1), d);
}

__global__ void __launch_bounds__(RB) k_depth_fwd(const DepthArgs a, const float* x, float* partials) {
    __shared__ float red[1][PB / 32];
    const float x0 = x[0], x1 = x[1];
    float acc[1] = {0.f};
    for (int64_t i = (int64_t)blockIdx.x * RB + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * RB) {
        float we;
        const float r = depth_residual(a, i, x0, x1, we);
        acc[0] += __fmul_rn(we, __fmul_rn(r, r));
    }
    block_sum<1>(acc, red);
    if (threadIdx.x == 0) partials[4 * blockIdx.x] = acc[0];
}

// d p = (g / n) * we * (2 r) * x0: the scale, the shift and the exp factor are detached in the reference
__global__ void __launch_bounds__(RB) k_depth_bwd(const DepthArgs a, const float* x, const float* g_out, float* __restrict__ d_p) {
    const float x0 = x[0], x1 = x[1];
    const float g = (float)((double)*g_out / (double)a.n);
    for (int64_t i = (int64_t)blockIdx.x * RB + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * RB) {
        float we;
        const float r = depth_residual(a, i, x0, x1, we);
        d_p[i] = __fmul_rn(__fmul_rn(__fmul_rn(g, we), __fmul_rn(2.0f, r)), x0);
    }
}

// ---- opacity_loss: mean(x); sparsity_loss: mean(log c + log(1 - c)), c = clamp(x, 1e-3, 1 - 1e-3) with float32 bounds
constexpr float SPARSE_LO = 1e-3f;
constexpr float SPARSE_HI = (float)(1.0 - 1e-3);

__device__ __forceinline__ float sparsity_term(float x) {
    const float c = x != x ? x : fminf(fmaxf(x, SPARSE_LO), SPARSE_HI);  // clamp keeps NaN
    return __fadd_rn(logf(c), logf(__fsub_rn(1.0f, c)));
}

template <bool SPARSE>
__global__ void __launch_bounds__(RB) k_opacity_fwd(int64_t n, const float* __restrict__ x, int64_t xs, float* partials) {
    __shared__ float red[1][PB / 32];
    float acc[1] = {0.f};
    for (int64_t i = (int64_t)blockIdx.x * RB + threadIdx.x; i < n; i += (int64_t)gridDim.x * RB) {
        const float v = x[i * xs];
        acc[0] += SPARSE ? sparsity_term(v) : v;
    }
    block_sum<1>(acc, red);
    if (threadIdx.x == 0) partials[4 * blockIdx.x] = acc[0];
}

// opacity: dx = g / n; sparsity: g / c - g / (1 - c) where 1e-3 <= x <= 1 - 1e-3 (clamp's backward passes both bounds), else 0
template <bool SPARSE>
__global__ void __launch_bounds__(RB) k_opacity_bwd(int64_t n, const float* __restrict__ x, int64_t xs, const float* g_out,
                                                    float* __restrict__ dx) {
    const float g = (float)((double)*g_out / (double)n);
    for (int64_t i = (int64_t)blockIdx.x * RB + threadIdx.x; i < n; i += (int64_t)gridDim.x * RB) {
        if (!SPARSE) {
            dx[i] = g;
            continue;
        }
        const float c = x[i * xs];
        dx[i] = c >= SPARSE_LO && c <= SPARSE_HI ? __fsub_rn(__fdiv_rn(g, c), __fdiv_rn(g, __fsub_rn(1.0f, c))) : 0.0f;
    }
}

// ---- entropy: -o log(o + 1e-10) - (1 - o) log(1 - o + 1e-10) over the Gaussians with radii > 0
constexpr float ENTROPY_EPS = 1e-10f;

__global__ void __launch_bounds__(RB) k_entropy_fwd(int64_t P, const float* __restrict__ o, int64_t os, const int32_t* __restrict__ radii,
                                                    int64_t rs, float* partials) {
    __shared__ float red[2][PB / 32];
    float acc[2] = {0.f, 0.f};  // sum of the terms, visible count
    for (int64_t i = (int64_t)blockIdx.x * RB + threadIdx.x; i < P; i += (int64_t)gridDim.x * RB) {
        if (radii[i * rs] <= 0) continue;
        const float v = o[i * os], u = __fsub_rn(1.0f, v);
        acc[0] += __fsub_rn(__fmul_rn(-v, logf(__fadd_rn(v, ENTROPY_EPS))), __fmul_rn(u, logf(__fadd_rn(u, ENTROPY_EPS))));
        acc[1] += 1.0f;
    }
    block_sum<2>(acc, red);
    if (threadIdx.x == 0) {
        partials[4 * blockIdx.x] = acc[0];
        partials[4 * blockIdx.x + 1] = acc[1];
    }
}

// torch's chain: -(g L1) + g (-o) / (o + eps) - ((-g) L2 + (-g) u / (u + eps)) with u = 1 - o; 0 where radii <= 0
__global__ void __launch_bounds__(RB) k_entropy_bwd(int64_t P, const float* __restrict__ o, int64_t os, const int32_t* __restrict__ radii,
                                                    int64_t rs, const double* totals, const float* g_out, float* __restrict__ d_o) {
    const float g = (float)((double)*g_out / totals[1]);
    for (int64_t i = (int64_t)blockIdx.x * RB + threadIdx.x; i < P; i += (int64_t)gridDim.x * RB) {
        float d = 0.0f;
        if (radii[i * rs] > 0) {
            const float v = o[i * os], u = __fsub_rn(1.0f, v);
            const float e1 = __fadd_rn(v, ENTROPY_EPS), e2 = __fadd_rn(u, ENTROPY_EPS);
            const float t1 = __fadd_rn(-__fmul_rn(g, logf(e1)), __fdiv_rn(__fmul_rn(g, -v), e1));
            const float t2 = __fadd_rn(__fmul_rn(-g, logf(e2)), __fdiv_rn(__fmul_rn(-g, u), e2));
            d = __fsub_rn(t1, t2);
        }
        d_o[i] = d;
    }
}

// ---- density-mode SDF estimation: e = d - exp(-0.5 s^2 / beta^2), mean |e| or mean e^2
struct DensityArgs {
    int64_t n;
    const float* d;
    int64_t d_s;
    const float* b;
    int64_t b_s;
    const float* s;
    int64_t s_s;
    int squared;
};

// the reference's expression with one rounding per torch op; t = exp(q), q = (-0.5 s^2) / beta^2, b2 = beta^2
__device__ __forceinline__ float density_error(const DensityArgs& a, int64_t i, float& t, float& q, float& b2) {
    const float s = a.s[i * a.s_s], beta = a.b[i * a.b_s];
    b2 = __fmul_rn(beta, beta);
    q = __fdiv_rn(__fmul_rn(-0.5f, __fmul_rn(s, s)), b2);
    t = expf(q);
    return __fsub_rn(a.d[i * a.d_s], t);
}

__global__ void __launch_bounds__(RB) k_density_fwd(const DensityArgs a, float* partials) {
    __shared__ float red[1][PB / 32];
    float acc[1] = {0.f};
    for (int64_t i = (int64_t)blockIdx.x * RB + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * RB) {
        float t, q, b2;
        const float e = density_error(a, i, t, q, b2);
        acc[0] += a.squared ? __fmul_rn(e, e) : fabsf(e);
    }
    block_sum<1>(acc, red);
    if (threadIdx.x == 0) partials[4 * blockIdx.x] = acc[0];
}

// torch's backward chain through pow(2) or abs, the subtraction, exp, the division ((-g q') / b2 and -g q' * (q / b2)), the -0.5
// factor and the two pow(2)s; sgn(0) = 0 makes every gradient of that sample zero, as in torch
__global__ void __launch_bounds__(RB) k_density_bwd(const DensityArgs a, const float* g_out, float* __restrict__ d_d,
                                                    float* __restrict__ d_b, float* __restrict__ d_s) {
    const float g = (float)((double)*g_out / (double)a.n);
    for (int64_t i = (int64_t)blockIdx.x * RB + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * RB) {
        float t, q, b2;
        const float e = density_error(a, i, t, q, b2);
        const float ge = a.squared ? __fmul_rn(g, __fmul_rn(2.0f, e)) : __fmul_rn(g, sgn(e));
        const float gq = __fmul_rn(-ge, t);
        const float gb2 = __fmul_rn(-gq, __fdiv_rn(q, b2));
        const float gs2 = __fmul_rn(__fdiv_rn(gq, b2), -0.5f);
        d_d[i] = ge;
        d_s[i] = __fmul_rn(gs2, __fmul_rn(2.0f, a.s[i * a.s_s]));
        d_b[i] = __fmul_rn(gb2, __fmul_rn(2.0f, a.b[i * a.b_s]));
    }
}

enum { FIN_PHOTO = 0, FIN_NORMAL = 1, FIN_MEAN = 2, FIN_RATIO = 3, FIN_DEPTH_SOLVE = 4 };

// one CTA: totals[k] = sum of partials[blk * stride + k] in double, thread-strided then tree order; then the mode's means
template <typename T>
__global__ void __launch_bounds__(RB) k_loss_finalize(int mode, const T* partials, int64_t blocks, int stride, int K, double n,
                                                      double* totals, float* out, float* out2) {
    __shared__ double sh[RB];
    for (int k = 0; k < K; ++k) {
        double s = 0.0;
        for (int64_t b = threadIdx.x; b < blocks; b += RB) s += (double)partials[b * stride + k];
        sh[threadIdx.x] = s;
        __syncthreads();
        for (int o = RB / 2; o > 0; o >>= 1) {
            if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
            __syncthreads();
        }
        if (threadIdx.x == 0) totals[k] = sh[0];
        __syncthreads();
    }
    if (threadIdx.x != 0) return;
    if (mode == FIN_PHOTO) {
        if (out) out[0] = (float)(totals[0] / n);
        out2[0] = (float)(totals[1] / n);
    } else if (mode == FIN_NORMAL) {  // l1 + 0.1 * cos, an empty selection is 0 / 0 = NaN as torch's mean of nothing
        const float l1 = (float)(totals[0] / (3.0 * totals[2])), cos = -(float)(totals[1] / totals[2]);
        out[0] = __fadd_rn(l1, __fmul_rn(0.1f, cos));
    } else if (mode == FIN_RATIO) {  // sum / count; no counted element is 0 / 0 = NaN
        out[0] = (float)(totals[0] / totals[1]);
    } else if (mode == FIN_DEPTH_SOLVE) {  // compute_scale_and_shift (LU/:65-92) on the sums rounded to float32, torch's order
        const float a00 = (float)totals[0], a01 = (float)totals[1], a11 = (float)totals[2];
        const float b0 = (float)totals[3], b1 = (float)totals[4];
        const float det = __fsub_rn(__fmul_rn(a00, a11), __fmul_rn(a01, a01));
        float x0 = __int_as_float(0x7fffffff), x1 = x0;  // det == 0: the reference fails; NaN here (INTEGRATION.md)
        if (det != 0.0f) {
            x0 = __fdiv_rn(__fsub_rn(__fmul_rn(a11, b0), __fmul_rn(a01, b1)), det);
            x1 = __fdiv_rn(__fadd_rn(__fmul_rn(-a01, b0), __fmul_rn(a00, b1)), det);
        }
        out[0] = x0;
        out[1] = x1;
    } else {
        out[0] = (float)(totals[0] / n);
    }
}

int reduce_blocks(int64_t n) {
    const int64_t b = (n + RB - 1) / RB;
    return (int)(b < RMAX_BLOCKS ? (b > 0 ? b : 1) : RMAX_BLOCKS);
}

bool photo_dims_ok(int B, int C, int H, int W) { return B > 0 && C > 0 && H > 0 && W > 0 && (int64_t)B * C < 65536; }

size_t photo_blocks(int B, int C, int H, int W) { return (size_t)((W + PT - 1) / PT) * ((H + PT - 1) / PT) * B * C; }

Window make_window(const float* w) {
    Window win;
    for (int k = 0; k < 2 * PR + 1; ++k) win.w[k] = w[k];
    return win;
}

}  // namespace

static int normal_args(const char* who, int64_t n, const float* pred, const int64_t* ps, const float* gt, const int64_t* gs,
                       const float* depth, int64_t d_sp, float scene_scale, NormalArgs& a) {
    if (n <= 0 || !pred || !ps || !gt || !gs) {
        set_error("%s: bad arguments (n %lld)", who, (long long)n);
        return GSR_ERR_INVALID;
    }
    a = NormalArgs{n, pred, ps[0], ps[1], gt, gs[0], gs[1], depth, d_sp, scene_scale};
    return GSR_OK;
}

static int check_reduce_ws(const char* who, const void* ws, size_t ws_bytes) {
    if (!ws || ws_bytes < GSR_LOSS_REDUCE_BYTES || ((uintptr_t)ws & 15u)) {
        set_error("%s: workspace of %zu bytes, GSR_LOSS_REDUCE_BYTES (%d) needed (16-byte aligned)", who, ws_bytes,
                  GSR_LOSS_REDUCE_BYTES);
        return GSR_ERR_WORKSPACE;
    }
    return GSR_OK;
}

}  // namespace gsr

using namespace gsr;

size_t gsr_photometric_loss_bytes(int32_t B, int32_t C, int32_t H, int32_t W, int32_t for_backward) {
    if (!photo_dims_ok(B, C, H, W)) return 0;
    const size_t n = (size_t)B * C * H * W;
    return 256 + align256(photo_blocks(B, C, H, W) * 2 * sizeof(float)) + (for_backward ? align256(3 * n * sizeof(float)) : 0);
}

int gsr_photometric_loss(int32_t B, int32_t C, int32_t H, int32_t W, const float* x, const int64_t* xs, const float* y,
                         const int64_t* ys, const float* window, int32_t for_backward, float* out_l1, float* out_ssim, void* ws,
                         size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_photometric_loss");
    const cudaStream_t st = (cudaStream_t)stream;
    if (!photo_dims_ok(B, C, H, W) || !x || !xs || !y || !ys || !window || !out_ssim) {
        set_error("gsr_photometric_loss: bad arguments (B %d, C %d, H %d, W %d)", B, C, H, W);
        return GSR_ERR_INVALID;
    }
    const bool store = for_backward != 0;
    const size_t need = gsr_photometric_loss_bytes(B, C, H, W, store);
    if (!ws || ws_bytes < need || ((uintptr_t)ws & 15u)) {
        set_error("gsr_photometric_loss: workspace of %zu bytes, %zu needed (16-byte aligned)", ws_bytes, need);
        return GSR_ERR_WORKSPACE;
    }
    PhotoArgs a;
    a.B = B; a.C = C; a.H = H; a.W = W;
    a.l1 = out_l1 != nullptr;
    a.store = store;
    a.x = x; a.y = y;
    a.sx = {xs[0], xs[1], xs[2], xs[3]};
    a.sy = {ys[0], ys[1], ys[2], ys[3]};
    a.win = make_window(window);
    char* base = (char*)ws;
    double* totals = (double*)base;
    a.partials = (float*)(base + 256);
    a.maps = (float*)(base + 256 + align256(photo_blocks(B, C, H, W) * 2 * sizeof(float)));
    const dim3 grid((W + PT - 1) / PT, (H + PT - 1) / PT, B * C);
    k_photo_fwd<<<grid, PB, 0, st>>>(a);
    k_loss_finalize<<<1, RB, 0, st>>>(FIN_PHOTO, a.partials, (int64_t)photo_blocks(B, C, H, W), 2, 2, (double)B * C * H * W, totals,
                                      out_l1, out_ssim);
    return check_launch("gsr_photometric_loss", false, st);
}

int gsr_photometric_loss_backward(int32_t B, int32_t C, int32_t H, int32_t W, const float* x, const int64_t* xs, const float* y,
                                  const int64_t* ys, const float* window, const float* g_l1, const float* g_ssim, float* dx,
                                  const void* ws, size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_photometric_loss_backward");
    const cudaStream_t st = (cudaStream_t)stream;
    if (!photo_dims_ok(B, C, H, W) || !x || !xs || !y || !ys || !window || !dx) {
        set_error("gsr_photometric_loss_backward: bad arguments (B %d, C %d, H %d, W %d)", B, C, H, W);
        return GSR_ERR_INVALID;
    }
    const size_t need = gsr_photometric_loss_bytes(B, C, H, W, 1);
    if (!ws || ws_bytes < need || ((uintptr_t)ws & 15u)) {
        set_error("gsr_photometric_loss_backward: workspace of %zu bytes, %zu needed (the forward's, with for_backward)",
                  ws_bytes, need);
        return GSR_ERR_WORKSPACE;
    }
    PhotoBwdArgs a;
    a.B = B; a.C = C; a.H = H; a.W = W;
    a.x = x; a.y = y;
    a.sx = {xs[0], xs[1], xs[2], xs[3]};
    a.sy = {ys[0], ys[1], ys[2], ys[3]};
    a.win = make_window(window);
    a.maps = (const float*)((const char*)ws + 256 + align256(photo_blocks(B, C, H, W) * 2 * sizeof(float)));
    a.g_l1 = g_l1; a.g_ssim = g_ssim; a.dx = dx;
    const dim3 grid((W + PT - 1) / PT, (H + PT - 1) / PT, B * C);
    k_photo_bwd<<<grid, PB, 0, st>>>(a);
    return check_launch("gsr_photometric_loss_backward", false, st);
}

int gsr_normal_loss(int64_t n, const float* pred, const int64_t* ps, const float* gt, const int64_t* gs, const float* depth,
                    int64_t d_sp, float scene_scale, float* out, void* ws, size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_normal_loss");
    const cudaStream_t st = (cudaStream_t)stream;
    NormalArgs a;
    int rc = normal_args("gsr_normal_loss", n, pred, ps, gt, gs, depth, d_sp, scene_scale, a);
    if (rc == GSR_OK && !out) { set_error("gsr_normal_loss: null output"); rc = GSR_ERR_INVALID; }
    if (rc == GSR_OK) rc = check_reduce_ws("gsr_normal_loss", ws, ws_bytes);
    if (rc != GSR_OK) return rc;
    const int blocks = reduce_blocks(n);
    float* partials = (float*)((char*)ws + 256);
    k_normal_fwd<<<blocks, RB, 0, st>>>(a, partials);
    k_loss_finalize<<<1, RB, 0, st>>>(FIN_NORMAL, partials, blocks, 4, 3, (double)n, (double*)ws, out, nullptr);
    return check_launch("gsr_normal_loss", false, st);
}

int gsr_normal_loss_backward(int64_t n, const float* pred, const int64_t* ps, const float* gt, const int64_t* gs,
                             const float* depth, int64_t d_sp, float scene_scale, const float* g_out, float* d_pred, const void* ws,
                             size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_normal_loss_backward");
    const cudaStream_t st = (cudaStream_t)stream;
    NormalArgs a;
    int rc = normal_args("gsr_normal_loss_backward", n, pred, ps, gt, gs, depth, d_sp, scene_scale, a);
    if (rc == GSR_OK && (!g_out || !d_pred)) { set_error("gsr_normal_loss_backward: null gradient"); rc = GSR_ERR_INVALID; }
    if (rc == GSR_OK) rc = check_reduce_ws("gsr_normal_loss_backward", ws, ws_bytes);
    if (rc != GSR_OK) return rc;
    k_normal_bwd<<<reduce_blocks(n), RB, 0, st>>>(a, (const double*)ws, g_out, d_pred);
    return check_launch("gsr_normal_loss_backward", false, st);
}

int gsr_anisotropic_loss(int64_t P, const float* scales, float r, float* out, void* ws, size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_anisotropic_loss");
    const cudaStream_t st = (cudaStream_t)stream;
    if (P <= 0 || !scales || !out) {
        set_error("gsr_anisotropic_loss: bad arguments (P %lld)", (long long)P);
        return GSR_ERR_INVALID;
    }
    const int rc = check_reduce_ws("gsr_anisotropic_loss", ws, ws_bytes);
    if (rc != GSR_OK) return rc;
    const int blocks = reduce_blocks(P);
    float* partials = (float*)((char*)ws + 256);
    k_aniso_fwd<<<blocks, RB, 0, st>>>(P, scales, r, partials);
    k_loss_finalize<<<1, RB, 0, st>>>(FIN_MEAN, partials, blocks, 4, 1, (double)P, (double*)ws, out, nullptr);
    return check_launch("gsr_anisotropic_loss", false, st);
}

int gsr_anisotropic_loss_backward(int64_t P, const float* scales, float r, const float* g_out, float* d_scales, void* stream) {
    NvtxRange nvtx_("gsr_anisotropic_loss_backward");
    const cudaStream_t st = (cudaStream_t)stream;
    if (P <= 0 || !scales || !g_out || !d_scales) {
        set_error("gsr_anisotropic_loss_backward: bad arguments (P %lld)", (long long)P);
        return GSR_ERR_INVALID;
    }
    k_aniso_bwd<<<reduce_blocks(P), RB, 0, st>>>(P, scales, r, g_out, d_scales);
    return check_launch("gsr_anisotropic_loss_backward", false, st);
}

int gsr_depth_loss(int64_t n, const float* pred, int64_t pred_stride, const float* gt, int64_t gt_stride, float scene_scale_inv,
                   float* out, void* ws, size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_depth_loss");
    const cudaStream_t st = (cudaStream_t)stream;
    if (n <= 0 || !pred || !gt || !out) {
        set_error("gsr_depth_loss: bad arguments (n %lld)", (long long)n);
        return GSR_ERR_INVALID;
    }
    const int rc = check_reduce_ws("gsr_depth_loss", ws, ws_bytes);
    if (rc != GSR_OK) return rc;
    const DepthArgs a{n, pred, pred_stride, gt, gt_stride, scene_scale_inv};
    double* totals = (double*)ws;
    float* x = (float*)((char*)ws + 128);
    void* partials = (char*)ws + 256;
    const int blocks = reduce_blocks(n), b64 = blocks < RMAX_BLOCKS64 ? blocks : RMAX_BLOCKS64;
    k_depth_sums<<<b64, RB, 0, st>>>(a, (double*)partials);
    k_loss_finalize<<<1, RB, 0, st>>>(FIN_DEPTH_SOLVE, (const double*)partials, b64, 8, 5, (double)n, totals, x, nullptr);
    k_depth_fwd<<<blocks, RB, 0, st>>>(a, x, (float*)partials);
    k_loss_finalize<<<1, RB, 0, st>>>(FIN_MEAN, (const float*)partials, blocks, 4, 1, (double)n, totals, out, nullptr);
    return check_launch("gsr_depth_loss", false, st);
}

int gsr_depth_loss_backward(int64_t n, const float* pred, int64_t pred_stride, const float* gt, int64_t gt_stride,
                            float scene_scale_inv, const float* g_out, float* d_pred, const void* ws, size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_depth_loss_backward");
    const cudaStream_t st = (cudaStream_t)stream;
    if (n <= 0 || !pred || !gt || !g_out || !d_pred) {
        set_error("gsr_depth_loss_backward: bad arguments (n %lld)", (long long)n);
        return GSR_ERR_INVALID;
    }
    const int rc = check_reduce_ws("gsr_depth_loss_backward", ws, ws_bytes);
    if (rc != GSR_OK) return rc;
    const DepthArgs a{n, pred, pred_stride, gt, gt_stride, scene_scale_inv};
    k_depth_bwd<<<reduce_blocks(n), RB, 0, st>>>(a, (const float*)((const char*)ws + 128), g_out, d_pred);
    return check_launch("gsr_depth_loss_backward", false, st);
}

static int opacity_fwd(const char* who, bool sparse, int64_t n, const float* x, int64_t xs, float* out, void* ws, size_t ws_bytes,
                       cudaStream_t st) {
    if (n <= 0 || !x || !out) {
        set_error("%s: bad arguments (n %lld)", who, (long long)n);
        return GSR_ERR_INVALID;
    }
    const int rc = check_reduce_ws(who, ws, ws_bytes);
    if (rc != GSR_OK) return rc;
    const int blocks = reduce_blocks(n);
    float* partials = (float*)((char*)ws + 256);
    if (sparse)
        k_opacity_fwd<true><<<blocks, RB, 0, st>>>(n, x, xs, partials);
    else
        k_opacity_fwd<false><<<blocks, RB, 0, st>>>(n, x, xs, partials);
    k_loss_finalize<<<1, RB, 0, st>>>(FIN_MEAN, (const float*)partials, blocks, 4, 1, (double)n, (double*)ws, out, nullptr);
    return check_launch(who, false, st);
}

int gsr_opacity_loss(int64_t n, const float* x, int64_t x_stride, float* out, void* ws, size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_opacity_loss");
    return opacity_fwd("gsr_opacity_loss", false, n, x, x_stride, out, ws, ws_bytes, (cudaStream_t)stream);
}

int gsr_opacity_loss_backward(int64_t n, const float* g_out, float* dx, void* stream) {
    NvtxRange nvtx_("gsr_opacity_loss_backward");
    const cudaStream_t st = (cudaStream_t)stream;
    if (n <= 0 || !g_out || !dx) {
        set_error("gsr_opacity_loss_backward: bad arguments (n %lld)", (long long)n);
        return GSR_ERR_INVALID;
    }
    k_opacity_bwd<false><<<reduce_blocks(n), RB, 0, st>>>(n, nullptr, 0, g_out, dx);
    return check_launch("gsr_opacity_loss_backward", false, st);
}

int gsr_sparsity_loss(int64_t n, const float* x, int64_t x_stride, float* out, void* ws, size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_sparsity_loss");
    return opacity_fwd("gsr_sparsity_loss", true, n, x, x_stride, out, ws, ws_bytes, (cudaStream_t)stream);
}

int gsr_sparsity_loss_backward(int64_t n, const float* x, int64_t x_stride, const float* g_out, float* dx, void* stream) {
    NvtxRange nvtx_("gsr_sparsity_loss_backward");
    const cudaStream_t st = (cudaStream_t)stream;
    if (n <= 0 || !x || !g_out || !dx) {
        set_error("gsr_sparsity_loss_backward: bad arguments (n %lld)", (long long)n);
        return GSR_ERR_INVALID;
    }
    k_opacity_bwd<true><<<reduce_blocks(n), RB, 0, st>>>(n, x, x_stride, g_out, dx);
    return check_launch("gsr_sparsity_loss_backward", false, st);
}

int gsr_entropy_loss(int64_t P, const float* opacities, int64_t o_stride, const int32_t* radii, int64_t r_stride, float* out, void* ws,
                     size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_entropy_loss");
    const cudaStream_t st = (cudaStream_t)stream;
    if (P <= 0 || !opacities || !radii || !out) {
        set_error("gsr_entropy_loss: bad arguments (P %lld)", (long long)P);
        return GSR_ERR_INVALID;
    }
    const int rc = check_reduce_ws("gsr_entropy_loss", ws, ws_bytes);
    if (rc != GSR_OK) return rc;
    const int blocks = reduce_blocks(P);
    float* partials = (float*)((char*)ws + 256);
    k_entropy_fwd<<<blocks, RB, 0, st>>>(P, opacities, o_stride, radii, r_stride, partials);
    k_loss_finalize<<<1, RB, 0, st>>>(FIN_RATIO, (const float*)partials, blocks, 4, 2, (double)P, (double*)ws, out, nullptr);
    return check_launch("gsr_entropy_loss", false, st);
}

int gsr_entropy_loss_backward(int64_t P, const float* opacities, int64_t o_stride, const int32_t* radii, int64_t r_stride,
                              const float* g_out, float* d_opacities, const void* ws, size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_entropy_loss_backward");
    const cudaStream_t st = (cudaStream_t)stream;
    if (P <= 0 || !opacities || !radii || !g_out || !d_opacities) {
        set_error("gsr_entropy_loss_backward: bad arguments (P %lld)", (long long)P);
        return GSR_ERR_INVALID;
    }
    const int rc = check_reduce_ws("gsr_entropy_loss_backward", ws, ws_bytes);
    if (rc != GSR_OK) return rc;
    k_entropy_bwd<<<reduce_blocks(P), RB, 0, st>>>(P, opacities, o_stride, radii, r_stride, (const double*)ws, g_out, d_opacities);
    return check_launch("gsr_entropy_loss_backward", false, st);
}

int gsr_density_estimation_loss(int64_t n, const float* density, int64_t d_stride, const float* beta, int64_t b_stride,
                                const float* sdf_estimation, int64_t s_stride, int32_t squared, float* out, void* ws, size_t ws_bytes,
                                void* stream) {
    NvtxRange nvtx_("gsr_density_estimation_loss");
    const cudaStream_t st = (cudaStream_t)stream;
    if (n <= 0 || !density || !beta || !sdf_estimation || !out) {
        set_error("gsr_density_estimation_loss: bad arguments (n %lld)", (long long)n);
        return GSR_ERR_INVALID;
    }
    const int rc = check_reduce_ws("gsr_density_estimation_loss", ws, ws_bytes);
    if (rc != GSR_OK) return rc;
    const DensityArgs a{n, density, d_stride, beta, b_stride, sdf_estimation, s_stride, squared != 0};
    const int blocks = reduce_blocks(n);
    float* partials = (float*)((char*)ws + 256);
    k_density_fwd<<<blocks, RB, 0, st>>>(a, partials);
    k_loss_finalize<<<1, RB, 0, st>>>(FIN_MEAN, (const float*)partials, blocks, 4, 1, (double)n, (double*)ws, out, nullptr);
    return check_launch("gsr_density_estimation_loss", false, st);
}

int gsr_density_estimation_loss_backward(int64_t n, const float* density, int64_t d_stride, const float* beta, int64_t b_stride,
                                         const float* sdf_estimation, int64_t s_stride, int32_t squared, const float* g_out,
                                         float* d_density, float* d_beta, float* d_sdf_estimation, void* stream) {
    NvtxRange nvtx_("gsr_density_estimation_loss_backward");
    const cudaStream_t st = (cudaStream_t)stream;
    if (n <= 0 || !density || !beta || !sdf_estimation || !g_out || !d_density || !d_beta || !d_sdf_estimation) {
        set_error("gsr_density_estimation_loss_backward: bad arguments (n %lld)", (long long)n);
        return GSR_ERR_INVALID;
    }
    const DensityArgs a{n, density, d_stride, beta, b_stride, sdf_estimation, s_stride, squared != 0};
    k_density_bwd<<<reduce_blocks(n), RB, 0, st>>>(a, g_out, d_density, d_beta, d_sdf_estimation);
    return check_launch("gsr_density_estimation_loss_backward", false, st);
}
