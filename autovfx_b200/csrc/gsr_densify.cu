// gsr_b200 densification: the per-step statistics and densify_and_prune of 3DGS's GaussianModel and SuGaR's SuGaRDensifier
// ("GS/" = sugar/gaussian_splatting/scene/gaussian_model.py:268-417, "SD/" = sugar/sugar_scene/sugar_densifier.py:48-246).
//
//   k_densify_stats    accum += |grad[i,:2]|, denom += 1, max_radii2D = max(max_radii2D, radii) on the masked rows.
//   k_plan_flags       the reference's clone, split and final-prune decisions for every original row, as 5 bits per row
//                      (original kept, clone kept, first split copy kept, second split copy kept, split-selected), and the
//                      per-block count of each bit.
//   k_rs_scan          (gsr_common.cuh) exclusive scan of the counts, laid out stream-major: the destination of every kept row in
//                      the reference's final order (originals, clones, first copies, second copies) and the split indices.
//   k_plan_offsets     per-row destinations (-1: no row) and the totals {S, P'}.
//   k_densify_apply    one pass over every element of every parameter group and both Adam moments: kept rows copied with
//                      their moments, new rows (clones, split children) written with zero moments.
//
// The decisions use torch's float32 roundings op by op: grads = accum / denom, norm = |g|, exp and sigmoid as ATen
// evaluates them (sigmoid = 1 / (1 + exp(-x))), maxima that propagate NaN, thresholds rounded to float by the caller.
#include "gsr_common.cuh"

namespace gsr {

namespace {

constexpr int PLAN_BLOCK = 1024;
constexpr int N_STREAMS = 5;  // 4 destination streams + the split index

__global__ void k_densify_stats(int P, int C, const float* __restrict__ grad, const uint8_t* __restrict__ mask,
                                const int32_t* __restrict__ radii, float* __restrict__ accum, float* __restrict__ denom,
                                float* __restrict__ max_radii) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P || !mask[i]) return;
    const float a = grad[(size_t)i * C], b = grad[(size_t)i * C + 1];
    // torch.norm(dim=-1) over 2 elements: each square rounded, then one add (the reduction's two accumulators)
    accum[i] = __fadd_rn(accum[i], __fsqrt_rn(__fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b))));
    denom[i] = __fadd_rn(denom[i], 1.0f);
    if (max_radii) {
        const float m = max_radii[i], r = __int2float_rn(radii[i]);
        max_radii[i] = (m != m || !(m < r)) ? m : r;  // torch.maximum: NaN propagates
    }
}

__device__ __forceinline__ float nanmax(float a, float b) { return (a != a || a > b) ? a : b; }
__device__ __forceinline__ float max3_exp(float s0, float s1, float s2) { return nanmax(nanmax(expf(s0), expf(s1)), expf(s2)); }
// torch: scaling_inverse_activation(get_scaling / (0.8 * 2)); ATen divides by a Python float as a multiply by 1.0f / float(x)
__device__ __forceinline__ float child_scale(float s) { return logf(__fmul_rn(expf(s), 1.0f / 1.6f)); }

struct PlanArgs {
    int P, nb;
    const float *accum, *denom, *scaling, *opacity;
    float max_grad, dense_thr, min_opacity, max_screen_size, big_thr;
    int use_screen;
    uint8_t* flags;
    uint32_t* hist;  // [N_STREAMS * nb + 1]
};

__global__ void __launch_bounds__(PLAN_BLOCK) k_plan_flags(PlanArgs a) {
    const int i = blockIdx.x * PLAN_BLOCK + threadIdx.x;
    uint32_t f = 0;
    if (i < a.P) {
        float g = __fdiv_rn(a.accum[i], a.denom[i]);
        if (g != g) g = 0.0f;
        const float s0 = a.scaling[3 * (size_t)i], s1 = a.scaling[3 * (size_t)i + 1], s2 = a.scaling[3 * (size_t)i + 2];
        const float mx = max3_exp(s0, s1, s2);
        // torch.norm over grads' single column is |g|: no rounded square, which would underflow for |g| < 1.1e-19
        const bool clone = fabsf(g) >= a.max_grad && mx <= a.dense_thr;
        const bool split = g >= a.max_grad && mx > a.dense_thr;
        const float op = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-a.opacity[i])));
        // the final prune sees max_radii2D = 0 (densification_postfix reset it)
        const bool low = op < a.min_opacity, big_vs = a.use_screen && 0.0f > a.max_screen_size;
        const bool prune = low || big_vs || (a.use_screen && mx > a.big_thr);
        if (split) {
            const bool prune_child = low || big_vs || (a.use_screen && max3_exp(child_scale(s0), child_scale(s1), child_scale(s2)) > a.big_thr);
            f = 16u | (prune_child ? 0u : 12u);
        } else {
            f = (prune ? 0u : 1u) | (clone && !prune ? 2u : 0u);
        }
        a.flags[i] = (uint8_t)f;
    }
#pragma unroll
    for (int s = 0; s < N_STREAMS; ++s) {
        const int c = __syncthreads_count((f >> s) & 1u);
        if (threadIdx.x == 0) a.hist[(size_t)s * a.nb + blockIdx.x] = (uint32_t)c;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) a.hist[(size_t)N_STREAMS * a.nb] = 0;
}

__global__ void __launch_bounds__(PLAN_BLOCK) k_plan_offsets(int P, int nb, const uint8_t* __restrict__ flags,
                                                             const uint32_t* __restrict__ hist, int32_t* __restrict__ dst,
                                                             int32_t* __restrict__ totals) {
    __shared__ uint32_t wcount[N_STREAMS][32];
    const int i = blockIdx.x * PLAN_BLOCK + threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t f = i < P ? flags[i] : 0u;
    uint32_t rank[N_STREAMS];
#pragma unroll
    for (int s = 0; s < N_STREAMS; ++s) {
        const uint32_t bal = __ballot_sync(GSR_FULL, (f >> s) & 1u);
        rank[s] = __popc(bal & ((1u << lane) - 1u));
        if (lane == 0) wcount[s][warp] = __popc(bal);
    }
    __syncthreads();
    if (warp < N_STREAMS) {  // exclusive scan of the 32 warp counts of stream `warp`
        const uint32_t v = wcount[warp][lane];
        uint32_t incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(GSR_FULL, incl, o);
            if (lane >= o) incl += t;
        }
        wcount[warp][lane] = incl - v;
    }
    __syncthreads();
    const uint32_t split_base = hist[(size_t)(N_STREAMS - 1) * nb];  // = P'
    if (i < P) {
#pragma unroll
        for (int s = 0; s < N_STREAMS; ++s) {
            const uint32_t d = hist[(size_t)s * nb + blockIdx.x] + wcount[s][warp] + rank[s] - (s == N_STREAMS - 1 ? split_base : 0u);
            dst[(size_t)s * P + i] = (f >> s) & 1u ? (int32_t)d : -1;
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        totals[0] = (int32_t)(hist[(size_t)N_STREAMS * nb] - split_base);
        totals[1] = (int32_t)split_base;
    }
}

// 3DGS build_rotation (GS/utils/general_utils.py:78-99): the raw quaternion over its norm, every torch op rounded on its own
__device__ void rotation_3dgs(const float* q4, float R[9]) {
    const float a = q4[0], b = q4[1], c = q4[2], d = q4[3];
    const float n = __fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b)), __fmul_rn(c, c)), __fmul_rn(d, d)));
    const float r = __fdiv_rn(a, n), x = __fdiv_rn(b, n), y = __fdiv_rn(c, n), z = __fdiv_rn(d, n);
    const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
    const float xy = __fmul_rn(x, y), xz = __fmul_rn(x, z), yz = __fmul_rn(y, z);
    const float rx = __fmul_rn(r, x), ry = __fmul_rn(r, y), rz = __fmul_rn(r, z);
    R[0] = __fsub_rn(1.0f, 2.0f * __fadd_rn(yy, zz));
    R[1] = 2.0f * __fsub_rn(xy, rz);
    R[2] = 2.0f * __fadd_rn(xz, ry);
    R[3] = 2.0f * __fadd_rn(xy, rz);
    R[4] = __fsub_rn(1.0f, 2.0f * __fadd_rn(xx, zz));
    R[5] = 2.0f * __fsub_rn(yz, rx);
    R[6] = 2.0f * __fsub_rn(xz, ry);
    R[7] = 2.0f * __fadd_rn(yz, rx);
    R[8] = __fsub_rn(1.0f, 2.0f * __fadd_rn(xx, yy));
}

// SuGaR: pytorch3d quaternion_to_matrix(F.normalize(q)); the 4-term sums are pairwise, as torch's reductions add them
__device__ void rotation_sugar(const float* q4, float R[9]) {
    const float a = q4[0], b = q4[1], c = q4[2], d = q4[3];
    const float n = fmaxf(__fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b)), __fadd_rn(__fmul_rn(c, c), __fmul_rn(d, d)))),
                          1e-12f);
    const float r = __fdiv_rn(a, n), i = __fdiv_rn(b, n), j = __fdiv_rn(c, n), k = __fdiv_rn(d, n);
    const float ts = __fdiv_rn(2.0f, __fadd_rn(__fadd_rn(__fmul_rn(r, r), __fmul_rn(i, i)), __fadd_rn(__fmul_rn(j, j), __fmul_rn(k, k))));
    const float ii = __fmul_rn(i, i), jj = __fmul_rn(j, j), kk = __fmul_rn(k, k);
    const float ij = __fmul_rn(i, j), ik = __fmul_rn(i, k), jk = __fmul_rn(j, k);
    const float ir = __fmul_rn(i, r), jr = __fmul_rn(j, r), kr = __fmul_rn(k, r);
    R[0] = __fsub_rn(1.0f, __fmul_rn(ts, __fadd_rn(jj, kk)));
    R[1] = __fmul_rn(ts, __fsub_rn(ij, kr));
    R[2] = __fmul_rn(ts, __fadd_rn(ik, jr));
    R[3] = __fmul_rn(ts, __fadd_rn(ij, kr));
    R[4] = __fsub_rn(1.0f, __fmul_rn(ts, __fadd_rn(ii, kk)));
    R[5] = __fmul_rn(ts, __fsub_rn(jk, ir));
    R[6] = __fmul_rn(ts, __fsub_rn(ik, jr));
    R[7] = __fmul_rn(ts, __fadd_rn(jk, ir));
    R[8] = __fsub_rn(1.0f, __fmul_rn(ts, __fadd_rn(ii, jj)));
}

struct ApplyArgs {
    int P, S, n_groups, rotation_mode;
    const int32_t* dst;  // [5, P]
    const float *xyz, *scaling, *rotation, *eps;
    gsr_densify_group g[GSR_DENSIFY_MAX_GROUPS];
};

__global__ void __launch_bounds__(256) k_densify_apply(ApplyArgs a) {
    const gsr_densify_group G = a.g[blockIdx.y];
    const int w = G.width;
    const size_t n = (size_t)a.P * w, P = (size_t)a.P;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
        const size_t i = e / w, c = e - i * w;
        const int d0 = a.dst[i], d1 = a.dst[P + i], d2 = a.dst[2 * P + i], d3 = a.dst[3 * P + i];
        if ((d0 & d1 & d2 & d3) < 0) continue;  // every stream -1: the row leaves no row
        const float v = G.src[e];
        if (d0 >= 0) {
            G.dst[(size_t)d0 * w + c] = v;
            if (G.m1_dst) G.m1_dst[(size_t)d0 * w + c] = G.m1_src[e];
            if (G.m2_dst) G.m2_dst[(size_t)d0 * w + c] = G.m2_src[e];
        }
        if (d1 >= 0) {
            G.dst[(size_t)d1 * w + c] = v;
            if (G.m1_dst) G.m1_dst[(size_t)d1 * w + c] = 0.0f;
            if (G.m2_dst) G.m2_dst[(size_t)d1 * w + c] = 0.0f;
        }
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const int d = k ? d3 : d2;
            if (d < 0) continue;
            float out = v;
            if (G.role == GSR_DENSIFY_ROLE_SCALING) {
                out = child_scale(v);
            } else if (G.role == GSR_DENSIFY_ROLE_XYZ) {
                // torch.normal(0, std) = normal_(0, 1) * std + 0 with std = get_scaling; then bmm(R, samples) + xyz
                const size_t row = (size_t)k * a.S + a.dst[4 * P + i];
                float R[9];
                if (a.rotation_mode == GSR_DENSIFY_ROTATION_SUGAR) rotation_sugar(a.rotation + 4 * i, R);
                else rotation_3dgs(a.rotation + 4 * i, R);
                float acc = 0.0f;
#pragma unroll
                for (int m = 0; m < 3; ++m) {
                    const float smp = __fadd_rn(__fmul_rn(a.eps[3 * row + m], expf(a.scaling[3 * i + m])), 0.0f);
                    const float rcm = c == 0 ? R[m] : (c == 1 ? R[3 + m] : R[6 + m]);  // constant indices: R stays in registers
                    acc = fmaf(rcm, smp, acc);
                }
                out = __fadd_rn(acc, a.xyz[3 * i + c]);
            }
            G.dst[(size_t)d * w + c] = out;
            if (G.m1_dst) G.m1_dst[(size_t)d * w + c] = 0.0f;
            if (G.m2_dst) G.m2_dst[(size_t)d * w + c] = 0.0f;
        }
    }
}

inline int nblocks_plan(int P) { return (P + PLAN_BLOCK - 1) / PLAN_BLOCK; }

}  // namespace

}  // namespace gsr

using namespace gsr;

int gsr_densify_stats(int32_t P, int32_t C, const float* grad, const uint8_t* mask, const int32_t* radii, float* accum, float* denom,
                      float* max_radii, void* stream) {
    NvtxRange nvtx_("gsr_densify_stats");
    const cudaStream_t st = (cudaStream_t)stream;
    if (P < 0 || C < 2) {
        set_error("gsr_densify_stats: P = %d and C = %d (need P >= 0, C >= 2)", P, C);
        return GSR_ERR_INVALID;
    }
    if (P == 0) return GSR_OK;
    if (!grad || !mask || !accum || !denom || (!max_radii) != (!radii)) {
        set_error("gsr_densify_stats: missing input (grad, mask, accum, denom are required; radii and max_radii2D go together)");
        return GSR_ERR_INVALID;
    }
    k_densify_stats<<<(P + 255) / 256, 256, 0, st>>>(P, C, grad, mask, radii, accum, denom, max_radii);
    return check_launch("gsr_densify_stats", false, st);
}

size_t gsr_densify_plan_bytes(int32_t P) {
    const size_t nb = P > 0 ? (size_t)nblocks_plan(P) : 0;
    return align_up((size_t)(P > 0 ? P : 0), 16) + 4 * (N_STREAMS * nb + 1);
}

int gsr_densify_plan(int32_t P, const float* accum, const float* denom, const float* scaling, const float* opacity, float max_grad,
                     float dense_thr, float min_opacity, int32_t use_screen, float max_screen_size, float big_thr, int32_t* dst,
                     int32_t* totals, void* ws, size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_densify_plan");
    const cudaStream_t st = (cudaStream_t)stream;
    if (P < 0 || P > INT32_MAX / 3) {
        set_error("gsr_densify_plan: P = %d outside 0..%d", P, INT32_MAX / 3);
        return GSR_ERR_INVALID;
    }
    if (!totals || (P > 0 && (!accum || !denom || !scaling || !opacity || !dst))) {
        set_error("gsr_densify_plan: missing input or output");
        return GSR_ERR_INVALID;
    }
    if (ws_bytes < gsr_densify_plan_bytes(P) || (P > 0 && !ws) || ((uintptr_t)ws & 15)) {
        set_error("gsr_densify_plan: workspace of %zu bytes (need %zu, 16-byte aligned)", ws_bytes, gsr_densify_plan_bytes(P));
        return GSR_ERR_WORKSPACE;
    }
    if (P == 0) {
        cudaMemsetAsync(totals, 0, 2 * sizeof(int32_t), st);
        return check_launch("gsr_densify_plan", false, st);
    }
    const int nb = nblocks_plan(P);
    uint8_t* flags = (uint8_t*)ws;
    uint32_t* hist = (uint32_t*)((char*)ws + align_up((size_t)P, 16));
    const PlanArgs a{P, nb, accum, denom, scaling, opacity, max_grad, dense_thr, min_opacity, max_screen_size, big_thr, use_screen,
                     flags, hist};
    k_plan_flags<<<nb, PLAN_BLOCK, 0, st>>>(a);
    k_rs_scan<<<1, 1024, 0, st>>>(hist, N_STREAMS * nb + 1);
    k_plan_offsets<<<nb, PLAN_BLOCK, 0, st>>>(P, nb, flags, hist, dst, totals);
    return check_launch("gsr_densify_plan", false, st);
}

int gsr_densify_apply(int32_t P, int32_t S, int32_t n_groups, const gsr_densify_group* groups, const int32_t* dst, const float* xyz,
                      const float* scaling, const float* rotation, const float* eps, int32_t rotation_mode, void* stream) {
    NvtxRange nvtx_("gsr_densify_apply");
    const cudaStream_t st = (cudaStream_t)stream;
    if (P < 0 || S < 0 || S > P || n_groups < 0 || n_groups > GSR_DENSIFY_MAX_GROUPS || (n_groups > 0 && !groups) ||
        (rotation_mode != GSR_DENSIFY_ROTATION_3DGS && rotation_mode != GSR_DENSIFY_ROTATION_SUGAR)) {
        set_error("gsr_densify_apply: P = %d, S = %d, %d groups (at most %d), rotation mode %d", P, S, n_groups, GSR_DENSIFY_MAX_GROUPS,
                  rotation_mode);
        return GSR_ERR_INVALID;
    }
    if (P == 0 || n_groups == 0) return GSR_OK;
    ApplyArgs a{};
    a.P = P, a.S = S, a.n_groups = n_groups, a.rotation_mode = rotation_mode, a.dst = dst;
    a.xyz = xyz, a.scaling = scaling, a.rotation = rotation, a.eps = eps;
    int wmax = 0;
    for (int g = 0; g < n_groups; ++g) {
        const gsr_densify_group& G = groups[g];
        const bool moments_ok = (!G.m1_src) == (!G.m1_dst) && (!G.m2_src) == (!G.m2_dst);
        const bool xyz_ok = G.role != GSR_DENSIFY_ROLE_XYZ || (G.width == 3 && xyz && scaling && rotation && (S == 0 || eps));
        const bool role_ok = G.role == GSR_DENSIFY_ROLE_COPY || G.role == GSR_DENSIFY_ROLE_XYZ ||
                             (G.role == GSR_DENSIFY_ROLE_SCALING && G.width == 3);
        if (G.width < 0 || (G.width > 0 && (!G.src || !G.dst)) || !moments_ok || !xyz_ok || !role_ok || !dst) {
            set_error("gsr_densify_apply: group %d is malformed (width %d, role %d)", g, G.width, G.role);
            return GSR_ERR_INVALID;
        }
        a.g[g] = G;
        wmax = wmax > G.width ? wmax : G.width;
    }
    if (wmax == 0) return GSR_OK;
    const size_t blocks = ((size_t)P * wmax + 255) / 256;
    const dim3 grid((unsigned)(blocks < 132 * 16 ? blocks : 132 * 16), (unsigned)n_groups);
    k_densify_apply<<<grid, 256, 0, st>>>(a);
    return check_launch("gsr_densify_apply", false, st);
}
