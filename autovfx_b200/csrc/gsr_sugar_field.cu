// gsr_b200 — SuGaR's SDF-regularisation field ("SS/" = sugar/sugar_scene/sugar_model.py): get_field_values (SS/:1118-1187),
// compute_density (SS/:1216-1239) and get_beta's 'average' mode (SS/:1063-1066), forward and backward, for N samples x K
// neighbours (K <= 32) over P Gaussians.
//
//   k_field_prepare   one thread per Gaussian: a 64-byte record {centre, density_factor * strength, A = get_covariance(
//                     return_full_matrix, return_sqrt, inverse_scales) (SS/:602-608), min scale and its index}, so that every
//                     (sample, neighbour) pair costs one aligned 64-byte gather
//   k_field<W>        one segment of W = pow2 >= K lanes per sample, lane = neighbour: the per-pair opacity, and the density and
//                     beta as fixed-order butterfly sums over the segment; then the sdf
//   k_field_backward<W>  recomputes the forward (nothing is kept between the calls), writes dL/dx per sample without atomics and
//                     accumulates the record gradients of every pair into a per-Gaussian 64-byte scratch with 16-byte RED.ADDs
//   k_field_chain     one thread per Gaussian: record gradients -> dL/dpoints, dL/dscaling (through 1 / clamp(s, 1e-8) and the
//                     min), dL/dquaternions (through pytorch3d's quaternion_to_matrix), dL/dstrengths
//   Under torch.use_deterministic_algorithms (gsr_sugar_field_backward_det) k_field_backward<W, true> emits one key per pair
//   instead of the RED.ADDs, group_ids (gsr_radix.cuh) sorts the pair ids by Gaussian, and k_field_reduce sums each Gaussian's
//   partials in ascending pair id before the same chain.  The better-normal kernels below do the same (DESIGN.md §4).
//
// Every elementwise torch op is one IEEE rounding here (explicit _rn intrinsics, accurate expf / logf / sqrtf, no FMA
// contraction) in the order SuGaR writes it.  torch's batched 3x3 matmul and its K-sum have no fixed order on the GPU, so the
// results are not claimed bit-identical to torch; the contract is the tolerance of tests/test_gpu_sugar_field.py.
#include "gsr_radix.cuh"

namespace gsr {

constexpr int FIELD_KMAX = 32;

struct FieldIn {
    int N, K, P, R;
    const float* x;            // [N,3]
    const int64_t* rows;       // [R,K] Gaussian indices
    const int64_t* row_idx;    // [N] row of each sample, NULL = identity (R == N)
    const float4* rec;         // [P] x 4 float4 records
    float opacity_min_clamp, sdf_offset;
};

// --- the record: r0 = (cx, cy, cz, fs), r1 = (A00, A01, A02, A10), r2 = (A11, A12, A20, A21), r3 = (A22, smin, kmin bits, 0),
//     A[i][j] = R[i][j] * (1 / clamp(s_j, 1e-8)), R = quaternion_to_matrix(q) (row i, column j), fs = density_factor * strength.
__device__ __forceinline__ float inv_scale_rn(float s) { return __frcp_rn(s < 1e-8f ? 1e-8f : s); }  // NaN passes as in clamp

__global__ void __launch_bounds__(256) k_field_prepare(int P, const float* __restrict__ points, const float* __restrict__ scaling,
                                                       const float* __restrict__ quaternions, const float* __restrict__ strengths,
                                                       float density_factor, float4* __restrict__ rec) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const size_t p3 = 3 * (size_t)p, p4 = 4 * (size_t)p;
    const float s0 = scaling[p3], s1 = scaling[p3 + 1], s2 = scaling[p3 + 2];
    float R[9], t;
    quat_to_matrix_rn(quaternions[p4], quaternions[p4 + 1], quaternions[p4 + 2], quaternions[p4 + 3], R, t);
    const float i0 = inv_scale_rn(s0), i1 = inv_scale_rn(s1), i2 = inv_scale_rn(s2);
    int km = 0;
    float sm = s0;
    if (s1 < sm) { sm = s1; km = 1; }
    if (s2 < sm) { sm = s2; km = 2; }
    float4* r = rec + 4 * (size_t)p;
    r[0] = make_float4(points[p3], points[p3 + 1], points[p3 + 2], __fmul_rn(density_factor, strengths[p]));
    r[1] = make_float4(__fmul_rn(R[0], i0), __fmul_rn(R[1], i1), __fmul_rn(R[2], i2), __fmul_rn(R[3], i0));
    r[2] = make_float4(__fmul_rn(R[4], i1), __fmul_rn(R[5], i2), __fmul_rn(R[6], i0), __fmul_rn(R[7], i1));
    r[3] = make_float4(__fmul_rn(R[8], i2), sm, __int_as_float(km), 0.0f);
}

// One (sample, neighbour) pair, recomputed identically by the forward and the backward.
struct FieldPair {
    bool ok;                 // the row and the Gaussian index are inside their arrays
    int64_t g;               // Gaussian index
    float sx, sy, sz;        // shift = x - centre
    float A[9];
    float w0, w1, w2;        // A^T shift
    float q;                 // (w0^2 + w1^2) + w2^2, unclamped
    float e, fs, o, smin;    // exp(-0.5 clamp(q, 0, 1e8)), density_factor * strength, fs * e, min scale
    int kmin;
};

__device__ __forceinline__ void field_pair(const FieldIn& a, int64_t n, int k, FieldPair& f) {
    const int64_t r = a.row_idx ? a.row_idx[n] : n;
    f.g = -1;
    if (r >= 0 && r < a.R) f.g = a.rows[r * a.K + k];
    f.ok = f.g >= 0 && f.g < a.P;
    if (!f.ok) {
        f.o = f.smin = __int_as_float(0x7fc00000);
        return;
    }
    const float4* rp = a.rec + 4 * f.g;
    const float4 r0 = __ldg(rp), r1 = __ldg(rp + 1), r2 = __ldg(rp + 2), r3 = __ldg(rp + 3);
    f.A[0] = r1.x; f.A[1] = r1.y; f.A[2] = r1.z; f.A[3] = r1.w; f.A[4] = r2.x; f.A[5] = r2.y; f.A[6] = r2.z; f.A[7] = r2.w; f.A[8] = r3.x;
    f.fs = r0.w; f.smin = r3.y; f.kmin = __float_as_int(r3.z);
    f.sx = __fsub_rn(a.x[3 * n], r0.x); f.sy = __fsub_rn(a.x[3 * n + 1], r0.y); f.sz = __fsub_rn(a.x[3 * n + 2], r0.z);
    // warped_shift = A^T @ shift: w_j = (A0j s0 + A1j s1) + A2j s2
    f.w0 = __fadd_rn(__fadd_rn(__fmul_rn(f.A[0], f.sx), __fmul_rn(f.A[3], f.sy)), __fmul_rn(f.A[6], f.sz));
    f.w1 = __fadd_rn(__fadd_rn(__fmul_rn(f.A[1], f.sx), __fmul_rn(f.A[4], f.sy)), __fmul_rn(f.A[7], f.sz));
    f.w2 = __fadd_rn(__fadd_rn(__fmul_rn(f.A[2], f.sx), __fmul_rn(f.A[5], f.sy)), __fmul_rn(f.A[8], f.sz));
    f.q = __fadd_rn(__fadd_rn(__fmul_rn(f.w0, f.w0), __fmul_rn(f.w1, f.w1)), __fmul_rn(f.w2, f.w2));
    const float qc = f.q > 1e8f ? 1e8f : f.q;  // clamp(min=0, max=1e8); q >= 0 by construction, NaN passes
    f.e = expf(__fmul_rn(-0.5f, qc));
    f.o = __fmul_rn(f.fs, f.e);
}

// Sum over the W lanes of a segment, the same butterfly order for every call; every lane of the segment gets the same value.
template <int W>
__device__ __forceinline__ float seg_sum(float v) {
#pragma unroll
    for (int off = W / 2; off >= 1; off >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, off));
    return v;
}

// d_hat = d / (d.detach() + 1e-12) where d >= 1 (SS/:1151-1152), then clamp(min=opacity_min_clamp); NaN passes.
__device__ __forceinline__ float field_dhat(float d) { return d >= 1.0f ? __fdiv_rn(d, __fadd_rn(d, 1e-12f)) : d; }
__device__ __forceinline__ float field_clampmin(float v, float lo) { return v < lo ? lo : v; }

template <int W>
__global__ void __launch_bounds__(256) k_field(FieldIn a, float* __restrict__ out_density, float* __restrict__ out_opac,
                                               float* __restrict__ out_beta, float* __restrict__ out_sdf) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t n = (int64_t)(t / W);
    const int k = (int)(t % W);
    const bool active = n < a.N && k < a.K;  // every lane takes part in the shuffles
    FieldPair f;
    f.o = f.smin = 0.0f;
    if (active) field_pair(a, n, k, f);
    const float d = seg_sum<W>(f.o);
    float bsum = 0.0f;
    if (out_beta || out_sdf) bsum = seg_sum<W>(f.smin);
    if (!active) return;
    if (out_opac) out_opac[n * a.K + k] = f.o;
    if (k != 0) return;
    if (out_density) out_density[n] = d;
    const float beta = __fdiv_rn(bsum, (float)a.K);  // .mean(dim=1)
    if (out_beta) out_beta[n] = beta;
    if (out_sdf) {
        const float cd = field_clampmin(field_dhat(d), a.opacity_min_clamp);
        out_sdf[n] = __fmul_rn(beta, __fsub_rn(sqrtf(__fmul_rn(-2.0f, logf(cd))), a.sdf_offset));
    }
}

struct FieldGrad {
    const float* g_density;  // [N]   dL/dfields['density'] (the clone before the normalisation)
    const float* g_opac;     // [N,K] dL/dneighbor_opacities
    const float* g_beta;     // [N]
    const float* g_sdf;      // [N]
    float* dx;               // [N,3]
    float4* grec;            // [P] x 4 float4: (dc0, dc1, dc2, dfs), (dA00..dA10), (dA11..dA21), (dA22, dsmin, 0, 0)
};

// The gradient reaching o_nk through every output of sample n but the opacities: the density's, and the sdf chain's (sqrt: g / (2
// result); -2 *: g * -2; log: g / x; clamp: where(x >= min); normalisation: g / (d + 1e-12)).  gbeta is dL/dbeta in, beta's
// sdf term added.  d is the segment's density sum, bsum its min-scale sum.
__device__ __forceinline__ float field_sample_grad(const FieldIn& a, const FieldGrad& b, int64_t n, float d, float bsum, float& gbeta) {
    float G = b.g_density ? b.g_density[n] : 0.0f;
    gbeta = b.g_beta ? b.g_beta[n] : 0.0f;
    if (b.g_sdf) {
        const float gs = b.g_sdf[n];
        const float beta = __fdiv_rn(bsum, (float)a.K);
        const float dh = field_dhat(d), cd = field_clampmin(dh, a.opacity_min_clamp);
        const float sq = sqrtf(__fmul_rn(-2.0f, logf(cd)));
        gbeta = __fadd_rn(gbeta, __fmul_rn(gs, __fsub_rn(sq, a.sdf_offset)));
        const float gm = __fdiv_rn(__fmul_rn(gs, beta), __fmul_rn(2.0f, sq));
        const float gcd = __fdiv_rn(__fmul_rn(gm, -2.0f), cd);
        const float gdh = dh >= a.opacity_min_clamp ? gcd : 0.0f;
        G = __fadd_rn(G, d >= 1.0f ? __fdiv_rn(gdh, __fadd_rn(d, 1e-12f)) : gdh);
    }
    return G;
}

// One pair's partials: dL/dshift ds and the record gradient r[0..12] = (-ds0, -ds1, -ds2, dfs, dA00, dA01, dA02, dA10, dA11, dA12,
// dA20, dA21, dA22), given G of its sample.  k_field_backward adds them with atomics, k_field_reduce in id order: one formula.
__device__ __forceinline__ void field_partial(const FieldIn& a, const FieldGrad& b, int64_t n, int k, const FieldPair& f, float G,
                                              float& ds0, float& ds1, float& ds2, float r[13]) {
    const float go = b.g_opac ? __fadd_rn(G, b.g_opac[n * a.K + k]) : G;
    const float dfs = __fmul_rn(go, f.e);
    const float dqc = __fmul_rn(__fmul_rn(__fmul_rn(go, f.fs), f.e), -0.5f);
    const float dq = (f.q <= 1e8f) ? dqc : 0.0f;  // clamp(0, 1e8) passes where 0 <= q <= 1e8
    const float dw0 = __fmul_rn(2.0f, __fmul_rn(dq, f.w0)), dw1 = __fmul_rn(2.0f, __fmul_rn(dq, f.w1)),
                dw2 = __fmul_rn(2.0f, __fmul_rn(dq, f.w2));
    ds0 = __fadd_rn(__fadd_rn(__fmul_rn(f.A[0], dw0), __fmul_rn(f.A[1], dw1)), __fmul_rn(f.A[2], dw2));
    ds1 = __fadd_rn(__fadd_rn(__fmul_rn(f.A[3], dw0), __fmul_rn(f.A[4], dw1)), __fmul_rn(f.A[5], dw2));
    ds2 = __fadd_rn(__fadd_rn(__fmul_rn(f.A[6], dw0), __fmul_rn(f.A[7], dw1)), __fmul_rn(f.A[8], dw2));
    r[0] = -ds0; r[1] = -ds1; r[2] = -ds2; r[3] = dfs;
    r[4] = __fmul_rn(dw0, f.sx); r[5] = __fmul_rn(dw1, f.sx); r[6] = __fmul_rn(dw2, f.sx);
    r[7] = __fmul_rn(dw0, f.sy); r[8] = __fmul_rn(dw1, f.sy); r[9] = __fmul_rn(dw2, f.sy);
    r[10] = __fmul_rn(dw0, f.sz); r[11] = __fmul_rn(dw1, f.sz); r[12] = __fmul_rn(dw2, f.sz);
}

// What DET adds to the default backward: per-sample scalars the partials need and one key per pair id n * K + k.
struct FieldDet {
    float* G;       // [N] field_sample_grad
    float* dmin;    // [N] the min scale's gradient, dL/dbeta / K
    uint32_t* key;  // [N*K] target Gaussian, P where the pair adds nothing
    uint32_t* id;   // [N*K] = the position
};

template <int W, bool DET>
__global__ void __launch_bounds__(256) k_field_backward(FieldIn a, FieldGrad b, FieldDet det) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t n = (int64_t)(t / W);
    const int k = (int)(t % W);
    const bool active = n < a.N && k < a.K;
    FieldPair f;
    f.o = f.smin = 0.0f;
    f.ok = false;
    if (active) field_pair(a, n, k, f);
    const float d = seg_sum<W>(f.o);
    float bsum = 0.0f;
    if (b.g_sdf) bsum = seg_sum<W>(f.smin);
    // One lane with an index outside its array makes d and beta NaN for the whole segment, so the sample adds nothing to any
    // Gaussian (not even through its valid lanes) and its dL/dx is NaN.
    const unsigned seg = W == 32 ? 0xffffffffu : ((1u << W) - 1u) << ((threadIdx.x & 31u) & ~(unsigned)(W - 1));
    const bool bad = (__ballot_sync(0xffffffffu, active && !f.ok) & seg) != 0u;
    float ds0 = 0.0f, ds1 = 0.0f, ds2 = 0.0f;  // dL/dshift of this pair
    if (DET && active) {
        const size_t pid = (size_t)n * a.K + k;
        det.key[pid] = bad ? (uint32_t)a.P : (uint32_t)f.g;
        det.id[pid] = (uint32_t)pid;
    }
    if (active && bad) {
        ds0 = ds1 = ds2 = __int_as_float(0x7fc00000);
    } else if (active) {  // every lane of the segment is inside its arrays
        float gbeta;
        const float G = field_sample_grad(a, b, n, d, bsum, gbeta);
        const float dmin = (b.g_beta || b.g_sdf) ? __fdiv_rn(gbeta, (float)a.K) : 0.0f;
        float r[13];
        field_partial(a, b, n, k, f, G, ds0, ds1, ds2, r);
        if (DET) {
            if (k == 0) { det.G[n] = G; det.dmin[n] = dmin; }
        } else {
            float4* gr = b.grec + 4 * f.g;
            atomicAdd(gr, make_float4(r[0], r[1], r[2], r[3]));
            atomicAdd(gr + 1, make_float4(r[4], r[5], r[6], r[7]));
            atomicAdd(gr + 2, make_float4(r[8], r[9], r[10], r[11]));
            atomicAdd(gr + 3, make_float4(r[12], dmin, 0.0f, 0.0f));
        }
    }
    ds0 = seg_sum<W>(ds0);
    ds1 = seg_sum<W>(ds1);
    ds2 = seg_sum<W>(ds2);
    if (active && k == 0 && b.dx) {
        b.dx[3 * n] = ds0; b.dx[3 * n + 1] = ds1; b.dx[3 * n + 2] = ds2;
    }
}

// DET: one thread per Gaussian g sums the partials of its pairs, recomputed with field_partial, in ascending pair id from +0.0, and
// writes g's record gradient for the unchanged k_field_chain.
__global__ void __launch_bounds__(256) k_field_reduce(FieldIn a, FieldGrad b, const float* __restrict__ G, const float* __restrict__ dmin,
                                                      const uint32_t* __restrict__ ids, const uint32_t* __restrict__ seg) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.P) return;
    float acc[14];
#pragma unroll
    for (int c = 0; c < 14; c++) acc[c] = 0.0f;
    const uint32_t e = seg[g + 1];
    for (uint32_t s = seg[g]; s < e; s++) {
        const uint32_t pid = ids[s];
        const int64_t n = pid / (uint32_t)a.K;
        const int k = (int)(pid - (uint32_t)n * (uint32_t)a.K);
        FieldPair f;
        field_pair(a, n, k, f);
        float ds0, ds1, ds2, r[13];
        field_partial(a, b, n, k, f, G[n], ds0, ds1, ds2, r);
#pragma unroll
        for (int c = 0; c < 13; c++) acc[c] = __fadd_rn(acc[c], r[c]);
        acc[13] = __fadd_rn(acc[13], dmin[n]);
    }
    float4* gr = b.grec + 4 * (size_t)g;
    gr[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    gr[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
    gr[2] = make_float4(acc[8], acc[9], acc[10], acc[11]);
    gr[3] = make_float4(acc[12], acc[13], 0.0f, 0.0f);
}

__global__ void __launch_bounds__(256) k_field_chain(int P, const float* __restrict__ scaling, const float* __restrict__ quaternions,
                                                     float density_factor, const float4* __restrict__ grec, float* __restrict__ d_points,
                                                     float* __restrict__ d_scaling, float* __restrict__ d_quaternions,
                                                     float* __restrict__ d_strengths) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const size_t p3 = 3 * (size_t)p, p4 = 4 * (size_t)p;
    const float4 g0 = grec[4 * (size_t)p], g1 = grec[4 * (size_t)p + 1], g2 = grec[4 * (size_t)p + 2], g3 = grec[4 * (size_t)p + 3];
    d_points[p3] = g0.x; d_points[p3 + 1] = g0.y; d_points[p3 + 2] = g0.z;
    d_strengths[p] = __fmul_rn(g0.w, density_factor);
    const float s[3] = {scaling[p3], scaling[p3 + 1], scaling[p3 + 2]};
    const float qr = quaternions[p4], qi = quaternions[p4 + 1], qj = quaternions[p4 + 2], qk = quaternions[p4 + 3];
    float R[9], t;
    quat_to_matrix_rn(qr, qi, qj, qk, R, t);
    const float inv[3] = {inv_scale_rn(s[0]), inv_scale_rn(s[1]), inv_scale_rn(s[2])};
    const float dA[9] = {g1.x, g1.y, g1.z, g1.w, g2.x, g2.y, g2.z, g2.w, g3.x};
    float dR[9];
#pragma unroll
    for (int e = 0; e < 9; e++) dR[e] = dA[e] * inv[e % 3];
    int km = 0;
    float sm = s[0];
    if (s[1] < sm) { sm = s[1]; km = 1; }
    if (s[2] < sm) { sm = s[2]; km = 2; }
#pragma unroll
    for (int j = 0; j < 3; j++) {
        // A = R * inv[None, :]: d inv_j = sum_i dA_ij R_ij; inv = reciprocal(clamp(s, 1e-8)): -g inv^2, zero below the clamp
        const float dinv = (dA[j] * R[j] + dA[3 + j] * R[3 + j]) + dA[6 + j] * R[6 + j];
        float ds = s[j] >= 1e-8f ? -(dinv * (inv[j] * inv[j])) : 0.0f;
        if (j == km) ds += g3.y;  // scaling.min(dim=-1)[0]: the gradient goes to the returned index
        d_scaling[p3 + j] = ds;
    }
    float dq[4];
    quat_to_matrix_vjp(qr, qi, qj, qk, t, dR, dq);
    d_quaternions[p4] = dq[0]; d_quaternions[p4 + 1] = dq[1]; d_quaternions[p4 + 2] = dq[2]; d_quaternions[p4 + 3] = dq[3];
}

static int field_check(const char* who, int N, int K, int P, int R, const float* x, const int64_t* rows, const int64_t* row_idx,
                       const float* points, const float* scaling, const float* quaternions, const float* strengths, bool want_sdf,
                       void* ws, size_t ws_bytes, size_t need) {
    if (N < 0 || P < 0 || R < 0) { set_error("%s: negative size (N = %d, P = %d, R = %d)", who, N, P, R); return GSR_ERR_INVALID; }
    if (K < 1 || K > FIELD_KMAX) { set_error("%s: K = %d outside 1..%d", who, K, FIELD_KMAX); return GSR_ERR_INVALID; }
    if (!row_idx && R != N) { set_error("%s: row_idx == NULL needs R == N (%d != %d)", who, R, N); return GSR_ERR_INVALID; }
    if (N == 0) return GSR_OK;
    if (!x || !rows || !points || !quaternions || !strengths) {
        set_error("%s: an output was requested without its inputs (x, rows, points, quaternions and strengths are required)", who);
        return GSR_ERR_INVALID;
    }
    if (!scaling) {
        set_error(want_sdf ? "%s: the sdf needs beta, whose input scaling is null" : "%s: scaling is null", who);
        return GSR_ERR_INVALID;
    }
    if (!ws || ((uintptr_t)ws & 15) || ws_bytes < need) {
        set_error("%s: workspace null, not 16-byte aligned or too small (%zu < %zu)", who, ws_bytes, need);
        return GSR_ERR_WORKSPACE;
    }
    return GSR_OK;
}

template <int W>
static void launch_field(const FieldIn& a, float* d, float* o, float* b, float* s, cudaStream_t st) {
    const size_t threads = (size_t)a.N * W;
    k_field<W><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(a, d, o, b, s);
}
template <int W>
static void launch_field_backward(const FieldIn& a, const FieldGrad& g, const FieldDet* det, cudaStream_t st) {
    const size_t threads = (size_t)a.N * W;
    if (det) k_field_backward<W, true><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(a, g, *det);
    else k_field_backward<W, false><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(a, g, FieldDet{});
}
static int seg_width(int K) { int w = 1; while (w < K) w <<= 1; return w; }

// det: the deterministic backward (gsr_sugar_field_backward_det); the workspace is then its scratch, laid out by FieldDetLayout.
struct FieldDetLayout {
    size_t G, dmin, group, total;
    GroupLayout gl;
    FieldDetLayout(int N, int K, int P) : gl((size_t)(N < 0 ? 0 : N) * (size_t)(K < 0 ? 0 : K), P < 0 ? 0 : P) {
        const size_t n = N < 0 ? 0 : N;
        size_t o = align_up(2 * gsr_sugar_field_bytes(P), 256);  // rec, grec: the default backward's workspace
        G = o;     o = align_up(o + 4 * n, 256);
        dmin = o;  o = align_up(o + 4 * n, 256);
        group = o;
        total = o + gl.total;
    }
};

static int det_scratch_check(const char* who, const void* scratch) {
    if (!scratch) { set_error("%s: scratch is NULL", who); return GSR_ERR_INVALID; }
    if ((uintptr_t)scratch & 15) { set_error("%s: scratch is not 16-byte aligned", who); return GSR_ERR_INVALID; }
    return GSR_OK;
}

static int det_ids_check(const char* who, int N, int K, int per_sample) {
    if (N > 0 && K >= 1 && K <= FIELD_KMAX && (uint64_t)N * (uint64_t)(K + per_sample) >= (1ull << 32)) {
        set_error("%s: %llu partial ids, at or above 2^32", who, (unsigned long long)((uint64_t)N * (uint64_t)(K + per_sample)));
        return GSR_ERR_INVALID;
    }
    return GSR_OK;
}

// ================================================================================================================================
// The better-normal regulariser and the projection estimate of the coarse trainers ("CD/" = sugar/sugar_trainers/coarse_density.py
// :704-707 and :756-780; coarse_sdf.py :735-759 is the same code), over the same samples and knn_idx rows as the field.  n_g is
// column k_g of quaternion_to_matrix(q_g), k_g the lowest index of min(s_g) (get_normals -> get_smallest_axis, SS/:801-839).
//
//   k_normal_prepare  one thread per Gaussian: a 32-byte record {p.xyz, c = clamp(min s, 1e-6)^2 | n.xyz, 0}, two aligned
//                     16-byte loads per pair
//   k_normal<W>       one segment of W = pow2 >= K lanes per sample, lane = neighbour j of knn_idx[i], i = sdf_gaussian_idx[n]:
//                     sigma_j = sign(n_j . n_i), w_j = (o_nj |(x - p_j) . sigma_j n_j|) / c_j, w_hat = w / clamp(sum w, 1e-6),
//                     r = n_i - sum_j w_hat_j sigma_j n_j, loss = (r0^2 + r1^2) + r2^2; and the estimate (x - p_i) . n_i
//   k_normal_backward<W>  recomputes the forward; dL/dx per sample without atomics, the normal (and, for the estimate, centre)
//                     gradients of every pair into a per-Gaussian 32-byte scratch with 16-byte RED.ADDs.  sigma, the weights,
//                     their sum, o and c are detached, as the trainer (sdf_better_normal_gradient_through_normal_only) has them
//   k_normal_chain    one thread per Gaussian: the normal gradient -> dL/dquaternions through column k_g of quaternion_to_matrix;
//                     dL/dpoints
//
// Dots are pinned as (a0 b0 + a1 b1) + a2 b2 and the K-sums are seg_sum's fixed butterfly; every other op is one IEEE rounding.
__global__ void __launch_bounds__(256) k_normal_prepare(int P, const float* __restrict__ points, const float* __restrict__ scaling,
                                                        const float* __restrict__ quaternions, float4* __restrict__ rec) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const size_t p3 = 3 * (size_t)p, p4 = 4 * (size_t)p;
    float R[9], t;
    quat_to_matrix_rn(quaternions[p4], quaternions[p4 + 1], quaternions[p4 + 2], quaternions[p4 + 3], R, t);
    int km = 0;
    float sm = scaling[p3];
    if (scaling[p3 + 1] < sm) { sm = scaling[p3 + 1]; km = 1; }
    if (scaling[p3 + 2] < sm) { sm = scaling[p3 + 2]; km = 2; }
    const float cm = sm < 1e-6f ? 1e-6f : sm;  // clamp(min=1e-6), NaN passes
    rec[2 * (size_t)p] = make_float4(points[p3], points[p3 + 1], points[p3 + 2], __fmul_rn(cm, cm));
    rec[2 * (size_t)p + 1] = make_float4(R[km], R[3 + km], R[6 + km], 0.0f);
}

struct NormalIn {
    int N, K, P;
    const float* x;          // [N,3] sdf_samples
    const int64_t* gidx;     // [N]   sdf_gaussian_idx
    const int64_t* knn;      // [P,K] knn_idx (loss only)
    const float* opac;       // [N,K] closest_gaussian_opacities (loss only)
    const float4* rec;       // [P] x 2 float4
};

__device__ __forceinline__ float dot3_rn(float a0, float a1, float a2, float b0, float b1, float b2) {
    return __fadd_rn(__fadd_rn(__fmul_rn(a0, b0), __fmul_rn(a1, b1)), __fmul_rn(a2, b2));
}

// The sample's own Gaussian i, read by every lane of the segment.
struct NormalSample {
    bool ok;          // i inside [0, P)
    int64_t i;
    float x0, x1, x2;
    float4 pc, nz;    // (p_i, c_i), (n_i, 0)
};

__device__ __forceinline__ void normal_sample(const NormalIn& a, int64_t n, NormalSample& s) {
    s.i = a.gidx[n];
    s.ok = s.i >= 0 && s.i < a.P;
    s.x0 = a.x[3 * n]; s.x1 = a.x[3 * n + 1]; s.x2 = a.x[3 * n + 2];
    const float nan = __int_as_float(0x7fc00000);
    s.pc = s.nz = make_float4(nan, nan, nan, nan);
    if (s.ok) { s.pc = __ldg(a.rec + 2 * s.i); s.nz = __ldg(a.rec + 2 * s.i + 1); }
}

// One (sample, neighbour) pair of the loss: sigma_j, n'_j = sigma_j n_j and the raw weight w_j.  An index outside its array is
// never read and gives w = NaN, which the segment sum spreads over the sample.
struct NormalPair {
    bool ok;
    int64_t j;
    float sg, m0, m1, m2, w;
};

__device__ __forceinline__ void normal_pair(const NormalIn& a, int64_t n, int k, const NormalSample& s, NormalPair& f) {
    f.j = s.ok ? a.knn[s.i * a.K + k] : -1;
    f.ok = s.ok && f.j >= 0 && f.j < a.P;
    if (!f.ok) {
        f.sg = f.m0 = f.m1 = f.m2 = f.w = __int_as_float(0x7fc00000);
        return;
    }
    const float4 pc = __ldg(a.rec + 2 * f.j), nz = __ldg(a.rec + 2 * f.j + 1);
    const float dt = dot3_rn(nz.x, nz.y, nz.z, s.nz.x, s.nz.y, s.nz.z);
    f.sg = (float)((0.0f < dt) - (dt < 0.0f));  // torch.sign: sign(0) = 0 drops the neighbour
    f.m0 = __fmul_rn(nz.x, f.sg); f.m1 = __fmul_rn(nz.y, f.sg); f.m2 = __fmul_rn(nz.z, f.sg);
    const float d = fabsf(dot3_rn(__fsub_rn(s.x0, pc.x), __fsub_rn(s.x1, pc.y), __fsub_rn(s.x2, pc.z), f.m0, f.m1, f.m2));
    f.w = __fdiv_rn(__fmul_rn(a.opac[n * a.K + k], d), pc.w);
}

__device__ __forceinline__ float normal_what(float w, float S) { return __fdiv_rn(w, S < 1e-6f ? 1e-6f : S); }  // clamp(min=1e-6), NaN passes

// The loss's segment reductions: w_hat of this lane and T = sum_j w_hat_j n'_j (every lane gets T); S = sum_j w_j.
template <int W>
__device__ __forceinline__ float normal_sums(const NormalPair& f, float& T0, float& T1, float& T2, float& S) {
    S = seg_sum<W>(f.w);
    const float wh = normal_what(f.w, S);
    T0 = seg_sum<W>(__fmul_rn(wh, f.m0));
    T1 = seg_sum<W>(__fmul_rn(wh, f.m1));
    T2 = seg_sum<W>(__fmul_rn(wh, f.m2));
    return wh;
}

template <int W>
__global__ void __launch_bounds__(256) k_normal(NormalIn a, float* __restrict__ out_loss, float* __restrict__ out_est) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t n = (int64_t)(t / W);
    const int k = (int)(t % W);
    const bool active = n < a.N && k < a.K;  // every lane takes part in the shuffles
    NormalSample s;
    if (active) normal_sample(a, n, s);
    if (out_loss) {
        NormalPair f;
        f.w = f.m0 = f.m1 = f.m2 = 0.0f;
        if (active) normal_pair(a, n, k, s, f);
        float T0, T1, T2, S;
        normal_sums<W>(f, T0, T1, T2, S);
        if (active && k == 0) {
            const float r0 = __fsub_rn(s.nz.x, T0), r1 = __fsub_rn(s.nz.y, T1), r2 = __fsub_rn(s.nz.z, T2);
            out_loss[n] = dot3_rn(r0, r1, r2, r0, r1, r2);
        }
    }
    if (out_est && active && k == 0)
        out_est[n] = dot3_rn(__fsub_rn(s.x0, s.pc.x), __fsub_rn(s.x1, s.pc.y), __fsub_rn(s.x2, s.pc.z), s.nz.x, s.nz.y, s.nz.z);
}

struct NormalGrad {
    const float* g_loss;  // [N] dL/dloss
    const float* g_est;   // [N] dL/destimate
    float* dx;            // [N,3]
    float4* grec;         // [P] x 2 float4: (dp.xyz, 0), (dn.xyz, 0)
};

// The loss's neighbour term, dL/dn_j of pair (n, j): -dn_i w_hat_j sigma_j, dn_i = dL/dloss * 2 r.  k_normal_backward adds it with
// atomics, k_normal_reduce in id order: one formula.
__device__ __forceinline__ float4 normal_neighbour_term(float dn0, float dn1, float dn2, float wh, float sg) {
    return make_float4(__fmul_rn(__fmul_rn(-dn0, wh), sg), __fmul_rn(__fmul_rn(-dn1, wh), sg), __fmul_rn(__fmul_rn(-dn2, wh), sg), 0.0f);
}

// What DET adds to the default backward: per-sample values the partials need and one key per partial id n * (KS + 1) + slot, KS
// = K neighbour slots with the loss, none without.
struct NormalDet {
    float4* sc;     // [N]   (the loss's dn_i, S = sum_j w_j)
    float4* own;    // [N,2] the sample's own term: (dn_i, 0), (-dx, 0)
    uint32_t* key;  // [N*(KS+1)] slot k < KS: knn[i, k], slot KS: i; P where the slot adds nothing
    uint32_t* id;   // [N*(KS+1)] = the position
    int KS;
};

template <int W, bool DET>
__global__ void __launch_bounds__(256) k_normal_backward(NormalIn a, NormalGrad b, NormalDet det) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t n = (int64_t)(t / W);
    const int k = (int)(t % W);
    const bool active = n < a.N && k < a.K;
    const size_t pid0 = (size_t)n * (det.KS + 1);  // DET: the sample's first partial id
    NormalSample s;
    s.ok = true;
    if (active) normal_sample(a, n, s);
    float dn0 = 0.0f, dn1 = 0.0f, dn2 = 0.0f;  // dL/dn_i of this sample (lane 0)
    bool bad = active && !s.ok;
    if (b.g_loss) {
        NormalPair f;
        f.w = f.m0 = f.m1 = f.m2 = 0.0f;
        f.ok = true;
        if (active) normal_pair(a, n, k, s, f);
        float T0, T1, T2, S;
        const float wh = normal_sums<W>(f, T0, T1, T2, S);
        if (seg_sum<W>(f.ok ? 0.0f : 1.0f) != 0.0f) bad = active;
        if (active && !bad) {
            // loss = sum_c r_c^2: dr = g * (2 r); r = n_i - T: dn_i = dr, dT = -dr; T = sum_j w_hat_j (sigma_j n_j)
            const float gl = b.g_loss[n];
            dn0 = __fmul_rn(gl, __fmul_rn(2.0f, __fsub_rn(s.nz.x, T0)));
            dn1 = __fmul_rn(gl, __fmul_rn(2.0f, __fsub_rn(s.nz.y, T1)));
            dn2 = __fmul_rn(gl, __fmul_rn(2.0f, __fsub_rn(s.nz.z, T2)));
            if (DET) {
                if (k == 0) det.sc[n] = make_float4(dn0, dn1, dn2, S);
            } else if (f.ok) {
                atomicAdd(b.grec + 2 * f.j + 1, normal_neighbour_term(dn0, dn1, dn2, wh, f.sg));
            }
        }
        if (DET && active) {
            det.key[pid0 + k] = bad || !f.ok ? (uint32_t)a.P : (uint32_t)f.j;
            det.id[pid0 + k] = (uint32_t)(pid0 + k);
        }
    }
    if (!active || k != 0) return;
    float dx0 = 0.0f, dx1 = 0.0f, dx2 = 0.0f;
    if (b.g_est && !bad) {
        // est = sum_c (x - p_i)_c n_ic: d(x - p_i) = g n_i, dn_i += g (x - p_i)
        const float ge = b.g_est[n];
        dx0 = __fmul_rn(ge, s.nz.x); dx1 = __fmul_rn(ge, s.nz.y); dx2 = __fmul_rn(ge, s.nz.z);
        dn0 = __fadd_rn(dn0, __fmul_rn(ge, __fsub_rn(s.x0, s.pc.x)));
        dn1 = __fadd_rn(dn1, __fmul_rn(ge, __fsub_rn(s.x1, s.pc.y)));
        dn2 = __fadd_rn(dn2, __fmul_rn(ge, __fsub_rn(s.x2, s.pc.z)));
        if (!DET) atomicAdd(b.grec + 2 * s.i, make_float4(-dx0, -dx1, -dx2, 0.0f));
    }
    if (DET) {
        const bool adds = !bad && (b.g_loss || b.g_est);
        det.key[pid0 + det.KS] = adds ? (uint32_t)s.i : (uint32_t)a.P;
        det.id[pid0 + det.KS] = (uint32_t)(pid0 + det.KS);
        if (adds) {
            det.own[2 * n] = make_float4(dn0, dn1, dn2, 0.0f);
            det.own[2 * n + 1] = b.g_est ? make_float4(-dx0, -dx1, -dx2, 0.0f) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        }
    } else if (!bad && (b.g_loss || b.g_est)) {
        atomicAdd(b.grec + 2 * s.i + 1, make_float4(dn0, dn1, dn2, 0.0f));
    }
    // an index outside its array: this sample adds nothing and its dL/dx is NaN
    if (bad) dx0 = dx1 = dx2 = __int_as_float(0x7fc00000);
    if (b.dx) { b.dx[3 * n] = dx0; b.dx[3 * n + 1] = dx1; b.dx[3 * n + 2] = dx2; }
}

// DET: one thread per Gaussian g sums its partials in ascending id from +0.0: a neighbour slot adds normal_neighbour_term
// (recomputed) to the normal, an own slot its stored (dn_i, -dx) to the normal and the centre.  Writes g's gradient record for
// the unchanged k_normal_chain.
__global__ void __launch_bounds__(256) k_normal_reduce(NormalIn a, float4* __restrict__ grec, const float4* __restrict__ sc,
                                                       const float4* __restrict__ own, int KS, const uint32_t* __restrict__ ids,
                                                       const uint32_t* __restrict__ seg) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.P) return;
    float p0 = 0.0f, p1 = 0.0f, p2 = 0.0f, n0 = 0.0f, n1 = 0.0f, n2 = 0.0f;
    const uint32_t e = seg[g + 1], K1 = (uint32_t)KS + 1;
    for (uint32_t q = seg[g]; q < e; q++) {
        const uint32_t pid = ids[q];
        const int64_t n = pid / K1;
        const int k = (int)(pid - (uint32_t)n * K1);
        float4 v;
        if (k == KS) {
            const float4 op = own[2 * n + 1];
            p0 = __fadd_rn(p0, op.x); p1 = __fadd_rn(p1, op.y); p2 = __fadd_rn(p2, op.z);
            v = own[2 * n];
        } else {
            NormalSample s;
            normal_sample(a, n, s);
            NormalPair f;
            normal_pair(a, n, k, s, f);
            const float4 c = sc[n];
            v = normal_neighbour_term(c.x, c.y, c.z, normal_what(f.w, c.w), f.sg);
        }
        n0 = __fadd_rn(n0, v.x); n1 = __fadd_rn(n1, v.y); n2 = __fadd_rn(n2, v.z);
    }
    grec[2 * (size_t)g] = make_float4(p0, p1, p2, 0.0f);
    grec[2 * (size_t)g + 1] = make_float4(n0, n1, n2, 0.0f);
}

__global__ void __launch_bounds__(256) k_normal_chain(int P, const float* __restrict__ scaling, const float* __restrict__ quaternions,
                                                      const float4* __restrict__ grec, float* __restrict__ d_points,
                                                      float* __restrict__ d_quaternions) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const size_t p3 = 3 * (size_t)p, p4 = 4 * (size_t)p;
    const float4 gp = grec[2 * (size_t)p], gn = grec[2 * (size_t)p + 1];
    d_points[p3] = gp.x; d_points[p3 + 1] = gp.y; d_points[p3 + 2] = gp.z;
    int km = 0;
    float sm = scaling[p3];
    if (scaling[p3 + 1] < sm) { sm = scaling[p3 + 1]; km = 1; }
    if (scaling[p3 + 2] < sm) km = 2;
    const float qr = quaternions[p4], qi = quaternions[p4 + 1], qj = quaternions[p4 + 2], qk = quaternions[p4 + 3];
    float R[9], t;
    quat_to_matrix_rn(qr, qi, qj, qk, R, t);
    float G[9] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};  // dL/dR: only column km (the gather's backward)
    G[km] = gn.x; G[3 + km] = gn.y; G[6 + km] = gn.z;
    float dq[4];
    quat_to_matrix_vjp(qr, qi, qj, qk, t, G, dq);
    d_quaternions[p4] = dq[0]; d_quaternions[p4 + 1] = dq[1]; d_quaternions[p4 + 2] = dq[2]; d_quaternions[p4 + 3] = dq[3];
}

static int normal_check(const char* who, int N, int K, int P, const float* x, const int64_t* gidx, const int64_t* knn,
                        const float* points, const float* scaling, const float* quaternions, const float* opac, bool want_loss,
                        void* ws, size_t ws_bytes, size_t need) {
    if (N < 0 || P < 0) { set_error("%s: negative size (N = %d, P = %d)", who, N, P); return GSR_ERR_INVALID; }
    if (K < 1 || K > FIELD_KMAX) { set_error("%s: K = %d outside 1..%d", who, K, FIELD_KMAX); return GSR_ERR_INVALID; }
    if (N == 0) return GSR_OK;
    if (!x || !gidx || !points || !scaling || !quaternions) {
        set_error("%s: an output was requested without its inputs (x, gidx, points, scaling and quaternions are required)", who);
        return GSR_ERR_INVALID;
    }
    if (want_loss && (!knn || !opac)) {
        set_error("%s: the better-normal loss needs knn_idx and the opacities", who);
        return GSR_ERR_INVALID;
    }
    if (!ws || ((uintptr_t)ws & 15) || ws_bytes < need) {
        set_error("%s: workspace null, not 16-byte aligned or too small (%zu < %zu)", who, ws_bytes, need);
        return GSR_ERR_WORKSPACE;
    }
    return GSR_OK;
}

// Without the loss every sample needs one lane.
static int normal_width(int K, bool loss) { return loss ? seg_width(K) : 1; }

template <int W>
static void launch_normal(const NormalIn& a, float* l, float* e, cudaStream_t st) {
    const size_t threads = (size_t)a.N * W;
    k_normal<W><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(a, l, e);
}
template <int W>
static void launch_normal_backward(const NormalIn& a, const NormalGrad& g, const NormalDet* det, cudaStream_t st) {
    const size_t threads = (size_t)a.N * W;
    if (det) k_normal_backward<W, true><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(a, g, *det);
    else k_normal_backward<W, false><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(a, g, NormalDet{});
}

// det: the deterministic backward (gsr_sugar_sdf_normal_backward_det); the workspace is then its scratch, laid out by NormalDetLayout
// for KS = K neighbour slots per sample with the loss, 0 without.
struct NormalDetLayout {
    size_t sc, own, group, total;
    GroupLayout gl;
    NormalDetLayout(int N, int KS, int P) : gl((size_t)(N < 0 ? 0 : N) * (size_t)(KS < 0 ? 1 : KS + 1), P < 0 ? 0 : P) {
        const size_t n = N < 0 ? 0 : N;
        size_t o = align_up(2 * gsr_sugar_sdf_normal_bytes(P), 256);  // rec, grec: the default backward's workspace
        sc = o;   o = align_up(o + 16 * n, 256);
        own = o;  o = align_up(o + 32 * n, 256);
        group = o;
        total = o + gl.total;
    }
};

}  // namespace gsr

using namespace gsr;

size_t gsr_sugar_field_bytes(int32_t P) { return 64 * (size_t)(P < 0 ? 0 : P); }

int gsr_sugar_field(int32_t N, int32_t K, int32_t P, int32_t R, const float* x, const int64_t* rows, const int64_t* row_idx,
                    const float* points, const float* scaling, const float* quaternions, const float* strengths, float density_factor,
                    float opacity_min_clamp, float sdf_offset, float* out_density, float* out_opac, float* out_beta, float* out_sdf,
                    void* ws, size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_sugar_field");
    const cudaStream_t st = (cudaStream_t)stream;
    int rc = field_check("gsr_sugar_field", N, K, P, R, x, rows, row_idx, points, scaling, quaternions, strengths, out_sdf != nullptr, ws,
                         ws_bytes, gsr_sugar_field_bytes(P));
    if (rc != GSR_OK || N == 0) return rc;
    if (!out_density && !out_opac && !out_beta && !out_sdf) return GSR_OK;
    float4* rec = (float4*)ws;
    if (P > 0) k_field_prepare<<<(P + 255) / 256, 256, 0, st>>>(P, points, scaling, quaternions, strengths, density_factor, rec);
    const FieldIn a{N, K, P, R, x, rows, row_idx, rec, opacity_min_clamp, sdf_offset};
    switch (seg_width(K)) {
        case 1: launch_field<1>(a, out_density, out_opac, out_beta, out_sdf, st); break;
        case 2: launch_field<2>(a, out_density, out_opac, out_beta, out_sdf, st); break;
        case 4: launch_field<4>(a, out_density, out_opac, out_beta, out_sdf, st); break;
        case 8: launch_field<8>(a, out_density, out_opac, out_beta, out_sdf, st); break;
        case 16: launch_field<16>(a, out_density, out_opac, out_beta, out_sdf, st); break;
        default: launch_field<32>(a, out_density, out_opac, out_beta, out_sdf, st); break;
    }
    return check_launch("gsr_sugar_field", false, st);
}

size_t gsr_sugar_field_backward_det_bytes(int32_t N, int32_t K, int32_t P) { return FieldDetLayout(N, K, P).total; }

static int sugar_field_backward_impl(int N, int K, int P, int R, const float* x, const int64_t* rows, const int64_t* row_idx,
                                     const float* points, const float* scaling, const float* quaternions, const float* strengths,
                                     float density_factor, float opacity_min_clamp, float sdf_offset, const float* g_density,
                                     const float* g_opac, const float* g_beta, const float* g_sdf, float* dx, float* d_points,
                                     float* d_scaling, float* d_quaternions, float* d_strengths, void* ws, size_t ws_bytes, bool det,
                                     cudaStream_t st) {
    const char* who = det ? "gsr_sugar_field_backward_det" : "gsr_sugar_field_backward";
    if (det) {
        int rc = det_ids_check(who, N, K, 0);
        if (rc == GSR_OK && N > 0) rc = det_scratch_check(who, ws);
        if (rc != GSR_OK) return rc;
    }
    int rc = field_check(who, N, K, P, R, x, rows, row_idx, points, scaling, quaternions, strengths, g_sdf != nullptr, ws, ws_bytes,
                         det ? gsr_sugar_field_backward_det_bytes(N, K, P) : 2 * gsr_sugar_field_bytes(P));
    if (rc != GSR_OK || N == 0) return rc;
    if (P > 0 && (!d_points || !d_scaling || !d_quaternions || !d_strengths)) {
        set_error("%s: dL_dpoints, dL_dscaling, dL_dquaternions and dL_dstrengths are required", who);
        return GSR_ERR_INVALID;
    }
    float4* rec = (float4*)ws;
    float4* grec = rec + 4 * (size_t)P;
    if (P > 0) {
        k_field_prepare<<<(P + 255) / 256, 256, 0, st>>>(P, points, scaling, quaternions, strengths, density_factor, rec);
        if (!det) cudaMemsetAsync(grec, 0, gsr_sugar_field_bytes(P), st);
    }
    const FieldIn a{N, K, P, R, x, rows, row_idx, rec, opacity_min_clamp, sdf_offset};
    const FieldGrad g{g_density, g_opac, g_beta, g_sdf, dx, grec};
    const FieldDetLayout L(N, K, P);
    char* w = (char*)ws;
    const FieldDet fd{(float*)(w + L.G), (float*)(w + L.dmin), (uint32_t*)(w + L.group + L.gl.keys0), (uint32_t*)(w + L.group + L.gl.vals0)};
    const FieldDet* dp = det ? &fd : nullptr;
    switch (seg_width(K)) {
        case 1: launch_field_backward<1>(a, g, dp, st); break;
        case 2: launch_field_backward<2>(a, g, dp, st); break;
        case 4: launch_field_backward<4>(a, g, dp, st); break;
        case 8: launch_field_backward<8>(a, g, dp, st); break;
        case 16: launch_field_backward<16>(a, g, dp, st); break;
        default: launch_field_backward<32>(a, g, dp, st); break;
    }
    if (det && P > 0) {
        const uint32_t* ids = group_ids((size_t)N * K, P, w + L.group, L.gl, st);
        k_field_reduce<<<(P + 255) / 256, 256, 0, st>>>(a, g, fd.G, fd.dmin, ids, (const uint32_t*)(w + L.group + L.gl.seg));
    }
    if (P > 0)
        k_field_chain<<<(P + 255) / 256, 256, 0, st>>>(P, scaling, quaternions, density_factor, grec, d_points, d_scaling, d_quaternions,
                                                        d_strengths);
    return check_launch(who, false, st);
}

int gsr_sugar_field_backward(int32_t N, int32_t K, int32_t P, int32_t R, const float* x, const int64_t* rows, const int64_t* row_idx,
                             const float* points, const float* scaling, const float* quaternions, const float* strengths,
                             float density_factor, float opacity_min_clamp, float sdf_offset, const float* dL_ddensity,
                             const float* dL_dopacities, const float* dL_dbeta, const float* dL_dsdf, float* dL_dx, float* dL_dpoints,
                             float* dL_dscaling, float* dL_dquaternions, float* dL_dstrengths, void* workspace, size_t workspace_bytes,
                             void* stream) {
    NvtxRange nvtx_("gsr_sugar_field_backward");
    return sugar_field_backward_impl(N, K, P, R, x, rows, row_idx, points, scaling, quaternions, strengths, density_factor,
                                     opacity_min_clamp, sdf_offset, dL_ddensity, dL_dopacities, dL_dbeta, dL_dsdf, dL_dx, dL_dpoints,
                                     dL_dscaling, dL_dquaternions, dL_dstrengths, workspace, workspace_bytes, false, (cudaStream_t)stream);
}

int gsr_sugar_field_backward_det(int32_t N, int32_t K, int32_t P, int32_t R, const float* x, const int64_t* rows, const int64_t* row_idx,
                                 const float* points, const float* scaling, const float* quaternions, const float* strengths,
                                 float density_factor, float opacity_min_clamp, float sdf_offset, const float* dL_ddensity,
                                 const float* dL_dopacities, const float* dL_dbeta, const float* dL_dsdf, float* dL_dx, float* dL_dpoints,
                                 float* dL_dscaling, float* dL_dquaternions, float* dL_dstrengths, void* scratch, size_t scratch_bytes,
                                 void* stream) {
    NvtxRange nvtx_("gsr_sugar_field_backward_det");
    return sugar_field_backward_impl(N, K, P, R, x, rows, row_idx, points, scaling, quaternions, strengths, density_factor,
                                     opacity_min_clamp, sdf_offset, dL_ddensity, dL_dopacities, dL_dbeta, dL_dsdf, dL_dx, dL_dpoints,
                                     dL_dscaling, dL_dquaternions, dL_dstrengths, scratch, scratch_bytes, true, (cudaStream_t)stream);
}

size_t gsr_sugar_sdf_normal_bytes(int32_t P) { return 32 * (size_t)(P < 0 ? 0 : P); }

int gsr_sugar_sdf_normal(int32_t N, int32_t K, int32_t P, const float* x, const int64_t* gidx, const int64_t* knn,
                         const float* points, const float* scaling, const float* quaternions, const float* opac, float* out_loss,
                         float* out_est, void* ws, size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_sugar_sdf_normal");
    const cudaStream_t st = (cudaStream_t)stream;
    int rc = normal_check("gsr_sugar_sdf_normal", N, K, P, x, gidx, knn, points, scaling, quaternions, opac, out_loss != nullptr, ws,
                          ws_bytes, gsr_sugar_sdf_normal_bytes(P));
    if (rc != GSR_OK || N == 0) return rc;
    if (!out_loss && !out_est) return GSR_OK;
    float4* rec = (float4*)ws;
    if (P > 0) k_normal_prepare<<<(P + 255) / 256, 256, 0, st>>>(P, points, scaling, quaternions, rec);
    const NormalIn a{N, K, P, x, gidx, knn, opac, rec};
    switch (normal_width(K, out_loss != nullptr)) {
        case 1: launch_normal<1>(a, out_loss, out_est, st); break;
        case 2: launch_normal<2>(a, out_loss, out_est, st); break;
        case 4: launch_normal<4>(a, out_loss, out_est, st); break;
        case 8: launch_normal<8>(a, out_loss, out_est, st); break;
        case 16: launch_normal<16>(a, out_loss, out_est, st); break;
        default: launch_normal<32>(a, out_loss, out_est, st); break;
    }
    return check_launch("gsr_sugar_sdf_normal", false, st);
}

size_t gsr_sugar_sdf_normal_backward_det_bytes(int32_t N, int32_t K, int32_t P, int with_loss) {
    return NormalDetLayout(N, with_loss ? K : 0, P).total;
}

static int sugar_sdf_normal_backward_impl(int N, int K, int P, const float* x, const int64_t* gidx, const int64_t* knn,
                                          const float* points, const float* scaling, const float* quaternions, const float* opac,
                                          const float* g_loss, const float* g_est, float* dx, float* d_points, float* d_quaternions,
                                          void* ws, size_t ws_bytes, bool det, cudaStream_t st) {
    const char* who = det ? "gsr_sugar_sdf_normal_backward_det" : "gsr_sugar_sdf_normal_backward";
    if (det) {
        int rc = g_loss ? det_ids_check(who, N, K, 1) : GSR_OK;
        if (rc == GSR_OK && N > 0) rc = det_scratch_check(who, ws);
        if (rc != GSR_OK) return rc;
    }
    int rc = normal_check(who, N, K, P, x, gidx, knn, points, scaling, quaternions, opac, g_loss != nullptr, ws, ws_bytes,
                          det ? gsr_sugar_sdf_normal_backward_det_bytes(N, K, P, g_loss != nullptr) : 2 * gsr_sugar_sdf_normal_bytes(P));
    if (rc != GSR_OK || N == 0) return rc;
    if (P > 0 && (!d_points || !d_quaternions)) {
        set_error("%s: dL_dpoints and dL_dquaternions are required", who);
        return GSR_ERR_INVALID;
    }
    float4* rec = (float4*)ws;
    float4* grec = rec + 2 * (size_t)P;
    if (P > 0) {
        k_normal_prepare<<<(P + 255) / 256, 256, 0, st>>>(P, points, scaling, quaternions, rec);
        if (!det) cudaMemsetAsync(grec, 0, gsr_sugar_sdf_normal_bytes(P), st);
    }
    const NormalIn a{N, K, P, x, gidx, knn, opac, rec};
    const NormalGrad g{g_loss, g_est, dx, grec};
    const int KS = g_loss ? K : 0;
    const NormalDetLayout L(N, KS, P);
    char* w = (char*)ws;
    const NormalDet nd{(float4*)(w + L.sc), (float4*)(w + L.own), (uint32_t*)(w + L.group + L.gl.keys0),
                       (uint32_t*)(w + L.group + L.gl.vals0), KS};
    const NormalDet* dp = det ? &nd : nullptr;
    switch (normal_width(K, g_loss != nullptr)) {
        case 1: launch_normal_backward<1>(a, g, dp, st); break;
        case 2: launch_normal_backward<2>(a, g, dp, st); break;
        case 4: launch_normal_backward<4>(a, g, dp, st); break;
        case 8: launch_normal_backward<8>(a, g, dp, st); break;
        case 16: launch_normal_backward<16>(a, g, dp, st); break;
        default: launch_normal_backward<32>(a, g, dp, st); break;
    }
    if (det && P > 0) {
        const uint32_t* ids = group_ids((size_t)N * (KS + 1), P, w + L.group, L.gl, st);
        k_normal_reduce<<<(P + 255) / 256, 256, 0, st>>>(a, grec, nd.sc, nd.own, KS, ids, (const uint32_t*)(w + L.group + L.gl.seg));
    }
    if (P > 0) k_normal_chain<<<(P + 255) / 256, 256, 0, st>>>(P, scaling, quaternions, grec, d_points, d_quaternions);
    return check_launch(who, false, st);
}

int gsr_sugar_sdf_normal_backward(int32_t N, int32_t K, int32_t P, const float* x, const int64_t* gidx, const int64_t* knn_idx,
                                  const float* points, const float* scaling, const float* quaternions, const float* opacities,
                                  const float* dL_dloss, const float* dL_destimate, float* dL_dx, float* dL_dpoints,
                                  float* dL_dquaternions, void* workspace, size_t workspace_bytes, void* stream) {
    NvtxRange nvtx_("gsr_sugar_sdf_normal_backward");
    return sugar_sdf_normal_backward_impl(N, K, P, x, gidx, knn_idx, points, scaling, quaternions, opacities, dL_dloss, dL_destimate,
                                          dL_dx, dL_dpoints, dL_dquaternions, workspace, workspace_bytes, false, (cudaStream_t)stream);
}

int gsr_sugar_sdf_normal_backward_det(int32_t N, int32_t K, int32_t P, const float* x, const int64_t* gidx, const int64_t* knn_idx,
                                      const float* points, const float* scaling, const float* quaternions, const float* opacities,
                                      const float* dL_dloss, const float* dL_destimate, float* dL_dx, float* dL_dpoints,
                                      float* dL_dquaternions, void* scratch, size_t scratch_bytes, void* stream) {
    NvtxRange nvtx_("gsr_sugar_sdf_normal_backward_det");
    return sugar_sdf_normal_backward_impl(N, K, P, x, gidx, knn_idx, points, scaling, quaternions, opacities, dL_dloss, dL_destimate,
                                          dL_dx, dL_dpoints, dL_dquaternions, scratch, scratch_bytes, true, (cudaStream_t)stream);
}
