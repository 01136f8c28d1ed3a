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
//
// Every elementwise torch op is one IEEE rounding here (explicit _rn intrinsics, accurate expf / logf / sqrtf, no FMA
// contraction) in the order SuGaR writes it.  torch's batched 3x3 matmul and its K-sum have no fixed order on the GPU, so the
// results are not claimed bit-identical to torch; the contract is the tolerance of tests/test_gpu_sugar_field.py.
#include "gsr_common.cuh"

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

template <int W>
__global__ void __launch_bounds__(256) k_field_backward(FieldIn a, FieldGrad b) {
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
    float ds0 = 0.0f, ds1 = 0.0f, ds2 = 0.0f;  // dL/dshift of this pair
    if (active) {
        // per-sample gradient reaching every o_nk through densities.sum(dim=-1)
        float G = b.g_density ? b.g_density[n] : 0.0f;
        float gbeta = b.g_beta ? b.g_beta[n] : 0.0f;
        if (b.g_sdf) {
            const float gs = b.g_sdf[n];
            const float beta = __fdiv_rn(bsum, (float)a.K);
            const float dh = field_dhat(d), cd = field_clampmin(dh, a.opacity_min_clamp);
            const float sq = sqrtf(__fmul_rn(-2.0f, logf(cd)));
            gbeta = __fadd_rn(gbeta, __fmul_rn(gs, __fsub_rn(sq, a.sdf_offset)));
            // sqrt: g / (2 result); -2 *: g * -2; log: g / x; clamp: where(x >= min); normalisation: g / (d + 1e-12)
            const float gm = __fdiv_rn(__fmul_rn(gs, beta), __fmul_rn(2.0f, sq));
            const float gcd = __fdiv_rn(__fmul_rn(gm, -2.0f), cd);
            const float gdh = dh >= a.opacity_min_clamp ? gcd : 0.0f;
            G = __fadd_rn(G, d >= 1.0f ? __fdiv_rn(gdh, __fadd_rn(d, 1e-12f)) : gdh);
        }
        if (f.ok) {
            const float go = b.g_opac ? __fadd_rn(G, b.g_opac[n * a.K + k]) : G;
            const float dfs = __fmul_rn(go, f.e);
            const float dqc = __fmul_rn(__fmul_rn(__fmul_rn(go, f.fs), f.e), -0.5f);
            const float dq = (f.q <= 1e8f) ? dqc : 0.0f;  // clamp(0, 1e8) passes where 0 <= q <= 1e8
            const float dw0 = __fmul_rn(2.0f, __fmul_rn(dq, f.w0)), dw1 = __fmul_rn(2.0f, __fmul_rn(dq, f.w1)),
                        dw2 = __fmul_rn(2.0f, __fmul_rn(dq, f.w2));
            ds0 = __fadd_rn(__fadd_rn(__fmul_rn(f.A[0], dw0), __fmul_rn(f.A[1], dw1)), __fmul_rn(f.A[2], dw2));
            ds1 = __fadd_rn(__fadd_rn(__fmul_rn(f.A[3], dw0), __fmul_rn(f.A[4], dw1)), __fmul_rn(f.A[5], dw2));
            ds2 = __fadd_rn(__fadd_rn(__fmul_rn(f.A[6], dw0), __fmul_rn(f.A[7], dw1)), __fmul_rn(f.A[8], dw2));
            const float dmin = (b.g_beta || b.g_sdf) ? __fdiv_rn(gbeta, (float)a.K) : 0.0f;
            float4* gr = b.grec + 4 * f.g;
            atomicAdd(gr, make_float4(-ds0, -ds1, -ds2, dfs));
            atomicAdd(gr + 1, make_float4(__fmul_rn(dw0, f.sx), __fmul_rn(dw1, f.sx), __fmul_rn(dw2, f.sx), __fmul_rn(dw0, f.sy)));
            atomicAdd(gr + 2, make_float4(__fmul_rn(dw1, f.sy), __fmul_rn(dw2, f.sy), __fmul_rn(dw0, f.sz), __fmul_rn(dw1, f.sz)));
            atomicAdd(gr + 3, make_float4(__fmul_rn(dw2, f.sz), dmin, 0.0f, 0.0f));
        } else {
            ds0 = ds1 = ds2 = __int_as_float(0x7fc00000);  // an index outside its array: NaN in this sample's dL/dx
        }
    }
    ds0 = seg_sum<W>(ds0);
    ds1 = seg_sum<W>(ds1);
    ds2 = seg_sum<W>(ds2);
    if (active && k == 0 && b.dx) {
        b.dx[3 * n] = ds0; b.dx[3 * n + 1] = ds1; b.dx[3 * n + 2] = ds2;
    }
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

size_t sugar_field_bytes(int P) { return 64 * (size_t)(P < 0 ? 0 : P); }

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
static void launch_field_backward(const FieldIn& a, const FieldGrad& g, cudaStream_t st) {
    const size_t threads = (size_t)a.N * W;
    k_field_backward<W><<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(a, g);
}
static int seg_width(int K) { int w = 1; while (w < K) w <<= 1; return w; }

int sugar_field_impl(int N, int K, int P, int R, const float* x, const int64_t* rows, const int64_t* row_idx, const float* points,
                     const float* scaling, const float* quaternions, const float* strengths, float density_factor,
                     float opacity_min_clamp, float sdf_offset, float* out_density, float* out_opac, float* out_beta, float* out_sdf,
                     void* ws, size_t ws_bytes, cudaStream_t st) {
    int rc = field_check("gsr_sugar_field", N, K, P, R, x, rows, row_idx, points, scaling, quaternions, strengths, out_sdf != nullptr, ws,
                         ws_bytes, sugar_field_bytes(P));
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

int sugar_field_backward_impl(int N, int K, int P, int R, const float* x, const int64_t* rows, const int64_t* row_idx,
                              const float* points, const float* scaling, const float* quaternions, const float* strengths,
                              float density_factor, float opacity_min_clamp, float sdf_offset, const float* g_density, const float* g_opac,
                              const float* g_beta, const float* g_sdf, float* dx, float* d_points, float* d_scaling, float* d_quaternions,
                              float* d_strengths, void* ws, size_t ws_bytes, cudaStream_t st) {
    int rc = field_check("gsr_sugar_field_backward", N, K, P, R, x, rows, row_idx, points, scaling, quaternions, strengths,
                         g_sdf != nullptr, ws, ws_bytes, 2 * sugar_field_bytes(P));
    if (rc != GSR_OK || N == 0) return rc;
    if (P > 0 && (!d_points || !d_scaling || !d_quaternions || !d_strengths)) {
        set_error("gsr_sugar_field_backward: dL_dpoints, dL_dscaling, dL_dquaternions and dL_dstrengths are required");
        return GSR_ERR_INVALID;
    }
    float4* rec = (float4*)ws;
    float4* grec = rec + 4 * (size_t)P;
    if (P > 0) {
        k_field_prepare<<<(P + 255) / 256, 256, 0, st>>>(P, points, scaling, quaternions, strengths, density_factor, rec);
        cudaMemsetAsync(grec, 0, sugar_field_bytes(P), st);
    }
    const FieldIn a{N, K, P, R, x, rows, row_idx, rec, opacity_min_clamp, sdf_offset};
    const FieldGrad g{g_density, g_opac, g_beta, g_sdf, dx, grec};
    switch (seg_width(K)) {
        case 1: launch_field_backward<1>(a, g, st); break;
        case 2: launch_field_backward<2>(a, g, st); break;
        case 4: launch_field_backward<4>(a, g, st); break;
        case 8: launch_field_backward<8>(a, g, st); break;
        case 16: launch_field_backward<16>(a, g, st); break;
        default: launch_field_backward<32>(a, g, st); break;
    }
    if (P > 0)
        k_field_chain<<<(P + 255) / 256, 256, 0, st>>>(P, scaling, quaternions, density_factor, grec, d_points, d_scaling, d_quaternions,
                                                        d_strengths);
    return check_launch("gsr_sugar_field_backward", false, st);
}

}  // namespace gsr
