// gsr_b200 — SuGaR.sample_points_in_gaussians ("SS/" = sugar/sugar_scene/sugar_model.py:757-799): the SDF-regularisation samples
// of the coarse trainers and the refinement, forward and backward, with no host round trip.
//
// SuGaR hands torch.multinomial cum_probs = cumsum(w) / sum(w) as the weights, so selected row k (in row order) is drawn with
// probability proportional to C_k = sum_{j <= k} w_j, not to w_k.  Over all P rows, with t_i = mask_i C_i:
//   k_sample_prefix<0>  w_i (0 on unselected rows) and the per-block sums of w
//   k_rs_scan<double>   (gsr_common.cuh) exclusive scan of those sums: the block offsets of C
//   k_sample_prefix<1>  C_i = offset + in-block inclusive sum; the per-block sums of t
//   k_rs_scan<double>   the block offsets of T
//   k_sample_prefix<2>  T_i = offset + in-block inclusive sum of t, stored as -T_i where t_i = 0
//   k_sample_points     per sample: the first row whose |T| exceeds u * total (total = |T_{P-1}|), one gathered record, the two
//                       Hamilton products of pytorch3d's quaternion_apply
// Searching the prefix of all P rows gives original row indices directly: no compaction, no count read back.  Everything is in
// float64 and in a fixed order, so a call is deterministic.  The float64 roundings of a parallel scan can leave a row with t = 0
// one ulp above its predecessor; the sign of T marks those rows, and a search that lands on one steps back to the last row of
// positive weight (a zero-weight row is never drawn; leading zero rows have T = 0 exactly and can never be landed on).
#include "gsr_radix.cuh"
#include <cfloat>

namespace gsr {
namespace {

constexpr int PREFIX_BLOCK = 1024;

struct PrefixArgs {
    int P, volume;
    const uint8_t* mask;     // [P] or NULL: every row
    const float* scaling;    // [P,3]
    const float* strengths;  // [P] or NULL: not proportional to opacity
    double* w_off;           // [nb] block sums of w, then their exclusive scan
    double* t_off;           // [nb] block sums of t, then their exclusive scan
    double* T;               // [P]
};

// inclusive scan of v over the block; *total = the block's sum (the last thread's inclusive value)
__device__ __forceinline__ double block_scan(double v, double* total) {
    __shared__ double wsum[PREFIX_BLOCK / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double t = __shfl_up_sync(GSR_FULL, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        const double s = wsum[lane];
        double si = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double t = __shfl_up_sync(GSR_FULL, si, o);
            if (lane >= o) si += t;
        }
        wsum[lane] = si;  // inclusive over the warps
    }
    __syncthreads();
    const double r = (warp ? wsum[warp - 1] : 0.0) + incl;
    *total = wsum[PREFIX_BLOCK / 32 - 1];
    __syncthreads();  // wsum is reused by the next call
    return r;
}

// SuGaR's areas: s0 * s1 * s2 (or 1), times the strength, abs; float32 as torch evaluates it
__device__ __forceinline__ double row_weight(const PrefixArgs& a, int i) {
    if (i >= a.P || (a.mask && !a.mask[i])) return 0.0;
    float w = 1.0f;
    if (a.volume) w = __fmul_rn(__fmul_rn(a.scaling[3 * (size_t)i], a.scaling[3 * (size_t)i + 1]), a.scaling[3 * (size_t)i + 2]);
    if (a.strengths) w = __fmul_rn(w, a.strengths[i]);
    return (double)fabsf(w);
}

template <int STAGE>
__global__ void __launch_bounds__(PREFIX_BLOCK) k_sample_prefix(PrefixArgs a) {
    const int i = blockIdx.x * PREFIX_BLOCK + threadIdx.x;
    const bool sel = i < a.P && (!a.mask || a.mask[i]);
    double tot;
    const double cw = block_scan(row_weight(a, i), &tot);
    if (STAGE == 0) {
        if (threadIdx.x == 0) a.w_off[blockIdx.x] = tot;
        return;
    }
    const double t = sel ? a.w_off[blockIdx.x] + cw : 0.0;
    const double ct = block_scan(t, &tot);
    if (STAGE == 1) {
        if (threadIdx.x == 0) a.t_off[blockIdx.x] = tot;
        return;
    }
    if (i < a.P) {
        const double T = a.t_off[blockIdx.x] + ct;
        a.T[i] = t > 0.0 ? T : -T;
    }
}

struct SampleArgs {
    int N, P;
    float f;
    const double *T, *u;
    const float *z, *points, *scaling, *quaternions;
    float* out_points;
    int64_t* out_idx;
    double* out_total;
};

__device__ __forceinline__ bool total_ok(double total) { return total > 0.0 && total <= DBL_MAX; }

__global__ void __launch_bounds__(256) k_sample_points(SampleArgs a) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= a.N) return;
    const double total = fabs(a.T[a.P - 1]);
    if (n == 0) *a.out_total = total;
    const bool ok = total_ok(total);
    int i = 0;
    if (ok) {
        double x = a.u[n] * total;
        // a guard only: for u < 1, fl(u * total) < total whenever the total is a normal float64, and a total built from float32
        // weights is at least 1.4e-45, far above float64's subnormal range
        if (!(x < total)) x = nextafter(total, 0.0);
        int lo = 0, hi = a.P - 1;                      // |T[P-1]| = total > x: the first crossing is at most P-1
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (fabs(a.T[mid]) > x) hi = mid;
            else lo = mid + 1;
        }
        i = lo;
        while (!(a.T[i] > 0.0)) --i;  // a zero-weight row raised by rounding: |T_i| > 0, so a positive row precedes it
    }
    float o0 = __int_as_float(0x7fffffff), o1 = o0, o2 = o0;
    if (ok) {
        const size_t r = (size_t)i;
        // v = (f * s) * z; then quaternion_raw_multiply(quaternion_raw_multiply(q, (0, v)), q * [1, -1, -1, -1])[1:]
        const float v0 = __fmul_rn(__fmul_rn(a.f, a.scaling[3 * r]), a.z[3 * (size_t)n]);
        const float v1 = __fmul_rn(__fmul_rn(a.f, a.scaling[3 * r + 1]), a.z[3 * (size_t)n + 1]);
        const float v2 = __fmul_rn(__fmul_rn(a.f, a.scaling[3 * r + 2]), a.z[3 * (size_t)n + 2]);
        const float qw = a.quaternions[4 * r], qx = a.quaternions[4 * r + 1], qy = a.quaternions[4 * r + 2], qz = a.quaternions[4 * r + 3];
        const float zero = 0.0f;
        const float aw = __fsub_rn(__fsub_rn(__fsub_rn(__fmul_rn(qw, zero), __fmul_rn(qx, v0)), __fmul_rn(qy, v1)), __fmul_rn(qz, v2));
        const float ax = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(qw, v0), __fmul_rn(qx, zero)), __fmul_rn(qy, v2)), __fmul_rn(qz, v1));
        const float ay = __fadd_rn(__fadd_rn(__fsub_rn(__fmul_rn(qw, v1), __fmul_rn(qx, v2)), __fmul_rn(qy, zero)), __fmul_rn(qz, v0));
        const float az = __fadd_rn(__fsub_rn(__fadd_rn(__fmul_rn(qw, v2), __fmul_rn(qx, v1)), __fmul_rn(qy, v0)), __fmul_rn(qz, zero));
        const float bw = qw, bx = -qx, by = -qy, bz = -qz;
        const float rx = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(aw, bx), __fmul_rn(ax, bw)), __fmul_rn(ay, bz)), __fmul_rn(az, by));
        const float ry = __fadd_rn(__fadd_rn(__fsub_rn(__fmul_rn(aw, by), __fmul_rn(ax, bz)), __fmul_rn(ay, bw)), __fmul_rn(az, bx));
        const float rz = __fadd_rn(__fsub_rn(__fadd_rn(__fmul_rn(aw, bz), __fmul_rn(ax, by)), __fmul_rn(ay, bx)), __fmul_rn(az, bw));
        o0 = __fadd_rn(a.points[3 * r], rx);
        o1 = __fadd_rn(a.points[3 * r + 1], ry);
        o2 = __fadd_rn(a.points[3 * r + 2], rz);
    }
    a.out_points[3 * (size_t)n] = o0;
    a.out_points[3 * (size_t)n + 1] = o1;
    a.out_points[3 * (size_t)n + 2] = o2;
    a.out_idx[n] = i;
}

struct SampleGradArgs {
    int N, P;
    float f;
    const int64_t* idx;
    const float *z, *scaling, *quaternions, *g;
    const double* total;
    float *d_points, *d_scaling, *d_quaternions;
};

// out = p + q (0, v) q* = p + (w^2 - u.u) v + 2 (u.v) u + 2 w (u x v), q = (w, u), v = (f s) z: any q, unit or not.  Sample n's
// partials to its Gaussian i: r = (dL/dpoints (3), dL/dscaling (3), dL/dquaternions (4)).  k_sample_backward adds them with atomics,
// k_sample_reduce in ascending n: one formula.
__device__ __forceinline__ void sample_partial(const SampleGradArgs& a, int n, int64_t i, float r[10]) {
    const float3 g = {a.g[3 * (size_t)n], a.g[3 * (size_t)n + 1], a.g[3 * (size_t)n + 2]};
    const float3 z = {a.z[3 * (size_t)n], a.z[3 * (size_t)n + 1], a.z[3 * (size_t)n + 2]};
    const float3 v = {a.f * a.scaling[3 * i] * z.x, a.f * a.scaling[3 * i + 1] * z.y, a.f * a.scaling[3 * i + 2] * z.z};
    const float w = a.quaternions[4 * i];
    const float3 u = {a.quaternions[4 * i + 1], a.quaternions[4 * i + 2], a.quaternions[4 * i + 3]};
    const float uu = u.x * u.x + u.y * u.y + u.z * u.z, ug = u.x * g.x + u.y * g.y + u.z * g.z;
    const float uv = u.x * v.x + u.y * v.y + u.z * v.z, gv = g.x * v.x + g.y * v.y + g.z * v.z;
    const float c = w * w - uu;
    // dL/dv = Q(q)^T g = (w^2 - u.u) g + 2 (u.g) u + 2 w (g x u)
    const float dvx = c * g.x + 2.0f * ug * u.x + 2.0f * w * (g.y * u.z - g.z * u.y);
    const float dvy = c * g.y + 2.0f * ug * u.y + 2.0f * w * (g.z * u.x - g.x * u.z);
    const float dvz = c * g.z + 2.0f * ug * u.z + 2.0f * w * (g.x * u.y - g.y * u.x);
    // dL/dw = 2 w (g.v) + 2 g.(u x v);  dL/du = -2 (g.v) u + 2 (u.g) v + 2 (u.v) g + 2 w (v x g)
    const float3 uxv = {u.y * v.z - u.z * v.y, u.z * v.x - u.x * v.z, u.x * v.y - u.y * v.x};
    const float3 vxg = {v.y * g.z - v.z * g.y, v.z * g.x - v.x * g.z, v.x * g.y - v.y * g.x};
    r[0] = g.x; r[1] = g.y; r[2] = g.z;
    r[3] = a.f * z.x * dvx; r[4] = a.f * z.y * dvy; r[5] = a.f * z.z * dvz;
    r[6] = 2.0f * (w * gv + (g.x * uxv.x + g.y * uxv.y + g.z * uxv.z));
    r[7] = 2.0f * (ug * v.x + uv * g.x + w * vxg.x - gv * u.x);
    r[8] = 2.0f * (ug * v.y + uv * g.y + w * vxg.y - gv * u.y);
    r[9] = 2.0f * (ug * v.z + uv * g.z + w * vxg.z - gv * u.z);
}

// DET: no atomics; key[n] = the sample's Gaussian, or P where it adds nothing (an index outside [0, P), a zero or non-finite
// total), id[n] = n.
template <bool DET>
__global__ void __launch_bounds__(256) k_sample_backward(SampleGradArgs a, uint32_t* __restrict__ key, uint32_t* __restrict__ id) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (DET) {
        if (n >= a.N) return;
        const int64_t i = a.idx[n];
        key[n] = total_ok(*a.total) && i >= 0 && i < a.P ? (uint32_t)i : (uint32_t)a.P;
        id[n] = (uint32_t)n;
        return;
    }
    if (n >= a.N || !total_ok(*a.total)) return;
    const int64_t i = a.idx[n];
    if (i < 0 || i >= a.P) return;
    float r[10];
    sample_partial(a, n, i, r);
    atomicAdd(a.d_points + 3 * i, r[0]);
    atomicAdd(a.d_points + 3 * i + 1, r[1]);
    atomicAdd(a.d_points + 3 * i + 2, r[2]);
    atomicAdd(a.d_scaling + 3 * i, r[3]);
    atomicAdd(a.d_scaling + 3 * i + 1, r[4]);
    atomicAdd(a.d_scaling + 3 * i + 2, r[5]);
    atomicAdd(a.d_quaternions + 4 * i, r[6]);
    atomicAdd(a.d_quaternions + 4 * i + 1, r[7]);
    atomicAdd(a.d_quaternions + 4 * i + 2, r[8]);
    atomicAdd(a.d_quaternions + 4 * i + 3, r[9]);
}

// DET: one thread per Gaussian g sums sample_partial over its samples in ascending n from +0.0 and writes g's three rows.
__global__ void __launch_bounds__(256) k_sample_reduce(SampleGradArgs a, const uint32_t* __restrict__ ids, const uint32_t* __restrict__ seg) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= a.P) return;
    float acc[10];
#pragma unroll
    for (int c = 0; c < 10; c++) acc[c] = 0.0f;
    const uint32_t e = seg[g + 1];
    for (uint32_t q = seg[g]; q < e; q++) {
        float r[10];
        sample_partial(a, (int)ids[q], g, r);
#pragma unroll
        for (int c = 0; c < 10; c++) acc[c] = __fadd_rn(acc[c], r[c]);
    }
    const size_t g3 = 3 * (size_t)g, g4 = 4 * (size_t)g;
    a.d_points[g3] = acc[0]; a.d_points[g3 + 1] = acc[1]; a.d_points[g3 + 2] = acc[2];
    a.d_scaling[g3] = acc[3]; a.d_scaling[g3 + 1] = acc[4]; a.d_scaling[g3 + 2] = acc[5];
    a.d_quaternions[g4] = acc[6]; a.d_quaternions[g4 + 1] = acc[7]; a.d_quaternions[g4 + 2] = acc[8]; a.d_quaternions[g4 + 3] = acc[9];
}

inline int nblocks_prefix(int P) { return (P + PREFIX_BLOCK - 1) / PREFIX_BLOCK; }

}  // namespace
}  // namespace gsr

using namespace gsr;

size_t gsr_sugar_sample_bytes(int32_t P) {
    if (P < 1) return 16;
    return align_up(8 * (size_t)P, 16) + 2 * align_up(8 * (size_t)nblocks_prefix(P), 16);
}

int gsr_sugar_sample(int32_t N, int32_t P, float f, int32_t volume, const uint8_t* mask, const float* strengths, const double* u,
                     const float* z, const float* points, const float* scaling, const float* quaternions, float* out_points,
                     int64_t* out_idx, double* out_total, void* ws, size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_sugar_sample");
    const cudaStream_t st = (cudaStream_t)stream;
    if (N < 0 || P < 1) {
        set_error("gsr_sugar_sample: N = %d and P = %d (need N >= 0, P >= 1)", N, P);
        return GSR_ERR_INVALID;
    }
    if (N == 0) return GSR_OK;
    if (!u || !z || !points || !scaling || !quaternions || !out_points || !out_idx || !out_total) {
        set_error("gsr_sugar_sample: missing input or output (only mask and strengths may be NULL)");
        return GSR_ERR_INVALID;
    }
    if (ws_bytes < gsr_sugar_sample_bytes(P) || !ws || ((uintptr_t)ws & 15)) {
        set_error("gsr_sugar_sample: workspace of %zu bytes (need %zu, 16-byte aligned)", ws_bytes, gsr_sugar_sample_bytes(P));
        return GSR_ERR_WORKSPACE;
    }
    const int nb = nblocks_prefix(P);
    char* w = (char*)ws;
    PrefixArgs a{P, volume ? 1 : 0, mask, scaling, strengths, nullptr, nullptr, (double*)w};
    w += align_up(8 * (size_t)P, 16);
    a.w_off = (double*)w;
    a.t_off = (double*)(w + align_up(8 * (size_t)nb, 16));
    k_sample_prefix<0><<<nb, PREFIX_BLOCK, 0, st>>>(a);
    k_rs_scan<double><<<1, 1024, 0, st>>>(a.w_off, nb);
    k_sample_prefix<1><<<nb, PREFIX_BLOCK, 0, st>>>(a);
    k_rs_scan<double><<<1, 1024, 0, st>>>(a.t_off, nb);
    k_sample_prefix<2><<<nb, PREFIX_BLOCK, 0, st>>>(a);
    const SampleArgs s{N, P, f, a.T, u, z, points, scaling, quaternions, out_points, out_idx, out_total};
    k_sample_points<<<(N + 255) / 256, 256, 0, st>>>(s);
    return check_launch("gsr_sugar_sample", false, st);
}

size_t gsr_sugar_sample_backward_det_bytes(int32_t N, int32_t P) { return GroupLayout((size_t)(N < 0 ? 0 : N), P < 0 ? 0 : P).total; }

// det: the deterministic backward (gsr_sugar_sample_backward_det) with `scratch` of scratch_bytes; otherwise scratch is unused.
static int sugar_sample_backward_impl(int N, int P, float f, const int64_t* idx, const float* z, const float* scaling,
                                      const float* quaternions, const double* total, const float* dL_dsamples, float* d_points,
                                      float* d_scaling, float* d_quaternions, bool det, void* scratch, size_t scratch_bytes,
                                      cudaStream_t st) {
    const char* who = det ? "gsr_sugar_sample_backward_det" : "gsr_sugar_sample_backward";
    if (N < 0 || P < 1) {
        set_error("%s: N = %d and P = %d (need N >= 0, P >= 1)", who, N, P);
        return GSR_ERR_INVALID;
    }
    if (!d_points || !d_scaling || !d_quaternions || (N > 0 && (!idx || !z || !scaling || !quaternions || !total || !dL_dsamples))) {
        set_error("%s: missing input or output", who);
        return GSR_ERR_INVALID;
    }
    const SampleGradArgs a{N, P, f, idx, z, scaling, quaternions, dL_dsamples, total, d_points, d_scaling, d_quaternions};
    if (det && N > 0) {
        if (!scratch) { set_error("%s: scratch is NULL", who); return GSR_ERR_INVALID; }
        if ((uintptr_t)scratch & 15) { set_error("%s: scratch is not 16-byte aligned", who); return GSR_ERR_INVALID; }
        const GroupLayout L((size_t)N, P);
        if (scratch_bytes < L.total) {
            set_error("%s: scratch too small (%zu < %zu)", who, scratch_bytes, L.total);
            return GSR_ERR_WORKSPACE;
        }
        char* w = (char*)scratch;
        k_sample_backward<true><<<(N + 255) / 256, 256, 0, st>>>(a, (uint32_t*)(w + L.keys0), (uint32_t*)(w + L.vals0));
        const uint32_t* ids = group_ids((size_t)N, P, w, L, st);
        k_sample_reduce<<<(P + 255) / 256, 256, 0, st>>>(a, ids, (const uint32_t*)(w + L.seg));
        return check_launch(who, false, st);
    }
    cudaMemsetAsync(d_points, 0, 12 * (size_t)P, st);
    cudaMemsetAsync(d_scaling, 0, 12 * (size_t)P, st);
    cudaMemsetAsync(d_quaternions, 0, 16 * (size_t)P, st);
    if (N > 0) k_sample_backward<false><<<(N + 255) / 256, 256, 0, st>>>(a, nullptr, nullptr);
    return check_launch(who, false, st);
}

int gsr_sugar_sample_backward(int32_t N, int32_t P, float sampling_scale_factor, const int64_t* idx, const float* z, const float* scaling,
                              const float* quaternions, const double* total, const float* dL_dsamples, float* dL_dpoints,
                              float* dL_dscaling, float* dL_dquaternions, void* stream) {
    NvtxRange nvtx_("gsr_sugar_sample_backward");
    return sugar_sample_backward_impl(N, P, sampling_scale_factor, idx, z, scaling, quaternions, total, dL_dsamples, dL_dpoints,
                                      dL_dscaling, dL_dquaternions, false, nullptr, 0, (cudaStream_t)stream);
}

int gsr_sugar_sample_backward_det(int32_t N, int32_t P, float sampling_scale_factor, const int64_t* idx, const float* z,
                                  const float* scaling, const float* quaternions, const double* total, const float* dL_dsamples,
                                  float* dL_dpoints, float* dL_dscaling, float* dL_dquaternions, void* scratch, size_t scratch_bytes,
                                  void* stream) {
    NvtxRange nvtx_("gsr_sugar_sample_backward_det");
    return sugar_sample_backward_impl(N, P, sampling_scale_factor, idx, z, scaling, quaternions, total, dL_dsamples, dL_dpoints,
                                      dL_dscaling, dL_dquaternions, true, scratch, scratch_bytes, (cudaStream_t)stream);
}
