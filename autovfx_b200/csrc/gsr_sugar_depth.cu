// gsr_b200 — coarse_sdf's depth-map SDF estimate ("CS/" = sugar/sugar_trainers/coarse_sdf.py, "SS/" = sugar/sugar_scene/
// sugar_model.py): the close-to-surface mask of the Gaussians (CS/:655-665) and the 'sdf' estimation loss (CS/:689-712), forward
// and backward, with no host round trip.
//
//   project, make_taps, sample_taps  pytorch3d's world-to-view transform_points, the camera's projection (FoVPerspectiveCameras with an SfM K:
//                      Transform3d(matrix=K^T), a plain division by w), SuGaR's rescaling by -min(H, W) / W and -min(H, W) / H
//                      (SS/:1193-1197) and torch's CUDA grid_sample(bilinear, border, align_corners=False) (SS/:1199-1203) of one
//                      point.  The mask and both loss kernels call it, so they all read the same taps with the same weights.
//   k_surface_mask     one thread per Gaussian: |map_z(centre) - z| < threshold * |s * quaternion_apply(quaternion_invert(q),
//                      normalize(c - p))|
//   k_depth_loss       one thread per sample: z > znear, term = clamp(|sdf - |map_z - z|| * (1 / std), max); fixed-tree block sums
//                      of the terms and the count (float64, uint64), k_depth_loss_final adds the block sums in block order and
//                      divides (0 / 0 = NaN for an empty mask, as torch's mean of an empty tensor)
//   k_depth_loss_backward  one thread per sample: dL/dsdf and dL/dsamples (through z, the projection and the bilinear weights)
//                      without atomics; dL/ddepth of the four taps with atomics or, under torch.use_deterministic_algorithms
//                      (gsr_sugar_depth_sdf_loss_backward_det), one key per (sample, tap) = texel, group_ids (gsr_radix.cuh) and
//                      k_depth_texel_reduce, one walker per texel that sums the partials of depth_sample_grad in ascending id.
//
// The lookup follows torch's source expressions (GridSampler.cuh / GridSampler.cu) including the multiply-adds nvcc contracts
// there: the unnormalize ((c + 1) * size - 1) / 2 and the tap accumulation out += v * w.  The 4x4 transforms are one fp32
// multiply-add chain in row order, as a GEMM of inner size 4 accumulates.  tests/test_gpu_sugar_depth.py pins what that gives.
#include "gsr_radix.cuh"

namespace gsr {
namespace {

struct DepthMap {
    int H, W;
    int64_t sh, sw;  // element strides of the [H, W] depth view
    const float* d;
    float sx, sy;    // SuGaR's factor / W and factor / H, rounded to float32 as torch multiplies by a Python double
};

// [p, 1] @ M, then the first three columns divided by the last (pytorch3d's transform_points with eps=None)
__device__ __forceinline__ float4 xform_row(float p0, float p1, float p2, const float* __restrict__ M) {
    float h[4];
#pragma unroll
    for (int k = 0; k < 4; k++) h[k] = __fadd_rn(__fmaf_rn(p2, M[8 + k], __fmaf_rn(p1, M[4 + k], __fmul_rn(p0, M[k]))), M[12 + k]);
    return make_float4(h[0], h[1], h[2], h[3]);
}

// torch's grid_sampler_unnormalize (align_corners=False) with nvcc's contraction of (c + 1) * size - 1
__device__ __forceinline__ float unnormalize(float c, int size) { return __fmul_rn(__fmaf_rn(__fadd_rn(c, 1.0f), (float)size, -1.0f), 0.5f); }

struct Taps {
    float ix, iy;     // the source coordinates after the border clip
    int x0, y0;       // floor(ix), floor(iy)
    float w[4];       // nw, ne, sw, se
    float gmx, gmy;   // d ix / d grid_x, d iy / d grid_y: size / 2 inside the clip range, 0 at or beyond a limit
};

__device__ __forceinline__ bool tap_in(const DepthMap& m, int x, int y) { return x >= 0 && x < m.W && y >= 0 && y < m.H; }
__device__ __forceinline__ int tap_x(const Taps& t, int k) { return t.x0 + (k & 1); }
__device__ __forceinline__ int tap_y(const Taps& t, int k) { return t.y0 + (k >> 1); }
__device__ __forceinline__ float tap_value(const DepthMap& m, int x, int y) { return m.d[(int64_t)y * m.sh + (int64_t)x * m.sw]; }

// BWD: grid_sampler_compute_source_index_set_grad (a coordinate at or beyond a limit has gradient 0; a NaN coordinate becomes
// -100, outside the map), else grid_sampler_compute_source_index (fmaxf sends NaN to 0; the border clip leaves every coordinate
// finite and inside the int range, so its safe_downgrade_to_int_range is the identity)
template <bool BWD>
__device__ __forceinline__ float clip_coord(float in, int size, float& g) {
    const float hi = (float)(size - 1);
    g = 0.5f * (float)size;
    if (!BWD) return fminf(hi, fmaxf(in, 0.0f));
    if (in <= 0.0f) { g = 0.0f; return 0.0f; }
    if (in >= hi) { g = 0.0f; return hi; }
    if (in != in) return -100.0f;
    return in;
}

template <bool BWD>
__device__ __forceinline__ Taps make_taps(const DepthMap& m, float gx, float gy) {
    Taps t;
    t.ix = clip_coord<BWD>(unnormalize(gx, m.W), m.W, t.gmx);
    t.iy = clip_coord<BWD>(unnormalize(gy, m.H), m.H, t.gmy);
    t.x0 = (int)floorf(t.ix);
    t.y0 = (int)floorf(t.iy);
    const float xe = __fsub_rn((float)(t.x0 + 1), t.ix), xw = __fsub_rn(t.ix, (float)t.x0);
    const float ys = __fsub_rn((float)(t.y0 + 1), t.iy), yn = __fsub_rn(t.iy, (float)t.y0);
    t.w[0] = __fmul_rn(xe, ys);
    t.w[1] = __fmul_rn(xw, ys);
    t.w[2] = __fmul_rn(xe, yn);
    t.w[3] = __fmul_rn(xw, yn);
    return t;
}

// bilinear value in torch's tap order, out_acc += v * w contracted
__device__ __forceinline__ float sample_taps(const DepthMap& m, const Taps& t) {
    float acc = 0.0f;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int x = tap_x(t, k), y = tap_y(t, k);
        if (tap_in(m, x, y)) acc = __fmaf_rn(tap_value(m, x, y), t.w[k], acc);
    }
    return acc;
}

struct Proj {
    float4 v;        // camera-space point (x, y, z) and the world-to-view w
    float4 h;        // [v, 1] @ K^T before the division
    float n0, n1;    // h.x / h.w, h.y / h.w
    float gx, gy;    // grid coordinates
};

// cam [36]: world-to-view matrix (16, row-major, row vectors: [p, 1] @ M), projection matrix (16, likewise K^T), znear,
// camera centre (3)
__device__ __forceinline__ Proj project(const DepthMap& m, const float* __restrict__ cam, float p0, float p1, float p2) {
    Proj r;
    const float4 hv = xform_row(p0, p1, p2, cam);
    r.v = make_float4(__fdiv_rn(hv.x, hv.w), __fdiv_rn(hv.y, hv.w), __fdiv_rn(hv.z, hv.w), hv.w);
    r.h = xform_row(r.v.x, r.v.y, r.v.z, cam + 16);
    r.n0 = __fdiv_rn(r.h.x, r.h.w);
    r.n1 = __fdiv_rn(r.h.y, r.h.w);
    r.gx = __fmul_rn(m.sx, r.n0);
    r.gy = __fmul_rn(m.sy, r.n1);
    return r;
}

// quaternion_apply(a, d) of pytorch3d, one rounding per torch op: raw_multiply(raw_multiply(a, (0, d)), quaternion_invert(a))
__device__ __forceinline__ float3 quat_apply_rn(float qw, float qx, float qy, float qz, float v0, float v1, float v2) {
    const float zero = 0.0f;
    const float aw = __fsub_rn(__fsub_rn(__fsub_rn(__fmul_rn(qw, zero), __fmul_rn(qx, v0)), __fmul_rn(qy, v1)), __fmul_rn(qz, v2));
    const float ax = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(qw, v0), __fmul_rn(qx, zero)), __fmul_rn(qy, v2)), __fmul_rn(qz, v1));
    const float ay = __fadd_rn(__fadd_rn(__fsub_rn(__fmul_rn(qw, v1), __fmul_rn(qx, v2)), __fmul_rn(qy, zero)), __fmul_rn(qz, v0));
    const float az = __fadd_rn(__fsub_rn(__fadd_rn(__fmul_rn(qw, v2), __fmul_rn(qx, v1)), __fmul_rn(qy, v0)), __fmul_rn(qz, zero));
    const float bw = qw, bx = -qx, by = -qy, bz = -qz;
    return make_float3(__fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(aw, bx), __fmul_rn(ax, bw)), __fmul_rn(ay, bz)), __fmul_rn(az, by)),
                       __fadd_rn(__fadd_rn(__fsub_rn(__fmul_rn(aw, by), __fmul_rn(ax, bz)), __fmul_rn(ay, bw)), __fmul_rn(az, bx)),
                       __fadd_rn(__fsub_rn(__fadd_rn(__fmul_rn(aw, bz), __fmul_rn(ax, by)), __fmul_rn(ay, bx)), __fmul_rn(az, bw)));
}

struct MaskArgs {
    int P;
    DepthMap m;
    const float *cam, *points, *scaling, *quaternions;
    float threshold;
    uint8_t* out;
    float* map_z;  // may be NULL
};

__global__ void __launch_bounds__(256) k_surface_mask(MaskArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.P) return;
    const size_t i3 = 3 * (size_t)i, i4 = 4 * (size_t)i;
    const float p0 = a.points[i3], p1 = a.points[i3 + 1], p2 = a.points[i3 + 2];
    const Proj pr = project(a.m, a.cam, p0, p1, p2);
    const float mz = sample_taps(a.m, make_taps<false>(a.m, pr.gx, pr.gy));
    float d0, d1, d2;
    normalize3_rn(__fsub_rn(a.cam[33], p0), __fsub_rn(a.cam[34], p1), __fsub_rn(a.cam[35], p2), d0, d1, d2);
    // quaternion_invert(q) = q * [1, -1, -1, -1]
    const float3 r = quat_apply_rn(a.quaternions[i4], -a.quaternions[i4 + 1], -a.quaternions[i4 + 2], -a.quaternions[i4 + 3], d0, d1, d2);
    const float sd = norm3_rn(__fmul_rn(a.scaling[i3], r.x), __fmul_rn(a.scaling[i3 + 1], r.y), __fmul_rn(a.scaling[i3 + 2], r.z));
    a.out[i] = fabsf(__fsub_rn(mz, pr.v.z)) < __fmul_rn(a.threshold, sd) ? 1 : 0;
    if (a.map_z) a.map_z[i] = mz;
}

struct LossArgs {
    int N;
    DepthMap m;
    const float *cam, *x, *sdf;
    float inv_std, clamp_max;
};

constexpr int LOSS_BLOCK = 256, LOSS_ITEMS = 8, LOSS_CHUNK = LOSS_BLOCK * LOSS_ITEMS;

// term of sample n (0 where z <= znear); *masked = z > znear
__device__ __forceinline__ float sample_term(const LossArgs& a, int n, bool* masked) {
    const size_t n3 = 3 * (size_t)n;
    const Proj pr = project(a.m, a.cam, a.x[n3], a.x[n3 + 1], a.x[n3 + 2]);
    *masked = pr.v.z > a.cam[32];
    if (!*masked) return 0.0f;
    const float est = __fsub_rn(sample_taps(a.m, make_taps<false>(a.m, pr.gx, pr.gy)), pr.v.z);
    const float t = __fmul_rn(fabsf(__fsub_rn(a.sdf[n], fabsf(est))), a.inv_std);
    return t > a.clamp_max ? a.clamp_max : t;  // clamp(max=): NaN stays NaN
}

__global__ void __launch_bounds__(LOSS_BLOCK) k_depth_loss(LossArgs a, double* __restrict__ part_sum, unsigned long long* __restrict__ part_cnt) {
    double s = 0.0;
    unsigned long long c = 0;
    const int base = blockIdx.x * LOSS_CHUNK + threadIdx.x;
#pragma unroll
    for (int k = 0; k < LOSS_ITEMS; k++) {
        const int n = base + k * LOSS_BLOCK;
        if (n < a.N) {
            bool msk;
            const float t = sample_term(a, n, &msk);
            if (msk) { s += (double)t; c++; }
        }
    }
    __shared__ double ws[LOSS_BLOCK / 32];
    __shared__ unsigned long long wc[LOSS_BLOCK / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(GSR_FULL, s, o);
        c += __shfl_xor_sync(GSR_FULL, c, o);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { ws[warp] = s; wc[warp] = c; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double bs = 0.0;
        unsigned long long bc = 0;
        for (int w = 0; w < LOSS_BLOCK / 32; w++) { bs += ws[w]; bc += wc[w]; }
        part_sum[blockIdx.x] = bs;
        part_cnt[blockIdx.x] = bc;
    }
}

// one thread adds the block sums in block order
__global__ void k_depth_loss_final(int nb, const double* __restrict__ part_sum, const unsigned long long* __restrict__ part_cnt,
                                   float* __restrict__ out, int64_t* __restrict__ count) {
    double s = 0.0;
    unsigned long long c = 0;
    for (int b = 0; b < nb; b++) { s += part_sum[b]; c += part_cnt[b]; }
    *out = (float)(s / (double)c);
    *count = (int64_t)c;
}

struct LossGradArgs {
    LossArgs f;
    const int64_t* count;
    const float* g;  // dL/dloss [1]
    float *d_x, *d_sdf, *d_depth;
};

struct SampleGrad {
    bool masked;
    float g_map;   // dL/dmap_z
    Taps t;        // the backward's taps
};

// dL/dmap_z of sample n and its taps; with dx / dsdf not NULL also dL/dx and dL/dsdf.  The atomic backward and the texel walker
// both take a tap's partial, g_map * w[k], from here.
__device__ __forceinline__ SampleGrad depth_sample_grad(const LossGradArgs& a, int n, float* dx, float* dsdf) {
    const LossArgs& f = a.f;
    const size_t n3 = 3 * (size_t)n;
    const float* M = f.cam;
    const float* K = f.cam + 16;
    SampleGrad r;
    const Proj pr = project(f.m, f.cam, f.x[n3], f.x[n3 + 1], f.x[n3 + 2]);
    r.masked = pr.v.z > f.cam[32];
    r.g_map = 0.0f;
    r.t = make_taps<true>(f.m, pr.gx, pr.gy);
    if (!r.masked) {
        if (dx) dx[0] = dx[1] = dx[2] = 0.0f;
        if (dsdf) *dsdf = 0.0f;
        return r;
    }
    const float mz = sample_taps(f.m, make_taps<false>(f.m, pr.gx, pr.gy));
    const float est = __fsub_rn(mz, pr.v.z);
    const float res = __fsub_rn(f.sdf[n], fabsf(est));
    const float t = __fmul_rn(fabsf(res), f.inv_std);
    const float gterm = (t <= f.clamp_max) ? __fdiv_rn(*a.g, (float)*a.count) : 0.0f;  // clamp's backward passes t == max
    const float sgn_r = (float)((res > 0.0f) - (res < 0.0f)), sgn_e = (float)((est > 0.0f) - (est < 0.0f));
    const float g_res = gterm * f.inv_std * sgn_r;
    const float g_est = -g_res * sgn_e;
    r.g_map = g_est;
    if (dsdf) *dsdf = g_res;
    if (!dx) return r;
    // dL/d(grid) through the bilinear weights, taps inside the map only (torch's grid_sampler_2d_backward)
    const Taps& tp = r.t;
    float gix = 0.0f, giy = 0.0f;
    const float xe = (float)(tp.x0 + 1) - tp.ix, xw = tp.ix - (float)tp.x0, ys = (float)(tp.y0 + 1) - tp.iy, yn = tp.iy - (float)tp.y0;
    const float dwx[4] = {-ys, ys, -yn, yn}, dwy[4] = {-xe, -xw, xe, xw};
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int x = tap_x(tp, k), y = tap_y(tp, k);
        if (tap_in(f.m, x, y)) {
            const float v = tap_value(f.m, x, y);
            gix += v * dwx[k];
            giy += v * dwy[k];
        }
    }
    const float gn0 = g_est * gix * tp.gmx * f.m.sx, gn1 = g_est * giy * tp.gmy * f.m.sy;
    // n = h.xy / h.w, h = [v, 1] @ K^T
    const float gh[4] = {gn0 / pr.h.w, gn1 / pr.h.w, 0.0f, -(gn0 * pr.n0 + gn1 * pr.n1) / pr.h.w};
    float gv[3];
#pragma unroll
    for (int i = 0; i < 3; i++) gv[i] = K[4 * i] * gh[0] + K[4 * i + 1] * gh[1] + K[4 * i + 3] * gh[3];
    gv[2] -= g_est;  // est = map_z - z
    // v = hv.xyz / hv.w, hv = [x, 1] @ M
    const float iw = 1.0f / pr.v.w;
    const float ghv[4] = {gv[0] * iw, gv[1] * iw, gv[2] * iw, -(gv[0] * pr.v.x + gv[1] * pr.v.y + gv[2] * pr.v.z) * iw};
#pragma unroll
    for (int j = 0; j < 3; j++) dx[j] = M[4 * j] * ghv[0] + M[4 * j + 1] * ghv[1] + M[4 * j + 2] * ghv[2] + M[4 * j + 3] * ghv[3];
    return r;
}

// DET: per-sample gradients, and key[4n + k] = the texel of tap k (H * W where the tap adds nothing), id[4n + k] = 4n + k
template <bool DET>
__global__ void __launch_bounds__(256) k_depth_loss_backward(LossGradArgs a, uint32_t* __restrict__ key, uint32_t* __restrict__ id) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= a.f.N) return;
    float dx[3], dsdf;
    const SampleGrad s = depth_sample_grad(a, n, dx, &dsdf);
    const size_t n3 = 3 * (size_t)n;
    a.d_x[n3] = dx[0]; a.d_x[n3 + 1] = dx[1]; a.d_x[n3 + 2] = dx[2];
    a.d_sdf[n] = dsdf;
    const DepthMap& m = a.f.m;
    const uint32_t none = (uint32_t)m.H * (uint32_t)m.W;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int x = tap_x(s.t, k), y = tap_y(s.t, k);
        const bool adds = s.masked && tap_in(m, x, y);
        if (DET) {
            key[4 * (size_t)n + k] = adds ? (uint32_t)y * (uint32_t)m.W + (uint32_t)x : none;
            id[4 * (size_t)n + k] = 4 * (uint32_t)n + k;
        } else if (adds) {
            atomicAdd(a.d_depth + (size_t)y * m.W + x, s.g_map * s.t.w[k]);
        }
    }
}

// DET: one thread per texel sums its partials in ascending id from +0.0
__global__ void __launch_bounds__(256) k_depth_texel_reduce(LossGradArgs a, const uint32_t* __restrict__ ids, const uint32_t* __restrict__ seg) {
    const uint32_t texel = blockIdx.x * blockDim.x + threadIdx.x;
    if (texel >= (uint32_t)a.f.m.H * (uint32_t)a.f.m.W) return;
    float acc = 0.0f;
    const uint32_t e = seg[texel + 1];
    for (uint32_t q = seg[texel]; q < e; q++) {
        const uint32_t i = ids[q];
        const SampleGrad s = depth_sample_grad(a, (int)(i >> 2), nullptr, nullptr);
        const uint32_t k = i & 3;  // a select, not a dynamic index into s.t.w (which would put it on the stack)
        const float w = k == 0 ? s.t.w[0] : k == 1 ? s.t.w[1] : k == 2 ? s.t.w[2] : s.t.w[3];
        acc = __fadd_rn(acc, s.g_map * w);
    }
    a.d_depth[texel] = acc;
}

inline int loss_blocks(int N) { return (N + LOSS_CHUNK - 1) / LOSS_CHUNK; }

// H * W below 2^31: texel indices, the sentinel H * W and the grouping's target count are int; per_item partial ids per item
// (4 for the loss's taps, 1 for the mask's Gaussians) below 2^32: the ids are uint32
bool depth_args_ok(const char* who, int N, int per_item, int H, int W, const float* depth, const float* camera) {
    if (N < 0 || H < 1 || W < 1 || (int64_t)H * W > (int64_t)INT32_MAX || (int64_t)N * per_item >= (int64_t)UINT32_MAX) {
        set_error("%s: N = %d, H = %d, W = %d (need N >= 0, H, W >= 1, H * W < 2^31 and %d N < 2^32)", who, N, H, W, per_item);
        return false;
    }
    if (N > 0 && (!depth || !camera)) {
        set_error("%s: depth and camera are required", who);
        return false;
    }
    return true;
}

}  // namespace
}  // namespace gsr

using namespace gsr;

int gsr_sugar_surface_mask(int32_t P, int32_t H, int32_t W, int64_t depth_stride_h, int64_t depth_stride_w, const float* depth,
                           float sx, float sy, const float* camera, const float* points, const float* scaling, const float* quaternions,
                           float threshold, uint8_t* out_mask, float* out_map_z, void* stream) {
    NvtxRange nvtx_("gsr_sugar_surface_mask");
    const char* who = "gsr_sugar_surface_mask";
    if (!depth_args_ok(who, P, 1, H, W, depth, camera)) return GSR_ERR_INVALID;
    if (P == 0) return GSR_OK;
    if (!points || !scaling || !quaternions || !out_mask) {
        set_error("%s: missing input or output (only out_map_z may be NULL)", who);
        return GSR_ERR_INVALID;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    const MaskArgs a{P, DepthMap{H, W, depth_stride_h, depth_stride_w, depth, sx, sy}, camera, points, scaling, quaternions, threshold,
                     out_mask, out_map_z};
    k_surface_mask<<<(P + 255) / 256, 256, 0, st>>>(a);
    return check_launch(who, false, st);
}

size_t gsr_sugar_depth_sdf_loss_bytes(int32_t N) { return 16 * (size_t)(N > 0 ? loss_blocks(N) : 1); }

int gsr_sugar_depth_sdf_loss(int32_t N, int32_t H, int32_t W, int64_t depth_stride_h, int64_t depth_stride_w, const float* depth,
                             float sx, float sy, const float* camera, const float* samples, const float* sdf_values, float inv_std,
                             float clamp_max, float* out_loss, int64_t* out_count, void* workspace, size_t workspace_bytes,
                             void* stream) {
    NvtxRange nvtx_("gsr_sugar_depth_sdf_loss");
    const char* who = "gsr_sugar_depth_sdf_loss";
    if (!depth_args_ok(who, N, 4, H, W, depth, camera)) return GSR_ERR_INVALID;
    if (!out_loss || !out_count || (N > 0 && (!samples || !sdf_values))) {
        set_error("%s: missing input or output", who);
        return GSR_ERR_INVALID;
    }
    if (workspace_bytes < gsr_sugar_depth_sdf_loss_bytes(N) || !workspace || ((uintptr_t)workspace & 15)) {
        set_error("%s: workspace of %zu bytes (need %zu, 16-byte aligned)", who, workspace_bytes, gsr_sugar_depth_sdf_loss_bytes(N));
        return GSR_ERR_WORKSPACE;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    const int nb = N > 0 ? loss_blocks(N) : 0;
    double* part_sum = (double*)workspace;
    unsigned long long* part_cnt = (unsigned long long*)((char*)workspace + 8 * (size_t)(nb > 0 ? nb : 1));
    const LossArgs a{N, DepthMap{H, W, depth_stride_h, depth_stride_w, depth, sx, sy}, camera, samples, sdf_values, inv_std, clamp_max};
    if (nb > 0) k_depth_loss<<<nb, LOSS_BLOCK, 0, st>>>(a, part_sum, part_cnt);
    k_depth_loss_final<<<1, 1, 0, st>>>(nb, part_sum, part_cnt, out_loss, out_count);
    return check_launch(who, false, st);
}

size_t gsr_sugar_depth_sdf_loss_backward_det_bytes(int32_t N, int32_t H, int32_t W) {
    const int64_t hw = (int64_t)(H > 0 ? H : 0) * (W > 0 ? W : 0);
    return hw > INT32_MAX ? 0 : GroupLayout(4 * (size_t)(N > 0 ? N : 0), (int)hw).total;  // such a map is rejected by the call
}

static int depth_loss_backward_impl(int N, int H, int W, int64_t sh, int64_t sw, const float* depth, float sx, float sy,
                                    const float* camera, const float* samples, const float* sdf_values, float inv_std, float clamp_max,
                                    const int64_t* count, const float* dL_dloss, float* dL_dsamples, float* dL_dsdf, float* dL_ddepth,
                                    bool det, void* scratch, size_t scratch_bytes, cudaStream_t st) {
    const char* who = det ? "gsr_sugar_depth_sdf_loss_backward_det" : "gsr_sugar_depth_sdf_loss_backward";
    if (!depth_args_ok(who, N, 4, H, W, depth, camera)) return GSR_ERR_INVALID;
    if (!dL_ddepth || (N > 0 && (!samples || !sdf_values || !count || !dL_dloss || !dL_dsamples || !dL_dsdf))) {
        set_error("%s: missing input or output", who);
        return GSR_ERR_INVALID;
    }
    const int HW = H * W;
    const LossGradArgs a{LossArgs{N, DepthMap{H, W, sh, sw, depth, sx, sy}, camera, samples, sdf_values, inv_std, clamp_max}, count,
                         dL_dloss, dL_dsamples, dL_dsdf, dL_ddepth};
    if (det && N > 0) {
        if (!scratch || ((uintptr_t)scratch & 15)) {
            set_error("%s: scratch is NULL or not 16-byte aligned", who);
            return GSR_ERR_INVALID;
        }
        const GroupLayout L(4 * (size_t)N, HW);
        if (scratch_bytes < L.total) {
            set_error("%s: scratch too small (%zu < %zu)", who, scratch_bytes, L.total);
            return GSR_ERR_WORKSPACE;
        }
        char* w = (char*)scratch;
        k_depth_loss_backward<true><<<(N + 255) / 256, 256, 0, st>>>(a, (uint32_t*)(w + L.keys0), (uint32_t*)(w + L.vals0));
        const uint32_t* ids = group_ids(4 * (size_t)N, HW, w, L, st);
        k_depth_texel_reduce<<<(HW + 255) / 256, 256, 0, st>>>(a, ids, (const uint32_t*)(w + L.seg));
        return check_launch(who, false, st);
    }
    cudaMemsetAsync(dL_ddepth, 0, 4 * (size_t)HW, st);
    if (N > 0) k_depth_loss_backward<false><<<(N + 255) / 256, 256, 0, st>>>(a, nullptr, nullptr);
    return check_launch(who, false, st);
}

int gsr_sugar_depth_sdf_loss_backward(int32_t N, int32_t H, int32_t W, int64_t depth_stride_h, int64_t depth_stride_w, const float* depth,
                                      float sx, float sy, const float* camera, const float* samples, const float* sdf_values, float inv_std,
                                      float clamp_max, const int64_t* count, const float* dL_dloss, float* dL_dsamples, float* dL_dsdf,
                                      float* dL_ddepth, void* stream) {
    NvtxRange nvtx_("gsr_sugar_depth_sdf_loss_backward");
    return depth_loss_backward_impl(N, H, W, depth_stride_h, depth_stride_w, depth, sx, sy, camera, samples, sdf_values, inv_std,
                                    clamp_max, count, dL_dloss, dL_dsamples, dL_dsdf, dL_ddepth, false, nullptr, 0, (cudaStream_t)stream);
}

int gsr_sugar_depth_sdf_loss_backward_det(int32_t N, int32_t H, int32_t W, int64_t depth_stride_h, int64_t depth_stride_w,
                                          const float* depth, float sx, float sy, const float* camera, const float* samples,
                                          const float* sdf_values, float inv_std, float clamp_max, const int64_t* count,
                                          const float* dL_dloss, float* dL_dsamples, float* dL_dsdf, float* dL_ddepth, void* scratch,
                                          size_t scratch_bytes, void* stream) {
    NvtxRange nvtx_("gsr_sugar_depth_sdf_loss_backward_det");
    return depth_loss_backward_impl(N, H, W, depth_stride_h, depth_stride_w, depth, sx, sy, camera, samples, sdf_values, inv_std,
                                    clamp_max, count, dL_dloss, dL_dsamples, dL_dsdf, dL_ddepth, true, scratch, scratch_bytes,
                                    (cudaStream_t)stream);
}
