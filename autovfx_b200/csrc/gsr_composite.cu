// Frame compositing of blender/blend_all.py:blend_frames (:185-342), the last numeric stage of render_scene
// (scene_representation.py:224-232):
//   k_pct_hist / k_pct_pick / k_pct_above / k_pct_final
//                    np.percentile(smoke_depth, 0.001) (:208) by a radix select on order-preserving keys, result on the device
//   k_composite<GS, SMOKE, FIRE>
//                    the per-pixel body :236-342 in one pass: 8-bit layers and float depths in, the uint8 RGBA frame out
// Every float operation is the float32 operation numpy performs, in numpy's order, written with _rn intrinsics so that nothing
// contracts into an FMA (NumPy >= 2: python scalars are weak, so /255., 1. - x, + 1e-6 and < 0.01 are float32 operations).
#include "gsr_common.cuh"

namespace gsr {

// ------------------------------------------------------------------------------------------------------ np.percentile(x, 0.001)
// numpy's 'linear' method on a float32 array under NumPy >= 2 (function_base._quantile): q = float32(0.001) / float32(100),
// v = float32(n - 1) * q, i = floor(v), t = v - i, the order statistics a = x_(i) and b = x_(i+1) (both x_(n-1) when
// v >= n - 1), then _lerp: a + (b - a) * t, or b - (b - a) * (1 - t) where t >= 0.5, all in float32.  Any NaN gives NaN.
// Keys: the float's bits with the sign bit flipped for positives and every bit flipped for negatives, so unsigned order is
// float order (-0.0 sorts below +0.0; numpy treats them as equal, so a result may differ from numpy's in the sign of a zero).
struct PctState {
    uint32_t hist[256];
    uint32_t prefix;    // key bits selected so far (high bits first)
    uint32_t rank;      // rank of x_(i) among the keys that share `prefix`
    uint32_t eq_after;  // keys equal to x_(i) at ranks above it (after the last pass)
    uint32_t nan;       // 1 when any element is NaN
    uint32_t above;     // smallest key greater than x_(i) (k_pct_above)
};
static_assert(sizeof(PctState) <= GSR_PERCENTILE_BYTES, "GSR_PERCENTILE_BYTES too small");

__device__ __forceinline__ uint32_t f2key(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

constexpr int PCT_THREADS = 256;
constexpr int PCT_ITEMS = 16;  // elements per thread per block tile

// Histogram of byte `pass` (0 = most significant) of the keys whose higher bytes equal the selected prefix.
__global__ void __launch_bounds__(PCT_THREADS) k_pct_hist(int64_t n, const float* __restrict__ x, int pass, PctState* __restrict__ st) {
    __shared__ uint32_t h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int shift = 24 - 8 * pass;
    const uint32_t mask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
    const uint32_t prefix = st->prefix;
    bool nan = false;
    const int64_t stride = (int64_t)gridDim.x * PCT_THREADS;
    for (int64_t i = (int64_t)blockIdx.x * PCT_THREADS + threadIdx.x; i < n; i += stride) {
        const float f = x[i];
        nan |= f != f;
        const uint32_t k = f2key(f);
        // warp-aggregated: a constant background (Blender's empty-pixel depth) would otherwise serialise on one bin
        const uint32_t b = (k & mask) == prefix ? ((k >> shift) & 255u) : 256u;
        const unsigned peers = __match_any_sync(__activemask(), b);
        if (b < 256u && (threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1)) atomicAdd(&h[b], (uint32_t)__popc(peers));
    }
    if (pass == 0 && __syncthreads_or(nan) && threadIdx.x == 0) st->nan = 1u;
    __syncthreads();
    if (h[threadIdx.x]) atomicAdd(&st->hist[threadIdx.x], h[threadIdx.x]);
}

// One CTA of 256: the bin holding `rank`, appended to the prefix; clears the histogram for the next pass.
__global__ void __launch_bounds__(256) k_pct_pick(int pass, PctState* __restrict__ st) {
    __shared__ uint32_t cum[256];
    const uint32_t c = st->hist[threadIdx.x];
    cum[threadIdx.x] = c;
    __syncthreads();
    for (int off = 1; off < 256; off <<= 1) {  // inclusive scan
        const uint32_t v = threadIdx.x >= off ? cum[threadIdx.x - off] : 0u;
        __syncthreads();
        cum[threadIdx.x] += v;
        __syncthreads();
    }
    const uint32_t rank = st->rank, lo = cum[threadIdx.x] - c;
    __syncthreads();
    if (c && lo <= rank && rank < lo + c) {
        st->prefix |= (uint32_t)threadIdx.x << (24 - 8 * pass);
        st->rank = rank - lo;
        st->eq_after = c - 1 - (rank - lo);
    }
    st->hist[threadIdx.x] = 0u;
}

// Smallest key above x_(i), needed only when no key equal to x_(i) sits at a higher rank.
__global__ void __launch_bounds__(PCT_THREADS) k_pct_above(int64_t n, const float* __restrict__ x, PctState* __restrict__ st) {
    if (st->eq_after != 0u) return;
    const uint32_t k0 = st->prefix;
    uint32_t best = 0xffffffffu;
    const int64_t stride = (int64_t)gridDim.x * PCT_THREADS;
    for (int64_t i = (int64_t)blockIdx.x * PCT_THREADS + threadIdx.x; i < n; i += stride) {
        const uint32_t k = f2key(x[i]);
        if (k > k0) best = min(best, k);
    }
    best = __reduce_min_sync(GSR_FULL, best);
    if ((threadIdx.x & 31) == 0 && best != 0xffffffffu) atomicMin(&st->above, best);
}

__global__ void k_pct_init(uint32_t rank, PctState* __restrict__ st) {
    st->hist[threadIdx.x] = 0u;
    if (threadIdx.x == 0) {
        st->prefix = 0u;
        st->rank = rank;
        st->eq_after = 0u;
        st->nan = 0u;
        st->above = 0xffffffffu;
    }
}

__global__ void k_pct_final(float t, int same, const PctState* __restrict__ st, float* __restrict__ out) {
    const float a = key2f(st->prefix);
    const float b = (same || st->eq_after != 0u) ? a : key2f(st->above);
    const float d = __fsub_rn(b, a);
    float r = __fadd_rn(a, __fmul_rn(d, t));
    if (t >= 0.5f) r = __fsub_rn(b, __fmul_rn(d, __fsub_rn(1.0f, t)));
    out[0] = st->nan ? __int_as_float(0x7fc00000) : r;
}

// ------------------------------------------------------------------------------------------------------------- the composite
__device__ __forceinline__ float byte_f(uint32_t px, int c) { return (float)((px >> (8 * c)) & 255u); }
__device__ __forceinline__ float alpha_f(uint32_t px) { return __fdiv_rn((float)(px >> 24), 255.0f); }  // rgb[..., 3] / 255.
// np.clip(v, 0, 255).astype(np.uint8): truncation; NaN would stay NaN through the clip and numpy's x86 cast gives 0, as this does
__device__ __forceinline__ uint32_t to_u8(float v) { return v != v ? 0u : (uint32_t)(v < 0.0f ? 0.0f : (v > 255.0f ? 255.0f : v)); }

template <bool GS, bool SMOKE, bool FIRE>
__global__ void __launch_bounds__(256) k_composite(int64_t HW, const uint32_t* __restrict__ frame, const uint32_t* __restrict__ obj,
                                                   const float* __restrict__ obj_d, const uint32_t* __restrict__ shadow,
                                                   const float* __restrict__ shadow_d, const uint32_t* __restrict__ all,
                                                   const uint32_t* __restrict__ gs, const float* __restrict__ gs_d,
                                                   const uint32_t* __restrict__ smoke, const float* __restrict__ smoke_d,
                                                   const float* __restrict__ smoke_pct, const uint32_t* __restrict__ fire,
                                                   uint32_t* __restrict__ out) {
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    const uint32_t o = obj[p], a = all[p];
    const float od = obj_d[p], sd = shadow_d[p];
    // step 1 (:255-273)
    float non_gs_alpha = 1.0f;
    bool gs_front = false;
    if (GS) {
        const float gd = gs_d[p];
        non_gs_alpha = sd <= gd ? 1.0f : __fsub_rn(1.0f, alpha_f(gs[p]));  // depth_check(s_d, o_gs_d) -> 1.0 (:259)
        gs_front = gd <= od;                                                  // :276
    }
    float obj_alpha = alpha_f(o);
    bool depth_mask = od <= sd;  // 'naive': d1 <= d2, NaN compares false
    float smoke_alpha = 0.0f;
    bool depth_mask_smoke = false;
    if (SMOKE) {
        const uint32_t sm = smoke[p];
        const float sfd = (sm >> 24) ? smoke_pct[0] : smoke_d[p];  // :207-208, alpha byte > 0 -> the percentile
        smoke_alpha = alpha_f(sm);
        depth_mask_smoke = sfd <= sd;
        obj_alpha = fmaxf(obj_alpha, smoke_alpha);  // both in [0, 1], never NaN
        depth_mask = depth_mask || depth_mask_smoke;
    }
    const bool mask = obj_alpha > 0.0f && depth_mask;
    if (!mask) obj_alpha = 0.0f;  // :272, before non_object_alpha
    const float non_obj_alpha = __fsub_rn(1.0f, obj_alpha);
    if (GS && gs_front) obj_alpha = __fmul_rn(obj_alpha, non_gs_alpha);  // :277, also where obj_alpha is 0
    float sca = __fmul_rn(non_obj_alpha, alpha_f(a));
    if (GS) sca = __fmul_rn(sca, non_gs_alpha);  // (non_object_alpha * fg_alpha) * non_obj_3dgs_alpha
    float cd[3] = {1.0f, 1.0f, 1.0f};
    if (sca > 0.0f) {
        const uint32_t s = shadow[p];
#pragma unroll
        for (int c = 0; c < 3; c++) cd[c] = fminf(fmaxf(__fdiv_rn(byte_f(a, c), __fadd_rn(byte_f(s, c), 1e-6f)), 0.0f), 1.0f);
    }
    // shadow_mask tests all four channels; the alpha channel of color_diff is 1, |1 - 1| < 0.01 always holds
    const bool shadow_mask = !(fabsf(__fsub_rn(cd[0], 1.0f)) < 0.01f && fabsf(__fsub_rn(cd[1], 1.0f)) < 0.01f &&
                               fabsf(__fsub_rn(cd[2], 1.0f)) < 0.01f);
    const uint32_t bg = frame[p];
    float f[4] = {byte_f(bg, 0), byte_f(bg, 1), byte_f(bg, 2), byte_f(bg, 3)};
    if (shadow_mask) {  // :292, all four channels: (f * cd) * sca + f * (1 - sca), with cd = 1 on alpha
        const float keep = __fsub_rn(1.0f, sca);
#pragma unroll
        for (int c = 0; c < 4; c++) f[c] = __fadd_rn(__fmul_rn(__fmul_rn(f[c], c < 3 ? cd[c] : 1.0f), sca), __fmul_rn(f[c], keep));
    }
    // step 2 (:297-302): both blends read frame_tmp; the fire pass overwrites the object's where both apply
    const float tmp[3] = {f[0], f[1], f[2]};
    if (mask) {
        const float keep = __fsub_rn(1.0f, obj_alpha);
#pragma unroll
        for (int c = 0; c < 3; c++) f[c] = __fadd_rn(__fmul_rn(byte_f(o, c), obj_alpha), __fmul_rn(tmp[c], keep));
    }
    if (FIRE && depth_mask_smoke) {
        const uint32_t fi = fire[p];
        const float keep = __fsub_rn(1.0f, smoke_alpha);
#pragma unroll
        for (int c = 0; c < 3; c++) f[c] = __fadd_rn(byte_f(fi, c), __fmul_rn(tmp[c], keep));
    }
    out[p] = to_u8(f[0]) | (to_u8(f[1]) << 8) | (to_u8(f[2]) << 16) | (to_u8(f[3]) << 24);
}

}  // namespace gsr

using namespace gsr;

int gsr_percentile_low(int64_t n, const float* x, float* out, void* ws, size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_percentile_low");
    const cudaStream_t s = (cudaStream_t)stream;
    if (n <= 0 || n > 0x7fffffffLL || !x || !out) { set_error("gsr_percentile_low: bad arguments (n %lld)", (long long)n); return GSR_ERR_INVALID; }
    if (!ws || ((uintptr_t)ws & 15) || ws_bytes < GSR_PERCENTILE_BYTES) {
        set_error("gsr_percentile_low: workspace of %zu bytes, GSR_PERCENTILE_BYTES (%d) needed (16-byte aligned)", ws_bytes, GSR_PERCENTILE_BYTES);
        return GSR_ERR_WORKSPACE;
    }
    // numpy's index arithmetic, in float32 as NumPy >= 2 does it for a float32 array
    const float q = 0.001f / 100.0f;
    const float v = (float)(n - 1) * q;
    const float fi = floorf(v);
    const bool top = v >= (float)(n - 1);  // only n = 1: both statistics are the maximum (index -1)
    const float t = top ? 1.0f : v - fi;   // numpy's gamma is v - (-1) there
    const uint32_t rank = top ? (uint32_t)(n - 1) : (uint32_t)fi;
    PctState* st = (PctState*)ws;
    k_pct_init<<<1, 256, 0, s>>>(rank, st);
    const int64_t tiles = (n + PCT_THREADS * PCT_ITEMS - 1) / (PCT_THREADS * PCT_ITEMS);
    const unsigned grid = (unsigned)(tiles < 2048 ? tiles : 2048);
    for (int pass = 0; pass < 4; pass++) {
        k_pct_hist<<<grid, PCT_THREADS, 0, s>>>(n, x, pass, st);
        k_pct_pick<<<1, 256, 0, s>>>(pass, st);
    }
    if (!top) k_pct_above<<<grid, PCT_THREADS, 0, s>>>(n, x, st);
    k_pct_final<<<1, 1, 0, s>>>(t, top ? 1 : 0, st, out);
    return check_launch("gsr_percentile_low", false, s);
}

int gsr_composite(int32_t W, int32_t H, const uint8_t* frame, const uint8_t* obj, const float* obj_d, const uint8_t* shadow,
                  const float* shadow_d, const uint8_t* all, const uint8_t* gs, const float* gs_d, const uint8_t* smoke,
                  const float* smoke_d, const float* smoke_pct, const uint8_t* fire, uint8_t* out, void* stream) {
    NvtxRange nvtx_("gsr_composite");
    const cudaStream_t s = (cudaStream_t)stream;
    if (W <= 0 || H <= 0) { set_error("gsr_composite: bad size (%d x %d)", W, H); return GSR_ERR_INVALID; }
    if (!frame || !obj || !obj_d || !shadow || !shadow_d || !all || !out) { set_error("gsr_composite: a required layer is NULL"); return GSR_ERR_INVALID; }
    if (!gs != !gs_d || !smoke != !smoke_d || !smoke != !smoke_pct || (fire && !smoke)) {
        set_error("gsr_composite: optional layers must come with their depth (and the smoke percentile); fire needs smoke");
        return GSR_ERR_INVALID;
    }
    for (const void* q : {(const void*)frame, (const void*)obj, (const void*)shadow, (const void*)all, (const void*)gs, (const void*)smoke,
                          (const void*)fire, (const void*)out})
        if ((uintptr_t)q & 3) { set_error("gsr_composite: 8-bit RGBA layers must be 4-byte aligned"); return GSR_ERR_INVALID; }
    const int64_t HW = (int64_t)W * H;
    const unsigned grid = (unsigned)((HW + 255) / 256);
    const auto* f32 = (const uint32_t*)frame;
    const auto *o32 = (const uint32_t*)obj, *s32 = (const uint32_t*)shadow, *a32 = (const uint32_t*)all;
    const auto *g32 = (const uint32_t*)gs, *m32 = (const uint32_t*)smoke, *x32 = (const uint32_t*)fire;
    auto* out32 = (uint32_t*)out;
#define GSR_COMPOSITE(G, S, F) \
    k_composite<G, S, F><<<grid, 256, 0, s>>>(HW, f32, o32, obj_d, s32, shadow_d, a32, g32, gs_d, m32, smoke_d, smoke_pct, x32, out32)
    const int sel = (gs ? 4 : 0) | (smoke ? 2 : 0) | (fire ? 1 : 0);
    switch (sel) {
        case 0: GSR_COMPOSITE(false, false, false); break;
        case 2: GSR_COMPOSITE(false, true, false); break;
        case 3: GSR_COMPOSITE(false, true, true); break;
        case 4: GSR_COMPOSITE(true, false, false); break;
        case 6: GSR_COMPOSITE(true, true, false); break;
        default: GSR_COMPOSITE(true, true, true); break;
    }
#undef GSR_COMPOSITE
    return check_launch("gsr_composite", false, s);
}
