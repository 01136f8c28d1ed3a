// gsr_b200 forward pass: projection -> tile histogram/scan -> colour + instance emission -> per-tile depth sort -> blend.
//
// Replaces CudaRasterizer::Rasterizer::forward (DGR/cuda_rasterizer/rasterizer_impl.cu:197-339) and the
// kernels it drives (forward.cu:155-256 preprocessCUDA, rasterizer_impl.cu:70-138 duplicateWithKeys /
// identifyTileRanges, CUB InclusiveSum + DeviceRadixSort, forward.cu:261-378 renderCUDA).
//
// Pipeline (results are identical, see DESIGN.md):
//   k_project     every Gaussian: near cull, conservative screen test, EWA projection, radius, tile rectangle, ranked per-tile
//                 tickets, the geometry part of the record, the compact list of visible Gaussians;
//   k_tile_scan   exclusive scan over the tiles: ranges, R and the overflow flag stay on the device (no host round trip);
//   k_color_emit  every VISIBLE Gaussian: SH -> RGB from a TMA-staged row, one (depth bits, id, footprint mask) pair per
//                 (Gaussian, tile) scattered to ranges[tile].x + rank;
//   k_sort_tiles  one CTA per tile sorts its bucket by (depth bits, id) — exactly the order of the reference's stable radix sort
//                 of (tile | depth) keys, because the reference emits every (tile, Gaussian) pair once in ascending Gaussian id
//                 (rasterizer_impl.cu:98-108) — and transposes the footprint masks into the ballot matrix;
//   k_blend_lists (gsr_blend.cu) one warp per 8x4-pixel footprint blends its survivors.
//   Record, 48 bytes per visible Gaussian: {x, y, conic.a, conic.b | conic.c, opacity, depth, radius | r, g, b, log2 opacity}.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "gsr_common.cuh"
#include "gsr_packed.cuh"

namespace gsr {

static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
}
const char* last_error() { return g_err; }
int check_launch(const char* what, bool debug, cudaStream_t stream) {
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess && debug) e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return GSR_ERR_CUDA;
    }
    return GSR_OK;
}

// =====================================================================================================
// Kernel 1: projection of every Gaussian (k_project); its colour is evaluated later, only for the visible ones (k_color_emit)
// =====================================================================================================
struct PreParams {
    int P, D, M, W, H, gx, gy;
    float scale_modifier, tanfovx, tanfovy, focal_x, focal_y;
    int prefiltered, for_backward, rot_vec, tight;
    const float *means3D, *shs, *colors_precomp, *opacities, *scales, *rotations, *cov3D_precomp, *view, *proj, *campos;
    float4* records;
    float* cov3D;
    uint8_t* clamped;
    int* radii;
    uint32_t* tile_count;
    uint32_t* tile_big;
    uint32_t* ranks;
    uint32_t* vis_list;
    gsr_counters* counters;
};

constexpr int PRE_THREADS = 128;

__host__ __device__ constexpr int sh_nf(int deg) { return 3 * (deg + 1) * (deg + 1); }
__host__ __device__ constexpr int sh_nv(int deg, bool win) { return (sh_nf(deg) + 3) / 4 + (win ? 1 : 0); }  // float4 per staged row
__host__ __device__ constexpr int sh_stride(int deg, bool vec, bool win = false) {
    // vec: rows of nv float4, padded so that (stride/4) is odd -> conflict-free LDS.128 across 8 lanes
    // scalar: odd number of words -> conflict-free LDS.32
    return vec ? (sh_nv(deg, win) % 2 == 0 ? (sh_nv(deg, win) + 1) * 4 : sh_nv(deg, win) * 4) : (sh_nf(deg) | 1);
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

// TMA bulk copy (cp.async.bulk, SASS UBLKCP) of one contiguous row global -> shared, completion on an mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}

// SH -> RGB for one Gaussian from its staged row (forward.cu:20-71).  Like cov3d_ref_rounding below, the
// roundings are pinned to the instruction sequence nvcc 12.9 emits for the reference (SASS of oracle/_ref):
// every coefficient C*poly(dir) is built from separate multiplies (only 3xx-yy, 4zz-xx, 2zz-3xx-3yy, xx-3yy use
// an FMA), and each term is accumulated with one FMA, in the reference's order.
template <int DEG>
__device__ __forceinline__ void sh_eval(const float* sh, float3 pos, const float* campos, float* rgb, unsigned& clamp_bits) {
    const float dx = __fsub_rn(pos.x, campos[0]), dy = __fsub_rn(pos.y, campos[1]), dz = __fsub_rn(pos.z, campos[2]);
    const float len = __fsqrt_rn(__fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy))));
    const float x = __fdiv_rn(dx, len), y = __fdiv_rn(dy, len), z = __fdiv_rn(dz, len);
    float k[16];
    k[0] = SH_C0;
    if (DEG > 0) {
        k[1] = -__fmul_rn(y, SH_C1);
        k[2] = __fmul_rn(z, SH_C1);
        k[3] = -__fmul_rn(x, SH_C1);
    }
    if (DEG > 1) {
        const float xy = __fmul_rn(y, x), yz = __fmul_rn(z, y), zz = __fmul_rn(z, z), xx = __fmul_rn(x, x), yy = __fmul_rn(y, y);
        const float xz = __fmul_rn(z, x), zz2 = __fadd_rn(zz, zz), xmy = __fsub_rn(xx, yy);
        k[4] = __fmul_rn(xy, SH_C2_0);
        k[5] = __fmul_rn(yz, SH_C2_1);
        k[6] = __fmul_rn(__fsub_rn(__fsub_rn(zz2, xx), yy), SH_C2_2);
        k[7] = __fmul_rn(xz, SH_C2_3);
        k[8] = __fmul_rn(xmy, SH_C2_4);
        if (DEG > 2) {
            const float f = __fsub_rn(__fmaf_rn(zz, 4.0f, -xx), yy);  // 4zz - xx - yy
            k[9] = __fmul_rn(__fmul_rn(y, SH_C3_0), __fmaf_rn(xx, 3.0f, -yy));
            k[10] = __fmul_rn(__fmul_rn(xy, SH_C3_1), z);
            k[11] = __fmul_rn(__fmul_rn(y, SH_C3_2), f);
            k[12] = __fmul_rn(__fmul_rn(z, SH_C3_3), __fmaf_rn(yy, -3.0f, __fmaf_rn(xx, -3.0f, zz2)));
            k[13] = __fmul_rn(__fmul_rn(x, SH_C3_4), f);
            k[14] = __fmul_rn(__fmul_rn(z, SH_C3_5), xmy);
            k[15] = __fmul_rn(__fmul_rn(x, SH_C3_6), __fmaf_rn(yy, -3.0f, xx));
        }
    }
    constexpr int NC = (DEG + 1) * (DEG + 1);
    clamp_bits = 0;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        float res = __fmul_rn(sh[c], k[0]);
#pragma unroll
        for (int i = 1; i < NC; i++) res = __fmaf_rn(k[i], sh[i * 3 + c], res);
        const float v = __fadd_rn(res, 0.5f);
        const bool neg = v < 0.f;  // == (res < -0.5f)
        if (neg) clamp_bits |= 1u << c;
        rgb[c] = neg ? 0.0f : v;
    }
}

// 3D covariance from scale / rotation (forward.cu:118-152: Sigma = (S R)^T (S R), quaternion not normalised).
// The roundings (which product of each sum is fused into an FMA, which terms multiply the structural zeros of
// S) are pinned with intrinsics to what nvcc 12.9 emits for the reference's GLM expression on sm_90a
// (read from the SASS of oracle/_ref), because the compiler's contraction choices depend on common
// sub-expression sharing and cannot be reproduced by writing "the same" C++ expression in another kernel.
// A 1-ulp difference here changes conic -> alpha -> the T < 1e-4 termination of a pixel now and then.
__device__ __forceinline__ void cov3d_ref_rounding(float sx, float sy, float sz, float mod, float4 q, float* c3) {
    const float r = q.x, x = q.y, y = q.z, z = q.w;
    const float xz = __fmul_rn(x, z), rx = __fmul_rn(r, x);
    const float A02 = __fmaf_rn(r, y, xz), A20 = __fmaf_rn(-r, y, xz);
    const float rz = __fmul_rn(r, z);
    const float A12 = __fmaf_rn(y, z, -rx), A21 = __fmaf_rn(y, z, rx);
    const float yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
    const float A01 = __fmaf_rn(x, y, -rz), A10 = __fmaf_rn(x, y, rz);
    const float B22 = __fmaf_rn(x, x, yy), B00 = __fadd_rn(yy, zz), B11 = __fmaf_rn(x, x, zz);
    const float s0 = __fmul_rn(mod, sx), s1 = __fmul_rn(mod, sy), s2 = __fmul_rn(mod, sz);
    // rotation matrix, R<c><r> = column c, row r
    const float R00 = __fsub_rn(1.f, __fadd_rn(B00, B00)), R01 = __fadd_rn(A01, A01), R02 = __fadd_rn(A02, A02);
    const float R10 = __fadd_rn(A10, A10), R11 = __fsub_rn(1.f, __fadd_rn(B11, B11)), R12 = __fadd_rn(A12, A12);
    const float R20 = __fadd_rn(A20, A20), R21 = __fadd_rn(A21, A21), R22 = __fsub_rn(1.f, __fadd_rn(B22, B22));
    // M = S * R with S = diag(s0, s1, s2): M<c><r> = S[0][r] R[c][0] + S[1][r] R[c][1] + S[2][r] R[c][2]
    const float z0 = __fmul_rn(0.f, R21), z00 = __fmul_rn(0.f, R00), z11 = __fmul_rn(0.f, R11);
    const float uM22 = __fmaf_rn(0.f, R20, z0), uM20 = __fmaf_rn(s0, R20, z0), uM21 = __fmaf_rn(0.f, R20, __fmul_rn(s1, R21));
    const float uM01 = __fmaf_rn(s1, R01, z00), uM02 = __fmaf_rn(0.f, R01, z00), uM00 = __fmaf_rn(0.f, R01, __fmul_rn(s0, R00));
    const float uM10 = __fmaf_rn(s0, R10, z11), uM11 = __fmaf_rn(0.f, R10, __fmul_rn(s1, R11)), uM12 = __fmaf_rn(0.f, R10, z11);
    const float M20 = __fmaf_rn(0.f, R22, uM20), M21 = __fmaf_rn(0.f, R22, uM21), M22 = __fmaf_rn(s2, R22, uM22);
    const float M00 = __fmaf_rn(0.f, R02, uM00), M01 = __fmaf_rn(0.f, R02, uM01), M02 = __fmaf_rn(s2, R02, uM02);
    const float M10 = __fmaf_rn(0.f, R12, uM10), M11 = __fmaf_rn(0.f, R12, uM11), M12 = __fmaf_rn(s2, R12, uM12);
    // Sigma = M^T M, upper triangle
    c3[0] = __fmaf_rn(M02, M02, __fmaf_rn(M00, M00, __fmul_rn(M01, M01)));
    c3[1] = __fmaf_rn(M02, M12, __fmaf_rn(M00, M10, __fmul_rn(M01, M11)));
    c3[2] = __fmaf_rn(M02, M22, __fmaf_rn(M00, M20, __fmul_rn(M01, M21)));
    c3[3] = __fmaf_rn(M12, M12, __fmaf_rn(M10, M10, __fmul_rn(M11, M11)));
    c3[4] = __fmaf_rn(M12, M22, __fmaf_rn(M10, M20, __fmul_rn(M11, M21)));
    c3[5] = __fmaf_rn(M22, M22, __fmaf_rn(M20, M20, __fmul_rn(M21, M21)));
}

// Kernel 1 of 5 (colour-agnostic; DEG / VEC / BULK / WIN only matter to k_color_emit below).
// Phase 1, one thread per Gaussian: load the 44 bytes of geometry, near cull, and a cheap CONSERVATIVE screen test — an upper
// bound of the splat radius (trace and norm bounds, see radius_bound) against the image rectangle; a Gaussian it rejects has an
// empty tile rectangle in the reference too (forward.cu:236), so it gets radius 0 without the projection math.  The survivors of
// the CTA are compacted through shared memory.  Phase 2, one thread per survivor (whole warps retire early): 3D covariance, EWA
// projection, conic, radius, tile rectangle (forward.cu:155-256 minus the colour), the per-tile histogram with ranked tickets,
// and the compact list of visible Gaussians the colour + emission kernel walks.  The 192-byte SH row is not touched here.
struct ProjCand {  // one phase-1 survivor
    float mx, my, mz, opacity;
    float a0, a1, a2, a3, a4, a5, a6;  // scale.xyz + rotation.rxyz, or cov3D[0..5]
    int idx;
};

template <int MINB, bool TIGHT>
__global__ void __launch_bounds__(PRE_THREADS, MINB) k_project(const PreParams p) {
    __shared__ CamConsts cam;
    __shared__ float s_w2;                       // upper bound of the squared spectral norm of the view matrix's 3x3 part
    __shared__ ProjCand s_cand[PRE_THREADS];
    __shared__ int s_wcnt[PRE_THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 16) cam.view[tid] = p.view[tid];
    else if (tid < 32) cam.proj[tid - 16] = p.proj[tid - 16];
    __syncthreads();
    if (tid == 0) {
        // rigid view matrices have orthonormal rows: then the norm is 1; anything else falls back to the Frobenius norm
        const float* v = cam.view;
        float dev = 0.f, frob = 0.f;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) {
                const float d = v[i] * v[j] + v[4 + i] * v[4 + j] + v[8 + i] * v[8 + j] - (i == j ? 1.f : 0.f);
                dev = fmaxf(dev, fabsf(d));
                frob += v[4 * j + i] * v[4 * j + i];
            }
        s_w2 = dev < 1.0e-3f ? 1.01f : frob * 1.01f;
    }
    __syncthreads();

    const int idx0 = blockIdx.x * PRE_THREADS + tid;
    const bool valid0 = idx0 < p.P;
    bool cand = false;
    ProjCand me;
    me.idx = idx0;
    if (valid0) {
        // all per-Gaussian inputs are requested up front (one memory round trip instead of three dependent ones)
        me.mx = p.means3D[3 * (size_t)idx0]; me.my = p.means3D[3 * (size_t)idx0 + 1]; me.mz = p.means3D[3 * (size_t)idx0 + 2];
        me.opacity = p.opacities[idx0];
        if (p.cov3D_precomp != nullptr) {
            const float* c = p.cov3D_precomp + 6 * (size_t)idx0;
            me.a0 = c[0]; me.a1 = c[1]; me.a2 = c[2]; me.a3 = c[3]; me.a4 = c[4]; me.a5 = c[5]; me.a6 = 0.f;
        } else {
            me.a0 = p.scales[3 * (size_t)idx0]; me.a1 = p.scales[3 * (size_t)idx0 + 1]; me.a2 = p.scales[3 * (size_t)idx0 + 2];
            float4 q;
            if (p.rot_vec) q = reinterpret_cast<const float4*>(p.rotations)[idx0];
            else q = make_float4(p.rotations[4 * (size_t)idx0], p.rotations[4 * (size_t)idx0 + 1], p.rotations[4 * (size_t)idx0 + 2], p.rotations[4 * (size_t)idx0 + 3]);
            me.a3 = q.x; me.a4 = q.y; me.a5 = q.z; me.a6 = q.w;
        }
        const float3 mean = {me.mx, me.my, me.mz};
        const float3 p_view = xform4x3(mean, cam.view);
        if (p_view.z <= 0.2f) {  // near cull (auxiliary.h:139-164): only view-space z is tested
            if (p.prefiltered) p.counters->trapped = 1;
        } else {
            // upper bound of the radius: lambda_max(cov2D) <= trace <= |J|_F^2 |W|_2^2 lambda_max(Sigma) + 0.6, and
            // lambda1 = mid + sqrt(max(0.1, mid^2 - det)) <= 2 mid + 0.32
            float lam;
            if (p.cov3D_precomp != nullptr) lam = me.a0 + me.a3 + me.a5;  // trace(Sigma)
            else {
                const float s2 = p.scale_modifier * p.scale_modifier * fmaxf(me.a0 * me.a0, fmaxf(me.a1 * me.a1, me.a2 * me.a2));
                const float n = me.a3 * me.a3 + me.a4 * me.a4 + me.a5 * me.a5 + me.a6 * me.a6;       // |q|^2 (not normalised by the rasterizer)
                const float r2 = fabsf(n - 1.f) < 1.0e-3f ? 1.01f : 9.f * (1.f + 2.f * n) * (1.f + 2.f * n);  // |R|_2^2 <= |R|_F^2 bound
                lam = s2 * r2;
            }
            const float limx = 1.3f * p.tanfovx, limy = 1.3f * p.tanfovy;
            const float cj = p.focal_x * p.focal_x * (1.f + limx * limx) + p.focal_y * p.focal_y * (1.f + limy * limy);
            const float l1 = cj * s_w2 * lam / (p_view.z * p_view.z) * 1.01f + 0.92f;
            const float rmax = ceilf(3.f * sqrtf(l1)) + 2.f;
            const float4 p_hom = xform4x4(mean, cam.proj);
            const float p_w = 1.0f / (p_hom.w + 0.0000001f);
            const float px = ((p_hom.x * p_w + 1.0f) * p.W - 1.0f) * 0.5f, py = ((p_hom.y * p_w + 1.0f) * p.H - 1.0f) * 0.5f;
            // empty tile rectangle (auxiliary.h:46-56): px + r < 1 or px - r >= 16 gx (same in y); one pixel of slack for the float evaluation
            const bool off = (px + rmax < -1.f) || (px - rmax > (float)(p.gx * GSR_TILE) + 1.f) || (py + rmax < -1.f) || (py - rmax > (float)(p.gy * GSR_TILE) + 1.f);
            cand = !off;
        }
        if (!cand) p.radii[idx0] = 0;
    }
    // ---- CTA-level compaction of the candidates ----
    const unsigned cm = __ballot_sync(GSR_FULL, cand);
    if (lane == 0) s_wcnt[warp] = __popc(cm);
    __syncthreads();
    int base = 0, ncand = 0;
#pragma unroll
    for (int w = 0; w < PRE_THREADS / 32; w++) {
        if (w < warp) base += s_wcnt[w];
        ncand += s_wcnt[w];
    }
    if (cand) s_cand[base + __popc(cm & ((1u << lane) - 1u))] = me;
    __syncthreads();
    if (warp * 32 >= ncand) return;  // whole warp without work

    // ---- phase 2 ----
    const bool valid = tid < ncand;
    const ProjCand c = s_cand[valid ? tid : 0];
    const int idx = c.idx;
    bool vis = false;
    int radius = 0, x0 = 0, y0 = 0, x1 = 0, y1 = 0;
    float px = 0, py = 0, depth = 0, con_a = 0, con_b = 0, con_c = 0;
    float c3[6] = {0, 0, 0, 0, 0, 0};
    const float opacity = c.opacity;
    if (valid) {
        const float3 mean = {c.mx, c.my, c.mz};
        if (p.cov3D_precomp != nullptr) { c3[0] = c.a0; c3[1] = c.a1; c3[2] = c.a2; c3[3] = c.a3; c3[4] = c.a4; c3[5] = c.a5; }
        float4 p_hom = xform4x4(mean, cam.proj);
        float p_w = 1.0f / (p_hom.w + 0.0000001f);
        float3 p_proj = {p_hom.x * p_w, p_hom.y * p_w, p_hom.z * p_w};
        float3 p_view = xform4x3(mean, cam.view);
        {
            // 3D covariance (forward.cu:118-152)
            if (p.cov3D_precomp == nullptr) cov3d_ref_rounding(c.a0, c.a1, c.a2, p.scale_modifier, make_float4(c.a3, c.a4, c.a5, c.a6), c3);
            // EWA 2D covariance (forward.cu:74-113)
            float3 t = xform4x3(mean, cam.view);
            const float limx = 1.3f * p.tanfovx, limy = 1.3f * p.tanfovy;
            const float txtz = t.x / t.z, tytz = t.y / t.z;
            t.x = min(limx, max(-limx, txtz)) * t.z;
            t.y = min(limy, max(-limy, tytz)) * t.z;
            m3 J = m3_make(p.focal_x / t.z, 0.0f, -(p.focal_x * t.x) / (t.z * t.z),
                           0.0f, p.focal_y / t.z, -(p.focal_y * t.y) / (t.z * t.z),
                           0, 0, 0);
            m3 Wm = m3_make(cam.view[0], cam.view[4], cam.view[8], cam.view[1], cam.view[5], cam.view[9],
                            cam.view[2], cam.view[6], cam.view[10]);
            m3 T = m3_mul(Wm, J);
            m3 Vrk = m3_make(c3[0], c3[1], c3[2], c3[1], c3[3], c3[4], c3[2], c3[4], c3[5]);
            m3 cov = m3_mul(m3_mul(m3_t(T), m3_t(Vrk)), T);
            cov.m[0][0] += 0.3f;
            cov.m[1][1] += 0.3f;
            const float cx = cov.m[0][0], cy = cov.m[0][1], cz = cov.m[1][1];
            // conic, radius, tile rectangle (forward.cu:217-237)
            float det = (cx * cz - cy * cy);
            if (det != 0.0f) {
                float det_inv = 1.f / det;
                con_a = cz * det_inv; con_b = -cy * det_inv; con_c = cx * det_inv;
                float mid = 0.5f * (cx + cz);
                float lambda1 = mid + sqrt(max(0.1f, mid * mid - det));
                float lambda2 = mid - sqrt(max(0.1f, mid * mid - det));
                float my_radius = ceil(3.f * sqrt(max(lambda1, lambda2)));
                px = ndc2pix(p_proj.x, p.W);
                py = ndc2pix(p_proj.y, p.H);
                tile_rect(px, py, (int)my_radius, p.gx, p.gy, x0, y0, x1, y1);
                if ((x1 - x0) * (y1 - y0) != 0) {
                    vis = true;
                    radius = (int)my_radius;
                    depth = p_view.z;
                }
            }
        }
    }
    if (!vis) { x0 = y0 = x1 = y1 = 0; }

    // Per-tile histogram.  Gaussians touching <= 8 tiles take a ranked ticket per tile (atomic with return) in COLUMN-major
    // order — the order k_color_emit walks them — and store the ranks, so the emission needs no atomics.  Larger rectangles
    // are counted separately, warp-cooperatively.  With p.tight a tile of the reference's rectangle only receives an instance
    // if the splat can reach alpha >= 1/255 at one of its pixel centres (opt-in: lists differ from the reference's, images do not).
    const float tau = footprint_tau(opacity);
    uint32_t rk[8];
    const int rect_h = y1 - y0, rect_n = (x1 - x0) * rect_h;
    if (rect_n > 0 && rect_n <= 8) {
        int tx = x0, ty = y0;
#pragma unroll
        for (int k = 0; k < 8; k++) {
            if (k < rect_n) {
                rk[k] = 0xffffffffu;
                if (!TIGHT || tile_may_touch(px, py, con_a, con_b, con_c, tau, tx, ty)) rk[k] = atomicAdd(&p.tile_count[ty * p.gx + tx], 1u);
                if (++ty == y1) { ty = y0; tx++; }
            }
        }
    }
    {
        const bool big = rect_n > 8;
        uint32_t* tb = p.tile_big;
        if (TIGHT) {
            const uint32_t pay[6] = {__float_as_uint(px), __float_as_uint(py), __float_as_uint(con_a), __float_as_uint(con_b),
                                     __float_as_uint(con_c), __float_as_uint(tau)};
            for_each_tile<0, 6>(big ? x0 : 0, big ? y0 : 0, big ? x1 : 0, big ? y1 : 0, p.gx, pay, [&](int tile, int tx, int ty, const uint32_t(&o)[6]) {
                if (tile_may_touch(__uint_as_float(o[0]), __uint_as_float(o[1]), __uint_as_float(o[2]), __uint_as_float(o[3]),
                                   __uint_as_float(o[4]), __uint_as_float(o[5]), tx, ty))
                    atomicAdd(&tb[tile], 1u);
            });
        } else {
            const uint32_t pay[1] = {0u};
            for_each_tile<0, 1>(big ? x0 : 0, big ? y0 : 0, big ? x1 : 0, big ? y1 : 0, p.gx, pay,
                                [&](int tile, int, int, const uint32_t(&)[1]) { atomicAdd(&tb[tile], 1u); });
        }
    }

    if (valid) {
        p.radii[idx] = radius;
        if (vis) {
            float4* rec = p.records + 3 * (size_t)idx;
            rec[0] = make_float4(px, py, con_a, con_b);
            rec[1] = make_float4(con_c, opacity, depth, __int_as_float(radius));
            rec[2] = make_float4(c.mx, c.my, c.mz, 0.0f);  // the mean, for k_color_emit's view direction (it overwrites the quad with the colour)
            if (rect_n <= 8) {
                uint4* rr = reinterpret_cast<uint4*>(p.ranks + 8 * (size_t)idx);
                rr[0] = make_uint4(rk[0], rk[1], rk[2], rk[3]);
                if (rect_n > 4) rr[1] = make_uint4(rk[4], rk[5], rk[6], rk[7]);
            }
            if (p.for_backward && p.cov3D_precomp == nullptr) {
#pragma unroll
                for (int k = 0; k < 6; k++) p.cov3D[6 * (size_t)idx + k] = c3[k];
            }
        }
    }
    // compact list of the visible Gaussians (order is irrelevant: every entry is processed independently)
    const unsigned vm = __ballot_sync(GSR_FULL, vis);
    if (vm) {
        uint32_t vbase = 0;
        if (lane == __ffs(vm) - 1) vbase = atomicAdd(&p.counters->num_visible, (uint32_t)__popc(vm));
        vbase = __shfl_sync(GSR_FULL, vbase, __ffs(vm) - 1);
        if (vis) p.vis_list[vbase + __popc(vm & ((1u << lane) - 1u))] = (uint32_t)idx;
    }
}

// =====================================================================================================
// Kernel 2: exclusive scan over the per-tile counts -> ranges, R, overflow flag (single CTA)
// =====================================================================================================
__global__ void __launch_bounds__(1024) k_tile_scan(const uint32_t* __restrict__ tile_count, const uint32_t* __restrict__ tile_big,
                                                    uint32_t* __restrict__ tile_fill, uint2* __restrict__ ranges,
                                                    gsr_counters* counters, int tiles, uint32_t capacity) {
    // Every thread owns SCAN_PER consecutive tiles (16-byte loads and stores; the arrays are 256-byte aligned), so a 1080p frame
    // (8,160 tiles) is one pass with two barriers instead of eight chunks of 1024 tiles with three barriers each.
    constexpr int SCAN_PER = 8;
    __shared__ uint32_t warp_sum[32];
    __shared__ uint32_t warp_max[32];
    __shared__ uint32_t chunk_total;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t carry = 0, lmax = 0;
    for (int base = 0; base < tiles; base += 1024 * SCAN_PER) {
        const int t0 = base + tid * SCAN_PER;
        uint32_t cs[SCAN_PER], c[SCAN_PER];
        if (t0 + SCAN_PER <= tiles) {
            const uint4 a0 = *reinterpret_cast<const uint4*>(tile_count + t0), a1 = *reinterpret_cast<const uint4*>(tile_count + t0 + 4);
            const uint4 b0 = *reinterpret_cast<const uint4*>(tile_big + t0), b1 = *reinterpret_cast<const uint4*>(tile_big + t0 + 4);
            cs[0] = a0.x; cs[1] = a0.y; cs[2] = a0.z; cs[3] = a0.w; cs[4] = a1.x; cs[5] = a1.y; cs[6] = a1.z; cs[7] = a1.w;
            c[0] = a0.x + b0.x; c[1] = a0.y + b0.y; c[2] = a0.z + b0.z; c[3] = a0.w + b0.w;
            c[4] = a1.x + b1.x; c[5] = a1.y + b1.y; c[6] = a1.z + b1.z; c[7] = a1.w + b1.w;
        } else {
#pragma unroll
            for (int k = 0; k < SCAN_PER; k++) {
                const int t = t0 + k;
                cs[k] = t < tiles ? tile_count[t] : 0u;
                c[k] = cs[k] + (t < tiles ? tile_big[t] : 0u);
            }
        }
        uint32_t sum = 0;
#pragma unroll
        for (int k = 0; k < SCAN_PER; k++) { sum += c[k]; lmax = max(lmax, c[k]); }
        uint32_t incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(GSR_FULL, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) warp_sum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const uint32_t s = warp_sum[lane];
            uint32_t si = s;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t v = __shfl_up_sync(GSR_FULL, si, o);
                if (lane >= o) si += v;
            }
            warp_sum[lane] = si - s;  // exclusive
            if (lane == 31) chunk_total = si;
        }
        __syncthreads();
        uint32_t start = carry + warp_sum[warp] + (incl - sum);
        uint2 rg[SCAN_PER];
        uint32_t fill[SCAN_PER];
#pragma unroll
        for (int k = 0; k < SCAN_PER; k++) {
            rg[k] = c[k] ? make_uint2(start, start + c[k]) : make_uint2(0u, 0u);
            fill[k] = start + cs[k];  // absolute cursor of the tile's un-ranked (large-rectangle) instances
            start += c[k];
        }
        if (t0 + SCAN_PER <= tiles) {
#pragma unroll
            for (int k = 0; k < SCAN_PER; k += 2) reinterpret_cast<uint4*>(ranges + t0)[k >> 1] = make_uint4(rg[k].x, rg[k].y, rg[k + 1].x, rg[k + 1].y);
            reinterpret_cast<uint4*>(tile_fill + t0)[0] = make_uint4(fill[0], fill[1], fill[2], fill[3]);
            reinterpret_cast<uint4*>(tile_fill + t0)[1] = make_uint4(fill[4], fill[5], fill[6], fill[7]);
        } else {
#pragma unroll
            for (int k = 0; k < SCAN_PER; k++)
                if (t0 + k < tiles) { ranges[t0 + k] = rg[k]; tile_fill[t0 + k] = fill[k]; }
        }
        carry += chunk_total;
        __syncthreads();
    }
    lmax = __reduce_max_sync(GSR_FULL, lmax);
    if (lane == 0) warp_max[warp] = lmax;
    __syncthreads();
    if (warp == 0) {
        const uint32_t m = __reduce_max_sync(GSR_FULL, warp_max[lane]);
        if (lane == 0) {
            counters->num_rendered = carry;
            counters->overflow = carry > capacity ? 1u : 0u;
            counters->max_tile = m;
        }
    }
}

// =====================================================================================================
// Kernel 3 of 5: colour + instance emission, one thread per VISIBLE Gaussian (the compact list k_project wrote), every
// lane busy.  (a) SH -> RGB (forward.cu:20-71) from the Gaussian's SH row, staged by ONE TMA bulk copy issued by its own
// lane; (b) the work of duplicateWithKeys (rasterizer_impl.cu:70-111): one (depth bits, id) pair per (Gaussian, tile)
// scattered to ranges[tile].x + rank — the ranks were drawn by k_project, so no atomics for rectangles of <= 8 tiles;
// (c) PACKED (P <= 2^24): the pair's low word is (id << 8 | mask), mask = which of the tile's eight 8x4 warp footprints the
// splat can touch (strip intervals, computed once per tile column of the rectangle), so k_sort_tiles needs no gather.
// The kernel streams 192 B of SH per thread and has issue slots to spare for (c).
// DEG = -1: colours are precomputed.  VEC: SH rows are 16-byte aligned (M % 4 == 0) -> 16-byte staging, either one TMA
// bulk copy per Gaussian (BULK) or coalesced cp.async by the whole warp.  WIN (with VEC and BULK): rows are only 4-byte
// aligned (M = 25, the SuGaR storage: 300-byte rows) — each lane bulk-copies the 16-byte aligned window that contains its
// coefficients (one extra float4) and evaluates from its row's offset inside the window.
// =====================================================================================================
struct EmitParams {
    int P, M, gx, gy, for_backward;
    const float *shs, *colors_precomp, *campos;
    float4* records;
    uint8_t* clamped;
    const uint32_t* ranks;
    const uint32_t* vis_list;
    const uint2* ranges;
    uint32_t* tile_fill;
    uint2* pairs;
    const gsr_counters* counters;
};

template <int DEG, bool VEC, bool BULK, bool WIN, bool TIGHT, bool PACKED>
__global__ void __launch_bounds__(PRE_THREADS, 8) k_color_emit(const EmitParams p) {
    constexpr int DG = DEG < 0 ? 0 : DEG;
    constexpr int NF = sh_nf(DG);
    constexpr int STRIDE = sh_stride(DG, VEC, WIN);
    __shared__ float campos[3];
    // per warp: the SH staging rows of its 32 Gaussians, later reused as the emission's owner table (16 words per Gaussian)
    constexpr int WSTAGE = (DEG < 0 || 32 * STRIDE < 16 * 32) ? 16 * 32 : 32 * STRIDE;
    __shared__ __align__(16) float stage[(PRE_THREADS / 32) * WSTAGE];
    __shared__ __align__(8) unsigned long long stage_bar[PRE_THREADS / 32];

    const uint32_t nvis = p.counters->num_visible;
    if (blockIdx.x * PRE_THREADS >= nvis) return;  // the grid is sized for P; blocks past the visible list leave at once
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (BULK && lane == 0) {
        mbar_init((uint32_t)__cvta_generic_to_shared(&stage_bar[warp]), 1u);
        mbar_fence_init();
    }
    if (tid < 3) campos[tid] = p.campos[tid];
    __syncthreads();

    const uint32_t k = blockIdx.x * PRE_THREADS + tid;
    const bool vis = k < nvis;
    const uint32_t idx = vis ? p.vis_list[k] : 0u;
    // the whole 48-byte record (two 32-byte sectors whichever part is read): geometry, radius, and the mean k_project parked in the colour quad
    float4 r0 = make_float4(0, 0, 0, 0), r1 = r0, r2 = r0;
    int radius = 0;
    if (vis) {
        r0 = p.records[3 * (size_t)idx];
        r1 = p.records[3 * (size_t)idx + 1];
        r2 = p.records[3 * (size_t)idx + 2];
        radius = __float_as_int(r1.w);
    }
    const float tau = footprint_tau(r1.y);  // = the value k_project used for its tight-tile decisions (same function of the same opacity)

    // ---- colour ----
    float rgb[3] = {0, 0, 0};
    unsigned clamp_bits = 0;
    float* wstage = stage + warp * WSTAGE;
    if constexpr (DEG < 0) {
        if (vis) {
            rgb[0] = p.colors_precomp[3 * (size_t)idx];
            rgb[1] = p.colors_precomp[3 * (size_t)idx + 1];
            rgb[2] = p.colors_precomp[3 * (size_t)idx + 2];
        }
    } else {
        const float3 mean = {r2.x, r2.y, r2.z};
        const unsigned vismask = __ballot_sync(GSR_FULL, vis);
        const size_t row_floats = (size_t)p.M * 3;
        int win_off = 0;  // floats between the start of the staged window and the row's first coefficient (WIN only)
        if (VEC && BULK) {
            constexpr int NV = sh_nv(DG, WIN);
            const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&stage_bar[warp]);
            if (vismask) {
                if (lane == 0) mbar_arrive_expect_tx(bar, (uint32_t)__popc(vismask) * NV * 16u);
                if (vis) {
                    const float* src = p.shs + (size_t)idx * row_floats;
                    if (WIN) {
                        win_off = (int)(((uintptr_t)src & 15u) >> 2);
                        src -= win_off;
                    }
                    bulk_g2s((uint32_t)__cvta_generic_to_shared(wstage + lane * STRIDE), src, NV * 16u, bar);
                }
                mbar_wait(bar, 0u);
            }
        } else if (VEC) {
            constexpr int NV = (NF + 3) / 4;
#pragma unroll
            for (int it = 0; it < NV; it++) {
                const int item = it * 32 + lane;
                const int gl = item / NV, part = item - gl * NV;
                const uint32_t gid = __shfl_sync(GSR_FULL, idx, gl);
                if ((vismask >> gl) & 1u) cp_async16(wstage + gl * STRIDE + part * 4, p.shs + (size_t)gid * row_floats + part * 4);
            }
            cp_async_wait_all();
        } else {
#pragma unroll 4
            for (int it = 0; it < NF; it++) {
                const int item = it * 32 + lane;
                const int gl = item / NF, part = item - gl * NF;
                const uint32_t gid = __shfl_sync(GSR_FULL, idx, gl);
                if ((vismask >> gl) & 1u) wstage[gl * STRIDE + part] = p.shs[(size_t)gid * row_floats + part];
            }
        }
        __syncwarp();
        if (vis) sh_eval<DG>(wstage + lane * STRIDE + win_off, mean, campos, rgb, clamp_bits);
    }
    if (vis) {
        p.records[3 * (size_t)idx + 2] = make_float4(rgb[0], rgb[1], rgb[2], log2f(r1.y));  // .w: log2(opacity) for the default blend
        if (p.for_backward) p.clamped[idx] = (uint8_t)clamp_bits;
    }

    // ---- emission ----
    // The (Gaussian, tile column) pairs of the warp's 32 Gaussians are FLATTENED into one work list and dealt to the lanes round
    // robin, so a lane whose Gaussian covers one tile does not idle while its neighbour walks a 3x3 rectangle: every owner parks
    // its rectangle, strip context and key words in shared memory, a warp scan of the per-Gaussian item counts gives each item
    // its owner (binary search over 32 prefix sums), and the item's lane evaluates the two strips of its column once and walks
    // the column's (at most 8) tiles.  Columns taller than 8 tiles (rectangles of > 8 tiles only) are split into chunks of 8 rows.
    if (p.counters->overflow) return;  // set by k_tile_scan: the binning buffer is too small for this frame
    int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
    if (vis) tile_rect(r0.x, r0.y, radius, p.gx, p.gy, x0, y0, x1, y1);
    const int w = x1 - x0, h = y1 - y0, cnt = w * h;
    const int cpc = (h + 7) >> 3;  // chunks per column
    const int n_items = w * cpc;
    float* own = wstage;  // the SH staging area is free after sh_eval
    __syncwarp();
    {
        StripCtx sc = {};
        if (PACKED && cnt > 0) {
            const float um = fmaxf(r0.x - (float)(x0 * GSR_TILE), (float)(x1 * GSR_TILE) - r0.x);
            const float vm = fmaxf(r0.y - (float)(y0 * GSR_TILE), (float)(y1 * GSR_TILE) - r0.y);
            sc = strip_ctx(r0.x, r0.y, r0.z, r0.w, r1.x, tau, um, vm);
        }
        own[0 * 32 + lane] = r0.x; own[1 * 32 + lane] = r0.y; own[2 * 32 + lane] = r0.w; own[3 * 32 + lane] = sc.det;
        own[4 * 32 + lane] = sc.rc; own[5 * 32 + lane] = sc.cT; own[6 * 32 + lane] = sc.sstar;
        own[7 * 32 + lane] = __uint_as_float((sc.ok ? 1u : 0u) | (sc.none ? 2u : 0u) | (cnt > 8 ? 4u : 0u));
        own[8 * 32 + lane] = __uint_as_float((uint32_t)x0 | ((uint32_t)y0 << 16));
        own[9 * 32 + lane] = __uint_as_float((uint32_t)w | ((uint32_t)h << 16));
        own[10 * 32 + lane] = __uint_as_float(idx);
        own[11 * 32 + lane] = r1.z;   // depth
        own[12 * 32 + lane] = r0.z;   // conic a
        own[13 * 32 + lane] = r1.x;   // conic c
        own[14 * 32 + lane] = tau;
    }
    int incl = n_items;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(GSR_FULL, incl, o);
        if (lane >= o) incl += v;
    }
    own[15 * 32 + lane] = __int_as_float(incl - n_items);  // exclusive prefix of the item counts
    const int total = __shfl_sync(GSR_FULL, incl, 31);
    __syncwarp();
    for (int j = lane; j < total; j += 32) {
        int g = 0;  // owner: the last Gaussian whose prefix is <= j
#pragma unroll
        for (int step = 16; step > 0; step >>= 1)
            if (__float_as_int(own[15 * 32 + g + step]) <= j) g += step;
        const int local = j - __float_as_int(own[15 * 32 + g]);
        const uint32_t wh = __float_as_uint(own[9 * 32 + g]), xy = __float_as_uint(own[8 * 32 + g]), fl = __float_as_uint(own[7 * 32 + g]);
        const int gh = (int)(wh >> 16), gx0 = (int)(xy & 0xffffu), gy0 = (int)(xy >> 16);
        const int gcpc = (gh + 7) >> 3;
        const int col = gcpc == 1 ? local : local / gcpc, chunk = local - col * gcpc;
        const int tx = gx0 + col, ty_lo = gy0 + 8 * chunk, ty_hi = min(gy0 + gh, ty_lo + 8);
        const uint32_t gid = __float_as_uint(own[10 * 32 + g]), dbits = __float_as_uint(own[11 * 32 + g]);
        const uint32_t lo_id = PACKED ? gid << 8 : gid;
        const bool big = fl & 4u;
        const float gpx = own[0 * 32 + g], gpy = own[1 * 32 + g], gb = own[2 * 32 + g];
        float ylo0 = 0.f, yhi0 = 0.f, ylo1 = 0.f, yhi1 = 0.f;
        bool v0 = false, v1 = false;
        if (PACKED && (fl & 1u) && !(fl & 2u)) {
            StripCtx c2;
            c2.px = gpx; c2.py = gpy; c2.b = gb; c2.det = own[3 * 32 + g]; c2.rc = own[4 * 32 + g]; c2.cT = own[5 * 32 + g]; c2.sstar = own[6 * 32 + g];
            c2.ok = true; c2.none = false;
            v0 = strip_rows(c2, (float)(tx * GSR_TILE), 8.f, ylo0, yhi0);
            v1 = strip_rows(c2, (float)(tx * GSR_TILE + 8), 8.f, ylo1, yhi1);
        }
        // The rows [ylo, yhi] a strip covers, as a bit mask over the (at most 32) 4-row bands of this column chunk: band k = rows
        // [Y0 + 4k, Y0 + 4k + 3] is touched iff ylo <= Y0 + 4k + 3 and yhi >= Y0 + 4k, i.e. ceil((ylo - Y0 - 3) / 4) <= k <= floor((yhi - Y0) / 4).
        // Two conversions per strip instead of eight comparisons per tile; near a band boundary the subtractions are exact (Y0 is an
        // integer within a factor two of y), and the strips carry a 0.01-pixel margin anyway.
        const float Y0 = (float)(ty_lo * GSR_TILE);
        auto band_bits = [&](const bool v, const float ylo, const float yhi) -> uint32_t {
            const float a = fminf(fmaxf((ylo - Y0 - 3.f) * 0.25f, -1.f), 33.f), b = fminf(fmaxf((yhi - Y0) * 0.25f, -1.f), 33.f);
            const int klo = max((int)ceilf(a), 0), khi = min((int)floorf(b), 31);
            return (v && klo <= khi) ? (0xffffffffu >> (31 - khi)) & (0xffffffffu << klo) : 0u;
        };
        const uint32_t bands0 = band_bits(v0, ylo0, yhi0), bands1 = band_bits(v1, ylo1, yhi1);
        // Slots of the column's (at most 8) tiles first — rank + start of the tile's bucket, or a ticket from the per-tile cursor for
        // rectangles of > 8 tiles — so that up to 16 independent loads / atomics are in flight while the masks are computed.
        const uint32_t* rk = p.ranks + 8 * (size_t)gid + col * gh + (ty_lo - gy0);  // column-major ranks of a <= 8-tile rectangle
        uint32_t pos[8];
#pragma unroll
        for (int r = 0; r < 8; r++) {
            pos[r] = 0xffffffffu;
            const int ty = ty_lo + r;
            if (ty < ty_hi) {
                const int tile = ty * p.gx + tx;
                if (!big) {
                    const uint32_t rank = rk[r];
                    const uint32_t start = p.ranges[tile].x;
                    pos[r] = (TIGHT && rank == 0xffffffffu) ? 0xffffffffu : start + rank;
                } else if (!TIGHT || tile_may_touch(gpx, gpy, own[12 * 32 + g], gb, own[13 * 32 + g], own[14 * 32 + g], tx, ty)) {
                    // the tight-tile test is re-evaluated on the same stored values k_project used (bitwise same decision)
                    pos[r] = atomicAdd(&p.tile_fill[tile], 1u);
                }
            }
        }
#pragma unroll
        for (int r = 0; r < 8; r++) {
            const int ty = ty_lo + r;
            if (ty < ty_hi && pos[r] != 0xffffffffu) {
                uint32_t mask = 0;
                if (PACKED) {
                    if (!(fl & 1u)) mask = tile_foot_mask(gpx, gpy, own[12 * 32 + g], gb, own[13 * 32 + g], own[14 * 32 + g], tx, ty);
                    else {  // the tile's four bands of both strips, interleaved: bit 2q + i = band q of strip i
                        uint32_t n0 = (bands0 >> (4 * r)) & 15u, n1 = (bands1 >> (4 * r)) & 15u;
                        n0 = (n0 | (n0 << 2)) & 0x33u; n0 = (n0 | (n0 << 1)) & 0x55u;
                        n1 = (n1 | (n1 << 2)) & 0x33u; n1 = (n1 | (n1 << 1)) & 0x55u;
                        mask = n0 | (n1 << 1);
                    }
                }
                p.pairs[pos[r]] = make_uint2(lo_id | mask, dbits);  // little endian: u64 = depth bits << 32 | low word
            }
        }
    }
}

// =====================================================================================================
// Kernel 4: per-tile sort of the bucket by (depth bits, id) -> point_list
// Normalised bitonic network (all compare-exchanges ascending), valid for any n by skipping partners >= n.
// =====================================================================================================
constexpr int SORT_THREADS = 256;
constexpr int SORT_CAP = 4096;  // u64 entries in shared memory (32 KB)

template <typename T>
__device__ __forceinline__ void cmpx(T* a, uint32_t i, uint32_t l) {
    const unsigned long long x = a[i], y = a[l];
    if (x > y) { a[i] = y; a[l] = x; }
}
// one "flip" step of block size k over the first N slots (N power of two), entries >= n are virtual +inf
__device__ __forceinline__ void step_flip(unsigned long long* a, uint32_t n, uint32_t N, uint32_t k) {
    const uint32_t half = k >> 1;
    for (uint32_t t = threadIdx.x; t < (N >> 1); t += SORT_THREADS) {
        const uint32_t i = ((t & ~(half - 1)) << 1) | (t & (half - 1));
        const uint32_t l = i ^ (k - 1);
        if (l < n) cmpx(a, i, l);
    }
}
__device__ __forceinline__ void step_j(unsigned long long* a, uint32_t n, uint32_t N, uint32_t j) {
    for (uint32_t t = threadIdx.x; t < (N >> 1); t += SORT_THREADS) {
        const uint32_t i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const uint32_t l = i + j;
        if (l < n) cmpx(a, i, l);
    }
}
__device__ __forceinline__ uint32_t next_pow2(uint32_t n) { return n <= 1 ? 1u : 1u << (32 - __clz(n - 1)); }

// full sort of a[0..n) (n <= SORT_CAP) in shared memory
__device__ void sort_smem(unsigned long long* s, uint32_t n) {
    const uint32_t N = next_pow2(n);
    for (uint32_t k = 2; k <= N; k <<= 1) {
        step_flip(s, n, N, k);
        __syncthreads();
        for (uint32_t j = k >> 2; j > 0; j >>= 1) {
            step_j(s, n, N, j);
            __syncthreads();
        }
    }
}

// ---- bucket sort for n <= SORT_CAP (the common case) -----------------------------------------------------
// The keys of one tile are (depth bits << 32 | id) with depths spread over [zmin, zmax] of the tile.  A monotone
// linear quantisation of the depth into B >= n/2 buckets (float subtract, multiply by a positive constant and
// truncation are all monotone) puts ~1 key in each bucket, so the sort is: histogram (shared atomics, the
// returned value is the key's slot in its bucket) -> exclusive scan -> scatter -> per-bucket insertion sort on
// the full 64-bit key, O(n) work instead of the O(n log^2 n) network.  The result is the unique ascending
// order, whatever order the atomics happened in.  Buckets holding more than SORT_BUCKET_MAX keys (all depths
// equal, or extreme clustering) trigger the generic network on the same shared array instead.
constexpr int SORT_BUCKETS = 2048;
constexpr int SORT_BUCKET_MAX = 24;

template <bool PACKED>
__device__ void sort_bucket(const unsigned long long* __restrict__ g, uint32_t n, uint32_t* __restrict__ out,
                            unsigned long long* __restrict__ gkeep, unsigned long long* s, uint32_t* hist /*[SORT_BUCKETS+1]*/) {
    __shared__ uint32_t red_min[SORT_THREADS / 32], red_max[SORT_THREADS / 32], wsum[SORT_THREADS / 32];
    __shared__ int fallback;
    const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const uint32_t B = min((uint32_t)SORT_BUCKETS, max(32u, next_pow2(n)));
    // the keys are read three times from global memory (L2 hits after the first pass) instead of being held in
    // up to 32 registers per thread: min/max, bucket + ticket, scatter
    uint32_t dmin = 0xffffffffu, dmax = 0u;
    for (uint32_t i = t; i < n; i += SORT_THREADS) {
        const uint32_t d = (uint32_t)(g[i] >> 32);
        dmin = min(dmin, d);
        dmax = max(dmax, d);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        dmin = min(dmin, __shfl_xor_sync(GSR_FULL, dmin, o));
        dmax = max(dmax, __shfl_xor_sync(GSR_FULL, dmax, o));
    }
    if (lane == 0) { red_min[warp] = dmin; red_max[warp] = dmax; }
    if (t == 0) fallback = 0;
    for (uint32_t b = t; b <= B; b += SORT_THREADS) hist[b] = 0;
    __syncthreads();
#pragma unroll
    for (int w = 0; w < SORT_THREADS / 32; w++) { dmin = min(dmin, red_min[w]); dmax = max(dmax, red_max[w]); }
    const float zmin = __uint_as_float(dmin), zmax = __uint_as_float(dmax);  // positive floats: bit order == value order
    const float scale = zmax > zmin ? (float)(B - 1) / (zmax - zmin) : 0.f;
    // ticket = (bucket << 16) | slot-in-bucket, parked in the output array until the scatter (a bucket with
    // >= 65536 keys cannot occur: n <= SORT_CAP)
    for (uint32_t i = t; i < n; i += SORT_THREADS) {
        const float d = __uint_as_float((uint32_t)(g[i] >> 32));
        const uint32_t b = min(B - 1, (uint32_t)((d - zmin) * scale));
        out[i] = (b << 16) | atomicAdd(&hist[b], 1u);
    }
    __syncthreads();
    {   // exclusive scan of hist[0..B) in place, hist[B] = n
        const uint32_t per = B / SORT_THREADS > 0 ? B / SORT_THREADS : 1;  // B is a power of two >= 32
        const uint32_t b0 = t * per;
        uint32_t loc[SORT_BUCKETS / SORT_THREADS];
        uint32_t sum = 0;
#pragma unroll
        for (uint32_t k = 0; k < SORT_BUCKETS / SORT_THREADS; k++) {
            loc[k] = 0;
            if (k < per && b0 + k < B) { loc[k] = hist[b0 + k]; }
            sum += loc[k];
        }
        uint32_t incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t x = __shfl_up_sync(GSR_FULL, incl, o);
            if (lane >= o) incl += x;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        uint32_t base = incl - sum;
#pragma unroll
        for (int w = 0; w < SORT_THREADS / 32; w++) base += (w < (int)warp) ? wsum[w] : 0u;
#pragma unroll
        for (uint32_t k = 0; k < SORT_BUCKETS / SORT_THREADS; k++) {
            if (k < per && b0 + k < B) { hist[b0 + k] = base; base += loc[k]; }
        }
        if (t == 0) hist[B] = n;
    }
    __syncthreads();
    for (uint32_t i = t; i < n; i += SORT_THREADS) {
        const uint32_t tk = out[i];
        s[hist[tk >> 16] + (tk & 0xffffu)] = g[i];
    }
    __syncthreads();
    for (uint32_t b = t; b < B; b += SORT_THREADS) {  // order the few keys that share a bucket
        const uint32_t lo = hist[b], c = hist[b + 1] - lo;
        if (c > (uint32_t)SORT_BUCKET_MAX) fallback = 1;
        else if (c > 1) {
            for (uint32_t i = 1; i < c; i++) {
                const unsigned long long x = s[lo + i];
                uint32_t j = i;
                while (j > 0 && s[lo + j - 1] > x) { s[lo + j] = s[lo + j - 1]; j--; }
                s[lo + j] = x;
            }
        }
    }
    __syncthreads();
    if (fallback) sort_smem(s, n);  // ends with a barrier
    for (uint32_t i = t; i < n; i += SORT_THREADS) {
        const unsigned long long x = s[i];
        const uint32_t id = PACKED ? (uint32_t)x >> 8 : (uint32_t)x;  // PACKED: low word = id << 8 | footprint mask
        out[i] = id;
        if (gkeep) gkeep[i] = (x & 0xffffffff00000000ull) | id;
    }
}

// bucket of a depth (bit pattern of a positive float): monotone, and pinned to one subtraction and one multiplication so that every
// evaluation for the same key yields the same bucket (sort_bucket_small evaluates it twice per key)
__device__ __forceinline__ uint32_t depth_bucket(uint32_t dbits, float zmin, float scale, uint32_t B) {
    return min(B - 1, (uint32_t)__fmul_rn(__fsub_rn(__uint_as_float(dbits), zmin), scale));
}

struct FootArgs;  // defined with the ballot matrix below
template <bool PACKED>
__device__ void foot_ballots(const FootArgs& fa, const unsigned long long* keys, uint32_t n, uint32_t range_x, int tile);
__device__ __forceinline__ uint32_t* foot_bal_rows(const FootArgs& fa, uint32_t range_x, int tile);

// ---- the same bucket sort for n <= SORT_SMALL: one pass over global memory -------------------------------------------------
// The shared key array is split into two halves: the keys are read from global memory ONCE into the first half (the depth
// range is reduced on the way), the tickets (bucket << 6 | slot) live in a 16-bit shared array instead of the output buffer, and
// the scatter goes shared -> shared into the second half.  A bucket with more than 63 keys (the ticket's slot field saturates)
// sorts the first half with the generic network instead.  The ids go to point_list and (PACKED) the footprint masks of 32
// consecutive sorted entries to one row of the ballot matrix in the same pass over the sorted keys.
constexpr int SORT_SMALL = SORT_CAP / 2;

template <bool PACKED>
__device__ void sort_bucket_small(const unsigned long long* __restrict__ g, uint32_t n, uint32_t* __restrict__ out,
                                  unsigned long long* __restrict__ gkeep, unsigned long long* s, uint32_t* hist, uint16_t* tk16,
                                  const FootArgs& fa, uint32_t range_x, int tile) {
    __shared__ uint32_t red_min[SORT_THREADS / 32], red_max[SORT_THREADS / 32], wsum[SORT_THREADS / 32];
    __shared__ int fallback;
    const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
    // n/2 .. n buckets (1 - 2 keys each): half the histogram / scan work of one bucket per key, measured 3 % faster; 4x fewer: slower.
    // B <= 1024 (n <= SORT_SMALL): a ticket is bucket (10 bits) | slot (6 bits), so a bucket may hold up to 63 keys before the
    // tile falls back to the generic network (depth outliers that stretch the tile's range crowd the other keys into few buckets)
    const uint32_t B = min((uint32_t)SORT_BUCKETS / 2, max(32u, next_pow2(n) >> 1));
    constexpr uint32_t SLOT_BITS = 6u, SLOT_MAX = (1u << SLOT_BITS) - 1u;
    unsigned long long* A = s;
    unsigned long long* Bf = s + SORT_SMALL;
    uint32_t dmin = 0xffffffffu, dmax = 0u;
#pragma unroll 4
    for (uint32_t i = t; i < n; i += SORT_THREADS) {
        const unsigned long long k = g[i];
        A[i] = k;
        const uint32_t d = (uint32_t)(k >> 32);
        dmin = min(dmin, d);
        dmax = max(dmax, d);
    }
    dmin = __reduce_min_sync(GSR_FULL, dmin);  // REDUX: one instruction per warp-wide reduction
    dmax = __reduce_max_sync(GSR_FULL, dmax);
    if (lane == 0) { red_min[warp] = dmin; red_max[warp] = dmax; }
    if (t == 0) fallback = 0;
    for (uint32_t b = t; b <= B; b += SORT_THREADS) hist[b] = 0;
    __syncthreads();
#pragma unroll
    for (int w = 0; w < SORT_THREADS / 32; w++) { dmin = min(dmin, red_min[w]); dmax = max(dmax, red_max[w]); }
    const float zmin = __uint_as_float(dmin), zmax = __uint_as_float(dmax);  // positive floats: bit order == value order
    const float scale = zmax > zmin ? (float)(B - 1) / (zmax - zmin) : 0.f;
    bool over = false;
    for (uint32_t i = t; i < n; i += SORT_THREADS) {
        const uint32_t b = depth_bucket((uint32_t)(A[i] >> 32), zmin, scale, B);
        const uint32_t slot = atomicAdd(&hist[b], 1u);
        over |= slot >= SLOT_MAX;
        tk16[i] = (uint16_t)((b << SLOT_BITS) | min(slot, SLOT_MAX));
    }
    if (over) fallback = 1;
    __syncthreads();
    if (fallback) {  // block-uniform
        sort_smem(A, n);  // ends with a barrier
    } else {
        {   // exclusive scan of hist[0..B) in place, hist[B] = n
            const uint32_t per = B / SORT_THREADS > 0 ? B / SORT_THREADS : 1;  // B is a power of two >= 32
            const uint32_t b0 = t * per;
            uint32_t loc[SORT_BUCKETS / SORT_THREADS];
            uint32_t sum = 0;
#pragma unroll
            for (uint32_t k = 0; k < SORT_BUCKETS / SORT_THREADS; k++) {
                loc[k] = 0;
                if (k < per && b0 + k < B) { loc[k] = hist[b0 + k]; }
                sum += loc[k];
            }
            uint32_t incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t x = __shfl_up_sync(GSR_FULL, incl, o);
                if (lane >= o) incl += x;
            }
            if (lane == 31) wsum[warp] = incl;
            __syncthreads();
            uint32_t base = incl - sum;
#pragma unroll
            for (int w = 0; w < SORT_THREADS / 32; w++) base += (w < (int)warp) ? wsum[w] : 0u;
#pragma unroll
            for (uint32_t k = 0; k < SORT_BUCKETS / SORT_THREADS; k++) {
                if (k < per && b0 + k < B) { hist[b0 + k] = base; base += loc[k]; }
            }
            if (t == 0) hist[B] = n;
        }
        __syncthreads();
        for (uint32_t i = t; i < n; i += SORT_THREADS) {
            const uint32_t tk = tk16[i];
            Bf[hist[tk >> SLOT_BITS] + (tk & SLOT_MAX)] = A[i];
        }
        __syncthreads();
        // Final order, one thread per KEY (balanced, no divergent insertion loops): a key's place inside its bucket is the number
        // of smaller keys in it (the keys are distinct: the id is part of them); bucket order -> sorted order, second half -> first.
        for (uint32_t i = t; i < n; i += SORT_THREADS) {  // in bucket order: neighbouring threads read neighbouring buckets
            const unsigned long long k = Bf[i];
            const uint32_t b = depth_bucket((uint32_t)(k >> 32), zmin, scale, B);  // the very same roundings as the ticket pass
            const uint32_t lo = hist[b], c = hist[b + 1] - lo;
            uint32_t rank = 0;
            for (uint32_t j = 0; j < c; j++) rank += Bf[lo + j] < k ? 1u : 0u;
            A[lo + rank] = k;
        }
        __syncthreads();
    }
    if (!PACKED) {  // masks from gathered records (P > 2^24): the general ballot routine
        for (uint32_t i = t; i < n; i += SORT_THREADS) {
            const unsigned long long x = A[i];
            out[i] = (uint32_t)x;
            if (gkeep) gkeep[i] = x;
        }
        foot_ballots<PACKED>(fa, A, n, range_x, tile);  // A[] is only read after the sort's last barrier
        return;
    }
    uint32_t* bal = foot_bal_rows(fa, range_x, tile);
    for (uint32_t base = warp * 32; base < n; base += SORT_THREADS) {  // warp-uniform: 32 consecutive sorted entries per warp and step
        const uint32_t i = base + lane;
        uint32_t m = 0;
        if (i < n) {
            const unsigned long long x = A[i];
            const uint32_t id = (uint32_t)x >> 8;  // low word = id << 8 | footprint mask
            m = (uint32_t)x & 0xffu;
            out[i] = id;
            if (gkeep) gkeep[i] = (x & 0xffffffff00000000ull) | id;
        }
        uint32_t mine = 0;
#pragma unroll
        for (int f = 0; f < GSR_FOOTS; f++) {
            const uint32_t b = __ballot_sync(GSR_FULL, (m >> f) & 1u);
            if (lane == (uint32_t)f) mine = b;
        }
        if (lane < GSR_FOOTS) bal[(base >> 5) * GSR_FOOTS + lane] = mine;  // one 32-byte row
    }
}

// ---- footprint ballot matrix ------------------------------------------------------------------------------------
// After the sort every entry of the tile carries an 8-bit mask: which of the tile's eight 8x4-pixel warp footprints the splat
// can touch (PACKED: the low byte of the key, computed by k_color_emit; otherwise the record is gathered and the mask computed
// here).  The masks of 32 consecutive list entries are transposed by eight ballots into one ROW of the ballot matrix:
// bal[row][f] = bit i set iff entry 32 row + i touches footprint f.  The blend warp that owns footprint f reads column f — one
// word per 32 entries — and expands it into the positions of its survivors on the fly, so the blend has no per-entry cull
// and no lists have to be allocated.  Rows of tile t start at (ranges[t].x >> 5) + t.
struct FootArgs {
    const float4* records;
    uint32_t* bal;  // [rows][GSR_FOOTS]
    int gx;
};

__device__ __forceinline__ uint32_t* foot_bal_rows(const FootArgs& fa, uint32_t range_x, int tile) { return fa.bal + bal_row_base(range_x, tile) * GSR_FOOTS; }

// keys: the n sorted keys of the tile (shared or global memory)
template <bool PACKED>
__device__ void foot_ballots(const FootArgs& fa, const unsigned long long* keys, uint32_t n, uint32_t range_x, int tile) {
    const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const uint32_t* klo = reinterpret_cast<const uint32_t*>(keys);  // low word of key i
    uint32_t* bal = fa.bal + bal_row_base(range_x, tile) * GSR_FOOTS;
    const int ty = tile / fa.gx, tx = tile - ty * fa.gx;
    for (uint32_t c0 = 0; c0 < n; c0 += 2 * SORT_THREADS) {
        float4 r0[2], r1[2];
        uint32_t lo[2];
#pragma unroll
        for (int u = 0; u < 2; u++) {  // two gathers in flight per thread on the general path
            const uint32_t i = c0 + u * SORT_THREADS + t;
            r0[u] = r1[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            lo[u] = 0;
            if (i < n) {
                lo[u] = klo[2 * i];
                if (!PACKED) {
                    const float4* r = fa.records + 3 * (size_t)lo[u];
                    r0[u] = r[0];
                    r1[u] = r[1];
                }
            }
        }
#pragma unroll
        for (int u = 0; u < 2; u++) {
            const uint32_t rbase = c0 + u * SORT_THREADS + warp * 32;  // warp-uniform
            if (rbase < n) {
                uint32_t m = 0;
                if (rbase + lane < n) m = PACKED ? lo[u] & 0xffu : tile_foot_mask_any(r0[u].x, r0[u].y, r0[u].z, r0[u].w, r1[u].x, footprint_tau(r1[u].y), tx, ty);
                uint32_t mine = 0;
#pragma unroll
                for (int f = 0; f < GSR_FOOTS; f++) {
                    const uint32_t b = __ballot_sync(GSR_FULL, (m >> f) & 1u);
                    if (lane == (uint32_t)f) mine = b;
                }
                if (lane < GSR_FOOTS) bal[(rbase >> 5) * GSR_FOOTS + lane] = mine;  // one 32-byte row
            }
        }
    }
}

// Sorts the bucket of one tile (pairs[rg.x..rg.y) by (depth bits, id)) and writes the ids to point_list.
// s: SORT_CAP u64 of shared memory, hist: SORT_BUCKETS+1 u32.  Block-wide (SORT_THREADS threads), ends without a barrier.
template <bool PACKED>
__device__ void sort_tile(const uint2 rg, unsigned long long* __restrict__ pairs, uint32_t* __restrict__ point_list, int keep_pairs,
                          unsigned long long* s, uint32_t* hist, uint16_t* tk16, const FootArgs& fa, int tile) {
    const uint32_t n = rg.y - rg.x;
    const uint32_t tid = threadIdx.x;
    if (n == 0) return;
    unsigned long long* g = pairs + rg.x;
    uint32_t* out = point_list + rg.x;
    if (n <= SORT_SMALL && tk16 != nullptr) {
        sort_bucket_small<PACKED>(g, n, out, keep_pairs ? g : nullptr, s, hist, tk16, fa, rg.x, tile);
        return;
    }
    if (n <= SORT_CAP) {
        sort_bucket<PACKED>(g, n, out, keep_pairs ? g : nullptr, s, hist);
        foot_ballots<PACKED>(fa, s, n, rg.x, tile);  // s[] still holds the sorted keys (only read after the sort's last barrier)
        return;
    }
    // ---- large tile: chunks sorted in shared memory, cross-chunk steps in global (L2) memory ----
    const uint32_t N = next_pow2(n);
    for (uint32_t c0 = 0; c0 < n; c0 += SORT_CAP) {
        const uint32_t m = min((uint32_t)SORT_CAP, n - c0);
        for (uint32_t i = tid; i < m; i += SORT_THREADS) s[i] = g[c0 + i];
        __syncthreads();
        sort_smem(s, m);
        for (uint32_t i = tid; i < m; i += SORT_THREADS) g[c0 + i] = s[i];
        __syncthreads();
    }
    for (uint32_t k = 2 * SORT_CAP; k <= N; k <<= 1) {
        step_flip(g, n, N, k);
        __syncthreads();
        uint32_t j = k >> 2;
        for (; j >= SORT_CAP; j >>= 1) {
            step_j(g, n, N, j);
            __syncthreads();
        }
        for (uint32_t c0 = 0; c0 < n; c0 += SORT_CAP) {
            const uint32_t m = min((uint32_t)SORT_CAP, n - c0);
            for (uint32_t i = tid; i < m; i += SORT_THREADS) s[i] = g[c0 + i];
            __syncthreads();
            for (uint32_t jj = SORT_CAP >> 1; jj > 0; jj >>= 1) {
                step_j(s, m, SORT_CAP, jj);
                __syncthreads();
            }
            for (uint32_t i = tid; i < m; i += SORT_THREADS) g[c0 + i] = s[i];
            __syncthreads();
        }
    }
    __syncthreads();
    foot_ballots<PACKED>(fa, g, n, rg.x, tile);
    __syncthreads();
    for (uint32_t i = tid; i < n; i += SORT_THREADS) {
        const unsigned long long x = g[i];
        const uint32_t id = PACKED ? (uint32_t)x >> 8 : (uint32_t)x;
        out[i] = id;
        if (PACKED && keep_pairs) g[i] = (x & 0xffffffff00000000ull) | id;
    }
}

// stand-alone per-tile sort kernel
template <bool PACKED>
__global__ void __launch_bounds__(SORT_THREADS, 5) k_sort_tiles(const uint2* __restrict__ ranges, unsigned long long* __restrict__ pairs,
                                                             uint32_t* __restrict__ point_list,
                                                             const gsr_counters* __restrict__ counters, int keep_pairs, const FootArgs fa,
                                                             const int sort_small_enabled) {
    if (counters->overflow) return;  // set by k_tile_scan, before this kernel started
    __shared__ unsigned long long s[SORT_CAP];
    __shared__ uint32_t hist[SORT_BUCKETS + 1];
    __shared__ uint16_t tk16[SORT_SMALL];
    sort_tile<PACKED>(ranges[blockIdx.x], pairs, point_list, keep_pairs, s, hist, sort_small_enabled ? tk16 : nullptr, fa, (int)blockIdx.x);
}

// =====================================================================================================
// Second pass over identical geometry (GSR_FLAG_REUSE_GEOMETRY): the product frame renders every camera twice with
// the same Gaussians — SH colours, then colors_precomp = normals (gaussian_renderer/__init__.py:151-185,
// sugar_model.py:2141-2183).  Projection, binning and sorting of the first pass stay valid; only the colour slot of
// the visible records is rewritten before the blend.
// =====================================================================================================
__global__ void __launch_bounds__(256) k_recolor(int P, const int* __restrict__ radii, const float* __restrict__ colors_precomp,
                                                 float4* __restrict__ records) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P || radii[idx] <= 0) return;
    float* c = reinterpret_cast<float*>(records + 3 * (size_t)idx + 2);  // .w (log2 opacity) stays
    c[0] = colors_precomp[3 * (size_t)idx];
    c[1] = colors_precomp[3 * (size_t)idx + 1];
    c[2] = colors_precomp[3 * (size_t)idx + 2];
}

// =====================================================================================================
// optional per-kernel timing (bench.py roofline): CUDA events recorded around each forward kernel on the
// launching stream; no effect unless gsr_profile_begin() was called.  Not thread safe (one profiled stream).
// =====================================================================================================
struct ProfileState {
    bool on = false;
    int max_frames = 0, frames = 0;
    int stride = 1, seen = 0;  // every stride-th forward call is timed (the event records cost ~1.5 % of a frame)
    cudaEvent_t* ev = nullptr;  // 6 per frame
    int allocated = 0;
};
static ProfileState g_prof;
static inline void prof_mark(int k, cudaStream_t st) {
    if (g_prof.on && g_prof.frames < g_prof.max_frames && g_prof.seen % g_prof.stride == 0) cudaEventRecord(g_prof.ev[g_prof.frames * 6 + k], st);
}
int profile_begin(int max_frames, int stride) {
    if (max_frames <= 0 || stride <= 0) { set_error("gsr_profile_begin: max_frames and stride must be > 0"); return GSR_ERR_INVALID; }
    if (g_prof.allocated < max_frames * 6) {
        cudaEvent_t* ne = new cudaEvent_t[max_frames * 6];
        for (int i = 0; i < max_frames * 6; i++) {
            if (i < g_prof.allocated) ne[i] = g_prof.ev[i];
            else if (cudaEventCreate(&ne[i]) != cudaSuccess) { set_error("gsr_profile_begin: cudaEventCreate failed"); return GSR_ERR_CUDA; }
        }
        delete[] g_prof.ev;
        g_prof.ev = ne;
        g_prof.allocated = max_frames * 6;
    }
    g_prof.max_frames = max_frames;
    g_prof.frames = 0;
    g_prof.stride = stride;
    g_prof.seen = 0;
    g_prof.on = true;
    return GSR_OK;
}
int profile_end(float* ms, int* frames) {
    g_prof.on = false;
    double acc[5] = {0, 0, 0, 0, 0};
    for (int f = 0; f < g_prof.frames; f++) {
        if (cudaEventSynchronize(g_prof.ev[f * 6 + 5]) != cudaSuccess) { set_error("gsr_profile_end: event sync failed"); return GSR_ERR_CUDA; }
        for (int k = 0; k < 5; k++) {
            float t = 0;
            cudaEventElapsedTime(&t, g_prof.ev[f * 6 + k], g_prof.ev[f * 6 + k + 1]);
            acc[k] += t;
        }
    }
    for (int k = 0; k < 5; k++) ms[k] = g_prof.frames ? (float)(acc[k] / g_prof.frames) : 0.f;
    if (frames) *frames = g_prof.frames;
    return GSR_OK;
}

// =====================================================================================================
// host side
// =====================================================================================================
static int sh_bulk_mode() {  // GSR_SH_STAGING=cpasync selects the LDGSTS path, default is the TMA bulk copy
    static int mode = -1;
    if (mode < 0) {
        const char* e = getenv("GSR_SH_STAGING");
        mode = (e && strcmp(e, "cpasync") == 0) ? 0 : 1;
    }
    return mode;
}
template <int DEG, bool TIGHT, bool PACKED>
static void launch_ce_v(bool vec, bool win, const EmitParams& ep, cudaStream_t st) {
    const int grid = (ep.P + PRE_THREADS - 1) / PRE_THREADS;  // sized for P; blocks past the visible list exit at once
    if (DEG < 0) k_color_emit<-1, false, false, false, TIGHT, PACKED><<<grid, PRE_THREADS, 0, st>>>(ep);
    else if (win && sh_bulk_mode()) k_color_emit<DEG, true, true, true, TIGHT, PACKED><<<grid, PRE_THREADS, 0, st>>>(ep);
    else if (vec && sh_bulk_mode()) k_color_emit<DEG, true, true, false, TIGHT, PACKED><<<grid, PRE_THREADS, 0, st>>>(ep);
    else if (vec) k_color_emit<DEG, true, false, false, TIGHT, PACKED><<<grid, PRE_THREADS, 0, st>>>(ep);
    else k_color_emit<DEG, false, false, false, TIGHT, PACKED><<<grid, PRE_THREADS, 0, st>>>(ep);
}
template <int DEG>
static void launch_color_emit(bool vec, bool win, bool tight, bool packed, const EmitParams& ep, cudaStream_t st) {
    if (tight) { if (packed) launch_ce_v<DEG, true, true>(vec, win, ep, st); else launch_ce_v<DEG, true, false>(vec, win, ep, st); }
    else       { if (packed) launch_ce_v<DEG, false, true>(vec, win, ep, st); else launch_ce_v<DEG, false, false>(vec, win, ep, st); }
}

static void launch_blend(const BlendArgs& a, cudaStream_t st) { launch_blend_lists(a, st); }

// process-wide experiment / tuning options of the forward (gsr_set_option)
struct ForwardOptions {
    int sort_single_pass = 1;  // tiles of <= SORT_SMALL instances are read from global memory once (sort_bucket_small)
};
static ForwardOptions g_opt;
int set_blend_persist(int k);
int set_option(const char* name, int value) {
    if (strcmp(name, "blend_persist") == 0) return set_blend_persist(value);
    if (strcmp(name, "sort_single_pass") == 0) { g_opt.sort_single_pass = value ? 1 : 0; return GSR_OK; }
    return GSR_ERR_INVALID;
}

int forward_impl(const gsr_frame* f, const gsr_workspace* ws, float* out_color, float* out_depth, float* out_alpha,
                 int32_t* radii, const float* extra_colors, float* out_extra, int flags, cudaStream_t st) {
    if (!f || !ws) { set_error("gsr_forward: null frame/workspace"); return GSR_ERR_INVALID; }
    if (f->P < 0 || f->W <= 0 || f->H <= 0) { set_error("gsr_forward: bad sizes P=%d W=%d H=%d", f->P, f->W, f->H); return GSR_ERR_INVALID; }
    if (!out_color || !out_depth || !out_alpha) { set_error("gsr_forward: null output image"); return GSR_ERR_INVALID; }
    if ((extra_colors == nullptr) != (out_extra == nullptr)) { set_error("gsr_forward_multi: extra_colors and out_extra go together"); return GSR_ERR_INVALID; }
    const size_t HW = (size_t)f->W * f->H;
    const ImageLayout il(f->W, f->H);
    if (!ws->image || ws->image_bytes < il.total) { set_error("gsr_forward: image workspace too small (%zu < %zu)", ws->image_bytes, il.total); return GSR_ERR_WORKSPACE; }
    char* img = (char*)ws->image;
    gsr_counters* counters = (gsr_counters*)(img + il.counters);
    const bool debug = f->debug != 0;
    if (f->P == 0) {  // rasterize_points.cu:68-71,82: zero images, nothing else runs
        cudaMemsetAsync(out_color, 0, 12 * HW, st);
        cudaMemsetAsync(out_depth, 0, 4 * HW, st);
        cudaMemsetAsync(out_alpha, 0, 4 * HW, st);
        if (out_extra) cudaMemsetAsync(out_extra, 0, 12 * HW, st);
        cudaMemsetAsync(img, 0, il.zero_bytes(), st);
        cudaMemsetAsync(img + il.ranges, 0, 8 * (size_t)il.tiles, st);
        return check_launch("gsr_forward(P=0)", debug, st);
    }
    if (!radii || !f->means3D || !f->opacities || !f->viewmatrix || !f->projmatrix || !f->campos || !f->bg) {
        set_error("gsr_forward: null required input");
        return GSR_ERR_INVALID;
    }
    if ((f->shs == nullptr) == (f->colors_precomp == nullptr)) { set_error("gsr_forward: provide exactly one of shs / colors_precomp"); return GSR_ERR_INVALID; }
    const bool has_sr = f->scales != nullptr && f->rotations != nullptr;
    if (has_sr == (f->cov3D_precomp != nullptr) || ((f->scales != nullptr) != (f->rotations != nullptr))) {
        set_error("gsr_forward: provide exactly one of scales+rotations / cov3D_precomp");
        return GSR_ERR_INVALID;
    }
    const int D = f->D < 0 ? 0 : (f->D > 3 ? 3 : f->D);
    if (f->shs && (D + 1) * (D + 1) > f->M) { set_error("gsr_forward: sh degree %d needs %d coefficients, shs has M=%d", D, (D + 1) * (D + 1), f->M); return GSR_ERR_INVALID; }
    const GeomLayout gl((size_t)f->P);
    if (!ws->geom || ws->geom_bytes < gl.total) { set_error("gsr_forward: geometry workspace too small (%zu < %zu)", ws->geom_bytes, gl.total); return GSR_ERR_WORKSPACE; }
    const size_t cap_nominal = ws->binning ? BinLayout::capacity_of(ws->binning_bytes) : 0;
    if (cap_nominal < 1) { set_error("gsr_forward: binning workspace too small"); return GSR_ERR_WORKSPACE; }
    const BinLayout bl(cap_nominal);
    // the ballot matrix needs capacity / 32 + tiles + 1 rows: images with more tiles than the fixed slack covers lower the usable capacity
    size_t cap = cap_nominal;
    if ((size_t)il.tiles + 1 > bl.bal_rows) { set_error("gsr_forward: binning workspace too small for %d tiles", il.tiles); return GSR_ERR_WORKSPACE; }
    if (cap / 32 + (size_t)il.tiles + 1 > bl.bal_rows) cap = 32 * (bl.bal_rows - (size_t)il.tiles - 1);
    if (cap < 1) { set_error("gsr_forward: binning workspace too small"); return GSR_ERR_WORKSPACE; }
    char* geo = (char*)ws->geom;
    char* bin = (char*)ws->binning;

    if (flags & GSR_FLAG_REUSE_GEOMETRY) {
        // `radii` is an INPUT here: the radii of the pass whose workspaces are being reused
        if (!f->colors_precomp) { set_error("gsr_forward: GSR_FLAG_REUSE_GEOMETRY needs colors_precomp"); return GSR_ERR_INVALID; }
        if (flags & GSR_FLAG_FOR_BACKWARD) { set_error("gsr_forward: GSR_FLAG_REUSE_GEOMETRY cannot be combined with GSR_FLAG_FOR_BACKWARD"); return GSR_ERR_INVALID; }
        k_recolor<<<(f->P + 255) / 256, 256, 0, st>>>(f->P, radii, f->colors_precomp, (float4*)(geo + gl.records));
        int rc0 = check_launch("gsr_forward/recolor", debug, st);
        if (rc0) return rc0;
        BlendArgs ba{(const uint2*)(img + il.ranges), (const uint32_t*)(bin + bl.point_list), (const float4*)(geo + gl.records), extra_colors,
                     f->W, f->H, il.gx, il.gy, f->bg, out_color, out_depth, out_alpha, out_extra, nullptr, counters,
                     (const uint32_t*)(bin + bl.bal), (flags & GSR_FLAG_EXACT_IMAGES) ? 1 : 0};
        launch_blend(ba, st);
        return check_launch("gsr_forward/blend(reuse)", debug, st);
    }

    // a frame can be issued in two calls — GSR_FLAG_BINNING_ONLY (projection + tile scan: the counters are final except for
    // exact_redos) and GSR_FLAG_RESUME (everything after it) — so that a caller who validates the capacity on the host can
    // start that round trip while the rest of the frame runs
    const bool resume = (flags & GSR_FLAG_RESUME) != 0;
    if ((flags & GSR_FLAG_BINNING_ONLY) && resume) { set_error("gsr_forward: GSR_FLAG_BINNING_ONLY and GSR_FLAG_RESUME are exclusive"); return GSR_ERR_INVALID; }
    if (!resume) {
        cudaMemsetAsync(img, 0, il.zero_bytes(), st);
        prof_mark(0, st);
    }

    PreParams pp;
    pp.P = f->P; pp.D = D; pp.M = f->M; pp.W = f->W; pp.H = f->H; pp.gx = il.gx; pp.gy = il.gy;
    pp.scale_modifier = f->scale_modifier; pp.tanfovx = f->tanfovx; pp.tanfovy = f->tanfovy;
    pp.focal_y = f->H / (2.0f * f->tanfovy);  // rasterizer_impl.cu:223-224
    pp.focal_x = f->W / (2.0f * f->tanfovx);
    pp.rot_vec = (((uintptr_t)f->rotations & 15) == 0) ? 1 : 0;
    pp.tight = (flags & GSR_FLAG_TIGHT_TILES) ? 1 : 0;
    pp.prefiltered = f->prefiltered; pp.for_backward = (flags & GSR_FLAG_FOR_BACKWARD) ? 1 : 0;
    pp.means3D = f->means3D; pp.shs = f->shs; pp.colors_precomp = f->colors_precomp; pp.opacities = f->opacities;
    pp.scales = f->scales; pp.rotations = f->rotations; pp.cov3D_precomp = f->cov3D_precomp;
    pp.view = f->viewmatrix; pp.proj = f->projmatrix; pp.campos = f->campos;
    pp.records = (float4*)(geo + gl.records); pp.cov3D = (float*)(geo + gl.cov3D); pp.clamped = (uint8_t*)(geo + gl.clamped);
    pp.radii = radii; pp.tile_count = (uint32_t*)(img + il.tile_count); pp.tile_big = (uint32_t*)(img + il.tile_big);
    pp.ranks = (uint32_t*)(geo + gl.ranks); pp.counters = counters;

    pp.vis_list = (uint32_t*)(geo + gl.vis_list);
    uint2* ranges = (uint2*)(img + il.ranges);
    int rc = GSR_OK;
    if (!resume) {
        static int minb = -1;  // GSR_PROJ_MINB=8|10|12: resident CTAs per SM the kernel is compiled for (experiment knob)
        if (minb < 0) { const char* e = getenv("GSR_PROJ_MINB"); minb = e ? atoi(e) : 8; }
        const int grid = (f->P + PRE_THREADS - 1) / PRE_THREADS;
        if (pp.tight) k_project<8, true><<<grid, PRE_THREADS, 0, st>>>(pp);
        else if (minb == 12) k_project<12, false><<<grid, PRE_THREADS, 0, st>>>(pp);
        else if (minb == 10) k_project<10, false><<<grid, PRE_THREADS, 0, st>>>(pp);
        else k_project<8, false><<<grid, PRE_THREADS, 0, st>>>(pp);
        prof_mark(1, st);
        if ((rc = check_launch("gsr_forward/project", debug, st))) return rc;

        k_tile_scan<<<1, 1024, 0, st>>>(pp.tile_count, pp.tile_big, (uint32_t*)(img + il.tile_fill), ranges, counters, il.tiles, (uint32_t)(cap > 0xffffffffull ? 0xffffffffull : cap));
        prof_mark(2, st);
        if ((rc = check_launch("gsr_forward/tile_scan", debug, st))) return rc;
    }
    if (flags & GSR_FLAG_BINNING_ONLY) return GSR_OK;

    // footprint masks travel in the low byte of the pair's id word when the ids fit 24 bits; GSR_PACKED_KEYS=0 forces the
    // general path (masks computed by k_sort_tiles from gathered records), which is what P > 2^24 uses
    static int packed_ok = -1;
    if (packed_ok < 0) { const char* e = getenv("GSR_PACKED_KEYS"); packed_ok = (e && e[0] == '0') ? 0 : 1; }
    const bool packed = packed_ok && f->P <= (1 << 24);
    EmitParams ep;
    ep.P = f->P; ep.M = f->M; ep.gx = il.gx; ep.gy = il.gy; ep.for_backward = pp.for_backward;
    ep.shs = f->shs; ep.colors_precomp = f->colors_precomp; ep.campos = f->campos;
    ep.records = pp.records; ep.clamped = pp.clamped; ep.ranks = pp.ranks; ep.vis_list = pp.vis_list;
    ep.ranges = ranges; ep.tile_fill = (uint32_t*)(img + il.tile_fill); ep.pairs = (uint2*)(bin + bl.pairs); ep.counters = counters;
    if (f->colors_precomp) launch_color_emit<-1>(false, false, pp.tight, packed, ep, st);
    else {
        const bool vec = (f->M % 4 == 0) && (((uintptr_t)f->shs & 15) == 0);
        // 4-byte aligned rows (e.g. M = 25): the aligned window of sh_nv(D, true) float4 must fit inside every row
        const bool win = !vec && (((uintptr_t)f->shs & 15) == 0) && (size_t)f->M * 12 >= (size_t)sh_nv(D, true) * 16;
        switch (D) {
            case 0: launch_color_emit<0>(vec, win, pp.tight, packed, ep, st); break;
            case 1: launch_color_emit<1>(vec, win, pp.tight, packed, ep, st); break;
            case 2: launch_color_emit<2>(vec, win, pp.tight, packed, ep, st); break;
            default: launch_color_emit<3>(vec, win, pp.tight, packed, ep, st); break;
        }
    }
    prof_mark(3, st);
    if ((rc = check_launch("gsr_forward/color_emit", debug, st))) return rc;

    const int keep_pairs = (flags & GSR_FLAG_SORTED_KEYS) ? 1 : 0;
    uint32_t* n_contrib = (flags & GSR_FLAG_FOR_BACKWARD) ? (uint32_t*)(img + il.n_contrib) : nullptr;
    FootArgs fa{pp.records, (uint32_t*)(bin + bl.bal), il.gx};
    if (packed) k_sort_tiles<true><<<il.tiles, SORT_THREADS, 0, st>>>(ranges, (unsigned long long*)(bin + bl.pairs), (uint32_t*)(bin + bl.point_list), counters, keep_pairs, fa, g_opt.sort_single_pass);
    else k_sort_tiles<false><<<il.tiles, SORT_THREADS, 0, st>>>(ranges, (unsigned long long*)(bin + bl.pairs), (uint32_t*)(bin + bl.point_list), counters, keep_pairs, fa, g_opt.sort_single_pass);
    prof_mark(4, st);
    if ((rc = check_launch("gsr_forward/sort", debug, st))) return rc;
    BlendArgs ba{ranges, (const uint32_t*)(bin + bl.point_list), pp.records, extra_colors, f->W, f->H, il.gx, il.gy, f->bg,
                 out_color, out_depth, out_alpha, out_extra, n_contrib, counters, (const uint32_t*)(bin + bl.bal),
                 (flags & GSR_FLAG_EXACT_IMAGES) ? 1 : 0};
    launch_blend(ba, st);
    prof_mark(5, st);
    if (g_prof.on) {
        if (g_prof.frames < g_prof.max_frames && g_prof.seen % g_prof.stride == 0) g_prof.frames++;
        g_prof.seen++;
    }
    return check_launch("gsr_forward/blend", debug, st);
}

}  // namespace gsr
