/* TEST INFRASTRUCTURE — CPU oracle, not product code.
 *
 * Plain-C restatement of the reference 3D-Gaussian-splatting rasterizer hot path
 * (haoyuhsu/autovfx, sugar/gaussian_splatting/submodules/diff-gaussian-rasterization = "DGR/",
 * .../simple-knn = "KNN/").  Each function cites the reference file:line it follows.  The
 * product path (autovfx_b200/csrc) never links or calls this file; only tests/, bench.py's
 * cpu_baseline / reference legs and __graft_entry__.smoke() do.
 *
 * Parity pinning: the reference ships no golden vectors (SURVEY §4), so this restatement is
 * pinned against outputs of the reference's own CUDA code (oracle/_ref/libref_dgr.so) run on a
 * GPU and committed under tests/golden/ (tests/golden/make_golden.py).  Arithmetic is fp32
 * without FMA contraction (-ffp-contract=off); the GPU reference contracts to FMA, so float
 * outputs agree to ~1e-6 relative, not bitwise.
 *
 * Stages are exposed separately (preprocess -> binning -> render, and the two backward stages)
 * with caller-owned buffers, mirroring the reference's GeometryState / BinningState / ImageState
 * (DGR/cuda_rasterizer/rasterizer_impl.h:30-63).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>

#define TILE 16 /* DGR/cuda_rasterizer/config.h:16-17 */

/* DGR/cuda_rasterizer/auxiliary.h:22-39 */
static const float SH_C0 = 0.28209479177387814f;
static const float SH_C1 = 0.4886025119029199f;
static const float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                               -1.0925484305920792f, 0.5462742152960396f};
static const float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                               0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                               -0.5900435899266435f};

static inline float fminf_(float a, float b) { return a < b ? a : b; }
static inline float fmaxf_(float a, float b) { return a > b ? a : b; }
static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int imax(int a, int b) { return a > b ? a : b; }

/* auxiliary.h:58-77 — row-vector times the row-major torch buffer. */
static inline void xform4x3(const float* p, const float* m, float* o) {
    o[0] = m[0] * p[0] + m[4] * p[1] + m[8] * p[2] + m[12];
    o[1] = m[1] * p[0] + m[5] * p[1] + m[9] * p[2] + m[13];
    o[2] = m[2] * p[0] + m[6] * p[1] + m[10] * p[2] + m[14];
}
static inline void xform4x4(const float* p, const float* m, float* o) {
    o[0] = m[0] * p[0] + m[4] * p[1] + m[8] * p[2] + m[12];
    o[1] = m[1] * p[0] + m[5] * p[1] + m[9] * p[2] + m[13];
    o[2] = m[2] * p[0] + m[6] * p[1] + m[10] * p[2] + m[14];
    o[3] = m[3] * p[0] + m[7] * p[1] + m[11] * p[2] + m[15];
}

/* auxiliary.h:41-44: the literals are double, so the expression is evaluated in double. */
static inline float ndc2pix(float v, int S) { return (float)(((v + 1.0) * S - 1.0) * 0.5); }

/* auxiliary.h:46-56 */
static inline void get_rect(float px, float py, int r, int gx, int gy, int* x0, int* y0, int* x1, int* y1) {
    *x0 = imin(gx, imax(0, (int)((px - r) / TILE)));
    *y0 = imin(gy, imax(0, (int)((py - r) / TILE)));
    *x1 = imin(gx, imax(0, (int)((px + r + TILE - 1) / TILE)));
    *y1 = imin(gy, imax(0, (int)((py + r + TILE - 1) / TILE)));
}

/* 3x3 column-major helpers with GLM's summation order (third_party/glm/glm/detail/type_mat3x3.inl:486-519):
 * R[c][r] = A[0][r]*B[c][0] + A[1][r]*B[c][1] + A[2][r]*B[c][2], left to right. */
typedef struct { float m[3][3]; } mat3; /* m[col][row] */
static inline mat3 mat3_mul(mat3 A, mat3 B) {
    mat3 R;
    for (int c = 0; c < 3; c++)
        for (int r = 0; r < 3; r++)
            R.m[c][r] = A.m[0][r] * B.m[c][0] + A.m[1][r] * B.m[c][1] + A.m[2][r] * B.m[c][2];
    return R;
}
static inline mat3 mat3_t(mat3 A) {
    mat3 R;
    for (int c = 0; c < 3; c++)
        for (int r = 0; r < 3; r++) R.m[c][r] = A.m[r][c];
    return R;
}

/* forward.cu:118-152 — quaternion (r,x,y,z) NOT normalised here (line 127 commented out). */
static void cov3d_from_scale_rot(const float* s, float mod, const float* q, float* cov3D) {
    mat3 S;
    memset(&S, 0, sizeof S);
    S.m[0][0] = mod * s[0];
    S.m[1][1] = mod * s[1];
    S.m[2][2] = mod * s[2];
    float r = q[0], x = q[1], y = q[2], z = q[3];
    mat3 R = {{{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
               {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
               {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}}};
    mat3 M = mat3_mul(S, R);
    mat3 Sigma = mat3_mul(mat3_t(M), M);
    cov3D[0] = Sigma.m[0][0];
    cov3D[1] = Sigma.m[0][1];
    cov3D[2] = Sigma.m[0][2];
    cov3D[3] = Sigma.m[1][1];
    cov3D[4] = Sigma.m[1][2];
    cov3D[5] = Sigma.m[2][2];
}

/* Shared by forward.cu:74-113 and backward.cu:160-196: builds T = W*J and cov2D (before the +0.3). */
static void cov2d_parts(const float* mean, float fx, float fy, float tanx, float tany, const float* cov3D,
                        const float* view, float* t_out, float* txtz_tytz, mat3* T_out, mat3* Vrk_out,
                        mat3* cov_out) {
    float t[3];
    xform4x3(mean, view, t);
    const float limx = 1.3f * tanx, limy = 1.3f * tany;
    const float txtz = t[0] / t[2], tytz = t[1] / t[2];
    t[0] = fminf_(limx, fmaxf_(-limx, txtz)) * t[2];
    t[1] = fminf_(limy, fmaxf_(-limy, tytz)) * t[2];
    mat3 J = {{{fx / t[2], 0.f, -(fx * t[0]) / (t[2] * t[2])}, {0.f, fy / t[2], -(fy * t[1]) / (t[2] * t[2])}, {0.f, 0.f, 0.f}}};
    mat3 W = {{{view[0], view[4], view[8]}, {view[1], view[5], view[9]}, {view[2], view[6], view[10]}}};
    mat3 T = mat3_mul(W, J);
    mat3 Vrk = {{{cov3D[0], cov3D[1], cov3D[2]}, {cov3D[1], cov3D[3], cov3D[4]}, {cov3D[2], cov3D[4], cov3D[5]}}};
    mat3 cov = mat3_mul(mat3_mul(mat3_t(T), mat3_t(Vrk)), T);
    if (t_out) { t_out[0] = t[0]; t_out[1] = t[1]; t_out[2] = t[2]; }
    if (txtz_tytz) { txtz_tytz[0] = txtz; txtz_tytz[1] = tytz; }
    if (T_out) *T_out = T;
    if (Vrk_out) *Vrk_out = Vrk;
    *cov_out = cov;
}

/* forward.cu:20-71 */
static void sh_to_rgb(int deg, int M, const float* pos, const float* campos, const float* sh /* [M][3] */,
                      float* rgb, unsigned char* clamped) {
    float d[3] = {pos[0] - campos[0], pos[1] - campos[1], pos[2] - campos[2]};
    float len = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    float x = d[0] / len, y = d[1] / len, z = d[2] / len;
    (void)M;
    for (int c = 0; c < 3; c++) {
#define SH(k) sh[(k)*3 + c]
        float res = SH_C0 * SH(0);
        if (deg > 0) {
            res = res - SH_C1 * y * SH(1) + SH_C1 * z * SH(2) - SH_C1 * x * SH(3);
            if (deg > 1) {
                float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                res = res + SH_C2[0] * xy * SH(4) + SH_C2[1] * yz * SH(5) + SH_C2[2] * (2.0f * zz - xx - yy) * SH(6) +
                      SH_C2[3] * xz * SH(7) + SH_C2[4] * (xx - yy) * SH(8);
                if (deg > 2) {
                    res = res + SH_C3[0] * y * (3.0f * xx - yy) * SH(9) + SH_C3[1] * xy * z * SH(10) +
                          SH_C3[2] * y * (4.0f * zz - xx - yy) * SH(11) +
                          SH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * SH(12) +
                          SH_C3[4] * x * (4.0f * zz - xx - yy) * SH(13) + SH_C3[5] * z * (xx - yy) * SH(14) +
                          SH_C3[6] * x * (xx - 3.0f * yy) * SH(15);
                }
            }
        }
#undef SH
        res += 0.5f;
        clamped[c] = (res < 0);
        rgb[c] = fmaxf_(res, 0.0f);
    }
}

/* FORWARD preprocess — forward.cu:155-256 (+ in_frustum auxiliary.h:139-164).
 * Null pointer == absent input.  Outputs are caller-allocated; rows of culled Gaussians keep radii = 0,
 * tiles_touched = 0 and are otherwise left untouched (the reference leaves them uninitialised).
 * Returns sum(tiles_touched) = num_rendered, or -1 if `prefiltered` and a point is culled (the
 * reference __trap()s, auxiliary.h:156-160). */
int64_t gsro_preprocess(int P, int D, int M, const float* means3D, const float* scales, float scale_modifier,
                        const float* rotations, const float* opacities, const float* shs,
                        const float* cov3D_precomp, const float* colors_precomp, const float* view,
                        const float* proj, const float* campos, int W, int H, float tanfovx, float tanfovy,
                        int prefiltered, int* radii, float* means2D, float* depths, float* cov3Ds, float* rgb,
                        float* conic_opacity, unsigned char* clamped, uint32_t* tiles_touched) {
    const float focal_y = H / (2.0f * tanfovy); /* rasterizer_impl.cu:223-224 */
    const float focal_x = W / (2.0f * tanfovx);
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    int64_t total = 0;
    int trapped = 0;
#pragma omp parallel for schedule(static) reduction(+ : total) reduction(| : trapped)
    for (int i = 0; i < P; i++) {
        radii[i] = 0;
        tiles_touched[i] = 0;
        const float* p = means3D + 3 * (size_t)i;
        float pv[3], ph[4];
        xform4x4(p, proj, ph);
        xform4x3(p, view, pv);
        if (pv[2] <= 0.2f) { /* auxiliary.h:154 — near cull only */
            if (prefiltered) trapped |= 1;
            continue;
        }
        float pw = 1.0f / (ph[3] + 0.0000001f);
        float pproj[2] = {ph[0] * pw, ph[1] * pw};
        const float* cov3D;
        if (cov3D_precomp) cov3D = cov3D_precomp + 6 * (size_t)i;
        else {
            cov3d_from_scale_rot(scales + 3 * (size_t)i, scale_modifier, rotations + 4 * (size_t)i, cov3Ds + 6 * (size_t)i);
            cov3D = cov3Ds + 6 * (size_t)i;
        }
        mat3 cov;
        cov2d_parts(p, focal_x, focal_y, tanfovx, tanfovy, cov3D, view, NULL, NULL, NULL, NULL, &cov);
        float cx = cov.m[0][0] + 0.3f, cy = cov.m[0][1], cz = cov.m[1][1] + 0.3f; /* forward.cu:110-112 */
        float det = cx * cz - cy * cy;
        if (det == 0.0f) continue;
        float det_inv = 1.f / det;
        float conic[3] = {cz * det_inv, -cy * det_inv, cx * det_inv};
        float mid = 0.5f * (cx + cz);
        float lambda1 = mid + sqrtf(fmaxf_(0.1f, mid * mid - det));
        float lambda2 = mid - sqrtf(fmaxf_(0.1f, mid * mid - det));
        float my_radius = ceilf(3.f * sqrtf(fmaxf_(lambda1, lambda2)));
        float pix[2] = {ndc2pix(pproj[0], W), ndc2pix(pproj[1], H)};
        int x0, y0, x1, y1;
        get_rect(pix[0], pix[1], (int)my_radius, gx, gy, &x0, &y0, &x1, &y1);
        if ((x1 - x0) * (y1 - y0) == 0) continue;
        if (!colors_precomp) sh_to_rgb(D, M, p, campos, shs + (size_t)i * M * 3, rgb + 3 * (size_t)i, clamped + 3 * (size_t)i);
        depths[i] = pv[2];
        radii[i] = (int)my_radius;
        means2D[2 * (size_t)i] = pix[0];
        means2D[2 * (size_t)i + 1] = pix[1];
        float* co = conic_opacity + 4 * (size_t)i;
        co[0] = conic[0]; co[1] = conic[1]; co[2] = conic[2]; co[3] = opacities[i];
        tiles_touched[i] = (uint32_t)((y1 - y0) * (x1 - x0));
        total += tiles_touched[i];
    }
    return trapped ? -1 : total;
}

/* rasterizer_impl.cu:35-50 */
static uint32_t higher_msb(uint32_t n) {
    uint32_t msb = sizeof(n) * 4, step = msb;
    while (step > 1) {
        step /= 2;
        if (n >> msb) msb += step; else msb -= step;
    }
    if (n >> msb) msb++;
    return msb;
}

/* BINNING — InclusiveSum (rasterizer_impl.cu:278), duplicateWithKeys (:70-111), stable LSD radix sort on
 * the low 32+bit key bits (:301-309), identifyTileRanges (:116-138, after the memset :311).
 * keys/point_list have R entries, ranges has 2*tiles entries. */
int gsro_binning(int P, int W, int H, const float* means2D, const float* depths, const int* radii,
                 const uint32_t* tiles_touched, int64_t R, uint64_t* keys, uint32_t* point_list,
                 uint32_t* ranges) {
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    memset(ranges, 0, sizeof(uint32_t) * 2 * (size_t)gx * gy);
    if (R == 0) return 0;
    uint64_t* k0 = (uint64_t*)malloc(sizeof(uint64_t) * R);
    uint32_t* v0 = (uint32_t*)malloc(sizeof(uint32_t) * R);
    uint64_t* k1 = (uint64_t*)malloc(sizeof(uint64_t) * R);
    uint32_t* v1 = (uint32_t*)malloc(sizeof(uint32_t) * R);
    if (!k0 || !v0 || !k1 || !v1) return -1;
    int64_t off = 0;
    for (int i = 0; i < P; i++) {
        if (radii[i] > 0) {
            int x0, y0, x1, y1;
            get_rect(means2D[2 * (size_t)i], means2D[2 * (size_t)i + 1], radii[i], gx, gy, &x0, &y0, &x1, &y1);
            uint32_t dbits;
            memcpy(&dbits, &depths[i], 4);
            for (int y = y0; y < y1; y++)
                for (int x = x0; x < x1; x++) {
                    uint64_t key = (uint64_t)(y * gx + x);
                    key <<= 32;
                    key |= dbits;
                    k0[off] = key;
                    v0[off] = (uint32_t)i;
                    off++;
                }
            (void)tiles_touched;
        }
    }
    if (off != R) { free(k0); free(v0); free(k1); free(v1); return -2; }
    const int end_bit = 32 + (int)higher_msb((uint32_t)(gx * gy));
    /* stable LSD radix sort, 11-bit digits, only bits [0,end_bit) take part (like CUB begin/end bit) */
    uint64_t mask = end_bit >= 64 ? ~0ull : ((1ull << end_bit) - 1);
    const int RB = 11;
    size_t* cnt = (size_t*)malloc(sizeof(size_t) * ((size_t)1 << RB));
    for (int shift = 0; shift < end_bit; shift += RB) {
        memset(cnt, 0, sizeof(size_t) * ((size_t)1 << RB));
        for (int64_t j = 0; j < R; j++) cnt[((k0[j] & mask) >> shift) & ((1u << RB) - 1)]++;
        size_t sum = 0;
        for (size_t d = 0; d < ((size_t)1 << RB); d++) { size_t c = cnt[d]; cnt[d] = sum; sum += c; }
        for (int64_t j = 0; j < R; j++) {
            size_t d = ((k0[j] & mask) >> shift) & ((1u << RB) - 1);
            k1[cnt[d]] = k0[j];
            v1[cnt[d]] = v0[j];
            cnt[d]++;
        }
        uint64_t* tk = k0; k0 = k1; k1 = tk;
        uint32_t* tv = v0; v0 = v1; v1 = tv;
    }
    memcpy(keys, k0, sizeof(uint64_t) * R);
    memcpy(point_list, v0, sizeof(uint32_t) * R);
    for (int64_t j = 0; j < R; j++) {
        uint32_t cur = (uint32_t)(keys[j] >> 32);
        if (j == 0) ranges[2 * cur] = 0;
        else {
            uint32_t prev = (uint32_t)(keys[j - 1] >> 32);
            if (cur != prev) { ranges[2 * prev + 1] = (uint32_t)j; ranges[2 * cur] = (uint32_t)j; }
        }
        if (j == R - 1) ranges[2 * cur + 1] = (uint32_t)R;
    }
    free(cnt); free(k0); free(v0); free(k1); free(v1);
    return 0;
}

/* FORWARD blend — forward.cu:261-378.  One pixel at a time; the per-pixel arithmetic order is the
 * reference's.  features = geom rgb or colors_precomp ([P,3]). */
void gsro_render(int W, int H, const uint32_t* ranges, const uint32_t* point_list, const float* means2D,
                 const float* features, const float* depths, const float* conic_opacity, const float* bg,
                 float* out_color, float* out_depth, float* out_alpha, uint32_t* n_contrib) {
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
#pragma omp parallel for schedule(dynamic, 4)
    for (int tile = 0; tile < gx * gy; tile++) {
        const int ty = tile / gx, tx = tile % gx;
        const uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
        for (int py = ty * TILE; py < imin(ty * TILE + TILE, H); py++)
            for (int px = tx * TILE; px < imin(tx * TILE + TILE, W); px++) {
                const float pxf = (float)px, pyf = (float)py;
                float T = 1.0f, C[3] = {0, 0, 0}, Dp = 0;
                uint32_t contributor = 0, last = 0;
                for (uint32_t j = r0; j < r1; j++) {
                    contributor++;
                    const uint32_t g = point_list[j];
                    const float dx = means2D[2 * (size_t)g] - pxf, dy = means2D[2 * (size_t)g + 1] - pyf;
                    const float* co = conic_opacity + 4 * (size_t)g;
                    const float power = -0.5f * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
                    if (power > 0.0f) continue;
                    const float alpha = fminf_(0.99f, co[3] * expf(power));
                    if (alpha < 1.0f / 255.0f) continue;
                    const float test_T = T * (1 - alpha);
                    if (test_T < 0.0001f) break; /* done = true; nothing after this is applied */
                    for (int ch = 0; ch < 3; ch++) C[ch] += features[3 * (size_t)g + ch] * alpha * T;
                    Dp += depths[g] * alpha * T;
                    T = test_T;
                    last = contributor;
                }
                const size_t pid = (size_t)W * py + px;
                out_alpha[pid] = 1 - T;
                n_contrib[pid] = last;
                for (int ch = 0; ch < 3; ch++) out_color[(size_t)ch * H * W + pid] = C[ch] + T * bg[ch];
                out_depth[pid] = Dp;
            }
    }
}

static inline void atomic_addf(float* p, float v) {
#pragma omp atomic
    *p += v;
}

/* BACKWARD blend — backward.cu:415-599.  Accumulates into zero-initialised dL_dmean2D[P*3] (x,y used),
 * dL_dconic[P*4] (slots 0,1,3), dL_dopacity[P], dL_dcolors[P*3], dL_ddepths[P]. */
void gsro_render_backward(int W, int H, const uint32_t* ranges, const uint32_t* point_list, const float* bg,
                          const float* means2D, const float* conic_opacity, const float* colors,
                          const float* depths, const float* accum_alphas, const uint32_t* n_contrib,
                          const float* dL_dpixels, const float* dL_dpixel_depths, const float* dL_dpixel_alphas,
                          float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolors,
                          float* dL_ddepths) {
    const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
    const float ddelx_dx = (float)(0.5 * W), ddely_dy = (float)(0.5 * H); /* backward.cu:488-489 */
#pragma omp parallel for schedule(dynamic, 4)
    for (int tile = 0; tile < gx * gy; tile++) {
        const int ty = tile / gx, tx = tile % gx;
        const uint32_t r0 = ranges[2 * tile], r1 = ranges[2 * tile + 1];
        for (int py = ty * TILE; py < imin(ty * TILE + TILE, H); py++)
            for (int px = tx * TILE; px < imin(tx * TILE + TILE, W); px++) {
                const size_t pid = (size_t)W * py + px;
                const float pxf = (float)px, pyf = (float)py;
                const float T_final = 1 - accum_alphas[pid];
                float T = T_final;
                const uint32_t last_contributor = n_contrib[pid];
                float accum_rec[3] = {0, 0, 0}, accum_red = 0, accum_rea = 0;
                float dLp[3] = {dL_dpixels[pid], dL_dpixels[(size_t)H * W + pid], dL_dpixels[2 * (size_t)H * W + pid]};
                const float dLd = dL_dpixel_depths[pid], dLa = dL_dpixel_alphas[pid];
                float last_alpha = 0, last_color[3] = {0, 0, 0}, last_depth = 0;
                /* back to front: entry k (1-based position in the tile list) from last_contributor down to 1 */
                for (uint32_t k = imin((int)last_contributor, (int)(r1 - r0)); k >= 1; k--) {
                    const uint32_t g = point_list[r0 + k - 1];
                    const float dx = means2D[2 * (size_t)g] - pxf, dy = means2D[2 * (size_t)g + 1] - pyf;
                    const float* co = conic_opacity + 4 * (size_t)g;
                    const float power = -0.5f * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
                    if (power > 0.0f) continue;
                    const float G = expf(power);
                    const float alpha = fminf_(0.99f, co[3] * G);
                    if (alpha < 1.0f / 255.0f) continue;
                    T = T / (1.f - alpha);
                    const float dchannel_dcolor = alpha * T;
                    float dL_dalpha = 0.0f;
                    for (int ch = 0; ch < 3; ch++) {
                        const float c = colors[3 * (size_t)g + ch];
                        accum_rec[ch] = last_alpha * last_color[ch] + (1.f - last_alpha) * accum_rec[ch];
                        last_color[ch] = c;
                        dL_dalpha += (c - accum_rec[ch]) * dLp[ch];
                        atomic_addf(&dL_dcolors[3 * (size_t)g + ch], dchannel_dcolor * dLp[ch]);
                    }
                    const float dep = depths[g];
                    accum_red = last_alpha * last_depth + (1.f - last_alpha) * accum_red;
                    last_depth = dep;
                    dL_dalpha += (dep - accum_red) * dLd;
                    atomic_addf(&dL_ddepths[g], dchannel_dcolor * dLd);
                    accum_rea = last_alpha + (1.f - last_alpha) * accum_rea;
                    dL_dalpha += (1 - accum_rea) * dLa;
                    dL_dalpha *= T;
                    last_alpha = alpha;
                    float bg_dot = 0;
                    for (int ch = 0; ch < 3; ch++) bg_dot += bg[ch] * dLp[ch];
                    dL_dalpha += (-T_final / (1.f - alpha)) * bg_dot;
                    const float dL_dG = co[3] * dL_dalpha;
                    const float gdx = G * dx, gdy = G * dy;
                    const float dG_ddelx = -gdx * co[0] - gdy * co[1];
                    const float dG_ddely = -gdy * co[2] - gdx * co[1];
                    atomic_addf(&dL_dmean2D[3 * (size_t)g + 0], dL_dG * dG_ddelx * ddelx_dx);
                    atomic_addf(&dL_dmean2D[3 * (size_t)g + 1], dL_dG * dG_ddely * ddely_dy);
                    atomic_addf(&dL_dconic[4 * (size_t)g + 0], -0.5f * gdx * dx * dL_dG);
                    atomic_addf(&dL_dconic[4 * (size_t)g + 1], -0.5f * gdx * dy * dL_dG);
                    atomic_addf(&dL_dconic[4 * (size_t)g + 3], -0.5f * gdy * dy * dL_dG);
                    atomic_addf(&dL_dopacity[g], G * dL_dalpha);
                }
            }
    }
}

/* auxiliary.h:106-118 */
static void dnormvdv3(const float* v, const float* dv, float* o) {
    float sum2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
    float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
    o[0] = ((+sum2 - v[0] * v[0]) * dv[0] - v[1] * v[0] * dv[1] - v[2] * v[0] * dv[2]) * invsum32;
    o[1] = (-v[0] * v[1] * dv[0] + (sum2 - v[1] * v[1]) * dv[1] - v[2] * v[1] * dv[2]) * invsum32;
    o[2] = (-v[0] * v[2] * dv[0] - v[1] * v[2] * dv[1] + (sum2 - v[2] * v[2]) * dv[2]) * invsum32;
}

/* backward.cu:20-139 */
static void sh_backward(int deg, int M, const float* pos, const float* campos, const float* sh,
                        const unsigned char* clamped, const float* dL_dcolor, float* dL_dmean, float* dL_dsh) {
    float dorig[3] = {pos[0] - campos[0], pos[1] - campos[1], pos[2] - campos[2]};
    float len = sqrtf(dorig[0] * dorig[0] + dorig[1] * dorig[1] + dorig[2] * dorig[2]);
    float x = dorig[0] / len, y = dorig[1] / len, z = dorig[2] / len;
    float dRGB[3];
    for (int c = 0; c < 3; c++) dRGB[c] = dL_dcolor[c] * (clamped[c] ? 0.f : 1.f);
    float dRGBdx[3] = {0, 0, 0}, dRGBdy[3] = {0, 0, 0}, dRGBdz[3] = {0, 0, 0};
    (void)M;
#define SHV(k, c) sh[(k)*3 + (c)]
#define DSH(k, w) for (int c = 0; c < 3; c++) dL_dsh[(k)*3 + c] = (w) * dRGB[c]
    DSH(0, SH_C0);
    if (deg > 0) {
        DSH(1, -SH_C1 * y);
        DSH(2, SH_C1 * z);
        DSH(3, -SH_C1 * x);
        for (int c = 0; c < 3; c++) {
            dRGBdx[c] = -SH_C1 * SHV(3, c);
            dRGBdy[c] = -SH_C1 * SHV(1, c);
            dRGBdz[c] = SH_C1 * SHV(2, c);
        }
        if (deg > 1) {
            float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            DSH(4, SH_C2[0] * xy);
            DSH(5, SH_C2[1] * yz);
            DSH(6, SH_C2[2] * (2.f * zz - xx - yy));
            DSH(7, SH_C2[3] * xz);
            DSH(8, SH_C2[4] * (xx - yy));
            for (int c = 0; c < 3; c++) {
                dRGBdx[c] += SH_C2[0] * y * SHV(4, c) + SH_C2[2] * 2.f * -x * SHV(6, c) + SH_C2[3] * z * SHV(7, c) + SH_C2[4] * 2.f * x * SHV(8, c);
                dRGBdy[c] += SH_C2[0] * x * SHV(4, c) + SH_C2[1] * z * SHV(5, c) + SH_C2[2] * 2.f * -y * SHV(6, c) + SH_C2[4] * 2.f * -y * SHV(8, c);
                dRGBdz[c] += SH_C2[1] * y * SHV(5, c) + SH_C2[2] * 2.f * 2.f * z * SHV(6, c) + SH_C2[3] * x * SHV(7, c);
            }
            if (deg > 2) {
                DSH(9, SH_C3[0] * y * (3.f * xx - yy));
                DSH(10, SH_C3[1] * xy * z);
                DSH(11, SH_C3[2] * y * (4.f * zz - xx - yy));
                DSH(12, SH_C3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy));
                DSH(13, SH_C3[4] * x * (4.f * zz - xx - yy));
                DSH(14, SH_C3[5] * z * (xx - yy));
                DSH(15, SH_C3[6] * x * (xx - 3.f * yy));
                for (int c = 0; c < 3; c++) {
                    dRGBdx[c] += (SH_C3[0] * SHV(9, c) * 3.f * 2.f * xy + SH_C3[1] * SHV(10, c) * yz + SH_C3[2] * SHV(11, c) * -2.f * xy +
                                  SH_C3[3] * SHV(12, c) * -3.f * 2.f * xz + SH_C3[4] * SHV(13, c) * (-3.f * xx + 4.f * zz - yy) +
                                  SH_C3[5] * SHV(14, c) * 2.f * xz + SH_C3[6] * SHV(15, c) * 3.f * (xx - yy));
                    dRGBdy[c] += (SH_C3[0] * SHV(9, c) * 3.f * (xx - yy) + SH_C3[1] * SHV(10, c) * xz +
                                  SH_C3[2] * SHV(11, c) * (-3.f * yy + 4.f * zz - xx) + SH_C3[3] * SHV(12, c) * -3.f * 2.f * yz +
                                  SH_C3[4] * SHV(13, c) * -2.f * xy + SH_C3[5] * SHV(14, c) * -2.f * yz +
                                  SH_C3[6] * SHV(15, c) * -3.f * 2.f * xy);
                    dRGBdz[c] += (SH_C3[1] * SHV(10, c) * xy + SH_C3[2] * SHV(11, c) * 4.f * 2.f * yz +
                                  SH_C3[3] * SHV(12, c) * 3.f * (2.f * zz - xx - yy) + SH_C3[4] * SHV(13, c) * 4.f * 2.f * xz +
                                  SH_C3[5] * SHV(14, c) * (xx - yy));
                }
            }
        }
    }
#undef SHV
#undef DSH
    float ddir[3] = {dRGBdx[0] * dRGB[0] + dRGBdx[1] * dRGB[1] + dRGBdx[2] * dRGB[2],
                     dRGBdy[0] * dRGB[0] + dRGBdy[1] * dRGB[1] + dRGBdy[2] * dRGB[2],
                     dRGBdz[0] * dRGB[0] + dRGBdz[1] * dRGB[1] + dRGBdz[2] * dRGB[2]};
    float dm[3];
    dnormvdv3(dorig, ddir, dm);
    dL_dmean[0] += dm[0];
    dL_dmean[1] += dm[1];
    dL_dmean[2] += dm[2];
}

/* backward.cu:278-341 (no quaternion-normalisation backward: line 340 comment) */
static void cov3d_backward(const float* s_in, float mod, const float* q, const float* dcov, float* dscale, float* drot) {
    float r = q[0], x = q[1], y = q[2], z = q[3];
    mat3 R = {{{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
               {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
               {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}}};
    mat3 S;
    memset(&S, 0, sizeof S);
    float s[3] = {mod * s_in[0], mod * s_in[1], mod * s_in[2]};
    S.m[0][0] = s[0]; S.m[1][1] = s[1]; S.m[2][2] = s[2];
    mat3 M = mat3_mul(S, R);
    mat3 dSigma = {{{dcov[0], 0.5f * dcov[1], 0.5f * dcov[2]}, {0.5f * dcov[1], dcov[3], 0.5f * dcov[4]}, {0.5f * dcov[2], 0.5f * dcov[4], dcov[5]}}};
    mat3 M2;
    for (int c = 0; c < 3; c++) for (int rr = 0; rr < 3; rr++) M2.m[c][rr] = 2.0f * M.m[c][rr]; /* 2.0f * M */
    mat3 dM = mat3_mul(M2, dSigma);
    mat3 Rt = mat3_t(R), dMt = mat3_t(dM);
    for (int k = 0; k < 3; k++) /* glm::dot: x*x' + y*y' + z*z' */
        dscale[k] = Rt.m[k][0] * dMt.m[k][0] + Rt.m[k][1] * dMt.m[k][1] + Rt.m[k][2] * dMt.m[k][2];
    for (int k = 0; k < 3; k++) for (int rr = 0; rr < 3; rr++) dMt.m[k][rr] *= s[k];
#define D(c, rr) dMt.m[c][rr]
    drot[0] = 2 * z * (D(0, 1) - D(1, 0)) + 2 * y * (D(2, 0) - D(0, 2)) + 2 * x * (D(1, 2) - D(2, 1));
    drot[1] = 2 * y * (D(1, 0) + D(0, 1)) + 2 * z * (D(2, 0) + D(0, 2)) + 2 * r * (D(1, 2) - D(2, 1)) - 4 * x * (D(2, 2) + D(1, 1));
    drot[2] = 2 * x * (D(1, 0) + D(0, 1)) + 2 * r * (D(2, 0) - D(0, 2)) + 2 * z * (D(1, 2) + D(2, 1)) - 4 * y * (D(2, 2) + D(0, 0));
    drot[3] = 2 * r * (D(0, 1) - D(1, 0)) + 2 * x * (D(2, 0) + D(0, 2)) + 2 * y * (D(1, 2) + D(2, 1)) - 4 * z * (D(1, 1) + D(0, 0));
#undef D
}

/* BACKWARD preprocess — computeCov2DCUDA (backward.cu:144-274) followed by preprocessCUDA (:346-412).
 * cov3Ds = cov3D_precomp if given else the forward's geom cov3D.  dL_dmean2D[P*3], dL_dconic[P*4],
 * dL_dcolor[P*3], dL_ddepth[P] are inputs (from the blend backward); dL_dmeans3D[P*3], dL_dcov3D[P*6],
 * dL_dsh[P*M*3], dL_dscale[P*3], dL_drot[P*4] are zero-initialised outputs. */
void gsro_preprocess_backward(int P, int D, int M, const float* means3D, const int* radii, const float* shs,
                              const unsigned char* clamped, const float* scales, const float* rotations,
                              float scale_modifier, const float* cov3Ds, const float* view, const float* proj,
                              int W, int H, float tanfovx, float tanfovy, const float* campos,
                              const float* dL_dmean2D, const float* dL_dconic, float* dL_dmeans3D,
                              const float* dL_dcolor, const float* dL_ddepth, float* dL_dcov3D, float* dL_dsh,
                              float* dL_dscale, float* dL_drot) {
    const float h_y = H / (2.0f * tanfovy), h_x = W / (2.0f * tanfovx);
#pragma omp parallel for schedule(static)
    for (int i = 0; i < P; i++) {
        if (!(radii[i] > 0)) continue;
        const float* mean = means3D + 3 * (size_t)i;
        /* ---- computeCov2DCUDA ---- */
        {
            const float* cov3D = cov3Ds + 6 * (size_t)i;
            float dcon[3] = {dL_dconic[4 * (size_t)i], dL_dconic[4 * (size_t)i + 1], dL_dconic[4 * (size_t)i + 3]};
            float t[3], tt[2];
            mat3 T, Vrk, cov2D;
            cov2d_parts(mean, h_x, h_y, tanfovx, tanfovy, cov3D, view, t, tt, &T, &Vrk, &cov2D);
            const float limx = 1.3f * tanfovx, limy = 1.3f * tanfovy;
            const float x_grad_mul = (tt[0] < -limx || tt[0] > limx) ? 0.f : 1.f;
            const float y_grad_mul = (tt[1] < -limy || tt[1] > limy) ? 0.f : 1.f;
            mat3 Wm = {{{view[0], view[4], view[8]}, {view[1], view[5], view[9]}, {view[2], view[6], view[10]}}};
            float a = cov2D.m[0][0] + 0.3f, b = cov2D.m[0][1], c = cov2D.m[1][1] + 0.3f;
            float denom = a * c - b * b;
            float dL_da = 0, dL_db = 0, dL_dc = 0;
            float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
            float* dcov = dL_dcov3D + 6 * (size_t)i;
            if (denom2inv != 0) {
                dL_da = denom2inv * (-c * c * dcon[0] + 2 * b * c * dcon[1] + (denom - a * c) * dcon[2]);
                dL_dc = denom2inv * (-a * a * dcon[2] + 2 * a * b * dcon[1] + (denom - a * c) * dcon[0]);
                dL_db = denom2inv * 2 * (b * c * dcon[0] - (denom + 2 * b * b) * dcon[1] + a * b * dcon[2]);
#define TT(c_, r_) T.m[c_][r_]
                dcov[0] = (TT(0, 0) * TT(0, 0) * dL_da + TT(0, 0) * TT(1, 0) * dL_db + TT(1, 0) * TT(1, 0) * dL_dc);
                dcov[3] = (TT(0, 1) * TT(0, 1) * dL_da + TT(0, 1) * TT(1, 1) * dL_db + TT(1, 1) * TT(1, 1) * dL_dc);
                dcov[5] = (TT(0, 2) * TT(0, 2) * dL_da + TT(0, 2) * TT(1, 2) * dL_db + TT(1, 2) * TT(1, 2) * dL_dc);
                dcov[1] = 2 * TT(0, 0) * TT(0, 1) * dL_da + (TT(0, 0) * TT(1, 1) + TT(0, 1) * TT(1, 0)) * dL_db + 2 * TT(1, 0) * TT(1, 1) * dL_dc;
                dcov[2] = 2 * TT(0, 0) * TT(0, 2) * dL_da + (TT(0, 0) * TT(1, 2) + TT(0, 2) * TT(1, 0)) * dL_db + 2 * TT(1, 0) * TT(1, 2) * dL_dc;
                dcov[4] = 2 * TT(0, 2) * TT(0, 1) * dL_da + (TT(0, 1) * TT(1, 2) + TT(0, 2) * TT(1, 1)) * dL_db + 2 * TT(1, 1) * TT(1, 2) * dL_dc;
            } else {
                for (int k = 0; k < 6; k++) dcov[k] = 0;
            }
#define VV(c_, r_) Vrk.m[c_][r_]
            float dT00 = 2 * (TT(0, 0) * VV(0, 0) + TT(0, 1) * VV(0, 1) + TT(0, 2) * VV(0, 2)) * dL_da + (TT(1, 0) * VV(0, 0) + TT(1, 1) * VV(0, 1) + TT(1, 2) * VV(0, 2)) * dL_db;
            float dT01 = 2 * (TT(0, 0) * VV(1, 0) + TT(0, 1) * VV(1, 1) + TT(0, 2) * VV(1, 2)) * dL_da + (TT(1, 0) * VV(1, 0) + TT(1, 1) * VV(1, 1) + TT(1, 2) * VV(1, 2)) * dL_db;
            float dT02 = 2 * (TT(0, 0) * VV(2, 0) + TT(0, 1) * VV(2, 1) + TT(0, 2) * VV(2, 2)) * dL_da + (TT(1, 0) * VV(2, 0) + TT(1, 1) * VV(2, 1) + TT(1, 2) * VV(2, 2)) * dL_db;
            float dT10 = 2 * (TT(1, 0) * VV(0, 0) + TT(1, 1) * VV(0, 1) + TT(1, 2) * VV(0, 2)) * dL_dc + (TT(0, 0) * VV(0, 0) + TT(0, 1) * VV(0, 1) + TT(0, 2) * VV(0, 2)) * dL_db;
            float dT11 = 2 * (TT(1, 0) * VV(1, 0) + TT(1, 1) * VV(1, 1) + TT(1, 2) * VV(1, 2)) * dL_dc + (TT(0, 0) * VV(1, 0) + TT(0, 1) * VV(1, 1) + TT(0, 2) * VV(1, 2)) * dL_db;
            float dT12 = 2 * (TT(1, 0) * VV(2, 0) + TT(1, 1) * VV(2, 1) + TT(1, 2) * VV(2, 2)) * dL_dc + (TT(0, 0) * VV(2, 0) + TT(0, 1) * VV(2, 1) + TT(0, 2) * VV(2, 2)) * dL_db;
#undef TT
#undef VV
            float dJ00 = Wm.m[0][0] * dT00 + Wm.m[0][1] * dT01 + Wm.m[0][2] * dT02;
            float dJ02 = Wm.m[2][0] * dT00 + Wm.m[2][1] * dT01 + Wm.m[2][2] * dT02;
            float dJ11 = Wm.m[1][0] * dT10 + Wm.m[1][1] * dT11 + Wm.m[1][2] * dT12;
            float dJ12 = Wm.m[2][0] * dT10 + Wm.m[2][1] * dT11 + Wm.m[2][2] * dT12;
            float tz = 1.f / t[2], tz2 = tz * tz, tz3 = tz2 * tz;
            float dtx = x_grad_mul * -h_x * tz2 * dJ02;
            float dty = y_grad_mul * -h_y * tz2 * dJ12;
            float dtz = -h_x * tz2 * dJ00 - h_y * tz2 * dJ11 + (2 * h_x * t[0]) * tz3 * dJ02 + (2 * h_y * t[1]) * tz3 * dJ12;
            float* dm = dL_dmeans3D + 3 * (size_t)i; /* transformVec4x3Transpose, auxiliary.h:89-97; plain store (:273) */
            dm[0] = view[0] * dtx + view[1] * dty + view[2] * dtz;
            dm[1] = view[4] * dtx + view[5] * dty + view[6] * dtz;
            dm[2] = view[8] * dtx + view[9] * dty + view[10] * dtz;
        }
        /* ---- preprocessCUDA (backward) ---- */
        {
            const float* m = mean;
            float mh[4];
            xform4x4(m, proj, mh);
            float m_w = 1.0f / (mh[3] + 0.0000001f);
            float mul1 = (proj[0] * m[0] + proj[4] * m[1] + proj[8] * m[2] + proj[12]) * m_w * m_w;
            float mul2 = (proj[1] * m[0] + proj[5] * m[1] + proj[9] * m[2] + proj[13]) * m_w * m_w;
            const float* d2 = dL_dmean2D + 3 * (size_t)i;
            float dmean[3];
            dmean[0] = (proj[0] * m_w - proj[3] * mul1) * d2[0] + (proj[1] * m_w - proj[3] * mul2) * d2[1];
            dmean[1] = (proj[4] * m_w - proj[7] * mul1) * d2[0] + (proj[5] * m_w - proj[7] * mul2) * d2[1];
            dmean[2] = (proj[8] * m_w - proj[11] * mul1) * d2[0] + (proj[9] * m_w - proj[11] * mul2) * d2[1];
            float* dm = dL_dmeans3D + 3 * (size_t)i;
            dm[0] += dmean[0]; dm[1] += dmean[1]; dm[2] += dmean[2];
            float mul3 = view[2] * m[0] + view[6] * m[1] + view[10] * m[2] + view[14];
            float dd = dL_ddepth[i];
            dm[0] += (view[2] - view[3] * mul3) * dd;
            dm[1] += (view[6] - view[7] * mul3) * dd;
            dm[2] += (view[10] - view[11] * mul3) * dd;
            if (shs)
                sh_backward(D, M, m, campos, shs + (size_t)i * M * 3, clamped + 3 * (size_t)i, dL_dcolor + 3 * (size_t)i, dm, dL_dsh + (size_t)i * M * 3);
            if (scales)
                cov3d_backward(scales + 3 * (size_t)i, scale_modifier, rotations + 4 * (size_t)i, dL_dcov3D + 6 * (size_t)i, dL_dscale + 3 * (size_t)i, dL_drot + 4 * (size_t)i);
        }
    }
}

/* checkFrustum — rasterizer_impl.cu:54-66 */
void gsro_mark_visible(int P, const float* means3D, const float* view, const float* proj, unsigned char* present) {
    (void)proj;
#pragma omp parallel for schedule(static)
    for (int i = 0; i < P; i++) {
        float pv[3];
        xform4x3(means3D + 3 * (size_t)i, view, pv);
        present[i] = !(pv[2] <= 0.2f);
    }
}

/* ---------------------------------------------------------------------------------------------------
 * distCUDA2 — KNN/simple_knn.cu:185-220.  The result is the exact mean squared distance to the 3
 * nearest neighbours (the Morton pass only orders points and seeds a conservative bound, SURVEY a17),
 * so this restatement keeps the Morton order + 1024-point boxes + pruning to stay fast, and a brute
 * force variant (gsro_dist2_brute) pins it at small P. */
static uint32_t prep_morton(uint32_t x) { /* simple_knn.cu:46-53 */
    x = (x | (x << 16)) & 0x030000FF;
    x = (x | (x << 8)) & 0x0300F00F;
    x = (x | (x << 4)) & 0x030C30C3;
    x = (x | (x << 2)) & 0x09249249;
    return x;
}
static inline void kbest3(const float* ref, const float* p, float* knn) { /* simple_knn.cu:130-145 */
    float d0 = p[0] - ref[0], d1 = p[1] - ref[1], d2 = p[2] - ref[2];
    float dist = d0 * d0 + d1 * d1 + d2 * d2;
    for (int j = 0; j < 3; j++)
        if (knn[j] > dist) { float t = knn[j]; knn[j] = dist; dist = t; }
}
typedef struct { uint32_t code, idx; } mpair;
static int cmp_mpair(const void* a, const void* b) {
    const mpair *x = (const mpair*)a, *y = (const mpair*)b;
    if (x->code != y->code) return x->code < y->code ? -1 : 1;
    return x->idx < y->idx ? -1 : (x->idx > y->idx);
}
void gsro_dist2(int P, const float* pts, float* out) {
    if (P == 0) return;
    float mn[3] = {0, 0, 0}, mx[3] = {0, 0, 0}; /* init {0,0,0}: bbox always contains the origin (:191) */
    for (int i = 0; i < P; i++)
        for (int k = 0; k < 3; k++) {
            mn[k] = fminf_(mn[k], pts[3 * (size_t)i + k]);
            mx[k] = fmaxf_(mx[k], pts[3 * (size_t)i + k]);
        }
    mpair* mp = (mpair*)malloc(sizeof(mpair) * P);
    for (int i = 0; i < P; i++) { /* coord2Morton :55-61 */
        uint32_t c[3];
        for (int k = 0; k < 3; k++)
            c[k] = prep_morton((uint32_t)(((pts[3 * (size_t)i + k] - mn[k]) / (mx[k] - mn[k])) * ((1 << 10) - 1)));
        mp[i].code = c[0] | (c[1] << 1) | (c[2] << 2);
        mp[i].idx = (uint32_t)i;
    }
    qsort(mp, P, sizeof(mpair), cmp_mpair); /* stable radix sort == sort by (code, original idx) */
    const int BOX = 1024;
    int nb = (P + BOX - 1) / BOX;
    float* boxes = (float*)malloc(sizeof(float) * 6 * nb);
    for (int b = 0; b < nb; b++) { /* boxMinMax :78-117 */
        float lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
        for (int i = b * BOX; i < imin(P, (b + 1) * BOX); i++)
            for (int k = 0; k < 3; k++) {
                float v = pts[3 * (size_t)mp[i].idx + k];
                lo[k] = fminf_(lo[k], v);
                hi[k] = fmaxf_(hi[k], v);
            }
        memcpy(boxes + 6 * b, lo, 12);
        memcpy(boxes + 6 * b + 3, hi, 12);
    }
#pragma omp parallel for schedule(dynamic, 256)
    for (int idx = 0; idx < P; idx++) { /* boxMeanDist :147-183 */
        const float* point = pts + 3 * (size_t)mp[idx].idx;
        float best[3] = {FLT_MAX, FLT_MAX, FLT_MAX};
        for (int i = imax(0, idx - 3); i <= imin(P - 1, idx + 3); i++) {
            if (i == idx) continue;
            kbest3(point, pts + 3 * (size_t)mp[i].idx, best);
        }
        float reject = best[2];
        best[0] = best[1] = best[2] = FLT_MAX;
        for (int b = 0; b < nb; b++) {
            const float* lo = boxes + 6 * b; const float* hi = lo + 3;
            float diff[3] = {0, 0, 0}; /* distBoxPoint :119-128 */
            for (int k = 0; k < 3; k++)
                if (point[k] < lo[k] || point[k] > hi[k]) diff[k] = fminf_(fabsf(point[k] - lo[k]), fabsf(point[k] - hi[k]));
            float dist = diff[0] * diff[0] + diff[1] * diff[1] + diff[2] * diff[2];
            if (dist > reject || dist > best[2]) continue;
            for (int i = b * BOX; i < imin(P, (b + 1) * BOX); i++) {
                if (i == idx) continue;
                kbest3(point, pts + 3 * (size_t)mp[i].idx, best);
            }
        }
        out[mp[idx].idx] = (best[0] + best[1] + best[2]) / 3.0f;
    }
    free(boxes);
    free(mp);
}

/* O(P^2) definition of the same quantity, for pinning gsro_dist2 at small P. */
void gsro_dist2_brute(int P, const float* pts, float* out) {
#pragma omp parallel for schedule(static)
    for (int i = 0; i < P; i++) {
        float best[3] = {FLT_MAX, FLT_MAX, FLT_MAX};
        for (int j = 0; j < P; j++)
            if (j != i) kbest3(pts + 3 * (size_t)i, pts + 3 * (size_t)j, best);
        out[i] = (best[0] + best[1] + best[2]) / 3.0f;
    }
}
