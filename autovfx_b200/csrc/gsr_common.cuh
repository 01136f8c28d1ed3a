// gsr_b200 — shared device/host helpers.  sm_90a (H100) only.
//
// Arithmetic note (bit-exact tile/key indexing, SURVEY §7 "hard parts"): every quantity that feeds an
// integer output of the reference (radii, tile rectangles, depth key bits) is computed with the same
// fp32 expression TREES as the reference's preprocess (DGR/cuda_rasterizer/forward.cu:74-256 and the
// GLM 3x3 product it uses, third_party/glm/glm/detail/type_mat3x3.inl:486-519), including the terms
// that multiply structural zeros, so that nvcc's FMA contraction produces the same roundings.  The
// memory access pattern, staging and parallel decomposition are ours.
#pragma once
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>  // header-only NVTX v3: the ranges cost nothing unless a profiler is attached
#include <stdint.h>
#include "../../include/gsr_b200.h"

#define GSR_TILE 16
#define GSR_TILE_PIX 256
#define GSR_FOOTS 8  // warp footprints (8x4 pixels) per tile
#define GSR_FULL 0xffffffffu

namespace gsr {

__host__ __device__ inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---- workspace layouts (pure functions of P / capacity / W,H) --------------------------------------
struct GeomLayout {
    size_t records, ranks, vis_list, cov3D, clamped, total;
    __host__ __device__ explicit GeomLayout(size_t P) {
        size_t o = 0;
        records = o; o = align_up(o + 48 * P, 256);
        ranks = o;   o = align_up(o + 32 * P, 256);  // 8 x u32 in-tile ranks for Gaussians touching <= 8 tiles
        vis_list = o; o = align_up(o + 4 * P, 256);  // ids of the visible Gaussians (k_project -> k_emit)
        cov3D = o;   o = align_up(o + 24 * P, 256);
        clamped = o; o = align_up(o + P, 256);
        total = o + 256;
    }
};
struct ImageLayout {
    size_t counters, tile_count, tile_big, tile_fill, ranges, n_contrib, total;
    int gx, gy, tiles;
    __host__ __device__ ImageLayout(int W, int H) {
        gx = (W + GSR_TILE - 1) / GSR_TILE;
        gy = (H + GSR_TILE - 1) / GSR_TILE;
        tiles = gx * gy;
        size_t o = 0;
        counters = o;   o = align_up(o + sizeof(gsr_counters), 256);
        tile_count = o; o = align_up(o + 4 * (size_t)tiles, 256);  // instances of Gaussians touching <= 8 tiles (ranked)
        tile_big = o;   o = align_up(o + 4 * (size_t)tiles, 256);  // instances of Gaussians touching > 8 tiles
        tile_fill = o;  o = align_up(o + 4 * (size_t)tiles, 256);  // cursor for the latter, written by the scan
        ranges = o;     o = align_up(o + 8 * (size_t)tiles, 256);
        n_contrib = o;  o = align_up(o + 4 * (size_t)W * H, 256);
        total = o + 256;
    }
    // bytes [0, zero_bytes) are cleared at the start of every frame (counters + tile_count + tile_big)
    __host__ __device__ size_t zero_bytes() const { return tile_fill; }
};
// Binning workspace: 8 (pair) + 4 (point_list) bytes per instance of capacity, plus the footprint ballot matrix: one 32-byte
// row per 32 list entries, rows of tile t starting at (ranges[t].x >> 5) + t -> at most capacity / 32 + tiles + 1 rows.
#define GSR_BAL_SLACK_TILES 131072  // tile count the fixed part of the workspace provides rows for (e.g. 8192 x 4096 pixels)
struct BinLayout {
    size_t pairs, point_list, bal, bal_rows, total, capacity;
    __host__ __device__ explicit BinLayout(size_t cap) {
        capacity = cap;
        pairs = 0;
        point_list = 8 * cap;
        bal = align_up(12 * cap, 256);
        bal_rows = cap / 32 + GSR_BAL_SLACK_TILES + 2;
        total = 13 * cap + fixed_bytes();  // >= bal + 32 * bal_rows
    }
    __host__ __device__ static size_t fixed_bytes() { return 32 * (size_t)GSR_BAL_SLACK_TILES + 512; }
    __host__ __device__ static size_t capacity_of(size_t bytes) { return bytes > fixed_bytes() ? (bytes - fixed_bytes()) / 13 : 0; }
    // Slab emission (slab stride S > 0): `slots` = tiles x S pairs occupy the END of the pairs region, 256-byte aligned, so the
    // offsets of every region stay a function of the workspace size alone (the backward and gsr_get_views do not know S).  The
    // compact capacity is what lies below the slab; 0 if the slab does not fit.
    __host__ __device__ static size_t slab_offset(size_t cap, size_t slots) { return slots < cap ? (8 * (cap - slots)) & ~(size_t)255 : 0; }
    __host__ __device__ static size_t bytes_with_slab(size_t cap, size_t slots) { return BinLayout(cap + slots + 32).total; }
};

// ---- camera block staged in shared memory ------------------------------------------------------------
struct CamConsts {
    float view[16];
    float proj[16];
    float campos[3];
};

// ---- minimal column-major 3x3 (m[col][row]) with the textbook product order --------------------------
struct m3 {
    float m[3][3];
};
__device__ __forceinline__ m3 m3_make(float a0, float a1, float a2, float b0, float b1, float b2, float c0, float c1, float c2) {
    m3 r;
    r.m[0][0] = a0; r.m[0][1] = a1; r.m[0][2] = a2;
    r.m[1][0] = b0; r.m[1][1] = b1; r.m[1][2] = b2;
    r.m[2][0] = c0; r.m[2][1] = c1; r.m[2][2] = c2;
    return r;
}
__device__ __forceinline__ m3 m3_mul(const m3& A, const m3& B) {
    m3 R;
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
        for (int r = 0; r < 3; r++)
            R.m[c][r] = A.m[0][r] * B.m[c][0] + A.m[1][r] * B.m[c][1] + A.m[2][r] * B.m[c][2];
    return R;
}
__device__ __forceinline__ m3 m3_t(const m3& A) {
    m3 R;
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
        for (int r = 0; r < 3; r++) R.m[c][r] = A.m[r][c];
    return R;
}

// row-vector * row-major buffer (DGR/cuda_rasterizer/auxiliary.h:58-77)
__device__ __forceinline__ float3 xform4x3(const float3& p, const float* m) {
    float3 t = {m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12], m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
                m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14]};
    return t;
}
__device__ __forceinline__ float4 xform4x4(const float3& p, const float* m) {
    float4 t = {m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12], m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
                m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14], m[3] * p.x + m[7] * p.y + m[11] * p.z + m[15]};
    return t;
}

// auxiliary.h:41-44 — double-precision literals make this a double expression
__device__ __forceinline__ float ndc2pix(float v, int S) { return ((v + 1.0) * S - 1.0) * 0.5; }

// auxiliary.h:46-56
__device__ __forceinline__ void tile_rect(float px, float py, int r, int gx, int gy, int& x0, int& y0, int& x1, int& y1) {
    x0 = min(gx, max(0, (int)((px - r) / GSR_TILE)));
    y0 = min(gy, max(0, (int)((py - r) / GSR_TILE)));
    x1 = min(gx, max(0, (int)((px + r + GSR_TILE - 1) / GSR_TILE)));
    y1 = min(gy, max(0, (int)((py + r + GSR_TILE - 1) / GSR_TILE)));
}

// Run op(tile_index, tx, ty, payload) once for every tile of this lane's rectangle; payload = NW 32-bit words of
// the lane that owns the rectangle.  Rectangles of up to SMALL tiles are walked by their own lane; larger ones are
// walked by the whole warp, 32 tiles at a time (the owner's payload is broadcast by shuffles first), so one huge
// splat does not serialise a warp.  Must be called by all 32 lanes (lanes with nothing to do pass an empty rectangle).
template <int SMALL, int NW, typename Op>
__device__ __forceinline__ void for_each_tile(int x0, int y0, int x1, int y1, int gx, const uint32_t (&pay)[NW], Op op) {
    const int w = x1 - x0;
    const int cnt = w * (y1 - y0);
    const int lane = threadIdx.x & 31;
    if (cnt > 0 && cnt <= SMALL) {
        for (int y = y0; y < y1; y++)
            for (int x = x0; x < x1; x++) op(y * gx + x, x, y, pay);
    }
    __syncwarp();
    unsigned big = __ballot_sync(GSR_FULL, cnt > SMALL);
    while (big) {
        const int src = __ffs(big) - 1;
        big &= big - 1;
        const int bx0 = __shfl_sync(GSR_FULL, x0, src), by0 = __shfl_sync(GSR_FULL, y0, src);
        const int bw = __shfl_sync(GSR_FULL, w, src), bn = __shfl_sync(GSR_FULL, cnt, src);
        uint32_t bp[NW];
#pragma unroll
        for (int k = 0; k < NW; k++) bp[k] = __shfl_sync(GSR_FULL, pay[k], src);
        const float inv_w = 1.0f / (float)bw;  // row of tile t without an integer division: (t + 0.5) / bw is at least 0.5/bw away from
        for (int t = lane; t < bn; t += 32) {  // an integer and the float product is off by < t * 2^-22 / bw, so it truncates exactly for t < 2^21
            const int row = (int)(((float)t + 0.5f) * inv_w);
            const int ty = by0 + row, tx = bx0 + (t - row * bw);
            op(ty * gx + tx, tx, ty, bp);
        }
        __syncwarp();
    }
}

// ---- warp-footprint culling shared by the forward and backward blend kernels ------------------------------
// A warp owns an 8x4 pixel footprint (half extents FOOT_HX x FOOT_HY around its centre).  A splat can reach
// alpha >= 1/255 at a pixel p only where power(p) = -q(p)/2 >= -tau, q(p) = (mu-p)^T A (mu-p) (A = conic),
// tau = ln(255*opacity).  The test computes the exact minimum of the convex form q over the footprint: it lies
// on one of the two box faces that face the splat centre, where q restricted to the face is a parabola.  Both
// face minima are evaluated branch-free (a face that does not separate the box from the centre yields a value
// >= the true minimum, so taking the smaller of the two is always right).  The reciprocals are approximate
// (MUFU.RCP): an imprecise minimiser only raises the evaluated q by a second-order amount.  Margins: 1e-3 on
// tau and 4e-6 of the magnitude of the terms (float rounding here and in the reference's own evaluation of
// `power`), so a rejected (footprint, splat) pair is one the reference skips at every pixel of the footprint.
// Non positive-definite conics and NaNs are never culled.
constexpr float FOOT_HX = 3.5f, FOOT_HY = 1.5f;
__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float sqrt_approx(float x) {
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float footprint_tau(float opacity) { return __logf(255.0f * opacity); }
// dx, dy: splat centre minus box centre; hx, hy: half extents of the box of pixel centres
__device__ __forceinline__ bool box_may_touch(float dx, float dy, float a, float b, float c, float tau, float hx, float hy) {
    const float uc = dx - fminf(fmaxf(dx, -hx), hx);  // signed distance of the box from the centre, 0 if it straddles
    const float vc = dy - fminf(fmaxf(dy, -hy), hy);
    const float vs = fminf(fmaxf(-b * uc * rcp_approx(c), dy - hy), dy + hy);  // minimiser on the face u = uc
    const float us = fminf(fmaxf(-b * vc * rcp_approx(a), dx - hx), dx + hx);  // minimiser on the face v = vc
    const float q1 = a * uc * uc + 2.f * b * uc * vs + c * vs * vs;
    const float q2 = a * us * us + 2.f * b * us * vc + c * vc * vc;
    const float um = fabsf(dx) + hx, vm = fabsf(dy) + hy;
    const float mag = a * um * um + c * vm * vm + 2.f * fabsf(b) * um * vm;
    const bool pd = a > 0.f && c > 0.f;
    return !(pd && 0.5f * fminf(q1, q2) > tau + 1.0e-3f + 4.0e-6f * mag);
}
__device__ __forceinline__ bool footprint_may_touch(float dx, float dy, float a, float b, float c, float tau) {
    return box_may_touch(dx, dy, a, b, c, tau, FOOT_HX, FOOT_HY);
}
// whole 16x16 tile (tx, ty): pixel centres [16 tx, 16 tx + 15] x [16 ty, 16 ty + 15]
__device__ __forceinline__ bool tile_may_touch(float px, float py, float a, float b, float c, float tau, int tx, int ty) {
    return box_may_touch(px - ((float)(tx * GSR_TILE) + 7.5f), py - ((float)(ty * GSR_TILE) + 7.5f), a, b, c, tau, 7.5f, 7.5f);
}

// All eight warp footprints of tile (tx, ty) at once, for one splat: bit w of the result is set if footprint w (origin
// ((w & 1) * 8, (w >> 1) * 4) inside the tile, 8x4 pixels) may be touched — the same exact box minimum as box_may_touch, with
// the per-column / per-row parts of the two face parabolas shared between the footprints and one (larger, hence still
// conservative) rounding margin for the whole tile.
__device__ __forceinline__ uint32_t tile_foot_mask(float px, float py, float a, float b, float c, float tau, int tx, int ty) {
    const float dxt = px - (float)(tx * GSR_TILE), dyt = py - (float)(ty * GSR_TILE);
    const bool pd = a > 0.f && c > 0.f;
    const float um = fabsf(dxt - 7.5f) + 7.5f, vm = fabsf(dyt - 7.5f) + 7.5f;
    const float mag = a * um * um + c * vm * vm + 2.f * fabsf(b) * um * vm;
    const float thr = 2.f * (tau + 1.0e-3f + 4.0e-6f * mag);
    const float nbrc = -b * rcp_approx(c), nbra = -b * rcp_approx(a), b2 = 2.f * b;
    float dxl[2], dxh[2], Auc[2], Buc[2], vs0[2];
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const float dx = dxt - (FOOT_HX + 8.f * i);
        const float uc = dx - fminf(fmaxf(dx, -FOOT_HX), FOOT_HX);
        dxl[i] = dx - FOOT_HX; dxh[i] = dx + FOOT_HX;
        Auc[i] = a * uc * uc; Buc[i] = b2 * uc; vs0[i] = nbrc * uc;
    }
    uint32_t mask = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const float dy = dyt - (FOOT_HY + 4.f * j);
        const float vc = dy - fminf(fmaxf(dy, -FOOT_HY), FOOT_HY);
        const float dyl = dy - FOOT_HY, dyh = dy + FOOT_HY;
        const float Cvc = c * vc * vc, Bvc = b2 * vc, us0 = nbra * vc;
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const float vs = fminf(fmaxf(vs0[i], dyl), dyh);
            const float us = fminf(fmaxf(us0, dxl[i]), dxh[i]);
            const float q1 = Auc[i] + vs * (Buc[i] + c * vs);
            const float q2 = Cvc + us * (Bvc + a * us);
            if (!(pd && fminf(q1, q2) > thr)) mask |= 1u << (2 * j + i);
        }
    }
    return mask;
}

// ---- footprint masks from strip intervals -------------------------------------------------------------------------
// The region where a splat can reach alpha >= 1/255 is the ellipse q(x, y) <= T around (px, py), T = 2 (tau + margins).
// For an 8-pixel-wide column strip [X, X+7] the ellipse covers the rows [py + tlo, py + thi]: on the line x = px + s the
// form has the roots t = (-b s +- sqrt(c T - det s^2)) / c, the upper one is largest at s = -b sqrt(T / (a det)) and the
// lower one smallest at the opposite point, both clamped to the strip (they lie inside the ellipse's x-extent whenever the
// strip meets it; D < 0 at both clamped points means it does not).  A footprint (strip, 4-row band) is touched iff the band
// meets that interval.  ~22 instructions per strip + 3 per footprint instead of ~37 per footprint for the box-minimum test;
// numerically it is a superset of it (T is inflated by 2e-3 relative for the approximate units and the cancellation in
// det, rows by 0.01 pixel; checked on 400k random splats: 0 misses, 0.15 % more survivors).  Needs a well-conditioned
// positive-definite conic (det > 1e-4 a c); everything else takes tile_foot_mask.
struct StripCtx {
    float px, py, b, det, rc, cT, sstar;
    bool ok;   // false: use tile_foot_mask (non positive-definite / ill-conditioned conic, NaNs)
    bool none; // the splat cannot reach alpha >= 1/255 anywhere
};
// um, vm: upper bounds of |x - px|, |y - py| over the pixels the masks will be asked for (rounding margin, like box_may_touch)
__device__ __forceinline__ StripCtx strip_ctx(float px, float py, float a, float b, float c, float tau, float um, float vm) {
    StripCtx s;
    const float det = fmaf(a, c, -b * b);
    const float mag = a * um * um + c * vm * vm + 2.f * fabsf(b) * um * vm;
    const float T = 2.004f * (tau + 1.0e-3f + 4.0e-6f * mag);
    s.ok = a > 0.f && c > 0.f && det > 1.0e-4f * (a * c) && T == T;
    s.none = s.ok && !(T > 0.f);
    s.px = px; s.py = py; s.b = b; s.det = det;
    s.rc = rcp_approx(c);
    s.cT = c * T;
    s.sstar = b * sqrt_approx(fmaxf(T, 0.f) * rcp_approx(a * det));
    return s;
}
// rows [ylo, yhi] covered inside the strip of pixel columns [X, X + w - 1]; false if the strip misses the ellipse
__device__ __forceinline__ bool strip_rows(const StripCtx& s, float X, float w, float& ylo, float& yhi) {
    const float sl = X - s.px, sh = sl + (w - 1.f);
    const float st = fminf(fmaxf(-s.sstar, sl), sh), sb = fminf(fmaxf(s.sstar, sl), sh);
    const float Dt = fmaf(-s.det, st * st, s.cT), Db = fmaf(-s.det, sb * sb, s.cT);
    yhi = s.py + (fmaf(-s.b, st, sqrt_approx(fmaxf(Dt, 0.f))) * s.rc + 0.01f);
    ylo = s.py + (fmaf(-s.b, sb, -sqrt_approx(fmaxf(Db, 0.f))) * s.rc - 0.01f);
    return Dt >= 0.f || Db >= 0.f;
}
// mask of the eight 8x4 footprints of tile (tx, ty) from the tile's two strips
__device__ __forceinline__ uint32_t strip_tile_mask(const StripCtx& s, int tx, int ty) {
    uint32_t mask = 0;
    const float Y = (float)(ty * GSR_TILE);
#pragma unroll
    for (int i = 0; i < 2; i++) {
        float ylo, yhi;
        const bool v = strip_rows(s, (float)(tx * GSR_TILE + 8 * i), 8.f, ylo, yhi);
#pragma unroll
        for (int j = 0; j < 4; j++)
            if (v && ylo <= Y + (4.f * j + 3.f) && yhi >= Y + 4.f * j) mask |= 1u << (2 * j + i);
    }
    return mask;
}
// The emission's masks (k_emit, and k_project on the slab path; both must produce the same bits): the rows [ylo, yhi] the two
// strips of tile column tx cover, as bit masks over the (at most 32) 4-row bands from row Y0 = 16 ty_lo down: band k = rows
// [Y0 + 4k, Y0 + 4k + 3] is touched iff ylo <= Y0 + 4k + 3 and yhi >= Y0 + 4k, i.e. ceil((ylo - Y0 - 3) / 4) <= k <= floor((yhi - Y0) / 4).
// Two conversions per strip instead of eight comparisons per tile; near a band boundary the subtractions are exact (Y0 is an
// integer within a factor two of y), and the strips carry a 0.01-pixel margin anyway.  strips = s.ok && !s.none.
__device__ __forceinline__ void column_bands(const StripCtx& s, bool strips, int tx, int ty_lo, uint32_t& bands0, uint32_t& bands1) {
    float ylo0 = 0.f, yhi0 = 0.f, ylo1 = 0.f, yhi1 = 0.f;
    bool v0 = false, v1 = false;
    if (strips) {
        v0 = strip_rows(s, (float)(tx * GSR_TILE), 8.f, ylo0, yhi0);
        v1 = strip_rows(s, (float)(tx * GSR_TILE + 8), 8.f, ylo1, yhi1);
    }
    const float Y0 = (float)(ty_lo * GSR_TILE);
    auto band_bits = [&](const bool v, const float ylo, const float yhi) -> uint32_t {
        const float a = fminf(fmaxf((ylo - Y0 - 3.f) * 0.25f, -1.f), 33.f), b = fminf(fmaxf((yhi - Y0) * 0.25f, -1.f), 33.f);
        const int klo = max((int)ceilf(a), 0), khi = min((int)floorf(b), 31);
        return (v && klo <= khi) ? (0xffffffffu >> (31 - khi)) & (0xffffffffu << klo) : 0u;
    };
    bands0 = band_bits(v0, ylo0, yhi0);
    bands1 = band_bits(v1, ylo1, yhi1);
}
// footprint mask of the tile r rows below ty_lo: its four bands of both strips, interleaved (bit 2q + i = band q of strip i)
__device__ __forceinline__ uint32_t bands_tile_mask(uint32_t bands0, uint32_t bands1, int r) {
    uint32_t n0 = (bands0 >> (4 * r)) & 15u, n1 = (bands1 >> (4 * r)) & 15u;
    n0 = (n0 | (n0 << 2)) & 0x33u; n0 = (n0 | (n0 << 1)) & 0x55u;
    n1 = (n1 | (n1 << 2)) & 0x33u; n1 = (n1 | (n1 << 1)) & 0x55u;
    return n0 | (n1 << 1);
}
// strip context of a splat over its whole tile rectangle [x0, x1) x [y0, y1) (the margins bound |x - px|, |y - py| over it)
__device__ __forceinline__ StripCtx rect_strip_ctx(float px, float py, float a, float b, float c, float tau, int x0, int y0, int x1, int y1) {
    const float um = fmaxf(px - (float)(x0 * GSR_TILE), (float)(x1 * GSR_TILE) - px);
    const float vm = fmaxf(py - (float)(y0 * GSR_TILE), (float)(y1 * GSR_TILE) - py);
    return strip_ctx(px, py, a, b, c, tau, um, vm);
}

// one (splat, tile) pair, any conic
__device__ __forceinline__ uint32_t tile_foot_mask_any(float px, float py, float a, float b, float c, float tau, int tx, int ty) {
    const float um = fabsf(px - ((float)(tx * GSR_TILE) + 7.5f)) + 7.5f, vm = fabsf(py - ((float)(ty * GSR_TILE) + 7.5f)) + 7.5f;
    const StripCtx s = strip_ctx(px, py, a, b, c, tau, um, vm);
    if (!s.ok) return tile_foot_mask(px, py, a, b, c, tau, tx, ty);
    if (s.none) return 0u;
    return strip_tile_mask(s, tx, ty);
}

// ---- the shading-normal decision of GaussianModel.get_normal (GM/:120-128, GU/:78-157) ------------------------------------
// One IEEE rounding per reference torch op, in the reference's order.  Shared by k_axis_normals (the forward) and
// k_activate_backward, which must differentiate through the very axis and flip the forward chose.
__device__ __forceinline__ float norm3_rn(float x, float y, float z) {
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}
// F.normalize(v, dim=-1) of one 3-vector: v / clamp_min(||v||, 1e-12).  Returns the unclamped norm (the backward's branch).
__device__ __forceinline__ float normalize3_rn(float x, float y, float z, float& vx, float& vy, float& vz) {
    const float n = norm3_rn(x, y, z), dn = fmaxf(n, 1e-12f);
    vx = __fdiv_rn(x, dn); vy = __fdiv_rn(y, dn); vz = __fdiv_rn(z, dn);
    return n;
}
// torch.sigmoid as 1 / (1 + exp(-x)) (GM/:95-115, SuGaR's strengths)
__device__ __forceinline__ float sigmoid_rn(float x) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-x))); }
struct AxisPick {
    int k;            // argsort(scales)[0]: the smallest scale, ties to the lowest index (GU/:137)
    bool flip;        // flip_align_view negated the axis (GU/:151-157)
    float qn;         // ||r||, the norm build_rotation divides by (no clamp, GU/:79)
    float w, x, y, z; // r / ||r||
    float a0, a1, a2; // column k of build_rotation(r), before the flip
};
__device__ __forceinline__ AxisPick axis_pick(float s0, float s1, float s2, float q0, float q1, float q2, float q3, float m0, float m1,
                                              float m2, const float* campos) {
    AxisPick p;
    p.k = 0;
    float sm = s0;
    if (s1 < sm) { sm = s1; p.k = 1; }
    if (s2 < sm) { sm = s2; p.k = 2; }
    // build_rotation (GU/:78-99): normalise, then the k-th COLUMN of R
    p.qn = __fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q0, q0), __fmul_rn(q1, q1)), __fmul_rn(q2, q2)), __fmul_rn(q3, q3)));
    const float r = __fdiv_rn(q0, p.qn), x = __fdiv_rn(q1, p.qn), y = __fdiv_rn(q2, p.qn), z = __fdiv_rn(q3, p.qn);
    p.w = r; p.x = x; p.y = y; p.z = z;
    if (p.k == 0) {
        p.a0 = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(y, y), __fmul_rn(z, z))));
        p.a1 = __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, y), __fmul_rn(r, z)));
        p.a2 = __fmul_rn(2.0f, __fsub_rn(__fmul_rn(x, z), __fmul_rn(r, y)));
    } else if (p.k == 1) {
        p.a0 = __fmul_rn(2.0f, __fsub_rn(__fmul_rn(x, y), __fmul_rn(r, z)));
        p.a1 = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, x), __fmul_rn(z, z))));
        p.a2 = __fmul_rn(2.0f, __fadd_rn(__fmul_rn(y, z), __fmul_rn(r, x)));
    } else {
        p.a0 = __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, z), __fmul_rn(r, y)));
        p.a1 = __fmul_rn(2.0f, __fsub_rn(__fmul_rn(y, z), __fmul_rn(r, x)));
        p.a2 = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y))));
    }
    // dir_pp_normalized (GR/:131-132) and flip_align_view (GU/:151-157): keep the axis if it faces the camera
    const float dx = __fsub_rn(m0, campos[0]), dy = __fsub_rn(m1, campos[1]), dz = __fsub_rn(m2, campos[2]);
    const float dn = norm3_rn(dx, dy, dz);
    const float vx = __fdiv_rn(dx, dn), vy = __fdiv_rn(dy, dn), vz = __fdiv_rn(dz, dn);
    const float dot = __fadd_rn(__fadd_rn(__fmul_rn(p.a0, -vx), __fmul_rn(p.a1, -vy)), __fmul_rn(p.a2, -vz));
    p.flip = !(dot >= 0.0f);
    return p;
}

// ---- SuGaR's shading-normal decision (sugar_model.py:801-815 get_smallest_axis, :2164-2168; GU/:151-157) -------------------------
// Not get_normal: the rotation is pytorch3d's quaternion_to_matrix of the RAW quaternion (two_s = 2 / |q|^2, no normalisation),
// the axis is torch.min(scaling, dim=-1)'s index (ties: the lowest index), and the view direction is F.normalize'd (1e-12 clamp).
// One IEEE rounding per torch op, in torch's order.  Shared by k_sugar_normals and k_sugar_normals_backward.
struct SugarAxisPick {
    int k;            // scaling.min(dim=-1)[1]
    bool flip;        // flip_align_view negated the axis
    float two_s;      // 2 / (r^2 + i^2 + j^2 + k^2), as torch evaluates `2.0 / t`: reciprocal(t) * 2
    float a0, a1, a2; // column k of quaternion_to_matrix(q), before the flip
};
__device__ __forceinline__ SugarAxisPick sugar_axis_pick(float s0, float s1, float s2, float r, float i, float j, float k, float m0,
                                                         float m1, float m2, const float* campos) {
    SugarAxisPick p;
    p.k = 0;
    float sm = s0;
    if (s1 < sm) { sm = s1; p.k = 1; }
    if (s2 < sm) { sm = s2; p.k = 2; }
    // (q * q).sum(-1), left to right, then 2.0 / that
    const float ss = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r, r), __fmul_rn(i, i)), __fmul_rn(j, j)), __fmul_rn(k, k));
    const float t = __fmul_rn(__frcp_rn(ss), 2.0f);
    p.two_s = t;
    // o = stack(1 - t(jj+kk), t(ij-kr), t(ik+jr), t(ij+kr), 1 - t(ii+kk), t(jk-ir), t(ik-jr), t(jk+ir), 1 - t(ii+jj)).view(3,3)
    if (p.k == 0) {
        p.a0 = __fsub_rn(1.0f, __fmul_rn(t, __fadd_rn(__fmul_rn(j, j), __fmul_rn(k, k))));
        p.a1 = __fmul_rn(t, __fadd_rn(__fmul_rn(i, j), __fmul_rn(k, r)));
        p.a2 = __fmul_rn(t, __fsub_rn(__fmul_rn(i, k), __fmul_rn(j, r)));
    } else if (p.k == 1) {
        p.a0 = __fmul_rn(t, __fsub_rn(__fmul_rn(i, j), __fmul_rn(k, r)));
        p.a1 = __fsub_rn(1.0f, __fmul_rn(t, __fadd_rn(__fmul_rn(i, i), __fmul_rn(k, k))));
        p.a2 = __fmul_rn(t, __fadd_rn(__fmul_rn(j, k), __fmul_rn(i, r)));
    } else {
        p.a0 = __fmul_rn(t, __fadd_rn(__fmul_rn(i, k), __fmul_rn(j, r)));
        p.a1 = __fmul_rn(t, __fsub_rn(__fmul_rn(j, k), __fmul_rn(i, r)));
        p.a2 = __fsub_rn(1.0f, __fmul_rn(t, __fadd_rn(__fmul_rn(i, i), __fmul_rn(j, j))));
    }
    // render_directions = F.normalize(positions - camera_center, dim=-1); keep the axis if dot(axis, -dir) >= 0
    const float dx = __fsub_rn(m0, campos[0]), dy = __fsub_rn(m1, campos[1]), dz = __fsub_rn(m2, campos[2]);
    float vx, vy, vz;
    normalize3_rn(dx, dy, dz, vx, vy, vz);
    const float dot = __fadd_rn(__fadd_rn(__fmul_rn(p.a0, -vx), __fmul_rn(p.a1, -vy)), __fmul_rn(p.a2, -vz));
    p.flip = !(dot >= 0.0f);
    return p;
}

// The whole of pytorch3d's quaternion_to_matrix(q) for a raw q = (r, i, j, k), row-major R[3 * row + col], with sugar_axis_pick's
// roundings; t = two_s = 2 / |q|^2 as torch evaluates it.
__device__ __forceinline__ void quat_to_matrix_rn(float r, float i, float j, float k, float (&R)[9], float& t) {
    const float ss = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r, r), __fmul_rn(i, i)), __fmul_rn(j, j)), __fmul_rn(k, k));
    t = __fmul_rn(__frcp_rn(ss), 2.0f);
    R[0] = __fsub_rn(1.0f, __fmul_rn(t, __fadd_rn(__fmul_rn(j, j), __fmul_rn(k, k))));
    R[1] = __fmul_rn(t, __fsub_rn(__fmul_rn(i, j), __fmul_rn(k, r)));
    R[2] = __fmul_rn(t, __fadd_rn(__fmul_rn(i, k), __fmul_rn(j, r)));
    R[3] = __fmul_rn(t, __fadd_rn(__fmul_rn(i, j), __fmul_rn(k, r)));
    R[4] = __fsub_rn(1.0f, __fmul_rn(t, __fadd_rn(__fmul_rn(i, i), __fmul_rn(k, k))));
    R[5] = __fmul_rn(t, __fsub_rn(__fmul_rn(j, k), __fmul_rn(i, r)));
    R[6] = __fmul_rn(t, __fsub_rn(__fmul_rn(i, k), __fmul_rn(j, r)));
    R[7] = __fmul_rn(t, __fadd_rn(__fmul_rn(j, k), __fmul_rn(i, r)));
    R[8] = __fsub_rn(1.0f, __fmul_rn(t, __fadd_rn(__fmul_rn(i, i), __fmul_rn(j, j))));
}
// Its vector-Jacobian product for dL/dR = G (row-major): with R = base + t u(q) and dt/dq = -t^2 q,
//   dL/dq = t * sum_ab G_ab du_ab/dq - t^2 * (sum_ab G_ab u_ab) * q.
// k_sugar_normals_backward is the special case of one non-zero column.
__device__ __forceinline__ void quat_to_matrix_vjp(float r, float i, float j, float k, float t, const float (&G)[9], float (&dq)[4]) {
    const float s01 = G[1] + G[3], s02 = G[2] + G[6], s12 = G[5] + G[7];  // symmetric parts
    const float a10 = G[3] - G[1], a02 = G[2] - G[6], a21 = G[7] - G[5];  // antisymmetric parts
    const float gr = k * a10 + j * a02 + i * a21;
    const float gi = j * s01 + k * s02 + r * a21 - 2.0f * i * (G[4] + G[8]);
    const float gj = i * s01 + k * s12 + r * a02 - 2.0f * j * (G[0] + G[8]);
    const float gk = i * s02 + j * s12 + r * a10 - 2.0f * k * (G[0] + G[4]);
    const float su = -G[0] * (j * j + k * k) - G[4] * (i * i + k * k) - G[8] * (i * i + j * j) + G[1] * (i * j - k * r) +
                     G[2] * (i * k + j * r) + G[3] * (i * j + k * r) + G[5] * (j * k - i * r) + G[6] * (i * k - j * r) +
                     G[7] * (j * k + i * r);
    const float tts = t * t * su;
    dq[0] = t * gr - tts * r; dq[1] = t * gi - tts * i; dq[2] = t * gj - tts * j; dq[3] = t * gk - tts * k;
}

// SH basis constants (auxiliary.h:22-39; degree 4: SuGaR's sugar_utils/spherical_harmonics.py:23-33)
constexpr float SH_C0 = 0.28209479177387814f;
constexpr float SH_C1 = 0.4886025119029199f;
constexpr float SH_C2_0 = 1.0925484305920792f, SH_C2_1 = -1.0925484305920792f, SH_C2_2 = 0.31539156525252005f,
                           SH_C2_3 = -1.0925484305920792f, SH_C2_4 = 0.5462742152960396f;
constexpr float SH_C3_0 = -0.5900435899266435f, SH_C3_1 = 2.890611442640554f, SH_C3_2 = -0.4570457994644658f,
                           SH_C3_3 = 0.3731763325901154f, SH_C3_4 = -0.4570457994644658f, SH_C3_5 = 1.445305721320277f,
                           SH_C3_6 = -0.5900435899266435f;
constexpr float SH_C4_0 = 2.5033429417967046f, SH_C4_1 = -1.7701307697799304f, SH_C4_2 = 0.9461746957575601f,
                           SH_C4_3 = -0.6690465435572892f, SH_C4_4 = 0.10578554691520431f, SH_C4_5 = -0.6690465435572892f,
                           SH_C4_6 = 0.47308734787878004f, SH_C4_7 = -1.7701307697799304f, SH_C4_8 = 0.6258357354491761f;

// arguments of the blend kernels (gsr_forward.cu builds them, gsr_blend.cu consumes them)
struct BlendArgs {
    const uint2* ranges; const uint32_t* point_list; const float4* records; const float* extra;
    int W, H, gx, gy; const float* bg; float *out_color, *out_depth, *out_alpha, *out_extra; uint32_t* n_contrib;
    gsr_counters* counters;
    const uint32_t* bal;  // footprint ballot matrix [rows][GSR_FOOTS], rows of tile t from bal_row_base(ranges[t].x, t)
    int exact;  // GSR_FLAG_EXACT_IMAGES
};
void launch_blend_lists(const BlendArgs& a, cudaStream_t st);
__host__ __device__ inline size_t bal_row_base(uint32_t range_x, int tile) { return (size_t)(range_x >> 5) + (size_t)tile; }

// Exclusive scan of n entries in place, one CTA of 1024 threads: uint32_t for the radix sort of gsr_knn / gsr_dist2 and for
// gsr_densify_plan, double for the prefix sums of gsr_sugar_sample.  Internal linkage: each translation unit has its own copy.
namespace {
template <typename T>
__global__ void __launch_bounds__(1024) k_rs_scan(T* hist, int n) {
    __shared__ T wsum[32];
    __shared__ T carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry = T(0);
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        const int i = base + tid;
        const T v = i < n ? hist[i] : T(0);
        T incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const T t = __shfl_up_sync(GSR_FULL, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const T s = wsum[lane];
            T si = s;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const T t = __shfl_up_sync(GSR_FULL, si, o);
                if (lane >= o) si += t;
            }
            wsum[lane] = si - s;
        }
        __syncthreads();
        const T excl = carry + wsum[warp] + incl - v;
        if (i < n) hist[i] = excl;
        __syncthreads();
        if (tid == 1023) carry = excl + v;
        __syncthreads();
    }
}
}  // namespace

void set_error(const char* fmt, ...);
int check_launch(const char* what, bool debug, cudaStream_t stream);

struct NvtxRange {  // one named range per C-ABI call (SURVEY §5: the reference has no instrumentation; this build adds NVTX)
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};

}  // namespace gsr
