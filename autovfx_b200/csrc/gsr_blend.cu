// gsr_b200 — forward alpha blend (replaces renderCUDA, DGR/cuda_rasterizer/forward.cu:261-378).
//
// One WARP per 8x4-pixel footprint, one lane per pixel.  The warp walks the footprint's own survivors — the entries of the
// tile's depth-sorted list whose mask says "this splat can reach alpha >= 1/255 somewhere in the footprint" — so there is no
// block-level staging, no barrier and no per-entry cull here; warps are completely independent.
//   expand : the warp's column of the tile's ballot matrix (k_sort_tiles: one 32-bit word per 32 list entries) is turned into
//            list positions: lane l takes row l of a 32-row block, a warp scan of the popcounts gives every lane the stream
//            offset of its survivors, and the lanes write their set bits' positions into a 256-entry ring in shared memory
//   gather : 32 survivors per batch, one per lane: ring -> position -> id (point_list) -> 48-byte record (three 16-byte loads);
//            the next batch's records and the batch-after-next's ids are in flight while the current batch is blended
//   stage  : the batch is transposed into the warp's shared-memory queue, two splats per 112-byte "pair" so that the
//            per-splat arithmetic runs on both lanes of two-lane fp32 values (f32x2, gsr_packed.cuh)
//   drain  : every lane evaluates every queued splat for its pixel (broadcast LDS.128), front to back.
//
// Two drains share the queue:
//   exact : the reference's fp32 instruction sequence (power, expf, opacity multiply, 0.99 clamp, the three skip rules,
//           colour*alpha then *T) — bit-identical images (GSR_FLAG_EXACT_IMAGES, and the repair path of the default mode).
//   fast  : (default) the same bit-exact `power`, then alpha = min(0.99, ex2.approx(power*log2e + log2(opacity))) — one FFMA
//           and one MUFU instead of expf's eight instructions and the opacity multiply — and a shorter serial part
//           (T' = fma(-T, alpha, T), weight = T*alpha, colours accumulated as two fma2).  alpha differs from the reference's by
//           < 1.3e-6 relative, which cannot move an image by 1e-4 — unless it flips a DECISION.  The two decisions are guarded:
//             * alpha < 1/255 (skip): each lane tracks min |log2(255*alpha)| over its evaluations; below BL_QBAND the
//               decision is inside the approximation's error band;
//             * T(1-alpha) < 1e-4 (terminate): the fast drain terminates at 1e-4*(1-BL_T_BAND), so a pixel whose decision could
//               differ from the reference's ends with |T| inside [1e-4*(1-BL_T_BAND), 1e-4*(1+BL_T_BAND)) and stays there.  The
//               band must cover how far the fast T drifts from the exact one: each unclamped splat in front moves it by
//               alpha/(1-alpha) times the relative difference of the two alphas, so two fronts near alpha 0.98 amplify it ~100x.
//               Measured on an H100 over 1080p stacks of one to three fronts with alpha up to 0.989 in front of a deciding
//               splat (tests/test_gpu_blend_decisions.py): the largest drift is 1.82e-5, which a band of 1e-5 let through;
//               BL_T_BAND = 4e-5 keeps 2.2x that.  (Alpha's worst-case relative difference, ~1e-6, times the largest possible
//               amplification, 2*99 for the fronts and 99 for the deciding splat, would ask for 3e-4: 17x the redos.)
//             * power > 0 (skip): cannot happen for a well-conditioned positive-definite conic (det > 1e-5*a*c, rounding of
//               the power expression is 4e-7 of its terms); batches holding any other splat are drained exactly.
//           A warp with any lane inside a band re-blends its whole list with the exact drain (counters->exact_redos: about
//           1,300 of 65,280 warps per 3M/1080p frame on an H100 80GB HBM3 at 700 W, 460 with a 1e-5 band), so the default
//           images carry the reference's decisions everywhere and n_contrib is identical to the exact mode's.
#include "gsr_common.cuh"
#include "gsr_packed.cuh"

namespace gsr {

constexpr float BL_LOG2E = 1.4426950408889634f;
constexpr float BL_LOG2_255 = 7.994353436858858f;
constexpr float BL_QBAND = 3.0e-6f;                     // |log2(255 alpha)| below this: the skip decision is re-done exactly
constexpr float BL_T_BAND = 4.0e-5f;                   // covers the fast T's relative drift from the exact T (see above)
constexpr float BL_T_LO = 0.0001f * (1.0f - BL_T_BAND);  // fast drain's termination threshold
constexpr float BL_T_HI = 0.0001f * (1.0f + BL_T_BAND);  // |T| below this at the end: termination decisions re-done exactly

template <int NX>
struct ListCfg {
    // one pair = two splats: {x0,x1},{y0,y1},{a0,a1},{-b0,-b1},{c0,c1},{lo0,lo1} | {r,g,b,depth}0 | {r,g,b,depth}1 | {o0,o1,pos0,pos1}
    // [| {e0,e1,e2,-}0 | {e0,e1,e2,-}1] + 16 bytes of padding (staging stores of neighbouring pairs hit different banks)
    static constexpr int PAIRB = NX ? 144 : 112;
    static constexpr int QB = 16 * PAIRB;  // 32 splats per warp
    static constexpr int RING = 256;       // expanded survivor positions per warp (u32)
    static constexpr int WB = QB + 4 * RING;  // shared memory per warp
};

// One work item: WARPS footprints of one tile (bx = tile column * PARTS + part, by = tile row), one warp per footprint.
template <int NX, bool NC, bool EXACT, int WARPS>
__device__ __forceinline__ void blend_item(const BlendArgs& a, const int bx, const int by, unsigned char* sq) {
    typedef ListCfg<NX> Cfg;
    constexpr int PAIRB = Cfg::PAIRB;
    constexpr int PARTS = GSR_FOOTS / WARPS;
    constexpr int RING = Cfg::RING;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tx = bx / PARTS, part = bx - tx * PARTS;
    const int f = part * WARPS + warp;
    const int tile = by * a.gx + tx;
    const int pxi = tx * GSR_TILE + (f & 1) * 8 + (lane & 7), pyi = by * GSR_TILE + (f >> 1) * 4 + (lane >> 3);
    const bool inside = pxi < a.W && pyi < a.H;
    const float pixx = (float)pxi, pixy = (float)pyi;
    const uint32_t q_base = (uint32_t)__cvta_generic_to_shared(sq) + (uint32_t)warp * Cfg::WB;
    uint32_t* ring = reinterpret_cast<uint32_t*>(sq + (size_t)warp * Cfg::WB + Cfg::QB);

    uint2 rg = a.ranges[tile];
    if (a.counters->overflow) rg = make_uint2(0u, 0u);
    const uint32_t n = rg.y - rg.x;                  // entries of the tile's list
    const uint32_t rows = (n + 31u) >> 5;            // rows of the tile's ballot matrix
    const uint32_t* __restrict__ balcol = a.bal + bal_row_base(rg.x, tile) * GSR_FOOTS + f;  // this footprint's column
    const uint32_t* __restrict__ plist = a.point_list + rg.x;

    // pixel state.  T: running transmittance; negative once the pixel has terminated (magnitude = final transmittance), so a
    // dead pixel fails every later `T' >= threshold` test by itself.  Pixels outside the image start dead.
    float T;
    f32x2 C01, C2D, E01, E2x;
    uint32_t last;
    float qmin;  // min |log2(255 alpha~)| seen by this lane (fast drain)

    const f32x2 npx2 = pk2(-pixx, -pixx), npy2 = pk2(-pixy, -pixy), mhalf2 = pk2(-0.5f, -0.5f);

    // ---- fast drain --------------------------------------------------------------------------------------------
    auto drain_fast = [&](int cnt) {
        const f32x2 l2e2 = pk2(BL_LOG2E, BL_LOG2E), l255 = pk2(BL_LOG2_255, BL_LOG2_255);
        uint32_t qa = q_base;
        const int np = (cnt + 1) >> 1;
#pragma unroll 2
        for (int k = 0; k < np; k++, qa += PAIRB) {
            const float4 L0 = lds128(qa), L1 = lds128(qa + 16), L2 = lds128(qa + 32), LA = lds128(qa + 48), LB = lds128(qa + 64);
            float2 ps = make_float2(0.f, 0.f);
            if (NC) ps = lds64(qa + 88);
            const f32x2 dx = add2(pk2(L0.x, L0.y), npx2), dy = add2(pk2(L0.z, L0.w), npy2);
            const f32x2 t1 = mul2(pk2(L2.x, L2.y), dy);   // c * dy            (the reference's rounding sequence for `power`,
            const f32x2 t3 = mul2(pk2(L1.x, L1.y), dx);   // a * dx             forward.cu:338: the conditioning of the conic
            const f32x2 t2 = mul2(pk2(L1.z, L1.w), dx);   // (-b) * dx          cannot amplify a difference between the two modes)
            const f32x2 t4 = mul2(dy, t1);
            const f32x2 t5 = mul2(dy, t2);
            const f32x2 t6 = fma2(dx, t3, t4);
            const f32x2 pw = fma2(t6, mhalf2, t5);        // power
            const f32x2 p2 = fma2(pw, l2e2, pk2(L2.z, L2.w));  // log2(alpha~) = power*log2e + log2(opacity)
            const f32x2 q2 = add2(p2, l255);              // log2(255 alpha~): the skip rule alpha < 1/255 is q < 0
            float p0, p1, q0, q1;
            upk2(p2, p0, p1);
            upk2(q2, q0, q1);
            const float a0 = q0 >= 0.0f ? fminf(ex2_approx(p0), 0.99f) : 0.0f;
            const float a1 = q1 >= 0.0f ? fminf(ex2_approx(p1), 0.99f) : 0.0f;
            qmin = fminf(qmin, fminf(fabsf(q0), fabsf(q1)));
            {
                const float tt = fmaf(-T, a0, T);
                const bool live = tt >= BL_T_LO;
                const float w = (live ? T : 0.0f) * a0;
                T = live ? tt : -fabsf(T);
                const f32x2 w2 = pk2(w, w);
                C01 = fma2(w2, pk2(LA.x, LA.y), C01);
                C2D = fma2(w2, pk2(LA.z, LA.w), C2D);
                if (NX) {
                    const float4 EA = lds128(qa + 96);
                    E01 = fma2(w2, pk2(EA.x, EA.y), E01);
                    E2x = fma2(w2, pk2(EA.z, EA.w), E2x);
                }
                if (NC) last = w > 0.0f ? __float_as_uint(ps.x) : last;
            }
            {
                const float tt = fmaf(-T, a1, T);
                const bool live = tt >= BL_T_LO;
                const float w = (live ? T : 0.0f) * a1;
                T = live ? tt : -fabsf(T);
                const f32x2 w2 = pk2(w, w);
                C01 = fma2(w2, pk2(LB.x, LB.y), C01);
                C2D = fma2(w2, pk2(LB.z, LB.w), C2D);
                if (NX) {
                    const float4 EB = lds128(qa + 112);
                    E01 = fma2(w2, pk2(EB.x, EB.y), E01);
                    E2x = fma2(w2, pk2(EB.z, EB.w), E2x);
                }
                if (NC) last = w > 0.0f ? __float_as_uint(ps.y) : last;
            }
        }
    };

    // ---- exact drain: the reference's arithmetic (forward.cu:330-366), bit for bit --------------------------------
    auto drain_exact = [&](int cnt) {
        const f32x2 mone2 = pk2(-1.0f, -1.0f), one2 = pk2(1.0f, 1.0f);
        float C0, C1, C2, Dp, E0 = 0.f, E1 = 0.f, E2 = 0.f, dummy;
        upk2(C01, C0, C1);
        upk2(C2D, C2, Dp);
        if (NX) { upk2(E01, E0, E1); upk2(E2x, E2, dummy); }
        uint32_t qa = q_base;
        const int np = (cnt + 1) >> 1;
        for (int k = 0; k < np; k++, qa += PAIRB) {
            const float4 L0 = lds128(qa), L1 = lds128(qa + 16), L2 = lds128(qa + 32), LA = lds128(qa + 48), LB = lds128(qa + 64),
                         L5 = lds128(qa + 80);
            const f32x2 dx = add2(pk2(L0.x, L0.y), npx2), dy = add2(pk2(L0.z, L0.w), npy2);
            const f32x2 t1 = mul2(pk2(L2.x, L2.y), dy);
            const f32x2 t3 = mul2(pk2(L1.x, L1.y), dx);
            const f32x2 t2 = mul2(pk2(L1.z, L1.w), dx);
            const f32x2 t4 = mul2(dy, t1);
            const f32x2 t5 = mul2(dy, t2);
            const f32x2 t6 = fma2(dx, t3, t4);
            const f32x2 pw = fma2(t6, mhalf2, t5);
            float p0, p1;
            upk2(pw, p0, p1);
            float a0, a1;
            upk2(mul2(pk2(L5.x, L5.y), pk2(exp(p0), exp(p1))), a0, a1);  // opacity * exp(power)
            a0 = min(0.99f, a0);
            a1 = min(0.99f, a1);
            const bool hit0 = !(p0 > 0.0f) && !(a0 < 1.0f / 255.0f), hit1 = !(p1 > 0.0f) && !(a1 < 1.0f / 255.0f);
            float om0, om1;
            upk2(fma2(pk2(a0, a1), mone2, one2), om0, om1);  // 1 - alpha
            {
                const float cr = __fmul_rn(LA.x, a0), cg = __fmul_rn(LA.y, a0), cb = __fmul_rn(LA.z, a0), cd = __fmul_rn(LA.w, a0);
                const bool act = hit0 && T > 0.0f;
                const float test_T = __fmul_rn(T, om0);
                const bool live = act && !(test_T < 0.0001f);
                const float Tw = live ? T : 0.0f;
                C0 = __fmaf_rn(Tw, cr, C0); C1 = __fmaf_rn(Tw, cg, C1); C2 = __fmaf_rn(Tw, cb, C2); Dp = __fmaf_rn(Tw, cd, Dp);
                if (NX) {
                    const float4 EA = lds128(qa + 96);
                    E0 = __fmaf_rn(Tw, __fmul_rn(EA.x, a0), E0); E1 = __fmaf_rn(Tw, __fmul_rn(EA.y, a0), E1); E2 = __fmaf_rn(Tw, __fmul_rn(EA.z, a0), E2);
                }
                T = act ? (live ? test_T : -T) : T;
                if (NC) last = live ? __float_as_uint(L5.z) : last;
            }
            {
                const float cr = __fmul_rn(LB.x, a1), cg = __fmul_rn(LB.y, a1), cb = __fmul_rn(LB.z, a1), cd = __fmul_rn(LB.w, a1);
                const bool act = hit1 && T > 0.0f;
                const float test_T = __fmul_rn(T, om1);
                const bool live = act && !(test_T < 0.0001f);
                const float Tw = live ? T : 0.0f;
                C0 = __fmaf_rn(Tw, cr, C0); C1 = __fmaf_rn(Tw, cg, C1); C2 = __fmaf_rn(Tw, cb, C2); Dp = __fmaf_rn(Tw, cd, Dp);
                if (NX) {
                    const float4 EB = lds128(qa + 112);
                    E0 = __fmaf_rn(Tw, __fmul_rn(EB.x, a1), E0); E1 = __fmaf_rn(Tw, __fmul_rn(EB.y, a1), E1); E2 = __fmaf_rn(Tw, __fmul_rn(EB.z, a1), E2);
                }
                T = act ? (live ? test_T : -T) : T;
                if (NC) last = live ? __float_as_uint(L5.w) : last;
            }
        }
        C01 = pk2(C0, C1);
        C2D = pk2(C2, Dp);
        if (NX) { E01 = pk2(E0, E1); E2x = pk2(E2, 0.0f); }
    };

    // ---- one pass over the footprint's survivors ----------------------------------------------------------------------
    auto run = [&](const bool exact) {
        T = inside ? 1.0f : -1.0f;
        C01 = C2D = E01 = E2x = pk2(0.0f, 0.0f);
        last = 0;
        qmin = 1.0e30f;
        // survivor stream: index s = 0, 1, 2, ... over the set bits of the column in list order.  ring[s % RING] = list position.
        uint32_t rbits = 0;       // this lane's remaining bits of its row in the current 32-row block
        uint32_t roff = 0;        // stream index of this lane's next survivor
        uint32_t rrow = 0;        // list position of bit 0 of this lane's row
        uint32_t sbase = 0;       // stream index after the blocks expanded so far (warp-uniform)
        uint32_t nblk = 0;        // 32-row blocks loaded so far
        uint32_t filled = 0;      // ring holds stream indices [consumed, filled) (warp-uniform)
        uint32_t consumed = 0;    // stream index of the next batch
        bool block_open = false;  // some lane still has unexpanded bits of the current block
        uint32_t wnext = lane < rows ? balcol[(size_t)lane * GSR_FOOTS] : 0u;  // column word of block 0, prefetched
        const uint32_t nblocks = (rows + 31u) >> 5;
        auto refill = [&]() {  // fill the ring up to stream index consumed + RING (or the end of the stream)
            const uint32_t limit = consumed + RING;
            while (true) {
                if (!block_open) {
                    if (nblk == nblocks) break;
                    rbits = wnext;
                    rrow = (nblk * 32u + (uint32_t)lane) * 32u;
                    nblk++;
                    const uint32_t r = nblk * 32u + (uint32_t)lane;
                    wnext = (nblk < nblocks && r < rows) ? balcol[(size_t)r * GSR_FOOTS] : 0u;  // next block's word in flight
                    const uint32_t c = (uint32_t)__popc(rbits);
                    uint32_t incl = c;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const uint32_t v = __shfl_up_sync(GSR_FULL, incl, o);
                        if (lane >= o) incl += v;
                    }
                    roff = sbase + incl - c;
                    sbase += __shfl_sync(GSR_FULL, incl, 31);
                    block_open = true;
                }
                while (rbits && roff < limit) {
                    const uint32_t bit = (uint32_t)__ffs(rbits) - 1u;
                    rbits &= rbits - 1u;
                    ring[roff & (RING - 1)] = rrow + bit;
                    roff++;
                }
                if (__any_sync(GSR_FULL, rbits != 0u)) { filled = limit; return; }  // ring full
                block_open = false;
                filled = sbase;
                if (filled >= limit) return;
            }
            filled = sbase;
        };
        float4 ra = make_float4(0, 0, 0, 0), rb = ra, rc = ra, rd = ra;
        uint32_t pos_c = 0, pos1 = 0, id1 = 0;
        auto load_rec = [&](uint32_t id) {
            const float4* r = a.records + 3 * (size_t)id;
            ra = r[0]; rb = r[1]; rc = r[2];
            if (NX) { const float* e = a.extra + 3 * (size_t)id; rd = make_float4(e[0], e[1], e[2], 0.0f); }
        };
        refill();
        __syncwarp();
        // prologue: records of batch 0, ids of batch 1
        if (consumed + lane < filled) { pos_c = ring[(consumed + lane) & (RING - 1)]; load_rec(plist[pos_c]); }
        if (consumed + 32 + lane < filled) { pos1 = ring[(consumed + 32 + lane) & (RING - 1)]; id1 = plist[pos1]; }
        while (consumed < filled) {
            const int cnt = (int)min(32u, filled - consumed);
            // stage this batch (registers -> queue)
            bool ill = false;
            {
                const uint32_t pb = q_base + (uint32_t)(lane >> 1) * PAIRB, h = (uint32_t)(lane & 1);
                if (lane < cnt) {
                    const float ca = ra.z, cb = ra.w, cc = rb.x, lo = rc.w;
                    ill = !(ca > 0.0f && cc > 0.0f && (ca * cc - cb * cb) > 1.0e-5f * (ca * cc) && lo == lo);
                    const uint32_t qa = pb + h * 4;
                    sts32(qa, ra.x); sts32(qa + 8, ra.y); sts32(qa + 16, ca); sts32(qa + 24, -cb); sts32(qa + 32, cc); sts32(qa + 40, lo);
                    sts128(pb + 48 + h * 16, make_float4(rc.x, rc.y, rc.z, rb.z));
                    sts32(qa + 80, rb.y);
                    sts32(qa + 88, __uint_as_float(pos_c + 1u));  // 1-based position in the tile's list (n_contrib)
                    if (NX) sts128(pb + 96 + h * 16, rd);
                } else if (lane == cnt && (cnt & 1)) {  // complete the last pair with a splat that can never hit
                    const uint32_t qa = pb + h * 4;
                    sts32(qa, 0.f); sts32(qa + 8, 0.f); sts32(qa + 16, 0.f); sts32(qa + 24, 0.f); sts32(qa + 32, 0.f);
                    sts32(qa + 40, __int_as_float(0xff800000));  // log2(0)
                    sts128(pb + 48 + h * 16, make_float4(0.f, 0.f, 0.f, 0.f));
                    sts32(qa + 80, 0.f); sts32(qa + 88, 0.f);
                    if (NX) sts128(pb + 96 + h * 16, make_float4(0.f, 0.f, 0.f, 0.f));
                }
            }
            const bool any_ill = __any_sync(GSR_FULL, ill);
            consumed += (uint32_t)cnt;
            // the ring must hold the two batches after this one; expand only when it runs short (one call fills up to RING entries ahead)
            if (filled - consumed < 96u && (block_open || nblk < nblocks)) refill();
            __syncwarp();   // staging + ring stores visible to every lane
            // next batch's records and the one after's ids go in flight now
            pos_c = pos1;
            if (consumed + lane < filled) load_rec(id1);
            if (consumed + 32 + lane < filled) { pos1 = ring[(consumed + 32 + lane) & (RING - 1)]; id1 = plist[pos1]; }
            if (EXACT || exact || any_ill) drain_exact(cnt);
            else drain_fast(cnt);
            __syncwarp();  // the queue is free again
            if (__all_sync(GSR_FULL, T < 0.0f)) break;  // every pixel of the footprint has terminated
        }
    };

    run(false);
    if (!EXACT) {
        const bool unc = inside && (qmin < BL_QBAND || fabsf(T) < BL_T_HI);
        if (__any_sync(GSR_FULL, unc)) {
            if (lane == 0) atomicAdd(&a.counters->exact_redos, 1u);
            run(true);
        }
    }

    if (inside) {
        const float T_out = fabsf(T);  // final transmittance, whether the pixel terminated or the list ran out
        const size_t pid = (size_t)a.W * pyi + pxi;
        const size_t HW = (size_t)a.H * a.W;
        float C0, C1, C2, Dp;
        upk2(C01, C0, C1);
        upk2(C2D, C2, Dp);
        a.out_alpha[pid] = 1 - T_out;
        if (NC) a.n_contrib[pid] = last;
        a.out_color[pid] = C0 + T_out * a.bg[0];
        a.out_color[HW + pid] = C1 + T_out * a.bg[1];
        a.out_color[2 * HW + pid] = C2 + T_out * a.bg[2];
        a.out_depth[pid] = Dp;
        if (NX) {
            float E0, E1, E2, dummy;
            upk2(E01, E0, E1);
            upk2(E2x, E2, dummy);
            a.out_extra[pid] = E0 + T_out * a.bg[0];
            a.out_extra[HW + pid] = E1 + T_out * a.bg[1];
            a.out_extra[2 * HW + pid] = E2 + T_out * a.bg[2];
        }
    }
}

// OCC: resident warps per SM the kernel is compiled for (32 -> 64 registers; 24 -> 80, which the second colour set needs)
template <int NX, bool NC, bool EXACT, int WARPS, int OCC>
__global__ void __launch_bounds__(WARPS * 32, OCC / WARPS) k_blend_lists(const BlendArgs a) {
    __shared__ __align__(16) unsigned char sq[WARPS * ListCfg<NX>::WB];
    blend_item<NX, NC, EXACT, WARPS>(a, (int)blockIdx.x, (int)blockIdx.y, sq);
}

template <int NX, bool NC, bool EXACT>
static void launch_w(const BlendArgs& a, cudaStream_t st) {
    constexpr int WARPS = 4;  // footprints per CTA
    const dim3 grid(a.gx * (GSR_FOOTS / WARPS), a.gy);
    k_blend_lists<NX, NC, EXACT, WARPS, (NX ? 24 : 32)><<<grid, WARPS * 32, 0, st>>>(a);
}
template <int NX, bool NC>
static void launch_e(const BlendArgs& a, cudaStream_t st) {
    if (a.exact) launch_w<NX, NC, true>(a, st);
    else launch_w<NX, NC, false>(a, st);
}
void launch_blend_lists(const BlendArgs& a, cudaStream_t st) {
    if (a.extra) { if (a.n_contrib) launch_e<3, true>(a, st); else launch_e<3, false>(a, st); }
    else         { if (a.n_contrib) launch_e<0, true>(a, st); else launch_e<0, false>(a, st); }
}

}  // namespace gsr
