// gsr_b200 — distCUDA2: mean squared distance to the 3 nearest neighbours.
//
// Replaces SimpleKNN::knn (KNN/simple_knn.cu:185-220).  Same result — the exact mean of the squared distances to the 3
// nearest neighbours (self skipped by index, duplicates count) — and the same first steps: Morton order over the bounding
// box (which always contains the origin, simple_knn.cu:191) and a per-point seed bound from the +-3 Morton neighbours.
// The search itself is organised for the GPU instead of one thread walking every 1024-point box through an index array:
//   * the points are gathered ONCE into Morton order as float4 (x, y, z, original index): every later access is contiguous;
//   * two levels of boxes: 1024-point boxes and their sixteen 64-point sub-boxes, each with an AABB;
//   * one CTA per 256 consecutive (hence spatially close) queries: the CTA's AABB and its largest seed bound select the
//     candidate 1024-point boxes ONCE for all 256 queries (box-to-box distance, the threads share the work), so a query loops over
//     a few dozen candidates instead of all P/1024 boxes; per query the reference's pruning rule (box farther than the seed
//     bound or than the current third-best) is applied to the box and then to its sub-boxes, and only surviving 64-point
//     sub-boxes are scanned.  Pruning is conservative at every level, so the three smallest distances are exact.
// No host round trip (the reference makes two blocking cudaMemcpy's of the bounding box, :197,:200), no cudaMalloc/cudaFree, no
// Thrust/CUB: the bounding box stays on the device, and the (morton, index) sort is a small hand-written stable LSD radix sort
// (one warp per 2048-key chunk, warp match_any ranking).  Init-time only (gaussian_model.py:144).
#include "gsr_common.cuh"
#include <cfloat>

namespace gsr {

constexpr int KNN_BOX = 1024;
constexpr int KNN_SUB = 64;      // points per sub-box (16 per box)
constexpr int KNN_QCTA = 256;    // queries per CTA of the search kernel
constexpr int KNN_MAXC = 1024;   // candidate boxes a CTA can list; beyond that it falls back to testing every box
constexpr int KNN_CHUNK = 2048;  // keys per warp in the radix sort

struct KnnLayout {
    size_t bbox, codes0, codes1, idx0, idx1, hist, boxes, subboxes, sorted, total;
    int nchunks, nboxes, nsub;
    __host__ __device__ explicit KnnLayout(size_t P) {
        nchunks = (int)((P + KNN_CHUNK - 1) / KNN_CHUNK);
        nboxes = (int)((P + KNN_BOX - 1) / KNN_BOX);
        nsub = nboxes * (KNN_BOX / KNN_SUB);
        size_t o = 0;
        bbox = o;   o = align_up(o + 32, 256);
        codes0 = o; o = align_up(o + 4 * P, 256);
        codes1 = o; o = align_up(o + 4 * P, 256);
        idx0 = o;   o = align_up(o + 4 * P, 256);
        idx1 = o;   o = align_up(o + 4 * P, 256);
        hist = o;   o = align_up(o + 4 * 256 * (size_t)nchunks, 256);
        boxes = o;  o = align_up(o + 24 * (size_t)nboxes, 256);
        subboxes = o; o = align_up(o + 24 * (size_t)nsub, 256);
        sorted = o; o = align_up(o + 16 * P, 256);  // float4 (x, y, z, original index) in Morton order
        total = o + 256;
    }
};
size_t dist2_bytes(int P) { return KnnLayout((size_t)(P < 0 ? 0 : P)).total; }

__device__ __forceinline__ uint32_t f2ord(float f) {
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord2f(uint32_t u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u); }

__global__ void k_bbox_init(uint32_t* bbox) {
    if (threadIdx.x < 6) bbox[threadIdx.x] = f2ord(0.0f);  // reduction init {0,0,0} (simple_knn.cu:191)
}
__global__ void __launch_bounds__(256) k_bbox(int P, const float* __restrict__ pts, uint32_t* bbox) {
    float mn[3] = {0, 0, 0}, mx[3] = {0, 0, 0};
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const float v = pts[3 * (size_t)i + k];
            mn[k] = fminf(mn[k], v);
            mx[k] = fmaxf(mx[k], v);
        }
    }
#pragma unroll
    for (int k = 0; k < 3; k++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn[k] = fminf(mn[k], __shfl_xor_sync(GSR_FULL, mn[k], o));
            mx[k] = fmaxf(mx[k], __shfl_xor_sync(GSR_FULL, mx[k], o));
        }
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 3; k++) {
            atomicMin(&bbox[k], f2ord(mn[k]));
            atomicMax(&bbox[3 + k], f2ord(mx[k]));
        }
    }
}

__device__ __forceinline__ uint32_t prep_morton(uint32_t x) {  // simple_knn.cu:46-53
    x = (x | (x << 16)) & 0x030000FF;
    x = (x | (x << 8)) & 0x0300F00F;
    x = (x | (x << 4)) & 0x030C30C3;
    x = (x | (x << 2)) & 0x09249249;
    return x;
}
__global__ void __launch_bounds__(256) k_morton(int P, const float* __restrict__ pts, const uint32_t* __restrict__ bbox,
                                                uint32_t* __restrict__ codes, uint32_t* __restrict__ idx) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float mnx = ord2f(bbox[0]), mny = ord2f(bbox[1]), mnz = ord2f(bbox[2]);
    const float mxx = ord2f(bbox[3]), mxy = ord2f(bbox[4]), mxz = ord2f(bbox[5]);
    const float3 c = {pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2]};
    const uint32_t x = prep_morton(((c.x - mnx) / (mxx - mnx)) * ((1 << 10) - 1));  // simple_knn.cu:55-61
    const uint32_t y = prep_morton(((c.y - mny) / (mxy - mny)) * ((1 << 10) - 1));
    const uint32_t z = prep_morton(((c.z - mnz) / (mxz - mnz)) * ((1 << 10) - 1));
    codes[i] = x | (y << 1) | (z << 2);
    idx[i] = (uint32_t)i;
}

// ---- stable LSD radix sort, 8-bit digits, one warp per chunk of KNN_CHUNK consecutive keys ----
constexpr int RS_WARPS = 4;
__global__ void __launch_bounds__(RS_WARPS * 32) k_rs_hist(int P, const uint32_t* __restrict__ keys, int shift, int nchunks,
                                                           uint32_t* __restrict__ hist) {
    __shared__ uint32_t cnt[RS_WARPS][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int chunk = blockIdx.x * RS_WARPS + warp;
    for (int d = lane; d < 256; d += 32) cnt[warp][d] = 0;
    __syncwarp();
    if (chunk < nchunks) {
        const int b = chunk * KNN_CHUNK, e = min(P, b + KNN_CHUNK);
        for (int i = b + lane; i < e; i += 32) atomicAdd(&cnt[warp][(keys[i] >> shift) & 255u], 1u);
        __syncwarp();
        for (int d = lane; d < 256; d += 32) hist[(size_t)d * nchunks + chunk] = cnt[warp][d];
    }
}
__global__ void __launch_bounds__(1024) k_rs_scan(uint32_t* hist, int n) {  // exclusive scan of n entries, one CTA
    __shared__ uint32_t wsum[32];
    __shared__ uint32_t carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        const int i = base + tid;
        const uint32_t v = i < n ? hist[i] : 0;
        uint32_t incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(GSR_FULL, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            const uint32_t s = wsum[lane];
            uint32_t si = s;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(GSR_FULL, si, o);
                if (lane >= o) si += t;
            }
            wsum[lane] = si - s;
        }
        __syncthreads();
        const uint32_t excl = carry + wsum[warp] + incl - v;
        if (i < n) hist[i] = excl;
        __syncthreads();
        if (tid == 1023) carry = excl + v;
        __syncthreads();
    }
}
__global__ void __launch_bounds__(RS_WARPS * 32) k_rs_scatter(int P, const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                                                              int shift, int nchunks, const uint32_t* __restrict__ hist,
                                                              uint32_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out) {
    __shared__ uint32_t off[RS_WARPS][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int chunk = blockIdx.x * RS_WARPS + warp;
    if (chunk >= nchunks) return;
    for (int d = lane; d < 256; d += 32) off[warp][d] = hist[(size_t)d * nchunks + chunk];
    __syncwarp();
    const int b = chunk * KNN_CHUNK, e = min(P, b + KNN_CHUNK);
    for (int i0 = b; i0 < e; i0 += 32) {
        const int i = i0 + lane;
        const bool act = i < e;
        const uint32_t k = act ? keys[i] : 0u, v = act ? vals[i] : 0u;
        const uint32_t d = act ? ((k >> shift) & 255u) : 256u + lane;  // inactive lanes get unique pseudo-digits
        const unsigned peers = __match_any_sync(GSR_FULL, d);
        const int leader = __ffs(peers) - 1;
        const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
        uint32_t basepos = 0;
        if (act && lane == leader) {
            basepos = off[warp][d];
            off[warp][d] = basepos + __popc(peers);
        }
        basepos = __shfl_sync(GSR_FULL, basepos, leader);
        if (act) {
            keys_out[basepos + rank] = k;
            vals_out[basepos + rank] = v;
        }
        __syncwarp();
    }
}

// ---- points in Morton order, box and sub-box AABBs ----
__global__ void __launch_bounds__(256) k_gather_sorted(int P, const float* __restrict__ pts, const uint32_t* __restrict__ order, float4* __restrict__ sorted) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const uint32_t id = order[i];
    sorted[i] = make_float4(pts[3 * (size_t)id], pts[3 * (size_t)id + 1], pts[3 * (size_t)id + 2], __uint_as_float(id));
}
// one warp per 64-point sub-box; the 16 warps of a CTA cover one 1024-point box and combine their results for its AABB
__global__ void __launch_bounds__(512) k_box_minmax(int P, const float4* __restrict__ sorted, float* __restrict__ boxes, float* __restrict__ subboxes) {
    __shared__ float red[16][6];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int b = blockIdx.x, sb = b * (KNN_BOX / KNN_SUB) + warp;
    float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
#pragma unroll
    for (int k = 0; k < KNN_SUB / 32; k++) {
        const int i = sb * KNN_SUB + k * 32 + lane;
        if (i < P) {
            const float4 v = sorted[i];
            mn[0] = fminf(mn[0], v.x); mn[1] = fminf(mn[1], v.y); mn[2] = fminf(mn[2], v.z);
            mx[0] = fmaxf(mx[0], v.x); mx[1] = fmaxf(mx[1], v.y); mx[2] = fmaxf(mx[2], v.z);
        }
    }
#pragma unroll
    for (int k = 0; k < 3; k++)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn[k] = fminf(mn[k], __shfl_xor_sync(GSR_FULL, mn[k], o));
            mx[k] = fmaxf(mx[k], __shfl_xor_sync(GSR_FULL, mx[k], o));
        }
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < 3; k++) { red[warp][k] = mn[k]; red[warp][3 + k] = mx[k]; subboxes[6 * (size_t)sb + k] = mn[k]; subboxes[6 * (size_t)sb + 3 + k] = mx[k]; }
    }
    __syncthreads();
    if (threadIdx.x < 6) {
        float v = red[0][threadIdx.x];
        for (int w = 1; w < 16; w++) v = threadIdx.x < 3 ? fminf(v, red[w][threadIdx.x]) : fmaxf(v, red[w][threadIdx.x]);
        boxes[6 * (size_t)b + threadIdx.x] = v;
    }
}

// insert a squared distance into the ascending triple of the three smallest seen so far
__device__ __forceinline__ void top3_insert(float d, float& b0, float& b1, float& b2) {
    const float m0 = fminf(b0, d), r0 = fmaxf(b0, d);
    const float m1 = fminf(b1, r0), r1 = fmaxf(b1, r0);
    b0 = m0; b1 = m1; b2 = fminf(b2, r1);
}
__device__ __forceinline__ float dist2_3(float3 a, float4 b) {
    const float dx = b.x - a.x, dy = b.y - a.y, dz = b.z - a.z;
    return dx * dx + dy * dy + dz * dz;
}
// squared distance from a point to an AABB {min xyz, max xyz}; 0 inside (distBoxPoint, simple_knn.cu:119-128: an empty box,
// min = +FLT_MAX, yields a huge distance and is never visited)
__device__ __forceinline__ float point_box_dist2(float3 p, const float* bx) {
    const float dx = fmaxf(fmaxf(bx[0] - p.x, p.x - bx[3]), 0.f), dy = fmaxf(fmaxf(bx[1] - p.y, p.y - bx[4]), 0.f),
                dz = fmaxf(fmaxf(bx[2] - p.z, p.z - bx[5]), 0.f);
    return dx * dx + dy * dy + dz * dz;
}

__global__ void __launch_bounds__(KNN_QCTA) k_knn_search(int P, const float4* __restrict__ sorted, const float* __restrict__ boxes,
                                                          const float* __restrict__ subboxes, int nboxes, float* __restrict__ dists) {
    __shared__ float s_red[KNN_QCTA / 32][7];
    __shared__ float s_q[7];           // the CTA's query AABB and its largest seed bound
    __shared__ uint32_t s_cand[KNN_MAXC];
    __shared__ uint32_t s_ncand;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int q = blockIdx.x * KNN_QCTA + tid;
    const bool valid = q < P;
    float3 pt = {0, 0, 0};
    uint32_t orig = 0;
    float reject = 0.f;
    if (valid) {
        const float4 me = sorted[q];
        pt = make_float3(me.x, me.y, me.z);
        orig = __float_as_uint(me.w);
        float s0 = FLT_MAX, s1 = FLT_MAX, s2 = FLT_MAX;  // seed: the 3 nearest among the +-3 Morton neighbours (simple_knn.cu:156-161)
        for (int i = max(0, q - 3); i <= min(P - 1, q + 3); i++)
            if (i != q) top3_insert(dist2_3(pt, sorted[i]), s0, s1, s2);
        reject = s2;
    }
    // CTA reduction: AABB of the queries, maximum of the seed bounds
    float mn[3] = {valid ? pt.x : FLT_MAX, valid ? pt.y : FLT_MAX, valid ? pt.z : FLT_MAX};
    float mx[3] = {valid ? pt.x : -FLT_MAX, valid ? pt.y : -FLT_MAX, valid ? pt.z : -FLT_MAX};
    float rmax = valid ? reject : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int k = 0; k < 3; k++) {
            mn[k] = fminf(mn[k], __shfl_xor_sync(GSR_FULL, mn[k], o));
            mx[k] = fmaxf(mx[k], __shfl_xor_sync(GSR_FULL, mx[k], o));
        }
        rmax = fmaxf(rmax, __shfl_xor_sync(GSR_FULL, rmax, o));
    }
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < 3; k++) { s_red[warp][k] = mn[k]; s_red[warp][3 + k] = mx[k]; }
        s_red[warp][6] = rmax;
    }
    if (tid == 0) s_ncand = 0;
    __syncthreads();
    if (tid < 7) {
        float v = s_red[0][tid];
        for (int w = 1; w < KNN_QCTA / 32; w++) v = tid < 3 ? fminf(v, s_red[w][tid]) : fmaxf(v, s_red[w][tid]);
        s_q[tid] = v;
    }
    __syncthreads();
    // candidate 1024-point boxes of the CTA: box-to-box distance within the largest seed bound (every query's own bound is smaller)
    for (int b = tid; b < nboxes; b += KNN_QCTA) {
        const float* bx = boxes + 6 * (size_t)b;
        const float dx = fmaxf(fmaxf(bx[0] - s_q[3], s_q[0] - bx[3]), 0.f), dy = fmaxf(fmaxf(bx[1] - s_q[4], s_q[1] - bx[4]), 0.f),
                    dz = fmaxf(fmaxf(bx[2] - s_q[5], s_q[2] - bx[5]), 0.f);
        if (dx * dx + dy * dy + dz * dz <= s_q[6]) {
            const uint32_t slot = atomicAdd(&s_ncand, 1u);
            if (slot < KNN_MAXC) s_cand[slot] = (uint32_t)b;
        }
    }
    __syncthreads();
    const uint32_t nlisted = s_ncand;
    const bool all_boxes = nlisted > KNN_MAXC;  // pathological (e.g. thousands of coincident points): test every box
    const int ncand = all_boxes ? nboxes : (int)nlisted;
    if (!valid) return;
    float b0 = FLT_MAX, b1 = FLT_MAX, b2 = FLT_MAX;
    for (int c = 0; c < ncand; c++) {
        const int b = all_boxes ? c : (int)s_cand[c];
        const float db = point_box_dist2(pt, boxes + 6 * (size_t)b);
        if (db > reject || db > b2) continue;  // the reference's rule (simple_knn.cu:168-170), applied to the box ...
        const int sb0 = b * (KNN_BOX / KNN_SUB);
        for (int sidx = sb0; sidx < sb0 + KNN_BOX / KNN_SUB; sidx++) {
            const int i0 = sidx * KNN_SUB;
            if (i0 >= P) break;
            const float ds = point_box_dist2(pt, subboxes + 6 * (size_t)sidx);
            if (ds > reject || ds > b2) continue;  // ... and to each of its sub-boxes
            const int i1 = min(P, i0 + KNN_SUB);
            for (int i = i0; i < i1; i++)
                if (i != q) top3_insert(dist2_3(pt, sorted[i]), b0, b1, b2);
        }
    }
    dists[orig] = (b0 + b1 + b2) / 3.0f;
}

int dist2_impl(int P, const float* points, float* out, void* ws, size_t ws_bytes, cudaStream_t st) {
    if (P < 0) { set_error("gsr_dist2: negative P"); return GSR_ERR_INVALID; }
    if (P == 0) return GSR_OK;
    if (!points || !out) { set_error("gsr_dist2: null pointer"); return GSR_ERR_INVALID; }
    const KnnLayout L((size_t)P);
    if (!ws || ws_bytes < L.total) { set_error("gsr_dist2: workspace too small (%zu < %zu)", ws_bytes, L.total); return GSR_ERR_WORKSPACE; }
    char* w = (char*)ws;
    uint32_t* bbox = (uint32_t*)(w + L.bbox);
    uint32_t *k0 = (uint32_t*)(w + L.codes0), *k1 = (uint32_t*)(w + L.codes1), *v0 = (uint32_t*)(w + L.idx0), *v1 = (uint32_t*)(w + L.idx1);
    uint32_t* hist = (uint32_t*)(w + L.hist);
    float* boxes = (float*)(w + L.boxes);
    k_bbox_init<<<1, 32, 0, st>>>(bbox);
    k_bbox<<<min(132 * 8, (P + 255) / 256), 256, 0, st>>>(P, points, bbox);
    k_morton<<<(P + 255) / 256, 256, 0, st>>>(P, points, bbox, k0, v0);
    const int rs_blocks = (L.nchunks + RS_WARPS - 1) / RS_WARPS;
    for (int pass = 0; pass < 4; pass++) {
        k_rs_hist<<<rs_blocks, RS_WARPS * 32, 0, st>>>(P, k0, pass * 8, L.nchunks, hist);
        k_rs_scan<<<1, 1024, 0, st>>>(hist, 256 * L.nchunks);
        k_rs_scatter<<<rs_blocks, RS_WARPS * 32, 0, st>>>(P, k0, v0, pass * 8, L.nchunks, hist, k1, v1);
        uint32_t* t = k0; k0 = k1; k1 = t;
        t = v0; v0 = v1; v1 = t;
    }
    float4* sorted = (float4*)(w + L.sorted);
    float* subboxes = (float*)(w + L.subboxes);
    k_gather_sorted<<<(P + 255) / 256, 256, 0, st>>>(P, points, v0, sorted);
    k_box_minmax<<<L.nboxes, 512, 0, st>>>(P, sorted, boxes, subboxes);
    k_knn_search<<<(P + KNN_QCTA - 1) / KNN_QCTA, KNN_QCTA, 0, st>>>(P, sorted, boxes, subboxes, L.nboxes, out);
    return check_launch("gsr_dist2", false, st);
}

}  // namespace gsr
