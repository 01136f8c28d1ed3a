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
// Thrust/CUB: the bounding box stays on the device, and the (morton, index) sort is the library's stable LSD radix sort (gsr_radix.cuh)
// (one warp per 2048-key chunk, warp match_any ranking).  Init-time only (gaussian_model.py:144).
//
// gsr_knn (below k_knn_search) runs the same pipeline for pytorch3d.ops.knn_points as SuGaR calls it: the K <= 32 nearest points
// of every query, the query set being the points themselves or a second cloud.
#include "gsr_radix.cuh"
#include <cfloat>

namespace gsr {

constexpr int KNN_BOX = 1024;
constexpr int KNN_SUB = 64;      // points per sub-box (16 per box)
constexpr int KNN_QCTA = 256;    // queries per CTA of the search kernel
constexpr int KNN_MAXC = 1024;   // candidate boxes a CTA can list; beyond that it falls back to testing every box
constexpr int KNN_CHUNK = RS_CHUNK;  // keys per warp in the radix sort (gsr_radix.cuh)

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

// ================================================================================================================================
// gsr_knn — exact K nearest neighbours (pytorch3d.ops.knn_points for N = 1, D = 3, K <= 32) on the same Morton boxes.
//
// Distance, pinned: d = (dx*dx + dy*dy) + dz*dz with dx = p.x - q.x, every operation rounded once (no contraction), so a float32
// restatement with separate ops reproduces it bit for bit.  The point-to-box bound is computed with the same rounding sequence
// from the box faces; rounding is monotone, so it never exceeds the computed distance of any point inside the box.
// Ranking is lexicographic on (distance, original index): among equal distances the lower index wins, and a box or sub-box is
// pruned only when its bound is STRICTLY greater than the current K-th distance.  Self is not excluded.
// ================================================================================================================================
constexpr int KNN_KMAX = 32;

__device__ __forceinline__ float knn_d2(float3 q, float4 p) {
    const float dx = __fsub_rn(p.x, q.x), dy = __fsub_rn(p.y, q.y), dz = __fsub_rn(p.z, q.z);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}
// lower bound of knn_d2 from q to any point of the AABB {lo[3], hi[3]}
__device__ __forceinline__ float knn_box_d2(float3 q, const float* lo, const float* hi) {
    const float gx = fmaxf(fmaxf(__fsub_rn(lo[0], q.x), __fsub_rn(q.x, hi[0])), 0.f);
    const float gy = fmaxf(fmaxf(__fsub_rn(lo[1], q.y), __fsub_rn(q.y, hi[1])), 0.f);
    const float gz = fmaxf(fmaxf(__fsub_rn(lo[2], q.z), __fsub_rn(q.z, hi[2])), 0.f);
    return __fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), __fmul_rn(gz, gz));
}
__device__ __forceinline__ bool knn_less(float da, uint32_t ia, float db, uint32_t ib) { return da < db || (da == db && ia < ib); }

// Ascending (distance, index) list of the K best, held in registers (every index is a compile-time constant after unrolling).
// The first KCAP - K slots are sentinels at distance -1 that no insertion passes, so the K-th best is always slot KCAP - 1.
template <int KCAP>
struct KnnTopK {
    float d[KCAP];
    uint32_t i[KCAP];
    __device__ __forceinline__ void reset(int K) {
#pragma unroll
        for (int j = 0; j < KCAP; j++) {
            d[j] = j < KCAP - K ? -1.f : INFINITY;
            i[j] = 0xffffffffu;
        }
    }
    __device__ __forceinline__ float kth() const { return d[KCAP - 1]; }
    __device__ __forceinline__ void insert(float dd, uint32_t ii) {
        if (!knn_less(dd, ii, d[KCAP - 1], i[KCAP - 1])) return;
        d[KCAP - 1] = dd;
        i[KCAP - 1] = ii;
#pragma unroll
        for (int j = KCAP - 1; j > 0; j--) {
            if (!knn_less(d[j], i[j], d[j - 1], i[j - 1])) break;
            const float td = d[j]; d[j] = d[j - 1]; d[j - 1] = td;
            const uint32_t ti = i[j]; i[j] = i[j - 1]; i[j - 1] = ti;
        }
    }
};

// One CTA per KNN_QCTA Morton-consecutive queries, as k_knn_search.  SELF: the queries are the points (qsorted == sorted) and the
// seed is the K-th best of the +-K Morton neighbours, the query included.  Otherwise the queries are Morton-sorted over the same
// box and the seed is the K-th best of the 2K points around the query's code in the points' sorted codes (P2 >= K: K exist).
template <int KCAP, bool SELF>
__global__ void __launch_bounds__(KNN_QCTA) k_knn_topk(int P1, int P2, int K, const float4* __restrict__ qsorted,
                                                       const uint32_t* __restrict__ qcodes, const float4* __restrict__ sorted,
                                                       const uint32_t* __restrict__ pcodes, const float* __restrict__ boxes,
                                                       const float* __restrict__ subboxes, int nboxes, float* __restrict__ out_d,
                                                       int64_t* __restrict__ out_i) {
    __shared__ float s_red[KNN_QCTA / 32][7];
    __shared__ float s_q[7];  // the CTA's query AABB and its largest seed bound
    __shared__ uint32_t s_cand[KNN_MAXC];
    __shared__ uint32_t s_ncand;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int q = blockIdx.x * KNN_QCTA + tid;
    const bool valid = q < P1;
    float3 pt = {0, 0, 0};
    uint32_t orig = 0;
    float reject = 0.f;
    KnnTopK<KCAP> top;
    if (valid) {
        const float4 me = qsorted[q];
        pt = make_float3(me.x, me.y, me.z);
        orig = __float_as_uint(me.w);
        int lo, hi;
        if (SELF) {
            lo = max(0, q - K);
            hi = min(P2, q + K + 1);
        } else {
            const uint32_t code = qcodes[q];
            int a = 0, b = P2;  // lower bound of the query's code
            while (a < b) {
                const int m = (a + b) >> 1;
                if (pcodes[m] < code) a = m + 1; else b = m;
            }
            lo = max(0, min(a - K, P2 - 2 * K));
            hi = min(P2, lo + 2 * K);
        }
        top.reset(K);
        for (int i = lo; i < hi; i++) {
            const float4 p = sorted[i];
            top.insert(knn_d2(pt, p), __float_as_uint(p.w));
        }
        reject = top.kth();
    }
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
    // candidate boxes: box-to-box bound (same rounding, so it bounds every query's point bound from below) within the largest seed
    for (int b = tid; b < nboxes; b += KNN_QCTA) {
        const float* bx = boxes + 6 * (size_t)b;
        const float gx = fmaxf(fmaxf(__fsub_rn(bx[0], s_q[3]), __fsub_rn(s_q[0], bx[3])), 0.f);
        const float gy = fmaxf(fmaxf(__fsub_rn(bx[1], s_q[4]), __fsub_rn(s_q[1], bx[4])), 0.f);
        const float gz = fmaxf(fmaxf(__fsub_rn(bx[2], s_q[5]), __fsub_rn(s_q[2], bx[5])), 0.f);
        if (__fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), __fmul_rn(gz, gz)) <= s_q[6]) {
            const uint32_t slot = atomicAdd(&s_ncand, 1u);
            if (slot < KNN_MAXC) s_cand[slot] = (uint32_t)b;
        }
    }
    __syncthreads();
    const uint32_t nlisted = s_ncand;
    const bool all_boxes = nlisted > KNN_MAXC;  // far queries, thousands of coincident points: test every box
    const int ncand = all_boxes ? nboxes : (int)nlisted;
    if (!valid) return;
    top.reset(K);
    for (int c = 0; c < ncand; c++) {
        const int b = all_boxes ? c : (int)s_cand[c];
        const float* bx = boxes + 6 * (size_t)b;
        const float db = knn_box_d2(pt, bx, bx + 3);
        if (db > reject || db > top.kth()) continue;
        const int sb0 = b * (KNN_BOX / KNN_SUB);
        for (int sidx = sb0; sidx < sb0 + KNN_BOX / KNN_SUB; sidx++) {
            const int i0 = sidx * KNN_SUB;
            if (i0 >= P2) break;
            const float* sbx = subboxes + 6 * (size_t)sidx;
            const float ds = knn_box_d2(pt, sbx, sbx + 3);
            if (ds > reject || ds > top.kth()) continue;
            const int i1 = min(P2, i0 + KNN_SUB);
            for (int i = i0; i < i1; i++) {
                const float4 p = sorted[i];
                const float d = knn_d2(pt, p);
                if (d <= reject) top.insert(d, __float_as_uint(p.w));  // beyond the seed bound a point cannot rank in the K best
            }
        }
    }
    const size_t row = (size_t)orig * K;
#pragma unroll
    for (int j = 0; j < KCAP; j++)
        if (j >= KCAP - K) {
            out_d[row + (j - (KCAP - K))] = top.d[j];
            out_i[row + (j - (KCAP - K))] = (int64_t)top.i[j];
        }
}

// Morton-sort P points of `pts` over the box in `bbox` with the layout L at `w`: afterwards L.codes0 holds the sorted codes and
// L.sorted the points as float4 (x, y, z, original index).
static void knn_morton_sort(int P, const float* pts, const uint32_t* bbox, char* w, const KnnLayout& L, cudaStream_t st) {
    uint32_t *k0 = (uint32_t*)(w + L.codes0), *k1 = (uint32_t*)(w + L.codes1), *v0 = (uint32_t*)(w + L.idx0), *v1 = (uint32_t*)(w + L.idx1);
    uint32_t* hist = (uint32_t*)(w + L.hist);
    k_morton<<<(P + 255) / 256, 256, 0, st>>>(P, pts, bbox, k0, v0);
    const int rs_blocks = (L.nchunks + RS_WARPS - 1) / RS_WARPS;
    for (int pass = 0; pass < 4; pass++) {  // an even number of passes: the result ends in codes0 / idx0
        k_rs_hist<<<rs_blocks, RS_WARPS * 32, 0, st>>>(P, k0, pass * 8, L.nchunks, hist);
        k_rs_scan<<<1, 1024, 0, st>>>(hist, 256 * L.nchunks);
        k_rs_scatter<<<rs_blocks, RS_WARPS * 32, 0, st>>>(P, k0, v0, pass * 8, L.nchunks, hist, k1, v1);
        uint32_t* t = k0; k0 = k1; k1 = t;
        t = v0; v0 = v1; v1 = t;
    }
    k_gather_sorted<<<(P + 255) / 256, 256, 0, st>>>(P, pts, v0, (float4*)(w + L.sorted));
}

template <int KCAP>
static void knn_launch(bool self, int P1, int P2, int K, const float4* qsorted, const uint32_t* qcodes, const float4* sorted,
                       const uint32_t* pcodes, const float* boxes, const float* subboxes, int nboxes, float* out_d, int64_t* out_i,
                       cudaStream_t st) {
    const int grid = (P1 + KNN_QCTA - 1) / KNN_QCTA;
    if (self)
        k_knn_topk<KCAP, true><<<grid, KNN_QCTA, 0, st>>>(P1, P2, K, qsorted, qcodes, sorted, pcodes, boxes, subboxes, nboxes, out_d, out_i);
    else
        k_knn_topk<KCAP, false><<<grid, KNN_QCTA, 0, st>>>(P1, P2, K, qsorted, qcodes, sorted, pcodes, boxes, subboxes, nboxes, out_d, out_i);
}

}  // namespace gsr

using namespace gsr;

size_t gsr_dist2_bytes(int32_t P) { return KnnLayout((size_t)(P < 0 ? 0 : P)).total; }

int gsr_dist2(int32_t P, const float* points, float* out, void* ws, size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_dist2");
    const cudaStream_t st = (cudaStream_t)stream;
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

// the points' layout, then (general queries only) the queries' layout; the workspace does not depend on K
size_t gsr_knn_bytes(int32_t P1, int32_t P2, int32_t K) {
    (void)K;
    return KnnLayout((size_t)max(P2, 0)).total + KnnLayout((size_t)max(P1, 0)).total;
}

int gsr_knn(int32_t P1, int32_t P2, int32_t K, const float* queries, const float* points, float* out_d, int64_t* out_i, void* ws,
            size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_knn");
    const cudaStream_t st = (cudaStream_t)stream;
    if (P1 < 0 || P2 < 0) { set_error("gsr_knn: negative size (P1 = %d, P2 = %d)", P1, P2); return GSR_ERR_INVALID; }
    if (K < 1 || K > KNN_KMAX) { set_error("gsr_knn: K = %d outside 1..%d", K, KNN_KMAX); return GSR_ERR_INVALID; }
    if (K > P2) { set_error("gsr_knn: K = %d > P2 = %d", K, P2); return GSR_ERR_INVALID; }
    if (!queries && P1 != P2) { set_error("gsr_knn: queries == NULL needs P1 == P2 (%d != %d)", P1, P2); return GSR_ERR_INVALID; }
    if (P1 == 0) return GSR_OK;
    if (!points || !out_d || !out_i) { set_error("gsr_knn: null pointer"); return GSR_ERR_INVALID; }
    const KnnLayout L((size_t)P2);
    const size_t need = L.total + (queries ? KnnLayout((size_t)P1).total : 0);
    if (!ws || ws_bytes < need) { set_error("gsr_knn: workspace too small (%zu < %zu)", ws_bytes, need); return GSR_ERR_WORKSPACE; }
    char* w = (char*)ws;
    uint32_t* bbox = (uint32_t*)(w + L.bbox);
    float* boxes = (float*)(w + L.boxes);
    float* subboxes = (float*)(w + L.subboxes);
    const float4* sorted = (const float4*)(w + L.sorted);
    // one box over both clouds (the atomics take the union), so every query's Morton coordinates lie in [0, 1023] as well
    k_bbox_init<<<1, 32, 0, st>>>(bbox);
    k_bbox<<<min(132 * 8, (P2 + 255) / 256), 256, 0, st>>>(P2, points, bbox);
    if (queries) k_bbox<<<min(132 * 8, (P1 + 255) / 256), 256, 0, st>>>(P1, queries, bbox);
    knn_morton_sort(P2, points, bbox, w, L, st);
    k_box_minmax<<<L.nboxes, 512, 0, st>>>(P2, sorted, boxes, subboxes);
    const float4* qsorted = sorted;
    const uint32_t* qcodes = (const uint32_t*)(w + L.codes0);
    if (queries) {
        const KnnLayout QL((size_t)P1);
        char* qw = w + L.total;
        knn_morton_sort(P1, queries, bbox, qw, QL, st);
        qsorted = (const float4*)(qw + QL.sorted);
        qcodes = (const uint32_t*)(qw + QL.codes0);
    }
    const uint32_t* pcodes = (const uint32_t*)(w + L.codes0);
    const bool self = queries == nullptr;
    if (K <= 4) knn_launch<4>(self, P1, P2, K, qsorted, qcodes, sorted, pcodes, boxes, subboxes, L.nboxes, out_d, out_i, st);
    else if (K <= 8) knn_launch<8>(self, P1, P2, K, qsorted, qcodes, sorted, pcodes, boxes, subboxes, L.nboxes, out_d, out_i, st);
    else if (K <= 16) knn_launch<16>(self, P1, P2, K, qsorted, qcodes, sorted, pcodes, boxes, subboxes, L.nboxes, out_d, out_i, st);
    else knn_launch<32>(self, P1, P2, K, qsorted, qcodes, sorted, pcodes, boxes, subboxes, L.nboxes, out_d, out_i, st);
    return check_launch("gsr_knn", false, st);
}
