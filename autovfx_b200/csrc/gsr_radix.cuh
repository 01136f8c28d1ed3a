// gsr_b200 — the library's stable LSD radix sort of (uint32 key, uint32 value) pairs, 8-bit digits, one warp per chunk of
// RS_CHUNK consecutive keys (warp match_any ranking), and a multi-CTA exclusive scan of uint32 counts.  gsr_knn / gsr_dist2 sort
// Morton codes with it; the deterministic SuGaR backwards (gsr_sugar_field.cu, gsr_sugar_sample.cu) group partial ids by Gaussian.
// Internal linkage, as k_rs_scan: each translation unit has its own copy.
#pragma once
#include "gsr_common.cuh"

namespace gsr {
namespace {

constexpr int RS_CHUNK = 2048;  // keys per warp
constexpr int RS_WARPS = 4;

// hist[d * nchunks + chunk] = the number of keys of the chunk whose digit at `shift` is d (column-major: an exclusive scan of the
// whole table gives every (digit, chunk) its first output position)
__global__ void __launch_bounds__(RS_WARPS * 32) k_rs_hist(uint32_t n, const uint32_t* __restrict__ keys, int shift, int nchunks,
                                                           uint32_t* __restrict__ hist) {
    __shared__ uint32_t cnt[RS_WARPS][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int chunk = blockIdx.x * RS_WARPS + warp;
    for (int d = lane; d < 256; d += 32) cnt[warp][d] = 0;
    __syncwarp();
    if (chunk < nchunks) {
        const size_t b = (size_t)chunk * RS_CHUNK, e = min((size_t)n, b + RS_CHUNK);
        for (size_t i = b + lane; i < e; i += 32) atomicAdd(&cnt[warp][(keys[i] >> shift) & 255u], 1u);
        __syncwarp();
        for (int d = lane; d < 256; d += 32) hist[(size_t)d * nchunks + chunk] = cnt[warp][d];
    }
}

// stable scatter of one digit pass: within a chunk the keys keep their order (lanes in order, rounds in order)
__global__ void __launch_bounds__(RS_WARPS * 32) k_rs_scatter(uint32_t n, const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                                                              int shift, int nchunks, const uint32_t* __restrict__ hist,
                                                              uint32_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out) {
    __shared__ uint32_t off[RS_WARPS][256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int chunk = blockIdx.x * RS_WARPS + warp;
    if (chunk >= nchunks) return;
    for (int d = lane; d < 256; d += 32) off[warp][d] = hist[(size_t)d * nchunks + chunk];
    __syncwarp();
    const size_t b = (size_t)chunk * RS_CHUNK, e = min((size_t)n, b + RS_CHUNK);
    for (size_t i0 = b; i0 < e; i0 += 32) {
        const size_t i = i0 + lane;
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

inline int rs_chunks(size_t n) { return (int)((n + RS_CHUNK - 1) / RS_CHUNK); }

// ---- exclusive scan of n uint32 counts over many CTAs: block sums, k_rs_scan of the sums, then each block's scan plus its offset.
// Integer sums: the result does not depend on the order.
constexpr int SCAN_BLOCK = 1024;

__device__ __forceinline__ uint32_t block_excl_scan_u32(uint32_t v, uint32_t* total) {
    __shared__ uint32_t wsum[SCAN_BLOCK / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(GSR_FULL, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t s = wsum[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(GSR_FULL, s, o);
            if (lane >= o) s += t;
        }
        wsum[lane] = s;  // inclusive over the warps
    }
    __syncthreads();
    *total = wsum[SCAN_BLOCK / 32 - 1];
    return (warp ? wsum[warp - 1] : 0u) + incl - v;
}

template <bool APPLY>
__global__ void __launch_bounds__(SCAN_BLOCK) k_scan_wide(uint32_t* __restrict__ v, size_t n, uint32_t* __restrict__ part) {
    const size_t i = (size_t)blockIdx.x * SCAN_BLOCK + threadIdx.x;
    const uint32_t x = i < n ? v[i] : 0u;
    uint32_t total;
    const uint32_t ex = block_excl_scan_u32(x, &total);
    if (!APPLY) {
        if (threadIdx.x == 0) part[blockIdx.x] = total;
    } else if (i < n) {
        v[i] = part[blockIdx.x] + ex;
    }
}

inline size_t scan_parts(size_t n) { return (n + SCAN_BLOCK - 1) / SCAN_BLOCK; }

// v[0..n) -> its exclusive scan in place; `part` holds scan_parts(n) entries
inline void scan_wide(uint32_t* v, size_t n, uint32_t* part, cudaStream_t st) {
    const size_t nb = scan_parts(n);
    if (nb == 0) return;
    k_scan_wide<false><<<(unsigned)nb, SCAN_BLOCK, 0, st>>>(v, n, part);
    k_rs_scan<uint32_t><<<1, 1024, 0, st>>>(part, (int)nb);
    k_scan_wide<true><<<(unsigned)nb, SCAN_BLOCK, 0, st>>>(v, n, part);
}

// ---- grouping of M partial ids by target Gaussian (the deterministic SuGaR backwards).  The emission kernel writes keys0[id] (the
// target Gaussian, or the sentinel P where the id adds nothing) and vals0[id] = id.  A stable sort on the low ceil(log2(P + 1)) bits
// then lists every Gaussian's ids in ascending order, and seg[g] .. seg[g + 1] (g < P) is Gaussian g's range of the sorted ids.
struct GroupLayout {
    size_t keys0, keys1, vals0, vals1, hist, part, seg, total;
    int nchunks, bits;
    GroupLayout(size_t M, int P) {
        nchunks = rs_chunks(M);
        bits = 0;
        while (bits < 32 && ((uint64_t)P >> bits) != 0) bits++;
        const size_t nhist = 256 * (size_t)nchunks, nseg = (size_t)P + 1;
        size_t o = 0;
        keys0 = o; o = align_up(o + 4 * M, 256);
        keys1 = o; o = align_up(o + 4 * M, 256);
        vals0 = o; o = align_up(o + 4 * M, 256);
        vals1 = o; o = align_up(o + 4 * M, 256);
        hist = o;  o = align_up(o + 4 * nhist, 256);
        part = o;  o = align_up(o + 4 * scan_parts(nhist > nseg ? nhist : nseg), 256);
        seg = o;   o = align_up(o + 4 * nseg, 256);
        total = o;
    }
};

__global__ void __launch_bounds__(256) k_seg_count(uint32_t M, const uint32_t* __restrict__ keys, uint32_t* __restrict__ seg) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < M) atomicAdd(seg + keys[i], 1u);  // integer counts: the order of the adds does not matter
}

// Sorts the emitted (key, id) pairs and builds seg; returns the sorted ids (vals0 or vals1 of the layout, by the pass count).
inline const uint32_t* group_ids(size_t M, int P, char* w, const GroupLayout& L, cudaStream_t st) {
    uint32_t *k0 = (uint32_t*)(w + L.keys0), *k1 = (uint32_t*)(w + L.keys1), *v0 = (uint32_t*)(w + L.vals0), *v1 = (uint32_t*)(w + L.vals1);
    uint32_t *hist = (uint32_t*)(w + L.hist), *part = (uint32_t*)(w + L.part), *seg = (uint32_t*)(w + L.seg);
    const int rs_blocks = (L.nchunks + RS_WARPS - 1) / RS_WARPS;
    for (int shift = 0; shift < L.bits; shift += 8) {
        k_rs_hist<<<rs_blocks, RS_WARPS * 32, 0, st>>>((uint32_t)M, k0, shift, L.nchunks, hist);
        scan_wide(hist, 256 * (size_t)L.nchunks, part, st);
        k_rs_scatter<<<rs_blocks, RS_WARPS * 32, 0, st>>>((uint32_t)M, k0, v0, shift, L.nchunks, hist, k1, v1);
        uint32_t* t = k0; k0 = k1; k1 = t;
        t = v0; v0 = v1; v1 = t;
    }
    cudaMemsetAsync(seg, 0, 4 * ((size_t)P + 1), st);
    k_seg_count<<<(unsigned)((M + 255) / 256), 256, 0, st>>>((uint32_t)M, k0, seg);
    scan_wide(seg, (size_t)P + 1, part, st);
    return v0;
}

}  // namespace
}  // namespace gsr
