// Scoring of extract_object's candidate Gaussian subsets (extract/extract_object.py:195-221, :314-340): per ratio the reference
// deep-copies the model, boolean-indexes it, renders every tracked view and counts (alpha >= 0.8) XOR (mask == 255) in numpy.
//   k_sel_count / k_rs_scan / k_sel_scatter
//                    t[keep] of means3D, opacities, scales and rotations in one scatter pass, rows in their original order
//   k_pack_masks     the tracking masks (uint8, == 255) as one bit per pixel
//   k_disagree       popcount((alpha >= thr) != maskbit) over one frame's alpha plane, one integer atomic per block
#include "gsr_common.cuh"

namespace gsr {

constexpr int SEL_THREADS = 256;
constexpr int SEL_ROUNDS = 4;  // a block selects from SEL_ROUNDS * SEL_THREADS consecutive rows
constexpr int SEL_TILE = SEL_THREADS * SEL_ROUNDS;

// Kept rows per tile; block_counts[tiles] is the scan's extra entry, which becomes the total.
__global__ void __launch_bounds__(SEL_THREADS) k_sel_count(int64_t P, const uint8_t* __restrict__ keep, uint32_t* __restrict__ block_counts,
                                                           int tiles) {
    __shared__ uint32_t warp_n[SEL_THREADS / 32];
    const int64_t base = (int64_t)blockIdx.x * SEL_TILE;
    uint32_t n = 0;
#pragma unroll
    for (int r = 0; r < SEL_ROUNDS; r++) {
        const int64_t i = base + r * SEL_THREADS + threadIdx.x;
        n += (i < P && keep[i]) ? 1u : 0u;
    }
    n = __reduce_add_sync(GSR_FULL, n);
    if ((threadIdx.x & 31) == 0) warp_n[threadIdx.x >> 5] = n;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t s = 0;
        for (int w = 0; w < SEL_THREADS / 32; w++) s += warp_n[w];
        block_counts[blockIdx.x] = s;
        if (blockIdx.x == 0) block_counts[tiles] = 0u;
    }
}

__device__ __forceinline__ void copy_row(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst, int64_t i, int64_t o, int w) {
    for (int c = 0; c < w; c++) dst[o * w + c] = src[i * w + c];
}

// Every kept row i goes to its rank among the kept rows: block offset (scanned counts) + rank inside the tile, in row order.
// Words are copied as integers, so every bit pattern (NaN payloads included) arrives unchanged, as with t[keep].
__global__ void __launch_bounds__(SEL_THREADS) k_sel_scatter(int64_t P, const uint8_t* __restrict__ keep, const uint32_t* __restrict__ offsets,
                                                             int tiles, const uint32_t* __restrict__ m, const uint32_t* __restrict__ op,
                                                             const uint32_t* __restrict__ sc, const uint32_t* __restrict__ ro,
                                                             uint32_t* __restrict__ m_out, uint32_t* __restrict__ op_out,
                                                             uint32_t* __restrict__ sc_out, uint32_t* __restrict__ ro_out,
                                                             int32_t* __restrict__ count) {
    __shared__ uint32_t warp_n[SEL_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t base = (int64_t)blockIdx.x * SEL_TILE;
    uint32_t run = offsets[blockIdx.x];
    for (int r = 0; r < SEL_ROUNDS; r++) {
        const int64_t i = base + r * SEL_THREADS + threadIdx.x;
        const bool k = i < P && keep[i];
        const unsigned bal = __ballot_sync(GSR_FULL, k);
        if (lane == 0) warp_n[warp] = __popc(bal);
        __syncthreads();
        uint32_t before = 0, total = 0;
        for (int w = 0; w < SEL_THREADS / 32; w++) {
            const uint32_t c = warp_n[w];
            before += w < warp ? c : 0u;
            total += c;
        }
        if (k) {
            const int64_t o = (int64_t)run + before + __popc(bal & ((1u << lane) - 1u));
            copy_row(m, m_out, i, o, 3);
            copy_row(op, op_out, i, o, 1);
            copy_row(sc, sc_out, i, o, 3);
            copy_row(ro, ro_out, i, o, 4);
        }
        run += total;
        __syncthreads();  // warp_n is rewritten by the next round
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *count = (int32_t)offsets[tiles];
}

// One warp per 32-pixel word: bit x & 31 of word (y, x >> 5) is mask[y, x] == 255; a row's bits past W stay 0.
__global__ void __launch_bounds__(256) k_pack_masks(int64_t words, int wpr, int W, const uint8_t* __restrict__ masks,
                                                    uint32_t* __restrict__ bits) {
    const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (wid >= words) return;  // whole warps leave together
    const int lane = threadIdx.x & 31;
    const int64_t row = wid / wpr;  // (view, y) flattened
    const int x = (int)(wid - row * wpr) * 32 + lane;
    const bool on = x < W && masks[row * W + x] == 255;
    const unsigned b = __ballot_sync(GSR_FULL, on);
    if (lane == 0) bits[wid] = b;
}

constexpr int DIS_THREADS = 256;

// count += number of pixels where (alpha >= thr) differs from the mask bit.  alpha >= thr is false for NaN, as numpy's >= is.
__global__ void __launch_bounds__(DIS_THREADS) k_disagree(int64_t words, int wpr, int W, const float* __restrict__ alpha, float thr,
                                                          const uint32_t* __restrict__ bits, unsigned long long* __restrict__ count) {
    __shared__ uint32_t warp_n[DIS_THREADS / 32];
    const int lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (DIS_THREADS / 32);
    uint32_t n = 0;
    for (int64_t wid = ((int64_t)blockIdx.x * DIS_THREADS + threadIdx.x) >> 5; wid < words; wid += warps) {
        const int64_t y = wid / wpr;
        const int x = (int)(wid - y * wpr) * 32 + lane;
        const bool in = x < W;
        const bool on = in && alpha[y * W + x] >= thr;
        const unsigned valid = __ballot_sync(GSR_FULL, in);
        const unsigned drawn = __ballot_sync(GSR_FULL, on);
        if (lane == 0) n += (uint32_t)__popc((drawn ^ bits[wid]) & valid);
    }
    if (lane == 0) warp_n[threadIdx.x >> 5] = n;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t s = 0;
        for (int w = 0; w < DIS_THREADS / 32; w++) s += warp_n[w];
        if (s) atomicAdd(count, (unsigned long long)s);
    }
}

}  // namespace gsr

using namespace gsr;

static int sel_tiles(int64_t P) { return (int)((P + SEL_TILE - 1) / SEL_TILE); }

size_t gsr_select_rows_bytes(int64_t P) {
    if (P < 0 || P > 0x7fffffffLL) return 0;
    return ((size_t)sel_tiles(P) + 1) * sizeof(uint32_t);
}

int gsr_select_rows(int64_t P, const uint8_t* keep, const float* means3D, const float* opacities, const float* scales, const float* rotations,
                    float* means3D_out, float* opacities_out, float* scales_out, float* rotations_out, int32_t* count, void* ws,
                    size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_select_rows");
    const cudaStream_t s = (cudaStream_t)stream;
    if (P < 0 || P > 0x7fffffffLL || !count) { set_error("gsr_select_rows: bad arguments (P %lld)", (long long)P); return GSR_ERR_INVALID; }
    if (P > 0 && (!keep || !means3D || !opacities || !scales || !rotations || !means3D_out || !opacities_out || !scales_out || !rotations_out)) {
        set_error("gsr_select_rows: a row array is NULL");
        return GSR_ERR_INVALID;
    }
    if (!ws || ((uintptr_t)ws & 3) || ws_bytes < gsr_select_rows_bytes(P)) {
        set_error("gsr_select_rows: workspace of %zu bytes, gsr_select_rows_bytes(%lld) = %zu needed (4-byte aligned)", ws_bytes, (long long)P,
                  gsr_select_rows_bytes(P));
        return GSR_ERR_WORKSPACE;
    }
    if (P == 0) {
        cudaMemsetAsync(count, 0, sizeof(int32_t), s);
        return check_launch("gsr_select_rows", false, s);
    }
    const int tiles = sel_tiles(P);
    uint32_t* counts = (uint32_t*)ws;
    k_sel_count<<<tiles, SEL_THREADS, 0, s>>>(P, keep, counts, tiles);
    k_rs_scan<uint32_t><<<1, 1024, 0, s>>>(counts, tiles + 1);
    k_sel_scatter<<<tiles, SEL_THREADS, 0, s>>>(P, keep, counts, tiles, (const uint32_t*)means3D, (const uint32_t*)opacities,
                                                (const uint32_t*)scales, (const uint32_t*)rotations, (uint32_t*)means3D_out,
                                                (uint32_t*)opacities_out, (uint32_t*)scales_out, (uint32_t*)rotations_out, count);
    return check_launch("gsr_select_rows", false, s);
}

int gsr_pack_masks(int32_t V, int32_t W, int32_t H, const uint8_t* masks, uint32_t* bits, void* stream) {
    NvtxRange nvtx_("gsr_pack_masks");
    const cudaStream_t s = (cudaStream_t)stream;
    if (V < 0 || W <= 0 || H <= 0 || (V > 0 && (!masks || !bits))) { set_error("gsr_pack_masks: bad arguments (V %d, %d x %d)", V, W, H); return GSR_ERR_INVALID; }
    const int wpr = (W + 31) / 32;
    const int64_t words = (int64_t)V * H * wpr;
    if (words == 0) return GSR_OK;
    k_pack_masks<<<(unsigned)((words * 32 + 255) / 256), 256, 0, s>>>(words, wpr, W, masks, bits);
    return check_launch("gsr_pack_masks", false, s);
}

int gsr_mask_disagreement(int32_t W, int32_t H, const float* alpha, const uint32_t* bits, float thr, int64_t* count, void* stream) {
    NvtxRange nvtx_("gsr_mask_disagreement");
    const cudaStream_t s = (cudaStream_t)stream;
    if (W <= 0 || H <= 0 || !alpha || !bits || !count) { set_error("gsr_mask_disagreement: bad arguments (%d x %d)", W, H); return GSR_ERR_INVALID; }
    if ((uintptr_t)count & 7) { set_error("gsr_mask_disagreement: count must be 8-byte aligned"); return GSR_ERR_INVALID; }
    const int wpr = (W + 31) / 32;
    const int64_t words = (int64_t)H * wpr;
    const int64_t want = (words + DIS_THREADS / 32 - 1) / (DIS_THREADS / 32);
    const unsigned grid = (unsigned)(want < 1024 ? want : 1024);
    k_disagree<<<grid, DIS_THREADS, 0, s>>>(words, wpr, W, alpha, thr, bits, (unsigned long long*)count);
    return check_launch("gsr_mask_disagreement", false, s);
}
