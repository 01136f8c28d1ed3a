// PNG encoding of 8-bit frames (the images, depth-colormap and normal-map files of the frame loop, and blend_frames' output):
//   k_png_filter   one CTA per scanline: the five PNG filters, libpng's heuristic (least sum of |residual| read as int8)
//   k_png_match    one CTA per 32 KiB chunk of the filtered stream: a hash chain over the chunk and the 32 KiB before it (built
//                  by one warp, 32 positions per step), then the longest match of every position (up to PNG_CHAIN candidates)
//   k_png_deflate  one CTA per chunk: greedy parse (parallel 32-byte segments joined where their paths converge), Huffman
//                  codes from the chunk's histogram, the smallest of a dynamic, fixed or stored block, bit packing, and the
//                  chunk's CRC-32 and Adler-32 sums
//   k_png_assemble one CTA per chunk copies it to its offset in the file; one CTA per image writes the signature, IHDR, the IDAT
//                  header and trailer (Adler-32 and CRC-32 combined over the chunks) and IEND, and the file size
// Every chunk but the last ends with an empty stored block (a sync flush), so the chunks are byte-aligned and concatenate.
// Matches may reach into the previous chunk.  Nothing depends on the order of atomics: the histograms are integer counts and
// the bit packing ORs disjoint bits, so the bytes depend only on the pixels and the shape.
#include <string.h>
#include "gsr_common.cuh"

namespace gsr {

constexpr int PNG_CHUNK = 32768;              // filtered bytes per deflate block
constexpr int PNG_HIST = 32768;               // deflate's window
constexpr int PNG_WIN = PNG_HIST + PNG_CHUNK; // history + chunk
constexpr int PNG_CAP = PNG_CHUNK + 256;      // scratch bytes per compressed chunk (a stored chunk takes PNG_CHUNK + 5)
constexpr int PNG_HASH_BITS = 13;
constexpr int PNG_CHAIN = 8;                  // candidates tried per position
constexpr int PNG_THREADS = 1024;
constexpr int PNG_SEG = PNG_CHUNK / PNG_THREADS;  // 32 parse positions per thread: one bit word
static_assert(PNG_SEG == 32, "one vis word per thread");
constexpr uint32_t PNG_NONE = 0xffffffffu;
constexpr int PNG_HEAD = 43;                  // signature 8 + IHDR 25 + IDAT length/type 8 + zlib header 2
constexpr int PNG_TAIL = 20;                  // Adler-32 4 + IDAT CRC 4 + IEND 12
constexpr uint32_t CRC_POLY = 0xedb88320u;

struct PngDesc {
    const uint8_t* src;
    const uint8_t* lut;
    int64_t sh, sw, sc;
    int32_t H, W, C, flags;   // C: channels in the file
    int64_t raw_off, raw_len; // the filtered stream in the workspace (also the offset of its match words)
    int64_t row_base;         // first k_png_filter block of this image
    int32_t chunk_base, nchunks;
    uint8_t* out;
    int64_t* size;
};

struct PngBatch {
    int32_t n, rows, chunks, pad_;
    uint8_t* raw;
    uint32_t* match;
    uint8_t* scratch;  // [chunks of the call, PNG_CAP]
    uint4* meta;       // per chunk: compressed bytes, CRC-32, Adler s1, Adler s2 (mod 65521)
    PngDesc d[GSR_PNG_MAX_BATCH];
};

__device__ __forceinline__ int png_image_of_chunk(const PngBatch& b, int c) {
    int i = 0;
    while (i + 1 < b.n && c >= b.d[i + 1].chunk_base) i++;
    return i;
}

// --------------------------------------------------------------------------------------------------------------- CRC-32 algebra
// Polynomials mod the CRC-32 generator, bit-reflected as zlib keeps them (x^0 is the top bit).
__device__ __host__ __forceinline__ uint32_t multmodp(uint32_t a, uint32_t b) {
    uint32_t m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ CRC_POLY : b >> 1;
    }
    return p;
}

// x^(8 n) mod p from x2n[k] = x^(2^k) mod p
__device__ __forceinline__ uint32_t x8nmodp(uint64_t n, const uint32_t* x2n) {
    uint32_t p = 1u << 31;
    int k = 3;
    while (n) {
        if (n & 1) p = multmodp(x2n[k & 31], p);
        n >>= 1;
        k++;
    }
    return p;
}

// crc32(A || B) from crc32(A), crc32(B) and |B|
__device__ __forceinline__ uint32_t crc_combine(uint32_t a, uint32_t b, uint64_t len_b, const uint32_t* x2n) {
    return multmodp(x8nmodp(len_b, x2n), a) ^ b;
}

__device__ void png_crc_tables(uint32_t* table, uint32_t* x2n) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        uint32_t c = (uint32_t)i;
        for (int k = 0; k < 8; k++) c = c & 1 ? (c >> 1) ^ CRC_POLY : c >> 1;
        table[i] = c;
    }
    if (threadIdx.x == 0) {
        uint32_t p = 1u << 30;  // x^1
        x2n[0] = p;
        for (int k = 1; k < 32; k++) x2n[k] = p = multmodp(p, p);
    }
}

__device__ __forceinline__ uint32_t crc_bytes_bitwise(uint32_t crc, const uint8_t* p, int n) {
    for (int i = 0; i < n; i++) {
        crc ^= p[i];
        for (int k = 0; k < 8; k++) crc = crc & 1 ? (crc >> 1) ^ CRC_POLY : crc >> 1;
    }
    return crc;
}

// ------------------------------------------------------------------------------------------------------------------- the filter
__device__ __forceinline__ uint32_t png_px(const PngDesc& d, int y, int j) {
    const int x = j / d.C, c = j - x * d.C;
    const uint8_t* p = d.src + (int64_t)y * d.sh + (int64_t)x * d.sw;
    if (d.lut) return d.lut[3 * (uint32_t)p[0] + c];
    const int cc = (d.flags & GSR_PNG_SWAP_RB) && c < 3 ? 2 - c : c;
    return p[(int64_t)cc * d.sc];
}

__device__ __forceinline__ uint32_t paeth(int a, int b, int c) {
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return (uint32_t)(pa <= pb && pa <= pc ? a : (pb <= pc ? b : c));
}

__global__ void __launch_bounds__(256) k_png_filter(const __grid_constant__ PngBatch b) {
    __shared__ uint32_t red[8][5];
    __shared__ int pick;
    int i = 0;
    while (i + 1 < b.n && (int64_t)blockIdx.x >= b.d[i + 1].row_base) i++;
    const PngDesc& d = b.d[i];
    const int y = (int)(blockIdx.x - d.row_base);
    const int L = d.W * d.C, bpp = d.C;
    uint32_t s[5] = {0, 0, 0, 0, 0};
    auto residuals = [&](int j, uint32_t r[5]) {
        const uint32_t x = png_px(d, y, j), a = j >= bpp ? png_px(d, y, j - bpp) : 0u;
        const uint32_t u = y > 0 ? png_px(d, y - 1, j) : 0u, c = (y > 0 && j >= bpp) ? png_px(d, y - 1, j - bpp) : 0u;
        r[0] = x & 255u;
        r[1] = (x - a) & 255u;
        r[2] = (x - u) & 255u;
        r[3] = (x - ((a + u) >> 1)) & 255u;
        r[4] = (x - paeth((int)a, (int)u, (int)c)) & 255u;
    };
    for (int j = threadIdx.x; j < L; j += 256) {
        uint32_t r[5];
        residuals(j, r);
#pragma unroll
        for (int f = 0; f < 5; f++) s[f] += (uint32_t)abs((int)(int8_t)(uint8_t)r[f]);
    }
#pragma unroll
    for (int f = 0; f < 5; f++) s[f] = __reduce_add_sync(GSR_FULL, s[f]);
    if ((threadIdx.x & 31) == 0)
        for (int f = 0; f < 5; f++) red[threadIdx.x >> 5][f] = s[f];
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t best = PNG_NONE;
        int bf = 0;
        for (int f = 0; f < 5; f++) {
            uint32_t t = 0;
            for (int w = 0; w < 8; w++) t += red[w][f];
            if (t < best) best = t, bf = f;
        }
        pick = bf;
    }
    __syncthreads();
    const int f = pick;
    uint8_t* row = b.raw + d.raw_off + (int64_t)y * (1 + L);
    if (threadIdx.x == 0) row[0] = (uint8_t)f;
    for (int j = threadIdx.x; j < L; j += 256) {
        uint32_t r[5];
        residuals(j, r);
        row[1 + j] = (uint8_t)r[f];
    }
}

// ------------------------------------------------------------------------------------------------------------ the match finder
// Match word of a position: (length << 16) | (distance - 1), 0 for a literal.
__global__ void __launch_bounds__(PNG_THREADS, 1) k_png_match(const __grid_constant__ PngBatch b) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t* win = smem;                                          // [PNG_WIN + 16]
    uint16_t* prev = (uint16_t*)(smem + PNG_WIN + 16);           // [PNG_WIN] distance to the previous same-hash position, 0 = none
    uint32_t* head = (uint32_t*)(smem + PNG_WIN + 16 + 2 * PNG_WIN);  // [1 << PNG_HASH_BITS]
    const int ci = blockIdx.x, im = png_image_of_chunk(b, ci);
    const PngDesc& d = b.d[im];
    const int j = ci - d.chunk_base;
    const int64_t c0 = (int64_t)j * PNG_CHUNK;
    const int clen = (int)min((int64_t)PNG_CHUNK, d.raw_len - c0);
    const int hist = (int)min((int64_t)PNG_HIST, c0);
    const uint8_t* src = b.raw + d.raw_off + c0 - hist;
    const int w0 = PNG_HIST - hist, wend = PNG_HIST + clen;
    for (int k = threadIdx.x; k < hist + clen; k += PNG_THREADS) win[w0 + k] = src[k];
    for (int k = threadIdx.x; k < (1 << PNG_HASH_BITS); k += PNG_THREADS) head[k] = PNG_NONE;
    __syncthreads();
    if (threadIdx.x < 32) {  // the chain: one warp, 32 consecutive positions per step, in stream order
        const int lane = threadIdx.x;
        for (int base = w0; base < wend; base += 32) {
            const int p = base + lane;
            const bool valid = p + 3 <= wend;
            const uint32_t h = valid ? ((((uint32_t)win[p] | ((uint32_t)win[p + 1] << 8) | ((uint32_t)win[p + 2] << 16)) * 2654435761u) >>
                                        (32 - PNG_HASH_BITS))
                                     : (1u << PNG_HASH_BITS) + lane;
            const unsigned peers = __match_any_sync(GSR_FULL, h);
            const unsigned lower = peers & ((1u << lane) - 1u);
            uint32_t q = PNG_NONE;
            if (valid) q = lower ? (uint32_t)(base + 31 - __clz(lower)) : head[h];
            __syncwarp();
            if (valid) {
                prev[p] = (q != PNG_NONE && (uint32_t)p - q <= (uint32_t)PNG_HIST) ? (uint16_t)((uint32_t)p - q) : (uint16_t)0;
                if (!(peers >> lane >> 1)) head[h] = (uint32_t)p;  // the last position of its hash in this step
            }
            __syncwarp();
        }
    }
    __syncthreads();
    uint32_t* mout = b.match + d.raw_off + c0;
    for (int k = threadIdx.x; k < clen; k += PNG_THREADS) {
        const int p = PNG_HIST + k;
        const int maxlen = min(258, wend - p);
        int best = 0, bd = 0;
        if (maxlen >= 3) {
            int q = p;
            for (int t = 0; t < PNG_CHAIN; t++) {
                const int dq = prev[q];
                if (dq == 0) break;
                q -= dq;
                const int dist = p - q;
                if (dist > PNG_HIST) break;
                if (win[q + best] != win[p + best]) continue;
                int l = 0;
                while (l < maxlen && win[q + l] == win[p + l]) l++;
                if (l > best) {
                    best = l, bd = dist;
                    if (l == maxlen) break;
                }
            }
        }
        mout[k] = (best >= 4 || (best == 3 && bd <= 4096)) ? ((uint32_t)best << 16) | (uint32_t)(bd - 1) : 0u;
    }
}

// --------------------------------------------------------------------------------------------------------------- Huffman codes
__device__ __forceinline__ int len_code(int len, int& ebits, int& eval) {  // 257..285
    const int v = len - 3;
    if (len == 258) { ebits = 0; eval = 0; return 285; }
    if (v < 8) { ebits = 0; eval = 0; return 257 + v; }
    const int l = 31 - __clz(v);
    ebits = l - 2;
    eval = v & ((1 << ebits) - 1);
    return 257 + 4 * (l - 1) + ((v >> (l - 2)) & 3);
}

__device__ __forceinline__ int dist_code(int dist, int& ebits, int& eval) {  // 0..29
    const int v = dist - 1;
    if (v < 4) { ebits = 0; eval = 0; return v; }
    const int l = 31 - __clz(v);
    ebits = l - 1;
    eval = v & ((1 << ebits) - 1);
    return 2 * l + ((v >> (l - 1)) & 1);
}

__device__ __forceinline__ int len_extra(int code) { return code < 265 || code == 285 ? 0 : (code - 261) / 4; }
__device__ __forceinline__ int dist_extra(int code) { return code < 4 ? 0 : code / 2 - 1; }
__device__ __forceinline__ int fixed_len(int sym) { return sym < 144 ? 8 : (sym < 256 ? 9 : (sym < 280 ? 7 : 8)); }

struct HuffScratch {
    uint32_t weight[2 * 288];
    uint16_t parent[2 * 288];
    uint16_t depth[2 * 288];
    uint16_t count[290];
};

// Code lengths (<= maxbits) of the m symbols `sorted` lists in ascending (weight, symbol) order, m >= 2: a Huffman tree by the
// two-queue method (ties take the leaf), then JPEG's Annex K.3 adjustment of the length counts, longest codes to the rarest.
__device__ void huff_build(const uint16_t* sorted, int m, const uint32_t* w, int maxbits, uint8_t* len, HuffScratch& s) {
    for (int i = 0; i < m; i++) s.weight[i] = w[sorted[i]];
    int li = 0, ii = m;
    for (int nid = m; nid < 2 * m - 1; nid++) {
        int pick[2];
        for (int k = 0; k < 2; k++) {
            if (li < m && (ii >= nid || s.weight[li] <= s.weight[ii])) pick[k] = li++;
            else pick[k] = ii++;
        }
        s.weight[nid] = s.weight[pick[0]] + s.weight[pick[1]];
        s.parent[pick[0]] = s.parent[pick[1]] = (uint16_t)nid;
    }
    s.depth[2 * m - 2] = 0;
    int maxd = 0;
    for (int k = 0; k <= 288; k++) s.count[k] = 0;
    for (int nd = 2 * m - 3; nd >= 0; nd--) {
        s.depth[nd] = s.depth[s.parent[nd]] + 1;
        if (nd < m) {
            s.count[s.depth[nd]]++;
            maxd = max(maxd, (int)s.depth[nd]);
        }
    }
    for (int i = maxd; i > maxbits; i--) {
        while (s.count[i] > 0) {
            int j = i - 2;
            while (s.count[j] == 0) j--;
            s.count[i] -= 2;
            s.count[i - 1] += 1;
            s.count[j + 1] += 2;
            s.count[j] -= 1;
        }
    }
    int k = 0;
    for (int l = min(maxd, maxbits); l >= 1; l--)
        for (int c = 0; c < s.count[l]; c++) len[sorted[k++]] = (uint8_t)l;
}

// Canonical codes, bit-reversed for deflate's LSB-first packing.  `more8` counts 8-bit codes of symbols past n (the fixed
// literal/length code defines 286 and 287, which never occur but take their places in the canonical order).
__device__ void huff_codes(const uint8_t* len, int n, uint16_t* code, int more8 = 0) {
    uint16_t cnt[16] = {0}, next[16];
    for (int i = 0; i < n; i++) cnt[len[i]]++;
    cnt[8] += more8;
    cnt[0] = 0;
    uint32_t c = 0;
    for (int l = 1; l < 16; l++) {
        c = (c + cnt[l - 1]) << 1;
        next[l] = (uint16_t)c;
    }
    for (int i = 0; i < n; i++)
        code[i] = len[i] ? (uint16_t)(__brev((uint32_t)next[len[i]]++) >> (32 - len[i])) : (uint16_t)0;
}

// ------------------------------------------------------------------------------------------------------------------ the deflater
struct DeflateShared {
    uint32_t match[PNG_CHUNK];
    uint32_t out[(PNG_CAP) / 4];
    uint8_t data[PNG_CHUNK];
    uint32_t vis[PNG_THREADS];  // bit k of word t: position 32 t + k starts a token
    uint32_t exitp[PNG_THREADS];
    uint32_t freq[286 + 30];    // literal/length then distance counts
    uint32_t wgt[286 + 30];     // counts used for the codes (absent symbols forced in where fewer than two are used)
    uint16_t sorted_ll[286], sorted_d[30];
    uint8_t len[286 + 30];
    uint16_t code[286 + 30];
    uint8_t cl_len[19];
    uint16_t cl_code[19];
    uint8_t rle_sym[286 + 30], rle_ext[286 + 30];
    HuffScratch hs[2];
    uint32_t crc_table[256], x2n[32];
    uint32_t scan[32];
    uint64_t red[32][2];
    int mode, n_rle, hlit, hdist, hclen;
    uint32_t hdr_bits, data_bits, total_bytes;
};
constexpr int PNG_MATCH_SMEM = PNG_WIN + 16 + 2 * PNG_WIN + 4 * (1 << PNG_HASH_BITS);
static_assert(sizeof(DeflateShared) <= 232448 && PNG_MATCH_SMEM <= 232448, "one CTA per SM of shared memory");

__device__ __forceinline__ void put_bits(uint32_t* out, uint32_t pos, uint32_t v, int n) {
    if (!n) return;
    const uint64_t x = (uint64_t)v << (pos & 31);
    atomicOr(&out[pos >> 5], (uint32_t)x);
    if (x >> 32) atomicOr(&out[(pos >> 5) + 1], (uint32_t)(x >> 32));
}

__device__ __forceinline__ int step_at(const uint32_t* match, int p) {
    const uint32_t m = match[p];
    return m ? (int)(m >> 16) : 1;
}

__constant__ uint8_t CL_ORDER[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

__global__ void __launch_bounds__(PNG_THREADS, 1) k_png_deflate(const __grid_constant__ PngBatch b) {
    extern __shared__ __align__(16) uint8_t smem[];
    DeflateShared& S = *(DeflateShared*)smem;
    const int tid = threadIdx.x, ci = blockIdx.x, im = png_image_of_chunk(b, ci);
    const PngDesc& d = b.d[im];
    const int j = ci - d.chunk_base;
    const bool final_ = j == d.nchunks - 1;
    const int64_t c0 = (int64_t)j * PNG_CHUNK;
    const int clen = (int)min((int64_t)PNG_CHUNK, d.raw_len - c0);
    const uint32_t* msrc = b.match + d.raw_off + c0;
    const uint8_t* dsrc = b.raw + d.raw_off + c0;
    for (int k = tid; k < clen; k += PNG_THREADS) {
        S.match[k] = msrc[k];
        S.data[k] = dsrc[k];
    }
    for (int k = tid; k < PNG_CAP / 4; k += PNG_THREADS) S.out[k] = 0u;
    for (int k = tid; k < 286 + 30; k += PNG_THREADS) S.freq[k] = 0u;
    png_crc_tables(S.crc_table, S.x2n);
    __syncthreads();

    // greedy parse: every thread walks its 32 positions from the segment's start ...
    const int nseg = (clen + 31) / 32;
    {
        const int s = 32 * tid, e = min(s + 32, clen);
        uint32_t word = 0;
        int p = s;
        while (p < e) {
            word |= 1u << (p - s);
            p += step_at(S.match, p);
        }
        S.vis[tid] = word;
        S.exitp[tid] = (uint32_t)p;
    }
    __syncthreads();
    // ... then one thread follows the true path from position 0, re-walking a segment only until it meets that segment's own path
    if (tid == 0) {
        int entry = 0;
        for (int t = 0; t < nseg; t++) {
            const int s = 32 * t, e = min(s + 32, clen);
            if (entry == s) {
                entry = (int)S.exitp[t];
                continue;
            }
            const uint32_t old = S.vis[t];
            if (entry >= e) {  // a match from an earlier segment covers this one
                S.vis[t] = 0u;
                continue;
            }
            uint32_t word = 0;
            int p = entry;
            while (p < e && !((old >> (p - s)) & 1u)) {
                word |= 1u << (p - s);
                p += step_at(S.match, p);
            }
            if (p < e) {  // converged at p: keep the old path from p on
                S.vis[t] = word | (old & (0xffffffffu << (p - s)));
                entry = (int)S.exitp[t];
            } else {
                S.vis[t] = word;
                entry = p;
            }
        }
    }
    __syncthreads();

    // histogram (integer counts) and the extra bits, the same for every block type
    uint32_t extra = 0;
    if (tid < nseg) {
        uint32_t w = S.vis[tid];
        while (w) {
            const int p = 32 * tid + __ffs(w) - 1;
            w &= w - 1;
            const uint32_t m = S.match[p];
            if (!m) {
                atomicAdd(&S.freq[S.data[p]], 1u);
            } else {
                int eb, ev, db, dv;
                const int lc = len_code((int)(m >> 16), eb, ev), dc = dist_code((int)(m & 0xffffu) + 1, db, dv);
                atomicAdd(&S.freq[lc], 1u);
                atomicAdd(&S.freq[286 + dc], 1u);
                extra += eb + db;
            }
        }
    }
    extra = __reduce_add_sync(GSR_FULL, extra);
    if ((tid & 31) == 0) S.scan[tid >> 5] = extra;
    if (tid == 0) S.freq[256] = 1u;  // end of block
    __syncthreads();
    // code weights: at least two symbols per alphabet, so that every code is complete
    if (tid < 32) {
        const int lane = tid;
        uint32_t cnt_ll = 0, cnt_d = 0;
        for (int k = lane; k < 286; k += 32) cnt_ll += S.freq[k] != 0;
        for (int k = lane; k < 30; k += 32) cnt_d += S.freq[286 + k] != 0;
        cnt_ll = __reduce_add_sync(GSR_FULL, cnt_ll);
        cnt_d = __reduce_add_sync(GSR_FULL, cnt_d);
        for (int k = lane; k < 316; k += 32) {
            uint32_t f = S.freq[k];
            if (!f && k < 286 && cnt_ll < 2 && k == 0) f = 1;
            if (!f && k >= 286 && cnt_d < 2 && (k == 286 || (k == 287 && (cnt_d == 0 || S.freq[286] != 0)))) f = 1;
            S.wgt[k] = f;
        }
        if (lane == 0) {
            uint32_t x = 0;
            for (int w = 0; w < 32; w++) x += S.scan[w];
            S.data_bits = x;  // the extra bits for now
        }
    }
    __syncthreads();
    // ascending (weight, symbol) order of the used symbols, by rank
    if (tid < 286 + 30) {
        const bool ll = tid < 286;
        const int lo = ll ? 0 : 286, hi = ll ? 286 : 316;
        const uint32_t w = S.wgt[tid];
        if (w) {
            int r = 0;
            for (int k = lo; k < hi; k++) {
                const uint32_t v = S.wgt[k];
                r += v && (v < w || (v == w && k < tid));
            }
            if (ll) S.sorted_ll[r] = (uint16_t)tid;
            else S.sorted_d[r] = (uint16_t)(tid - 286);
        }
        S.len[tid] = 0;
    }
    __syncthreads();
    if (tid == 0 || tid == 32) {
        const bool ll = tid == 0;
        const int lo = ll ? 0 : 286, n = ll ? 286 : 30;
        int m = 0;
        for (int k = 0; k < n; k++) m += S.wgt[lo + k] != 0;
        huff_build(ll ? S.sorted_ll : S.sorted_d, m, S.wgt + lo, 15, S.len + lo, S.hs[ll ? 0 : 1]);
    }
    __syncthreads();

    if (tid == 0) {
        const uint32_t xbits = S.data_bits;
        int hlit = 286, hdist = 30;
        while (hlit > 257 && !S.len[hlit - 1]) hlit--;
        while (hdist > 1 && !S.len[286 + hdist - 1]) hdist--;
        // run-length code of the code lengths (literal/length then distance, one sequence)
        uint8_t seq[316];
        int n = 0;
        for (int k = 0; k < hlit; k++) seq[n++] = S.len[k];
        for (int k = 0; k < hdist; k++) seq[n++] = S.len[286 + k];
        int nr = 0;
        uint32_t clf[19] = {0};
        for (int i = 0; i < n;) {
            const int v = seq[i];
            int run = 1;
            while (i + run < n && seq[i + run] == v) run++;
            int r = run;
            if (v == 0) {
                while (r >= 11) {
                    const int k = min(r, 138);
                    S.rle_sym[nr] = 18, S.rle_ext[nr++] = (uint8_t)(k - 11), clf[18]++;
                    r -= k;
                }
                if (r >= 3) {
                    S.rle_sym[nr] = 17, S.rle_ext[nr++] = (uint8_t)(r - 3), clf[17]++;
                    r = 0;
                }
                for (; r > 0; r--) S.rle_sym[nr] = 0, S.rle_ext[nr++] = 0, clf[0]++;
            } else {
                S.rle_sym[nr] = (uint8_t)v, S.rle_ext[nr++] = 0, clf[v]++;
                r--;
                while (r >= 3) {
                    const int k = min(r, 6);
                    S.rle_sym[nr] = 16, S.rle_ext[nr++] = (uint8_t)(k - 3), clf[16]++;
                    r -= k;
                }
                for (; r > 0; r--) S.rle_sym[nr] = (uint8_t)v, S.rle_ext[nr++] = 0, clf[v]++;
            }
            i += run;
        }
        // the code-length code (7 bits), insertion-sorted: 19 symbols
        uint32_t clw[19];
        int used = 0;
        for (int k = 0; k < 19; k++) used += clf[k] != 0;
        for (int k = 0; k < 19; k++) clw[k] = clf[k] ? clf[k] : (used < 2 && (k == 0 || k == 1) ? 1u : 0u);
        uint16_t srt[19];
        int m = 0;
        for (int k = 0; k < 19; k++) {
            if (!clw[k]) continue;
            int pos = m++;
            while (pos > 0 && clw[srt[pos - 1]] > clw[k]) {
                srt[pos] = srt[pos - 1];
                pos--;
            }
            srt[pos] = (uint16_t)k;
        }
        for (int k = 0; k < 19; k++) S.cl_len[k] = 0;
        huff_build(srt, m, clw, 7, S.cl_len, S.hs[0]);
        int hclen = 19;
        while (hclen > 4 && !S.cl_len[CL_ORDER[hclen - 1]]) hclen--;
        uint64_t hdr = 3 + 14 + 3 * hclen;
        for (int k = 0; k < nr; k++) {
            const int sy = S.rle_sym[k];
            hdr += S.cl_len[sy] + (sy == 16 ? 2 : sy == 17 ? 3 : sy == 18 ? 7 : 0);
        }
        uint64_t dyn = xbits, fix = xbits;
        for (int k = 0; k < 286; k++) {
            dyn += (uint64_t)S.freq[k] * S.len[k];
            fix += (uint64_t)S.freq[k] * fixed_len(k);
        }
        for (int k = 0; k < 30; k++) {
            dyn += (uint64_t)S.freq[286 + k] * S.len[286 + k];
            fix += (uint64_t)S.freq[286 + k] * 5;
        }
        const uint32_t flush_bits = final_ ? 0u : 3u, flush_bytes = final_ ? 0u : 4u;
        const uint32_t bytes_dyn = (uint32_t)((hdr + dyn + flush_bits + 7) / 8) + flush_bytes;
        const uint32_t bytes_fix = (uint32_t)((3 + fix + flush_bits + 7) / 8) + flush_bytes;
        const uint32_t bytes_st = 5u + (uint32_t)clen;
        int mode = 2;  // dynamic
        uint32_t best = bytes_dyn;
        if (bytes_fix < best) mode = 1, best = bytes_fix;
        if (bytes_st < best) mode = 0, best = bytes_st;
        S.mode = mode;
        S.total_bytes = best;
        S.hlit = hlit, S.hdist = hdist, S.hclen = hclen, S.n_rle = nr;
        if (mode == 1) {
            for (int k = 0; k < 286; k++) S.len[k] = (uint8_t)fixed_len(k);
            for (int k = 0; k < 30; k++) S.len[286 + k] = 5;
        }
        if (mode) {
            huff_codes(S.len, 286, S.code, mode == 1 ? 2 : 0);
            huff_codes(S.len + 286, 30, S.code + 286);
            uint32_t pos = 0;
            put_bits(S.out, pos, (final_ ? 1u : 0u) | ((uint32_t)mode << 1), 3);
            pos += 3;
            if (mode == 2) {
                huff_codes(S.cl_len, 19, S.cl_code);
                put_bits(S.out, pos, hlit - 257, 5), pos += 5;
                put_bits(S.out, pos, hdist - 1, 5), pos += 5;
                put_bits(S.out, pos, hclen - 4, 4), pos += 4;
                for (int k = 0; k < hclen; k++) put_bits(S.out, pos, S.cl_len[CL_ORDER[k]], 3), pos += 3;
                for (int k = 0; k < nr; k++) {
                    const int sy = S.rle_sym[k];
                    put_bits(S.out, pos, S.cl_code[sy], S.cl_len[sy]), pos += S.cl_len[sy];
                    const int eb = sy == 16 ? 2 : sy == 17 ? 3 : sy == 18 ? 7 : 0;
                    put_bits(S.out, pos, S.rle_ext[k], eb), pos += eb;
                }
            }
            S.hdr_bits = pos;
            const uint32_t data_end = pos + (uint32_t)(mode == 2 ? dyn : fix);
            const uint32_t eob = data_end - S.len[256];
            put_bits(S.out, eob, S.code[256], S.len[256]);
            if (!final_) {  // sync flush: an empty stored block after a 3-bit header, LEN 0000, NLEN ffff
                const uint32_t nb = (data_end + 3 + 7) / 8;
                put_bits(S.out, (nb + 2) * 8, 0xffffu, 16);
            }
        }
    }
    __syncthreads();
    const int mode = S.mode;
    if (mode) {
        // bits of each segment's tokens, an exclusive scan over the block, then the tokens
        uint32_t nbits = 0;
        const uint32_t w0 = tid < nseg ? S.vis[tid] : 0u;
        for (uint32_t w = w0; w; w &= w - 1) {
            const int p = 32 * tid + __ffs(w) - 1;
            const uint32_t m = S.match[p];
            if (!m) {
                nbits += S.len[S.data[p]];
            } else {
                int eb, ev, db, dv;
                const int lc = len_code((int)(m >> 16), eb, ev), dc = dist_code((int)(m & 0xffffu) + 1, db, dv);
                nbits += S.len[lc] + eb + S.len[286 + dc] + db;
            }
        }
        uint32_t incl = nbits;
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(GSR_FULL, incl, o);
            if ((tid & 31) >= o) incl += t;
        }
        __syncthreads();
        if ((tid & 31) == 31) S.scan[tid >> 5] = incl;
        __syncthreads();
        if (tid < 32) {
            const uint32_t v = S.scan[tid];
            uint32_t x = v;
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(GSR_FULL, x, o);
                if (tid >= o) x += t;
            }
            S.scan[tid] = x - v;
        }
        __syncthreads();
        uint32_t pos = S.hdr_bits + S.scan[tid >> 5] + incl - nbits;
        for (uint32_t w = w0; w; w &= w - 1) {
            const int p = 32 * tid + __ffs(w) - 1;
            const uint32_t m = S.match[p];
            if (!m) {
                const int sy = S.data[p];
                put_bits(S.out, pos, S.code[sy], S.len[sy]), pos += S.len[sy];
            } else {
                int eb, ev, db, dv;
                const int lc = len_code((int)(m >> 16), eb, ev), dc = dist_code((int)(m & 0xffffu) + 1, db, dv);
                put_bits(S.out, pos, S.code[lc], S.len[lc]), pos += S.len[lc];
                put_bits(S.out, pos, (uint32_t)ev, eb), pos += eb;
                put_bits(S.out, pos, S.code[286 + dc], S.len[286 + dc]), pos += S.len[286 + dc];
                put_bits(S.out, pos, (uint32_t)dv, db), pos += db;
            }
        }
        __syncthreads();
    }

    // the chunk's bytes to the scratch, its CRC-32 (per-thread pieces combined in a tree) and Adler-32 sums
    const uint32_t total = S.total_bytes;
    const uint8_t* o8 = (const uint8_t*)S.out;
    auto obyte = [&](uint32_t k) -> uint8_t {
        if (mode) return o8[k];
        if (k == 0) return final_ ? 1 : 0;
        if (k == 1) return (uint8_t)clen;
        if (k == 2) return (uint8_t)(clen >> 8);
        if (k == 3) return (uint8_t)~clen;
        if (k == 4) return (uint8_t)(~clen >> 8);
        return S.data[k - 5];
    };
    uint8_t* dst = b.scratch + (int64_t)ci * PNG_CAP;
    for (uint32_t k = tid; k < total; k += PNG_THREADS) dst[k] = obyte(k);
    const uint32_t per = (total + PNG_THREADS - 1) / PNG_THREADS;
    const uint32_t a0 = min(total, per * tid), a1 = min(total, a0 + per);
    uint32_t crc = 0xffffffffu;
    for (uint32_t k = a0; k < a1; k++) crc = S.crc_table[(crc ^ obyte(k)) & 255u] ^ (crc >> 8);
    uint32_t* crc_part = S.vis;  // the parse words are no longer needed
    uint32_t* crc_len = S.exitp;
    __syncthreads();
    crc_part[tid] = ~crc;
    crc_len[tid] = a1 - a0;
    uint64_t s1 = 0, s2 = 0;
    for (int k = tid; k < clen; k += PNG_THREADS) {
        const uint64_t v = S.data[k];
        s1 += v;
        s2 += v * (uint64_t)(clen - k);
    }
    s1 = __reduce_add_sync(GSR_FULL, (uint32_t)s1);  // < 2^32: at most 32 x 255 per lane
    for (int o = 16; o; o >>= 1) s2 += __shfl_down_sync(GSR_FULL, s2, o);
    if ((tid & 31) == 0) S.red[tid >> 5][0] = s1, S.red[tid >> 5][1] = s2;
    __syncthreads();
    for (int st = 1; st < PNG_THREADS; st <<= 1) {
        if ((tid & (2 * st - 1)) == 0) {
            crc_part[tid] = crc_combine(crc_part[tid], crc_part[tid + st], crc_len[tid + st], S.x2n);
            crc_len[tid] += crc_len[tid + st];
        }
        __syncthreads();
    }
    if (tid == 0) {
        uint64_t t1 = 0, t2 = 0;
        for (int w = 0; w < 32; w++) t1 += S.red[w][0], t2 += S.red[w][1];
        b.meta[ci] = make_uint4(total, crc_part[0], (uint32_t)(t1 % 65521u), (uint32_t)(t2 % 65521u));
    }
}

// ------------------------------------------------------------------------------------------------------------------ the file
__device__ __forceinline__ void put_be32(uint8_t* p, uint32_t v) {
    p[0] = (uint8_t)(v >> 24), p[1] = (uint8_t)(v >> 16), p[2] = (uint8_t)(v >> 8), p[3] = (uint8_t)v;
}

__global__ void __launch_bounds__(256) k_png_assemble(const __grid_constant__ PngBatch b) {
    __shared__ uint64_t red[8];
    __shared__ uint32_t crc_part[256], crc_len[256], x2n[32], table_unused[256];
    const int tid = threadIdx.x;
    if ((int)blockIdx.x < b.chunks) {  // copy one chunk to its place
        const int ci = blockIdx.x, im = png_image_of_chunk(b, ci);
        const PngDesc& d = b.d[im];
        uint64_t off = 0;
        for (int k = d.chunk_base + tid; k < ci; k += 256) off += b.meta[k].x;
        for (int o = 16; o; o >>= 1) off += __shfl_down_sync(GSR_FULL, off, o);
        if ((tid & 31) == 0) red[tid >> 5] = off;
        __syncthreads();
        off = 0;
        for (int w = 0; w < 8; w++) off += red[w];
        const uint32_t n = b.meta[ci].x;
        const uint8_t* src = b.scratch + (int64_t)ci * PNG_CAP;
        uint8_t* dst = d.out + PNG_HEAD + off;
        for (uint32_t k = tid; k < n; k += 256) dst[k] = src[k];
        return;
    }
    // one image: headers, trailer and size
    const PngDesc& d = b.d[blockIdx.x - b.chunks];
    png_crc_tables(table_unused, x2n);
    __syncthreads();
    const int nc = d.nchunks;
    const int per = (nc + 255) / 256, k0 = min(nc, per * tid), k1 = min(nc, k0 + per);
    uint32_t crc = 0, clen_sum = 0;
    uint64_t a1 = 0, a2 = 0, bytes = 0;
    for (int k = k0; k < k1; k++) {
        const uint4 m = b.meta[d.chunk_base + k];
        crc = crc_combine(crc, m.y, m.x, x2n);
        clen_sum += m.x;
        const int64_t after = d.raw_len - (int64_t)(k + 1) * PNG_CHUNK;  // bytes of the stream after chunk k
        a1 += m.z;
        a2 += m.w + (uint64_t)((after > 0 ? after : 0) % 65521) * m.z % 65521;
    }
    bytes = clen_sum;
    crc_part[tid] = crc, crc_len[tid] = clen_sum;
    for (int o = 16; o; o >>= 1) {
        a1 += __shfl_down_sync(GSR_FULL, a1, o);
        a2 += __shfl_down_sync(GSR_FULL, a2, o);
        bytes += __shfl_down_sync(GSR_FULL, bytes, o);
    }
    __shared__ uint64_t sums[8][3];
    if ((tid & 31) == 0) sums[tid >> 5][0] = a1, sums[tid >> 5][1] = a2, sums[tid >> 5][2] = bytes;
    __syncthreads();
    for (int st = 1; st < 256; st <<= 1) {
        if ((tid & (2 * st - 1)) == 0) {
            crc_part[tid] = crc_combine(crc_part[tid], crc_part[tid + st], crc_len[tid + st], x2n);
            crc_len[tid] += crc_len[tid + st];
        }
        __syncthreads();
    }
    if (tid != 0) return;
    uint64_t S1 = 0, S2 = 0, Z = 0;
    for (int w = 0; w < 8; w++) S1 += sums[w][0], S2 += sums[w][1], Z += sums[w][2];
    const uint32_t ad_a = (uint32_t)((1 + S1) % 65521), ad_b = (uint32_t)(((uint64_t)(d.raw_len % 65521) + S2) % 65521);
    const uint32_t adler = (ad_b << 16) | ad_a;
    uint8_t* o = d.out;
    const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
    for (int k = 0; k < 8; k++) o[k] = sig[k];
    uint8_t ihdr[17] = {'I', 'H', 'D', 'R'};
    put_be32(ihdr + 4, (uint32_t)d.W);
    put_be32(ihdr + 8, (uint32_t)d.H);
    ihdr[12] = 8;
    ihdr[13] = d.C == 4 ? 6 : (d.C == 3 ? 2 : 0);
    ihdr[14] = ihdr[15] = ihdr[16] = 0;
    put_be32(o + 8, 13);
    for (int k = 0; k < 17; k++) o[12 + k] = ihdr[k];
    put_be32(o + 29, ~crc_bytes_bitwise(0xffffffffu, ihdr, 17));
    const uint32_t zlen = (uint32_t)(2 + Z + 4);
    put_be32(o + 33, zlen);
    const uint8_t idat[6] = {'I', 'D', 'A', 'T', 0x78, 0x01};
    for (int k = 0; k < 6; k++) o[37 + k] = idat[k];
    uint8_t ad[4];
    put_be32(ad, adler);
    uint32_t c = ~crc_bytes_bitwise(0xffffffffu, idat, 6);
    c = crc_combine(c, crc_part[0], Z, x2n);
    c = crc_combine(c, ~crc_bytes_bitwise(0xffffffffu, ad, 4), 4, x2n);
    uint8_t* t = o + PNG_HEAD + Z;
    for (int k = 0; k < 4; k++) t[k] = ad[k];
    put_be32(t + 4, c);
    const uint8_t iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xae, 0x42, 0x60, 0x82};
    for (int k = 0; k < 12; k++) t[8 + k] = iend[k];
    d.size[0] = (int64_t)(PNG_HEAD + Z + PNG_TAIL);
}

// ------------------------------------------------------------------------------------------------------------------ host side
int64_t png_raw_bytes(int32_t H, int32_t W, int32_t C) { return (int64_t)H * (1 + (int64_t)W * C); }
int64_t png_chunks(int64_t raw) { return (raw + PNG_CHUNK - 1) / PNG_CHUNK; }
int64_t align256(int64_t x) { return (x + 255) & ~(int64_t)255; }
constexpr int64_t PNG_MAX_RAW = 0x7fff0000LL;  // the IDAT length is a 31-bit field

int png_file_channels(const gsr_png_image& im) { return im.lut ? 3 : im.C; }

bool png_check(const gsr_png_image& im, int i) {
    if (!im.data) { set_error("gsr_png: image %d has no data", i); return false; }
    if (im.H < 1 || im.W < 1) { set_error("gsr_png: image %d is empty (%d x %d)", i, im.H, im.W); return false; }
    if (im.C != 1 && im.C != 3 && im.C != 4) { set_error("gsr_png: image %d has %d channels (1, 3 or 4)", i, im.C); return false; }
    if (im.lut && im.C != 1) { set_error("gsr_png: image %d has a lookup table and %d channels (needs 1)", i, im.C); return false; }
    if (im.flags & ~GSR_PNG_SWAP_RB) { set_error("gsr_png: image %d has unknown flags %d", i, im.flags); return false; }
    if (png_raw_bytes(im.H, im.W, png_file_channels(im)) > PNG_MAX_RAW) { set_error("gsr_png: image %d is too large for one IDAT chunk", i); return false; }
    return true;
}

struct PngLayout {
    int64_t raw, match, scratch, meta, total;
};

PngLayout png_layout(int n, const gsr_png_image* images) {
    PngLayout L = {0, 0, 0, 0, 0};
    int64_t chunks = 0;
    for (int i = 0; i < n; i++) {
        const int64_t r = png_raw_bytes(images[i].H, images[i].W, png_file_channels(images[i]));
        L.raw += align256(r);
        chunks += png_chunks(r);
    }
    L.match = L.raw;  // match words share the stream's offsets
    L.scratch = L.raw + 4 * L.raw;
    L.meta = L.scratch + chunks * PNG_CAP;
    L.total = L.meta + align256(chunks * 16);
    return L;
}

}  // namespace gsr

using namespace gsr;

size_t gsr_png_bound(int32_t H, int32_t W, int32_t C) {
    if (H < 1 || W < 1 || (C != 1 && C != 3 && C != 4)) return 0;
    const int64_t raw = png_raw_bytes(H, W, C);
    if (raw > PNG_MAX_RAW) return 0;
    return (size_t)(PNG_HEAD + PNG_TAIL + raw + 5 * png_chunks(raw));
}

size_t gsr_png_workspace_bytes(int32_t n, const gsr_png_image* images) {
    if (n < 0 || (n > 0 && !images)) return 0;
    for (int i = 0; i < n; i++)
        if (images[i].H < 1 || images[i].W < 1 || images[i].C < 1 || images[i].C > 4) return 0;
    return (size_t)png_layout(n, images).total;
}

int gsr_png_encode(const gsr_png_image* images, int32_t n, uint8_t* const* outputs, int64_t* sizes, void* workspace, size_t workspace_bytes,
                   void* stream) {
    NvtxRange nvtx_("gsr_png_encode");
    const cudaStream_t s = (cudaStream_t)stream;
    if (n == 0) return GSR_OK;
    if (n < 0 || !images || !outputs || !sizes) { set_error("gsr_png_encode: bad arguments (n %d)", n); return GSR_ERR_INVALID; }
    for (int i = 0; i < n; i++) {
        if (!png_check(images[i], i)) return GSR_ERR_INVALID;
        if (!outputs[i]) { set_error("gsr_png_encode: output %d is NULL", i); return GSR_ERR_INVALID; }
    }
    if ((uintptr_t)sizes & 7) { set_error("gsr_png_encode: sizes must be 8-byte aligned"); return GSR_ERR_INVALID; }
    const PngLayout L = png_layout(n, images);
    if (!workspace || ((uintptr_t)workspace & 255)) { set_error("gsr_png_encode: the workspace must be 256-byte aligned"); return GSR_ERR_INVALID; }
    if (workspace_bytes < (size_t)L.total) {
        set_error("gsr_png_encode: workspace of %zu bytes, gsr_png_workspace_bytes gives %lld", workspace_bytes, (long long)L.total);
        return GSR_ERR_WORKSPACE;
    }
    cudaFuncSetAttribute(k_png_match, cudaFuncAttributeMaxDynamicSharedMemorySize, PNG_MATCH_SMEM);
    cudaFuncSetAttribute(k_png_deflate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DeflateShared));
    uint8_t* ws = (uint8_t*)workspace;
    int64_t raw_off = 0, chunk_off = 0;
    for (int i0 = 0; i0 < n; i0 += GSR_PNG_MAX_BATCH) {
        PngBatch b;
        memset(&b, 0, sizeof(b));
        b.n = min(n - i0, GSR_PNG_MAX_BATCH);
        b.raw = ws;
        b.match = (uint32_t*)(ws + L.match);
        b.scratch = ws + L.scratch + chunk_off * PNG_CAP;
        b.meta = (uint4*)(ws + L.meta) + chunk_off;
        int64_t rows = 0, chunks = 0;
        for (int k = 0; k < b.n; k++) {
            const gsr_png_image& im = images[i0 + k];
            PngDesc& d = b.d[k];
            d.src = im.data, d.lut = im.lut;
            d.sh = im.stride_h, d.sw = im.stride_w, d.sc = im.stride_c;
            d.H = im.H, d.W = im.W, d.C = png_file_channels(im), d.flags = im.flags;
            d.raw_len = png_raw_bytes(d.H, d.W, d.C);
            d.raw_off = raw_off;
            raw_off += align256(d.raw_len);
            d.row_base = rows;
            rows += d.H;
            d.chunk_base = (int32_t)chunks;
            d.nchunks = (int32_t)png_chunks(d.raw_len);
            chunks += d.nchunks;
            d.out = outputs[i0 + k];
            d.size = sizes + i0 + k;
        }
        if (rows > 0x7fffffffLL || chunks > 0x7fffffffLL - GSR_PNG_MAX_BATCH) { set_error("gsr_png_encode: batch too large"); return GSR_ERR_INVALID; }
        b.rows = (int32_t)rows, b.chunks = (int32_t)chunks;
        chunk_off += chunks;
        k_png_filter<<<(unsigned)rows, 256, 0, s>>>(b);
        k_png_match<<<(unsigned)chunks, PNG_THREADS, PNG_MATCH_SMEM, s>>>(b);
        k_png_deflate<<<(unsigned)chunks, PNG_THREADS, sizeof(DeflateShared), s>>>(b);
        k_png_assemble<<<(unsigned)(chunks + b.n), 256, 0, s>>>(b);
    }
    return check_launch("gsr_png_encode", false, s);
}
