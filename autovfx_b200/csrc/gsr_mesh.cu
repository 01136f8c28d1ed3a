// First-hit ray casts against a triangle mesh: trimesh's `mesh.ray.intersects_first` / `intersects_location(multiple_hits=False)`
// as AutoVFX calls them (extract/extract_object.py, dataset_readers.py's ray-mesh initialisation, edit_utils.py,
// estimate_scene_scale.py), on an LBVH (Karras 2012) built on the device.
//   build:  k_mesh_prep    per triangle: validity (finite vertices, non-zero float64 edge cross product), float32 centroid,
//                          the centroid box and the scene's largest |coordinate| (ordered-integer atomics)
//           k_mesh_morton  30-bit Morton codes of the centroids; invalid triangles get 0xffffffff (they sort last)
//           k_rs_hist / scan / k_rs_scatter   the library's stable radix sort (gsr_radix.cuh): ties keep the lower index
//           k_mesh_leaves  float64 triangles and original indices in leaf order; leaf boxes rounded outwards to float32
//           k_mesh_tree    the radix tree of the sorted codes, ties split on the leaf position (Karras 2012, §4)
//           k_mesh_fit     bottom-up box fit, the second thread to reach a node carries on
//   query:  k_first_hit    one ray per thread, caller order, a 64-entry stack: the watertight test (Woop, Benthin and Wald 2013)
//                          in float64 with every operation rounded on its own (no FMA contraction), smallest t, then lowest index
//           k_inpaint_mask the inpainting mask of extract_object.py:563-606 from two casts' hits
// DESIGN.md §4 argues why the box test never culls a triangle the exact test hits.
#include "gsr_radix.cuh"
#include <cfloat>
#include <cstddef>

namespace gsr {
namespace {

constexpr int MESH_THREADS = 256;
constexpr int MESH_STACK = 64;  // > the deepest path of a radix tree over 30-bit codes + 31-bit positions
constexpr uint32_t MESH_INVALID_CODE = 0xffffffffu;

// BVH buffer: header | nodes | leaf triangles | leaf ids
struct MeshHeader {
    int32_t F;
    float coord_max;  // the largest |vertex coordinate| of the valid triangles, rounded up to float32
    int32_t pad[14];
};
struct MeshNode {        // an internal node holds its two children's boxes
    float4 a, b, c;      // lo_l.xyz hi_l.x | hi_l.yz lo_r.xy | lo_r.z hi_r.xyz
    int32_t left, right;  // >= 0: internal node; < 0: leaf ~k
    int32_t pad[2];
};
static_assert(sizeof(MeshNode) == 64, "one node per 64-byte line");

struct MeshBvh {
    size_t nodes, tris, ids, total;
    explicit MeshBvh(size_t F) {
        size_t o = align_up(sizeof(MeshHeader), 256);
        nodes = o; o = align_up(o + 64 * (F > 1 ? F - 1 : 0), 256);
        tris = o;  o = align_up(o + 72 * F, 256);
        ids = o;   o = align_up(o + 4 * F, 256);
        total = o;
    }
};

struct MeshBuild {
    size_t scal, cent, codes0, codes1, vals0, vals1, hist, part, leafbox, parent, leaf_parent, flags, total;
    int nchunks;
    explicit MeshBuild(size_t F) {
        nchunks = rs_chunks(F);
        const size_t nhist = 256 * (size_t)nchunks;
        size_t o = 0;
        scal = o;    o = align_up(o + 64, 256);
        cent = o;    o = align_up(o + 12 * F, 256);
        codes0 = o;  o = align_up(o + 4 * F, 256);
        codes1 = o;  o = align_up(o + 4 * F, 256);
        vals0 = o;   o = align_up(o + 4 * F, 256);
        vals1 = o;   o = align_up(o + 4 * F, 256);
        hist = o;    o = align_up(o + 4 * nhist, 256);
        part = o;    o = align_up(o + 4 * scan_parts(nhist), 256);
        leafbox = o; o = align_up(o + 24 * F, 256);
        parent = o;  o = align_up(o + 4 * F, 256);
        leaf_parent = o; o = align_up(o + 4 * F, 256);
        flags = o;   o = align_up(o + 4 * F, 256);
        total = o;
    }
};

__device__ __forceinline__ uint32_t mesh_f2ord(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float mesh_ord2f(uint32_t u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u); }

__device__ __forceinline__ double dsub(double a, double b) { return __dadd_rn(a, -b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }

// scal: [0..2] ordered min of the centroids, [3..5] ordered max, [6] float bits of the largest |coordinate|
__global__ void k_mesh_scal_init(uint32_t* scal) {
    if (threadIdx.x < 3) scal[threadIdx.x] = mesh_f2ord(FLT_MAX);
    else if (threadIdx.x < 6) scal[threadIdx.x] = mesh_f2ord(-FLT_MAX);
    else if (threadIdx.x == 6) scal[6] = 0u;
}

__device__ __forceinline__ bool load_tri(int64_t V, const double* __restrict__ verts, const int64_t* __restrict__ faces, int64_t f, double v[9]) {
    bool ok = true;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const int64_t vi = faces[3 * f + k];
        if (vi < 0 || vi >= V) {
            ok = false;
            v[3 * k] = v[3 * k + 1] = v[3 * k + 2] = 0.0;
            continue;
        }
#pragma unroll
        for (int c = 0; c < 3; c++) {
            v[3 * k + c] = verts[3 * vi + c];
            ok = ok && isfinite(v[3 * k + c]);
        }
    }
    return ok;
}

// A triangle is valid when its vertices are finite and (v1 - v0) x (v2 - v0), each operation rounded on its own, is not zero.
__device__ __forceinline__ bool tri_valid(const double v[9]) {
    const double e1x = dsub(v[3], v[0]), e1y = dsub(v[4], v[1]), e1z = dsub(v[5], v[2]);
    const double e2x = dsub(v[6], v[0]), e2y = dsub(v[7], v[1]), e2z = dsub(v[8], v[2]);
    const double nx = dsub(dmul(e1y, e2z), dmul(e1z, e2y));
    const double ny = dsub(dmul(e1z, e2x), dmul(e1x, e2z));
    const double nz = dsub(dmul(e1x, e2y), dmul(e1y, e2x));
    return nx != 0.0 || ny != 0.0 || nz != 0.0;
}

__global__ void __launch_bounds__(MESH_THREADS) k_mesh_prep(int32_t F, int64_t V, const double* __restrict__ verts, const int64_t* __restrict__ faces,
                                                            float* __restrict__ cent, uint32_t* __restrict__ scal) {
    const int f = blockIdx.x * MESH_THREADS + threadIdx.x;
    float c[3] = {0.f, 0.f, 0.f}, mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX}, amax = 0.f;
    if (f < F) {
        double v[9];
        const bool finite = load_tri(V, verts, faces, f, v);
        if (finite && tri_valid(v)) {
#pragma unroll
            for (int k = 0; k < 3; k++) {
                c[k] = (float)((v[k] + v[3 + k] + v[6 + k]) / 3.0);
                mn[k] = mx[k] = c[k];
            }
            double m = 0.0;
#pragma unroll
            for (int k = 0; k < 9; k++) m = fmax(m, fabs(v[k]));
            amax = __double2float_ru(m);
        } else {
            c[0] = c[1] = c[2] = __int_as_float(0x7fc00000);  // NaN: k_mesh_morton files it last
        }
        cent[3 * (size_t)f] = c[0]; cent[3 * (size_t)f + 1] = c[1]; cent[3 * (size_t)f + 2] = c[2];
    }
#pragma unroll
    for (int k = 0; k < 3; k++)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn[k] = fminf(mn[k], __shfl_xor_sync(GSR_FULL, mn[k], o));
            mx[k] = fmaxf(mx[k], __shfl_xor_sync(GSR_FULL, mx[k], o));
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(GSR_FULL, amax, o));
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 3; k++) {
            atomicMin(&scal[k], mesh_f2ord(mn[k]));
            atomicMax(&scal[3 + k], mesh_f2ord(mx[k]));
        }
        atomicMax(&scal[6], __float_as_uint(amax));  // non-negative floats order as their bits
    }
}

__device__ __forceinline__ uint32_t mesh_spread10(uint32_t x) {
    x = (x | (x << 16)) & 0x030000FF;
    x = (x | (x << 8)) & 0x0300F00F;
    x = (x | (x << 4)) & 0x030C30C3;
    x = (x | (x << 2)) & 0x09249249;
    return x;
}

__global__ void __launch_bounds__(MESH_THREADS) k_mesh_morton(int32_t F, const float* __restrict__ cent, const uint32_t* __restrict__ scal,
                                                              uint32_t* __restrict__ codes, uint32_t* __restrict__ vals) {
    const int f = blockIdx.x * MESH_THREADS + threadIdx.x;
    if (f >= F) return;
    uint32_t code = MESH_INVALID_CODE;
    const float cx = cent[3 * (size_t)f];
    if (!isnan(cx)) {
        code = 0;
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const float lo = mesh_ord2f(scal[k]), hi = mesh_ord2f(scal[3 + k]);
            const float ext = hi - lo;
            float q = ext > 0.f ? (cent[3 * (size_t)f + k] - lo) / ext * 1023.f : 0.f;
            q = fminf(fmaxf(q, 0.f), 1023.f);
            code |= mesh_spread10((uint32_t)q) << k;
        }
    }
    codes[f] = code;
    vals[f] = (uint32_t)f;
}

__global__ void __launch_bounds__(MESH_THREADS) k_mesh_leaves(int32_t F, int64_t V, const double* __restrict__ verts, const int64_t* __restrict__ faces,
                                                              const uint32_t* __restrict__ order, const uint32_t* __restrict__ codes,
                                                              double* __restrict__ tris, int32_t* __restrict__ ids, float* __restrict__ leafbox) {
    const int k = blockIdx.x * MESH_THREADS + threadIdx.x;
    if (k >= F) return;
    const uint32_t f = order[k];
    double v[9];
    load_tri(V, verts, faces, f, v);
    const bool valid = codes[k] != MESH_INVALID_CODE;
#pragma unroll
    for (int c = 0; c < 9; c++) tris[9 * (size_t)k + c] = v[c];
    ids[k] = valid ? (int32_t)f : -1;
    float* b = leafbox + 6 * (size_t)k;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        // rounded outwards: the float32 box holds the float64 vertices; an invalid leaf gets an empty box
        b[c] = valid ? __double2float_rd(fmin(fmin(v[c], v[3 + c]), v[6 + c])) : INFINITY;
        b[3 + c] = valid ? __double2float_ru(fmax(fmax(v[c], v[3 + c]), v[6 + c])) : -INFINITY;
    }
}

// common prefix length of the augmented keys (code, position) at positions i and j; -1 outside [0, n)
__device__ __forceinline__ int mesh_delta(const uint32_t* __restrict__ codes, int n, int i, int64_t j) {
    if (j < 0 || j >= n) return -1;
    const uint32_t a = codes[i], b = codes[j];
    return a != b ? __clz(a ^ b) : 32 + __clz((uint32_t)i ^ (uint32_t)j);
}

__global__ void __launch_bounds__(MESH_THREADS) k_mesh_tree(int32_t F, const uint32_t* __restrict__ codes, MeshNode* __restrict__ nodes,
                                                            int32_t* __restrict__ parent, int32_t* __restrict__ leaf_parent, int32_t* __restrict__ flags) {
    const int i = blockIdx.x * MESH_THREADS + threadIdx.x;
    if (i >= F - 1) return;
    const int d = mesh_delta(codes, F, i, i + 1) - mesh_delta(codes, F, i, i - 1) > 0 ? 1 : -1;
    const int dmin = mesh_delta(codes, F, i, i - d);
    int64_t lmax = 2;
    while (mesh_delta(codes, F, i, i + lmax * d) > dmin) lmax <<= 1;
    int l = 0;
    for (int64_t t = lmax >> 1; t >= 1; t >>= 1)
        if (mesh_delta(codes, F, i, i + (l + t) * d) > dmin) l += t;
    const int j = i + l * d;
    const int dnode = mesh_delta(codes, F, i, j);
    int s = 0;
    for (int t = (l + 1) >> 1;; t = (t + 1) >> 1) {
        if (mesh_delta(codes, F, i, i + (s + t) * d) > dnode) s += t;
        if (t == 1) break;
    }
    const int gamma = i + s * d + min(d, 0);
    const int lo = min(i, j), hi = max(i, j);
    const int left = lo == gamma ? ~gamma : gamma;
    const int right = hi == gamma + 1 ? ~(gamma + 1) : gamma + 1;
    nodes[i].left = left;
    nodes[i].right = right;
    if (left < 0) leaf_parent[~left] = i; else parent[left] = i;
    if (right < 0) leaf_parent[~right] = i; else parent[right] = i;
    flags[i] = 0;
}

__device__ __forceinline__ void node_box_store(MeshNode* n, int slot, const float b[6]) {
    float* f = reinterpret_cast<float*>(n) + 6 * slot;
#pragma unroll
    for (int c = 0; c < 6; c++) f[c] = b[c];
}

__global__ void __launch_bounds__(MESH_THREADS) k_mesh_fit(int32_t F, const float* __restrict__ leafbox, MeshNode* nodes, const int32_t* __restrict__ parent,
                                                           const int32_t* __restrict__ leaf_parent, int32_t* flags) {
    const int k = blockIdx.x * MESH_THREADS + threadIdx.x;
    if (k >= F) return;
    float b[6];
#pragma unroll
    for (int c = 0; c < 6; c++) b[c] = leafbox[6 * (size_t)k + c];
    int child = ~k, p = leaf_parent[k];
    while (true) {
        const int slot = nodes[p].left == child ? 0 : 1;
        node_box_store(nodes + p, slot, b);
        __threadfence();
        if (atomicAdd(flags + p, 1) == 0) return;  // the sibling's thread carries on
        __threadfence();
        const volatile float* o = reinterpret_cast<const volatile float*>(nodes + p) + 6 * (1 - slot);
#pragma unroll
        for (int c = 0; c < 3; c++) {
            b[c] = fminf(b[c], o[c]);
            b[3 + c] = fmaxf(b[3 + c], o[3 + c]);
        }
        if (p == 0) return;
        child = p;
        p = parent[p];
    }
}

// ---- query ----
struct Ray {
    double o[3], d[3];
    int kx, ky, kz;
    double Sx, Sy, Sz;
    double inv[3];
    double pad;  // the spatial slack of the box test (DESIGN.md §4)
};

// The watertight test in float64, every operation rounded on its own, in this order (tests/raycast_ref.py restates it).
__device__ __forceinline__ bool tri_test(const Ray& r, const double* __restrict__ v, double* t_out) {
    const double Akx = dsub(v[r.kx], r.o[r.kx]), Aky = dsub(v[r.ky], r.o[r.ky]), Akz = dsub(v[r.kz], r.o[r.kz]);
    const double Bkx = dsub(v[3 + r.kx], r.o[r.kx]), Bky = dsub(v[3 + r.ky], r.o[r.ky]), Bkz = dsub(v[3 + r.kz], r.o[r.kz]);
    const double Ckx = dsub(v[6 + r.kx], r.o[r.kx]), Cky = dsub(v[6 + r.ky], r.o[r.ky]), Ckz = dsub(v[6 + r.kz], r.o[r.kz]);
    const double Ax = dsub(Akx, dmul(r.Sx, Akz)), Ay = dsub(Aky, dmul(r.Sy, Akz));
    const double Bx = dsub(Bkx, dmul(r.Sx, Bkz)), By = dsub(Bky, dmul(r.Sy, Bkz));
    const double Cx = dsub(Ckx, dmul(r.Sx, Ckz)), Cy = dsub(Cky, dmul(r.Sy, Ckz));
    const double U = dsub(dmul(Cx, By), dmul(Cy, Bx));
    const double V = dsub(dmul(Ax, Cy), dmul(Ay, Cx));
    const double W = dsub(dmul(Bx, Ay), dmul(By, Ax));
    if ((U < 0.0 || V < 0.0 || W < 0.0) && (U > 0.0 || V > 0.0 || W > 0.0)) return false;
    const double det = dadd(dadd(U, V), W);
    if (det == 0.0) return false;
    const double Az = dmul(r.Sz, Akz), Bz = dmul(r.Sz, Bkz), Cz = dmul(r.Sz, Ckz);
    const double T = dadd(dadd(dmul(U, Az), dmul(V, Bz)), dmul(W, Cz));
    const double t = __ddiv_rn(T, det);
    *t_out = t;
    return t > 0.0 && t < INFINITY;  // false for NaN
}

// The box test: the ray's line meets the box grown by r.pad (all three slabs), and the kz-slab interval, which bounds every t
// the exact test can return inside the box (DESIGN.md §4), reaches t > 0 and not beyond best_t.  *key orders the two children.
__device__ __forceinline__ bool box_test(const Ray& r, const float* b, double best_t, double* key) {
    double tmin = -INFINITY, tmax = INFINITY;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const double lo = dsub((double)b[c], r.pad), hi = dadd((double)b[3 + c], r.pad);
        const bool neg = signbit(r.inv[c]);
        const double tn = dmul(dsub(neg ? hi : lo, r.o[c]), r.inv[c]);
        const double tf = dmul(dsub(neg ? lo : hi, r.o[c]), r.inv[c]);
        tmin = fmax(tmin, tn);  // fmax / fmin drop the NaN of 0 * inf (the origin on a slab plane of a parallel ray)
        tmax = fmin(tmax, tf);
    }
    if (!(tmin <= tmax)) return false;
    // the kz slab of the unpadded box, computed as the exact test computes Az: rn(Sz * rn(v - o)) is monotonic in v
    const double z0 = dmul(r.Sz, dsub((double)b[r.kz], r.o[r.kz])), z1 = dmul(r.Sz, dsub((double)b[3 + r.kz], r.o[r.kz]));
    const double zn = fmin(z0, z1), zf = fmax(z0, z1);
    const double slack = dmul(0x1p-40, fmax(fabs(zn), fabs(zf)));
    if (!(dadd(zf, slack) > 0.0) || dsub(zn, slack) > best_t) return false;
    *key = tmin;
    return true;
}

template <typename T>
__global__ void __launch_bounds__(MESH_THREADS) k_first_hit(int64_t N, int32_t F, const MeshHeader* __restrict__ hdr, const MeshNode* __restrict__ nodes,
                                                            const double* __restrict__ tris, const int32_t* __restrict__ ids,
                                                            const T* __restrict__ orig, const T* __restrict__ dir, const int64_t* __restrict__ active,
                                                            int64_t* __restrict__ tri_out, double* __restrict__ t_out) {
    const int64_t i = (int64_t)blockIdx.x * MESH_THREADS + threadIdx.x;
    if (i >= N) return;
    double best_t = INFINITY;
    int32_t best = -1;
    Ray r;
    bool ok = active == nullptr || active[i] >= 0;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        r.o[c] = (double)orig[3 * i + c];
        r.d[c] = (double)dir[3 * i + c];
        ok = ok && isfinite(r.o[c]) && isfinite(r.d[c]);
    }
    ok = ok && (r.d[0] != 0.0 || r.d[1] != 0.0 || r.d[2] != 0.0);
    if (ok && F > 0) {
        r.kz = 0;
        if (fabs(r.d[1]) > fabs(r.d[r.kz])) r.kz = 1;
        if (fabs(r.d[2]) > fabs(r.d[r.kz])) r.kz = 2;
        r.kx = r.kz == 2 ? 0 : r.kz + 1;
        r.ky = r.kx == 2 ? 0 : r.kx + 1;
        if (r.d[r.kz] < 0.0) { const int s = r.kx; r.kx = r.ky; r.ky = s; }
        r.Sx = __ddiv_rn(r.d[r.kx], r.d[r.kz]);
        r.Sy = __ddiv_rn(r.d[r.ky], r.d[r.kz]);
        r.Sz = __ddiv_rn(1.0, r.d[r.kz]);
#pragma unroll
        for (int c = 0; c < 3; c++) r.inv[c] = __ddiv_rn(1.0, r.d[c]);
        r.pad = dmul(0x1p-24, dadd(fmax(fmax(fabs(r.o[0]), fabs(r.o[1])), fabs(r.o[2])), (double)hdr->coord_max));

        auto leaf = [&](int k) {
            const int32_t id = ids[k];
            if (id < 0) return;
            double v[9];
#pragma unroll
            for (int c = 0; c < 9; c++) v[c] = tris[9 * (size_t)k + c];
            double t;
            if (tri_test(r, v, &t) && (t < best_t || (t == best_t && id < best))) {
                best_t = t;
                best = id;
            }
        };
        if (F == 1) {
            leaf(0);
        } else {
            int stack[MESH_STACK];
            int sp = 0, node = 0;
            while (true) {
                const MeshNode n = nodes[node];
                const float bl[6] = {n.a.x, n.a.y, n.a.z, n.a.w, n.b.x, n.b.y};
                const float br[6] = {n.b.z, n.b.w, n.c.x, n.c.y, n.c.z, n.c.w};
                double kl, kr;
                bool hl = box_test(r, bl, best_t, &kl), hr = box_test(r, br, best_t, &kr);
                if (hl && n.left < 0) { leaf(~n.left); hl = false; }
                if (hr && n.right < 0) { leaf(~n.right); hr = false; }
                if (hl && hr) {
                    const bool lfirst = kl <= kr;
                    stack[sp++] = lfirst ? n.right : n.left;
                    node = lfirst ? n.left : n.right;
                } else if (hl) {
                    node = n.left;
                } else if (hr) {
                    node = n.right;
                } else {
                    if (sp == 0) break;
                    node = stack[--sp];
                }
            }
        }
    }
    tri_out[i] = best;
    if (t_out) t_out[i] = best_t;
}

// extract_object.py:563-606 for one view, from the planar cast (tri_p, t_p) and the combined-mesh cast (tri_a, t_a) of the
// same rays: location = o + t d per component (one multiply, one add), depth = ((x w20 + y w21) + z w22) + w23, depth_all = 0
// where the combined mesh is missed, mask = 255 where |depth_all - depth_planar| < 0.01.  counts[0] += planar hits,
// counts[1] += planar-hit rays that also hit the combined mesh.
template <typename T>
__global__ void __launch_bounds__(MESH_THREADS) k_inpaint_mask(int64_t N, const T* __restrict__ orig, const T* __restrict__ dir,
                                                               const int64_t* __restrict__ tri_p, const double* __restrict__ t_p,
                                                               const int64_t* __restrict__ tri_a, const double* __restrict__ t_a,
                                                               const double* __restrict__ w2c, uint8_t* __restrict__ mask,
                                                               unsigned long long* __restrict__ counts) {
    const int64_t i = (int64_t)blockIdx.x * MESH_THREADS + threadIdx.x;
    bool hp = false, ha = false;
    if (i < N) {
        uint8_t m = 0;
        hp = tri_p[i] >= 0;
        if (hp) {
            ha = tri_a[i] >= 0;
            double o[3], d[3];
#pragma unroll
            for (int c = 0; c < 3; c++) { o[c] = (double)orig[3 * i + c]; d[c] = (double)dir[3 * i + c]; }
            auto depth = [&](double t) {
                const double x = dadd(o[0], dmul(t, d[0])), y = dadd(o[1], dmul(t, d[1])), z = dadd(o[2], dmul(t, d[2]));
                return dadd(dadd(dadd(dmul(x, w2c[8]), dmul(y, w2c[9])), dmul(z, w2c[10])), w2c[11]);
            };
            const double dp = depth(t_p[i]);
            const double da = ha ? depth(t_a[i]) : 0.0;
            m = fabs(dsub(da, dp)) < 0.01 ? 255 : 0;
        }
        mask[i] = m;
    }
    const unsigned bp = __ballot_sync(GSR_FULL, hp), ba = __ballot_sync(GSR_FULL, ha);
    if ((threadIdx.x & 31) == 0 && bp) {
        atomicAdd(counts, (unsigned long long)__popc(bp));
        if (ba) atomicAdd(counts + 1, (unsigned long long)__popc(ba));
    }
}

}  // namespace
}  // namespace gsr

using namespace gsr;

size_t gsr_mesh_bvh_bytes(int32_t F) { return F < 0 ? 0 : MeshBvh((size_t)F).total; }

size_t gsr_mesh_build_bytes(int32_t F) { return F < 0 ? 0 : MeshBuild((size_t)F).total; }

int gsr_mesh_build(int64_t V, int32_t F, const double* vertices, const int64_t* faces, void* bvh, size_t bvh_bytes, void* ws, size_t ws_bytes,
                   void* stream) {
    NvtxRange nvtx_("gsr_mesh_build");
    const cudaStream_t st = (cudaStream_t)stream;
    if (V < 0 || F < 0 || (F > 0 && (!vertices || !faces))) {
        set_error("gsr_mesh_build: bad arguments (V %lld, F %d)", (long long)V, F);
        return GSR_ERR_INVALID;
    }
    const MeshBvh B((size_t)F);
    const MeshBuild L((size_t)F);
    if (!bvh || ((uintptr_t)bvh & 255) || bvh_bytes < B.total) {
        set_error("gsr_mesh_build: BVH buffer of %zu bytes, gsr_mesh_bvh_bytes(%d) = %zu needed (256-byte aligned)", bvh_bytes, F, B.total);
        return GSR_ERR_WORKSPACE;
    }
    if (!ws || ((uintptr_t)ws & 255) || ws_bytes < L.total) {
        set_error("gsr_mesh_build: workspace of %zu bytes, gsr_mesh_build_bytes(%d) = %zu needed (256-byte aligned)", ws_bytes, F, L.total);
        return GSR_ERR_WORKSPACE;
    }
    char* b = (char*)bvh;
    char* w = (char*)ws;
    uint32_t* scal = (uint32_t*)(w + L.scal);
    MeshHeader h{};
    h.F = F;
    cudaMemcpyAsync(b, &h, sizeof(h), cudaMemcpyHostToDevice, st);  // F; coord_max follows from the device below
    if (F == 0) return check_launch("gsr_mesh_build", false, st);
    const unsigned grid = (unsigned)((F + MESH_THREADS - 1) / MESH_THREADS);
    k_mesh_scal_init<<<1, 32, 0, st>>>(scal);
    k_mesh_prep<<<grid, MESH_THREADS, 0, st>>>(F, V, vertices, faces, (float*)(w + L.cent), scal);
    cudaMemcpyAsync(b + offsetof(MeshHeader, coord_max), scal + 6, 4, cudaMemcpyDeviceToDevice, st);
    uint32_t *k0 = (uint32_t*)(w + L.codes0), *k1 = (uint32_t*)(w + L.codes1), *v0 = (uint32_t*)(w + L.vals0), *v1 = (uint32_t*)(w + L.vals1);
    uint32_t *hist = (uint32_t*)(w + L.hist), *part = (uint32_t*)(w + L.part);
    k_mesh_morton<<<grid, MESH_THREADS, 0, st>>>(F, (const float*)(w + L.cent), scal, k0, v0);
    const int rs_blocks = (L.nchunks + RS_WARPS - 1) / RS_WARPS;
    for (int shift = 0; shift < 32; shift += 8) {
        k_rs_hist<<<rs_blocks, RS_WARPS * 32, 0, st>>>((uint32_t)F, k0, shift, L.nchunks, hist);
        scan_wide(hist, 256 * (size_t)L.nchunks, part, st);
        k_rs_scatter<<<rs_blocks, RS_WARPS * 32, 0, st>>>((uint32_t)F, k0, v0, shift, L.nchunks, hist, k1, v1);
        uint32_t* t = k0; k0 = k1; k1 = t;
        t = v0; v0 = v1; v1 = t;
    }
    MeshNode* nodes = (MeshNode*)(b + B.nodes);
    float* leafbox = (float*)(w + L.leafbox);
    k_mesh_leaves<<<grid, MESH_THREADS, 0, st>>>(F, V, vertices, faces, v0, k0, (double*)(b + B.tris), (int32_t*)(b + B.ids), leafbox);
    if (F > 1) {
        int32_t *parent = (int32_t*)(w + L.parent), *leaf_parent = (int32_t*)(w + L.leaf_parent), *flags = (int32_t*)(w + L.flags);
        k_mesh_tree<<<(unsigned)((F - 1 + MESH_THREADS - 1) / MESH_THREADS), MESH_THREADS, 0, st>>>(F, k0, nodes, parent, leaf_parent, flags);
        k_mesh_fit<<<grid, MESH_THREADS, 0, st>>>(F, leafbox, nodes, parent, leaf_parent, flags);
    }
    return check_launch("gsr_mesh_build", false, st);
}

int gsr_mesh_first_hit(int32_t F, const void* bvh, int64_t N, const void* origins, const void* directions, int32_t f64, const int64_t* active,
                       int64_t* tri, double* t, void* stream) {
    NvtxRange nvtx_("gsr_mesh_first_hit");
    const cudaStream_t st = (cudaStream_t)stream;
    if (F < 0 || !bvh || ((uintptr_t)bvh & 255) || N < 0 || (f64 != 0 && f64 != 1) || (N > 0 && (!origins || !directions || !tri))) {
        set_error("gsr_mesh_first_hit: bad arguments (F %d, N %lld, f64 %d)", F, (long long)N, f64);
        return GSR_ERR_INVALID;
    }
    if (N == 0) return GSR_OK;
    const MeshBvh B((size_t)F);
    const char* b = (const char*)bvh;
    const MeshHeader* h = (const MeshHeader*)b;
    const MeshNode* nodes = (const MeshNode*)(b + B.nodes);
    const double* tris = (const double*)(b + B.tris);
    const int32_t* ids = (const int32_t*)(b + B.ids);
    const unsigned grid = (unsigned)((N + MESH_THREADS - 1) / MESH_THREADS);
    if (f64)
        k_first_hit<double><<<grid, MESH_THREADS, 0, st>>>(N, F, h, nodes, tris, ids, (const double*)origins, (const double*)directions, active, tri, t);
    else
        k_first_hit<float><<<grid, MESH_THREADS, 0, st>>>(N, F, h, nodes, tris, ids, (const float*)origins, (const float*)directions, active, tri, t);
    return check_launch("gsr_mesh_first_hit", false, st);
}

int gsr_mesh_inpaint_mask(int64_t N, const void* origins, const void* directions, int32_t f64, const int64_t* tri_planar, const double* t_planar,
                          const int64_t* tri_all, const double* t_all, const double* w2c, uint8_t* mask, int64_t* counts, void* stream) {
    NvtxRange nvtx_("gsr_mesh_inpaint_mask");
    const cudaStream_t st = (cudaStream_t)stream;
    if (N < 0 || (f64 != 0 && f64 != 1) || !counts || ((uintptr_t)counts & 7) ||
        (N > 0 && (!origins || !directions || !tri_planar || !t_planar || !tri_all || !t_all || !w2c || !mask))) {
        set_error("gsr_mesh_inpaint_mask: bad arguments (N %lld, f64 %d)", (long long)N, f64);
        return GSR_ERR_INVALID;
    }
    cudaMemsetAsync(counts, 0, 2 * sizeof(int64_t), st);
    if (N > 0) {
        const unsigned grid = (unsigned)((N + MESH_THREADS - 1) / MESH_THREADS);
        unsigned long long* c = (unsigned long long*)counts;
        if (f64)
            k_inpaint_mask<double><<<grid, MESH_THREADS, 0, st>>>(N, (const double*)origins, (const double*)directions, tri_planar, t_planar, tri_all,
                                                                  t_all, w2c, mask, c);
        else
            k_inpaint_mask<float><<<grid, MESH_THREADS, 0, st>>>(N, (const float*)origins, (const float*)directions, tri_planar, t_planar, tri_all,
                                                                 t_all, w2c, mask, c);
    }
    return check_launch("gsr_mesh_inpaint_mask", false, st);
}
