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
//           k_closest_morton / k_rs_hist / scan / k_rs_scatter   the queries' order along a Morton curve in the root box
//           k_closest      open3d's compute_closest_points on the same BVH: one point per thread in that order, nearer child first;
//                          Ericson's closest-point test in float64, every operation rounded on its own, smallest d2, then lowest index
//           k_isin_flags / k_isin_count / k_rs_scan / k_isin_scatter
//                          np.isin(tri, query_tri) and the boolean indexing of the melting-mesh frame, rows in their original order
// DESIGN.md §4 argues why the box tests never cull a triangle the exact tests would pick.
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

__device__ __forceinline__ double ddot(const double u[3], const double w[3]) { return dadd(dadd(dmul(u[0], w[0]), dmul(u[1], w[1])), dmul(u[2], w[2])); }

// The squared distance from p to its closest point q on triangle (a, b, c): Ericson's ClosestPtPointTriangle (Real-Time Collision
// Detection §5.1.5) in float64, every operation rounded on its own, in this order (tests/closest_ref.py restates it):
//   ab = b - a, ac = c - a, ap = p - a, bp = p - b, cp = p - c per component; dot(u, w) = (ux wx + uy wy) + uz wz
//   d1 = dot(ab, ap), d2 = dot(ac, ap)                        d1 <= 0 and d2 <= 0:                    q = a
//   d3 = dot(ab, bp), d4 = dot(ac, bp)                        d3 >= 0 and d4 <= d3:                   q = b
//   vc = d1 d4 - d3 d2                                        vc <= 0 and d1 >= 0 and d3 <= 0:        q = a + (d1 / (d1 - d3)) ab
//   d5 = dot(ab, cp), d6 = dot(ac, cp)                        d6 >= 0 and d5 <= d6:                   q = c
//   vb = d5 d2 - d1 d6                                        vb <= 0 and d2 >= 0 and d6 <= 0:        q = a + (d2 / (d2 - d6)) ac
//   va = d3 d6 - d5 d4, e = d4 - d3, f = d5 - d6              va <= 0 and e >= 0 and f >= 0:          q = b + (e / (e + f)) (c - b)
//   otherwise den = (va + vb) + vc, v = vb / den, w = vc / den:                                      q = (a + v ab) + w ac
//   and the result ((p - q)x^2 + (p - q)y^2) + (p - q)z^2, with s x = rn(s * x) and a + s x = rn(a + rn(s * x)) per component.
__device__ __forceinline__ double closest_d2(const double p[3], const double* __restrict__ t) {
    const double* a = t;
    const double* b = t + 3;
    const double* c = t + 6;
    double ab[3], ac[3], ap[3], bp[3], cp[3], q[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        ab[k] = dsub(b[k], a[k]);
        ac[k] = dsub(c[k], a[k]);
        ap[k] = dsub(p[k], a[k]);
        bp[k] = dsub(p[k], b[k]);
        cp[k] = dsub(p[k], c[k]);
    }
    const double d1 = ddot(ab, ap), d2 = ddot(ac, ap);
    const double d3 = ddot(ab, bp), d4 = ddot(ac, bp);
    const double d5 = ddot(ab, cp), d6 = ddot(ac, cp);
    const double vc = dsub(dmul(d1, d4), dmul(d3, d2));
    const double vb = dsub(dmul(d5, d2), dmul(d1, d6));
    const double va = dsub(dmul(d3, d6), dmul(d5, d4));
    const double e = dsub(d4, d3), f = dsub(d5, d6);
    if (d1 <= 0.0 && d2 <= 0.0) {
#pragma unroll
        for (int k = 0; k < 3; k++) q[k] = a[k];
    } else if (d3 >= 0.0 && d4 <= d3) {
#pragma unroll
        for (int k = 0; k < 3; k++) q[k] = b[k];
    } else if (vc <= 0.0 && d1 >= 0.0 && d3 <= 0.0) {
        const double v = __ddiv_rn(d1, dsub(d1, d3));
#pragma unroll
        for (int k = 0; k < 3; k++) q[k] = dadd(a[k], dmul(v, ab[k]));
    } else if (d6 >= 0.0 && d5 <= d6) {
#pragma unroll
        for (int k = 0; k < 3; k++) q[k] = c[k];
    } else if (vb <= 0.0 && d2 >= 0.0 && d6 <= 0.0) {
        const double w = __ddiv_rn(d2, dsub(d2, d6));
#pragma unroll
        for (int k = 0; k < 3; k++) q[k] = dadd(a[k], dmul(w, ac[k]));
    } else if (va <= 0.0 && e >= 0.0 && f >= 0.0) {
        const double w = __ddiv_rn(e, dadd(e, f));
#pragma unroll
        for (int k = 0; k < 3; k++) q[k] = dadd(b[k], dmul(w, dsub(c[k], b[k])));
    } else {
        const double den = dadd(dadd(va, vb), vc);
        const double v = __ddiv_rn(vb, den), w = __ddiv_rn(vc, den);
#pragma unroll
        for (int k = 0; k < 3; k++) q[k] = dadd(dadd(a[k], dmul(v, ab[k])), dmul(w, ac[k]));
    }
    const double ex = dsub(p[0], q[0]), ey = dsub(p[1], q[1]), ez = dsub(p[2], q[2]);
    return dadd(dadd(dmul(ex, ex), dmul(ey, ey)), dmul(ez, ez));
}

// The lower bound of the box test: the squared distance from p to the box grown by pad, per-axis gaps clamped at 0.  It never
// exceeds the computed squared distance of a valid triangle inside the box (DESIGN.md §4); an empty box gives +inf.
__device__ __forceinline__ double box_lower(const double p[3], const float* b, double pad) {
    double g[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const double lo = dsub((double)b[k], pad), hi = dadd((double)b[3 + k], pad);
        g[k] = fmax(fmax(dsub(lo, p[k]), dsub(p[k], hi)), 0.0);
    }
    return dadd(dadd(dmul(g[0], g[0]), dmul(g[1], g[1])), dmul(g[2], g[2]));
}

template <typename T>
__global__ void __launch_bounds__(MESH_THREADS) k_closest(int64_t N, int32_t F, const MeshHeader* __restrict__ hdr, const MeshNode* __restrict__ nodes,
                                                          const double* __restrict__ tris, const int32_t* __restrict__ ids,
                                                          const T* __restrict__ pts, const uint32_t* __restrict__ order,
                                                          int64_t* __restrict__ tri_out, double* __restrict__ d2_out) {
    const int64_t k = (int64_t)blockIdx.x * MESH_THREADS + threadIdx.x;
    if (k >= N) return;
    const int64_t i = order ? (int64_t)order[k] : k;  // neighbouring threads take spatially close points; results go to row i
    double best_d2 = INFINITY;
    int32_t best = -1;
    double p[3];
    bool ok = true;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        p[c] = (double)pts[3 * i + c];
        ok = ok && isfinite(p[c]);
    }
    if (ok && F > 0) {
        const double pad = dmul(0x1p-24, dadd(fmax(fmax(fabs(p[0]), fabs(p[1])), fabs(p[2])), (double)hdr->coord_max));
        // a candidate wins with a smaller d2, or the same d2 and a lower index; NaN and +inf (overflow) never win
        auto leaf = [&](int k) {
            const int32_t id = ids[k];
            if (id < 0) return;
            const double dd = closest_d2(p, tris + 9 * (size_t)k);
            if (dd < best_d2 || (dd == best_d2 && id < best)) {
                best_d2 = dd;
                best = id;
            }
        };
        // culled: a lower bound strictly above the best d2 (a tie at a lower index stays reachable), or +inf
        auto keep = [&](double lb) { return lb < INFINITY && !(lb > best_d2); };
        if (F == 1) {
            leaf(0);
        } else {
            int stack[MESH_STACK];
            int sp = 0, node = 0;
            while (true) {
                const MeshNode n = nodes[node];
                const float bl[6] = {n.a.x, n.a.y, n.a.z, n.a.w, n.b.x, n.b.y};
                const float br[6] = {n.b.z, n.b.w, n.c.x, n.c.y, n.c.z, n.c.w};
                const double kl = box_lower(p, bl, pad), kr = box_lower(p, br, pad);
                bool hl = keep(kl), hr = keep(kr);
                if (hl && n.left < 0) { leaf(~n.left); hl = false; }
                if (hr && n.right < 0) { leaf(~n.right); hr = false; }
                // the pushed child is tested again when popped: the best d2 may have shrunk meanwhile
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
    if (d2_out) d2_out[i] = best_d2;
}

// Query order for k_closest: 30-bit Morton codes of the points in the root box (float32 arithmetic, clamped; a non-finite point gets
// 0xffffffff), sorted with their row indices.  Only the order of the work changes, never a result.
template <typename T>
__global__ void __launch_bounds__(MESH_THREADS) k_closest_morton(int64_t N, const MeshNode* __restrict__ nodes, const T* __restrict__ pts,
                                                                 uint32_t* __restrict__ codes, uint32_t* __restrict__ vals) {
    const int64_t i = (int64_t)blockIdx.x * MESH_THREADS + threadIdx.x;
    if (i >= N) return;
    const MeshNode n = nodes[0];
    const float lo[3] = {fminf(n.a.x, n.b.z), fminf(n.a.y, n.b.w), fminf(n.a.z, n.c.x)};
    const float hi[3] = {fmaxf(n.a.w, n.c.y), fmaxf(n.b.x, n.c.z), fmaxf(n.b.y, n.c.w)};
    uint32_t code = 0;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float x = (float)pts[3 * i + k];
        if (!isfinite(x)) code = MESH_INVALID_CODE;
        const float ext = hi[k] - lo[k];
        float q = ext > 0.f ? (x - lo[k]) / ext * 1023.f : 0.f;
        q = fminf(fmaxf(q, 0.f), 1023.f);  // also maps NaN to 0
        if (code != MESH_INVALID_CODE) code |= mesh_spread10((uint32_t)q) << k;
    }
    codes[i] = code;
    vals[i] = (uint32_t)i;
}

struct ClosestWs {
    size_t codes0, codes1, vals0, vals1, hist, part, total;
    int nchunks;
    explicit ClosestWs(size_t N) {
        nchunks = rs_chunks(N);
        const size_t nhist = 256 * (size_t)nchunks;
        size_t o = 0;
        codes0 = o; o = align_up(o + 4 * N, 256);
        codes1 = o; o = align_up(o + 4 * N, 256);
        vals0 = o;  o = align_up(o + 4 * N, 256);
        vals1 = o;  o = align_up(o + 4 * N, 256);
        hist = o;   o = align_up(o + 4 * nhist, 256);
        part = o;   o = align_up(o + 4 * scan_parts(nhist), 256);
        total = o;
    }
};

constexpr int ISIN_THREADS = 256;
constexpr int ISIN_ROUNDS = 4;  // a block selects from ISIN_ROUNDS * ISIN_THREADS consecutive rows
constexpr int ISIN_TILE = ISIN_THREADS * ISIN_ROUNDS;
constexpr int ISIN_MAX_ARRAYS = 8;

struct IsinArrays {
    const uint32_t* src[ISIN_MAX_ARRAYS];
    uint32_t* dst[ISIN_MAX_ARRAYS];
    int32_t words[ISIN_MAX_ARRAYS];
    int32_t K;
};

__global__ void __launch_bounds__(ISIN_THREADS) k_isin_flags(int64_t Q, const int64_t* __restrict__ query, int32_t F, uint8_t* __restrict__ flags) {
    const int64_t j = (int64_t)blockIdx.x * ISIN_THREADS + threadIdx.x;
    if (j >= Q) return;
    const int64_t t = query[j];
    if (t >= 0 && t < F) flags[t] = 1;
}

__device__ __forceinline__ bool isin_keep(int64_t N, const int64_t* __restrict__ tri, int32_t F, const uint8_t* __restrict__ flags, int64_t i) {
    if (i >= N) return false;
    const int64_t t = tri[i];
    return t >= 0 && t < F && flags[t] != 0;
}

// Kept rows per tile; block_counts[tiles] is the scan's extra entry, which becomes the total.
__global__ void __launch_bounds__(ISIN_THREADS) k_isin_count(int64_t N, const int64_t* __restrict__ tri, int32_t F, const uint8_t* __restrict__ flags,
                                                             uint32_t* __restrict__ block_counts, int tiles) {
    __shared__ uint32_t warp_n[ISIN_THREADS / 32];
    const int64_t base = (int64_t)blockIdx.x * ISIN_TILE;
    uint32_t n = 0;
#pragma unroll
    for (int r = 0; r < ISIN_ROUNDS; r++) n += isin_keep(N, tri, F, flags, base + r * ISIN_THREADS + threadIdx.x) ? 1u : 0u;
    n = __reduce_add_sync(GSR_FULL, n);
    if ((threadIdx.x & 31) == 0) warp_n[threadIdx.x >> 5] = n;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t s = 0;
        for (int w = 0; w < ISIN_THREADS / 32; w++) s += warp_n[w];
        block_counts[blockIdx.x] = s;
        if (blockIdx.x == 0) block_counts[tiles] = 0u;
    }
}

// Every kept row i goes to its rank among the kept rows (block offset + rank inside the tile), in row order; words are copied as
// integers, so every bit pattern arrives unchanged, as with t[mask].
__global__ void __launch_bounds__(ISIN_THREADS) k_isin_scatter(int64_t N, const int64_t* __restrict__ tri, int32_t F, const uint8_t* __restrict__ flags,
                                                               const uint32_t* __restrict__ offsets, int tiles, IsinArrays A,
                                                               int64_t* __restrict__ count) {
    __shared__ uint32_t warp_n[ISIN_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t base = (int64_t)blockIdx.x * ISIN_TILE;
    uint32_t run = offsets[blockIdx.x];
    for (int r = 0; r < ISIN_ROUNDS; r++) {
        const int64_t i = base + r * ISIN_THREADS + threadIdx.x;
        const bool k = isin_keep(N, tri, F, flags, i);
        const unsigned bal = __ballot_sync(GSR_FULL, k);
        if (lane == 0) warp_n[warp] = __popc(bal);
        __syncthreads();
        uint32_t before = 0, total = 0;
        for (int w = 0; w < ISIN_THREADS / 32; w++) {
            const uint32_t c = warp_n[w];
            before += w < warp ? c : 0u;
            total += c;
        }
        if (k) {
            const int64_t o = (int64_t)run + before + __popc(bal & ((1u << lane) - 1u));
            for (int a = 0; a < A.K; a++) {
                const int w = A.words[a];
                for (int c = 0; c < w; c++) A.dst[a][o * w + c] = A.src[a][i * w + c];
            }
        }
        run += total;
        __syncthreads();  // warp_n is rewritten by the next round
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *count = (int64_t)offsets[tiles];
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

size_t gsr_mesh_closest_bytes(int64_t N) { return N < 0 || N > 0x7fffffffLL ? 0 : ClosestWs((size_t)N).total; }

int gsr_mesh_closest(int32_t F, const void* bvh, int64_t N, const void* points, int32_t f64, int64_t* tri, double* d2, void* ws, size_t ws_bytes,
                     void* stream) {
    NvtxRange nvtx_("gsr_mesh_closest");
    const cudaStream_t st = (cudaStream_t)stream;
    if (F < 0 || !bvh || ((uintptr_t)bvh & 255) || N < 0 || N > 0x7fffffffLL || (f64 != 0 && f64 != 1) || (N > 0 && (!points || !tri))) {
        set_error("gsr_mesh_closest: bad arguments (F %d, N %lld, f64 %d)", F, (long long)N, f64);
        return GSR_ERR_INVALID;
    }
    const ClosestWs L((size_t)N);
    if (!ws || ((uintptr_t)ws & 255) || ws_bytes < L.total) {
        set_error("gsr_mesh_closest: workspace of %zu bytes, gsr_mesh_closest_bytes(%lld) = %zu needed (256-byte aligned)", ws_bytes, (long long)N,
                  L.total);
        return GSR_ERR_WORKSPACE;
    }
    if (N == 0) return GSR_OK;
    const MeshBvh B((size_t)F);
    const char* b = (const char*)bvh;
    const MeshHeader* h = (const MeshHeader*)b;
    const MeshNode* nodes = (const MeshNode*)(b + B.nodes);
    const double* tris = (const double*)(b + B.tris);
    const int32_t* ids = (const int32_t*)(b + B.ids);
    const unsigned grid = (unsigned)((N + MESH_THREADS - 1) / MESH_THREADS);
    const uint32_t* order = nullptr;
    if (F > 1) {  // sort the queries along a Morton curve (DESIGN.md §4: trained models keep their rows in no spatial order)
        char* w = (char*)ws;
        uint32_t *k0 = (uint32_t*)(w + L.codes0), *k1 = (uint32_t*)(w + L.codes1), *v0 = (uint32_t*)(w + L.vals0), *v1 = (uint32_t*)(w + L.vals1);
        uint32_t *hist = (uint32_t*)(w + L.hist), *part = (uint32_t*)(w + L.part);
        if (f64)
            k_closest_morton<double><<<grid, MESH_THREADS, 0, st>>>(N, nodes, (const double*)points, k0, v0);
        else
            k_closest_morton<float><<<grid, MESH_THREADS, 0, st>>>(N, nodes, (const float*)points, k0, v0);
        const int rs_blocks = (L.nchunks + RS_WARPS - 1) / RS_WARPS;
        for (int shift = 0; shift < 32; shift += 8) {
            k_rs_hist<<<rs_blocks, RS_WARPS * 32, 0, st>>>((uint32_t)N, k0, shift, L.nchunks, hist);
            scan_wide(hist, 256 * (size_t)L.nchunks, part, st);
            k_rs_scatter<<<rs_blocks, RS_WARPS * 32, 0, st>>>((uint32_t)N, k0, v0, shift, L.nchunks, hist, k1, v1);
            uint32_t* t = k0; k0 = k1; k1 = t;
            t = v0; v0 = v1; v1 = t;
        }
        order = v0;
    }
    if (f64)
        k_closest<double><<<grid, MESH_THREADS, 0, st>>>(N, F, h, nodes, tris, ids, (const double*)points, order, tri, d2);
    else
        k_closest<float><<<grid, MESH_THREADS, 0, st>>>(N, F, h, nodes, tris, ids, (const float*)points, order, tri, d2);
    return check_launch("gsr_mesh_closest", false, st);
}

static int isin_tiles(int64_t N) { return (int)((N + ISIN_TILE - 1) / ISIN_TILE); }

size_t gsr_mesh_isin_rows_bytes(int64_t N, int32_t F) {
    if (N < 0 || N > 0x7fffffffLL || F < 0) return 0;
    return align_up((size_t)F, 256) + ((size_t)isin_tiles(N) + 1) * sizeof(uint32_t);
}

int gsr_mesh_isin_rows(int64_t N, const int64_t* tri, int64_t Q, const int64_t* query_tri, int32_t F, int32_t K, const void* const* src,
                       void* const* dst, const int32_t* words, int64_t* count, void* ws, size_t ws_bytes, void* stream) {
    NvtxRange nvtx_("gsr_mesh_isin_rows");
    const cudaStream_t st = (cudaStream_t)stream;
    if (N < 0 || N > 0x7fffffffLL || Q < 0 || F < 0 || K < 0 || K > ISIN_MAX_ARRAYS || !count || ((uintptr_t)count & 7) ||
        (N > 0 && !tri) || (Q > 0 && !query_tri) || (K > 0 && (!src || !dst || !words))) {
        set_error("gsr_mesh_isin_rows: bad arguments (N %lld, Q %lld, F %d, K %d)", (long long)N, (long long)Q, F, K);
        return GSR_ERR_INVALID;
    }
    IsinArrays A{};
    A.K = K;
    for (int a = 0; a < K; a++) {
        if (words[a] < 0 || (words[a] > 0 && N > 0 && (!src[a] || !dst[a]))) {
            set_error("gsr_mesh_isin_rows: array %d has %d words per row or a NULL pointer", a, words[a]);
            return GSR_ERR_INVALID;
        }
        A.src[a] = (const uint32_t*)src[a];
        A.dst[a] = (uint32_t*)dst[a];
        A.words[a] = words[a];
    }
    if (!ws || ((uintptr_t)ws & 3) || ws_bytes < gsr_mesh_isin_rows_bytes(N, F)) {
        set_error("gsr_mesh_isin_rows: workspace of %zu bytes, gsr_mesh_isin_rows_bytes(%lld, %d) = %zu needed (4-byte aligned)", ws_bytes,
                  (long long)N, F, gsr_mesh_isin_rows_bytes(N, F));
        return GSR_ERR_WORKSPACE;
    }
    if (N == 0) {
        cudaMemsetAsync(count, 0, sizeof(int64_t), st);
        return check_launch("gsr_mesh_isin_rows", false, st);
    }
    uint8_t* flags = (uint8_t*)ws;
    uint32_t* counts = (uint32_t*)((char*)ws + align_up((size_t)F, 256));
    if (F > 0) cudaMemsetAsync(flags, 0, (size_t)F, st);
    if (F > 0 && Q > 0) k_isin_flags<<<(unsigned)((Q + ISIN_THREADS - 1) / ISIN_THREADS), ISIN_THREADS, 0, st>>>(Q, query_tri, F, flags);
    const int tiles = isin_tiles(N);
    k_isin_count<<<tiles, ISIN_THREADS, 0, st>>>(N, tri, F, flags, counts, tiles);
    k_rs_scan<uint32_t><<<1, 1024, 0, st>>>(counts, tiles + 1);
    k_isin_scatter<<<tiles, ISIN_THREADS, 0, st>>>(N, tri, F, flags, counts, tiles, A, count);
    return check_launch("gsr_mesh_isin_rows", false, st);
}
