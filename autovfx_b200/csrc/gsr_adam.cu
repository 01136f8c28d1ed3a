// gsr_b200 Adam step: torch.optim.Adam's default (foreach) update of every parameter and both moments in one launch
// (torch/optim/adam.py:_multi_tensor_adam, the path of `torch.optim.Adam(l, lr=0.0, eps=1e-15)` in every trainer of the
// reference: GS/train.py:183-184, scene_representation.py:538-540, sugar_trainers/coarse_density.py:822).
//
//   k_adam   one grid-stride pass over the concatenated tensors, 4 elements per item: float4 loads and stores where all four
//            tensors of a descriptor are 16-byte aligned, scalar elements elsewhere and in each tensor's tail.
//
// torch runs the update as seven list ops, each rounding to float32 through memory.  Each is restated with explicit intrinsics so
// that nvcc contracts nothing across those roundings (as read from torch's own SASS and ATen/native/cuda/DeviceAddCmulCdiv.cuh):
//   _foreach_lerp_(m, g, w)          at::native::lerp: |w| < 0.5 ? fma(g - m, w, m) : fma(-(1 - w), g - m, g)
//   _foreach_mul_(v, beta2)          v * beta2
//   _foreach_addcmul_(v, g, g, c)    fma(c, g * g, v), or fma(g, g, v) when c == 1      (pointwise_op_impl)
//   _foreach_sqrt                    IEEE square root
//   _foreach_div_(s, bc2_sqrt)       IEEE division (MUFU.RCP + FCHK + slow path in torch's build, not a reciprocal multiply)
//   _foreach_add_(s, eps)            s + eps
//   _foreach_addcdiv_(p, m, s, a)    fma(a, m / s, p), or p + m / s when a == 1          (pointwise_op_impl)
// The per-tensor scalars are the host's Python doubles rounded to float, as the foreach kernels receive them.  NaN and Inf
// propagate through these operations exactly as in torch; nothing is guarded.
#include "gsr_common.cuh"

namespace gsr {

namespace {

constexpr int ADAM_BLOCK = 256;

struct AdamArgs {
    int n;
    uint32_t vec;                           // bit t: all four pointers of tensor t are 16-byte aligned
    int64_t start[GSR_ADAM_MAX_TENSORS + 1];  // first item (4 elements) of each tensor; start[n] = total
    gsr_adam_tensor t[GSR_ADAM_MAX_TENSORS];
};

struct AdamScalars {
    float w, one_minus_w, beta2, c, bc2, eps, a;
    bool small_w, c_one, a_one;
};

__device__ __forceinline__ AdamScalars adam_scalars(const gsr_adam_tensor& T) {
    AdamScalars s;
    s.w = T.lerp_weight;
    s.one_minus_w = __fsub_rn(1.0f, T.lerp_weight);
    s.small_w = fabsf(T.lerp_weight) < 0.5f;
    s.beta2 = T.beta2;
    s.c = T.one_minus_beta2;
    s.c_one = T.one_minus_beta2 == 1.0f;
    s.bc2 = T.bias_correction2_sqrt;
    s.eps = T.eps;
    s.a = T.step_size;
    s.a_one = T.step_size == 1.0f;
    return s;
}

__device__ __forceinline__ void adam_elem(const AdamScalars& s, float& p, float g, float& m, float& v) {
    const float d = __fsub_rn(g, m);
    m = s.small_w ? __fmaf_rn(d, s.w, m) : __fmaf_rn(-s.one_minus_w, d, g);
    v = __fmul_rn(v, s.beta2);
    v = s.c_one ? __fmaf_rn(g, g, v) : __fmaf_rn(s.c, __fmul_rn(g, g), v);
    float den = __fsqrt_rn(v);
    den = __fdiv_rn(den, s.bc2);
    den = __fadd_rn(den, s.eps);
    const float q = __fdiv_rn(m, den);
    p = s.a_one ? __fadd_rn(p, q) : __fmaf_rn(s.a, q, p);
}

// one 16-byte store: nvcc split a float4 assignment here into four 4-byte stores
__device__ __forceinline__ void st4(float* ptr, const float (&x)[4]) {
    asm volatile("st.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(ptr), "f"(x[0]), "f"(x[1]), "f"(x[2]), "f"(x[3]) : "memory");
}

__global__ void __launch_bounds__(ADAM_BLOCK) k_adam(const __grid_constant__ AdamArgs a) {
    const int64_t total = a.start[a.n];
    const int64_t stride = (int64_t)gridDim.x * ADAM_BLOCK;
    int t = 0;
    for (int64_t i = (int64_t)blockIdx.x * ADAM_BLOCK + threadIdx.x; i < total; i += stride) {
        while (i >= a.start[t + 1]) ++t;  // items only grow along the loop: the tensor index only moves forward
        const gsr_adam_tensor& T = a.t[t];
        const AdamScalars s = adam_scalars(T);
        const int64_t e = (i - a.start[t]) * 4;
        const int64_t rem = T.numel - e;
        if (rem >= 4 && ((a.vec >> t) & 1u)) {
            const float4 p4 = *reinterpret_cast<const float4*>(T.param + e);
            const float4 g = __ldg(reinterpret_cast<const float4*>(T.grad + e));
            const float4 m4 = *reinterpret_cast<const float4*>(T.exp_avg + e);
            const float4 v4 = *reinterpret_cast<const float4*>(T.exp_avg_sq + e);
            float p[4] = {p4.x, p4.y, p4.z, p4.w}, m[4] = {m4.x, m4.y, m4.z, m4.w}, v[4] = {v4.x, v4.y, v4.z, v4.w};
            const float gg[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) adam_elem(s, p[k], gg[k], m[k], v[k]);
            st4(T.param + e, p);
            st4(T.exp_avg + e, m);
            st4(T.exp_avg_sq + e, v);
        } else {
            const int k_end = rem < 4 ? (int)rem : 4;
            for (int k = 0; k < k_end; ++k) {
                float p = T.param[e + k], m = T.exp_avg[e + k], v = T.exp_avg_sq[e + k];
                adam_elem(s, p, __ldg(T.grad + e + k), m, v);
                T.param[e + k] = p;
                T.exp_avg[e + k] = m;
                T.exp_avg_sq[e + k] = v;
            }
        }
    }
}

bool aligned16(const void* ptr) { return ((uintptr_t)ptr & 15u) == 0; }

// one wave of resident CTAs on the current device (cached per device): the grid-stride loop covers the rest
int adam_grid_cap() {
    static int cap[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132 * 8;
    if (cap[dev] == 0) {
        int sms = 0, per_sm = 0;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_adam, ADAM_BLOCK, 0);
        cap[dev] = sms > 0 && per_sm > 0 ? sms * per_sm : 132 * 8;
    }
    return cap[dev];
}

}  // namespace
}  // namespace gsr

using namespace gsr;

int gsr_adam_step(int32_t n, const gsr_adam_tensor* tensors, void* stream) {
    NvtxRange nvtx_("gsr_adam_step");
    const cudaStream_t st = (cudaStream_t)stream;
    if (n < 0 || (n > 0 && !tensors)) {
        set_error("gsr_adam_step: %d tensors", n);
        return GSR_ERR_INVALID;
    }
    for (int i = 0; i < n; ++i) {
        const gsr_adam_tensor& T = tensors[i];
        if (T.numel < 0 || (T.numel > 0 && (!T.param || !T.grad || !T.exp_avg || !T.exp_avg_sq))) {
            set_error("gsr_adam_step: tensor %d is malformed (numel %lld)", i, (long long)T.numel);
            return GSR_ERR_INVALID;
        }
    }
    if (n == 0) return GSR_OK;
    const int64_t cap = adam_grid_cap();
    // descriptors travel in the kernel parameters: one launch per GSR_ADAM_MAX_TENSORS of them
    for (int first = 0; first < n; first += GSR_ADAM_MAX_TENSORS) {
        AdamArgs a{};
        a.n = n - first < GSR_ADAM_MAX_TENSORS ? n - first : GSR_ADAM_MAX_TENSORS;
        int64_t items = 0;
        for (int k = 0; k < a.n; ++k) {
            const gsr_adam_tensor& T = tensors[first + k];
            a.t[k] = T;
            a.start[k] = items;
            items += (T.numel + 3) / 4;
            if (aligned16(T.param) && aligned16(T.grad) && aligned16(T.exp_avg) && aligned16(T.exp_avg_sq)) a.vec |= 1u << k;
        }
        a.start[a.n] = items;
        if (items == 0) continue;
        const int64_t blocks = (items + ADAM_BLOCK - 1) / ADAM_BLOCK;
        k_adam<<<(unsigned)(blocks < cap ? blocks : cap), ADAM_BLOCK, 0, st>>>(a);
        const int rc = check_launch("gsr_adam_step", false, st);
        if (rc != GSR_OK) return rc;
    }
    return GSR_OK;
}
