// Fused optimizer kernels for sm_90a: Adam/AdamW, Lion, LAMB, Adagrad, SGD(momentum), plus the
// gradient utilities that surround them in a ZeRO step (sum-of-squares + inf/nan scan, scale).
//
// Role parity: reference csrc/adam/multi_tensor_adam.cu (N1), csrc/lion/multi_tensor_lion.cu and
// csrc/lamb/fused_lamb_cuda_kernel.cu (N4).  Design differences (H100-first):
//   * ZeRO keeps each rank's shard as ONE flat buffer, so the primary entry points are flat
//     kernels moving 8 elements / thread / iteration with 16-byte streaming accesses; the
//     multi-tensor variant walks a device-resident chunk table (no 4 KB kernel-arg struct, no
//     re-launch every 320 blocks).
//   * mixed precision in one pass: fp32 master/m/v are updated and the bf16/fp16 model copy is
//     written by the same kernel (the reference runs a separate fp32->bf16 copy kernel).
//   * the combined unscale*clip factor and the overflow "skip" flag are read from device memory,
//     so the step needs no host synchronisation and can be captured in a CUDA graph.
#include "dsb_common.cuh"

namespace dsb {

template <typename T>
__device__ __forceinline__ void load8(const T* p, float* out);
template <>
__device__ __forceinline__ void load8<float>(const float* p, float* out)
{
    Vec16 a = ld_stream(p), b = ld_stream(p + 4);
    Elem<float>::unpack(a, out);
    Elem<float>::unpack(b, out + 4);
}
template <>
__device__ __forceinline__ void load8<__nv_bfloat16>(const __nv_bfloat16* p, float* out)
{
    Elem<__nv_bfloat16>::unpack(ld_stream(p), out);
}
template <>
__device__ __forceinline__ void load8<__half>(const __half* p, float* out)
{
    Elem<__half>::unpack(ld_stream(p), out);
}

template <typename T>
__device__ __forceinline__ void store8(T* p, const float* in);
template <>
__device__ __forceinline__ void store8<float>(float* p, const float* in)
{
    st_stream(p, Elem<float>::pack(in));
    st_stream(p + 4, Elem<float>::pack(in + 4));
}
template <>
__device__ __forceinline__ void store8<__nv_bfloat16>(__nv_bfloat16* p, const float* in)
{
    st_stream(p, Elem<__nv_bfloat16>::pack(in));
}
template <>
__device__ __forceinline__ void store8<__half>(__half* p, const float* in)
{
    st_stream(p, Elem<__half>::pack(in));
}

struct AdamArgs {
    float lr, beta1, beta2, eps, weight_decay;
    float bc1, bc2;       // bias corrections 1-beta^t (1.0 when disabled)
    int adamw;            // 1 = decoupled weight decay, 0 = L2 into the gradient
    float grad_scale;     // host-side multiplier applied to the gradient (1/loss_scale etc.)
};

__device__ __forceinline__ void adam_math(float& p, float& m, float& v, float g, const AdamArgs& a,
                                          float gs)
{
    g *= gs;
    if (!a.adamw) g = fmaf(a.weight_decay, p, g);
    m = fmaf(a.beta1, m, (1.f - a.beta1) * g);
    v = fmaf(a.beta2, v, (1.f - a.beta2) * g * g);
    const float mh = m / a.bc1;
    const float vh = v / a.bc2;
    float upd = mh / (sqrtf(vh) + a.eps);
    if (a.adamw) upd = fmaf(a.weight_decay, p, upd);
    p = fmaf(-a.lr, upd, p);
}

// Grid-stride scalar form of adam_flat_kernel for pointers that are not 16-byte aligned.  Kept out of line:
// inlined, it made ptxas spill 8 bytes in the fp32-master kernels' vector path.
template <typename PT, typename GT, typename ST, typename OT, bool kHasOut>
__device__ __noinline__ void adam_flat_scalar(PT* __restrict__ p, const GT* __restrict__ g, ST* __restrict__ m,
                                              ST* __restrict__ v, OT* __restrict__ out, int64_t n, AdamArgs a,
                                              float gs)
{
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        float pf = Elem<PT>::to_f(p[i]), mf = Elem<ST>::to_f(m[i]), vf = Elem<ST>::to_f(v[i]);
        adam_math(pf, mf, vf, Elem<GT>::to_f(g[i]), a, gs);
        p[i] = Elem<PT>::from_f(pf);
        m[i] = Elem<ST>::from_f(mf);
        v[i] = Elem<ST>::from_f(vf);
        if (kHasOut) out[i] = Elem<OT>::from_f(pf);
    }
}

// PT: master/param dtype, GT: grad dtype, ST: state dtype, OT: low-precision copy dtype.
template <typename PT, typename GT, typename ST, typename OT, bool kHasOut>
__global__ void __launch_bounds__(256) adam_flat_kernel(PT* __restrict__ p, const GT* __restrict__ g,
                                                         ST* __restrict__ m, ST* __restrict__ v,
                                                         OT* __restrict__ out, int64_t n, AdamArgs a,
                                                         const float* __restrict__ d_gscale,
                                                         const int* __restrict__ d_skip)
{
    if (d_skip != nullptr && *d_skip != 0) return;
    const float gs = a.grad_scale * (d_gscale ? *d_gscale : 1.f);
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    // The 16-byte vector path needs every pointer 16-byte aligned (ZeRO arenas are; arbitrary views of
    // them need not be).  The test is uniform across the grid, so a misaligned call runs the scalar loop.
    const bool aligned = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) |
                           reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v) |
                           reinterpret_cast<uintptr_t>(out)) & 15) == 0;
    if (!aligned) {
        adam_flat_scalar<PT, GT, ST, OT, kHasOut>(p, g, m, v, out, n, a, gs);
        return;
    }
    const int64_t n8 = n >> 3;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8; i += stride) {
        const int64_t o = i << 3;
        float pf[8], gf[8], mf[8], vf[8];
        load8<PT>(p + o, pf);
        load8<GT>(g + o, gf);
        load8<ST>(m + o, mf);
        load8<ST>(v + o, vf);
#pragma unroll
        for (int k = 0; k < 8; ++k) adam_math(pf[k], mf[k], vf[k], gf[k], a, gs);
        store8<PT>(p + o, pf);
        store8<ST>(m + o, mf);
        store8<ST>(v + o, vf);
        if (kHasOut) store8<OT>(out + o, pf);
    }
    // tail (< 8 elements) handled by the first threads of block 0
    if (blockIdx.x == 0) {
        const int64_t t = (n8 << 3) + threadIdx.x;
        if (t < n) {
            float pf = Elem<PT>::to_f(p[t]), mf = Elem<ST>::to_f(m[t]), vf = Elem<ST>::to_f(v[t]);
            adam_math(pf, mf, vf, Elem<GT>::to_f(g[t]), a, gs);
            p[t] = Elem<PT>::from_f(pf);
            m[t] = Elem<ST>::from_f(mf);
            v[t] = Elem<ST>::from_f(vf);
            if (kHasOut) out[t] = Elem<OT>::from_f(pf);
        }
    }
}

// ---- multi-tensor: a device chunk table {tensor, start} drives the same math ------------------
struct TensorDesc {
    void* p;
    const void* g;
    void* m;
    void* v;
    void* out;  // may be null
    int64_t n;
};
struct ChunkDesc {
    int32_t tensor;
    int32_t pad;
    int64_t start;
};
constexpr int kChunkElems = 65536;

template <typename PT, typename GT, typename ST, typename OT>
__global__ void __launch_bounds__(256) adam_multi_kernel(const TensorDesc* __restrict__ tensors,
                                                          const ChunkDesc* __restrict__ chunks,
                                                          AdamArgs a, const float* __restrict__ d_gscale,
                                                          const int* __restrict__ d_skip)
{
    if (d_skip != nullptr && *d_skip != 0) return;
    const float gs = a.grad_scale * (d_gscale ? *d_gscale : 1.f);
    const ChunkDesc c = chunks[blockIdx.x];
    const TensorDesc t = tensors[c.tensor];
    PT* p = static_cast<PT*>(t.p) + c.start;
    const GT* g = static_cast<const GT*>(t.g) + c.start;
    ST* m = static_cast<ST*>(t.m) + c.start;
    ST* v = static_cast<ST*>(t.v) + c.start;
    OT* out = t.out ? static_cast<OT*>(t.out) + c.start : nullptr;
    int64_t len = t.n - c.start;
    if (len > kChunkElems) len = kChunkElems;
    // Vector path only when every pointer is 16-byte aligned.
    const bool aligned = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) |
                           reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v) |
                           reinterpret_cast<uintptr_t>(out)) & 15) == 0;
    int64_t done = 0;
    if (aligned) {
        const int64_t n8 = len >> 3;
        for (int64_t i = threadIdx.x; i < n8; i += blockDim.x) {
            const int64_t o = i << 3;
            float pf[8], gf[8], mf[8], vf[8];
            load8<PT>(p + o, pf);
            load8<GT>(g + o, gf);
            load8<ST>(m + o, mf);
            load8<ST>(v + o, vf);
#pragma unroll
            for (int k = 0; k < 8; ++k) adam_math(pf[k], mf[k], vf[k], gf[k], a, gs);
            store8<PT>(p + o, pf);
            store8<ST>(m + o, mf);
            store8<ST>(v + o, vf);
            if (out) store8<OT>(out + o, pf);
        }
        done = n8 << 3;
    }
    for (int64_t i = done + threadIdx.x; i < len; i += blockDim.x) {
        float pf = Elem<PT>::to_f(p[i]), mf = Elem<ST>::to_f(m[i]), vf = Elem<ST>::to_f(v[i]);
        adam_math(pf, mf, vf, Elem<GT>::to_f(g[i]), a, gs);
        p[i] = Elem<PT>::from_f(pf);
        m[i] = Elem<ST>::from_f(mf);
        v[i] = Elem<ST>::from_f(vf);
        if (out) out[i] = Elem<OT>::from_f(pf);
    }
}

// ---- Lion --------------------------------------------------------------------------------------
struct LionArgs {
    float lr, beta1, beta2, weight_decay, grad_scale;
};

template <typename PT, typename GT, typename ST, typename OT, bool kHasOut>
__global__ void __launch_bounds__(256) lion_flat_kernel(PT* __restrict__ p, const GT* __restrict__ g,
                                                         ST* __restrict__ m, OT* __restrict__ out, int64_t n,
                                                         LionArgs a, const float* __restrict__ d_gscale,
                                                         const int* __restrict__ d_skip)
{
    if (d_skip != nullptr && *d_skip != 0) return;
    const float gs = a.grad_scale * (d_gscale ? *d_gscale : 1.f);
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        float pf = Elem<PT>::to_f(p[i]);
        float mf = Elem<ST>::to_f(m[i]);
        const float gf = Elem<GT>::to_f(g[i]) * gs;
        const float c = fmaf(a.beta1, mf, (1.f - a.beta1) * gf);
        const float sgn = (c > 0.f) ? 1.f : ((c < 0.f) ? -1.f : 0.f);
        pf = pf * (1.f - a.lr * a.weight_decay) - a.lr * sgn;
        mf = fmaf(a.beta2, mf, (1.f - a.beta2) * gf);
        p[i] = Elem<PT>::from_f(pf);
        m[i] = Elem<ST>::from_f(mf);
        if (kHasOut) out[i] = Elem<OT>::from_f(pf);
    }
}

// ---- Adagrad / SGD -----------------------------------------------------------------------------
template <typename PT, typename GT, typename OT, bool kHasOut>
__global__ void __launch_bounds__(256) adagrad_flat_kernel(PT* __restrict__ p, const GT* __restrict__ g,
                                                            float* __restrict__ h, OT* __restrict__ out,
                                                            int64_t n, float lr, float eps, float wd,
                                                            float grad_scale)
{
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        float pf = Elem<PT>::to_f(p[i]);
        float gf = Elem<GT>::to_f(g[i]) * grad_scale;
        gf = fmaf(wd, pf, gf);
        const float hf = h[i] + gf * gf;
        pf -= lr * gf / (sqrtf(hf) + eps);
        h[i] = hf;
        p[i] = Elem<PT>::from_f(pf);
        if (kHasOut) out[i] = Elem<OT>::from_f(pf);
    }
}

template <typename PT, typename GT, typename OT, bool kHasOut>
__global__ void __launch_bounds__(256) sgd_flat_kernel(PT* __restrict__ p, const GT* __restrict__ g,
                                                        float* __restrict__ buf, OT* __restrict__ out,
                                                        int64_t n, float lr, float momentum, float dampening,
                                                        float wd, int nesterov, int first, float grad_scale)
{
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        float pf = Elem<PT>::to_f(p[i]);
        float gf = Elem<GT>::to_f(g[i]) * grad_scale;
        gf = fmaf(wd, pf, gf);
        if (momentum != 0.f) {
            float b = first ? gf : fmaf(momentum, buf[i], (1.f - dampening) * gf);
            buf[i] = b;
            gf = nesterov ? fmaf(momentum, b, gf) : b;
        }
        pf -= lr * gf;
        p[i] = Elem<PT>::from_f(pf);
        if (kHasOut) out[i] = Elem<OT>::from_f(pf);
    }
}

// ---- LAMB: phase 1 computes the Adam direction + per-block |p|^2, |u|^2; phase 2 applies --------
template <typename PT, typename GT>
__global__ void __launch_bounds__(256) lamb_phase1_kernel(const PT* __restrict__ p, const GT* __restrict__ g,
                                                           float* __restrict__ m, float* __restrict__ v,
                                                           float* __restrict__ upd, int64_t n, AdamArgs a,
                                                           float* __restrict__ partials /*[grid][2]*/)
{
    __shared__ float scratch[64];
    float sp = 0.f, su = 0.f;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float pf = Elem<PT>::to_f(p[i]);
        float gf = Elem<GT>::to_f(g[i]) * a.grad_scale;
        float mf = fmaf(a.beta1, m[i], (1.f - a.beta1) * gf);
        float vf = fmaf(a.beta2, v[i], (1.f - a.beta2) * gf * gf);
        m[i] = mf;
        v[i] = vf;
        float u = (mf / a.bc1) / (sqrtf(vf / a.bc2) + a.eps);
        u = fmaf(a.weight_decay, pf, u);
        upd[i] = u;
        sp = fmaf(pf, pf, sp);
        su = fmaf(u, u, su);
    }
    float2 r = block_reduce_sum2(sp, su, scratch);
    if (threadIdx.x == 0) {
        partials[2 * blockIdx.x] = r.x;
        partials[2 * blockIdx.x + 1] = r.y;
    }
}

template <typename PT, typename OT, bool kHasOut>
__global__ void __launch_bounds__(256) lamb_phase2_kernel(PT* __restrict__ p, const float* __restrict__ upd,
                                                           OT* __restrict__ out, int64_t n, float lr,
                                                           const float* __restrict__ partials, int nparts,
                                                           float max_coeff, float min_coeff,
                                                           float* __restrict__ coeff_out)
{
    __shared__ float scratch[64];
    // every block re-reduces the (small) partial array: deterministic, no extra launch
    float sp = 0.f, su = 0.f;
    for (int i = threadIdx.x; i < nparts; i += blockDim.x) {
        sp += partials[2 * i];
        su += partials[2 * i + 1];
    }
    float2 r = block_reduce_sum2(sp, su, scratch);
    const float pn = sqrtf(r.x), un = sqrtf(r.y);
    float coeff = 1.f;
    if (pn != 0.f && un != 0.f) coeff = fminf(fmaxf(pn / un, min_coeff), max_coeff);
    if (blockIdx.x == 0 && threadIdx.x == 0 && coeff_out) *coeff_out = coeff;
    const float step = lr * coeff;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        float pf = Elem<PT>::to_f(p[i]) - step * upd[i];
        p[i] = Elem<PT>::from_f(pf);
        if (kHasOut) out[i] = Elem<OT>::from_f(pf);
    }
}

// ---- gradient utilities ------------------------------------------------------------------------
// Per-block partial sum of squares + sticky inf/nan flag.  A second launch (or the consumer)
// reduces the partials deterministically.
template <typename T>
__global__ void __launch_bounds__(512) sumsq_partial_kernel(const T* __restrict__ x, int64_t n,
                                                             float* __restrict__ partials,
                                                             int* __restrict__ found_inf)
{
    __shared__ float scratch[32];
    constexpr int kPer = Elem<T>::kPerVec;
    float acc = 0.f;
    bool bad = false;
    const int64_t nv = n / kPer;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    const bool aligned = (reinterpret_cast<uintptr_t>(x) & 15) == 0;
    int64_t done = 0;
    if (aligned) {
        for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nv; i += stride) {
            float f[kPer];
            Elem<T>::unpack(ld_stream(x + i * kPer), f);
#pragma unroll
            for (int k = 0; k < kPer; ++k) {
                acc = fmaf(f[k], f[k], acc);
                bad |= !isfinite(f[k]);
            }
        }
        done = nv * kPer;
    }
    for (int64_t i = done + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float f = Elem<T>::to_f(x[i]);
        acc = fmaf(f, f, acc);
        bad |= !isfinite(f);
    }
    acc = block_reduce<SumOp>(acc, scratch);
    if (threadIdx.x == 0) partials[blockIdx.x] = acc;
    if (bad && found_inf) atomicOr(found_inf, 1);
}

// out[0] (+)= sum(partials); single block, fixed order => deterministic.
__global__ void __launch_bounds__(1024) reduce_partials_kernel(const float* __restrict__ partials, int n,
                                                                float* __restrict__ out, int accumulate)
{
    __shared__ float scratch[32];
    float acc = 0.f;
    for (int i = threadIdx.x; i < n; i += blockDim.x) acc += partials[i];
    acc = block_reduce<SumOp>(acc, scratch);
    if (threadIdx.x == 0) out[0] = accumulate ? out[0] + acc : acc;
}

// Device-side clip coefficient: gscale = (1/loss_scale) * min(1, max_norm / (norm/loss_scale + eps));
// skip = found_inf.  Keeps the whole unscale/clip/overflow decision off the host.
__global__ void clip_coeff_kernel(const float* __restrict__ sumsq, const int* __restrict__ found_inf,
                                  float inv_loss_scale, float max_norm, float* __restrict__ gscale,
                                  int* __restrict__ skip, float* __restrict__ norm_out)
{
    const float ss = *sumsq;
    const bool bad = (found_inf && *found_inf != 0) || !isfinite(ss);
    const float norm = sqrtf(ss) * inv_loss_scale;
    float c = inv_loss_scale;
    if (max_norm > 0.f) {
        const float clip = max_norm / (norm + 1e-6f);
        if (clip < 1.f) c *= clip;
    }
    *gscale = bad ? 0.f : c;
    if (skip) *skip = bad ? 1 : 0;
    if (norm_out) *norm_out = bad ? INFINITY : norm;
}

// y = a*x (+ y when accumulate) with dtype conversion: used for unscale, grad-accumulate into
// the fp32 shard and bf16<->fp32 casts of flat buffers.
template <typename TI, typename TO>
__global__ void __launch_bounds__(256) scale_cast_kernel(const TI* __restrict__ x, TO* __restrict__ y,
                                                          int64_t n, float a, int accumulate,
                                                          const float* __restrict__ d_scale)
{
    const float s = a * (d_scale ? *d_scale : 1.f);
    // in-place scaling by exactly 1 (a device-resident factor that is almost always 1, e.g. the LM-head gradient's loss
    // re-scale) is the identity: every thread sees the same scalar, so the whole grid leaves before touching memory
    if (!accumulate && s == 1.f && static_cast<const void*>(x) == static_cast<const void*>(y)) return;
    const int64_t n8 = n >> 3;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    const bool aligned =
        ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;
    int64_t done = 0;
    if (aligned) {
        for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8; i += stride) {
            const int64_t o = i << 3;
            float f[8];
            load8<TI>(x + o, f);
            if (accumulate) {
                float acc[8];
                load8<TO>(y + o, acc);
#pragma unroll
                for (int k = 0; k < 8; ++k) f[k] = fmaf(s, f[k], acc[k]);
            } else {
#pragma unroll
                for (int k = 0; k < 8; ++k) f[k] *= s;
            }
            store8<TO>(y + o, f);
        }
        done = n8 << 3;
    }
    for (int64_t i = done + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        float f = Elem<TI>::to_f(x[i]) * s;
        if (accumulate) f += Elem<TO>::to_f(y[i]);
        y[i] = Elem<TO>::from_f(f);
    }
}

}  // namespace dsb

using namespace dsb;

// ------------------------------------------------------------------------------------------------
// C ABI.  dtype codes: 0 fp32, 1 fp16, 2 bf16.  `out` may be null.
// ------------------------------------------------------------------------------------------------
#define DISPATCH_16(code, T, ...)                     \
    if ((code) == kBF16) {                            \
        using T = __nv_bfloat16;                      \
        __VA_ARGS__                                   \
    } else if ((code) == kF16) {                      \
        using T = __half;                             \
        __VA_ARGS__                                   \
    } else if ((code) == kF32) {                      \
        using T = float;                              \
        __VA_ARGS__                                   \
    } else {                                          \
        return -1;                                    \
    }

// state dtype is either fp32 or the same as the param dtype (keeps instantiation count sane)
#define DISPATCH_STATE(s_code, p_code, PT, ST, ...)   \
    if ((s_code) == kF32) {                           \
        using ST = float;                             \
        __VA_ARGS__                                   \
    } else if ((s_code) == (p_code)) {                \
        using ST = PT;                                \
        __VA_ARGS__                                   \
    } else {                                          \
        return -1;                                    \
    }

DSB_EXPORT int dsb_adam_flat(void* p, const void* g, void* m, void* v, void* out, int64_t n, int p_dtype,
                             int g_dtype, int s_dtype, int o_dtype, float lr, float beta1, float beta2,
                             float eps, float wd, float bc1, float bc2, int adamw, float grad_scale,
                             const float* d_gscale, const int* d_skip, cudaStream_t stream)
{
    if (n <= 0) return 0;
    AdamArgs a{lr, beta1, beta2, eps, wd, bc1, bc2, adamw, grad_scale};
    const int threads = 256;
    const int grid = flat_grid(n >> 3, threads, 8);
    DISPATCH_16(p_dtype, PT, DISPATCH_16(g_dtype, GT, DISPATCH_STATE(s_dtype, p_dtype, PT, ST, {
        if (out == nullptr) {
            adam_flat_kernel<PT, GT, ST, __nv_bfloat16, false><<<grid, threads, 0, stream>>>(
                (PT*)p, (const GT*)g, (ST*)m, (ST*)v, nullptr, n, a, d_gscale, d_skip);
        } else if (o_dtype == kBF16) {
            adam_flat_kernel<PT, GT, ST, __nv_bfloat16, true><<<grid, threads, 0, stream>>>(
                (PT*)p, (const GT*)g, (ST*)m, (ST*)v, (__nv_bfloat16*)out, n, a, d_gscale, d_skip);
        } else if (o_dtype == kF16) {
            adam_flat_kernel<PT, GT, ST, __half, true><<<grid, threads, 0, stream>>>(
                (PT*)p, (const GT*)g, (ST*)m, (ST*)v, (__half*)out, n, a, d_gscale, d_skip);
        } else {
            return -1;
        }
    })))
    DSB_CHECK_LAUNCH();
    return 0;
}

// tensors / chunks are device pointers prepared by the caller (see ops/adam/fused_adam.py).
DSB_EXPORT int dsb_adam_multi(const void* tensors, const void* chunks, int n_chunks, int p_dtype, int g_dtype,
                              int s_dtype, int o_dtype, float lr, float beta1, float beta2, float eps,
                              float wd, float bc1, float bc2, int adamw, float grad_scale,
                              const float* d_gscale, const int* d_skip, cudaStream_t stream)
{
    if (n_chunks <= 0) return 0;
    AdamArgs a{lr, beta1, beta2, eps, wd, bc1, bc2, adamw, grad_scale};
    DISPATCH_16(p_dtype, PT, DISPATCH_16(g_dtype, GT, DISPATCH_STATE(s_dtype, p_dtype, PT, ST, {
        if (o_dtype == kF16) {
            adam_multi_kernel<PT, GT, ST, __half><<<n_chunks, 256, 0, stream>>>(
                (const TensorDesc*)tensors, (const ChunkDesc*)chunks, a, d_gscale, d_skip);
        } else {
            adam_multi_kernel<PT, GT, ST, __nv_bfloat16><<<n_chunks, 256, 0, stream>>>(
                (const TensorDesc*)tensors, (const ChunkDesc*)chunks, a, d_gscale, d_skip);
        }
    })))
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_lion_flat(void* p, const void* g, void* m, void* out, int64_t n, int p_dtype, int g_dtype,
                             int s_dtype, int o_dtype, float lr, float beta1, float beta2, float wd,
                             float grad_scale, const float* d_gscale, const int* d_skip, cudaStream_t stream)
{
    if (n <= 0) return 0;
    LionArgs a{lr, beta1, beta2, wd, grad_scale};
    const int threads = 256;
    const int grid = flat_grid(n, threads, 16);
    DISPATCH_16(p_dtype, PT, DISPATCH_16(g_dtype, GT, DISPATCH_STATE(s_dtype, p_dtype, PT, ST, {
        if (out == nullptr) {
            lion_flat_kernel<PT, GT, ST, __nv_bfloat16, false><<<grid, threads, 0, stream>>>(
                (PT*)p, (const GT*)g, (ST*)m, nullptr, n, a, d_gscale, d_skip);
        } else if (o_dtype == kBF16) {
            lion_flat_kernel<PT, GT, ST, __nv_bfloat16, true><<<grid, threads, 0, stream>>>(
                (PT*)p, (const GT*)g, (ST*)m, (__nv_bfloat16*)out, n, a, d_gscale, d_skip);
        } else {
            lion_flat_kernel<PT, GT, ST, __half, true><<<grid, threads, 0, stream>>>(
                (PT*)p, (const GT*)g, (ST*)m, (__half*)out, n, a, d_gscale, d_skip);
        }
    })))
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_adagrad_flat(void* p, const void* g, float* h, void* out, int64_t n, int p_dtype,
                                int g_dtype, int o_dtype, float lr, float eps, float wd, float grad_scale,
                                cudaStream_t stream)
{
    if (n <= 0) return 0;
    const int threads = 256;
    const int grid = flat_grid(n, threads, 16);
    DISPATCH_16(p_dtype, PT, DISPATCH_16(g_dtype, GT, {
        if (out == nullptr) {
            adagrad_flat_kernel<PT, GT, __nv_bfloat16, false>
                <<<grid, threads, 0, stream>>>((PT*)p, (const GT*)g, h, nullptr, n, lr, eps, wd, grad_scale);
        } else if (o_dtype == kBF16) {
            adagrad_flat_kernel<PT, GT, __nv_bfloat16, true><<<grid, threads, 0, stream>>>(
                (PT*)p, (const GT*)g, h, (__nv_bfloat16*)out, n, lr, eps, wd, grad_scale);
        } else {
            adagrad_flat_kernel<PT, GT, __half, true>
                <<<grid, threads, 0, stream>>>((PT*)p, (const GT*)g, h, (__half*)out, n, lr, eps, wd, grad_scale);
        }
    }))
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_sgd_flat(void* p, const void* g, float* buf, void* out, int64_t n, int p_dtype, int g_dtype,
                            int o_dtype, float lr, float momentum, float dampening, float wd, int nesterov,
                            int first, float grad_scale, cudaStream_t stream)
{
    if (n <= 0) return 0;
    const int threads = 256;
    const int grid = flat_grid(n, threads, 16);
    DISPATCH_16(p_dtype, PT, DISPATCH_16(g_dtype, GT, {
        if (out == nullptr) {
            sgd_flat_kernel<PT, GT, __nv_bfloat16, false><<<grid, threads, 0, stream>>>(
                (PT*)p, (const GT*)g, buf, nullptr, n, lr, momentum, dampening, wd, nesterov, first, grad_scale);
        } else if (o_dtype == kBF16) {
            sgd_flat_kernel<PT, GT, __nv_bfloat16, true><<<grid, threads, 0, stream>>>(
                (PT*)p, (const GT*)g, buf, (__nv_bfloat16*)out, n, lr, momentum, dampening, wd, nesterov, first,
                grad_scale);
        } else {
            sgd_flat_kernel<PT, GT, __half, true><<<grid, threads, 0, stream>>>(
                (PT*)p, (const GT*)g, buf, (__half*)out, n, lr, momentum, dampening, wd, nesterov, first,
                grad_scale);
        }
    }))
    DSB_CHECK_LAUNCH();
    return 0;
}

// LAMB.  `upd` (n floats) and `partials` (2*grid floats) are caller-provided scratch.
DSB_EXPORT int dsb_lamb_grid(int64_t n) { return flat_grid(n, 256, 4); }

DSB_EXPORT int dsb_lamb_flat(void* p, const void* g, float* m, float* v, void* out, float* upd,
                             float* partials, float* coeff_out, int64_t n, int p_dtype, int g_dtype,
                             int o_dtype, float lr, float beta1, float beta2, float eps, float wd, float bc1,
                             float bc2, float max_coeff, float min_coeff, float grad_scale,
                             cudaStream_t stream)
{
    if (n <= 0) return 0;
    AdamArgs a{lr, beta1, beta2, eps, wd, bc1, bc2, 1, grad_scale};
    const int threads = 256;
    const int grid = flat_grid(n, threads, 4);
    DISPATCH_16(p_dtype, PT, DISPATCH_16(g_dtype, GT, {
        lamb_phase1_kernel<PT, GT><<<grid, threads, 0, stream>>>((const PT*)p, (const GT*)g, m, v, upd, n, a,
                                                                   partials);
        if (out == nullptr) {
            lamb_phase2_kernel<PT, __nv_bfloat16, false><<<grid, threads, 0, stream>>>(
                (PT*)p, upd, nullptr, n, lr, partials, grid, max_coeff, min_coeff, coeff_out);
        } else if (o_dtype == kBF16) {
            lamb_phase2_kernel<PT, __nv_bfloat16, true><<<grid, threads, 0, stream>>>(
                (PT*)p, upd, (__nv_bfloat16*)out, n, lr, partials, grid, max_coeff, min_coeff, coeff_out);
        } else {
            lamb_phase2_kernel<PT, __half, true><<<grid, threads, 0, stream>>>(
                (PT*)p, upd, (__half*)out, n, lr, partials, grid, max_coeff, min_coeff, coeff_out);
        }
    }))
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_sumsq_grid(int64_t n) { return flat_grid(n / 8 + 1, 512, 4); }

// out[0] (+)= sum(x^2); found_inf |= any(!finite(x)).  partials: >= dsb_sumsq_grid(n) floats.
DSB_EXPORT int dsb_sumsq(const void* x, int64_t n, int dtype, float* partials, float* out, int* found_inf,
                         int accumulate, cudaStream_t stream)
{
    if (n <= 0) {
        if (!accumulate) cudaMemsetAsync(out, 0, sizeof(float), stream);
        return 0;
    }
    const int grid = flat_grid(n / 8 + 1, 512, 4);
    DISPATCH_16(dtype, T, {
        sumsq_partial_kernel<T><<<grid, 512, 0, stream>>>((const T*)x, n, partials, found_inf);
    })
    reduce_partials_kernel<<<1, 1024, 0, stream>>>(partials, grid, out, accumulate);
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_clip_coeff(const float* sumsq, const int* found_inf, float inv_loss_scale, float max_norm,
                              float* gscale, int* skip, float* norm_out, cudaStream_t stream)
{
    clip_coeff_kernel<<<1, 1, 0, stream>>>(sumsq, found_inf, inv_loss_scale, max_norm, gscale, skip, norm_out);
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_scale_cast(const void* x, void* y, int64_t n, int in_dtype, int out_dtype, float a,
                              int accumulate, const float* d_scale, cudaStream_t stream)
{
    if (n <= 0) return 0;
    const int threads = 256;
    const int grid = flat_grid(n >> 3, threads, 8);
    DISPATCH_16(in_dtype, TI, DISPATCH_16(out_dtype, TO, {
        scale_cast_kernel<TI, TO>
            <<<grid, threads, 0, stream>>>((const TI*)x, (TO*)y, n, a, accumulate, d_scale);
    }))
    DSB_CHECK_LAUNCH();
    return 0;
}
