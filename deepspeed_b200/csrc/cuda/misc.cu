// Remaining device ops of the reference kernel inventory, re-implemented for sm_90a:
//   * dropout forward / backward with a counter-based RNG (+bias, +residual fusions)        [N7 dropout_kernels.cu]
//   * masked attention softmax forward / backward over [b, h, sq, sk] (causal / additive mask / alibi /
//     local window)                                                       [N7 softmax_kernels.cu, N8 softmax.cu]
//   * bias-add + [b, s, 3, h, d] -> [3, b, h, s, d] permute and its inverse      [N7/N8 transform kernels]
//   * random-LTD: token index sort, token gather / scatter, attention-mask slicing  [N14 csrc/random_ltd]
//   * NHWC bias-add fusions for diffusion UNet / VAE                                  [N13 csrc/spatial]
#include "dsb_common.cuh"

namespace dsb {
namespace misc {

__device__ __forceinline__ uint32_t mix32(uint32_t x)
{
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}
// Counter-based: the mask of element i depends only on (seed, offset + i) -> backward can regenerate it.
__device__ __forceinline__ float uniform01(uint64_t seed, uint64_t idx)
{
    const uint32_t lo = mix32(static_cast<uint32_t>(idx) ^ static_cast<uint32_t>(seed));
    const uint32_t hi = mix32(static_cast<uint32_t>(idx >> 32) + static_cast<uint32_t>(seed >> 32) + lo);
    return (hi >> 8) * (1.0f / 16777216.0f);
}

// y = dropout(x + bias) + residual ; mask (uint8) optionally stored.
template <typename T>
__global__ void __launch_bounds__(256)
dropout_kernel(const T* __restrict__ x, const T* __restrict__ bias, const T* __restrict__ residual, T* __restrict__ y,
               uint8_t* __restrict__ mask, int64_t n, int cols, float p, uint64_t seed, uint64_t offset)
{
    const float scale = 1.f / (1.f - p);
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        float f = Elem<T>::to_f(x[i]);
        if (bias) f += Elem<T>::to_f(bias[i % cols]);
        const bool keep = uniform01(seed, offset + static_cast<uint64_t>(i)) >= p;
        f = keep ? f * scale : 0.f;
        if (residual) f += Elem<T>::to_f(residual[i]);
        y[i] = Elem<T>::from_f(f);
        if (mask) mask[i] = keep ? 1 : 0;
    }
}

template <typename T>
__global__ void __launch_bounds__(256)
dropout_bwd_kernel(const T* __restrict__ dy, const uint8_t* __restrict__ mask, T* __restrict__ dx, int64_t n, float p,
                   uint64_t seed, uint64_t offset)
{
    const float scale = 1.f / (1.f - p);
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        const bool keep = mask ? mask[i] != 0 : uniform01(seed, offset + static_cast<uint64_t>(i)) >= p;
        dx[i] = Elem<T>::from_f(keep ? Elem<T>::to_f(dy[i]) * scale : 0.f);
    }
}

// ---- attention softmax -------------------------------------------------------------------------------------------
// scores [b, h, sq, sk] in place.  One warp per row.  mask (additive, T) broadcast as [b, 1, 1|sq, sk];
// causal: key j visible iff j <= i + (sk - sq);  window > 0 limits to the last `window` keys;
// alibi slopes [h] add slope * (j - i_abs).
template <typename T>
__global__ void __launch_bounds__(256)
attn_softmax_kernel(T* __restrict__ s, const T* __restrict__ mask, const float* __restrict__ alibi, int b, int h,
                    int sq, int sk, float scale, int causal, int window, int mask_sq)
{
    const int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const int64_t rows = static_cast<int64_t>(b) * h * sq;
    if (row >= rows) return;
    const int i = static_cast<int>(row % sq);
    const int hh = static_cast<int>((row / sq) % h);
    const int bb = static_cast<int>(row / (static_cast<int64_t>(sq) * h));
    T* r = s + row * sk;
    const T* m = mask ? mask + (static_cast<int64_t>(bb) * mask_sq + (mask_sq > 1 ? i : 0)) * sk : nullptr;
    const int i_abs = i + (sk - sq);
    const float slope = alibi ? alibi[hh] : 0.f;
    float mx = -INFINITY;
    for (int j = lane; j < sk; j += 32) {
        float v = Elem<T>::to_f(r[j]) * scale;
        if (m) v += Elem<T>::to_f(m[j]);
        if (alibi) v += slope * static_cast<float>(j - i_abs);
        if ((causal && j > i_abs) || (window > 0 && j <= i_abs - window)) v = -INFINITY;
        mx = fmaxf(mx, v);
    }
    mx = warp_reduce<MaxOp>(mx);
    float sum = 0.f;
    for (int j = lane; j < sk; j += 32) {
        float v = Elem<T>::to_f(r[j]) * scale;
        if (m) v += Elem<T>::to_f(m[j]);
        if (alibi) v += slope * static_cast<float>(j - i_abs);
        if ((causal && j > i_abs) || (window > 0 && j <= i_abs - window)) v = -INFINITY;
        sum += (mx == -INFINITY) ? 0.f : __expf(v - mx);
    }
    sum = warp_reduce<SumOp>(sum);
    const float inv = sum > 0.f ? 1.f / sum : 0.f;
    for (int j = lane; j < sk; j += 32) {
        float v = Elem<T>::to_f(r[j]) * scale;
        if (m) v += Elem<T>::to_f(m[j]);
        if (alibi) v += slope * static_cast<float>(j - i_abs);
        const bool dead = (causal && j > i_abs) || (window > 0 && j <= i_abs - window) || mx == -INFINITY;
        r[j] = Elem<T>::from_f(dead ? 0.f : __expf(v - mx) * inv);
    }
}

// dS = (dP - sum(dP * P)) * P * scale, in place on dP.
template <typename T>
__global__ void __launch_bounds__(256)
attn_softmax_bwd_kernel(T* __restrict__ dp, const T* __restrict__ p, int64_t rows, int sk, float scale)
{
    const int64_t row = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    T* d = dp + row * sk;
    const T* q = p + row * sk;
    float dot = 0.f;
    for (int j = lane; j < sk; j += 32) dot = fmaf(Elem<T>::to_f(d[j]), Elem<T>::to_f(q[j]), dot);
    dot = warp_reduce<SumOp>(dot);
    for (int j = lane; j < sk; j += 32) {
        const float pv = Elem<T>::to_f(q[j]);
        d[j] = Elem<T>::from_f((Elem<T>::to_f(d[j]) - dot) * pv * scale);
    }
}

// ---- QKV bias + permute -------------------------------------------------------------------------------------------
// in [b, s, n3, h, d] (+ bias [n3*h*d])  ->  out [n3, b, h, s, d]
template <typename T>
__global__ void __launch_bounds__(256)
bias_transform_0213_kernel(const T* __restrict__ in, const T* __restrict__ bias, T* __restrict__ out, int b, int s,
                           int n3, int h, int d)
{
    const int64_t total = static_cast<int64_t>(b) * s * n3 * h * d;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
        int64_t r = i;
        const int dd = static_cast<int>(r % d); r /= d;
        const int hh = static_cast<int>(r % h); r /= h;
        const int nn = static_cast<int>(r % n3); r /= n3;
        const int ss = static_cast<int>(r % s); r /= s;
        const int bb = static_cast<int>(r);
        float v = Elem<T>::to_f(in[i]);
        if (bias) v += Elem<T>::to_f(bias[(static_cast<int64_t>(nn) * h + hh) * d + dd]);
        out[(((static_cast<int64_t>(nn) * b + bb) * h + hh) * s + ss) * d + dd] = Elem<T>::from_f(v);
    }
}

// in [b, h, s, d] -> out [b, s, h, d]
template <typename T>
__global__ void __launch_bounds__(256)
transform4d_0213_kernel(const T* __restrict__ in, T* __restrict__ out, int b, int h, int s, int d)
{
    const int64_t total = static_cast<int64_t>(b) * h * s * d;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
        int64_t r = i;
        const int dd = static_cast<int>(r % d); r /= d;
        const int ss = static_cast<int>(r % s); r /= s;
        const int hh = static_cast<int>(r % h); r /= h;
        const int bb = static_cast<int>(r);
        out[((static_cast<int64_t>(bb) * s + ss) * h + hh) * d + dd] = in[i];
    }
}

// ---- random-LTD -----------------------------------------------------------------------------------------------------
// Sort each row of `idx` [rows, k] ascending (k <= 4096): bitonic sort in shared memory.
__global__ void __launch_bounds__(1024) token_sort_kernel(int32_t* __restrict__ idx, int k, int kpow2)
{
    extern __shared__ int32_t sh[];
    int32_t* row = idx + static_cast<int64_t>(blockIdx.x) * k;
    for (int i = threadIdx.x; i < kpow2; i += blockDim.x) sh[i] = i < k ? row[i] : 0x7fffffff;
    __syncthreads();
    for (int size = 2; size <= kpow2; size <<= 1) {
        for (int st = size >> 1; st > 0; st >>= 1) {
            for (int i = threadIdx.x; i < kpow2; i += blockDim.x) {
                const int j = i ^ st;
                if (j > i) {
                    const bool up = (i & size) == 0;
                    const int32_t a = sh[i], c = sh[j];
                    if ((a > c) == up) {
                        sh[i] = c;
                        sh[j] = a;
                    }
                }
            }
            __syncthreads();
        }
    }
    for (int i = threadIdx.x; i < k; i += blockDim.x) row[i] = sh[i];
}

// out[b, j, :] = x[b, idx[b, j], :]   (batch_first) ; scatter is the inverse write.
template <typename T>
__global__ void __launch_bounds__(256)
token_gather_kernel(const T* __restrict__ x, const int32_t* __restrict__ idx, T* __restrict__ out, int batch, int seq,
                    int k, int hidden, int scatter)
{
    const int bj = blockIdx.x;
    if (bj >= batch * k) return;
    const int bb = bj / k;
    const int src_tok = idx[bj];
    const T* a = scatter ? x + static_cast<int64_t>(bj) * hidden : x + (static_cast<int64_t>(bb) * seq + src_tok) * hidden;
    T* o = scatter ? out + (static_cast<int64_t>(bb) * seq + src_tok) * hidden : out + static_cast<int64_t>(bj) * hidden;
    for (int i = threadIdx.x; i < hidden; i += blockDim.x) o[i] = a[i];
}

// mask [b, 1, s, s] -> out [b, 1, k, k] restricted to the kept token indices (BERT-style full mask)
template <typename T>
__global__ void __launch_bounds__(256)
mask_gather_kernel(const T* __restrict__ mask, const int32_t* __restrict__ idx, T* __restrict__ out, int batch, int seq,
                   int k)
{
    const int64_t total = static_cast<int64_t>(batch) * k * k;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int c = static_cast<int>(i % k);
        const int r = static_cast<int>((i / k) % k);
        const int bb = static_cast<int>(i / (static_cast<int64_t>(k) * k));
        out[i] = mask[(static_cast<int64_t>(bb) * seq + idx[bb * k + r]) * seq + idx[bb * k + c]];
    }
}

// ---- NHWC bias add ------------------------------------------------------------------------------------------------------
// y = (x + bias_x) [+ (other [+ bias_o])]   with channel-last layout: channel = i % C
template <typename T>
__global__ void __launch_bounds__(256)
nhwc_bias_add_kernel(const T* __restrict__ x, const T* __restrict__ bias_x, const T* __restrict__ other,
                     const T* __restrict__ bias_o, T* __restrict__ y, int64_t n, int C)
{
    constexpr int kPer = Elem<T>::kPerVec;
    const int64_t nv = n / kPer;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t v = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; v < nv; v += stride) {
        const int c0 = static_cast<int>((v * kPer) % C);
        float f[kPer], g[kPer];
        Elem<T>::unpack(ld_stream(x + v * kPer), f);
        Elem<T>::unpack(ld_plain(bias_x + c0), g);
#pragma unroll
        for (int e = 0; e < kPer; ++e) f[e] += g[e];
        if (other) {
            Elem<T>::unpack(ld_stream(other + v * kPer), g);
#pragma unroll
            for (int e = 0; e < kPer; ++e) f[e] += g[e];
            if (bias_o) {
                Elem<T>::unpack(ld_plain(bias_o + c0), g);
#pragma unroll
                for (int e = 0; e < kPer; ++e) f[e] += g[e];
            }
        }
        st_plain(y + v * kPer, Elem<T>::pack(f));
    }
}

}  // namespace misc
}  // namespace dsb

using namespace dsb;
using namespace dsb::misc;

#define DISPATCH_XT(code, T, ...)  \
    if ((code) == kBF16) {         \
        using T = __nv_bfloat16;   \
        __VA_ARGS__                \
    } else if ((code) == kF16) {   \
        using T = __half;          \
        __VA_ARGS__                \
    } else if ((code) == kF32) {   \
        using T = float;           \
        __VA_ARGS__                \
    } else {                       \
        return -1;                 \
    }

DSB_EXPORT int dsb_dropout(const void* x, const void* bias, const void* residual, void* y, uint8_t* mask, int64_t n,
                           int cols, float p, uint64_t seed, uint64_t offset, int dtype, cudaStream_t stream)
{
    if (n <= 0) return 0;
    const int grid = flat_grid(n, 256, 16);
    DISPATCH_XT(dtype, T, {
        dropout_kernel<T><<<grid, 256, 0, stream>>>((const T*)x, (const T*)bias, (const T*)residual, (T*)y, mask, n, cols, p,
                                                     seed, offset);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_dropout_bwd(const void* dy, const uint8_t* mask, void* dx, int64_t n, float p, uint64_t seed,
                               uint64_t offset, int dtype, cudaStream_t stream)
{
    if (n <= 0) return 0;
    const int grid = flat_grid(n, 256, 16);
    DISPATCH_XT(dtype, T, {
        dropout_bwd_kernel<T><<<grid, 256, 0, stream>>>((const T*)dy, mask, (T*)dx, n, p, seed, offset);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_attn_softmax(void* s, const void* mask, const float* alibi, int b, int h, int sq, int sk, float scale,
                                int causal, int window, int mask_sq, int dtype, cudaStream_t stream)
{
    const int64_t rows = static_cast<int64_t>(b) * h * sq;
    if (rows <= 0) return 0;
    const int grid = static_cast<int>((rows * 32 + 255) / 256);
    DISPATCH_XT(dtype, T, {
        attn_softmax_kernel<T><<<grid, 256, 0, stream>>>((T*)s, (const T*)mask, alibi, b, h, sq, sk, scale, causal, window,
                                                          mask_sq);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_attn_softmax_bwd(void* dp, const void* p, int64_t rows, int sk, float scale, int dtype,
                                    cudaStream_t stream)
{
    if (rows <= 0) return 0;
    const int grid = static_cast<int>((rows * 32 + 255) / 256);
    DISPATCH_XT(dtype, T, { attn_softmax_bwd_kernel<T><<<grid, 256, 0, stream>>>((T*)dp, (const T*)p, rows, sk, scale); })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_bias_transform_0213(const void* in, const void* bias, void* out, int b, int s, int n3, int h, int d,
                                       int dtype, cudaStream_t stream)
{
    const int64_t total = static_cast<int64_t>(b) * s * n3 * h * d;
    if (total <= 0) return 0;
    const int grid = flat_grid(total, 256, 16);
    DISPATCH_XT(dtype, T, {
        bias_transform_0213_kernel<T><<<grid, 256, 0, stream>>>((const T*)in, (const T*)bias, (T*)out, b, s, n3, h, d);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_transform4d_0213(const void* in, void* out, int b, int h, int s, int d, int dtype, cudaStream_t stream)
{
    const int64_t total = static_cast<int64_t>(b) * h * s * d;
    if (total <= 0) return 0;
    const int grid = flat_grid(total, 256, 16);
    DISPATCH_XT(dtype, T, { transform4d_0213_kernel<T><<<grid, 256, 0, stream>>>((const T*)in, (T*)out, b, h, s, d); })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_token_sort(int32_t* idx, int rows, int k, cudaStream_t stream)
{
    if (rows <= 0 || k <= 1) return 0;
    int p2 = 1;
    while (p2 < k) p2 <<= 1;
    if (p2 > 8192) return -2;
    token_sort_kernel<<<rows, p2 < 1024 ? (p2 < 32 ? 32 : p2) : 1024, p2 * sizeof(int32_t), stream>>>(idx, k, p2);
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_token_gather(const void* x, const int32_t* idx, void* out, int batch, int seq, int k, int hidden,
                                int scatter, int dtype, cudaStream_t stream)
{
    if (batch * k <= 0) return 0;
    DISPATCH_XT(dtype, T, {
        token_gather_kernel<T><<<batch * k, 256, 0, stream>>>((const T*)x, idx, (T*)out, batch, seq, k, hidden, scatter);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_mask_gather(const void* mask, const int32_t* idx, void* out, int batch, int seq, int k, int dtype,
                               cudaStream_t stream)
{
    const int64_t total = static_cast<int64_t>(batch) * k * k;
    if (total <= 0) return 0;
    const int grid = flat_grid(total, 256, 16);
    DISPATCH_XT(dtype, T, { mask_gather_kernel<T><<<grid, 256, 0, stream>>>((const T*)mask, idx, (T*)out, batch, seq, k); })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_nhwc_bias_add(const void* x, const void* bias_x, const void* other, const void* bias_o, void* y,
                                 int64_t n, int C, int dtype, cudaStream_t stream)
{
    if (n <= 0) return 0;
    const int per = dtype == kF32 ? 4 : 8;
    if (C % per || n % per) return -2;
    const int grid = flat_grid(n / per, 256, 16);
    DISPATCH_XT(dtype, T, {
        nhwc_bias_add_kernel<T><<<grid, 256, 0, stream>>>((const T*)x, (const T*)bias_x, (const T*)other, (const T*)bias_o,
                                                           (T*)y, n, C);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------
// 1-bit (sign) compression with error feedback for the compressed all-reduce of 1-bit Adam / 0-1 Adam / 1-bit LAMB.
// Reference: runtime/comm/nccl.py:51 compressed_allreduce (cupy packbits + torch ops: ~8 element-wise passes per phase);
// here each phase is ONE pass: 8 values -> 1 byte (MSB first) and the error feedback  e = w - scale * sign(w)  in the same
// kernel; the server side fuses unpack + scale + average over the ranks.
// ---------------------------------------------------------------------------------------------------------------------------
namespace dsb {
__global__ void __launch_bounds__(256)
onebit_pack_kernel(const float* __restrict__ work, const float* __restrict__ scale_ptr, uint8_t* __restrict__ packed,
                   float* __restrict__ err, int64_t n8)
{
    const float s = *scale_ptr;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8; i += stride) {
        float w[8], e[8];
        Elem<float>::unpack(ld_stream(work + i * 8), w);
        Elem<float>::unpack(ld_stream(work + i * 8 + 4), w + 4);
        uint32_t byte = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const bool pos = w[k] >= 0.f;
            byte |= (pos ? 1u : 0u) << (7 - k);
            e[k] = w[k] - (pos ? s : -s);
        }
        packed[i] = static_cast<uint8_t>(byte);
        st_plain(err + i * 8, Elem<float>::pack(e));
        st_plain(err + i * 8 + 4, Elem<float>::pack(e + 4));
    }
}

// out[8 i + k] = inv * sum_r (bit(packed[r][i], k) ? scales[r] : -scales[r])
__global__ void __launch_bounds__(256)
onebit_unpack_avg_kernel(const uint8_t* __restrict__ packed, const float* __restrict__ scales, float* __restrict__ out,
                         int64_t n8, int ranks, float inv)
{
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8; i += stride) {
        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.f;
        for (int r = 0; r < ranks; ++r) {
            const uint32_t byte = packed[static_cast<int64_t>(r) * n8 + i];
            const float s = scales[r];
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[k] += ((byte >> (7 - k)) & 1u) ? s : -s;
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] *= inv;
        st_plain(out + i * 8, Elem<float>::pack(acc));
        st_plain(out + i * 8 + 4, Elem<float>::pack(acc + 4));
    }
}
}  // namespace dsb

DSB_EXPORT int dsb_onebit_pack(const float* work, const float* scale, uint8_t* packed, float* err, int64_t n,
                               cudaStream_t stream)
{
    if (n <= 0) return 0;
    if (n % 8) return -2;
    dsb::onebit_pack_kernel<<<dsb::flat_grid(n / 8, 256, 16), 256, 0, stream>>>(work, scale, packed, err, n / 8);
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_onebit_unpack_avg(const uint8_t* packed, const float* scales, float* out, int64_t n, int ranks, float inv,
                                     cudaStream_t stream)
{
    if (n <= 0) return 0;
    if (n % 8) return -2;
    dsb::onebit_unpack_avg_kernel<<<dsb::flat_grid(n / 8, 256, 16), 256, 0, stream>>>(packed, scales, out, n / 8, ranks, inv);
    DSB_CHECK_LAUNCH();
    return 0;
}
