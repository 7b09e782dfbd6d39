// Transformer elementwise / normalisation kernels for sm_90a (training + inference):
//   RMSNorm / LayerNorm forward+backward (optional fused residual add), rotary embedding
//   forward+backward, gated activations (SwiGLU / GEGLU / ReGLU) forward+backward, bias+activation,
//   fused softmax-cross-entropy forward+backward (in-place gradient), bias/residual adds.
//
// Role parity: reference csrc/transformer/{normalize,gelu,general}_kernels.cu (N7),
// csrc/transformer/inference/csrc/{layer_norm,rms_norm,apply_rotary_pos_emb,gelu,relu,
// pointwise_ops}.cu (N8) and inference/v2 core_ops norms / gated activations (N9a).
// All kernels are HBM-bound: one pass over the data with 16-byte accesses, the row cached in
// registers between the statistics pass and the output pass, fp32 math.
#include <cstdlib>
#include "dsb_common.cuh"

namespace dsb {

constexpr int kMaxVecPerThread = 4;  // 16-byte vectors cached in registers per thread

// ------------------------------------------------------------------------------------------------
// Norm forward.  kLN=false: RMSNorm, kLN=true: LayerNorm.  If `residual` != null the input is
// x + residual and that sum is written to `res_out` (pre-norm residual stream update).
// ------------------------------------------------------------------------------------------------
template <typename T, bool kLN>
__global__ void __launch_bounds__(1024)
norm_fwd_kernel(const T* __restrict__ x, const T* __restrict__ residual, const T* __restrict__ w,
                const T* __restrict__ b, T* __restrict__ y, T* __restrict__ res_out,
                float* __restrict__ mean_out, float* __restrict__ rstd_out, int rows, int hidden, float eps)
{
    __shared__ float scratch[64];
    constexpr int kPer = Elem<T>::kPerVec;
    const int nvec = hidden / kPer;
    for (int row = blockIdx.x; row < rows; row += gridDim.x) {
        const T* xr = x + static_cast<int64_t>(row) * hidden;
        const T* rr = residual ? residual + static_cast<int64_t>(row) * hidden : nullptr;
        Vec16 cache[kMaxVecPerThread];
        float s = 0.f, ss = 0.f;
#pragma unroll
        for (int k = 0; k < kMaxVecPerThread; ++k) {
            const int v = threadIdx.x + k * blockDim.x;
            if (v < nvec) {
                float f[kPer];
                Elem<T>::unpack(ld_stream(xr + v * kPer), f);
                if (rr) {
                    float r[kPer];
                    Elem<T>::unpack(ld_stream(rr + v * kPer), r);
#pragma unroll
                    for (int e = 0; e < kPer; ++e) f[e] += r[e];
                    cache[k] = Elem<T>::pack(f);
                    // re-unpack so the statistics see the rounded residual stream value
                    Elem<T>::unpack(cache[k], f);
                    if (res_out) st_plain(res_out + static_cast<int64_t>(row) * hidden + v * kPer, cache[k]);
                } else {
                    cache[k] = Elem<T>::pack(f);
                }
#pragma unroll
                for (int e = 0; e < kPer; ++e) {
                    s += f[e];
                    ss = fmaf(f[e], f[e], ss);
                }
            }
        }
        float mean = 0.f, rstd;
        if (kLN) {
            float2 r = block_reduce_sum2(s, ss, scratch);
            mean = r.x / hidden;
            const float var = fmaxf(r.y / hidden - mean * mean, 0.f);
            rstd = rsqrtf(var + eps);
        } else {
            const float tot = block_reduce<SumOp>(ss, scratch);
            rstd = rsqrtf(tot / hidden + eps);
        }
        if (threadIdx.x == 0) {
            if (rstd_out) rstd_out[row] = rstd;
            if (kLN && mean_out) mean_out[row] = mean;
        }
        T* yr = y + static_cast<int64_t>(row) * hidden;
#pragma unroll
        for (int k = 0; k < kMaxVecPerThread; ++k) {
            const int v = threadIdx.x + k * blockDim.x;
            if (v < nvec) {
                float f[kPer], wf[kPer];
                Elem<T>::unpack(cache[k], f);
                Elem<T>::unpack(ld_plain(w + v * kPer), wf);
                if (kLN) {
                    float bf[kPer];
                    if (b) Elem<T>::unpack(ld_plain(b + v * kPer), bf);
#pragma unroll
                    for (int e = 0; e < kPer; ++e) f[e] = fmaf((f[e] - mean) * rstd, wf[e], b ? bf[e] : 0.f);
                } else {
#pragma unroll
                    for (int e = 0; e < kPer; ++e) f[e] = f[e] * rstd * wf[e];
                }
                st_plain(yr + v * kPer, Elem<T>::pack(f));
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// Norm backward.  Persistent blocks loop over rows and keep per-column dw/db partial sums in
// registers; partials land in dw_part/db_part [gridDim.x, hidden] and a column-sum kernel
// finishes.  If dres != null it is added to dx (gradient of the residual branch).
// ------------------------------------------------------------------------------------------------
template <typename T, bool kLN>
__global__ void __launch_bounds__(512)
norm_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ x, const T* __restrict__ w,
                const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                const T* __restrict__ dres, T* __restrict__ dx, float* __restrict__ dw_part,
                float* __restrict__ db_part, int rows, int hidden)
{
    __shared__ float scratch[64];
    extern __shared__ __align__(16) uint8_t w_smem_raw[];  // the weight vector, staged once per block
    T* w_s = reinterpret_cast<T*>(w_smem_raw);
    constexpr int kPer = Elem<T>::kPerVec;
    const int nvec = hidden / kPer;
    for (int v = threadIdx.x; v < nvec; v += blockDim.x)
        *reinterpret_cast<Vec16*>(w_s + v * kPer) = ld_plain(w + v * kPer);  // generic store: w_s is shared memory
    __syncthreads();
    float dw_acc[kMaxVecPerThread][kPer];
    float db_acc[kMaxVecPerThread][kPer];
#pragma unroll
    for (int k = 0; k < kMaxVecPerThread; ++k) {
#pragma unroll
        for (int e = 0; e < kPer; ++e) {
            dw_acc[k][e] = 0.f;
            db_acc[k][e] = 0.f;
        }
    }
    for (int row = blockIdx.x; row < rows; row += gridDim.x) {
        const int64_t base = static_cast<int64_t>(row) * hidden;
        const float rstd = rstd_in[row];
        const float mean = kLN ? mean_in[row] : 0.f;
        // issue every global load of the row up front (x, dy and the residual-branch gradient): 12 x 16 B in flight
        // per thread instead of 8 followed by a dependent 4 after the block reduction
        Vec16 cx[kMaxVecPerThread], cdy[kMaxVecPerThread], cres[kMaxVecPerThread];
#pragma unroll
        for (int k = 0; k < kMaxVecPerThread; ++k) {
            const int v = threadIdx.x + k * blockDim.x;
            if (v < nvec) {
                cx[k] = ld_stream(x + base + v * kPer);
                cdy[k] = ld_stream(dy + base + v * kPer);
                if (dres) cres[k] = ld_stream(dres + base + v * kPer);
            }
        }
        float s1 = 0.f, s2 = 0.f;  // sum(g), sum(g * xhat)   with g = dy * w
#pragma unroll
        for (int k = 0; k < kMaxVecPerThread; ++k) {
            const int v = threadIdx.x + k * blockDim.x;
            if (v < nvec) {
                float xf[kPer], df[kPer], wf[kPer];
                Elem<T>::unpack(cx[k], xf);
                Elem<T>::unpack(cdy[k], df);
                Elem<T>::unpack(*reinterpret_cast<const Vec16*>(w_s + v * kPer), wf);
#pragma unroll
                for (int e = 0; e < kPer; ++e) {
                    const float xhat = (xf[e] - mean) * rstd;
                    const float g = df[e] * wf[e];
                    s1 += g;
                    s2 = fmaf(g, xhat, s2);
                    dw_acc[k][e] = fmaf(df[e], xhat, dw_acc[k][e]);
                    if (kLN) db_acc[k][e] += df[e];
                }
            }
        }
        float m1 = 0.f, m2;
        if (kLN) {
            float2 r = block_reduce_sum2(s1, s2, scratch);
            m1 = r.x / hidden;
            m2 = r.y / hidden;
        } else {
            m2 = block_reduce<SumOp>(s2, scratch) / hidden;
        }
#pragma unroll
        for (int k = 0; k < kMaxVecPerThread; ++k) {
            const int v = threadIdx.x + k * blockDim.x;
            if (v < nvec) {
                float xf[kPer], df[kPer], wf[kPer], o[kPer];
                Elem<T>::unpack(cx[k], xf);
                Elem<T>::unpack(cdy[k], df);
                Elem<T>::unpack(*reinterpret_cast<const Vec16*>(w_s + v * kPer), wf);
#pragma unroll
                for (int e = 0; e < kPer; ++e) {
                    const float xhat = (xf[e] - mean) * rstd;
                    const float g = df[e] * wf[e];
                    o[e] = rstd * (g - m1 - xhat * m2);
                }
                if (dres) {
                    float r[kPer];
                    Elem<T>::unpack(cres[k], r);
#pragma unroll
                    for (int e = 0; e < kPer; ++e) o[e] += r[e];
                }
                st_plain(dx + base + v * kPer, Elem<T>::pack(o));
            }
        }
    }
#pragma unroll
    for (int k = 0; k < kMaxVecPerThread; ++k) {
        const int v = threadIdx.x + k * blockDim.x;
        if (v < nvec) {
            float* dst = dw_part + static_cast<int64_t>(blockIdx.x) * hidden + v * kPer;
#pragma unroll
            for (int e = 0; e < kPer; ++e) dst[e] = dw_acc[k][e];
            if (kLN && db_part) {
                float* d2 = db_part + static_cast<int64_t>(blockIdx.x) * hidden + v * kPer;
#pragma unroll
                for (int e = 0; e < kPer; ++e) d2[e] = db_acc[k][e];
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// RMSNorm backward, bulk-async edition (bf16, hidden % 1024 == 0, hidden <= 8192): the register-cached kernel above keeps
// 4 CTAs x 3 rows in flight per SM and stalls every row on load -> reduce -> store; here one producer thread streams whole
// rows (x | dy | dres) through a 4-stage shared-memory ring with cp.async.bulk + mbarrier complete_tx, 4 compute warps
// consume them (conflict-free 16-byte shared loads), so ~190 KB per SM are in flight and loads never wait for math.
// ------------------------------------------------------------------------------------------------
namespace nb {
constexpr int kStages = 4;
constexpr int kComputeThreads = 128;
__device__ __forceinline__ uint32_t s32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mb_init(uint32_t bar, uint32_t n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(n)); }
__device__ __forceinline__ void mb_expect(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mb_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mb_wait(uint32_t bar, uint32_t parity)
{
    asm volatile(
        "{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D_%=;\nbra W_%=;\nD_%=:\n}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
                 "r"(bytes), "r"(bar)
                 : "memory");
}
}  // namespace nb

template <int VPT>  // 16-byte vectors per compute thread per tensor: hidden = 128 * VPT * 8
__global__ void __launch_bounds__(nb::kComputeThreads + 32)
rmsnorm_bwd_bulk_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                        const __nv_bfloat16* __restrict__ w, const float* __restrict__ rstd_in,
                        const __nv_bfloat16* __restrict__ dres, __nv_bfloat16* __restrict__ dx,
                        float* __restrict__ dw_part, int rows, int hidden)
{
    using namespace nb;
    extern __shared__ __align__(128) uint8_t sm_raw[];
    const uint32_t row_bytes = static_cast<uint32_t>(hidden) * 2;
    const int n_in = dres ? 3 : 2;
    // [stage][x | dy | dres] rows, then the weight row, the reduction scratch and the barriers
    uint8_t* ring = sm_raw;
    __nv_bfloat16* w_s = reinterpret_cast<__nv_bfloat16*>(sm_raw + kStages * 3 * row_bytes);
    float* red = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(w_s) + row_bytes);
    const uint32_t bar0 = s32(red + 8);
    auto full = [&](int s) { return bar0 + 8 * s; };
    auto empty = [&](int s) { return bar0 + 8 * (kStages + s); };
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        for (int s = 0; s < kStages; ++s) {
            mb_init(full(s), 1);
            mb_init(empty(s), kComputeThreads / 32);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int v = tid; v < hidden / 8; v += blockDim.x) reinterpret_cast<Vec16*>(w_s)[v] = ld_plain(w + v * 8);
    __syncthreads();
    const int n_my = rows > static_cast<int>(blockIdx.x) ? (rows - 1 - static_cast<int>(blockIdx.x)) / static_cast<int>(gridDim.x) + 1 : 0;

    if (warp == kComputeThreads / 32) {
        // ---------------- producer: one thread issues the bulk copies ----------------
        if (lane == 0) {
            for (int i = 0; i < n_my; ++i) {
                const int st = i % kStages;
                const int64_t row = static_cast<int64_t>(blockIdx.x) + static_cast<int64_t>(i) * gridDim.x;
                mb_wait(empty(st), ((i / kStages) & 1) ^ 1);
                mb_expect(full(st), n_in * row_bytes);
                const uint32_t dst = s32(ring + st * 3 * row_bytes);
                bulk_load(dst, x + row * hidden, row_bytes, full(st));
                bulk_load(dst + row_bytes, dy + row * hidden, row_bytes, full(st));
                if (dres) bulk_load(dst + 2 * row_bytes, dres + row * hidden, row_bytes, full(st));
            }
        }
        return;
    }
    // ---------------- consumers ----------------
    float dw_acc[VPT][8];
#pragma unroll
    for (int k = 0; k < VPT; ++k)
#pragma unroll
        for (int e = 0; e < 8; ++e) dw_acc[k][e] = 0.f;
    for (int i = 0; i < n_my; ++i) {
        const int st = i % kStages;
        const int64_t row = static_cast<int64_t>(blockIdx.x) + static_cast<int64_t>(i) * gridDim.x;
        const float rstd = rstd_in[row];
        mb_wait(full(st), (i / kStages) & 1);
        const uint8_t* base = ring + st * 3 * row_bytes;
        Vec16 cx[VPT], cdy[VPT], cres[VPT];
        float s2 = 0.f;
#pragma unroll
        for (int k = 0; k < VPT; ++k) {
            const int v = tid + k * kComputeThreads;
            cx[k] = *reinterpret_cast<const Vec16*>(base + v * 16);
            cdy[k] = *reinterpret_cast<const Vec16*>(base + row_bytes + v * 16);
            if (dres) cres[k] = *reinterpret_cast<const Vec16*>(base + 2 * row_bytes + v * 16);
            float xf[8], df[8], wf[8];
            Elem<__nv_bfloat16>::unpack(cx[k], xf);
            Elem<__nv_bfloat16>::unpack(cdy[k], df);
            Elem<__nv_bfloat16>::unpack(reinterpret_cast<const Vec16*>(w_s)[v], wf);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float xhat = xf[e] * rstd;
                s2 = fmaf(df[e] * wf[e], xhat, s2);
                dw_acc[k][e] = fmaf(df[e], xhat, dw_acc[k][e]);
            }
        }
        // the row is in registers: give the slot back before the reduction / stores
        __syncwarp();
        if (lane == 0) mb_arrive(empty(st));
        s2 = warp_reduce<SumOp>(s2);
        const int slot = (i & 1) * 4;  // two rotating scratch rows: a fast warp may already be one row ahead
        if (lane == 0) red[slot + warp] = s2;
        asm volatile("bar.sync 1, %0;" ::"n"(kComputeThreads) : "memory");
        const float m2 = (red[slot] + red[slot + 1] + red[slot + 2] + red[slot + 3]) / hidden;
#pragma unroll
        for (int k = 0; k < VPT; ++k) {
            const int v = tid + k * kComputeThreads;
            float xf[8], df[8], wf[8], o[8];
            Elem<__nv_bfloat16>::unpack(cx[k], xf);
            Elem<__nv_bfloat16>::unpack(cdy[k], df);
            Elem<__nv_bfloat16>::unpack(reinterpret_cast<const Vec16*>(w_s)[v], wf);
#pragma unroll
            for (int e = 0; e < 8; ++e) o[e] = rstd * (df[e] * wf[e] - xf[e] * rstd * m2);
            if (dres) {
                float r[8];
                Elem<__nv_bfloat16>::unpack(cres[k], r);
#pragma unroll
                for (int e = 0; e < 8; ++e) o[e] += r[e];
            }
            st_plain(dx + row * hidden + v * 8, Elem<__nv_bfloat16>::pack(o));
        }
    }
#pragma unroll
    for (int k = 0; k < VPT; ++k) {
        float* dst = dw_part + static_cast<int64_t>(blockIdx.x) * hidden + (tid + k * kComputeThreads) * 8;
#pragma unroll
        for (int e = 0; e < 8; ++e) dst[e] = dw_acc[k][e];
    }
}

// out[c] = sum_r part[r, c]  (fixed order -> deterministic); optional accumulate into out.
// A CTA owns 32 columns; its 8 warps stride over the rows (coalesced 128-byte row segments), partial sums meet in shared
// memory in a fixed order.  (One thread per column left only hidden/256 CTAs on the chip: 35 us for a 10 MB reduction.)
template <typename TO>
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ part, TO* __restrict__ out,
                                                      int nrows, int ncols, int accumulate)
{
    __shared__ float red[8][33];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + lane;
    float acc = 0.f;
    if (c < ncols) {
        int r = w;
        for (; r + 24 < nrows; r += 32) {  // 4 independent loads in flight per thread
            const float a0 = part[static_cast<int64_t>(r) * ncols + c];
            const float a1 = part[static_cast<int64_t>(r + 8) * ncols + c];
            const float a2 = part[static_cast<int64_t>(r + 16) * ncols + c];
            const float a3 = part[static_cast<int64_t>(r + 24) * ncols + c];
            acc += (a0 + a1) + (a2 + a3);
        }
        for (; r < nrows; r += 8) acc += part[static_cast<int64_t>(r) * ncols + c];
    }
    red[w][lane] = acc;
    __syncthreads();
    if (w == 0 && c < ncols) {
        float t = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) t += red[k][lane];
        if (accumulate) t += Elem<TO>::to_f(out[c]);
        out[c] = Elem<TO>::from_f(t);
    }
}

// ------------------------------------------------------------------------------------------------
// Rotary embedding (rotate-half convention), in place on a strided [tokens, heads, dim] view.
// cos/sin: fp32 tables [max_pos, rot_dim/2].  positions: int32 [tokens] or null (pos = token %
// seq_len).  sign = +1 forward, -1 backward (the transpose rotation).
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
rope_kernel(T* __restrict__ x, const float* __restrict__ cos_t, const float* __restrict__ sin_t,
            const int* __restrict__ positions, int64_t tokens, int heads, int head_dim, int rot_dim,
            int64_t token_stride, int seq_len, float sign)
{
    constexpr int kPer = Elem<T>::kPerVec;
    const int half = rot_dim / 2;
    const int vec_per_head = half / kPer;  // vectors in one half
    const int64_t total = tokens * heads * vec_per_head;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int v = static_cast<int>(i % vec_per_head);
        const int64_t th = i / vec_per_head;
        const int h = static_cast<int>(th % heads);
        const int64_t t = th / heads;
        const int pos = positions ? positions[t] : static_cast<int>(t % seq_len);
        T* base = x + t * token_stride + static_cast<int64_t>(h) * head_dim;
        float a[kPer], b[kPer], c[kPer], s[kPer];
        Elem<T>::unpack(ld_plain(base + v * kPer), a);
        Elem<T>::unpack(ld_plain(base + half + v * kPer), b);
        const float* cp = cos_t + static_cast<int64_t>(pos) * half + v * kPer;
        const float* sp = sin_t + static_cast<int64_t>(pos) * half + v * kPer;
#pragma unroll
        for (int e = 0; e < kPer; e += 4) {
            const float4 c4 = *reinterpret_cast<const float4*>(cp + e);
            const float4 s4 = *reinterpret_cast<const float4*>(sp + e);
            c[e] = c4.x; c[e + 1] = c4.y; c[e + 2] = c4.z; c[e + 3] = c4.w;
            s[e] = s4.x; s[e + 1] = s4.y; s[e + 2] = s4.z; s[e + 3] = s4.w;
        }
        float o1[kPer], o2[kPer];
#pragma unroll
        for (int e = 0; e < kPer; ++e) {
            const float sn = s[e] * sign;
            o1[e] = fmaf(a[e], c[e], -b[e] * sn);
            o2[e] = fmaf(b[e], c[e], a[e] * sn);
        }
        st_plain(base + v * kPer, Elem<T>::pack(o1));
        st_plain(base + half + v * kPer, Elem<T>::pack(o2));
    }
}

// ------------------------------------------------------------------------------------------------
// QK-norm + rotary embedding (Qwen3 attention), in place on the Q|K heads of a packed
// [tokens, (hq + 2 hkv) * head_dim] buffer with an arbitrary token stride:
//   q_h <- rope(w_q * q_h * rsqrt(mean(q_h^2) + eps)) for every query head, the same with w_k for every key head.
// One 16-byte vector per lane: a head spans L = head_dim / kPer lanes (8, 16 or 32), a warp holds 32 / L heads, and both
// the sum of squares and the rotate-half partner (element i <-> i + head_dim / 2, lane ^ L/2) move through shuffles.
// All arithmetic is fp32 and each output is rounded once.  rot_dim == head_dim.
// ------------------------------------------------------------------------------------------------
template <int L>
__device__ __forceinline__ float head_sum(float v)
{
#pragma unroll
    for (int o = L / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <int kPer>
__device__ __forceinline__ void ld_table(const float* p, float (&f)[kPer])
{
#pragma unroll
    for (int e = 0; e < kPer; e += 4) {
        const float4 q = *reinterpret_cast<const float4*>(p + e);
        f[e] = q.x; f[e + 1] = q.y; f[e + 2] = q.z; f[e + 3] = q.w;
    }
}

// Forward.  Also copies the pre-norm Q|K into `raw` [tokens, (hq + hkv) * head_dim] (contiguous) unless it is null: the
// backward reads it and derives rstd from it again.
template <typename T, int L>
__global__ void __launch_bounds__(256)
qk_norm_rope_kernel(T* __restrict__ qkv, T* __restrict__ raw, const float* __restrict__ cos_t,
                    const float* __restrict__ sin_t, const int* __restrict__ positions, const T* __restrict__ w_q,
                    const T* __restrict__ w_k, int64_t tokens, int hq, int hkv, int64_t token_stride, int seq_len,
                    float eps)
{
    constexpr int kPer = Elem<T>::kPerVec;
    constexpr int kDim = L * kPer, kHeadsPerWarp = 32 / L;
    const int lane = threadIdx.x & 31, v = lane % L;
    const bool upper = v >= L / 2;
    const int hv = (upper ? v - L / 2 : v) * kPer;  // offset into a [rot_dim / 2] table row
    const float rsign = upper ? 1.f : -1.f;
    const int heads = hq + hkv;
    const int64_t items = tokens * heads;
    const int64_t groups = ceil_div(items, kHeadsPerWarp);
    const int64_t nwarps = static_cast<int64_t>(gridDim.x) * (blockDim.x / 32);
    for (int64_t g = static_cast<int64_t>(blockIdx.x) * (blockDim.x / 32) + threadIdx.x / 32; g < groups; g += nwarps) {
        const int64_t item = g * kHeadsPerWarp + lane / L;
        const bool ok = item < items;  // a whole head group is in or out: the shuffles below stay within it
        const int64_t t = ok ? item / heads : 0;
        const int h = ok ? static_cast<int>(item - t * heads) : 0;
        T* px = qkv + t * token_stride + static_cast<int64_t>(h) * kDim + v * kPer;
        Vec16 xv{};
        float x[kPer], w[kPer] = {}, c[kPer] = {}, s[kPer] = {};
        if (ok) {
            xv = ld_plain(px);
            Elem<T>::unpack(ld_plain((h < hq ? w_q : w_k) + v * kPer), w);
            const int pos = positions ? positions[t] : static_cast<int>(t % seq_len);
            ld_table<kPer>(cos_t + static_cast<int64_t>(pos) * (kDim / 2) + hv, c);
            ld_table<kPer>(sin_t + static_cast<int64_t>(pos) * (kDim / 2) + hv, s);
        }
        Elem<T>::unpack(xv, x);
        float ss = 0.f;
#pragma unroll
        for (int e = 0; e < kPer; ++e) ss = fmaf(x[e], x[e], ss);
        const float rstd = rsqrtf(head_sum<L>(ss) / kDim + eps);
        float n[kPer], o[kPer];
#pragma unroll
        for (int e = 0; e < kPer; ++e) n[e] = x[e] * rstd * w[e];
#pragma unroll
        for (int e = 0; e < kPer; ++e) {
            const float p = __shfl_xor_sync(0xffffffffu, n[e], L / 2);
            o[e] = fmaf(n[e], c[e], rsign * p * s[e]);
        }
        if (ok) {
            if (raw) st_plain(raw + item * kDim + v * kPer, xv);
            st_plain(px, Elem<T>::pack(o));
        }
    }
}

// Backward, in place on the dQ|dK heads of the packed gradient: r = rope^-1(dy), g = w * r,
// dx = rstd * (g - xhat * mean(g * xhat)).  dw_q / dw_k partial sums of r * xhat over the CTA's heads of each kind land in
// dw_part [gridDim.x, 2 * head_dim] (q | k) in a fixed order; colsum_kernel finishes them, so dw is bit-reproducible.
template <typename T, int L>
__global__ void __launch_bounds__(256)
qk_norm_rope_bwd_kernel(T* __restrict__ dqkv, const T* __restrict__ raw, const float* __restrict__ cos_t,
                        const float* __restrict__ sin_t, const int* __restrict__ positions, const T* __restrict__ w_q,
                        const T* __restrict__ w_k, float* __restrict__ dw_part, int64_t tokens, int hq, int hkv,
                        int64_t token_stride, int seq_len, float eps)
{
    constexpr int kPer = Elem<T>::kPerVec;
    constexpr int kDim = L * kPer, kHeadsPerWarp = 32 / L, kWarps = 8;
    __shared__ float red[kWarps][2 * kDim];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, v = lane % L;
    const bool upper = v >= L / 2;
    const int hv = (upper ? v - L / 2 : v) * kPer;
    const float rsign = upper ? -1.f : 1.f;  // the transpose rotation
    const int heads = hq + hkv;
    const int64_t items = tokens * heads;
    const int64_t groups = ceil_div(items, kHeadsPerWarp);
    const int64_t nwarps = static_cast<int64_t>(gridDim.x) * kWarps;
    float acc_q[kPer], acc_k[kPer];
#pragma unroll
    for (int e = 0; e < kPer; ++e) acc_q[e] = acc_k[e] = 0.f;
    for (int64_t g = static_cast<int64_t>(blockIdx.x) * kWarps + warp; g < groups; g += nwarps) {
        const int64_t item = g * kHeadsPerWarp + lane / L;
        const bool ok = item < items;
        const int64_t t = ok ? item / heads : 0;
        const int h = ok ? static_cast<int>(item - t * heads) : 0;
        T* pd = dqkv + t * token_stride + static_cast<int64_t>(h) * kDim + v * kPer;
        Vec16 dv{}, xv{};
        float dy[kPer], x[kPer], w[kPer] = {}, c[kPer] = {}, s[kPer] = {};
        if (ok) {
            dv = ld_plain(pd);
            xv = ld_stream(raw + item * kDim + v * kPer);
            Elem<T>::unpack(ld_plain((h < hq ? w_q : w_k) + v * kPer), w);
            const int pos = positions ? positions[t] : static_cast<int>(t % seq_len);
            ld_table<kPer>(cos_t + static_cast<int64_t>(pos) * (kDim / 2) + hv, c);
            ld_table<kPer>(sin_t + static_cast<int64_t>(pos) * (kDim / 2) + hv, s);
        }
        Elem<T>::unpack(dv, dy);
        Elem<T>::unpack(xv, x);
        float r[kPer], ss = 0.f;
#pragma unroll
        for (int e = 0; e < kPer; ++e) {
            const float p = __shfl_xor_sync(0xffffffffu, dy[e], L / 2);
            r[e] = fmaf(dy[e], c[e], rsign * p * s[e]);
            ss = fmaf(x[e], x[e], ss);
        }
        const float rstd = rsqrtf(head_sum<L>(ss) / kDim + eps);
        float s2 = 0.f;
#pragma unroll
        for (int e = 0; e < kPer; ++e) s2 = fmaf(w[e] * r[e], x[e] * rstd, s2);
        const float m2 = head_sum<L>(s2) / kDim;
        float o[kPer];
#pragma unroll
        for (int e = 0; e < kPer; ++e) {
            const float xhat = x[e] * rstd;
            o[e] = rstd * (w[e] * r[e] - xhat * m2);
            if (ok && h < hq) acc_q[e] = fmaf(r[e], xhat, acc_q[e]);
            if (ok && h >= hq) acc_k[e] = fmaf(r[e], xhat, acc_k[e]);
        }
        if (ok) st_plain(pd, Elem<T>::pack(o));
    }
    // the warp's head groups, then the CTA's warps, each in a fixed order
#pragma unroll
    for (int e = 0; e < kPer; ++e) {
#pragma unroll
        for (int o = L; o < 32; o <<= 1) {
            acc_q[e] += __shfl_xor_sync(0xffffffffu, acc_q[e], o);
            acc_k[e] += __shfl_xor_sync(0xffffffffu, acc_k[e], o);
        }
    }
    if (lane < L) {
#pragma unroll
        for (int e = 0; e < kPer; ++e) {
            red[warp][v * kPer + e] = acc_q[e];
            red[warp][kDim + v * kPer + e] = acc_k[e];
        }
    }
    __syncthreads();
    for (int col = threadIdx.x; col < 2 * kDim; col += blockDim.x) {
        float sum = 0.f;
#pragma unroll
        for (int k = 0; k < kWarps; ++k) sum += red[k][col];
        dw_part[static_cast<int64_t>(blockIdx.x) * 2 * kDim + col] = sum;
    }
}

// ------------------------------------------------------------------------------------------------
// Gated activation: out[t, i] = act(gate[t, i]) * up[t, i], gate_up = [T, 2I] (gate | up).
// act: 0 SiLU (SwiGLU), 1 GELU-tanh (GEGLU), 2 ReLU (ReGLU), 3 GELU-erf.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float act_fwd(float g, int act)
{
    switch (act) {
        case 0: return g / (1.f + __expf(-g));
        case 1: {
            const float u = 0.7978845608028654f * (g + 0.044715f * g * g * g);
            return 0.5f * g * (1.f + tanhf(u));
        }
        case 2: return fmaxf(g, 0.f);
        default: return 0.5f * g * (1.f + erff(g * 0.7071067811865476f));
    }
}

__device__ __forceinline__ float act_bwd(float g, int act)
{
    switch (act) {
        case 0: {
            const float s = 1.f / (1.f + __expf(-g));
            return s * (1.f + g * (1.f - s));
        }
        case 1: {
            const float k = 0.7978845608028654f;
            const float u = k * (g + 0.044715f * g * g * g);
            const float t = tanhf(u);
            return 0.5f * (1.f + t) + 0.5f * g * (1.f - t * t) * k * (1.f + 3.f * 0.044715f * g * g);
        }
        case 2: return g > 0.f ? 1.f : 0.f;
        default: {
            const float cdf = 0.5f * (1.f + erff(g * 0.7071067811865476f));
            const float pdf = 0.3989422804014327f * __expf(-0.5f * g * g);
            return cdf + g * pdf;
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(256)
gated_act_fwd_kernel(const T* __restrict__ gate_up, T* __restrict__ out, int64_t tokens, int inter, int act)
{
    constexpr int kPer = Elem<T>::kPerVec;
    const int vpr = inter / kPer;
    const int64_t total = tokens * vpr;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int64_t t = i / vpr;
        const int v = static_cast<int>(i % vpr);
        const T* row = gate_up + t * 2 * inter;
        float g[kPer], u[kPer];
        Elem<T>::unpack(ld_stream(row + v * kPer), g);
        Elem<T>::unpack(ld_stream(row + inter + v * kPer), u);
#pragma unroll
        for (int e = 0; e < kPer; ++e) g[e] = act_fwd(g[e], act) * u[e];
        st_plain(out + t * inter + v * kPer, Elem<T>::pack(g));
    }
}

// kAct: also write act_out = act(gate) * up, computed exactly as gated_act_fwd_kernel does, so a caller that did not
// keep the forward's output gets it back bit for bit from the same read of gate_up.  A template flag rather than a null
// check, so the plain backward compiles to the same code (and register count) as without the extra output.
template <typename T, bool kAct>
__global__ void __launch_bounds__(256)
gated_act_bwd_kernel(const T* __restrict__ dout, const T* __restrict__ gate_up, T* __restrict__ dgate_up,
                     T* __restrict__ act_out, int64_t tokens, int inter, int act)
{
    constexpr int kPer = Elem<T>::kPerVec;
    const int vpr = inter / kPer;
    const int64_t total = tokens * vpr;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int64_t t = i / vpr;
        const int v = static_cast<int>(i % vpr);
        const T* row = gate_up + t * 2 * inter;
        float g[kPer], u[kPer], d[kPer], dg[kPer], du[kPer];
        Elem<T>::unpack(ld_stream(row + v * kPer), g);
        Elem<T>::unpack(ld_stream(row + inter + v * kPer), u);
        Elem<T>::unpack(ld_stream(dout + t * inter + v * kPer), d);
#pragma unroll
        for (int e = 0; e < kPer; ++e) {
            const float a = act_fwd(g[e], act);
            dg[e] = d[e] * u[e] * act_bwd(g[e], act);
            du[e] = d[e] * a;
            if constexpr (kAct) g[e] = a * u[e];
        }
        T* orow = dgate_up + t * 2 * inter;
        st_plain(orow + v * kPer, Elem<T>::pack(dg));
        st_plain(orow + inter + v * kPer, Elem<T>::pack(du));
        if constexpr (kAct) st_plain(act_out + t * inter + v * kPer, Elem<T>::pack(g));
    }
}

// y = act(x + bias) (+ residual).  act: -1 none, else as above.  bias/residual nullable.
template <typename T>
__global__ void __launch_bounds__(256)
bias_act_kernel(const T* __restrict__ x, const T* __restrict__ bias, const T* __restrict__ residual,
                T* __restrict__ y, int64_t rows, int cols, int act)
{
    constexpr int kPer = Elem<T>::kPerVec;
    const int vpr = cols / kPer;
    const int64_t total = rows * vpr;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int v = static_cast<int>(i % vpr);
        float f[kPer];
        Elem<T>::unpack(ld_stream(x + i * kPer), f);
        if (bias) {
            float bf[kPer];
            Elem<T>::unpack(ld_plain(bias + v * kPer), bf);
#pragma unroll
            for (int e = 0; e < kPer; ++e) f[e] += bf[e];
        }
        if (act >= 0) {
#pragma unroll
            for (int e = 0; e < kPer; ++e) f[e] = act_fwd(f[e], act);
        }
        if (residual) {
            float rf[kPer];
            Elem<T>::unpack(ld_stream(residual + i * kPer), rf);
#pragma unroll
            for (int e = 0; e < kPer; ++e) f[e] += rf[e];
        }
        st_plain(y + i * kPer, Elem<T>::pack(f));
    }
}

// dx = dy * act'(x + bias); used by the bias-GELU backward of the BERT-style training layer.
template <typename T>
__global__ void __launch_bounds__(256)
bias_act_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ x, const T* __restrict__ bias,
                    T* __restrict__ dx, int64_t rows, int cols, int act)
{
    constexpr int kPer = Elem<T>::kPerVec;
    const int vpr = cols / kPer;
    const int64_t total = rows * vpr;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int v = static_cast<int>(i % vpr);
        float f[kPer], d[kPer];
        Elem<T>::unpack(ld_stream(x + i * kPer), f);
        Elem<T>::unpack(ld_stream(dy + i * kPer), d);
        if (bias) {
            float bf[kPer];
            Elem<T>::unpack(ld_plain(bias + v * kPer), bf);
#pragma unroll
            for (int e = 0; e < kPer; ++e) f[e] += bf[e];
        }
#pragma unroll
        for (int e = 0; e < kPer; ++e) d[e] *= act_bwd(f[e], act);
        st_plain(dx + i * kPer, Elem<T>::pack(d));
    }
}

// ------------------------------------------------------------------------------------------------
// Fused softmax cross-entropy.  One block per row.  Pass 1: online max / sum-exp.  Pass 2 (second
// read hits L2): loss and, if dlogits != null, gradient (softmax - onehot) * gscale written to
// dlogits (may alias logits for in-place).  Rows whose label is ignore_index or outside [0, vocab) give
// loss 0 / grad 0.
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(1024)
softmax_xent_kernel(const T* logits, const int64_t* __restrict__ labels, float* __restrict__ loss,
                    float* __restrict__ lse_out, T* dlogits, int vocab, int64_t row_stride,
                    int64_t ignore_index, float gscale, const float* __restrict__ d_gscale)
{
    __shared__ float scratch[64];
    constexpr int kPer = Elem<T>::kPerVec;
    const int64_t row = blockIdx.x;
    const T* lr = logits + row * row_stride;
    const int64_t label = labels[row];
    const bool ignored = (label == ignore_index) || label < 0 || label >= vocab;
    // read the label's logit before the block reductions: their barriers order it ahead of the in-place gradient
    // stores, which other warps start as soon as the last reduction returns
    const float x_label = (threadIdx.x == 0 && !ignored) ? Elem<T>::to_f(lr[label]) : 0.f;
    const int nvec = vocab / kPer;
    const bool aligned = (row_stride % kPer) == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0;
    float mx = -INFINITY, sum = 0.f;
    auto upd = [&](float f) {
        if (f == -INFINITY) return;
        if (f > mx) {
            sum = sum * __expf(mx - f) + 1.f;
            mx = f;
        } else {
            sum += __expf(f - mx);
        }
    };
    int done = 0;
    if (aligned) {
        for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
            float f[kPer];
            Elem<T>::unpack(ld_plain(lr + v * kPer), f);
            float lm = f[0];
#pragma unroll
            for (int e = 1; e < kPer; ++e) lm = fmaxf(lm, f[e]);
            if (lm == -INFINITY) continue;
            if (lm > mx) {
                sum *= __expf(mx - lm);
                mx = lm;
            }
#pragma unroll
            for (int e = 0; e < kPer; ++e) sum += __expf(f[e] - mx);
        }
        done = nvec * kPer;
    }
    for (int i = done + threadIdx.x; i < vocab; i += blockDim.x) upd(Elem<T>::to_f(lr[i]));
    // combine (max, sum) pairs across the block
    const float gmx = block_reduce<MaxOp>(mx, scratch);
    const float part = (mx == -INFINITY) ? 0.f : sum * __expf(mx - gmx);
    const float gsum = block_reduce<SumOp>(part, scratch);
    const float lse = gmx + __logf(gsum);
    if (threadIdx.x == 0) {
        loss[row] = ignored ? 0.f : (lse - x_label);
        if (lse_out) lse_out[row] = lse;
    }
    if (dlogits == nullptr) return;
    const float gs = ignored ? 0.f : gscale * (d_gscale ? *d_gscale : 1.f);
    T* dr = dlogits + row * row_stride;
    done = 0;
    if (aligned && (reinterpret_cast<uintptr_t>(dlogits) & 15) == 0) {
        for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
            float f[kPer];
            Elem<T>::unpack(ld_plain(lr + v * kPer), f);
            const int basei = v * kPer;
#pragma unroll
            for (int e = 0; e < kPer; ++e) {
                float p = __expf(f[e] - lse);
                if (basei + e == label) p -= 1.f;
                f[e] = p * gs;
            }
            st_plain(dr + v * kPer, Elem<T>::pack(f));
        }
        done = nvec * kPer;
    }
    for (int i = done + threadIdx.x; i < vocab; i += blockDim.x) {
        float p = __expf(Elem<T>::to_f(lr[i]) - lse);
        if (i == label) p -= 1.f;
        dr[i] = Elem<T>::from_f(p * gs);
    }
}

// n-ary add: y = a + b (+ c) (+ d) with optional scale on the result.
template <typename T>
__global__ void __launch_bounds__(256)
fused_add_kernel(const T* __restrict__ a, const T* __restrict__ b, const T* __restrict__ c,
                 const T* __restrict__ d, T* __restrict__ y, int64_t n, float scale)
{
    constexpr int kPer = Elem<T>::kPerVec;
    const int64_t nv = n / kPer;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nv; i += stride) {
        float f[kPer], g[kPer];
        Elem<T>::unpack(ld_stream(a + i * kPer), f);
        Elem<T>::unpack(ld_stream(b + i * kPer), g);
#pragma unroll
        for (int e = 0; e < kPer; ++e) f[e] += g[e];
        if (c) {
            Elem<T>::unpack(ld_stream(c + i * kPer), g);
#pragma unroll
            for (int e = 0; e < kPer; ++e) f[e] += g[e];
        }
        if (d) {
            Elem<T>::unpack(ld_stream(d + i * kPer), g);
#pragma unroll
            for (int e = 0; e < kPer; ++e) f[e] += g[e];
        }
#pragma unroll
        for (int e = 0; e < kPer; ++e) f[e] *= scale;
        st_plain(y + i * kPer, Elem<T>::pack(f));
    }
    for (int64_t i = nv * kPer + static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        float f = Elem<T>::to_f(a[i]) + Elem<T>::to_f(b[i]);
        if (c) f += Elem<T>::to_f(c[i]);
        if (d) f += Elem<T>::to_f(d[i]);
        y[i] = Elem<T>::from_f(f * scale);
    }
}

}  // namespace dsb

using namespace dsb;

#define DISPATCH_T(code, T, ...)   \
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

static inline int norm_threads(int hidden, int per_vec)
{
    const int nvec = hidden / per_vec;
    int t = (nvec + kMaxVecPerThread - 1) / kMaxVecPerThread;
    t = ((t + 31) / 32) * 32;
    if (t < 32) t = 32;
    return t;  // caller checks <= 1024
}

// kind: 0 RMSNorm, 1 LayerNorm.  Returns -2 when the row does not fit the register cache.
DSB_EXPORT int dsb_norm_fwd(const void* x, const void* residual, const void* w, const void* b, void* y,
                            void* res_out, float* mean, float* rstd, int rows, int hidden, float eps, int kind,
                            int dtype, cudaStream_t stream)
{
    if (rows <= 0) return 0;
    const int per = (dtype == kF32) ? 4 : 8;
    if (hidden % per != 0) return -2;
    const int threads = norm_threads(hidden, per);
    if (threads > 1024) return -2;
    const int grid = rows;
    DISPATCH_T(dtype, T, {
        if (kind == 0)
            norm_fwd_kernel<T, false><<<grid, threads, 0, stream>>>((const T*)x, (const T*)residual, (const T*)w,
                                                                     (const T*)b, (T*)y, (T*)res_out, mean, rstd,
                                                                     rows, hidden, eps);
        else
            norm_fwd_kernel<T, true><<<grid, threads, 0, stream>>>((const T*)x, (const T*)residual, (const T*)w,
                                                                    (const T*)b, (T*)y, (T*)res_out, mean, rstd,
                                                                    rows, hidden, eps);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

static bool dsb_norm_bwd_bulk_disabled()
{
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("DSB200_NORM_BWD_BULK");
        v = (e && e[0] == '0') ? 1 : 0;
    }
    return v == 1;
}

DSB_EXPORT int dsb_norm_bwd_grid(int rows)
{
    // HBM-bound persistent kernel: exactly one wave of resident CTAs (4 per SM at 128 threads x ~120 registers); more
    // CTAs only add a second, half-empty wave and more dw partial rows for the column-sum pass.
    const int cap = kSmCountH100 * 4;
    return rows < cap ? rows : cap;
}

// Which kernel dsb_norm_bwd launches: 1 the bulk-async RMSNorm kernel, 0 the register-cached kernel.  `aligned`: dy, x,
// dres (when given) and dx all start on 16-byte boundaries.
DSB_EXPORT int dsb_norm_bwd_path(int rows, int hidden, int kind, int dtype, int aligned)
{
    return kind == 0 && dtype == kBF16 && hidden % 1024 == 0 && hidden <= 8192 && rows >= 1024 && aligned &&
           !dsb_norm_bwd_bulk_disabled();
}

// dw_part/db_part: fp32 scratch [dsb_norm_bwd_grid(rows), hidden].  dw/db: outputs in `wdtype`.
DSB_EXPORT int dsb_norm_bwd(const void* dy, const void* x, const void* w, const float* mean, const float* rstd,
                            const void* dres, void* dx, float* dw_part, float* db_part, void* dw, void* db,
                            int rows, int hidden, int kind, int dtype, int wdtype, int accumulate_dw,
                            cudaStream_t stream)
{
    if (rows <= 0) return 0;
    const int per = (dtype == kF32) ? 4 : 8;
    if (hidden % per != 0) return -2;
    const int threads = norm_threads(hidden, per);
    if (threads > 512) return -2;
    int grid = dsb_norm_bwd_grid(rows);
    const bool aligned = ((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dres) |
                           reinterpret_cast<uintptr_t>(dx)) & 15) == 0;
    const bool bulk = dsb_norm_bwd_path(rows, hidden, kind, dtype, aligned) == 1;
    if (bulk) {
        // 2 CTAs per SM: 4 stages x 3 rows each
        const int vpt = hidden / 1024;
        const size_t smem = static_cast<size_t>(nb::kStages) * 3 * hidden * 2 + hidden * 2 + 64 + 16 * nb::kStages + 64;
        const int per_sm = smem <= 110 * 1024 ? 2 : 1;
        const int g2 = rows < kSmCountH100 * per_sm ? rows : kSmCountH100 * per_sm;
        grid = g2;
        cudaError_t e = cudaSuccess;
#define DSB_LAUNCH_NB(V)                                                                                                    \
    {                                                                                                                       \
        static size_t attr = 0;                                                                                             \
        if (smem > attr) {                                                                                                  \
            e = cudaFuncSetAttribute(rmsnorm_bwd_bulk_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize,               \
                                     static_cast<int>(smem));                                                              \
            attr = smem;                                                                                                    \
        }                                                                                                                   \
        rmsnorm_bwd_bulk_kernel<V><<<grid, nb::kComputeThreads + 32, smem, stream>>>(                                       \
            (const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, (const __nv_bfloat16*)w, rstd, (const __nv_bfloat16*)dres,    \
            (__nv_bfloat16*)dx, dw_part, rows, hidden);                                                                     \
    }
        switch (vpt) {
            case 1: DSB_LAUNCH_NB(1) break;
            case 2: DSB_LAUNCH_NB(2) break;
            case 3: DSB_LAUNCH_NB(3) break;
            case 4: DSB_LAUNCH_NB(4) break;
            case 5: DSB_LAUNCH_NB(5) break;
            case 6: DSB_LAUNCH_NB(6) break;
            case 7: DSB_LAUNCH_NB(7) break;
            default: DSB_LAUNCH_NB(8) break;
        }
#undef DSB_LAUNCH_NB
        if (e != cudaSuccess) return static_cast<int>(e);
    } else
    DISPATCH_T(dtype, T, {
        if (kind == 0)
            norm_bwd_kernel<T, false><<<grid, threads, hidden * sizeof(T), stream>>>((const T*)dy, (const T*)x, (const T*)w, mean,
                                                                     rstd, (const T*)dres, (T*)dx, dw_part, db_part,
                                                                     rows, hidden);
        else
            norm_bwd_kernel<T, true><<<grid, threads, hidden * sizeof(T), stream>>>((const T*)dy, (const T*)x, (const T*)w, mean,
                                                                    rstd, (const T*)dres, (T*)dx, dw_part, db_part,
                                                                    rows, hidden);
    })
    const int cg = (hidden + 31) / 32;
    DISPATCH_T(wdtype, TO, {
        colsum_kernel<TO><<<cg, 256, 0, stream>>>(dw_part, (TO*)dw, grid, hidden, accumulate_dw);
        if (kind == 1 && db != nullptr)
            colsum_kernel<TO><<<cg, 256, 0, stream>>>(db_part, (TO*)db, grid, hidden, accumulate_dw);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_colsum(const float* part, void* out, int nrows, int ncols, int out_dtype, int accumulate,
                          cudaStream_t stream)
{
    const int cg = (ncols + 31) / 32;
    DISPATCH_T(out_dtype, TO, { colsum_kernel<TO><<<cg, 256, 0, stream>>>(part, (TO*)out, nrows, ncols, accumulate); })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_rope(void* x, const float* cos_t, const float* sin_t, const int* positions, int64_t tokens,
                        int heads, int head_dim, int rot_dim, int64_t token_stride, int seq_len, int backward,
                        int dtype, cudaStream_t stream)
{
    if (tokens <= 0 || heads <= 0) return 0;
    const int per = (dtype == kF32) ? 4 : 8;
    if ((rot_dim / 2) % per != 0 || token_stride % per != 0 || head_dim % per != 0) return -2;
    const int64_t total = tokens * heads * ((rot_dim / 2) / per);
    const int grid = flat_grid(total, 256, 16);
    DISPATCH_T(dtype, T, {
        rope_kernel<T><<<grid, 256, 0, stream>>>((T*)x, cos_t, sin_t, positions, tokens, heads, head_dim, rot_dim,
                                                 token_stride, seq_len, backward ? -1.f : 1.f);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

// The QK-norm kernels take head dim 64 or 128; L = head_dim / (elements per 16-byte vector) lanes per head.
#define DSB_DISPATCH_QK_HEAD_DIM(head_dim, T, L, ...) \
    if ((head_dim) == 64) {                           \
        constexpr int L = 64 / Elem<T>::kPerVec;      \
        __VA_ARGS__                                   \
    } else {                                          \
        constexpr int L = 128 / Elem<T>::kPerVec;     \
        __VA_ARGS__                                   \
    }

// In place on the Q|K heads of `qkv` [tokens, (hq + 2 hkv) * head_dim] (row stride token_stride elements, 16-byte aligned),
// cos/sin [max_pos, head_dim / 2] fp32, positions int32 [tokens] or null (pos = token % seq_len), w_q / w_k [head_dim] in
// the buffer's dtype.  raw: [tokens, (hq + hkv) * head_dim] contiguous, receives the pre-norm Q|K; null when no backward
// follows.
DSB_EXPORT int dsb_qk_norm_rope(void* qkv, void* raw, const float* cos_t, const float* sin_t, const int* positions,
                                const void* w_q, const void* w_k, int64_t tokens, int hq, int hkv, int head_dim,
                                int64_t token_stride, int seq_len, float eps, int dtype, cudaStream_t stream)
{
    const int per = (dtype == kF32) ? 4 : 8;
    if ((head_dim != 64 && head_dim != 128) || token_stride % per != 0) return -2;
    if (tokens <= 0 || hq + hkv <= 0) return 0;
    const int64_t warps = ceil_div(tokens * (hq + hkv), 32 / (head_dim / per));
    const int grid = flat_grid(warps * 32, 256, 8);
    DISPATCH_T(dtype, T, {
        DSB_DISPATCH_QK_HEAD_DIM(head_dim, T, L, {
            qk_norm_rope_kernel<T, L><<<grid, 256, 0, stream>>>((T*)qkv, (T*)raw, cos_t, sin_t, positions, (const T*)w_q,
                                                                (const T*)w_k, tokens, hq, hkv, token_stride, seq_len, eps);
        })
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

// Rows of the dw_part scratch dsb_qk_norm_rope_bwd needs ([rows, 2 * head_dim] fp32): its grid.
DSB_EXPORT int dsb_qk_norm_rope_bwd_grid(int64_t tokens, int heads, int head_dim, int dtype)
{
    const int per = (dtype == kF32) ? 4 : 8;
    return flat_grid(ceil_div(tokens * heads, 32 / (head_dim / per)) * 32, 256, 4);
}

// Backward of dsb_qk_norm_rope, in place on the dQ|dK heads of `dqkv` (same layout as qkv; dV untouched), from the `raw`
// the forward wrote.  dw: [2 * head_dim] in `wdtype` (dw_q | dw_k), overwritten.
DSB_EXPORT int dsb_qk_norm_rope_bwd(void* dqkv, const void* raw, const float* cos_t, const float* sin_t,
                                    const int* positions, const void* w_q, const void* w_k, float* dw_part, void* dw,
                                    int64_t tokens, int hq, int hkv, int head_dim, int64_t token_stride, int seq_len,
                                    float eps, int dtype, int wdtype, cudaStream_t stream)
{
    const int per = (dtype == kF32) ? 4 : 8;
    if ((head_dim != 64 && head_dim != 128) || token_stride % per != 0) return -2;
    // no tokens: the kernel writes zero partials, so dw is zero
    const int grid = dsb_qk_norm_rope_bwd_grid(tokens, hq + hkv, head_dim, dtype);
    DISPATCH_T(dtype, T, {
        DSB_DISPATCH_QK_HEAD_DIM(head_dim, T, L, {
            qk_norm_rope_bwd_kernel<T, L><<<grid, 256, 0, stream>>>((T*)dqkv, (const T*)raw, cos_t, sin_t, positions,
                                                                    (const T*)w_q, (const T*)w_k, dw_part, tokens, hq,
                                                                    hkv, token_stride, seq_len, eps);
        })
    })
    DISPATCH_T(wdtype, TO, {
        colsum_kernel<TO><<<(2 * head_dim + 31) / 32, 256, 0, stream>>>(dw_part, (TO*)dw, grid, 2 * head_dim, 0);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}
#undef DSB_DISPATCH_QK_HEAD_DIM

DSB_EXPORT int dsb_gated_act_fwd(const void* gate_up, void* out, int64_t tokens, int inter, int act, int dtype,
                                 cudaStream_t stream)
{
    if (tokens <= 0) return 0;
    const int per = (dtype == kF32) ? 4 : 8;
    if (inter % per != 0) return -2;
    const int grid = flat_grid(tokens * (inter / per), 256, 16);
    DISPATCH_T(dtype, T, {
        gated_act_fwd_kernel<T><<<grid, 256, 0, stream>>>((const T*)gate_up, (T*)out, tokens, inter, act);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_gated_act_bwd(const void* dout, const void* gate_up, void* dgate_up, void* act_out, int64_t tokens,
                                 int inter, int act, int dtype, cudaStream_t stream)
{
    if (tokens <= 0) return 0;
    const int per = (dtype == kF32) ? 4 : 8;
    if (inter % per != 0) return -2;
    const int grid = flat_grid(tokens * (inter / per), 256, 16);
    DISPATCH_T(dtype, T, {
        if (act_out != nullptr) {
            gated_act_bwd_kernel<T, true><<<grid, 256, 0, stream>>>((const T*)dout, (const T*)gate_up, (T*)dgate_up,
                                                                    (T*)act_out, tokens, inter, act);
        } else {
            gated_act_bwd_kernel<T, false><<<grid, 256, 0, stream>>>((const T*)dout, (const T*)gate_up, (T*)dgate_up,
                                                                     nullptr, tokens, inter, act);
        }
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_bias_act(const void* x, const void* bias, const void* residual, void* y, int64_t rows, int cols,
                            int act, int dtype, cudaStream_t stream)
{
    if (rows <= 0) return 0;
    const int per = (dtype == kF32) ? 4 : 8;
    if (cols % per != 0) return -2;
    const int grid = flat_grid(rows * (cols / per), 256, 16);
    DISPATCH_T(dtype, T, {
        bias_act_kernel<T>
            <<<grid, 256, 0, stream>>>((const T*)x, (const T*)bias, (const T*)residual, (T*)y, rows, cols, act);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_bias_act_bwd(const void* dy, const void* x, const void* bias, void* dx, int64_t rows, int cols,
                                int act, int dtype, cudaStream_t stream)
{
    if (rows <= 0) return 0;
    const int per = (dtype == kF32) ? 4 : 8;
    if (cols % per != 0) return -2;
    const int grid = flat_grid(rows * (cols / per), 256, 16);
    DISPATCH_T(dtype, T, {
        bias_act_bwd_kernel<T>
            <<<grid, 256, 0, stream>>>((const T*)dy, (const T*)x, (const T*)bias, (T*)dx, rows, cols, act);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_softmax_xent(const void* logits, const int64_t* labels, float* loss, float* lse, void* dlogits,
                                int64_t rows, int vocab, int64_t row_stride, int64_t ignore_index, float gscale,
                                const float* d_gscale, int dtype, cudaStream_t stream)
{
    if (rows <= 0) return 0;
    const int threads = vocab >= 8192 ? 1024 : (vocab >= 2048 ? 256 : 128);
    DISPATCH_T(dtype, T, {
        softmax_xent_kernel<T><<<static_cast<unsigned>(rows), threads, 0, stream>>>(
            (const T*)logits, labels, loss, lse, (T*)dlogits, vocab, row_stride, ignore_index, gscale, d_gscale);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_fused_add(const void* a, const void* b, const void* c, const void* d, void* y, int64_t n,
                             float scale, int dtype, cudaStream_t stream)
{
    if (n <= 0) return 0;
    const int per = (dtype == kF32) ? 4 : 8;
    const int grid = flat_grid(n / per + 1, 256, 16);
    DISPATCH_T(dtype, T, {
        fused_add_kernel<T>
            <<<grid, 256, 0, stream>>>((const T*)a, (const T*)b, (const T*)c, (const T*)d, (T*)y, n, scale);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}
