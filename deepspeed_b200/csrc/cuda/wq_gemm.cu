// Weight-only-quantised linear for decode-sized inputs:  out[M, N] = x[M, K] @ dequant(Wq)[N, K]^T,  M <= 64.
//
// Role parity: reference inference/v2/kernels/core_ops/cuda_linear (FP6-LLM `QUANT_GEMM_Kernel`, N9a) and the cutlass
// `mixed_gemm` (N9c): weights stay packed in HBM (int8 or int4 + one fp32 scale per group of `group_size` consecutive K
// elements, the layout produced by quant.cu / ops/quantizer) and are dequantised in registers on their way to the tensor
// cores, so a decode step streams 1 (int8) or 0.5 (int4) bytes per weight instead of 2.
//
// The op is pure weight bandwidth, so the layout is chosen for the loads, not the math: a CTA owns NT*8 output features, its 8
// warps split K in chunks (64 int8 / 128 int4 weights per feature), and inside a chunk lane (g, t) of a warp fetches ONE
// 16-byte packet of feature g: the 4 t-lanes of a feature cover the chunk contiguously.  The MMA's logical k order is
// arbitrary as long as A and B agree, so packet element 4j+{0..3} of lane t becomes k = {2t, 2t+1, 2t+8, 2t+9} of the j-th
// m16n8k16 MMA; the matching activation fragment is then 8 contiguous bytes of x per row.  The B fragments carry the exact
// integers (int8: byte-permute into the mantissa of 2^23 and subtract; int4: two nibbles at a time OR-ed into the mantissa of
// a 16-bit 128.0 / 1024.0 pair and one packed subtract, with the activation pairs permuted to match), each chunk accumulates
// into its own fp32 tile and the group scale is applied to that tile in fp32 -- scaling before the rounding to bf16 would
// cost an instruction per weight and lose bits.  Partial sums of the 8 warps are reduced through shared memory.
// (mma.sync on purpose: at M <= 64 a wgmma tile would be >75% padding and the kernel is bound by the weight stream.)
#include <cuda_fp8.h>
#include <type_traits>
#include "dsb_common.cuh"

namespace dsb {
namespace wq {

constexpr int kWarps = 8;

template <typename T>
struct Frag;
template <>
struct Frag<__nv_bfloat16> {
    static __device__ __forceinline__ uint32_t pack(float lo, float hi)
    {
        __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
        return *reinterpret_cast<uint32_t*>(&v);
    }
    // u holds (q+8) in bits 0..3 and 16..19 -> packed pair of exact q
    static __device__ __forceinline__ uint32_t i4pair(uint32_t u)
    {
        uint32_t v = u | 0x43004300u;  // bf16 128 + (q+8)
        const uint32_t off = 0x43084308u;  // bf16 136
        __nv_bfloat162 r = __hsub2(*reinterpret_cast<__nv_bfloat162*>(&v), *reinterpret_cast<const __nv_bfloat162*>(&off));
        return *reinterpret_cast<uint32_t*>(&r);
    }
    static __device__ __forceinline__ void mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1)
    {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
};
template <>
struct Frag<__half> {
    static __device__ __forceinline__ uint32_t pack(float lo, float hi)
    {
        __half2 v = __floats2half2_rn(lo, hi);
        return *reinterpret_cast<uint32_t*>(&v);
    }
    static __device__ __forceinline__ uint32_t i4pair(uint32_t u)
    {
        uint32_t v = u | 0x64006400u;  // fp16 1024 + (q+8)
        const uint32_t off = 0x64086408u;  // fp16 1032
        __half2 r = __hsub2(*reinterpret_cast<__half2*>(&v), *reinterpret_cast<const __half2*>(&off));
        return *reinterpret_cast<uint32_t*>(&r);
    }
    static __device__ __forceinline__ void mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1)
    {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
};

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))), "l"(gmem)
                 : "memory");
}
// activations: every CTA re-reads the same few KB, so let them allocate in L1 instead of all hammering the same L2 lines
__device__ __forceinline__ void cp_async16_l1(void* smem, const void* gmem)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))), "l"(gmem)
                 : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(smem))), "l"(gmem)
                 : "memory");
}

// int8 element e (0..15) of a 16-byte packet as an exact fp32 integer: the stored two's-complement byte xor 0x80 is q+128;
// dropped into the mantissa of 2^23 it reads 8388608+128+q.
__device__ __forceinline__ float dq8(const Vec16& pk, int e)
{
    return __uint_as_float(__byte_perm(pk.w[e >> 2] ^ 0x80808080u, 0x4B000000u, 0x7650 | (e & 3))) - (8388608.f + 128.f);
}

// two e4m3 codes (the low / high half of a packet word) -> one packed fragment register; e4m3 values are exact in bf16
template <typename T>
__device__ __forceinline__ uint32_t fp8x2_frag(uint32_t word, int hi)
{
    const __nv_fp8x2_storage_t two = static_cast<__nv_fp8x2_storage_t>(hi ? (word >> 16) : (word & 0xffffu));
    const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2(two, __NV_E4M3);
    if constexpr (sizeof(T) == 2 && std::is_same<T, __half>::value) {
        return *reinterpret_cast<const uint32_t*>(&h);
    } else {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h));
        return Frag<T>::pack(f.x, f.y);
    }
}

template <typename T, int BITS, int NT, int MT, bool FP8 = false>
__global__ void __launch_bounds__(kWarps * 32)
wq_mma_kernel(const T* __restrict__ x, const int8_t* __restrict__ wq, const float* __restrict__ scales,
              const T* __restrict__ bias, T* __restrict__ out, int M, int N, int K, int group_size, int S)
{
    constexpr int CK = BITS == 8 ? 64 : 128;  // weights per feature per chunk (4 lanes x 16 bytes)
    constexpr int EPL = CK / 4;               // weights per lane packet
    constexpr int XQ = EPL / 8;               // 16-byte pieces of activations per lane and row (the same k range as the packet)
    // Per-warp private prefetch ring in shared memory, filled with cp.async: the weight stream needs tens of KB in flight per SM
    // and the activation fragments (L2 latency, consumed immediately by the MMAs) must be prefetched just as far ahead.
    // One stage = the warp's chunk: NT weight packets per lane | xh*XQ activation pieces per lane | NT*8 group scales.
    const int xh = (M + 7) >> 3;  // 8-row halves of the activation tile that hold real rows
    const int w_bytes = NT * 512, x_bytes = xh * XQ * 512, stage_bytes = w_bytes + x_bytes + 128;
    extern __shared__ __align__(16) unsigned char ring[];
    float (*red)[MT * 16][NT * 8 + 1] = reinterpret_cast<float (*)[MT * 16][NT * 8 + 1]>(ring);  // reused after the K loop

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int n0 = blockIdx.x * NT * 8;
    const int64_t row_bytes = static_cast<int64_t>(K) * BITS / 8;
    const int gpr = K / group_size, cpg = group_size / CK;  // groups per weight row, chunks per group
    const int8_t* wrow[NT];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        int n = n0 + nt * 8 + g;
        n = n < N ? n : N - 1;  // clamped rows are computed and dropped at the store
        wrow[nt] = wq + n * row_bytes;
    }
    int ns = n0 + lane;  // lanes < NT*8 fetch the scale of feature n0+lane
    ns = ns < N ? ns : N - 1;
    const float* srow = scales + static_cast<int64_t>(ns) * gpr;
    float acc[MT][NT][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;

    const int chunks = K / CK;
    const int n_my = chunks > warp ? (chunks - warp + kWarps - 1) / kWarps : 0;
    unsigned char* my_ring = ring + warp * (S * stage_bytes);
    auto issue = [&](int i, int slot_idx) {
        const int c = warp + i * kWarps, kb = c * CK + t * EPL;
        unsigned char* slot = my_ring + slot_idx * stage_bytes;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) cp_async16(slot + (nt * 32 + lane) * 16, wrow[nt] + static_cast<int64_t>(kb) * BITS / 8);
        for (int hh = 0; hh < xh; ++hh) {
            int r = hh * 8 + g;
            r = r < M ? r : M - 1;  // rows past M repeat the last one; their outputs are never stored
            const T* xr = x + static_cast<int64_t>(r) * K + kb;
#pragma unroll
            for (int q = 0; q < XQ; ++q) cp_async16_l1(slot + w_bytes + ((hh * XQ + q) * 32 + lane) * 16, xr + q * 8);
        }
        if (lane < NT * 8) cp_async4(slot + w_bytes + x_bytes + lane * 4, srow + c / cpg);  // group_size % CK == 0
    };
    for (int i = 0; i < S - 1; ++i) {
        if (i < n_my) issue(i, i);
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    int rd = 0, wr = S - 1;  // ring positions of the stage consumed / filled this iteration
    for (int i = 0; i < n_my; ++i) {
        __syncwarp();  // all lanes finished reading the stage that is refilled now (scales are read across lanes)
        if (i + S - 1 < n_my) issue(i + S - 1, wr);
        asm volatile("cp.async.commit_group;" ::: "memory");
        switch (S) {
            case 2: asm volatile("cp.async.wait_group 1;" ::: "memory"); break;
            case 3: asm volatile("cp.async.wait_group 2;" ::: "memory"); break;
            case 4: asm volatile("cp.async.wait_group 3;" ::: "memory"); break;
            case 5: asm volatile("cp.async.wait_group 4;" ::: "memory"); break;
            default: asm volatile("cp.async.wait_group 5;" ::: "memory"); break;
        }
        __syncwarp();
        const unsigned char* slot = my_ring + rd * stage_bytes;
        const unsigned char* xs = slot + w_bytes + lane * 16;
        rd = rd + 1 == S ? 0 : rd + 1;
        wr = wr + 1 == S ? 0 : wr + 1;
        Vec16 cur[NT];
        float2 cs[NT];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            cur[nt] = *reinterpret_cast<const Vec16*>(slot + (nt * 32 + lane) * 16);
            cs[nt] = *reinterpret_cast<const float2*>(slot + w_bytes + x_bytes + (nt * 8 + 2 * t) * 4);
        }
        float tmp[MT][NT][4];
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int nt = 0; nt < NT; ++nt)
#pragma unroll
                for (int i2 = 0; i2 < 4; ++i2) tmp[mt][nt][i2] = 0.f;
        // activation piece q of 8-row half hh (zero when the half holds no real row)
        auto xpiece = [&](int hh, int q) {
            uint4 v = make_uint4(0u, 0u, 0u, 0u);
            if (hh < xh) v = *reinterpret_cast<const uint4*>(xs + (hh * XQ + q) * 512);
            return v;
        };
        if constexpr (BITS == 8) {
#pragma unroll
            for (int jp = 0; jp < 2; ++jp) {  // 16 bytes of x per row feed two MMAs
                uint32_t a[2][MT][4];
#pragma unroll
                for (int mt = 0; mt < MT; ++mt) {
                    const uint4 v0 = xpiece(2 * mt, jp), v1 = xpiece(2 * mt + 1, jp);
                    a[0][mt][0] = v0.x, a[0][mt][1] = v1.x, a[0][mt][2] = v0.y, a[0][mt][3] = v1.y;
                    a[1][mt][0] = v0.z, a[1][mt][1] = v1.z, a[1][mt][2] = v0.w, a[1][mt][3] = v1.w;
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int j = 2 * jp + h;
#pragma unroll
                    for (int nt = 0; nt < NT; ++nt) {
                        uint32_t b0, b1;
                        if constexpr (FP8) {
                            b0 = fp8x2_frag<T>(cur[nt].w[j], 0);
                            b1 = fp8x2_frag<T>(cur[nt].w[j], 1);
                        } else {
                            b0 = Frag<T>::pack(dq8(cur[nt], 4 * j), dq8(cur[nt], 4 * j + 1));
                            b1 = Frag<T>::pack(dq8(cur[nt], 4 * j + 2), dq8(cur[nt], 4 * j + 3));
                        }
#pragma unroll
                        for (int mt = 0; mt < MT; ++mt) Frag<T>::mma(tmp[mt][nt], a[h][mt], b0, b1);
                    }
                }
            }
        } else {
            // word w of the packet = weights 8w..8w+7; nibble pairs (i, i+4) share a 32-bit lane after shift+mask, so the
            // two MMAs of a word see k order (0,4 | 1,5) and (2,6 | 3,7); the activation pairs are permuted to match.
#pragma unroll
            for (int w = 0; w < 4; ++w) {
                uint32_t aA[MT][4], aB[MT][4];
#pragma unroll
                for (int mt = 0; mt < MT; ++mt) {
                    const uint4 v0 = xpiece(2 * mt, w), v1 = xpiece(2 * mt + 1, w);
                    aA[mt][0] = __byte_perm(v0.x, v0.z, 0x5410), aA[mt][2] = __byte_perm(v0.x, v0.z, 0x7632);
                    aA[mt][1] = __byte_perm(v1.x, v1.z, 0x5410), aA[mt][3] = __byte_perm(v1.x, v1.z, 0x7632);
                    aB[mt][0] = __byte_perm(v0.y, v0.w, 0x5410), aB[mt][2] = __byte_perm(v0.y, v0.w, 0x7632);
                    aB[mt][1] = __byte_perm(v1.y, v1.w, 0x5410), aB[mt][3] = __byte_perm(v1.y, v1.w, 0x7632);
                }
#pragma unroll
                for (int nt = 0; nt < NT; ++nt) {
                    const uint32_t u = cur[nt].w[w] ^ 0x88888888u;
                    const uint32_t p0 = Frag<T>::i4pair(u & 0x000f000fu), p1 = Frag<T>::i4pair((u >> 4) & 0x000f000fu);
                    const uint32_t p2 = Frag<T>::i4pair((u >> 8) & 0x000f000fu), p3 = Frag<T>::i4pair((u >> 12) & 0x000f000fu);
#pragma unroll
                    for (int mt = 0; mt < MT; ++mt) {
                        Frag<T>::mma(tmp[mt][nt], aA[mt], p0, p1);
                        Frag<T>::mma(tmp[mt][nt], aB[mt], p2, p3);
                    }
                }
            }
        }
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int nt = 0; nt < NT; ++nt) {
                acc[mt][nt][0] = fmaf(tmp[mt][nt][0], cs[nt].x, acc[mt][nt][0]);
                acc[mt][nt][1] = fmaf(tmp[mt][nt][1], cs[nt].y, acc[mt][nt][1]);
                acc[mt][nt][2] = fmaf(tmp[mt][nt][2], cs[nt].x, acc[mt][nt][2]);
                acc[mt][nt][3] = fmaf(tmp[mt][nt][3], cs[nt].y, acc[mt][nt][3]);
            }
    }
    __syncthreads();  // every warp is done with its ring before the reduction buffer overlays it
    // C fragment: c0,c1 = (row g, cols 2t, 2t+1); c2,c3 = (row g+8, same cols)
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            red[warp][mt * 16 + g][nt * 8 + 2 * t] = acc[mt][nt][0];
            red[warp][mt * 16 + g][nt * 8 + 2 * t + 1] = acc[mt][nt][1];
            red[warp][mt * 16 + g + 8][nt * 8 + 2 * t] = acc[mt][nt][2];
            red[warp][mt * 16 + g + 8][nt * 8 + 2 * t + 1] = acc[mt][nt][3];
        }
    __syncthreads();
    for (int i = threadIdx.x; i < MT * 16 * NT * 8; i += kWarps * 32) {
        const int m = i / (NT * 8), col = i % (NT * 8), n = n0 + col;
        if (m < M && n < N) {
            float v = 0.f;
#pragma unroll
            for (int w = 0; w < kWarps; ++w) v += red[w][m][col];
            if (bias) v += Elem<T>::to_f(bias[n]);
            out[static_cast<int64_t>(m) * N + n] = Elem<T>::from_f(v);
        }
    }
}

template <typename T, int BITS, bool FP8 = false>
void launch(const void* x, const void* wq, const float* scales, const void* bias, void* out, int M, int N, int K, int gs,
            cudaStream_t stream)
{
    constexpr int kSmemBudget = 80 * 1024;  // two CTAs per SM and ~90 KB of L1 left for the activations
#define WQ_GO(NT, MT)                                                                                                   \
    do {                                                                                                                \
        auto kern = wq_mma_kernel<T, BITS, NT, MT, FP8>;                                                                  \
        const int stage = NT * 512 + ((M + 7) / 8) * (BITS == 8 ? 2 : 4) * 512 + 128;                                   \
        int S = kSmemBudget / (kWarps * stage);                                                                         \
        S = S < 2 ? 2 : (S > 4 ? 4 : S);                                                                                \
        const int red_b = kWarps * MT * 16 * (NT * 8 + 1) * 4;                                                          \
        const int ring_b = kWarps * S * stage;                                                                          \
        const int smem = ring_b > red_b ? ring_b : red_b;                                                               \
        static bool attr = false;                                                                                       \
        if (!attr) {                                                                                                    \
            cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);                        \
            attr = true;                                                                                                \
        }                                                                                                               \
        kern<<<(N + NT * 8 - 1) / (NT * 8), kWarps * 32, smem, stream>>>((const T*)x, (const int8_t*)wq, scales,        \
                                                                         (const T*)bias, (T*)out, M, N, K, gs, S);      \
    } while (0)
    // wide CTAs (32 features) once there are enough of them to fill the machine twice over; otherwise 16 features per CTA
    const bool wide = N / 32 >= 2 * kSmCountH100;
    if (M <= 16) {
        if (wide) WQ_GO(4, 1); else WQ_GO(2, 1);
    } else {
        if (wide) WQ_GO(4, 2); else WQ_GO(2, 2);
    }
#undef WQ_GO
}

}  // namespace wq
}  // namespace dsb

using namespace dsb;

// x [M, K] (bf16/fp16, contiguous), wq packed [N, K*bits/8], scales fp32 [N*K/group_size], out [M, N].
// Returns -3 when the shape is not eligible (caller falls back to dequantise + GEMM).
DSB_EXPORT int dsb_wq_gemv(const void* x, const void* wq, const float* scales, const void* bias, void* out, int M, int N, int K,
                           int bits, int group_size, int dtype, cudaStream_t stream)
{
    if (M <= 0 || N <= 0) return 0;
    if (M > 32 || (bits != 8 && bits != 4)) return -3;  // beyond 32 rows dequantise + tensor-core GEMM is faster
    const int ck = bits == 8 ? 64 : 128;
    if (K % ck || group_size % ck || K % group_size) return -3;
    if (dtype != kBF16 && dtype != kF16) return -3;
    if (dtype == kBF16) {
        if (bits == 8) wq::launch<__nv_bfloat16, 8>(x, wq, scales, bias, out, M, N, K, group_size, stream);
        else wq::launch<__nv_bfloat16, 4>(x, wq, scales, bias, out, M, N, K, group_size, stream);
    } else {
        if (bits == 8) wq::launch<__half, 8>(x, wq, scales, bias, out, M, N, K, group_size, stream);
        else wq::launch<__half, 4>(x, wq, scales, bias, out, M, N, K, group_size, stream);
    }
    DSB_CHECK_LAUNCH();
    return 0;
}

// FP8 (e4m3 codes + one fp32 scale per group) weights: same kernel, the codes are converted with the hardware
// fp8x2 -> f16x2 instruction on their way into the fragments.
DSB_EXPORT int dsb_wq_gemv_fp8(const void* x, const void* wq, const float* scales, const void* bias, void* out, int M, int N, int K,
                               int group_size, int dtype, cudaStream_t stream)
{
    if (M <= 0 || N <= 0) return 0;
    if (M > 32 || K % 64 || group_size % 64 || K % group_size) return -3;
    if (dtype == kBF16)
        wq::launch<__nv_bfloat16, 8, true>(x, wq, scales, bias, out, M, N, K, group_size, stream);
    else if (dtype == kF16)
        wq::launch<__half, 8, true>(x, wq, scales, bias, out, M, N, K, group_size, stream);
    else
        return -3;
    DSB_CHECK_LAUNCH();
    return 0;
}
