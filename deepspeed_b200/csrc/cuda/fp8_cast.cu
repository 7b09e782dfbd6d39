// Tensorwise FP8 quantisation for training (the casts around the FP8 GEMM of gemm_sm90.cu).
//
// Recipe ("tensorwise current scaling", power-of-two scales): one fp32 scale per tensor, computed on the device from the
// tensor's amax at the time of the cast,
//     scale = 2^e,  e = floor(log2(FMAX / amax)) clamped to [-126, 126],    q = fp8_rne(x * scale),    scale_inv = 2^-e
// (FMAX = 448 for e4m3, 57344 for e5m2).  e is found from amax's exponent and significand, so it is the exact floor: no
// rounding of FMAX / amax can push amax * scale past FMAX, and no finite value saturates.  amax == 0 gives scale 1; a
// non-finite amax (an inf or NaN in the tensor) gives a NaN scale and scale_inv, so everything computed from the tensor
// is NaN instead of silently clipped.  Both scales are finite normal floats otherwise, so scaling and unscaling are exact.
//
//   * dsb_fp8_amax: multi-CTA max |x| into one device fp32 word by atomicMax on the bit pattern of |x| (exact; a NaN's
//     pattern is above inf's, so a NaN propagates);
//   * dsb_fp8_cast: reads that word and writes the row-major fp8 [R, C], the transposed fp8 [C, R] (through shared
//     memory, in the same pass), or both, and scale_inv.  The transposed copies exist because fp8 wgmma takes K-major
//     shared operands only: dgrad needs W^T and wgrad needs dY^T and X^T.
#include <cuda_fp8.h>

#include "dsb_common.cuh"

namespace dsb {
namespace fp8 {

constexpr int kTile = 64;  // cast tile: [64 rows x 64 columns]
constexpr int kThreads = 256;

__device__ __forceinline__ uint32_t abs_bits(__nv_bfloat16 v) { return __float_as_uint(__bfloat162float(v)) & 0x7fffffffu; }

template <bool kVec>
__global__ void __launch_bounds__(kThreads) amax_kernel(const __nv_bfloat16* __restrict__ x, int64_t R, int64_t C, int64_t ld,
                                                        uint32_t* amax_bits)
{
    // one warp per row (grid-stride over rows), 8 columns per lane and step
    const int lane = threadIdx.x & 31;
    const int64_t warps = static_cast<int64_t>(gridDim.x) * (kThreads / 32);
    uint32_t m = 0;
    for (int64_t r = static_cast<int64_t>(blockIdx.x) * (kThreads / 32) + (threadIdx.x >> 5); r < R; r += warps) {
        const __nv_bfloat16* row = x + r * ld;
        for (int64_t c = 8 * lane; c < C; c += 256) {
            if (kVec) {
                const uint4 v = *reinterpret_cast<const uint4*>(row + c);
                const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(&v);
#pragma unroll
                for (int i = 0; i < 8; ++i) m = max(m, abs_bits(h[i]));
            } else {
                const int64_t n = C - c < 8 ? C - c : 8;
                for (int64_t i = 0; i < n; ++i) m = max(m, abs_bits(row[c + i]));
            }
        }
    }
    m = __reduce_max_sync(0xffffffffu, m);
    __shared__ uint32_t part[kThreads / 32];
    if (lane == 0) part[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kThreads / 32; ++w) m = max(m, part[w]);
        atomicMax(amax_bits, m);
    }
}

// scale = 2^e and scale_inv = 2^-e for the tensor's amax (see the file header)
__device__ __forceinline__ void scale_of(float amax, int emax, float& scale, float& scale_inv)
{
    if (!(amax <= 3.402823466e38f)) {  // inf or NaN
        scale = scale_inv = __int_as_float(0x7fffffff);
        return;
    }
    if (amax == 0.f) {
        scale = scale_inv = 1.f;
        return;
    }
    int x;
    const float m = frexpf(amax, &x);  // amax = m 2^x, m in [0.5, 1): amax 2^e <= 1.75 2^emax  <=>  e <= emax - x + 1 - [m > 0.875]
    int e = emax - x + 1 - (m > 0.875f ? 1 : 0);
    e = e < -126 ? -126 : (e > 126 ? 126 : e);
    scale = __int_as_float((127 + e) << 23);
    scale_inv = __int_as_float((127 - e) << 23);
}

template <bool kE5M2>
__device__ __forceinline__ uint16_t cvt2(float a, float b)
{
    return __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, kE5M2 ? __NV_E5M2 : __NV_E4M3);
}

// One CTA per [64 x 64] tile; a thread converts two groups of 8 consecutive columns of one row.
template <bool kE5M2, bool kRow, bool kCol>
__global__ void __launch_bounds__(kThreads) cast_kernel(const __nv_bfloat16* __restrict__ x, int64_t R, int64_t C, int64_t ld,
                                                        const float* amax, uint8_t* __restrict__ q, int64_t ld_q,
                                                        uint8_t* __restrict__ qt, int64_t ld_t, float* scale_inv_out)
{
    __shared__ __align__(8) uint8_t tile[kTile][kTile + 8];
    float scale, scale_inv;
    scale_of(*amax, kE5M2 ? 15 : 8, scale, scale_inv);
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *scale_inv_out = scale_inv;
    const int64_t r0 = static_cast<int64_t>(blockIdx.y) * kTile, c0 = static_cast<int64_t>(blockIdx.x) * kTile;
    const bool vec_in = ((ld & 7) == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
    const bool vec_out = kRow && ((ld_q & 7) == 0) && ((reinterpret_cast<uintptr_t>(q) & 7) == 0);
#pragma unroll
    for (int it = 0; it < 2; ++it) {
        const int g = threadIdx.x + kThreads * it;
        const int lr = g >> 3, lc = (g & 7) * 8;
        const int64_t r = r0 + lr, c = c0 + lc;
        if (r >= R || c >= C) continue;
        const __nv_bfloat16* src = x + r * ld + c;
        float f[8];
        if (vec_in && c + 8 <= C) {
            const uint4 v = *reinterpret_cast<const uint4*>(src);
            const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(&v);
#pragma unroll
            for (int i = 0; i < 8; ++i) f[i] = __bfloat162float(h[i]) * scale;
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) f[i] = c + i < C ? __bfloat162float(src[i]) * scale : 0.f;
        }
        // bytes 0-3 / 4-7 of the group, little-endian
        const uint2 w = make_uint2(cvt2<kE5M2>(f[0], f[1]) | (uint32_t(cvt2<kE5M2>(f[2], f[3])) << 16),
                                   cvt2<kE5M2>(f[4], f[5]) | (uint32_t(cvt2<kE5M2>(f[6], f[7])) << 16));
        if (kRow) {
            uint8_t* dst = q + r * ld_q + c;
            if (vec_out && c + 8 <= C) {
                *reinterpret_cast<uint2*>(dst) = w;
            } else {
                for (int i = 0; i < 8 && c + i < C; ++i) dst[i] = static_cast<uint8_t>((i < 4 ? w.x : w.y) >> (8 * (i & 3)));
            }
        }
        if (kCol) *reinterpret_cast<uint2*>(&tile[lr][lc]) = w;
    }
    if (kCol) {
        __syncthreads();
        // qt [C, R]: thread writes 8 consecutive rows of x (bytes) of one column; R % 16 == 0 and ld_t % 16 == 0, so a
        // group of 8 is either wholly inside R and 8-byte aligned or wholly outside
#pragma unroll
        for (int it = 0; it < 2; ++it) {
            const int g = threadIdx.x + kThreads * it;
            const int lc = g >> 3, lr = (g & 7) * 8;
            const int64_t c = c0 + lc, r = r0 + lr;
            if (c >= C || r >= R) continue;
            uint2 v = make_uint2(0, 0);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                v.x |= uint32_t(tile[lr + i][lc]) << (8 * i);
                v.y |= uint32_t(tile[lr + 4 + i][lc]) << (8 * i);
            }
            *reinterpret_cast<uint2*>(qt + c * ld_t + r) = v;
        }
    }
}

}  // namespace fp8
}  // namespace dsb

using namespace dsb::fp8;

// max |x| of the bf16 matrix x [R, C] (row stride ld, elements) into *amax (device fp32; overwritten, not accumulated).
// Host-checked (-2, nothing launched): R, C >= 1, ld >= C, x 2-byte aligned, amax not null.
DSB_EXPORT int dsb_fp8_amax(const void* x, int64_t R, int64_t C, int64_t ld, float* amax, cudaStream_t stream)
{
    if (R < 1 || C < 1 || ld < C || !x || !amax || (reinterpret_cast<uintptr_t>(x) & 1)) return -2;
    cudaError_t e = cudaMemsetAsync(amax, 0, sizeof(float), stream);
    if (e != cudaSuccess) return static_cast<int>(e);
    int64_t blocks = (R + kThreads / 32 - 1) / (kThreads / 32);
    if (blocks > 4 * dsb::kSmCountH100) blocks = 4 * dsb::kSmCountH100;
    const bool vec = C % 8 == 0 && ld % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
    uint32_t* bits = reinterpret_cast<uint32_t*>(amax);
    if (vec) amax_kernel<true><<<static_cast<int>(blocks), kThreads, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), R, C, ld, bits);
    else amax_kernel<false><<<static_cast<int>(blocks), kThreads, 0, stream>>>(static_cast<const __nv_bfloat16*>(x), R, C, ld, bits);
    DSB_CHECK_LAUNCH();
    return 0;
}

template <bool kE5M2>
static int launch_cast(const void* x, int64_t R, int64_t C, int64_t ld, const float* amax, void* q, int64_t ld_q, void* qt,
                       int64_t ld_t, float* scale_inv, cudaStream_t stream)
{
    const dim3 grid(static_cast<unsigned>((C + kTile - 1) / kTile), static_cast<unsigned>((R + kTile - 1) / kTile));
    auto xs = static_cast<const __nv_bfloat16*>(x);
    auto qs = static_cast<uint8_t*>(q);
    auto ts = static_cast<uint8_t*>(qt);
    if (q && qt) cast_kernel<kE5M2, true, true><<<grid, kThreads, 0, stream>>>(xs, R, C, ld, amax, qs, ld_q, ts, ld_t, scale_inv);
    else if (q) cast_kernel<kE5M2, true, false><<<grid, kThreads, 0, stream>>>(xs, R, C, ld, amax, qs, ld_q, ts, ld_t, scale_inv);
    else cast_kernel<kE5M2, false, true><<<grid, kThreads, 0, stream>>>(xs, R, C, ld, amax, qs, ld_q, ts, ld_t, scale_inv);
    DSB_CHECK_LAUNCH();
    return 0;
}

// Quantise the bf16 matrix x [R, C] (row stride ld) with the scale of *amax (device fp32, from dsb_fp8_amax) to fmt
// (5 = e4m3, 6 = e5m2, the dtype codes of dsb_common.cuh): q [R, C] (row stride ld_q; nullable) and / or its transpose
// qt [C, R] (row stride ld_t; nullable), and *scale_inv (device fp32).  Elements outside [R, C] / [C, R] are not written.
// Host-checked (-2, nothing launched): R, C >= 1 and R <= 65535 * 64; ld >= C; x 2-byte aligned; amax and scale_inv not null;
// fmt 5 or 6; at least one of q, qt; q: ld_q >= C, 16-byte aligned; qt: R % 16 == 0, ld_t >= R, ld_t % 16 == 0, 16-byte
// aligned (qt is a TMA operand: its row stride must be a multiple of 16 bytes).
DSB_EXPORT int dsb_fp8_cast(const void* x, int64_t R, int64_t C, int64_t ld, const float* amax, int fmt, void* q,
                            int64_t ld_q, void* qt, int64_t ld_t, float* scale_inv, cudaStream_t stream)
{
    if (R < 1 || C < 1 || R > int64_t(65535) * kTile || ld < C || !x || (reinterpret_cast<uintptr_t>(x) & 1)) return -2;
    if (!amax || !scale_inv || (fmt != dsb::kF8E4M3 && fmt != dsb::kF8E5M2) || (!q && !qt)) return -2;
    if (q && (ld_q < C || (reinterpret_cast<uintptr_t>(q) & 15))) return -2;
    if (qt && (R % 16 || ld_t < R || ld_t % 16 || (reinterpret_cast<uintptr_t>(qt) & 15))) return -2;
    return fmt == dsb::kF8E5M2 ? launch_cast<true>(x, R, C, ld, amax, q, ld_q, qt, ld_t, scale_inv, stream)
                               : launch_cast<false>(x, R, C, ld, amax, q, ld_q, qt, ld_t, scale_inv, stream);
}
