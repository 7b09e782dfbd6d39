// FP8 quantisation for training (the casts around the FP8 GEMMs of gemm_sm90.cu): tensorwise, then blockwise.
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
//   * dsb_fp8_cast_block: the same rule with one scale per 1 x 128 strip or 128 x 128 block, amax and cast in one pass
//     (documented at the entry point).
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

// ---- blockwise scaling: one pass over the source, the amaxes found inside the tile -----------------------------------------
// Scaling of an output copy: none (copy not written), one scale per 1 x 128 strip along the copy's columns (an A operand
// of the blockwise GEMM), or one scale for the [128 x 128] tile (a B operand).
constexpr int kNone = 0, kStrip = 1, kBlock = 2;
constexpr int kBlk = 128;  // scaling block and cast tile: [128 rows x 128 columns]

// One CTA per [128 x 128] tile of x, read once into registers: a thread holds 8 groups of 8 consecutive columns, group
// `it` in row 16 it + tid / 16 at columns 8 (tid % 16).  Row-strip amaxes come from shuffles over the 16 lanes of a row,
// column-strip and tile amaxes from shared-memory atomics; elements outside [R, C] count as zeros.
template <bool kE5M2, int kRow, int kCol>
__global__ void __launch_bounds__(kThreads) cast_block_kernel(const __nv_bfloat16* __restrict__ x, int64_t R, int64_t C, int64_t ld,
                                                              uint8_t* __restrict__ q, int64_t ld_q, float* __restrict__ sq,
                                                              int64_t ld_sq, uint8_t* __restrict__ qt, int64_t ld_t,
                                                              float* __restrict__ st, int64_t ld_st)
{
    __shared__ __align__(8) uint8_t tile[kCol ? kBlk : 1][kBlk + 8];
    __shared__ uint32_t col_bits[kBlk];
    __shared__ uint32_t tile_bits;
    constexpr int emax = kE5M2 ? 15 : 8;
    constexpr bool kTileAmax = kRow == kBlock || kCol == kBlock;
    const int tid = threadIdx.x;
    const int lr0 = tid >> 4, lc = (tid & 15) * 8;
    const int64_t r0 = static_cast<int64_t>(blockIdx.y) * kBlk, c0 = static_cast<int64_t>(blockIdx.x) * kBlk;
    const int64_t c = c0 + lc;
    const bool vec_in = ((ld & 7) == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
    if (kCol == kStrip && tid < kBlk) col_bits[tid] = 0;
    if (kTileAmax && tid == 0) tile_bits = 0;
    if (kCol == kStrip || kTileAmax) __syncthreads();

    uint32_t h[8][4];  // the tile as packed bf16 pairs; fp32 bits of element i: low half shifted up, or the high half
    auto f32_bits = [](uint32_t pair, int i) { return (i & 1) ? (pair & 0xffff0000u) : (pair << 16); };
    uint32_t row_max[8], col_max[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) col_max[i] = 0;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int64_t r = r0 + lr0 + 16 * it;
        const __nv_bfloat16* src = x + r * ld + c;
        if (r < R && vec_in && c + 8 <= C) {
            const uint4 v = *reinterpret_cast<const uint4*>(src);
            h[it][0] = v.x, h[it][1] = v.y, h[it][2] = v.z, h[it][3] = v.w;
        } else {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const uint32_t lo = r < R && c + 2 * i < C ? __bfloat16_as_ushort(src[2 * i]) : 0;
                const uint32_t hi = r < R && c + 2 * i + 1 < C ? __bfloat16_as_ushort(src[2 * i + 1]) : 0;
                h[it][i] = lo | (hi << 16);
            }
        }
        uint32_t m = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const uint32_t b = f32_bits(h[it][i >> 1], i) & 0x7fffffffu;
            m = max(m, b);
            col_max[i] = max(col_max[i], b);
        }
#pragma unroll
        for (int o = 1; o < 16; o <<= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
        row_max[it] = m;
    }
    if (kCol == kStrip) {
#pragma unroll
        for (int i = 0; i < 8; ++i) atomicMax(&col_bits[lc + i], col_max[i]);
    }
    if (kTileAmax) {
        uint32_t m = 0;
#pragma unroll
        for (int it = 0; it < 8; ++it) m = max(m, row_max[it]);
        m = __reduce_max_sync(0xffffffffu, m);
        if ((tid & 31) == 0) atomicMax(&tile_bits, m);
    }
    if (kCol == kStrip || kTileAmax) __syncthreads();

    float tile_scale = 1.f, tile_inv = 1.f;
    if (kTileAmax) {
        scale_of(__uint_as_float(tile_bits), emax, tile_scale, tile_inv);
        if (tid == 0) {
            if (kRow == kBlock) sq[blockIdx.y * ld_sq + blockIdx.x] = tile_inv;
            if (kCol == kBlock) st[blockIdx.x * ld_st + blockIdx.y] = tile_inv;
        }
    }
    float col_scale[8];
    if (kCol == kStrip) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float inv;
            scale_of(__uint_as_float(col_bits[lc + i]), emax, col_scale[i], inv);
        }
        if (tid < kBlk && c0 + tid < C) {
            float s, inv;
            scale_of(__uint_as_float(col_bits[tid]), emax, s, inv);
            st[blockIdx.y * ld_st + c0 + tid] = inv;
        }
    }
    const bool vec_out = kRow && ((ld_q & 7) == 0) && ((reinterpret_cast<uintptr_t>(q) & 7) == 0);
#pragma unroll
    for (int it = 0; it < 8; ++it) {
        const int lr = lr0 + 16 * it;
        const int64_t r = r0 + lr;
        float f[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) f[i] = __uint_as_float(f32_bits(h[it][i >> 1], i));
        if (kRow) {
            float s = tile_scale;
            if (kRow == kStrip) {
                float inv;
                scale_of(__uint_as_float(row_max[it]), emax, s, inv);
                if ((tid & 15) == 0 && r < R) sq[blockIdx.x * ld_sq + r] = inv;
            }
            if (r < R && c < C) {
                const uint2 w = make_uint2(cvt2<kE5M2>(f[0] * s, f[1] * s) | (uint32_t(cvt2<kE5M2>(f[2] * s, f[3] * s)) << 16),
                                           cvt2<kE5M2>(f[4] * s, f[5] * s) | (uint32_t(cvt2<kE5M2>(f[6] * s, f[7] * s)) << 16));
                uint8_t* dst = q + r * ld_q + c;
                if (vec_out && c + 8 <= C) {
                    *reinterpret_cast<uint2*>(dst) = w;
                } else {
#pragma unroll
                    for (int i = 0; i < 8; ++i)
                        if (c + i < C) dst[i] = static_cast<uint8_t>((i < 4 ? w.x : w.y) >> (8 * (i & 3)));
                }
            }
        }
        if (kCol) {
            if (kCol == kBlock) {
#pragma unroll
                for (int i = 0; i < 8; ++i) f[i] *= tile_scale;
            } else {
#pragma unroll
                for (int i = 0; i < 8; ++i) f[i] *= col_scale[i];
            }
            *reinterpret_cast<uint2*>(&tile[lr][lc]) =
                make_uint2(cvt2<kE5M2>(f[0], f[1]) | (uint32_t(cvt2<kE5M2>(f[2], f[3])) << 16),
                           cvt2<kE5M2>(f[4], f[5]) | (uint32_t(cvt2<kE5M2>(f[6], f[7])) << 16));
        }
    }
    if (kCol) {
        __syncthreads();
        // qt [C, R]: a thread writes 8 consecutive rows of x (bytes) of one column; R % 16 == 0 and ld_t % 16 == 0, so a
        // group of 8 is either wholly inside R and 8-byte aligned or wholly outside
#pragma unroll
        for (int it = 0; it < 8; ++it) {
            const int tc = lr0 + 16 * it, tr = lc;
            if (c0 + tc >= C || r0 + tr >= R) continue;
            uint2 v = make_uint2(0, 0);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                v.x |= uint32_t(tile[tr + i][tc]) << (8 * i);
                v.y |= uint32_t(tile[tr + 4 + i][tc]) << (8 * i);
            }
            *reinterpret_cast<uint2*>(qt + (c0 + tc) * ld_t + r0 + tr) = v;
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

template <bool kE5M2, int kRow>
static int launch_cast_block_col(int col_mode, dim3 grid, const __nv_bfloat16* x, int64_t R, int64_t C, int64_t ld, uint8_t* q,
                                 int64_t ld_q, float* sq, int64_t ld_sq, uint8_t* qt, int64_t ld_t, float* st, int64_t ld_st,
                                 cudaStream_t stream)
{
    if (col_mode == kNone) cast_block_kernel<kE5M2, kRow, kNone><<<grid, kThreads, 0, stream>>>(x, R, C, ld, q, ld_q, sq, ld_sq, qt, ld_t, st, ld_st);
    else if (col_mode == kStrip) cast_block_kernel<kE5M2, kRow, kStrip><<<grid, kThreads, 0, stream>>>(x, R, C, ld, q, ld_q, sq, ld_sq, qt, ld_t, st, ld_st);
    else cast_block_kernel<kE5M2, kRow, kBlock><<<grid, kThreads, 0, stream>>>(x, R, C, ld, q, ld_q, sq, ld_sq, qt, ld_t, st, ld_st);
    DSB_CHECK_LAUNCH();
    return 0;
}

template <bool kE5M2>
static int launch_cast_block(int row_mode, int col_mode, dim3 grid, const __nv_bfloat16* x, int64_t R, int64_t C, int64_t ld,
                             uint8_t* q, int64_t ld_q, float* sq, int64_t ld_sq, uint8_t* qt, int64_t ld_t, float* st,
                             int64_t ld_st, cudaStream_t stream)
{
    if (row_mode == kNone) return launch_cast_block_col<kE5M2, kNone>(col_mode, grid, x, R, C, ld, q, ld_q, sq, ld_sq, qt, ld_t, st, ld_st, stream);
    if (row_mode == kStrip) return launch_cast_block_col<kE5M2, kStrip>(col_mode, grid, x, R, C, ld, q, ld_q, sq, ld_sq, qt, ld_t, st, ld_st, stream);
    return launch_cast_block_col<kE5M2, kBlock>(col_mode, grid, x, R, C, ld, q, ld_q, sq, ld_sq, qt, ld_t, st, ld_st, stream);
}

// Blockwise-scaled cast in one pass: quantise the bf16 matrix x [R, C] (row stride ld) to fmt (5 = e4m3, 6 = e5m2) with a
// power-of-two scale per block (the rule of the file header applied to the block's amax; a trailing partial block takes
// its amax over the elements that exist).  No amax launch comes first: a CTA finds the amaxes of its [128 x 128] tile.
//   q  [R, C] (row stride ld_q), row_mode 1: one scale per 1 x 128 strip of a row,   sq [ceil(C/128), R]  (row stride ld_sq)
//                                row_mode 2: one scale per 128 x 128 block,           sq [ceil(R/128), ceil(C/128)]
//   qt [C, R] (row stride ld_t), col_mode 1: one scale per 1 x 128 strip of a row of qt (128 rows of one column of x),
//                                                                                     st [ceil(R/128), C]  (row stride ld_st)
//                                col_mode 2: one scale per 128 x 128 block,           st [ceil(C/128), ceil(R/128)]
// sq / st hold scale_inv (fp32).  Strip scales are stored k-block-major -- row kb holds the scales of every row of the copy
// for its columns [128 kb, 128 kb + 128) -- the layout dsb_gemm_fp8_block reads for its A operand: the rows a warp
// holds are contiguous.  Block scales are the [n-block, k-block] grid of its B operand; a block of x and the same block
// of qt share their scale, so a matrix cast with row_mode 2 and col_mode 2 gets st = sq^T.  Mode 0 leaves that copy (and
// its scales) unwritten; elements outside [R, C] / [C, R] and scales outside the shapes above are not written.
// Host-checked (-2, nothing launched): R, C >= 1 and R <= 65535 * 128; ld >= C; x 2-byte aligned; fmt 5 or 6; row_mode and
// col_mode in 0..2, not both 0; row_mode != 0: q and sq not null, ld_q >= C, q 16-byte aligned, ld_sq >= R (mode 1) or
// ceil(C/128) (mode 2); col_mode != 0: qt and st not null, R % 16 == 0, ld_t >= R, ld_t % 16 == 0, qt 16-byte aligned (qt
// is a TMA operand), ld_st >= C (mode 1) or ceil(R/128) (mode 2).
DSB_EXPORT int dsb_fp8_cast_block(const void* x, int64_t R, int64_t C, int64_t ld, int fmt, int row_mode, void* q, int64_t ld_q,
                                  float* sq, int64_t ld_sq, int col_mode, void* qt, int64_t ld_t, float* st, int64_t ld_st,
                                  cudaStream_t stream)
{
    if (R < 1 || C < 1 || R > int64_t(65535) * kBlk || ld < C || !x || (reinterpret_cast<uintptr_t>(x) & 1)) return -2;
    if ((fmt != dsb::kF8E4M3 && fmt != dsb::kF8E5M2) || row_mode < 0 || row_mode > 2 || col_mode < 0 || col_mode > 2) return -2;
    if (row_mode == kNone && col_mode == kNone) return -2;
    const int64_t rb = (R + kBlk - 1) / kBlk, cb = (C + kBlk - 1) / kBlk;
    if (row_mode && (!q || !sq || ld_q < C || (reinterpret_cast<uintptr_t>(q) & 15) || ld_sq < (row_mode == kStrip ? R : cb)))
        return -2;
    if (col_mode && (!qt || !st || R % 16 || ld_t < R || ld_t % 16 || (reinterpret_cast<uintptr_t>(qt) & 15) ||
                     ld_st < (col_mode == kStrip ? C : rb)))
        return -2;
    const dim3 grid(static_cast<unsigned>(cb), static_cast<unsigned>(rb));
    auto xs = static_cast<const __nv_bfloat16*>(x);
    auto qs = static_cast<uint8_t*>(q);
    auto ts = static_cast<uint8_t*>(qt);
    return fmt == dsb::kF8E5M2
               ? launch_cast_block<true>(row_mode, col_mode, grid, xs, R, C, ld, qs, ld_q, sq, ld_sq, ts, ld_t, st, ld_st, stream)
               : launch_cast_block<false>(row_mode, col_mode, grid, xs, R, C, ld, qs, ld_q, sq, ld_sq, ts, ld_t, st, ld_st, stream);
}
