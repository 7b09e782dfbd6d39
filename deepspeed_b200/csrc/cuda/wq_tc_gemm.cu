// Weight-only-quantised linear on the Hopper tensor cores for 32 < M <= a few hundred rows (batched decode, chunked
// prefill, MoE expert slices):   out[M, N] = x[M, K] @ dequant(Wq)[N, K]^T   with Wq in FP6 (E3M2) / FP8 (E4M3) / INT8 /
// INT4, one fp32 scale per group of `group_size` consecutive K elements.
//
// The packed weights are the only large operand, so they go where wgmma wants the 64-row operand ("swap AB"):
//   D^T[128 features, 128 tokens] = Wdq[128 features, K] * x[128 tokens, K]^T
//   * the two consumer warpgroups (64 feature rows each, two threads per row, 32 K-elements each per step) stream their
//     rows' packed bytes straight from global memory one pipeline step AHEAD into registers (the load latency of step
//     k+1 hides behind the decode of step k), decode to bf16 with the group scale folded in, and write the
//     128-byte-swizzled K-major A tile in shared memory -- the dequantised weight never exists in HBM (the reference's
//     FP6-LLM kernel dequantises in registers for mma.sync, inference/v2/kernels/core_ops/cuda_linear/include/
//     kernel_matmul.cuh:22; cutlass mixed_gemm does the same for int8/int4)
//   * a producer warp TMA-loads the activation tile x[128 tokens, 64] (B operand: up to 128 rows reuse one pass over the
//     weights); each warpgroup issues wgmma.m64n128k16 on its own 64 rows; 4-stage ring, accumulators in registers
//   * epilogue: add the bias and store the transposed tile.
// For M <= 32 the mma.sync kernel of wq_gemm.cu (no padding waste) stays faster; for very large M dequantise-once + the
// bf16 GEMM amortises better -- the Python layer picks (inference/quantization/layers.py).
#include <cuda_fp8.h>
#include "dsb_tc.cuh"

namespace dsb {
namespace wqtc {
using namespace dsb::tc;

constexpr int BF = 128;   // features per CTA (two warpgroups x 64)
constexpr int BK = 64;    // K elements per pipeline step (one 128-byte swizzle row of bf16)
constexpr int BT = 128;   // tokens per CTA (MMA N)
constexpr int kStages = 4;
constexpr int kConsumerThreads = 256;
constexpr int kThreads = kConsumerThreads + 32;
constexpr uint32_t A_BYTES = BF * BK * 2;  // 16 KiB
constexpr uint32_t B_BYTES = BT * BK * 2;  // 16 KiB
constexpr uint32_t SM_A = 0, SM_B = kStages * A_BYTES, SM_BAR = SM_B + kStages * B_BYTES;
constexpr uint32_t SM_TOTAL = SM_BAR + 256 + 1024;

enum Mode : int { kInt8 = 0, kInt4 = 1, kFp8 = 2, kFp6 = 3 };

struct Params {
    const uint8_t* wq;     // packed weights, row-major [N, K] in the group byte-stream layout of quant.cu
    const float* scales;   // [N * K / group_size]
    const __nv_bfloat16* bias;
    __nv_bfloat16* out;    // [M, N]
    int M, N, K, group_size, ldo;
    // grouped (MoE) form: rows of x / out are sorted by expert, expert e owns rows offsets[e] .. offsets[e+1] (device
    // array, no host sync) and uses the e-th [N, K] slab of wq / scales / bias; blockIdx.z = expert
    const int* offsets;
};

// decode 8 consecutive K elements of one feature row into 8 scaled floats
template <int MODE>
__device__ __forceinline__ void decode8(const uint8_t* src, float scale, float* f);

template <>
__device__ __forceinline__ void decode8<kInt8>(const uint8_t* src, float scale, float* f)
{
    const uint2 w = *reinterpret_cast<const uint2*>(src);
    const int8_t* q = reinterpret_cast<const int8_t*>(&w);
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = static_cast<float>(q[e]) * scale;
}
template <>
__device__ __forceinline__ void decode8<kInt4>(const uint8_t* src, float scale, float* f)
{
    const uint32_t w = *reinterpret_cast<const uint32_t*>(src);  // 8 two's-complement nibbles, low nibble first
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = static_cast<float>(static_cast<int>(w << (28 - 4 * e)) >> 28) * scale;
}
template <>
__device__ __forceinline__ void decode8<kFp8>(const uint8_t* src, float scale, float* f)
{
    const uint2 w = *reinterpret_cast<const uint2*>(src);
    const uint16_t* pr = reinterpret_cast<const uint16_t*>(&w);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const __half2_raw h2 = __nv_cvt_fp8x2_to_halfraw2(pr[e], __NV_E4M3);
        const float2 v = __half22float2(*reinterpret_cast<const __half2*>(&h2));
        f[2 * e] = v.x * scale;
        f[2 * e + 1] = v.y * scale;
    }
}
__device__ __forceinline__ float fp6_to_float(uint32_t c)
{
    // E3M2, bias 3, no inf/nan: normal -> exponent field + 124 in fp32, 2 mantissa bits on top; subnormal = m / 16
    const uint32_t sign = (c & 0x20u) << 26;
    const uint32_t ef = (c >> 2) & 7u, mf = c & 3u;
    const uint32_t norm = ((ef + 124u) << 23) | (mf << 21);
    const float v = ef ? __uint_as_float(norm) : static_cast<float>(mf) * 0.0625f;
    return __uint_as_float(__float_as_uint(v) | sign);
}
template <>
__device__ __forceinline__ void decode8<kFp6>(const uint8_t* src, float scale, float* f)
{
    // 8 codes = 48 bits = 6 bytes (two little-endian 24-bit words of 4 codes each); src is only 2-byte aligned
    const uint16_t* p16 = reinterpret_cast<const uint16_t*>(src);
    const uint32_t lo = p16[0] | (static_cast<uint32_t>(p16[1]) << 16);
    const uint32_t hi = p16[2];
    const uint32_t w0 = lo & 0xffffffu;
    const uint32_t w1 = (lo >> 24) | (hi << 8);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        f[e] = fp6_to_float((w0 >> (6 * e)) & 0x3fu) * scale;
        f[4 + e] = fp6_to_float((w1 >> (6 * e)) & 0x3fu) * scale;
    }
}
template <int MODE>
__host__ __device__ constexpr int bytes_per_8()
{
    return MODE == kInt4 ? 4 : (MODE == kFp6 ? 6 : 8);
}

template <int MODE>
__global__ void __launch_bounds__(kThreads, 1)
wq_tc_kernel(const __grid_constant__ CUtensorMap map_x, const Params p)
{
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const uint32_t sbase = smem_u32(smem);
    const uint32_t bar = sbase + SM_BAR;
    auto b_full = [&](int s) { return bar + 8 * s; };
    auto b_empty = [&](int s) { return bar + 8 * (kStages + s); };

    const int f0 = blockIdx.x * BF;  // first feature of this CTA
    int t0 = blockIdx.y * BT;        // first token
    int t_end = p.M;
    const int expert = blockIdx.z;
    if (p.offsets != nullptr) {
        t0 += p.offsets[expert];
        t_end = p.offsets[expert + 1];
    }
    if (t0 >= t_end) return;  // this expert has fewer token tiles (uniform for the CTA: nothing was initialised yet)
    const int num_k = p.K / BK;

    if (threadIdx.x == kConsumerThreads) {
        prefetch_map(&map_x);
        for (int s = 0; s < kStages; ++s) {
            mbar_init(b_full(s), 1);
            mbar_init(b_empty(s), kConsumerThreads / 32);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (threadIdx.x >= kConsumerThreads) {
        if (threadIdx.x == kConsumerThreads) {
            for (int kb = 0; kb < num_k; ++kb) {
                const int st = kb % kStages;
                mbar_wait(b_empty(st), ((kb / kStages) & 1) ^ 1);
                mbar_expect_tx(b_full(st), B_BYTES);
                tma_load_2d(sbase + SM_B + st * B_BYTES, &map_x, b_full(st), kb * BK, t0);
            }
        }
        return;
    }

    // ---- consumers: dequantise this warpgroup's 64 feature rows, multiply, store ------------------------------------------
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = warp >> 2;
    const int tw = threadIdx.x & 127;
    const int r = wg * 64 + (tw & 63);   // feature row inside the CTA tile
    const int hk = tw >> 6;              // which half of the K step this thread decodes
    const int feat = f0 + r;
    const bool feat_ok = feat < p.N;
    constexpr int B8 = bytes_per_8<MODE>();
    constexpr int NR = 4 * B8 / 8;       // 8-byte words of packed weights per thread and step
    const int64_t row_bytes = static_cast<int64_t>(p.K) / 8 * B8;
    const int64_t slab = static_cast<int64_t>(expert) * p.N;  // rows of the stacked [E, N, K] weight before this expert
    const uint8_t* wrow = p.wq + (slab + (feat_ok ? feat : 0)) * row_bytes + hk * 4 * B8;
    const float* srow = p.scales + (slab + (feat_ok ? feat : 0)) * (p.K / p.group_size);
    uint2 cur[NR], nxt[NR];
    float sc_cur, sc_nxt = 0.f;
    auto fetch = [&](int kb, uint2* dst, float& sc) {
        const uint2* g = reinterpret_cast<const uint2*>(wrow + static_cast<int64_t>(kb) * (BK / 8) * B8);
#pragma unroll
        for (int i = 0; i < NR; ++i) dst[i] = feat_ok ? __ldg(g + i) : make_uint2(0u, 0u);
        sc = feat_ok ? __ldg(srow + (kb * BK) / p.group_size) : 0.f;
    };
    float acc[64];
    fetch(0, cur, sc_cur);
    for (int kb = 0; kb < num_k; ++kb) {
        const int st = kb % kStages;
        if (kb + 1 < num_k) fetch(kb + 1, nxt, sc_nxt);  // in flight while this step is decoded
        // the products that last read this A slot (step kb - kStages) retired: at most one group is left in flight
        uint8_t* arow = smem + SM_A + st * A_BYTES + r * 128;
        const uint8_t* raw = reinterpret_cast<const uint8_t*>(cur);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float f[8];
            decode8<MODE>(raw + j * B8, sc_cur, f);
            const int c = hk * 4 + j;
            *reinterpret_cast<Vec16*>(arow + ((c ^ (r & 7)) << 4)) = Elem<__nv_bfloat16>::pack(f);
        }
        fence_async_smem();
        named_sync(1 + wg, 128);
        mbar_wait(b_full(st), (kb / kStages) & 1);
        const uint64_t da = desc_kmajor_sw128(sbase + SM_A + st * A_BYTES + wg * (A_BYTES / 2));
        const uint64_t db = desc_kmajor_sw128(sbase + SM_B + st * B_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) wgmma_m64n128k16_ss<0, 0>(acc, da + 2 * k, db + 2 * k, (kb > 0 || k > 0) ? 1 : 0);
        wgmma_commit();
        wgmma_wait<1>();
        if (kb > 0 && lane == 0) mbar_arrive(b_empty((kb - 1) % kStages));
#pragma unroll
        for (int i = 0; i < NR; ++i) cur[i] = nxt[i];
        sc_cur = sc_nxt;
    }
    wgmma_wait<0>();
    fence_regs<64>(acc);
    // ---- epilogue: transposed store of D^T[feature, token] --------------------------------------------------------------
    const int fr = f0 + wg * 64 + 16 * (warp & 3) + (lane >> 2);  // this thread's features: fr, fr + 8
    const int c_in = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int f = fr + 8 * i;
        if (f >= p.N) continue;
        const float bias = p.bias != nullptr ? __bfloat162float(p.bias[slab + f]) : 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int tok = t0 + 8 * j + c_in + e;
                if (tok < t_end) p.out[static_cast<int64_t>(tok) * p.ldo + f] = __float2bfloat16_rn(acc[4 * j + 2 * i + e] + bias);
            }
    }
}

template <int MODE>
static int launch(const CUtensorMap& mx, const Params& p, int experts, cudaStream_t stream)
{
    static bool attr = false;
    if (!attr) {
        cudaError_t e = cudaFuncSetAttribute(wq_tc_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM_TOTAL);
        if (e != cudaSuccess) return static_cast<int>(e);
        attr = true;
    }
    dim3 grid((p.N + BF - 1) / BF, (p.M + BT - 1) / BT, experts);
    wq_tc_kernel<MODE><<<grid, kThreads, SM_TOTAL, stream>>>(mx, p);
    return 0;
}

}  // namespace wqtc
}  // namespace dsb

using namespace dsb::wqtc;

// mode: 0 int8, 1 int4 (two's-complement nibbles, low first), 2 fp8 e4m3, 3 fp6 e3m2.  x [M, K] bf16 (row stride ldx), out [M, N] bf16.
// K % 64 == 0, group_size % 64 == 0 (a K step never straddles two scale groups), K % group_size == 0.
static int wq_tc_impl(const void* x, const void* wq, const float* scales, const void* bias, void* out, int M, int N, int K,
                      int mode, int group_size, int ldx, int ldo, const int* offsets, int experts, cudaStream_t stream);

DSB_EXPORT int dsb_wq_tc_gemm(const void* x, const void* wq, const float* scales, const void* bias, void* out, int M, int N,
                              int K, int mode, int group_size, int ldx, int ldo, cudaStream_t stream)
{
    return wq_tc_impl(x, wq, scales, bias, out, M, N, K, mode, group_size, ldx, ldo, nullptr, 1, stream);
}

// Grouped (MoE) form: x / out rows sorted by expert, `offsets` int32 [E + 1] ON THE DEVICE, wq / scales / bias stacked [E, ...].
// M = total rows (an upper bound for every expert's row count: the grid covers ceil(M / 128) token tiles per expert and CTAs
// beyond an expert's range exit at once) -- no host synchronisation, CUDA-graph capturable.
DSB_EXPORT int dsb_wq_tc_gemm_grouped(const void* x, const void* wq, const float* scales, const void* bias, void* out,
                                      const int* offsets, int E, int M, int N, int K, int mode, int group_size, int ldx,
                                      int ldo, cudaStream_t stream)
{
    if (E <= 0 || offsets == nullptr) return -3;
    return wq_tc_impl(x, wq, scales, bias, out, M, N, K, mode, group_size, ldx, ldo, offsets, E, stream);
}

static int wq_tc_impl(const void* x, const void* wq, const float* scales, const void* bias, void* out, int M, int N, int K,
                      int mode, int group_size, int ldx, int ldo, const int* offsets, int experts, cudaStream_t stream)
{
    if (M <= 0 || N <= 0) return 0;
    if (K % BK || group_size % BK || K % group_size || ldx % 8 || mode < 0 || mode > 3) return -3;
    if (reinterpret_cast<uintptr_t>(x) & 15) return -3;
    CUtensorMap mx;
    if (make_map(&mx, x, M, K, ldx, BT)) return -3;
    Params p;
    p.wq = static_cast<const uint8_t*>(wq);
    p.scales = scales;
    p.bias = static_cast<const __nv_bfloat16*>(bias);
    p.out = static_cast<__nv_bfloat16*>(out);
    p.M = M;
    p.N = N;
    p.K = K;
    p.group_size = group_size;
    p.ldo = ldo;
    p.offsets = offsets;
    int rc;
    switch (mode) {
        case kInt8: rc = launch<kInt8>(mx, p, experts, stream); break;
        case kInt4: rc = launch<kInt4>(mx, p, experts, stream); break;
        case kFp8: rc = launch<kFp8>(mx, p, experts, stream); break;
        default: rc = launch<kFp6>(mx, p, experts, stream); break;
    }
    if (rc) return rc;
    DSB_CHECK_LAUNCH();
    return 0;
}
