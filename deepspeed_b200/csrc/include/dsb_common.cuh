// Shared device helpers for the deepspeed_b200 sm_90a kernels.
//
// Role parity: reference csrc/includes/{memory_access_utils.h, reduction_utils.h,
// conversion_utils.h} (N20 in SURVEY.md).  Written from scratch for sm_90a: 16-byte vector
// accesses with explicit cache policies, warp-shuffle + smem block reductions, and packed
// bf16/fp16 <-> fp32 conversion helpers.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define DSB_EXPORT extern "C" __attribute__((visibility("default")))

#define DSB_CHECK_LAUNCH()                                 \
    do {                                                   \
        cudaError_t _e = cudaPeekAtLastError();            \
        if (_e != cudaSuccess) return static_cast<int>(_e); \
    } while (0)

namespace dsb {

constexpr int kWarp = 32;
constexpr int kSmCountH100 = 132;

// dtype codes shared with Python (deepspeed_b200/ops/native.py)
enum DType : int { kF32 = 0, kF16 = 1, kBF16 = 2, kI8 = 3, kU8 = 4, kF8E4M3 = 5, kF8E5M2 = 6 };

// ---------------------------------------------------------------------------------------------
// 16-byte vector type
// ---------------------------------------------------------------------------------------------
struct __align__(16) Vec16 {
    uint32_t w[4];
};

__device__ __forceinline__ Vec16 ld_stream(const void* p)
{
    // Streaming read: data is touched once -> do not pollute L1.  (Not .nc: several kernels
    // read-modify-write the same flat buffer in place.)
    Vec16 v;
    asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
                 : "l"(p));
    return v;
}

__device__ __forceinline__ Vec16 ld_plain(const void* p)
{
    Vec16 v;
    asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
                 : "l"(p));
    return v;
}

__device__ __forceinline__ void st_stream(void* p, const Vec16& v)
{
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.w[0]),
                 "r"(v.w[1]), "r"(v.w[2]), "r"(v.w[3])
                 : "memory");
}

__device__ __forceinline__ void st_plain(void* p, const Vec16& v)
{
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.w[0]), "r"(v.w[1]),
                 "r"(v.w[2]), "r"(v.w[3])
                 : "memory");
}

// Peer / system-coherent accesses (NVLink-mapped addresses): relaxed.sys so they are not
// served from a stale L1 line.
__device__ __forceinline__ Vec16 ld_peer(const void* p)
{
    Vec16 v;
    asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
                 : "l"(p)
                 : "memory");
    return v;
}

__device__ __forceinline__ void st_peer(void* p, const Vec16& v)
{
    asm volatile("st.relaxed.sys.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.w[0]),
                 "r"(v.w[1]), "r"(v.w[2]), "r"(v.w[3])
                 : "memory");
}

// ---------------------------------------------------------------------------------------------
// conversions
// ---------------------------------------------------------------------------------------------
template <typename T>
struct Elem;

template <>
struct Elem<float> {
    static constexpr int kPerVec = 4;
    __device__ static __forceinline__ void unpack(const Vec16& v, float* out)
    {
#pragma unroll
        for (int i = 0; i < 4; ++i) out[i] = __uint_as_float(v.w[i]);
    }
    __device__ static __forceinline__ Vec16 pack(const float* in)
    {
        Vec16 v;
#pragma unroll
        for (int i = 0; i < 4; ++i) v.w[i] = __float_as_uint(in[i]);
        return v;
    }
    __device__ static __forceinline__ float to_f(float x) { return x; }
    __device__ static __forceinline__ float from_f(float x) { return x; }
};

template <>
struct Elem<__nv_bfloat16> {
    static constexpr int kPerVec = 8;
    __device__ static __forceinline__ void unpack(const Vec16& v, float* out)
    {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            // bf16 -> fp32 is a 16-bit shift: exact and cheaper than cvt.
            out[2 * i] = __uint_as_float(v.w[i] << 16);
            out[2 * i + 1] = __uint_as_float(v.w[i] & 0xffff0000u);
        }
    }
    __device__ static __forceinline__ Vec16 pack(const float* in)
    {
        Vec16 v;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            __nv_bfloat162 h = __floats2bfloat162_rn(in[2 * i], in[2 * i + 1]);
            v.w[i] = *reinterpret_cast<uint32_t*>(&h);
        }
        return v;
    }
    __device__ static __forceinline__ float to_f(__nv_bfloat16 x) { return __bfloat162float(x); }
    __device__ static __forceinline__ __nv_bfloat16 from_f(float x) { return __float2bfloat16_rn(x); }
};

template <>
struct Elem<__half> {
    static constexpr int kPerVec = 8;
    __device__ static __forceinline__ void unpack(const Vec16& v, float* out)
    {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            __half2 h = *reinterpret_cast<const __half2*>(&v.w[i]);
            float2 f = __half22float2(h);
            out[2 * i] = f.x;
            out[2 * i + 1] = f.y;
        }
    }
    __device__ static __forceinline__ Vec16 pack(const float* in)
    {
        Vec16 v;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            __half2 h = __floats2half2_rn(in[2 * i], in[2 * i + 1]);
            v.w[i] = *reinterpret_cast<uint32_t*>(&h);
        }
        return v;
    }
    __device__ static __forceinline__ float to_f(__half x) { return __half2float(x); }
    __device__ static __forceinline__ __half from_f(float x) { return __float2half_rn(x); }
};

// ---------------------------------------------------------------------------------------------
// reductions
// ---------------------------------------------------------------------------------------------
struct SumOp {
    __device__ __forceinline__ float operator()(float a, float b) const { return a + b; }
    __host__ __device__ static constexpr float identity() { return 0.f; }
};
struct MaxOp {
    __device__ __forceinline__ float operator()(float a, float b) const { return fmaxf(a, b); }
    __host__ __device__ static constexpr float identity() { return -3.402823466e+38f; }
};

template <typename Op>
__device__ __forceinline__ float warp_reduce(float v, Op op = Op())
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Block-wide all-reduce; `scratch` must hold >= 32 floats of shared memory.  All threads get
// the result.  Safe to call repeatedly with the same scratch (trailing barrier).
template <typename Op>
__device__ __forceinline__ float block_reduce(float v, float* scratch, Op op = Op())
{
    const int lane = threadIdx.x & 31;
    const int wid = threadIdx.x >> 5;
    const int nw = (blockDim.x + 31) >> 5;
    v = warp_reduce<Op>(v, op);
    if (lane == 0) scratch[wid] = v;
    __syncthreads();
    float r = (lane < nw) ? scratch[lane] : Op::identity();
    r = warp_reduce<Op>(r, op);
    __syncthreads();
    return r;
}

// Two values at once (sum, sumsq) to halve barrier count.
__device__ __forceinline__ float2 block_reduce_sum2(float a, float b, float* scratch)
{
    const int lane = threadIdx.x & 31;
    const int wid = threadIdx.x >> 5;
    const int nw = (blockDim.x + 31) >> 5;
    a = warp_reduce<SumOp>(a);
    b = warp_reduce<SumOp>(b);
    if (lane == 0) {
        scratch[wid] = a;
        scratch[32 + wid] = b;
    }
    __syncthreads();
    float ra = (lane < nw) ? scratch[lane] : 0.f;
    float rb = (lane < nw) ? scratch[32 + lane] : 0.f;
    ra = warp_reduce<SumOp>(ra);
    rb = warp_reduce<SumOp>(rb);
    __syncthreads();
    return make_float2(ra, rb);
}

__host__ __device__ __forceinline__ int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Grid sizing for bandwidth-bound flat kernels: a multiple of the SM count, capped so each
// block has enough work to amortise launch (grid-stride loops handle the rest).
inline int flat_grid(int64_t n_vec, int threads, int blocks_per_sm = 8, int sm_count = kSmCountH100)
{
    int64_t need = ceil_div(n_vec, threads);
    int64_t cap = static_cast<int64_t>(sm_count) * blocks_per_sm;
    if (need < 1) need = 1;
    return static_cast<int>(need < cap ? need : cap);
}

}  // namespace dsb
