// Quantization kernels for sm_90a.
//   * group-wise INT8 / INT4 symmetric + asymmetric quantize / dequantize (ZeRO++ qwZ weights)
//   * swizzled quantize: quantize AND lay partitions out in (device, node) order for the 2-hop all-to-all (qgZ)
//   * fused dequantize -> reduce -> requantize across the chunks received from N peers (qgZ middle step),
//     plus LoCo error-feedback variants
//   * fake quantization (quantize-dequantize in one pass) with optional stochastic rounding (MoQ / QAT)
//   * minifloat group quantization: FP8 (E4M3 / E5M2), FP6 (E3M2), FP4 (E2M1), FP12 (E4M7) with per-group
//     fp32 scales, stochastic rounding, dequantize and index-selected dequantize (LoRA base weights)
//
// Role parity: reference csrc/quantization/{quantize,dequantize,swizzled_quantize,quant_reduce,
// fake_quantizer,quantize_intX}.cu (N5) and csrc/fp_quantizer/fp_quantize.cu (N6).  Independent design:
// one CTA per quantization group with 16-byte loads, the group cached in registers between the
// range pass and the encode pass, and one generic minifloat codec instead of per-format kernels.
#include <cuda_fp8.h>
#include "dsb_common.cuh"

namespace dsb {
namespace quant {

constexpr int kThreads = 256;
constexpr int kMaxCache = 4;  // 16-byte vectors cached per thread (covers groups up to 8192 16-bit elements)

__device__ __forceinline__ uint32_t hash_u32(uint32_t x)
{
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}
// uniform in [0,1)
__device__ __forceinline__ float rand01(uint32_t seed, uint32_t idx) { return (hash_u32(seed ^ (idx * 0x9e3779b9u)) >> 8) * (1.0f / 16777216.0f); }

// floor(t + r) for r in [0, 1), exactly: the fp32 sum itself can round up to the next integer (0.5 - 2^-25 + 0.5 is 1)
__device__ __forceinline__ float floor_add(float t, float r)
{
    const float q = floorf(t);
    return (t - q) >= 1.f - r ? q + 1.f : q;
}

struct Range {
    float lo, hi;
};

// Non-finite groups: the range reductions propagate NaN (fmaxf would drop it), so a group holding a NaN or an inf
// has a non-finite range, gets a NaN scale, and every element of it dequantizes to NaN.  So does an asymmetric group
// whose range hi - lo overflows fp32: no finite scale spans it.  Its codes are whatever the NaN quotient clamps to;
// only the scale carries the information.
__device__ __forceinline__ float nan_max(float a, float b) { return (a > b || a != a) ? a : b; }
struct NanMaxOp {
    __device__ __forceinline__ float operator()(float a, float b) const { return nan_max(a, b); }
    __host__ __device__ static constexpr float identity() { return -3.402823466e+38f; }
};

// Scale of a group whose range is `span` (amax, or hi - lo) spread over `levels` steps.  NaN when the range is not
// finite; at least the smallest fp32 subnormal, so that a tiny group keeps a non-zero scale.
__device__ __forceinline__ float group_scale(float span, float levels)
{
    if (!isfinite(span)) return __int_as_float(0x7fc00000);
    return span > 0.f ? fmaxf(span / levels, 1.401298464e-45f) : 1.f;
}

// x / scale through the fp32 reciprocal `inv`; when 1/scale overflows (scale below 2^-128) divide instead, so that
// a zero still encodes to zero.
__device__ __forceinline__ float to_grid(float x, float scale, float inv) { return isfinite(inv) ? x * inv : x / scale; }

// Block-wide min/max of one group (elements [base, base+n)); leaves the unpacked group in `cache`.
template <typename T>
__device__ __forceinline__ Range group_range(const T* __restrict__ x, int n, float cache[kMaxCache][Elem<T>::kPerVec],
                                             float* scratch)
{
    constexpr int kPer = Elem<T>::kPerVec;
    const int nvec = n / kPer;
    float lo = 3.402823466e+38f, hi = -3.402823466e+38f;
#pragma unroll
    for (int k = 0; k < kMaxCache; ++k) {
        const int v = threadIdx.x + k * blockDim.x;
        if (v < nvec) {
            Elem<T>::unpack(ld_stream(x + v * kPer), cache[k]);
#pragma unroll
            for (int e = 0; e < kPer; ++e) {
                lo = -nan_max(-lo, -cache[k][e]);
                hi = nan_max(hi, cache[k][e]);
            }
        }
    }
    // (n is required to be a multiple of kPer and <= kMaxCache * blockDim * kPer by the host wrapper)
    hi = block_reduce<NanMaxOp>(hi, scratch);
    lo = -block_reduce<NanMaxOp>(-lo, scratch);
    return Range{lo, hi};
}

// ---- integer group quantization ----------------------------------------------------------------------------
// params layout: symmetric -> [groups] scale ; asymmetric -> [groups, 2] (scale, offset) with x ~ q*scale + offset
template <typename T, int BITS, bool SYM>
__global__ void __launch_bounds__(kThreads)
quantize_kernel(const T* __restrict__ x, int8_t* __restrict__ q, float* __restrict__ params, int group_size,
                int64_t out_group_stride_bytes, const int* __restrict__ group_perm, int stochastic, uint32_t seed)
{
    __shared__ float scratch[32];
    constexpr int kPer = Elem<T>::kPerVec;
    const int g = blockIdx.x;
    const T* xg = x + static_cast<int64_t>(g) * group_size;
    float cache[kMaxCache][kPer];
    const Range r = group_range<T>(xg, group_size, cache, scratch);
    constexpr float qmax = static_cast<float>((1 << (BITS - 1)) - 1);
    constexpr float qmin_asym = 0.f, qmax_asym = static_cast<float>((1 << BITS) - 1);
    float scale, offset = 0.f;
    if (SYM) {
        const float amax = fmaxf(fabsf(r.lo), fabsf(r.hi));
        scale = group_scale(amax, qmax + 1.f);  // amax -> 2^(b-1); +side saturates
    } else {
        scale = group_scale(r.hi - r.lo, qmax_asym + 1.f);
        offset = r.lo;
    }
    const float inv = 1.f / scale;
    const int og = group_perm ? group_perm[g] : g;
    if (threadIdx.x == 0) {
        if (SYM) {
            params[og] = scale;
        } else {
            params[2 * og] = scale;
            params[2 * og + 1] = offset;
        }
    }
    int8_t* qg = q + static_cast<int64_t>(og) * out_group_stride_bytes;
    const int nvec = group_size / kPer;
#pragma unroll
    for (int k = 0; k < kMaxCache; ++k) {
        const int v = threadIdx.x + k * blockDim.x;
        if (v < nvec) {
            int qi[kPer];
#pragma unroll
            for (int e = 0; e < kPer; ++e) {
                float f = to_grid(cache[k][e] - offset, scale, inv);
                if (stochastic) {
                    f = floor_add(f, rand01(seed, static_cast<uint32_t>(g * group_size + v * kPer + e)));
                } else {
                    f = rintf(f);
                }
                f = SYM ? fminf(fmaxf(f, -qmax - 1.f), qmax) : fminf(fmaxf(f, qmin_asym), qmax_asym);
                qi[e] = static_cast<int>(f);
            }
            if (BITS == 8) {
#pragma unroll
                for (int e = 0; e < kPer; ++e) qg[v * kPer + e] = static_cast<int8_t>(SYM ? qi[e] : qi[e] - 128);
            } else {  // 4-bit: two values per byte, low nibble first
#pragma unroll
                for (int e = 0; e < kPer; e += 2) {
                    const int a = SYM ? (qi[e] & 0xf) : qi[e];
                    const int b = SYM ? (qi[e + 1] & 0xf) : qi[e + 1];
                    qg[(v * kPer + e) >> 1] = static_cast<int8_t>((b << 4) | (a & 0xf));
                }
            }
        }
    }
}

// ---- LoCo (error-feedback) quantisation: q = Q(x + err);  err <- beta * err + (1 - beta) * ((x + err) - deQ(q)) -------------
// One pass: the compensated values and the old error stay in registers between the range reduction and the write-back
// (reference csrc/quantization/swizzled_quantize.cu loco_swizzled_quant_kernel).  Symmetric, 4 or 8 bits.
template <typename T, int BITS>
__global__ void __launch_bounds__(kThreads)
loco_quantize_kernel(const T* __restrict__ x, float* __restrict__ err, int8_t* __restrict__ q, float* __restrict__ params,
                     int group_size, int64_t out_group_stride_bytes, float beta, int reset)
{
    __shared__ float scratch[32];
    constexpr int kPer = Elem<T>::kPerVec;
    const int g = blockIdx.x;
    const T* xg = x + static_cast<int64_t>(g) * group_size;
    float* eg = err + static_cast<int64_t>(g) * group_size;
    float comp[kMaxCache][kPer], old[kMaxCache][kPer];
    const int nvec = group_size / kPer;
    float amax = 0.f;
#pragma unroll
    for (int k = 0; k < kMaxCache; ++k) {
        const int v = threadIdx.x + k * blockDim.x;
        if (v < nvec) {
            Elem<T>::unpack(ld_stream(xg + v * kPer), comp[k]);
#pragma unroll
            for (int e = 0; e < kPer; ++e) {
                old[k][e] = eg[v * kPer + e];
                comp[k][e] += old[k][e];
                amax = nan_max(amax, fabsf(comp[k][e]));
            }
        }
    }
    amax = block_reduce<NanMaxOp>(amax, scratch);
    constexpr float qmax = static_cast<float>((1 << (BITS - 1)) - 1);
    const float scale = group_scale(amax, qmax + 1.f);  // amax -> 2^(b-1); +side saturates
    const float inv = 1.f / scale;
    const bool finite = isfinite(scale);  // a non-finite group leaves its error slice as it was: that step is skipped
    if (threadIdx.x == 0) params[g] = scale;
    int8_t* qg = q + static_cast<int64_t>(g) * out_group_stride_bytes;
#pragma unroll
    for (int k = 0; k < kMaxCache; ++k) {
        const int v = threadIdx.x + k * blockDim.x;
        if (v < nvec) {
            int qi[kPer];
#pragma unroll
            for (int e = 0; e < kPer; ++e) {
                float f = fminf(fmaxf(rintf(to_grid(comp[k][e], scale, inv)), -qmax - 1.f), qmax);
                qi[e] = static_cast<int>(f);
                const float new_err = __fmaf_rn(-f, scale, comp[k][e]);
                if (finite) eg[v * kPer + e] = reset ? 0.f : __fmaf_rn(beta, old[k][e], __fmul_rn(1.f - beta, new_err));
            }
            if (BITS == 8) {
#pragma unroll
                for (int e = 0; e < kPer; ++e) qg[v * kPer + e] = static_cast<int8_t>(qi[e]);
            } else {
#pragma unroll
                for (int e = 0; e < kPer; e += 2)
                    qg[(v * kPer + e) >> 1] = static_cast<int8_t>(((qi[e + 1] & 0xf) << 4) | (qi[e] & 0xf));
            }
        }
    }
}

__device__ __forceinline__ float dequant_one(const int8_t* qg, int i, int bits, bool sym, float scale, float offset)
{
    int v;
    if (bits == 8) {
        v = sym ? static_cast<int>(qg[i]) : static_cast<int>(qg[i]) + 128;
    } else {
        const int byte = static_cast<uint8_t>(qg[i >> 1]);
        v = (i & 1) ? (byte >> 4) : (byte & 0xf);
        if (sym && (v & 8)) v -= 16;
    }
    return __fmaf_rn(static_cast<float>(v), scale, offset);
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
dequantize_kernel(const int8_t* __restrict__ q, const float* __restrict__ params, T* __restrict__ out, int group_size,
                  int64_t total, int bits, int sym)
{
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    const int bytes_per_group = bits == 8 ? group_size : group_size / 2;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int64_t g = i / group_size;
        const int e = static_cast<int>(i - g * group_size);
        const float scale = sym ? params[g] : params[2 * g];
        const float off = sym ? 0.f : params[2 * g + 1];
        out[i] = Elem<T>::from_f(dequant_one(q + g * bytes_per_group, e, bits, sym != 0, scale, off));
    }
}

// ---- dequant -> reduce -> requant (qgZ) -------------------------------------------------------------------------
// input: `peers` chunks, each [out_groups, group_size] quantized (+ params [peers, out_groups(,2)]).
// output group g = requant( sum_p dequant(chunk_p[g]) ).  Optional LoCo error feedback: err[g,:] (fp32)
// is added before requantisation and updated with the new quantisation error.
template <int BITS, bool SYM>
__global__ void __launch_bounds__(kThreads)
dequant_reduce_kernel(const int8_t* __restrict__ qin, const float* __restrict__ pin, int8_t* __restrict__ qout,
                      float* __restrict__ pout, int peers, int out_groups, int group_size, float* __restrict__ err,
                      float err_beta)
{
    __shared__ float scratch[32];
    extern __shared__ float acc[];  // group_size floats
    const int g = blockIdx.x;
    const int bpg = BITS == 8 ? group_size : group_size / 2;
    for (int i = threadIdx.x; i < group_size; i += blockDim.x) {
        float s = 0.f;
        for (int p = 0; p < peers; ++p) {
            const int64_t gi = static_cast<int64_t>(p) * out_groups + g;
            const float scale = SYM ? pin[gi] : pin[2 * gi];
            const float off = SYM ? 0.f : pin[2 * gi + 1];
            s += dequant_one(qin + gi * bpg, i, BITS, SYM, scale, off);
        }
        if (err) s = __fmaf_rn(err_beta, err[static_cast<int64_t>(g) * group_size + i], s);
        acc[i] = s;
    }
    __syncthreads();
    float lo = 3.402823466e+38f, hi = -3.402823466e+38f;
    for (int i = threadIdx.x; i < group_size; i += blockDim.x) {
        lo = -nan_max(-lo, -acc[i]);
        hi = nan_max(hi, acc[i]);
    }
    hi = block_reduce<NanMaxOp>(hi, scratch);
    lo = -block_reduce<NanMaxOp>(-lo, scratch);
    constexpr float qmax = static_cast<float>((1 << (BITS - 1)) - 1);
    constexpr float qmax_asym = static_cast<float>((1 << BITS) - 1);
    float scale, offset = 0.f;
    if (SYM) {
        const float amax = fmaxf(fabsf(lo), fabsf(hi));
        scale = group_scale(amax, qmax + 1.f);  // amax -> 2^(b-1); +side saturates
    } else {
        scale = group_scale(hi - lo, qmax_asym + 1.f);
        offset = lo;
    }
    if (threadIdx.x == 0) {
        if (SYM) {
            pout[g] = scale;
        } else {
            pout[2 * g] = scale;
            pout[2 * g + 1] = offset;
        }
    }
    const float inv = 1.f / scale;
    int8_t* qg = qout + static_cast<int64_t>(g) * bpg;
    const int step = BITS == 8 ? 1 : 2;
    for (int i = threadIdx.x * step; i < group_size; i += blockDim.x * step) {
        int qi[2];
        for (int e = 0; e < step; ++e) {
            float f = rintf(to_grid(acc[i + e] - offset, scale, inv));
            f = SYM ? fminf(fmaxf(f, -qmax - 1.f), qmax) : fminf(fmaxf(f, 0.f), qmax_asym);
            qi[e] = static_cast<int>(f);
            if (err && isfinite(scale))  // a non-finite group leaves its error slice as it was
                err[static_cast<int64_t>(g) * group_size + i + e] = acc[i + e] - __fmaf_rn(f, scale, offset);
        }
        if (BITS == 8)
            qg[i] = static_cast<int8_t>(SYM ? qi[0] : qi[0] - 128);
        else
            qg[i >> 1] = static_cast<int8_t>(((SYM ? (qi[1] & 0xf) : qi[1]) << 4) | ((SYM ? qi[0] : qi[0]) & 0xf));
    }
}

// ---- fake quantization (MoQ / QAT): x <- dequant(quant(x)) in place ---------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads)
fake_quant_kernel(T* __restrict__ x, int group_size, int bits, int sym, int stochastic, uint32_t seed)
{
    __shared__ float scratch[32];
    constexpr int kPer = Elem<T>::kPerVec;
    const int g = blockIdx.x;
    T* xg = x + static_cast<int64_t>(g) * group_size;
    float cache[kMaxCache][kPer];
    const Range r = group_range<T>(xg, group_size, cache, scratch);
    const float levels = static_cast<float>((1 << bits) - 1);
    const float qmax = static_cast<float>((1 << (bits - 1)) - 1);
    float scale, offset = 0.f, lo_q, hi_q;
    if (sym) {
        const float amax = fmaxf(fabsf(r.lo), fabsf(r.hi));
        scale = group_scale(amax, qmax + 1.f);  // amax -> 2^(b-1); +side saturates
        lo_q = -qmax - 1.f;
        hi_q = qmax;
    } else {
        scale = group_scale(r.hi - r.lo, levels + 1.f);
        offset = r.lo;
        lo_q = 0.f;
        hi_q = levels;
    }
    const float inv = 1.f / scale;
    const int nvec = group_size / kPer;
#pragma unroll
    for (int k = 0; k < kMaxCache; ++k) {
        const int v = threadIdx.x + k * blockDim.x;
        if (v < nvec) {
            float o[kPer];
#pragma unroll
            for (int e = 0; e < kPer; ++e) {
                float f = to_grid(cache[k][e] - offset, scale, inv);
                f = stochastic ? floor_add(f, rand01(seed, static_cast<uint32_t>(g * group_size + v * kPer + e))) : rintf(f);
                f = fminf(fmaxf(f, lo_q), hi_q);
                o[e] = __fmaf_rn(f, scale, offset);
            }
            st_plain(xg + v * kPer, Elem<T>::pack(o));
        }
    }
}

// ---- minifloat codec --------------------------------------------------------------------------------------------------
// Generic sign/exponent/mantissa format without inf/nan codes (FP6 E3M2, FP4 E2M1, FP12 E4M7); FP8 uses the
// hardware conversions.  `rnd` in [0,1): 0.5 gives round-to-nearest (ties away), anything else is stochastic.
__device__ __forceinline__ float minifloat_max(int E, int M)
{
    const int bias = (1 << (E - 1)) - 1;
    return (2.f - ldexpf(1.f, -M)) * ldexpf(1.f, ((1 << E) - 1) - bias);
}

__device__ __forceinline__ uint32_t minifloat_encode(float x, int E, int M, float rnd)
{
    const int bias = (1 << (E - 1)) - 1;
    const uint32_t sign = x < 0.f ? 1u : 0u;
    float a = fminf(fabsf(x), minifloat_max(E, M));
    uint32_t code;
    const float min_normal = ldexpf(1.f, 1 - bias);
    if (a < min_normal) {
        const float q = floor_add(a * ldexpf(1.f, M - (1 - bias)), rnd);  // units of the subnormal step
        code = static_cast<uint32_t>(q);                                 // == 1<<M rolls into the first normal
    } else {
        int e;
        const float fr = frexpf(a, &e);  // a = fr * 2^e, fr in [0.5,1)
        e -= 1;                          // a = (2*fr) * 2^e with 2*fr in [1,2)
        float m = floor_add((2.f * fr - 1.f) * static_cast<float>(1 << M), rnd);
        if (m >= static_cast<float>(1 << M)) {
            m = 0.f;
            e += 1;
        }
        const int emax = ((1 << E) - 1) - bias;
        if (e > emax) {
            e = emax;
            m = static_cast<float>((1 << M) - 1);
        }
        code = (static_cast<uint32_t>(e + bias) << M) | static_cast<uint32_t>(m);
    }
    return (sign << (E + M)) | code;
}

__device__ __forceinline__ float minifloat_decode(uint32_t code, int E, int M)
{
    const int bias = (1 << (E - 1)) - 1;
    const uint32_t sign = (code >> (E + M)) & 1u;
    const uint32_t ef = (code >> M) & ((1u << E) - 1u);
    const uint32_t mf = code & ((1u << M) - 1u);
    float v;
    if (ef == 0)
        v = static_cast<float>(mf) * ldexpf(1.f, (1 - bias) - M);
    else
        v = (1.f + static_cast<float>(mf) * ldexpf(1.f, -M)) * ldexpf(1.f, static_cast<int>(ef) - bias);
    return sign ? -v : v;
}

__device__ __forceinline__ float fp_format_max(int bits, int M)
{
    if (bits == 8) return M == 3 ? 448.f : 57344.f;
    return minifloat_max(bits - 1 - M, M);
}

__device__ __forceinline__ float fp_decode(uint32_t code, int bits, int M)
{
    if (bits == 8) {
        const __half_raw h = __nv_cvt_fp8_to_halfraw(static_cast<__nv_fp8_storage_t>(code), M == 3 ? __NV_E4M3 : __NV_E5M2);
        return __half2float(*reinterpret_cast<const __half*>(&h));
    }
    return minifloat_decode(code, bits - 1 - M, M);
}

__device__ __forceinline__ uint32_t fp_encode(float x, int bits, int M, float rnd)
{
    if (bits == 8) {
        const __nv_fp8_interpretation_t fmt = M == 3 ? __NV_E4M3 : __NV_E5M2;
        if (rnd != 0.5f && x == x) {
            // stochastic: floor(|x| / ulp + rnd) * ulp, with ulp the grid spacing at |x| (the subnormal step below
            // the smallest normal).  The hardware only rounds to nearest, so convert |x| + rnd * ulp and step one
            // code down when that rounded up.
            const float ax = fabsf(x);
            const int emin = M == 3 ? -6 : -14;  // exponent of the smallest normal
            int e;
            frexpf(ax, &e);  // ax in [2^(e-1), 2^e)
            const float ulp = ldexpf(1.f, (ax < ldexpf(1.f, emin) ? emin : e - 1) - M);
            const float y = ax + rnd * ulp;
            uint32_t c = __nv_cvt_float_to_fp8(y, __NV_SATFINITE, fmt);
            if (fp_decode(c, 8, M) > y) c -= 1;
            return x < 0.f ? (c | 0x80u) : c;
        }
        return static_cast<uint32_t>(__nv_cvt_float_to_fp8(x, __NV_SATFINITE, fmt));
    }
    return minifloat_encode(x, bits - 1 - M, M, rnd);
}

// Packed code storage: codes of `bits` width are written little-endian into a byte stream per group.
__device__ __forceinline__ void put_bits(uint8_t* base, int64_t bitpos, uint32_t code, int bits)
{
    // only used for 6- and 12-bit formats by a single thread per 4 (resp. 2) codes -> no races
    for (int b = 0; b < bits; ++b) {
        const int64_t p = bitpos + b;
        const uint8_t mask = static_cast<uint8_t>(1u << (p & 7));
        if ((code >> b) & 1u)
            base[p >> 3] |= mask;
        else
            base[p >> 3] &= static_cast<uint8_t>(~mask);
    }
}
__device__ __forceinline__ uint32_t get_bits(const uint8_t* base, int64_t bitpos, int bits)
{
    uint32_t v = 0;
    const int64_t byte0 = bitpos >> 3;
    const int shift = static_cast<int>(bitpos & 7);
    uint32_t window = base[byte0] | (static_cast<uint32_t>(base[byte0 + 1]) << 8);
    if (shift + bits > 16) window |= static_cast<uint32_t>(base[byte0 + 2]) << 16;
    v = (window >> shift) & ((1u << bits) - 1u);
    return v;
}

// One warp per group (like the reference: 8 groups per 256-thread CTA).  Layout of one output group:
// ceil(group_size * bits / 8) payload bytes followed (in a separate array) by one fp32 scale.
template <typename T>
__global__ void __launch_bounds__(kThreads)
fp_quantize_kernel(const T* __restrict__ x, uint8_t* __restrict__ q, float* __restrict__ scales, int64_t groups,
                   int group_size, int bits, int M, int stochastic, uint32_t seed)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t g = static_cast<int64_t>(blockIdx.x) * (kThreads / 32) + warp;
    if (g >= groups) return;
    const T* xg = x + g * group_size;
    float amax = 0.f;
    for (int i = lane; i < group_size; i += 32) amax = nan_max(amax, fabsf(Elem<T>::to_f(xg[i])));
    amax = warp_reduce<NanMaxOp>(amax);
    const float scale = group_scale(amax, fp_format_max(bits, M));
    const float inv = 1.f / scale;
    if (lane == 0) scales[g] = scale;
    const int64_t bytes_per_group = (static_cast<int64_t>(group_size) * bits + 7) / 8;
    uint8_t* qg = q + g * bytes_per_group;
    // each lane encodes runs of `per` codes that fill whole bytes: 8-bit:1, 4-bit:2, 6-bit:4 (3 B), 12-bit:2 (3 B)
    const int per = bits == 8 ? 1 : (bits == 6 ? 4 : 2);
    for (int i0 = lane * per; i0 < group_size; i0 += 32 * per) {
        uint32_t codes[4];
        for (int e = 0; e < per; ++e) {
            const int i = i0 + e;
            const float v = i < group_size ? to_grid(Elem<T>::to_f(xg[i]), scale, inv) : 0.f;
            const float rnd = stochastic ? rand01(seed, static_cast<uint32_t>(g * group_size + i)) : 0.5f;
            codes[e] = fp_encode(v, bits, M, rnd);
        }
        if (bits == 8) {
            qg[i0] = static_cast<uint8_t>(codes[0]);
        } else if (bits == 4) {
            qg[i0 >> 1] = static_cast<uint8_t>((codes[0] & 0xf) | ((codes[1] & 0xf) << 4));
        } else if (bits == 6) {
            const uint32_t w = (codes[0] & 0x3f) | ((codes[1] & 0x3f) << 6) | ((codes[2] & 0x3f) << 12) |
                               ((codes[3] & 0x3f) << 18);
            uint8_t* d = qg + (i0 / 4) * 3;
            d[0] = static_cast<uint8_t>(w);
            d[1] = static_cast<uint8_t>(w >> 8);
            d[2] = static_cast<uint8_t>(w >> 16);
        } else {  // 12
            const uint32_t w = (codes[0] & 0xfff) | ((codes[1] & 0xfff) << 12);
            uint8_t* d = qg + (i0 / 2) * 3;
            d[0] = static_cast<uint8_t>(w);
            d[1] = static_cast<uint8_t>(w >> 8);
            d[2] = static_cast<uint8_t>(w >> 16);
        }
    }
}

__device__ __forceinline__ uint32_t fp_fetch(const uint8_t* qg, int i, int bits)
{
    if (bits == 8) return qg[i];
    if (bits == 4) return (qg[i >> 1] >> ((i & 1) * 4)) & 0xf;
    if (bits == 6) {
        const uint8_t* d = qg + (i / 4) * 3;
        const uint32_t w = d[0] | (static_cast<uint32_t>(d[1]) << 8) | (static_cast<uint32_t>(d[2]) << 16);
        return (w >> ((i & 3) * 6)) & 0x3f;
    }
    const uint8_t* d = qg + (i / 2) * 3;
    const uint32_t w = d[0] | (static_cast<uint32_t>(d[1]) << 8) | (static_cast<uint32_t>(d[2]) << 16);
    return (w >> ((i & 1) * 12)) & 0xfff;
}

// rows (optional): dequantize only the listed groups-of-rows (selective dequantize); row r of the output
// corresponds to input row rows[r]; each row spans `groups_per_row` groups.
template <typename T>
__global__ void __launch_bounds__(kThreads)
fp_dequantize_kernel(const uint8_t* __restrict__ q, const float* __restrict__ scales, T* __restrict__ out,
                     int64_t out_groups, int group_size, int bits, int M, const int* __restrict__ rows,
                     int groups_per_row)
{
    const int64_t bytes_per_group = (static_cast<int64_t>(group_size) * bits + 7) / 8;
    const int64_t total = out_groups * group_size;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
    for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int64_t og = i / group_size;
        const int e = static_cast<int>(i - og * group_size);
        int64_t ig = og;
        if (rows) ig = static_cast<int64_t>(rows[og / groups_per_row]) * groups_per_row + (og % groups_per_row);
        const uint32_t code = fp_fetch(q + ig * bytes_per_group, e, bits);
        out[i] = Elem<T>::from_f(fp_decode(code, bits, M) * scales[ig]);
    }
}

}  // namespace quant
}  // namespace dsb

using namespace dsb;
using namespace dsb::quant;

#define DISPATCH_QT(code, T, ...)  \
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

static inline bool group_ok(int group_size, int dtype)
{
    const int per = dtype == kF32 ? 4 : 8;
    return group_size % per == 0 && group_size <= kMaxCache * kThreads * per && group_size % 2 == 0;
}

// group_perm (device int32[groups], nullable) sends input group g to output slot group_perm[g] (swizzle).
DSB_EXPORT int dsb_quantize(const void* x, void* q, float* params, int64_t groups, int group_size, int bits, int sym,
                            int dtype, const int* group_perm, int stochastic, uint32_t seed, cudaStream_t stream)
{
    if (groups <= 0) return 0;
    if (!group_ok(group_size, dtype) || (bits != 4 && bits != 8)) return -2;
    const int64_t obytes = bits == 8 ? group_size : group_size / 2;
    DISPATCH_QT(dtype, T, {
        if (bits == 8 && sym)
            quantize_kernel<T, 8, true><<<groups, kThreads, 0, stream>>>((const T*)x, (int8_t*)q, params, group_size,
                                                                          obytes, group_perm, stochastic, seed);
        else if (bits == 8)
            quantize_kernel<T, 8, false><<<groups, kThreads, 0, stream>>>((const T*)x, (int8_t*)q, params, group_size,
                                                                           obytes, group_perm, stochastic, seed);
        else if (sym)
            quantize_kernel<T, 4, true><<<groups, kThreads, 0, stream>>>((const T*)x, (int8_t*)q, params, group_size,
                                                                          obytes, group_perm, stochastic, seed);
        else
            quantize_kernel<T, 4, false><<<groups, kThreads, 0, stream>>>((const T*)x, (int8_t*)q, params, group_size,
                                                                           obytes, group_perm, stochastic, seed);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

// x [groups * group_size] (T), err fp32 same length (updated in place), q int8 (4-bit: two per byte), params fp32 [groups]
DSB_EXPORT int dsb_loco_quantize(const void* x, float* err, void* q, float* params, int64_t groups, int group_size, int bits,
                                 int dtype, float beta, int reset, cudaStream_t stream)
{
    if (groups <= 0) return 0;
    if (!group_ok(group_size, dtype) || (bits != 4 && bits != 8)) return -2;
    const int64_t obytes = bits == 8 ? group_size : group_size / 2;
    DISPATCH_QT(dtype, T, {
        if (bits == 8)
            loco_quantize_kernel<T, 8><<<groups, kThreads, 0, stream>>>((const T*)x, err, (int8_t*)q, params, group_size, obytes,
                                                                        beta, reset);
        else
            loco_quantize_kernel<T, 4><<<groups, kThreads, 0, stream>>>((const T*)x, err, (int8_t*)q, params, group_size, obytes,
                                                                        beta, reset);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_dequantize(const void* q, const float* params, void* out, int64_t groups, int group_size, int bits,
                              int sym, int out_dtype, cudaStream_t stream)
{
    if (groups <= 0) return 0;
    if ((bits != 4 && bits != 8) || group_size % 2) return -2;
    const int64_t total = groups * group_size;
    const int grid = flat_grid(total, kThreads, 16);
    DISPATCH_QT(out_dtype, T, {
        dequantize_kernel<T><<<grid, kThreads, 0, stream>>>((const int8_t*)q, params, (T*)out, group_size, total, bits, sym);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

template <int BITS, bool SYM>
static void launch_dequant_reduce(const void* qin, const float* pin, void* qout, float* pout, int peers, int out_groups,
                                  int group_size, float* err, float err_beta, size_t smem, cudaStream_t stream)
{
    // the kernel's static scratch comes on top of the dynamic accumulators: past the default 48 KB in all for the
    // largest groups, so opt in to 48 KB of dynamic shared memory
    if (smem > 46 * 1024)
        cudaFuncSetAttribute(dequant_reduce_kernel<BITS, SYM>, cudaFuncAttributeMaxDynamicSharedMemorySize, 48 * 1024);
    dequant_reduce_kernel<BITS, SYM><<<out_groups, kThreads, smem, stream>>>((const int8_t*)qin, pin, (int8_t*)qout, pout,
                                                                            peers, out_groups, group_size, err, err_beta);
}

DSB_EXPORT int dsb_dequant_reduce(const void* qin, const float* pin, void* qout, float* pout, int peers, int out_groups,
                                  int group_size, int bits, int sym, float* err, float err_beta, cudaStream_t stream)
{
    if (out_groups <= 0) return 0;
    if (group_size % 2 || (bits != 4 && bits != 8)) return -2;
    const size_t smem = static_cast<size_t>(group_size) * sizeof(float);
    if (smem > 48 * 1024) return -2;
    if (bits == 8 && sym)
        launch_dequant_reduce<8, true>(qin, pin, qout, pout, peers, out_groups, group_size, err, err_beta, smem, stream);
    else if (bits == 8)
        launch_dequant_reduce<8, false>(qin, pin, qout, pout, peers, out_groups, group_size, err, err_beta, smem, stream);
    else if (sym)
        launch_dequant_reduce<4, true>(qin, pin, qout, pout, peers, out_groups, group_size, err, err_beta, smem, stream);
    else
        launch_dequant_reduce<4, false>(qin, pin, qout, pout, peers, out_groups, group_size, err, err_beta, smem, stream);
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_fake_quantize(void* x, int64_t groups, int group_size, int bits, int sym, int dtype, int stochastic,
                                 uint32_t seed, cudaStream_t stream)
{
    if (groups <= 0) return 0;
    if (!group_ok(group_size, dtype) || bits < 2 || bits > 16) return -2;
    DISPATCH_QT(dtype, T, {
        fake_quant_kernel<T><<<groups, kThreads, 0, stream>>>((T*)x, group_size, bits, sym, stochastic, seed);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

// bits in {4, 6, 8, 12}; mantissa bits M: FP8 E4M3 -> 3, E5M2 -> 2, FP6 -> 2, FP4 -> 1, FP12 -> 7
static inline bool fp_format_ok(int bits, int M)
{
    return (bits == 8 && (M == 3 || M == 2)) || (bits == 6 && M == 2) || (bits == 4 && M == 1) || (bits == 12 && M == 7);
}

DSB_EXPORT int dsb_fp_quantize(const void* x, void* q, float* scales, int64_t groups, int group_size, int bits, int M,
                               int dtype, int stochastic, uint32_t seed, cudaStream_t stream)
{
    if (groups <= 0) return 0;
    if (!fp_format_ok(bits, M) || group_size % 4) return -2;
    const int grid = static_cast<int>((groups + (kThreads / 32) - 1) / (kThreads / 32));
    DISPATCH_QT(dtype, T, {
        fp_quantize_kernel<T><<<grid, kThreads, 0, stream>>>((const T*)x, (uint8_t*)q, scales, groups, group_size, bits, M,
                                                             stochastic, seed);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_fp_dequantize(const void* q, const float* scales, void* out, int64_t out_groups, int group_size,
                                 int bits, int M, int out_dtype, const int* rows, int groups_per_row, cudaStream_t stream)
{
    if (out_groups <= 0) return 0;
    if (!fp_format_ok(bits, M) || group_size % 4) return -2;
    const int grid = flat_grid(out_groups * group_size, kThreads, 16);
    DISPATCH_QT(out_dtype, T, {
        fp_dequantize_kernel<T><<<grid, kThreads, 0, stream>>>((const uint8_t*)q, scales, (T*)out, out_groups, group_size,
                                                               bits, M, rows, groups_per_row);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}
