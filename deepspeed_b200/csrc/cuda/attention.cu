// Paged-KV attention for ragged (continuous-batching) inference on sm_90a.
//
// One CTA per (query token, query head).  K/V live in a blocked cache laid out by `kv_rotary_append`
// (moe_ragged.cu): cache[block][slot][k|v][kv_head][d].  Each warp walks a strided subset of the visible
// keys with an online softmax (running max / sum, fp32 accumulators), lanes split the head dimension;
// the four per-warp partial states are merged through shared memory.  GQA: query head h reads kv head
// h / (hq / hkv).  Causality: query token with absolute position p sees keys [0, p].
//
// Role parity: reference inference/v2/kernels/ragged_ops/blocked_flash (N9b, a wrapper over the external
// `dskernels` flash-attention build) and the v1 `softmax_context` decode path (N8).  Prefill-sized work goes
// through the training attention path (ops/attention.py); this kernel is the decode / short-chunk path.
#include <cstdlib>
#include "dsb_common.cuh"

namespace dsb {
namespace pattn {

constexpr int kWarps = 4;
constexpr int kMaxPerLane = 8;  // head_dim <= 256

template <typename T>
__global__ void __launch_bounds__(kWarps * 32)
paged_attention_kernel(const T* __restrict__ q, const T* __restrict__ cache, T* __restrict__ out,
                       const int32_t* __restrict__ seq_of, const int32_t* __restrict__ pos_of,
                       const int32_t* __restrict__ block_table, int hq, int hkv, int d, int q_stride, int block_size,
                       int max_blocks, float scale)
{
    __shared__ float sm_m[kWarps], sm_l[kWarps];
    __shared__ float sm_o[kWarps][256];
    const int t = blockIdx.x, h = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int seq = seq_of[t];
    const int kv_len = pos_of[t] + 1;
    const int kvh = h / (hq / hkv);
    const int per = (d + 31) / 32;
    float qv[kMaxPerLane], acc[kMaxPerLane];
    const T* qrow = q + static_cast<int64_t>(t) * q_stride + static_cast<int64_t>(h) * d;
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) {
        const int e = lane + i * 32;
        qv[i] = (i < per && e < d) ? Elem<T>::to_f(qrow[e]) * scale : 0.f;
        acc[i] = 0.f;
    }
    float m = -INFINITY, l = 0.f;
    const int64_t tok_stride = static_cast<int64_t>(2) * hkv * d;
    for (int j = warp; j < kv_len; j += kWarps) {
        const int blk = block_table[seq * max_blocks + j / block_size];
        const T* kb = cache + (static_cast<int64_t>(blk) * block_size + (j % block_size)) * tok_stride +
                      static_cast<int64_t>(kvh) * d;
        const T* vb = kb + static_cast<int64_t>(hkv) * d;
        float dot = 0.f;
#pragma unroll
        for (int i = 0; i < kMaxPerLane; ++i) {
            const int e = lane + i * 32;
            if (i < per && e < d) dot = fmaf(qv[i], Elem<T>::to_f(kb[e]), dot);
        }
        dot = warp_reduce<SumOp>(dot);
        const float nm = fmaxf(m, dot);
        const float corr = __expf(m - nm);
        const float p = __expf(dot - nm);
        l = l * corr + p;
#pragma unroll
        for (int i = 0; i < kMaxPerLane; ++i) {
            const int e = lane + i * 32;
            if (i < per && e < d) acc[i] = fmaf(p, Elem<T>::to_f(vb[e]), acc[i] * corr);
        }
        m = nm;
    }
    if (lane == 0) {
        sm_m[warp] = m;
        sm_l[warp] = l;
    }
#pragma unroll
    for (int i = 0; i < kMaxPerLane; ++i) {
        const int e = lane + i * 32;
        if (i < per && e < d) sm_o[warp][e] = acc[i];
    }
    __syncthreads();
    float gm = -INFINITY;
    for (int w = 0; w < kWarps; ++w) gm = fmaxf(gm, sm_m[w]);
    float gl = 0.f;
    for (int w = 0; w < kWarps; ++w) gl += (sm_m[w] == -INFINITY) ? 0.f : sm_l[w] * __expf(sm_m[w] - gm);
    const float inv = gl > 0.f ? 1.f / gl : 0.f;
    T* orow = out + static_cast<int64_t>(t) * hq * d + static_cast<int64_t>(h) * d;
    for (int e = threadIdx.x; e < d; e += blockDim.x) {
        float o = 0.f;
        for (int w = 0; w < kWarps; ++w)
            if (sm_m[w] != -INFINITY) o += sm_o[w][e] * __expf(sm_m[w] - gm);
        orow[e] = Elem<T>::from_f(o * inv);
    }
}


// ------------------------------------------------------------------------------------------------------------------
// Decode-optimised variant ("flash decoding" shape): one CTA per (token, KV head, KV split).
//   * GQA sharing: the REP = hq/hkv query heads that read the same KV head are processed together, so K/V bytes are
//     fetched once per KV head instead of once per query head.
//   * memory-level parallelism: every lane keeps U=4 independent 16-byte K loads and 4 V loads in flight; a warp
//     load instruction covers 32/LPK whole keys (LPK = D/8 lanes per key), i.e. 512 contiguous-row bytes.
//   * split-KV: long contexts are cut into `nsplit` ranges so small decode batches still fill 132 SMs; partial
//     (m, l, acc) triples go to a workspace and a tiny merge kernel combines them.
// The per-key dot product is reduced over only LPK lanes; the running max is shared by the whole warp so all lanes
// rescale identically.
// ------------------------------------------------------------------------------------------------------------------
template <typename T, int D, int REP>
__global__ void __launch_bounds__(128)
paged_decode_kernel(const T* __restrict__ q, const T* __restrict__ cache, T* __restrict__ out, float* __restrict__ ws_acc,
                    float* __restrict__ ws_ml, const int32_t* __restrict__ seq_of, const int32_t* __restrict__ pos_of,
                    const int32_t* __restrict__ block_table, int hq, int hkv, int q_stride, int block_size, int max_blocks,
                    float scale, int nsplit)
{
    constexpr int LPK = D / 8;     // lanes per key (8 bf16/half elements per 16-byte vector)
    constexpr int KPW = 32 / LPK;  // keys per warp-wide load
    constexpr int U = 4;
    constexpr int kW = 4;
    __shared__ float sm_m[kW][REP], sm_l[kW][REP];
    __shared__ float sm_acc[kW][REP][D];
    const int t = blockIdx.x, kvh = blockIdx.y, sp = blockIdx.z;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int sub = lane / LPK, dl = lane % LPK;
    const int kv_len = pos_of[t] + 1;
    const int seq = seq_of[t];
    const int per = (kv_len + nsplit - 1) / nsplit;
    const int k0 = sp * per;
    const int k1 = min(kv_len, k0 + per);
    float qf[REP][8], acc[REP][8], m[REP], l[REP];
#pragma unroll
    for (int r = 0; r < REP; ++r) {
        const T* qrow = q + static_cast<int64_t>(t) * q_stride + static_cast<int64_t>(kvh * REP + r) * D + dl * 8;
        Elem<T>::unpack(ld_plain(qrow), qf[r]);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            qf[r][e] *= scale;
            acc[r][e] = 0.f;
        }
        m[r] = -INFINITY;
        l[r] = 0.f;
    }
    const int32_t* bt = block_table + static_cast<int64_t>(seq) * max_blocks;
    const int64_t tok_stride = static_cast<int64_t>(2) * hkv * D;
    for (int base = k0 + warp * KPW * U; base < k1; base += kW * KPW * U) {
        Vec16 kx[U], vx[U];
        bool ok[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int j = base + u * KPW + sub;
            ok[u] = j < k1;
            const int jj = ok[u] ? j : k0;  // always a valid address
            const int blk = bt[jj / block_size];
            const T* row = cache + (static_cast<int64_t>(blk) * block_size + (jj % block_size)) * tok_stride +
                           static_cast<int64_t>(kvh) * D + dl * 8;
            kx[u] = ld_stream(row);
            vx[u] = ld_stream(row + static_cast<int64_t>(hkv) * D);
        }
        float s[REP][U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            float kf[8];
            Elem<T>::unpack(kx[u], kf);
#pragma unroll
            for (int r = 0; r < REP; ++r) {
                float d = 0.f;
#pragma unroll
                for (int e = 0; e < 8; ++e) d = fmaf(qf[r][e], kf[e], d);
#pragma unroll
                for (int o = LPK / 2; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
                s[r][u] = ok[u] ? d : -INFINITY;
            }
        }
#pragma unroll
        for (int r = 0; r < REP; ++r) {
            float mx = s[r][0];
#pragma unroll
            for (int u = 1; u < U; ++u) mx = fmaxf(mx, s[r][u]);
#pragma unroll
            for (int o = LPK; o < 32; o <<= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            const float mn = fmaxf(m[r], mx);
            const float alpha = (m[r] == -INFINITY) ? 0.f : __expf(m[r] - mn);
            m[r] = mn;
            l[r] *= alpha;
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[r][e] *= alpha;
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            float vf[8];
            Elem<T>::unpack(vx[u], vf);
#pragma unroll
            for (int r = 0; r < REP; ++r) {
                const float p = (ok[u] && m[r] != -INFINITY) ? __expf(s[r][u] - m[r]) : 0.f;
                l[r] += p;
#pragma unroll
                for (int e = 0; e < 8; ++e) acc[r][e] = fmaf(p, vf[e], acc[r][e]);
            }
        }
    }
    // lanes with the same `dl` but different `sub` saw different keys under the same running max: add them up
#pragma unroll
    for (int r = 0; r < REP; ++r) {
#pragma unroll
        for (int o = LPK; o < 32; o <<= 1) {
            l[r] += __shfl_xor_sync(0xffffffffu, l[r], o);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[r][e] += __shfl_xor_sync(0xffffffffu, acc[r][e], o);
        }
        if (lane == 0) {
            sm_m[warp][r] = m[r];
            sm_l[warp][r] = l[r];
        }
        if (sub == 0) {
#pragma unroll
            for (int e = 0; e < 8; ++e) sm_acc[warp][r][dl * 8 + e] = acc[r][e];
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < REP * D; i += blockDim.x) {
        const int r = i / D, e = i % D;
        float gm = -INFINITY;
#pragma unroll
        for (int w = 0; w < kW; ++w) gm = fmaxf(gm, sm_m[w][r]);
        float gl = 0.f, o = 0.f;
#pragma unroll
        for (int w = 0; w < kW; ++w) {
            const float f = (sm_m[w][r] == -INFINITY) ? 0.f : __expf(sm_m[w][r] - gm);
            gl = fmaf(sm_l[w][r], f, gl);
            o = fmaf(sm_acc[w][r][e], f, o);
        }
        const int h = kvh * REP + r;
        if (nsplit == 1) {
            out[static_cast<int64_t>(t) * hq * D + static_cast<int64_t>(h) * D + e] = Elem<T>::from_f(gl > 0.f ? o / gl : 0.f);
        } else {
            const int64_t slot = (static_cast<int64_t>(t) * hq + h) * nsplit + sp;
            ws_acc[slot * D + e] = o;
            if (e == 0) {
                ws_ml[slot * 2] = gm;
                ws_ml[slot * 2 + 1] = gl;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Tensor-core decode attention.  The CUDA-core kernel above is issue-bound (ncu: 65 % SM throughput at 47 % of copy
// bandwidth): per key it spends ~55 warp instructions on FMAs, shuffles and exps.  Here one warp processes 16 keys per
// iteration with mma.sync.m16n8k16: rows = the (<= 8) query heads of one GQA group, so K and V are still read exactly once
// per group.  No shared-memory staging and no ldmatrix: the MMA's k order is arbitrary as long as A and B agree, so
//   * S = Q K^T: lane (g, t) loads 16-byte pieces of key g's row at d = 32 i + 8 t; piece element pairs (0,1),(2,3) /
//     (4,5),(6,7) are the B fragments of two k-steps, the matching Q fragment is the same 16 bytes of the query row;
//   * O = P V: the S accumulators of two 8-key tiles ARE the A fragment (keys 2t,2t+1 | 2t+8,2t+9); lane (g, t) loads
//     16 bytes at d = 64 G + 8 g of those four keys' V rows and packs (V[2t][d], V[2t+1][d]) with one byte-permute, i.e.
//     output column g of n-tile j is d = 64 G + 8 g + j (undone when the result is written).
// (mma.sync on purpose: M is 1..8 useful rows - a wgmma tile would be > 90 % padding - and the kernel is bound by the
// KV stream.)
// ---------------------------------------------------------------------------------------------------------------------
template <typename T>
struct MmaT;
template <>
struct MmaT<__nv_bfloat16> {
    static __device__ __forceinline__ void mma(float& c0, float& c1, float& z0, float& z1, uint32_t a0, uint32_t a2, uint32_t b0,
                                               uint32_t b1)
    {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(c0), "+f"(c1), "+f"(z0), "+f"(z1)
                     : "r"(a0), "r"(0u), "r"(a2), "r"(0u), "r"(b0), "r"(b1));
    }
    static __device__ __forceinline__ uint32_t pack(float lo, float hi)
    {
        __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
        return *reinterpret_cast<uint32_t*>(&v);
    }
};
template <>
struct MmaT<__half> {
    static __device__ __forceinline__ void mma(float& c0, float& c1, float& z0, float& z1, uint32_t a0, uint32_t a2, uint32_t b0,
                                               uint32_t b1)
    {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(c0), "+f"(c1), "+f"(z0), "+f"(z1)
                     : "r"(a0), "r"(0u), "r"(a2), "r"(0u), "r"(b0), "r"(b1));
    }
    static __device__ __forceinline__ uint32_t pack(float lo, float hi)
    {
        __half2 v = __floats2half2_rn(lo, hi);
        return *reinterpret_cast<uint32_t*>(&v);
    }
};

template <typename T, int D>
__global__ void __launch_bounds__(128)
paged_decode_mma_kernel(const T* __restrict__ q, const T* __restrict__ cache, T* __restrict__ out, float* __restrict__ ws_acc,
                        float* __restrict__ ws_ml, const int32_t* __restrict__ seq_of, const int32_t* __restrict__ pos_of,
                        const int32_t* __restrict__ block_table, int hq, int hkv, int rep, int q_stride, int block_size,
                        int max_blocks, float scale, int nsplit)
{
    constexpr int kW = 4;
    constexpr int NC = D / 32;  // 16-byte pieces of a K row per lane
    constexpr int NG = D / 64;  // 64-wide d groups of a V row
    constexpr int NO = D / 8;   // output n-tiles
    __shared__ float sm_m[kW][8], sm_l[kW][8];
    __shared__ float sm_acc[kW][8][D];
    const int t = blockIdx.x, kvh = blockIdx.y, sp = blockIdx.z;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, tq = lane & 3;
    const int kv_len = pos_of[t] + 1;
    const int seq = seq_of[t];
    const int per = (((kv_len + nsplit - 1) / nsplit) + 15) & ~15;  // splits start on 16-key boundaries
    const int k0 = sp * per;
    const int k1 = min(kv_len, k0 + per);
    const int32_t* bt = block_table + static_cast<int64_t>(seq) * max_blocks;
    const int64_t tok_stride = static_cast<int64_t>(2) * hkv * D;
    const T* kbase = cache + static_cast<int64_t>(kvh) * D;
    const T* vbase = kbase + static_cast<int64_t>(hkv) * D;

    // query fragments as stored, zero rows for g >= rep.  The softmax scale is applied to the fp32 scores after the MMA:
    // q * scale rounded back to bf16 / fp16 would add a relative error of up to 2^-9 / 2^-12 to every logit.
    Vec16 qv[NC];
#pragma unroll
    for (int i = 0; i < NC; ++i) {
        if (g < rep) {
            qv[i] = ld_plain(q + static_cast<int64_t>(t) * q_stride + static_cast<int64_t>(kvh * rep + g) * D + 32 * i + 8 * tq);
        } else {
#pragma unroll
            for (int w = 0; w < 4; ++w) qv[i].w[w] = 0u;
        }
    }
    float o[NO][2];
#pragma unroll
    for (int n = 0; n < NO; ++n) o[n][0] = o[n][1] = 0.f;
    float z0 = 0.f, z1 = 0.f;  // rows 8..15 of every accumulator: A rows 8..15 are zero, so these stay zero
    float m = -INFINITY, l = 0.f;

    auto row_of = [&](int key) -> int64_t {
        const int kk = key < k1 ? key : k0;  // always a valid address; masked below
        return (static_cast<int64_t>(bt[kk / block_size]) * block_size + (kk % block_size)) * tok_stride;
    };

    // Register double buffering: the loads of the NEXT 16-key block are in flight while the current one is being multiplied,
    // so every warp keeps ~8 KB outstanding at all times (2 CTAs x 4 warps per SM -> ~64 KB per SM, enough for HBM speed).
    auto load_block = [&](int kb, Vec16 (&kx)[2][NC], Vec16 (&vx)[4][NG]) {
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
            const T* row = kbase + row_of(kb + 8 * nt + g) + 8 * tq;
#pragma unroll
            for (int i = 0; i < NC; ++i) kx[nt][i] = ld_stream(row + 32 * i);
        }
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            const int key = kb + 2 * tq + (kk & 1) + 8 * (kk >> 1);
            const T* row = vbase + row_of(key) + 8 * g;
#pragma unroll
            for (int G = 0; G < NG; ++G) vx[kk][G] = ld_stream(row + 64 * G);
        }
    };
    auto compute_block = [&](int kb, Vec16 (&kx)[2][NC], Vec16 (&vx)[4][NG]) {
        // ---- S = Q K^T for 2 x 8 keys
        float s[2][2];
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
            s[nt][0] = s[nt][1] = 0.f;
#pragma unroll
            for (int i = 0; i < NC; ++i) {
                MmaT<T>::mma(s[nt][0], s[nt][1], z0, z1, qv[i].w[0], qv[i].w[1], kx[nt][i].w[0], kx[nt][i].w[1]);
                MmaT<T>::mma(s[nt][0], s[nt][1], z0, z1, qv[i].w[2], qv[i].w[3], kx[nt][i].w[2], kx[nt][i].w[3]);
            }
            const int key = kb + 8 * nt + 2 * tq;
            s[nt][0] = key < k1 ? s[nt][0] * scale : -INFINITY;
            s[nt][1] = key + 1 < k1 ? s[nt][1] * scale : -INFINITY;
        }
        // ---- online softmax for row g (values spread over the 4 t-lanes)
        float mx = fmaxf(fmaxf(s[0][0], s[0][1]), fmaxf(s[1][0], s[1][1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float mn = fmaxf(m, mx);  // finite: every 16-key block this loop visits has at least one valid key
        const float alpha = (m == -INFINITY) ? 0.f : __expf(m - mn);
        m = mn;
        float p[2][2];
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
            p[nt][0] = __expf(s[nt][0] - mn);
            p[nt][1] = __expf(s[nt][1] - mn);
        }
        l = l * alpha + (p[0][0] + p[0][1] + p[1][0] + p[1][1]);
#pragma unroll
        for (int n = 0; n < NO; ++n) {
            o[n][0] *= alpha;
            o[n][1] *= alpha;
        }
        const uint32_t pa0 = MmaT<T>::pack(p[0][0], p[0][1]);  // keys 2t, 2t+1
        const uint32_t pa2 = MmaT<T>::pack(p[1][0], p[1][1]);  // keys 2t+8, 2t+9
        // ---- O += P V
#pragma unroll
        for (int G = 0; G < NG; ++G) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const uint32_t sel = (j & 1) ? 0x7632u : 0x5410u;
                const uint32_t b0 = __byte_perm(vx[0][G].w[j >> 1], vx[1][G].w[j >> 1], sel);
                const uint32_t b1 = __byte_perm(vx[2][G].w[j >> 1], vx[3][G].w[j >> 1], sel);
                MmaT<T>::mma(o[G * 8 + j][0], o[G * 8 + j][1], z0, z1, pa0, pa2, b0, b1);
            }
        }
    };
    {
        Vec16 kA[2][NC], vA[4][NG], kB[2][NC], vB[4][NG];
        int kb = k0 + warp * 16;
        if (kb < k1) load_block(kb, kA, vA);
        while (kb < k1) {
            int nb = kb + kW * 16;
            if (nb < k1) load_block(nb, kB, vB);
            compute_block(kb, kA, vA);
            kb = nb;
            if (kb >= k1) break;
            nb = kb + kW * 16;
            if (nb < k1) load_block(nb, kA, vA);
            compute_block(kb, kB, vB);
            kb = nb;
        }
    }
    // ---- per-warp result -> shared: row g, column (2t, 2t+1) of n-tile G*8+j is d = 64 G + 8 (2t | 2t+1) + j
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    if (g < rep) {
        if (tq == 0) {
            sm_m[warp][g] = m;
            sm_l[warp][g] = l;
        }
#pragma unroll
        for (int G = 0; G < NG; ++G)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                sm_acc[warp][g][64 * G + 8 * (2 * tq) + j] = o[G * 8 + j][0];
                sm_acc[warp][g][64 * G + 8 * (2 * tq + 1) + j] = o[G * 8 + j][1];
            }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < rep * D; i += blockDim.x) {
        const int r = i / D, e = i % D;
        float gm = -INFINITY;
#pragma unroll
        for (int w = 0; w < kW; ++w) gm = fmaxf(gm, sm_m[w][r]);
        float gl = 0.f, acc = 0.f;
#pragma unroll
        for (int w = 0; w < kW; ++w) {
            const float f = (sm_m[w][r] == -INFINITY) ? 0.f : __expf(sm_m[w][r] - gm);
            gl = fmaf(sm_l[w][r], f, gl);
            acc = fmaf(sm_acc[w][r][e], f, acc);
        }
        const int h = kvh * rep + r;
        if (nsplit == 1) {
            out[static_cast<int64_t>(t) * hq * D + static_cast<int64_t>(h) * D + e] = Elem<T>::from_f(gl > 0.f ? acc / gl : 0.f);
        } else {
            const int64_t slot = (static_cast<int64_t>(t) * hq + h) * nsplit + sp;
            ws_acc[slot * D + e] = acc;
            if (e == 0) {
                ws_ml[slot * 2] = gm;
                ws_ml[slot * 2 + 1] = gl;
            }
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(128)
paged_decode_merge_kernel(const float* __restrict__ ws_acc, const float* __restrict__ ws_ml, T* __restrict__ out, int hq,
                          int d, int nsplit)
{
    const int t = blockIdx.x, h = blockIdx.y;
    const int64_t base = (static_cast<int64_t>(t) * hq + h) * nsplit;
    float gm = -INFINITY;
    for (int s = 0; s < nsplit; ++s) gm = fmaxf(gm, ws_ml[(base + s) * 2]);
    float gl = 0.f;
    for (int s = 0; s < nsplit; ++s) {
        const float mm = ws_ml[(base + s) * 2];
        gl += (mm == -INFINITY) ? 0.f : ws_ml[(base + s) * 2 + 1] * __expf(mm - gm);
    }
    const float inv = gl > 0.f ? 1.f / gl : 0.f;
    for (int e = threadIdx.x; e < d; e += blockDim.x) {
        float o = 0.f;
        for (int s = 0; s < nsplit; ++s) {
            const float mm = ws_ml[(base + s) * 2];
            if (mm != -INFINITY) o = fmaf(ws_acc[(base + s) * d + e], __expf(mm - gm), o);
        }
        out[static_cast<int64_t>(t) * hq * d + static_cast<int64_t>(h) * d + e] = Elem<T>::from_f(o * inv);
    }
}

}  // namespace pattn
}  // namespace dsb

using namespace dsb;

// q: [tokens, q_stride] with head h at offset h*d (a packed qkv buffer works with q_stride = (hq+2hkv)*d).
DSB_EXPORT int dsb_paged_attention(const void* q, const void* cache, void* out, const int32_t* seq_of,
                                   const int32_t* pos_of, const int32_t* block_table, int tokens, int hq, int hkv, int d,
                                   int q_stride, int block_size, int max_blocks, float scale, int dtype,
                                   cudaStream_t stream)
{
    if (tokens <= 0) return 0;
    if (d > 256 || hq % hkv) return -2;
    dim3 grid(tokens, hq);
    if (dtype == kBF16)
        pattn::paged_attention_kernel<__nv_bfloat16><<<grid, pattn::kWarps * 32, 0, stream>>>(
            (const __nv_bfloat16*)q, (const __nv_bfloat16*)cache, (__nv_bfloat16*)out, seq_of, pos_of, block_table, hq, hkv,
            d, q_stride, block_size, max_blocks, scale);
    else if (dtype == kF16)
        pattn::paged_attention_kernel<__half><<<grid, pattn::kWarps * 32, 0, stream>>>(
            (const __half*)q, (const __half*)cache, (__half*)out, seq_of, pos_of, block_table, hq, hkv, d, q_stride,
            block_size, max_blocks, scale);
    else if (dtype == kF32)
        pattn::paged_attention_kernel<float><<<grid, pattn::kWarps * 32, 0, stream>>>(
            (const float*)q, (const float*)cache, (float*)out, seq_of, pos_of, block_table, hq, hkv, d, q_stride,
            block_size, max_blocks, scale);
    else
        return -1;
    DSB_CHECK_LAUNCH();
    return 0;
}


// Decode-optimised entry: eligible when dtype is bf16/fp16, d in {64,128,256} and hq/hkv in {1,2,4,8}.
// ws_acc: float [tokens*hq*nsplit*d], ws_ml: float [tokens*hq*nsplit*2] (unused when nsplit == 1).
// Returns -3 when the shape is not eligible (caller falls back to dsb_paged_attention).
#define DSB_PD_LAUNCH(TT, DD, RR)                                                                                        \
    pattn::paged_decode_kernel<TT, DD, RR><<<grid, 128, 0, stream>>>((const TT*)q, (const TT*)cache, (TT*)out, ws_acc,   \
                                                                     ws_ml, seq_of, pos_of, block_table, hq, hkv, q_stride, \
                                                                     block_size, max_blocks, scale, nsplit)
#define DSB_PD_REP(TT, DD)                          \
    switch (rep) {                                   \
        case 1: DSB_PD_LAUNCH(TT, DD, 1); break;     \
        case 2: DSB_PD_LAUNCH(TT, DD, 2); break;     \
        case 4: DSB_PD_LAUNCH(TT, DD, 4); break;     \
        case 8: DSB_PD_LAUNCH(TT, DD, 8); break;     \
        default: return -3;                          \
    }
#define DSB_PD_D(TT)                                 \
    switch (d) {                                     \
        case 64: DSB_PD_REP(TT, 64) break;           \
        case 128: DSB_PD_REP(TT, 128) break;         \
        case 256: DSB_PD_REP(TT, 256) break;         \
        default: return -3;                          \
    }

DSB_EXPORT int dsb_paged_decode(const void* q, const void* cache, void* out, float* ws_acc, float* ws_ml,
                                const int32_t* seq_of, const int32_t* pos_of, const int32_t* block_table, int tokens, int hq,
                                int hkv, int d, int q_stride, int block_size, int max_blocks, float scale, int nsplit,
                                int dtype, cudaStream_t stream)
{
    if (tokens <= 0) return 0;
    if (hq % hkv || nsplit < 1 || q_stride % 8) return -3;
    const int rep = hq / hkv;
    if (dtype != kBF16 && dtype != kF16) return -3;
    dim3 grid(tokens, hkv, nsplit);
    static const bool use_mma = [] {
        const char* e = getenv("DSB200_PAGED_DECODE_MMA");
        return !(e && e[0] == '0');
    }();
    if (use_mma && rep <= 8 && (d == 64 || d == 128)) {
#define DSB_PDM(TT, DD)                                                                                                    \
    pattn::paged_decode_mma_kernel<TT, DD><<<grid, 128, 0, stream>>>((const TT*)q, (const TT*)cache, (TT*)out, ws_acc, ws_ml, \
                                                                     seq_of, pos_of, block_table, hq, hkv, rep, q_stride,   \
                                                                     block_size, max_blocks, scale, nsplit)
        if (dtype == kBF16) {
            if (d == 64) DSB_PDM(__nv_bfloat16, 64); else DSB_PDM(__nv_bfloat16, 128);
        } else {
            if (d == 64) DSB_PDM(__half, 64); else DSB_PDM(__half, 128);
        }
#undef DSB_PDM
    } else if (dtype == kBF16) {
        DSB_PD_D(__nv_bfloat16)
    } else {
        DSB_PD_D(__half)
    }
    if (nsplit > 1) {
        dim3 g2(tokens, hq);
        if (dtype == kBF16)
            pattn::paged_decode_merge_kernel<__nv_bfloat16><<<g2, 128, 0, stream>>>(ws_acc, ws_ml, (__nv_bfloat16*)out, hq, d,
                                                                                  nsplit);
        else
            pattn::paged_decode_merge_kernel<__half><<<g2, 128, 0, stream>>>(ws_acc, ws_ml, (__half*)out, hq, d, nsplit);
    }
    DSB_CHECK_LAUNCH();
    return 0;
}
