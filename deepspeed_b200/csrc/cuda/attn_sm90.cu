// Training attention for sm_90a: causal / full softmax(Q K^T / sqrt(d)) V with grouped-query heads, head dim 64 or 128
// (the template parameter kD of every kernel), bf16.
//
// Forward -- one CTA per (128 query rows, query head, batch):
//   warp 8      TMA producer: Q once, then a 3-stage ring of K and V tiles (64 keys x kD dims: 16 KiB at kD = 128, 8 KiB
//               at kD = 64)
//   warps 0-7   two consumer warpgroups, 64 query rows each: S = Q K_j^T with wgmma (both operands in shared memory,
//               accumulators in registers), online softmax in the log2 domain (ex2.approx) on the accumulator fragments,
//               then O += P V_j with P taken straight from registers as the A operand (the m64n64 accumulator layout is the
//               m64k16 A-fragment layout) and V_j read MN-major from shared memory; at the end O / l -> bf16 -> global and
//               the log-sum-exp for backward.
//   S, P never touch shared or global memory; K/V tiles are shared by the query heads of a GQA group through L2.
// Backward recomputes S / P per (query block, key block) pair from Q, K and the saved LSE with the same tile machinery
// and produces dQ, dK, dV.
//
// Reference role: the reference has no training attention kernel of its own for HF-style models (it calls flash-attn,
// sequence/fpdt_layer.py:235); its BERT-era fused layer is csrc/transformer/softmax_kernels.cu + cuBLAS strided batched GEMMs.
#include "dsb_tc.cuh"

namespace dsb {
namespace attn {
using namespace dsb::tc;

constexpr int BQ = 128, BS = 64;
constexpr int kThreads = 288;                            // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int kProducer = 256;                           // thread index of the producer
constexpr uint32_t BOX = BS * 64 * 2;                    // 8 KiB TMA box [64 x 64] bf16 (one 128-byte swizzle span per row)
template <int kD>
constexpr uint32_t kTile = BS * kD * 2;                  // [64 x kD] bf16 tile of one head = kD / 64 boxes
constexpr float kNegInf = -__builtin_huge_valf();

// Operand descriptors of a [64 x kD] tile at `t`:
//   K-major over the kD columns (S = Q K^T: Q as A, K as B): 16-column step kk in 0..kD/16-1, the second box from kk = 4
__device__ __forceinline__ uint64_t desc_k(uint32_t t, int kk) { return desc_kmajor_sw128(t + (kk >> 2) * BOX + (kk & 3) * 32); }
//   MN-major, rows as the reduction dimension, the kD columns as N (O = P V: V as B): 16-row step kk in 0..3.  The LBO
//   (the distance to the second 64-wide atom) is unused at kD = 64.
__device__ __forceinline__ uint64_t desc_mn(uint32_t t, int kk) { return desc_mnmajor_sw128(t + kk * 2048, BOX); }

template <int kD>
__device__ __forceinline__ void load_tile(uint32_t dst, const CUtensorMap* map, uint32_t bar, int col, int row)
{
    static_assert(kD == 64 || kD == 128, "head dim 64 or 128");
    tma_load_2d(dst, map, bar, col, row);
    if constexpr (kD == 128) tma_load_2d(dst + BOX, map, bar, col + 64, row);
}

// acc = A_tile(64 rows) x B_tile(64 rows)^T over the kD columns: m64n64, kD / 16 steps
template <int kD>
__device__ __forceinline__ void mma_rows_x_rows(float* acc, uint32_t a, uint32_t b)
{
#pragma unroll
    for (int kk = 0; kk < kD / 16; ++kk) wgmma_m64n64k16_ss<0, 0>(acc, desc_k(a, kk), desc_k(b, kk), kk > 0 ? 1 : 0);
}
// acc[64 x kD] += P[64 x 64] (register fragments of an m64n64 fp32 block) x tile[64 rows x kD]
template <int kD>
__device__ __forceinline__ void mma_regs_x_tile(float* acc, const uint32_t (*frag)[4], uint32_t t)
{
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        if constexpr (kD == 128)
            wgmma_m64n128k16_rs<1>(acc, frag[kk], desc_mn(t, kk), 1);
        else
            wgmma_m64n64k16_rs<1>(acc, frag[kk], desc_mn(t, kk), 1);
    }
}
// m64n64 fp32 accumulator -> bf16 A fragments of four k16 steps
__device__ __forceinline__ void to_frags(const float* s, uint32_t (*f)[4])
{
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        f[kk][0] = pack_bf16(s[8 * kk + 0], s[8 * kk + 1]);
        f[kk][1] = pack_bf16(s[8 * kk + 2], s[8 * kk + 3]);
        f[kk][2] = pack_bf16(s[8 * kk + 4], s[8 * kk + 5]);
        f[kk][3] = pack_bf16(s[8 * kk + 6], s[8 * kk + 7]);
    }
}
__device__ __forceinline__ float quad_max(float v)
{
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v)
{
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
// store a 64 x kD fp32 accumulator (times `mul`) as bf16 rows `row0 + r` (r < rows) of a [*, ld] matrix at column col0
template <int kD>
__device__ __forceinline__ void store_acc(const float* acc, __nv_bfloat16* base, int64_t ld, int row_local, int rows, int col0,
                                          int c_in, float mul0, float mul1)
{
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int r = row_local + 8 * i;
        if (r >= rows) continue;
        const float m = i ? mul1 : mul0;
        __nv_bfloat16* dst = base + static_cast<int64_t>(r) * ld + col0 + c_in;
#pragma unroll
        for (int j = 0; j < kD / 8; ++j)
            *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16(acc[4 * j + 2 * i] * m, acc[4 * j + 2 * i + 1] * m);
    }
}

struct FwdParams {
    __nv_bfloat16* o;   // [B*S, ld_o], head h at columns [h*D, (h+1)*D)
    float* lse;         // [B, Hq, S] natural-log sum-exp of the scaled scores (varlen: [Hq, T] by absolute token row)
    int ld_o;
    int S, Hq, Hkv;
    float scale_log2;   // softmax scale * log2(e)
    int causal;
    const int* cu;      // varlen only: document offsets [n_docs + 1] into the T token rows
    int T;              // varlen only: token rows
    int window;         // sliding window only: row i sees keys i - window < j <= i (1 <= window <= S)
};

// Packed sequences (varlen): blockIdx.z is a document, not a batch row.  Returns false for a CTA with nothing to do -- its
// first row is past the document's end, or the offsets are malformed -- so the whole CTA exits before any barrier exists.
template <bool kVarlen>
__device__ __forceinline__ bool doc_rows(const int* cu, int T, int S, int b, int first, int& row_base, int& len)
{
    if constexpr (kVarlen) {
        const int start = cu[b], end = cu[b + 1];
        if (start < 0 || start > end || end > T || first >= end - start) return false;
        row_base = start;
        len = end - start;
    } else {
        row_base = b * S;
        len = S;
    }
    return true;
}

// Sliding window: the first 64-key block a CTA whose first query row is q0 can see.  The producer and the consumers both
// start there and count ring stages and phases from it.
template <bool kWindow>
__device__ __forceinline__ int first_key_block(int q0, int window)
{
    return kWindow ? max(0, q0 - window + 1) / BS : 0;
}

template <int kD>
struct kf {  // forward shared-memory plan
    static constexpr int KV_STAGES = 3;
    static constexpr uint32_t TILE = kTile<kD>;
    static constexpr uint32_t SM_Q = 0;                         // 2 tiles (one per consumer warpgroup)
    static constexpr uint32_t SM_KV = SM_Q + 2 * TILE;          // KV_STAGES x (K tile, V tile)
    static constexpr uint32_t SM_BAR = SM_KV + KV_STAGES * 2 * TILE;
    static constexpr uint32_t SM_TOTAL = SM_BAR + 256 + 1024;
};

template <int kD, bool kVarlen, bool kWindow>
__global__ void __launch_bounds__(kThreads, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                const __grid_constant__ CUtensorMap map_v, const FwdParams p)
{
    using Plan = kf<kD>;
    constexpr int KV_STAGES = Plan::KV_STAGES;
    constexpr uint32_t TILE = Plan::TILE, SM_Q = Plan::SM_Q, SM_KV = Plan::SM_KV, SM_BAR = Plan::SM_BAR;
    const int q0 = blockIdx.x * BQ, h = blockIdx.y, b = blockIdx.z;
    int row_base, len;  // first token row and length of this sequence
    if (!doc_rows<kVarlen>(p.cu, p.T, p.S, b, q0, row_base, len)) return;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const uint32_t sbase = smem_u32(smem);
    const uint32_t q_full = sbase + SM_BAR;
    auto kv_full = [&](int s) { return sbase + SM_BAR + 8 * (1 + s); };
    auto kv_empty = [&](int s) { return sbase + SM_BAR + 8 * (1 + KV_STAGES + s); };

    const int kvh = h / (p.Hq / p.Hkv);
    const int n_blocks = (len + BS - 1) / BS;
    const int n_kv = p.causal ? min(n_blocks, (q0 + BQ) / BS) : n_blocks;
    const int j0 = first_key_block<kWindow>(q0, p.window);

    if (threadIdx.x == kProducer) {
        mbar_init(q_full, 1);
        for (int s = 0; s < KV_STAGES; ++s) {
            mbar_init(kv_full(s), 1);
            mbar_init(kv_empty(s), 8);  // one arrival per consumer warp
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (threadIdx.x >= kProducer) {
        if (threadIdx.x == kProducer) {
            prefetch_map(&map_q);
            prefetch_map(&map_k);
            prefetch_map(&map_v);
            mbar_expect_tx(q_full, 2 * TILE);
            load_tile<kD>(sbase + SM_Q, &map_q, q_full, h * kD, row_base + q0);
            load_tile<kD>(sbase + SM_Q + TILE, &map_q, q_full, h * kD, row_base + q0 + BS);
            for (int j = j0; j < n_kv; ++j) {
                const int s = (j - j0) % KV_STAGES;
                mbar_wait(kv_empty(s), (((j - j0) / KV_STAGES) & 1) ^ 1);
                mbar_expect_tx(kv_full(s), 2 * TILE);
                const uint32_t dst = sbase + SM_KV + s * 2 * TILE;
                load_tile<kD>(dst, &map_k, kv_full(s), kvh * kD, row_base + j * BS);
                load_tile<kD>(dst + TILE, &map_v, kv_full(s), kvh * kD, row_base + j * BS);
            }
        }
        return;
    }

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = warp >> 2;
    const int qr0 = q0 + wg * BS;                              // first query row of this warpgroup
    const int r_loc = 16 * (warp & 3) + (lane >> 2);          // this thread's rows: qr0 + r_loc (+8)
    const int c_in = 2 * (lane & 3);
    const uint32_t sq = sbase + SM_Q + wg * TILE;
    float o[kD / 2];
#pragma unroll
    for (int i = 0; i < kD / 2; ++i) o[i] = 0.f;
    float m_run[2] = {kNegInf, kNegInf}, l_run[2] = {0.f, 0.f};
    mbar_wait(q_full, 0);

    for (int j = j0; j < n_kv; ++j) {
        const int s = (j - j0) % KV_STAGES;
        mbar_wait(kv_full(s), ((j - j0) / KV_STAGES) & 1);
        // a block entirely above the diagonal, or entirely before the window of every row here, contributes nothing
        if (!(p.causal && j * BS > qr0 + BS - 1) && !(kWindow && j * BS + BS - 1 < qr0 - p.window + 1)) {
            const uint32_t sk = sbase + SM_KV + s * 2 * TILE, sv = sk + TILE;
            float sc[32];
            wgmma_fence();
            mma_rows_x_rows<kD>(sc, sq, sk);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs<32>(sc);
            float mx[2] = {kNegInf, kNegInf};
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int key = j * BS + 8 * jj + c_in + e;
                        const int row = qr0 + r_loc + 8 * i;
                        float x = sc[4 * jj + 2 * i + e] * p.scale_log2;
                        if (key >= len || (p.causal && key > row) || (kWindow && key <= row - p.window)) x = kNegInf;
                        sc[4 * jj + 2 * i + e] = x;
                        mx[i] = fmaxf(mx[i], x);
                    }
            float alpha[2], m_use[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const float m_new = fmaxf(m_run[i], quad_max(mx[i]));
                m_use[i] = m_new == kNegInf ? 0.f : m_new;  // a row with nothing visible yet keeps zero state
                alpha[i] = ex2(m_run[i] - m_use[i]);        // 0 on the first block (m_run = -inf)
                m_run[i] = m_new;
                l_run[i] *= alpha[i];
            }
#pragma unroll
            for (int jj = 0; jj < kD / 8; ++jj)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    o[4 * jj + 2 * i] *= alpha[i];
                    o[4 * jj + 2 * i + 1] *= alpha[i];
                }
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float pe = ex2(sc[4 * jj + 2 * i + e] - m_use[i]);
                        sc[4 * jj + 2 * i + e] = pe;
                        l_run[i] += pe;
                    }
            uint32_t pf[4][4];
            to_frags(sc, pf);
            wgmma_fence();
            mma_regs_x_tile<kD>(o, pf, sv);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs<kD / 2>(o);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(kv_empty(s));
    }

    // ---- epilogue: O / l -> bf16 -> global, LSE ----------------------------------------------------------------------------
    float inv[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        l_run[i] = quad_sum(l_run[i]);
        inv[i] = l_run[i] > 0.f ? 1.f / l_run[i] : 0.f;
    }
    const int rows = len - qr0;  // rows of this warpgroup inside the sequence
    store_acc<kD>(o, p.o + static_cast<int64_t>(row_base + qr0) * p.ld_o, p.ld_o, r_loc, rows < BS ? rows : BS, h * kD, c_in,
                  inv[0], inv[1]);
    if (p.lse != nullptr && (lane & 3) == 0) {
        float* lse = kVarlen ? p.lse + static_cast<int64_t>(h) * p.T + row_base
                             : p.lse + (static_cast<int64_t>(b) * p.Hq + h) * p.S;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int row = qr0 + r_loc + 8 * i;
            if (row < len) lse[row] = (m_run[i] + log2f(l_run[i])) * 0.6931471805599453f;
        }
    }
}

// =============================================================================================================================
// Backward.  Two kernels, no atomics, every accumulator in registers:
//   (A) dK / dV: one CTA per (128 keys, KV head, batch), 64 keys per consumer warpgroup, keeps K_j, V_j resident and streams
//       (query head of the GQA group) x (64-row query block): dP^T = V dO^T and S^T = K Q^T (M = keys), P^T = 2^(S^T*c -
//       lse[q]) and dS^T = P^T (dP^T - delta[q]) * scale on the fragments, then dV += P^T dO and dK += dS^T Q with P^T / dS^T
//       as register A operands; dK / dV accumulate over ALL query heads of the group -- GQA needs no reduction pass.
//   (B) dQ: one CTA per (128 queries, query head, batch) keeps Q, dO resident and streams 64-key blocks:
//       S = Q K^T, dP = dO V^T, dS on the fragments, dQ += dS K.
// S / P / dS are recomputed on chip; only Q, K, V, O, dO, LSE are read.  `delta = rowsum(dO * O)` and `lse * log2(e)` come
// from a small pre-pass.
// =============================================================================================================================
struct BwdParams {
    __nv_bfloat16 *dq, *dk, *dv;  // outputs, 2-D [B*S, ld]: head h at columns [h*D, +D)
    int ld_dq, ld_dk, ld_dv;
    const float* lse2;   // [B, Hq, S]  log-sum-exp * log2(e)       (varlen: [Hq, T])
    const float* delta;  // [B, Hq, S]  rowsum(dO * O)              (varlen: [Hq, T])
    int S, Hq, Hkv;
    float scale, scale_log2;
    int causal;
    const int* cu;       // varlen only, as in FwdParams
    int T;
    int window;          // sliding window only, as in FwdParams
};

// Per-row statistics (lse2 / delta) of query head h of this sequence, indexed by the row inside the sequence.
template <bool kVarlen>
__device__ __forceinline__ int64_t stat_base(const BwdParams& p, int b, int h, int row_base)
{
    return kVarlen ? static_cast<int64_t>(h) * p.T + row_base : (static_cast<int64_t>(b) * p.Hq + h) * p.S;
}

// delta[b,h,s] = sum_d dO * O ; lse2 = lse * log2(e).  One warp per (token, head) row of kD elements, 4 per lane: at
// kD = 64 lanes 16-31 add zeros, so delta is summed in the order the kD = 128 kernel uses on a head padded with zero
// columns, and the backward of a d = 64 head is bit-equal to the d = 128 backward of the zero-padded head.
// The varlen [Hq, T] layout is this kernel's B = 1, S = T.
template <int kD>
__global__ void __launch_bounds__(256)
attn_bwd_prep_kernel(const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ d_o, const float* __restrict__ lse,
                     float* __restrict__ delta, float* __restrict__ lse2, int B, int S, int Hq, int ld_o, int ld_do)
{
    const int64_t w = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const int64_t rows = static_cast<int64_t>(B) * S * Hq;
    if (w >= rows) return;
    const int h = static_cast<int>(w % Hq);
    const int64_t t = w / Hq;  // token row b*S + s
    float acc = 0.f;
    if (kD == 128 || lane < kD / 4) {
        const __nv_bfloat16* po = o + t * ld_o + h * kD + lane * 4;
        const __nv_bfloat16* pd = d_o + t * ld_do + h * kD + lane * 4;
        const uint2 a = *reinterpret_cast<const uint2*>(po);
        const uint2 g = *reinterpret_cast<const uint2*>(pd);
        acc = fmaf(__uint_as_float(a.x << 16), __uint_as_float(g.x << 16), acc);
        acc = fmaf(__uint_as_float(a.x & 0xffff0000u), __uint_as_float(g.x & 0xffff0000u), acc);
        acc = fmaf(__uint_as_float(a.y << 16), __uint_as_float(g.y << 16), acc);
        acc = fmaf(__uint_as_float(a.y & 0xffff0000u), __uint_as_float(g.y & 0xffff0000u), acc);
    }
    acc = warp_reduce<SumOp>(acc);
    if (lane == 0) {
        const int b = static_cast<int>(t / S), s_ = static_cast<int>(t % S);
        const int64_t idx = (static_cast<int64_t>(b) * Hq + h) * S + s_;
        delta[idx] = acc;
        lse2[idx] = lse[idx] * 1.4426950408889634f;
    }
}

template <int kD>
struct kb {  // shared-memory plan of both backward kernels: 4 resident tiles + 2 stages x 2 streamed tiles
    static constexpr int STAGES = 2;
    static constexpr uint32_t TILE = kTile<kD>;
    static constexpr uint32_t SM_RES = 0;                       // [X_wg0, X_wg1, Y_wg0, Y_wg1]
    static constexpr uint32_t SM_STR = SM_RES + 4 * TILE;       // STAGES x (X tile, Y tile)
    static constexpr uint32_t SM_BAR = SM_STR + STAGES * 2 * TILE;
    static constexpr uint32_t SM_TOTAL = SM_BAR + 256 + 1024;
};

// ---- (A) dK, dV ---------------------------------------------------------------------------------------------------------------
// dK and dV both live in registers (kD fp32 per thread), so at kD = 128, at the 168 registers a 288-thread CTA can launch
// with, the compiler spills a little and serialises the wgmma issue of this kernel.
// Varlen: the query blocks cover ceil(len / 64) blocks; queries past `len` (the next document's rows, or TMA zero fill) get
// P = 0 and dS = 0 explicitly -- the causal mask does not remove them.  Key rows past `len` are computed and never stored.
// Sliding window: the query blocks stop after the last query that sees the CTA's last key (k0 + 127 + window - 1).
template <int kD, bool kVarlen, bool kWindow>
__global__ void __launch_bounds__(kThreads, 1)
attn_bwd_dkdv_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                     const __grid_constant__ CUtensorMap map_v, const __grid_constant__ CUtensorMap map_do, const BwdParams p)
{
    using Plan = kb<kD>;
    constexpr int STAGES = Plan::STAGES;
    constexpr uint32_t TILE = Plan::TILE, SM_RES = Plan::SM_RES, SM_STR = Plan::SM_STR, SM_BAR = Plan::SM_BAR;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const uint32_t sbase = smem_u32(smem);
    const uint32_t res_full = sbase + SM_BAR;
    auto full = [&](int s) { return sbase + SM_BAR + 8 * (1 + s); };
    auto empty = [&](int s) { return sbase + SM_BAR + 8 * (1 + STAGES + s); };

    const int k0 = blockIdx.x * BQ, kvh = blockIdx.y, b = blockIdx.z;
    const int rep = p.Hq / p.Hkv;
    int row_base, len;
    if (!doc_rows<kVarlen>(p.cu, p.T, p.S, b, k0, row_base, len)) return;  // before any barrier exists
    const int qb0 = p.causal ? k0 / BS : 0;  // query blocks before the first key of the CTA see none of its keys
    const int n_qb_all = kVarlen ? (len + BS - 1) / BS : len / BS;
    const int n_qb = kWindow ? min(n_qb_all, (k0 + BQ - 1 + p.window - 1) / BS + 1) : n_qb_all;

    if (threadIdx.x == kProducer) {
        mbar_init(res_full, 1);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(full(s), 1);
            mbar_init(empty(s), 8);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (threadIdx.x >= kProducer) {
        if (threadIdx.x == kProducer) {
            mbar_expect_tx(res_full, 4 * TILE);
            for (int w = 0; w < 2; ++w) {
                load_tile<kD>(sbase + SM_RES + w * TILE, &map_k, res_full, kvh * kD, row_base + k0 + w * BS);
                load_tile<kD>(sbase + SM_RES + (2 + w) * TILE, &map_v, res_full, kvh * kD, row_base + k0 + w * BS);
            }
            int it = 0;
            for (int qh = kvh * rep; qh < (kvh + 1) * rep; ++qh)
                for (int qb = qb0; qb < n_qb; ++qb, ++it) {
                    const int s = it % STAGES;
                    mbar_wait(empty(s), ((it / STAGES) & 1) ^ 1);
                    mbar_expect_tx(full(s), 2 * TILE);
                    const uint32_t dst = sbase + SM_STR + s * 2 * TILE;
                    load_tile<kD>(dst, &map_q, full(s), qh * kD, row_base + qb * BS);
                    load_tile<kD>(dst + TILE, &map_do, full(s), qh * kD, row_base + qb * BS);
                }
        }
        return;
    }

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = warp >> 2;
    const int kr0 = k0 + wg * BS;
    const int r_loc = 16 * (warp & 3) + (lane >> 2);
    const int c_in = 2 * (lane & 3);
    const uint32_t sk = sbase + SM_RES + wg * TILE, sv = sbase + SM_RES + (2 + wg) * TILE;
    float dk[kD / 2], dv[kD / 2];
#pragma unroll
    for (int i = 0; i < kD / 2; ++i) dk[i] = dv[i] = 0.f;
    mbar_wait(res_full, 0);

    int it = 0;
    for (int qh = kvh * rep; qh < (kvh + 1) * rep; ++qh) {
        const float* lse2 = p.lse2 + stat_base<kVarlen>(p, b, qh, row_base);
        const float* delta = p.delta + stat_base<kVarlen>(p, b, qh, row_base);
        for (int qb = qb0; qb < n_qb; ++qb, ++it) {
            const int s = it % STAGES;
            mbar_wait(full(s), (it / STAGES) & 1);
            if (!(p.causal && qb * BS + BS - 1 < kr0) && !(kWindow && qb * BS > kr0 + BS - 1 + p.window - 1)) {
                const uint32_t sq = sbase + SM_STR + s * 2 * TILE, sdo = sq + TILE;
                float st[32], dpt[32];
                wgmma_fence();
                mma_rows_x_rows<kD>(dpt, sv, sdo);  // dP^T = V dO^T
                mma_rows_x_rows<kD>(st, sk, sq);    // S^T  = K Q^T
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs<32>(st);
                fence_regs<32>(dpt);
#pragma unroll
                for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int q = qb * BS + 8 * jj + c_in + e;
                        const bool q_in = !kVarlen || q < len;
                        const float l2 = q_in ? __ldg(lse2 + q) : 0.f, dl = q_in ? __ldg(delta + q) : 0.f;
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            const int key = kr0 + r_loc + 8 * i;
                            const int x = 4 * jj + 2 * i + e;
                            const float pe = ((p.causal && q < key) || (kWindow && q - key >= p.window))
                                                 ? 0.f
                                                 : ex2(fmaf(st[x], p.scale_log2, -l2));
                            st[x] = q_in ? pe : 0.f;
                            dpt[x] = q_in ? pe * (dpt[x] - dl) * p.scale : 0.f;
                        }
                    }
                uint32_t pf[4][4], df[4][4];
                to_frags(st, pf);
                to_frags(dpt, df);
                wgmma_fence();
                mma_regs_x_tile<kD>(dv, pf, sdo);  // dV += P^T dO
                mma_regs_x_tile<kD>(dk, df, sq);   // dK += dS^T Q
                wgmma_commit();
                wgmma_wait<0>();
                fence_regs<kD / 2>(dv);
                fence_regs<kD / 2>(dk);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty(s));
        }
    }
    const int64_t r0 = row_base + kr0;
    const int rows = kVarlen ? min(len - kr0, BS) : BS;
    store_acc<kD>(dk, p.dk + r0 * p.ld_dk, p.ld_dk, r_loc, rows, kvh * kD, c_in, 1.f, 1.f);
    store_acc<kD>(dv, p.dv + r0 * p.ld_dv, p.ld_dv, r_loc, rows, kvh * kD, c_in, 1.f, 1.f);
}

// ---- (B) dQ -------------------------------------------------------------------------------------------------------------------
// Varlen: keys past `len` get P = 0 and dS = 0; rows past `len` read no statistics and are never stored.
// Sliding window: the key blocks start at the forward's first block, keys before a row's window get P = 0 and dS = 0.
template <int kD, bool kVarlen, bool kWindow>
__global__ void __launch_bounds__(kThreads, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                   const __grid_constant__ CUtensorMap map_v, const __grid_constant__ CUtensorMap map_do, const BwdParams p)
{
    using Plan = kb<kD>;
    constexpr int STAGES = Plan::STAGES;
    constexpr uint32_t TILE = Plan::TILE, SM_RES = Plan::SM_RES, SM_STR = Plan::SM_STR, SM_BAR = Plan::SM_BAR;
    const int q0 = blockIdx.x * BQ, h = blockIdx.y, b = blockIdx.z;
    int row_base, len;
    if (!doc_rows<kVarlen>(p.cu, p.T, p.S, b, q0, row_base, len)) return;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const uint32_t sbase = smem_u32(smem);
    const uint32_t res_full = sbase + SM_BAR;
    auto full = [&](int s) { return sbase + SM_BAR + 8 * (1 + s); };
    auto empty = [&](int s) { return sbase + SM_BAR + 8 * (1 + STAGES + s); };

    const int kvh = h / (p.Hq / p.Hkv);
    const int n_blocks = kVarlen ? (len + BS - 1) / BS : len / BS;
    const int n_kv = p.causal ? (kVarlen ? min(n_blocks, (q0 + BQ) / BS) : (q0 + BQ) / BS) : n_blocks;
    const int j0 = first_key_block<kWindow>(q0, p.window);

    if (threadIdx.x == kProducer) {
        mbar_init(res_full, 1);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(full(s), 1);
            mbar_init(empty(s), 8);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (threadIdx.x >= kProducer) {
        if (threadIdx.x == kProducer) {
            mbar_expect_tx(res_full, 4 * TILE);
            for (int w = 0; w < 2; ++w) {
                load_tile<kD>(sbase + SM_RES + w * TILE, &map_q, res_full, h * kD, row_base + q0 + w * BS);
                load_tile<kD>(sbase + SM_RES + (2 + w) * TILE, &map_do, res_full, h * kD, row_base + q0 + w * BS);
            }
            for (int j = j0; j < n_kv; ++j) {
                const int s = (j - j0) % STAGES;
                mbar_wait(empty(s), (((j - j0) / STAGES) & 1) ^ 1);
                mbar_expect_tx(full(s), 2 * TILE);
                const uint32_t dst = sbase + SM_STR + s * 2 * TILE;
                load_tile<kD>(dst, &map_k, full(s), kvh * kD, row_base + j * BS);
                load_tile<kD>(dst + TILE, &map_v, full(s), kvh * kD, row_base + j * BS);
            }
        }
        return;
    }

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = warp >> 2;
    const int qr0 = q0 + wg * BS;
    const int r_loc = 16 * (warp & 3) + (lane >> 2);
    const int c_in = 2 * (lane & 3);
    const uint32_t sq = sbase + SM_RES + wg * TILE, sdo = sbase + SM_RES + (2 + wg) * TILE;
    const int64_t stat = stat_base<kVarlen>(p, b, h, row_base) + qr0 + r_loc;
    const bool in0 = !kVarlen || qr0 + r_loc < len, in1 = !kVarlen || qr0 + r_loc + 8 < len;
    const float l2[2] = {in0 ? p.lse2[stat] : 0.f, in1 ? p.lse2[stat + 8] : 0.f};
    const float dl[2] = {in0 ? p.delta[stat] : 0.f, in1 ? p.delta[stat + 8] : 0.f};
    float dq[kD / 2];
#pragma unroll
    for (int i = 0; i < kD / 2; ++i) dq[i] = 0.f;
    mbar_wait(res_full, 0);

    for (int j = j0; j < n_kv; ++j) {
        const int s = (j - j0) % STAGES;
        mbar_wait(full(s), ((j - j0) / STAGES) & 1);
        if (!(p.causal && j * BS > qr0 + BS - 1) && !(kWindow && j * BS + BS - 1 < qr0 - p.window + 1)) {
            const uint32_t sk = sbase + SM_STR + s * 2 * TILE, sv = sk + TILE;
            float sc[32], dp[32];
            wgmma_fence();
            mma_rows_x_rows<kD>(sc, sq, sk);   // S  = Q K^T
            mma_rows_x_rows<kD>(dp, sdo, sv);  // dP = dO V^T
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs<32>(sc);
            fence_regs<32>(dp);
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int key = j * BS + 8 * jj + c_in + e;
                        const int row = qr0 + r_loc + 8 * i;
                        const int x = 4 * jj + 2 * i + e;
                        const float pe = ((p.causal && key > row) || (kWindow && key <= row - p.window))
                                             ? 0.f
                                             : ex2(fmaf(sc[x], p.scale_log2, -l2[i]));
                        dp[x] = (kVarlen && key >= len) ? 0.f : pe * (dp[x] - dl[i]) * p.scale;
                    }
            uint32_t df[4][4];
            to_frags(dp, df);
            wgmma_fence();
            mma_regs_x_tile<kD>(dq, df, sk);  // dQ += dS K
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs<kD / 2>(dq);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(empty(s));
    }
    store_acc<kD>(dq, p.dq + static_cast<int64_t>(row_base + qr0) * p.ld_dq, p.ld_dq, r_loc,
                  kVarlen ? min(len - qr0, BS) : BS, h * kD, c_in, 1.f, 1.f);
}

// ---- launches ------------------------------------------------------------------------------------------------------------------
// Dense: n_seq = B sequences of S rows, T = B * S.  Varlen: n_seq = n_docs documents at offsets cu[0..n_docs], S = the longest
// document (it sizes the grid), T = cu[n_docs].  The tensor maps cover all T rows, so a tile that runs past a document reads
// the next document's rows (masked in the kernels) or TMA zero fill past T.
// head_dim is 64 or 128 (checked by the entry points); it picks the kernel instantiations and their shared-memory plan.
template <bool kVarlen, bool kWindow>
int launch_fwd(int head_dim, const void* q, const void* k, const void* v, void* o, float* lse, const int* cu, int n_seq, int S,
               int T, int Hq, int Hkv, int ld_q, int ld_k, int ld_v, int ld_o, int q_cols, int k_cols, int v_cols, float scale,
               int causal, int window, cudaStream_t stream)
{
    CUtensorMap mq, mk, mv;
    int rc;
    const uint64_t rows = static_cast<uint64_t>(T);
    if ((rc = make_map(&mq, q, rows, q_cols, ld_q, BS))) return rc;
    if ((rc = make_map(&mk, k, rows, k_cols, ld_k, BS))) return rc;
    if ((rc = make_map(&mv, v, rows, v_cols, ld_v, BS))) return rc;
    const bool d64 = head_dim == 64;
    const auto kernel = d64 ? attn_fwd_kernel<64, kVarlen, kWindow> : attn_fwd_kernel<128, kVarlen, kWindow>;
    const uint32_t smem = d64 ? kf<64>::SM_TOTAL : kf<128>::SM_TOTAL;
    static bool attr[2] = {false, false};
    if (!attr[d64]) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return static_cast<int>(e);
        attr[d64] = true;
    }
    FwdParams p;
    p.o = static_cast<__nv_bfloat16*>(o);
    p.lse = lse;
    p.ld_o = ld_o;
    p.S = S;
    p.Hq = Hq;
    p.Hkv = Hkv;
    p.scale_log2 = scale * 1.4426950408889634f;
    p.causal = causal;
    p.cu = cu;
    p.T = T;
    p.window = kWindow ? min(window, S) : 0;  // a window of S rows or more masks nothing
    dim3 grid((S + BQ - 1) / BQ, Hq, n_seq);
    kernel<<<grid, kThreads, smem, stream>>>(mq, mk, mv, p);
    DSB_CHECK_LAUNCH();
    return 0;
}

template <bool kVarlen, bool kWindow>
int launch_bwd(int head_dim, const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
               void* dq, void* dk, void* dv, float* work, const int* cu, int n_seq, int S, int T, int Hq, int Hkv, int ld_q,
               int ld_k, int ld_v, int ld_o, int ld_do, int ld_dq, int ld_dk, int ld_dv, int q_cols, int k_cols, int v_cols,
               float scale, int causal, int window, cudaStream_t stream)
{
    CUtensorMap mq, mk, mv, mdo;
    int rc;
    const uint64_t rows = static_cast<uint64_t>(T);
    if ((rc = make_map(&mq, q, rows, q_cols, ld_q, BS))) return rc;
    if ((rc = make_map(&mk, k, rows, k_cols, ld_k, BS))) return rc;
    if ((rc = make_map(&mv, v, rows, v_cols, ld_v, BS))) return rc;
    if ((rc = make_map(&mdo, d_o, rows, static_cast<uint64_t>(Hq) * head_dim, ld_do, BS))) return rc;
    const bool d64 = head_dim == 64;
    const auto dkdv = d64 ? attn_bwd_dkdv_kernel<64, kVarlen, kWindow> : attn_bwd_dkdv_kernel<128, kVarlen, kWindow>;
    const auto dq_kernel = d64 ? attn_bwd_dq_kernel<64, kVarlen, kWindow> : attn_bwd_dq_kernel<128, kVarlen, kWindow>;
    const auto prep = d64 ? attn_bwd_prep_kernel<64> : attn_bwd_prep_kernel<128>;
    const uint32_t smem = d64 ? kb<64>::SM_TOTAL : kb<128>::SM_TOTAL;
    static bool attr[2] = {false, false};
    if (!attr[d64]) {
        cudaError_t e = cudaFuncSetAttribute(dkdv, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return static_cast<int>(e);
        e = cudaFuncSetAttribute(dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return static_cast<int>(e);
        attr[d64] = true;
    }
    float* delta = work;
    float* lse2 = work + static_cast<int64_t>(T) * Hq;
    const int64_t prep_rows = static_cast<int64_t>(T) * Hq;
    // the varlen [Hq, T] statistics are the dense [B, Hq, S] layout with B = 1, S = T
    const int prep_b = kVarlen ? 1 : n_seq, prep_s = kVarlen ? T : S;
    prep<<<static_cast<unsigned>((prep_rows * 32 + 255) / 256), 256, 0, stream>>>(
        static_cast<const __nv_bfloat16*>(o), static_cast<const __nv_bfloat16*>(d_o), lse, delta, lse2, prep_b, prep_s, Hq,
        ld_o, ld_do);
    BwdParams p;
    p.dq = static_cast<__nv_bfloat16*>(dq);
    p.dk = static_cast<__nv_bfloat16*>(dk);
    p.dv = static_cast<__nv_bfloat16*>(dv);
    p.ld_dq = ld_dq;
    p.ld_dk = ld_dk;
    p.ld_dv = ld_dv;
    p.lse2 = lse2;
    p.delta = delta;
    p.S = S;
    p.Hq = Hq;
    p.Hkv = Hkv;
    p.scale = scale;
    p.scale_log2 = scale * 1.4426950408889634f;
    p.causal = causal;
    p.cu = cu;
    p.T = T;
    p.window = kWindow ? min(window, S) : 0;  // a window of S rows or more masks nothing
    const int nx = (S + BQ - 1) / BQ;
    dkdv<<<dim3(nx, Hkv, n_seq), kThreads, smem, stream>>>(mq, mk, mv, mdo, p);
    dq_kernel<<<dim3(nx, Hq, n_seq), kThreads, smem, stream>>>(mq, mk, mv, mdo, p);
    DSB_CHECK_LAUNCH();
    return 0;
}

}  // namespace attn
}  // namespace dsb

using namespace dsb::attn;

// The backward's operands must be 16-byte aligned: the tensor maps of q / k / v / d_o need it, the prep pass loads O as
// 8-byte words and store_acc writes dQ / dK / dV as 4-byte words, so a misaligned view is refused here instead of faulting.
static bool bwd_misaligned(const void* q, const void* k, const void* v, const void* o, const void* d_o, const void* dq,
                           const void* dk, const void* dv)
{
    return ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
             reinterpret_cast<uintptr_t>(o) | reinterpret_cast<uintptr_t>(d_o) | reinterpret_cast<uintptr_t>(dq) |
             reinterpret_cast<uintptr_t>(dk) | reinterpret_cast<uintptr_t>(dv)) & 15) != 0;
}

// q / k / v: 2-D bf16 tensors [B*S, *] (row stride ld_*), head `i` at columns [i*head_dim, +head_dim) -- for a packed QKV
// projection output all three point into the same buffer.  o: [B*S, ld_o] (head h at h*head_dim).  head_dim: 64 or 128.  lse: fp32 [B, Hq, S] or null.
// window > 0: causal sliding-window attention, row i sees keys i - window < j <= i (flash-attn's window_size = (window - 1,
// 0)); window <= 0: no window.  A window needs causal.
DSB_EXPORT int dsb_attn_fwd_bf16(const void* q, const void* k, const void* v, void* o, float* lse, int B, int S, int Hq,
                                 int Hkv, int head_dim, int ld_q, int ld_k, int ld_v, int ld_o, int q_cols, int k_cols,
                                 int v_cols, float scale, int causal, int window, cudaStream_t stream)
{
    if ((head_dim != 64 && head_dim != 128) || S <= 0 || Hq % Hkv || ld_q % 8 || ld_k % 8 || ld_v % 8 || ld_o % 8) return -2;
    if (B > 1 && S % BQ) return -2;  // ragged lengths: one sequence per launch (rows of the next one would be read as keys)
    if (window > 0 && !causal) return -2;
    if ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
         reinterpret_cast<uintptr_t>(o)) & 15)
        return -2;
    if (window > 0)
        return launch_fwd<false, true>(head_dim, q, k, v, o, lse, nullptr, B, S, B * S, Hq, Hkv, ld_q, ld_k, ld_v, ld_o, q_cols, k_cols,
                                       v_cols, scale, causal, window, stream);
    return launch_fwd<false, false>(head_dim, q, k, v, o, lse, nullptr, B, S, B * S, Hq, Hkv, ld_q, ld_k, ld_v, ld_o, q_cols, k_cols,
                                    v_cols, scale, causal, 0, stream);
}

// Backward.  q/k/v as in the forward; o, d_o: [B*S, ld] with head h at h*head_dim; lse from the forward.
// dq / dk / dv: 2-D outputs (may be column ranges of ONE packed buffer).  work: fp32 scratch of 2 * B * Hq * S elements.
// window: the forward's.
DSB_EXPORT int dsb_attn_bwd_bf16(const void* q, const void* k, const void* v, const void* o, const void* d_o, const float* lse,
                                 void* dq, void* dk, void* dv, float* work, int B, int S, int Hq, int Hkv, int head_dim,
                                 int ld_q, int ld_k, int ld_v, int ld_o, int ld_do, int ld_dq, int ld_dk, int ld_dv, int q_cols,
                                 int k_cols, int v_cols, float scale, int causal, int window, cudaStream_t stream)
{
    if ((head_dim != 64 && head_dim != 128) || S % BQ || Hq % Hkv || (ld_q | ld_k | ld_v | ld_o | ld_do | ld_dq | ld_dk | ld_dv) % 8) return -2;
    if (window > 0 && !causal) return -2;
    if (bwd_misaligned(q, k, v, o, d_o, dq, dk, dv)) return -2;
    if (window > 0)
        return launch_bwd<false, true>(head_dim, q, k, v, o, d_o, lse, dq, dk, dv, work, nullptr, B, S, B * S, Hq, Hkv, ld_q, ld_k, ld_v,
                                       ld_o, ld_do, ld_dq, ld_dk, ld_dv, q_cols, k_cols, v_cols, scale, causal, window, stream);
    return launch_bwd<false, false>(head_dim, q, k, v, o, d_o, lse, dq, dk, dv, work, nullptr, B, S, B * S, Hq, Hkv, ld_q, ld_k, ld_v,
                                    ld_o, ld_do, ld_dq, ld_dk, ld_dv, q_cols, k_cols, v_cols, scale, causal, 0, stream);
}

// Packed sequences (document-masked attention).  q / k / v / o as in dsb_attn_fwd_bf16 over T = cu_seqlens[n_docs] token
// rows; cu_seqlens: int32 device array of n_docs + 1 non-decreasing offsets from 0 to T (empty documents allowed);
// max_seqlen: the longest document (or more).  Each token attends only within its document.  lse: fp32 [Hq, T] or null.
// window as in dsb_attn_fwd_bf16, measured inside each document.
DSB_EXPORT int dsb_attn_varlen_fwd_bf16(const void* q, const void* k, const void* v, void* o, float* lse,
                                        const int* cu_seqlens, int n_docs, int max_seqlen, int T, int Hq, int Hkv,
                                        int head_dim, int ld_q, int ld_k, int ld_v, int ld_o, int q_cols, int k_cols,
                                        int v_cols, float scale, int causal, int window, cudaStream_t stream)
{
    if ((head_dim != 64 && head_dim != 128) || Hq % Hkv || ld_q % 8 || ld_k % 8 || ld_v % 8 || ld_o % 8) return -2;
    if (T < 0 || n_docs < 0 || n_docs > 65535 || (T > 0 && max_seqlen <= 0) || cu_seqlens == nullptr) return -2;
    if (window > 0 && !causal) return -2;
    if ((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
         reinterpret_cast<uintptr_t>(o)) & 15)
        return -2;
    if (T == 0 || n_docs == 0) return 0;
    if (window > 0)
        return launch_fwd<true, true>(head_dim, q, k, v, o, lse, cu_seqlens, n_docs, max_seqlen, T, Hq, Hkv, ld_q, ld_k, ld_v, ld_o,
                                      q_cols, k_cols, v_cols, scale, causal, window, stream);
    return launch_fwd<true, false>(head_dim, q, k, v, o, lse, cu_seqlens, n_docs, max_seqlen, T, Hq, Hkv, ld_q, ld_k, ld_v, ld_o, q_cols,
                                   k_cols, v_cols, scale, causal, 0, stream);
}

// Backward of dsb_attn_varlen_fwd_bf16 (same cu_seqlens / max_seqlen / window; lse [Hq, T] from it).  dq / dk / dv may be
// column ranges of one packed buffer.  work: fp32 scratch of 2 * Hq * T elements.
DSB_EXPORT int dsb_attn_varlen_bwd_bf16(const void* q, const void* k, const void* v, const void* o, const void* d_o,
                                        const float* lse, void* dq, void* dk, void* dv, float* work, const int* cu_seqlens,
                                        int n_docs, int max_seqlen, int T, int Hq, int Hkv, int head_dim, int ld_q, int ld_k,
                                        int ld_v, int ld_o, int ld_do, int ld_dq, int ld_dk, int ld_dv, int q_cols,
                                        int k_cols, int v_cols, float scale, int causal, int window, cudaStream_t stream)
{
    if ((head_dim != 64 && head_dim != 128) || Hq % Hkv || (ld_q | ld_k | ld_v | ld_o | ld_do | ld_dq | ld_dk | ld_dv) % 8) return -2;
    if (T < 0 || n_docs < 0 || n_docs > 65535 || (T > 0 && max_seqlen <= 0) || cu_seqlens == nullptr) return -2;
    if (window > 0 && !causal) return -2;
    if (bwd_misaligned(q, k, v, o, d_o, dq, dk, dv)) return -2;
    if (T == 0 || n_docs == 0) return 0;
    if (window > 0)
        return launch_bwd<true, true>(head_dim, q, k, v, o, d_o, lse, dq, dk, dv, work, cu_seqlens, n_docs, max_seqlen, T, Hq, Hkv, ld_q,
                                      ld_k, ld_v, ld_o, ld_do, ld_dq, ld_dk, ld_dv, q_cols, k_cols, v_cols, scale, causal,
                                      window, stream);
    return launch_bwd<true, false>(head_dim, q, k, v, o, d_o, lse, dq, dk, dv, work, cu_seqlens, n_docs, max_seqlen, T, Hq, Hkv, ld_q,
                                   ld_k, ld_v, ld_o, ld_do, ld_dq, ld_dk, ld_dv, q_cols, k_cols, v_cols, scale, causal, 0,
                                   stream);
}
