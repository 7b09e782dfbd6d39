// Flash attention with additive biases and a block-sparsity layout, forward + backward, for SMALL head dims (16 / 32 / 64).
//
// Two users (SURVEY.md N12 and P40):
//   * Evoformer attention (reference csrc/deepspeed4science/evoformer_attn/{kernel_forward.h:109, kernel_backward.h} behind
//     ops/deepspeed4science/evoformer_attn.py:15): Q/K/V [*, L, H, D], a per-key mask bias [B, N, 1, 1, L] and a pair bias
//     [B, 1, H, L, L] shared by all N rows of the MSA; the backward also produces both bias gradients.
//   * Block-sparse attention (reference Triton SDD / DSD / softmax in ops/sparse_attention/{matmul.py, softmax.py}): a
//     [H, L/bs, L/bs] 0/1 layout decides which score blocks exist; key-padding / attention masks ride the two bias slots.
//
// Why mma.sync and not wgmma here: with D <= 64 the two GEMMs of a score tile are 4*D <= 256 FLOP per score while every
// score still costs one exp2 and (backward) one registers read each for S and dP.  At registers's ~16 fp32 / clk / SM the wgmma
// formulation is capped at the SFU rate before the tensor core matters, and the fixed 128-row tile wastes most of an MSA
// row of 100-300 residues.  Register accumulators (m16n8k16, 16 query rows per warp) have no such read port: S, P, dP, dS
// never leave the register file, P / dS are re-used in place as the A operand of the second GEMM.
//
// Structure: a CTA is 4 warps x 16 rows = 64 rows; K / V (forward, dQ) or Q / dO (dK / dV) tiles of 64 rows stream through
// a 2-stage cp.async ring (row pitch padded by 16 B: ldmatrix conflict-free for every D) -- together with the matching
// [64 x 64] pair-bias tile and the 64 per-key bias values, so no bias load sits on the softmax's critical path.  The
// block-sparsity layout is turned into a compacted list of active tiles (+ a 4 x 4 sub-block mask each) once per CTA.  Backward is two kernels and has
// no dQ atomics: (A) one CTA per 64 keys computes the TRANSPOSED scores S^T = K Q^T so P^T / dS^T are already the A operand
// of dV += P^T dO and dK += dS^T Q, and reduces dS over queries into the mask-bias gradient; (B) one CTA per 64 queries
// recomputes S, forms dQ += dS K and adds dS into the pair-bias gradient (fp32 vector reductions: the sum over the N rows
// of the MSA crosses CTAs).
#include <type_traits>
#include "dsb_common.cuh"

namespace dsb {
namespace battn {

struct Params {
    const void* q;
    const void* k;
    const void* v;
    void* o;
    float* lse;  // [NB, H, Lq], natural log; +inf for rows without any visible key
    const void* bias1;
    const void* bias2;
    const uint8_t* layout;
    const void* d_o;
    void* dq;
    void* dk;
    void* dv;
    float* delta;  // [NB, H, Lq]
    float* db1;    // [NB1, Lk] fp32 (same batch stride rule as bias1)
    float* db2;    // fp32, contiguous [B2, H2, Lq, Lk]
    int NB, H, Lq, Lk;
    int64_t q_b, q_h, q_r, k_b, k_h, k_r, v_b, v_h, v_r, o_b, o_h, o_r;  // element strides (dq/dk/dv/dO follow q/k/v/o)
    int64_t b1_b;                                                          // bias1 / db1 batch stride (0 = shared)
    int b2_div;                                                            // bias2 batch index = nb / b2_div
    int64_t b2_b, b2_h, b2_r;                                              // bias2 strides
    int64_t g2_b, g2_h;                                                    // db2 strides (row stride = Lk)
    int lay_bs, lay_nq, lay_nk;  // lay_bs is a power of two >= 16; lay_sh = log2(lay_bs)
    int lay_sh;
    int64_t lay_h;
    int stage_bias;  // both biases are 16-byte tileable: stream them through shared memory with the K/V (Q/dO) tiles
    int list_cap;    // capacity (tiles) of the active-tile list in shared memory
    float scale;
    int causal;
};

constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

template <typename T>
struct Mma;
template <>
struct Mma<__nv_bfloat16> {
    static __device__ __forceinline__ void run(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
    {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
    static __device__ __forceinline__ uint32_t pack(float lo, float hi)
    {
        __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
        return *reinterpret_cast<uint32_t*>(&v);
    }
    static __device__ __forceinline__ float to_f(__nv_bfloat16 x) { return __bfloat162float(x); }
};
template <>
struct Mma<__half> {
    static __device__ __forceinline__ void run(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
    {
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
    }
    static __device__ __forceinline__ uint32_t pack(float lo, float hi)
    {
        __half2 v = __floats2half2_rn(lo, hi);
        return *reinterpret_cast<uint32_t*>(&v);
    }
    static __device__ __forceinline__ float to_f(__half x) { return __half2float(x); }
};

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3)
{
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3)
{
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
                 : "r"(addr));
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool valid)
{
    const int n = valid ? 16 : 0;  // src-size 0: the 16 destination bytes are zero-filled, nothing is read
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait()
{
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ float fast_exp2(float x)
{
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t ld_u32(const void* p) { return *reinterpret_cast<const uint32_t*>(p); }
__device__ __forceinline__ void red_add_v2(float* p, float a, float b)
{
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}

constexpr int kThreads = 128;
constexpr int kTile = 64;  // rows of a CTA / rows of a streamed tile

template <int D>
struct Cfg {
    static constexpr int KS = D / 16;            // k-steps of a [*, D] contraction
    static constexpr int ON = D / 8;             // n-tiles of a [*, D] output
    static constexpr int NT = kTile / 8;         // n-tiles across a streamed tile
    static constexpr int PITCH = D * 2 + 16;     // bytes per smem row
    static constexpr int TILE_BYTES = kTile * PITCH;
    static constexpr int CHUNKS = D / 8;         // 16-byte pieces per row
};

// Copies rows [row0, row0 + 64) of a [L, D] operand (row stride `rs` elements) into a padded smem tile.
template <typename T, int D>
__device__ __forceinline__ void load_tile(uint32_t dst, const T* base, int64_t rs, int row0, int L, int tid)
{
    using C = Cfg<D>;
#pragma unroll
    for (int i = tid; i < kTile * C::CHUNKS; i += kThreads) {
        const int r = i / C::CHUNKS, c = i % C::CHUNKS;
        const bool ok = row0 + r < L;
        cp_async16(dst + r * C::PITCH + c * 16, base + (ok ? static_cast<int64_t>(row0 + r) * rs + c * 8 : 0), ok);
    }
}

// A fragments of 16 rows [r0 + g, r0 + g + 8] x D taken straight from global memory (done once per CTA).
template <typename T, int D>
__device__ __forceinline__ void load_a_frag(uint32_t (&f)[Cfg<D>::KS][4], const T* base, int64_t rs, int r_lo, int L, int t)
{
    const int r_hi = r_lo + 8;
#pragma unroll
    for (int ks = 0; ks < Cfg<D>::KS; ++ks) {
        const int c = ks * 16 + 2 * t;
        f[ks][0] = r_lo < L ? ld_u32(base + static_cast<int64_t>(r_lo) * rs + c) : 0u;
        f[ks][1] = r_hi < L ? ld_u32(base + static_cast<int64_t>(r_hi) * rs + c) : 0u;
        f[ks][2] = r_lo < L ? ld_u32(base + static_cast<int64_t>(r_lo) * rs + c + 8) : 0u;
        f[ks][3] = r_hi < L ? ld_u32(base + static_cast<int64_t>(r_hi) * rs + c + 8) : 0u;
    }
}

// acc[j] (16 x 8 each, j over the 64 streamed rows) += A[16 x D] * tile[64 x D]^T   (tile rows are the n index)
template <typename T, int D>
__device__ __forceinline__ void mma_a_tileT(float (&acc)[8][4], const uint32_t (&a)[Cfg<D>::KS][4], uint32_t tile, int lane)
{
    using C = Cfg<D>;
    const int mi = lane >> 3;
    const uint32_t lane_off = ((lane & 7) + (mi >> 1) * 8) * C::PITCH + (mi & 1) * 16;
#pragma unroll
    for (int ks = 0; ks < C::KS; ++ks) {
#pragma unroll
        for (int jp = 0; jp < C::NT / 2; ++jp) {
            uint32_t r0, r1, r2, r3;
            ldsm_x4(tile + jp * 16 * C::PITCH + ks * 32 + lane_off, r0, r1, r2, r3);
            Mma<T>::run(acc[2 * jp], a[ks], r0, r1);
            Mma<T>::run(acc[2 * jp + 1], a[ks], r2, r3);
        }
    }
}

// out[dn] (16 x 8 each over D) += P[16 x 64] * tile[64 x D]   (tile rows are the k index); P given as packed A fragments.
template <typename T, int D>
__device__ __forceinline__ void mma_p_tile(float (&out)[Cfg<D>::ON][4], const uint32_t (&pa)[4][4], uint32_t tile, int lane)
{
    using C = Cfg<D>;
    const int mi = lane >> 3;
    const uint32_t lane_off = ((lane & 7) + (mi & 1) * 8) * C::PITCH + (mi >> 1) * 16;
#pragma unroll
    for (int kk = 0; kk < kTile / 16; ++kk) {
#pragma unroll
        for (int dn = 0; dn < C::ON / 2; ++dn) {
            uint32_t r0, r1, r2, r3;
            ldsm_x4_t(tile + kk * 16 * C::PITCH + dn * 32 + lane_off, r0, r1, r2, r3);
            Mma<T>::run(out[2 * dn], pa[kk], r0, r1);
            Mma<T>::run(out[2 * dn + 1], pa[kk], r2, r3);
        }
    }
}

// ---- block-sparsity layout ------------------------------------------------------------------------------------------------
// A CTA first builds, in parallel, the list of streamed tiles that contain at least one active layout block together with a
// 16-bit mask of the (up to 4 x 4) layout blocks inside each 64 x 64 score tile; the main loop then walks the compacted list
// (no dependent global loads, no divisions on the critical path).  mask bit = q_sub * nsb + k_sub.
__device__ __forceinline__ uint32_t tile_mask(const Params& p, const uint8_t* lay, int qt, int kt)
{
    if (lay == nullptr) return 0xffffu;
    const int sh = p.lay_sh;
    const int nsb = sh >= 6 ? 1 : (kTile >> sh);
    uint32_t m = 0;
    for (int a = 0; a < nsb; ++a) {
        const int qa = min((qt * kTile + (a << sh)) >> sh, p.lay_nq - 1);
        const bool q_in = sh >= 6 || (qt * kTile + (a << sh)) < (p.lay_nq << sh);
        for (int b = 0; b < nsb; ++b) {
            const int kb = min((kt * kTile + (b << sh)) >> sh, p.lay_nk - 1);
            const bool k_in = sh >= 6 || (kt * kTile + (b << sh)) < (p.lay_nk << sh);
            if (q_in && k_in && lay[qa * p.lay_nk + kb]) m |= 1u << (a * nsb + b);
        }
    }
    return m;
}

// Fills idx[0 .. n) with the active tiles of [first, n_tiles) (ascending) and mask[tile] for every tile; returns n.
// `fixed_is_q`: the CTA owns query tile `fixed` and streams key tiles (forward, dQ) -- otherwise it owns a key tile.
__device__ __forceinline__ int build_tile_list(const Params& p, const uint8_t* lay, bool fixed_is_q, int fixed, int first,
                                               int n_tiles, uint16_t* idx, uint16_t* mask, int* count_slot)
{
    const int tid = threadIdx.x;
    for (int t = first + tid; t < n_tiles; t += blockDim.x)
        mask[t] = static_cast<uint16_t>(fixed_is_q ? tile_mask(p, lay, fixed, t) : tile_mask(p, lay, t, fixed));
    __syncthreads();
    if (tid < 32) {
        int count = 0;
        for (int base = first; base < n_tiles; base += 32) {
            const int t = base + tid;
            const bool on = t < n_tiles && mask[t] != 0;
            const uint32_t bal = __ballot_sync(0xffffffffu, on);
            if (on) idx[count + __popc(bal & ((1u << tid) - 1u))] = static_cast<uint16_t>(t);
            count += __popc(bal);
        }
        if (tid == 0) *count_slot = count;
    }
    __syncthreads();
    return *count_slot;
}
// is layout block (row sub-block of `row_in_tile`, col sub-block of `col_in_tile`) of a tile with mask `m` active?
__device__ __forceinline__ bool sub_on(const Params& p, uint32_t m, int q_in_tile, int k_in_tile)
{
    const int sh = p.lay_sh;
    if (sh >= 6) return m != 0;
    const int nsb = kTile >> sh;
    return (m >> ((q_in_tile >> sh) * nsb + (k_in_tile >> sh))) & 1u;
}

__device__ __forceinline__ bool all_sub_on(const Params& p, uint32_t m)
{
    if (p.lay_sh >= 6) return m != 0;
    const int nsb = kTile >> p.lay_sh;
    const uint32_t full = (1u << (nsb * nsb)) - 1u;
    return (m & full) == full;
}

// ---- bias tiles in shared memory ----------------------------------------------------------------------------------------------
constexpr int kBiasPitch = kTile * 2 + 16;                       // bytes per row of a staged [64 x 64] pair-bias tile
constexpr int kBiasStage = kTile * kBiasPitch + kTile * 2;       // pair-bias tile + 64 per-key bias values
template <typename T>
__device__ __forceinline__ void load_bias_tile(uint32_t dst, const T* b2, int64_t b2_r, int row0, int n_rows, int col0, int n_cols,
                                               const T* b1, int tid)
{
    if (b2 != nullptr) {
#pragma unroll
        for (int i = tid; i < kTile * 8; i += kThreads) {
            const int r = i >> 3, c = i & 7;
            const bool ok = row0 + r < n_rows && col0 + c * 8 < n_cols;
            cp_async16(dst + r * kBiasPitch + c * 16, b2 + (ok ? static_cast<int64_t>(row0 + r) * b2_r + col0 + c * 8 : 0), ok);
        }
    }
    if (b1 != nullptr && tid < 8) {
        const bool ok = col0 + tid * 8 < n_cols;
        cp_async16(dst + kTile * kBiasPitch + tid * 16, b1 + (ok ? col0 + tid * 8 : 0), ok);
    }
}
template <typename T>
__device__ __forceinline__ float2 lds_pair(const uint8_t* p)
{
    const uint32_t w = *reinterpret_cast<const uint32_t*>(p);
    if constexpr (sizeof(T) == 2 && std::is_same<T, __nv_bfloat16>::value) {
        return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
    } else {
        const __half2 h = *reinterpret_cast<const __half2*>(&w);
        return __half22float2(h);
    }
}

template <typename T>
__device__ __forceinline__ float ldb(const T* p, int64_t i)
{
    return Mma<T>::to_f(p[i]);
}

// ---- forward -------------------------------------------------------------------------------------------------------------------
template <typename T, int D>
__global__ void __launch_bounds__(kThreads) fwd_kernel(const Params p)
{
    using C = Cfg<D>;
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t sb = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int qt = blockIdx.x, h = blockIdx.y, nb = blockIdx.z;
    const int r_lo = qt * kTile + warp * 16 + g, r_hi = r_lo + 8;

    const T* qp = static_cast<const T*>(p.q) + nb * p.q_b + h * p.q_h;
    const T* kp = static_cast<const T*>(p.k) + nb * p.k_b + h * p.k_h;
    const T* vp = static_cast<const T*>(p.v) + nb * p.v_b + h * p.v_h;
    const T* b1 = p.bias1 ? static_cast<const T*>(p.bias1) + nb * p.b1_b : nullptr;
    const T* b2 = p.bias2 ? static_cast<const T*>(p.bias2) + (nb / p.b2_div) * p.b2_b + h * p.b2_h : nullptr;
    const uint8_t* lay = p.layout ? p.layout + h * p.lay_h : nullptr;

    uint32_t qf[C::KS][4];
    load_a_frag<T, D>(qf, qp, p.q_r, r_lo, p.Lq, t);

    int n_kt = (p.Lk + kTile - 1) / kTile;
    if (p.causal) n_kt = min(n_kt, qt + 1);
    const bool staged = p.stage_bias && (b1 != nullptr || b2 != nullptr);
    const uint32_t bias_off = 4 * C::TILE_BYTES;
    uint8_t* list_base = smem + bias_off + (staged ? 2 * kBiasStage : 0);
    uint16_t* tl_idx = reinterpret_cast<uint16_t*>(list_base);
    uint16_t* tl_mask = tl_idx + p.list_cap;
    int* tl_count = reinterpret_cast<int*>(tl_mask + p.list_cap);
    const int n_act = build_tile_list(p, lay, true, qt, 0, n_kt, tl_idx, tl_mask, tl_count);
    auto issue = [&](int kt, int buf) {
        load_tile<T, D>(sb + buf * 2 * C::TILE_BYTES, kp, p.k_r, kt * kTile, p.Lk, tid);
        load_tile<T, D>(sb + buf * 2 * C::TILE_BYTES + C::TILE_BYTES, vp, p.v_r, kt * kTile, p.Lk, tid);
        if (staged) load_bias_tile<T>(sb + bias_off + buf * kBiasStage, b2, p.b2_r, qt * kTile, p.Lq, kt * kTile, p.Lk, b1, tid);
        cp_async_commit();
    };

    float o[C::ON][4];
#pragma unroll
    for (int i = 0; i < C::ON; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m_lo = -INFINITY, m_hi = -INFINITY, l_lo = 0.f, l_hi = 0.f;
    const float sc2 = p.scale * kLog2e;

    int buf = 0;
    if (n_act > 0) issue(tl_idx[0], 0);
    for (int it = 0; it < n_act; ++it) {
        const int kt = tl_idx[it];
        const uint32_t tmask = tl_mask[kt];
        if (it + 1 < n_act) {
            issue(tl_idx[it + 1], buf ^ 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const uint8_t* bst = smem + bias_off + buf * kBiasStage;  // staged pair-bias tile | per-key bias
        const uint32_t kb = sb + buf * 2 * C::TILE_BYTES, vb = kb + C::TILE_BYTES;
        float s[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
        mma_a_tileT<T, D>(s, qf, kb, lane);

        // additive bias (times log2 e) of score columns (c0, c0 + 1) of n-tile j for this thread's two rows
        auto bias_pair = [&](int j, float2& lo, float2& hi) {
            float2 k1 = make_float2(0.f, 0.f);
            lo = hi = k1;
            if (staged) {
                const int cb = (j * 8 + 2 * t) * 2;
                if (b1) k1 = lds_pair<T>(bst + kTile * kBiasPitch + cb);
                if (b2) {
                    lo = lds_pair<T>(bst + (warp * 16 + g) * kBiasPitch + cb);
                    hi = lds_pair<T>(bst + (warp * 16 + g + 8) * kBiasPitch + cb);
                }
            } else {  // unaligned shapes: clamped direct loads (out-of-range entries are masked below)
                const int ca = min(kt * kTile + j * 8 + 2 * t, p.Lk - 1), cb = min(kt * kTile + j * 8 + 2 * t + 1, p.Lk - 1);
                if (b1) k1 = make_float2(ldb(b1, ca), ldb(b1, cb));
                if (b2) {
                    const int64_t ra = static_cast<int64_t>(min(r_lo, p.Lq - 1)) * p.b2_r, rb = static_cast<int64_t>(min(r_hi, p.Lq - 1)) * p.b2_r;
                    lo = make_float2(ldb(b2, ra + ca), ldb(b2, ra + cb));
                    hi = make_float2(ldb(b2, rb + ca), ldb(b2, rb + cb));
                }
            }
            lo.x = (lo.x + k1.x) * kLog2e;
            lo.y = (lo.y + k1.y) * kLog2e;
            hi.x = (hi.x + k1.x) * kLog2e;
            hi.y = (hi.y + k1.y) * kLog2e;
        };
        const bool has_bias = b1 != nullptr || b2 != nullptr;
        // a tile entirely inside the sequence, below the causal diagonal and with every layout block on needs no masking
        const bool plain = (kt * kTile + kTile <= p.Lk) && !(p.causal && kt * kTile + kTile - 1 > qt * kTile + warp * 16) &&
                           all_sub_on(p, tmask);
        float mx_lo = -INFINITY, mx_hi = -INFINITY;
        if (plain) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float2 lo = make_float2(0.f, 0.f), hi = lo;
                if (has_bias) bias_pair(j, lo, hi);
                s[j][0] = fmaf(s[j][0], sc2, lo.x);
                s[j][1] = fmaf(s[j][1], sc2, lo.y);
                s[j][2] = fmaf(s[j][2], sc2, hi.x);
                s[j][3] = fmaf(s[j][3], sc2, hi.y);
                mx_lo = fmaxf(mx_lo, fmaxf(s[j][0], s[j][1]));
                mx_hi = fmaxf(mx_hi, fmaxf(s[j][2], s[j][3]));
            }
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c0 = kt * kTile + j * 8 + 2 * t;
                const bool on = sub_on(p, tmask, warp * 16, j * 8);
                float2 lo = make_float2(0.f, 0.f), hi = lo;
                if (has_bias) bias_pair(j, lo, hi);
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = c0 + e;
                    const bool in = col < p.Lk && on;
                    const bool v_lo = in && !(p.causal && col > r_lo), v_hi = in && !(p.causal && col > r_hi);
                    s[j][e] = v_lo ? fmaf(s[j][e], sc2, e ? lo.y : lo.x) : -INFINITY;
                    s[j][2 + e] = v_hi ? fmaf(s[j][2 + e], sc2, e ? hi.y : hi.x) : -INFINITY;
                    mx_lo = fmaxf(mx_lo, s[j][e]);
                    mx_hi = fmaxf(mx_hi, s[j][2 + e]);
                }
            }
        }
        mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1));
        mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
        mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1));
        mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));
        const float mn_lo = fmaxf(m_lo, mx_lo), mn_hi = fmaxf(m_hi, mx_hi);
        const float mu_lo = mn_lo == -INFINITY ? 0.f : mn_lo, mu_hi = mn_hi == -INFINITY ? 0.f : mn_hi;
        const float al_lo = fast_exp2(m_lo - mu_lo), al_hi = fast_exp2(m_hi - mu_hi);
        m_lo = mn_lo;
        m_hi = mn_hi;
        float sum_lo = 0.f, sum_hi = 0.f;
        uint32_t pa[4][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float p0 = fast_exp2(s[j][0] - mu_lo), p1 = fast_exp2(s[j][1] - mu_lo);
            const float p2 = fast_exp2(s[j][2] - mu_hi), p3 = fast_exp2(s[j][3] - mu_hi);
            sum_lo += p0 + p1;
            sum_hi += p2 + p3;
            pa[j >> 1][(j & 1) * 2] = Mma<T>::pack(p0, p1);
            pa[j >> 1][(j & 1) * 2 + 1] = Mma<T>::pack(p2, p3);
        }
        l_lo = l_lo * al_lo + sum_lo;
        l_hi = l_hi * al_hi + sum_hi;
#pragma unroll
        for (int i = 0; i < C::ON; ++i) {
            o[i][0] *= al_lo;
            o[i][1] *= al_lo;
            o[i][2] *= al_hi;
            o[i][3] *= al_hi;
        }
        mma_p_tile<T, D>(o, pa, vb, lane);
        __syncthreads();
        buf ^= 1;
    }
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 1);
    l_lo += __shfl_xor_sync(0xffffffffu, l_lo, 2);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 1);
    l_hi += __shfl_xor_sync(0xffffffffu, l_hi, 2);
    const float inv_lo = l_lo > 0.f ? 1.f / l_lo : 0.f, inv_hi = l_hi > 0.f ? 1.f / l_hi : 0.f;
    T* op = static_cast<T*>(p.o) + nb * p.o_b + h * p.o_h;
#pragma unroll
    for (int i = 0; i < C::ON; ++i) {
        const int c = i * 8 + 2 * t;
        if (r_lo < p.Lq)
            *reinterpret_cast<uint32_t*>(op + static_cast<int64_t>(r_lo) * p.o_r + c) = Mma<T>::pack(o[i][0] * inv_lo, o[i][1] * inv_lo);
        if (r_hi < p.Lq)
            *reinterpret_cast<uint32_t*>(op + static_cast<int64_t>(r_hi) * p.o_r + c) = Mma<T>::pack(o[i][2] * inv_hi, o[i][3] * inv_hi);
    }
    if (p.lse != nullptr && t == 0) {
        float* lp = p.lse + (static_cast<int64_t>(nb) * p.H + h) * p.Lq;
        if (r_lo < p.Lq) lp[r_lo] = l_lo > 0.f ? (m_lo + log2f(l_lo)) * kLn2 : INFINITY;
        if (r_hi < p.Lq) lp[r_hi] = l_hi > 0.f ? (m_hi + log2f(l_hi)) * kLn2 : INFINITY;
    }
}

// ---- backward prep: delta = rowsum(dO * O) ---------------------------------------------------------------------------------------
template <typename T, int D>
__global__ void __launch_bounds__(256) delta_kernel(const Params p)
{
    constexpr int LPR = D / 8;  // lanes per row (16-byte pieces)
    const int64_t idx = static_cast<int64_t>(blockIdx.x) * 256 + threadIdx.x;
    const int64_t row = idx / LPR;
    const int c = static_cast<int>(idx % LPR);
    const int64_t total = static_cast<int64_t>(p.NB) * p.H * p.Lq;
    float acc = 0.f;
    if (row < total) {
        const int r = static_cast<int>(row % p.Lq);
        const int h = static_cast<int>((row / p.Lq) % p.H);
        const int64_t nb = row / (static_cast<int64_t>(p.Lq) * p.H);
        const int64_t off = nb * p.o_b + h * p.o_h + static_cast<int64_t>(r) * p.o_r + c * 8;
        const Vec16 a = ld_plain(static_cast<const T*>(p.o) + off), b = ld_plain(static_cast<const T*>(p.d_o) + off);
        const T* ap = reinterpret_cast<const T*>(&a);
        const T* bp = reinterpret_cast<const T*>(&b);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc += Mma<T>::to_f(ap[e]) * Mma<T>::to_f(bp[e]);
    }
#pragma unroll
    for (int sft = 1; sft < LPR; sft <<= 1) acc += __shfl_xor_sync(0xffffffffu, acc, sft);
    if (row < total && c == 0) p.delta[row] = acc;
}

// ---- backward (A): dK, dV, d(mask bias) -- one CTA per 64 keys, transposed scores ------------------------------------------------
template <typename T, int D>
__global__ void __launch_bounds__(kThreads) bwd_dkdv_kernel(const Params p)
{
    using C = Cfg<D>;
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t sb = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
    float* stat = reinterpret_cast<float*>(smem + 4 * C::TILE_BYTES);  // [2 stages][lse2 | delta][64]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int kt = blockIdx.x, h = blockIdx.y, nb = blockIdx.z;
    const int k_lo = kt * kTile + warp * 16 + g, k_hi = k_lo + 8;  // this thread's two key rows

    const T* qp = static_cast<const T*>(p.q) + nb * p.q_b + h * p.q_h;
    const T* kp = static_cast<const T*>(p.k) + nb * p.k_b + h * p.k_h;
    const T* vp = static_cast<const T*>(p.v) + nb * p.v_b + h * p.v_h;
    const T* dop = static_cast<const T*>(p.d_o) + nb * p.o_b + h * p.o_h;
    const T* b1 = p.bias1 ? static_cast<const T*>(p.bias1) + nb * p.b1_b : nullptr;
    const T* b2 = p.bias2 ? static_cast<const T*>(p.bias2) + (nb / p.b2_div) * p.b2_b + h * p.b2_h : nullptr;
    const uint8_t* lay = p.layout ? p.layout + h * p.lay_h : nullptr;
    const float* lse = p.lse + (static_cast<int64_t>(nb) * p.H + h) * p.Lq;
    const float* dl = p.delta + (static_cast<int64_t>(nb) * p.H + h) * p.Lq;

    uint32_t kf[C::KS][4], vf[C::KS][4];
    load_a_frag<T, D>(kf, kp, p.k_r, k_lo, p.Lk, t);
    load_a_frag<T, D>(vf, vp, p.v_r, k_lo, p.Lk, t);
    const float b1_lo = (b1 && k_lo < p.Lk) ? ldb(b1, k_lo) * kLog2e : 0.f;
    const float b1_hi = (b1 && k_hi < p.Lk) ? ldb(b1, k_hi) * kLog2e : 0.f;

    const int n_qt = (p.Lq + kTile - 1) / kTile;
    const int q_first = p.causal ? kt : 0;
    const bool staged = p.stage_bias && b2 != nullptr;  // (the per-key bias is a per-thread constant here)
    const uint32_t bias_off = 4 * C::TILE_BYTES + 2 * 128 * 4;
    uint8_t* list_base = smem + bias_off + (staged ? 2 * kBiasStage : 0);
    uint16_t* tl_idx = reinterpret_cast<uint16_t*>(list_base);
    uint16_t* tl_mask = tl_idx + p.list_cap;
    int* tl_count = reinterpret_cast<int*>(tl_mask + p.list_cap);
    const int n_act = build_tile_list(p, lay, false, kt, q_first, n_qt, tl_idx, tl_mask, tl_count);
    auto issue = [&](int qt, int buf) {
        load_tile<T, D>(sb + buf * 2 * C::TILE_BYTES, qp, p.q_r, qt * kTile, p.Lq, tid);
        load_tile<T, D>(sb + buf * 2 * C::TILE_BYTES + C::TILE_BYTES, dop, p.o_r, qt * kTile, p.Lq, tid);
        if (staged)
            load_bias_tile<T>(sb + bias_off + buf * kBiasStage, b2, p.b2_r, qt * kTile, p.Lq, kt * kTile, p.Lk,
                              static_cast<const T*>(nullptr), tid);
        cp_async_commit();
        if (tid < kTile) {
            const int r = qt * kTile + tid;
            stat[buf * 128 + tid] = r < p.Lq ? lse[r] * kLog2e : INFINITY;
            stat[buf * 128 + 64 + tid] = r < p.Lq ? dl[r] : 0.f;
        }
    };

    float dk[C::ON][4], dv[C::ON][4];
#pragma unroll
    for (int i = 0; i < C::ON; ++i) {
        dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f;
        dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
    }
    float g1_lo = 0.f, g1_hi = 0.f;
    const float sc2 = p.scale * kLog2e;

    int buf = 0;
    if (n_act > 0) issue(tl_idx[0], 0);
    for (int it = 0; it < n_act; ++it) {
        const int qt = tl_idx[it];
        const uint32_t tmask = tl_mask[qt];
        if (it + 1 < n_act) {
            issue(tl_idx[it + 1], buf ^ 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const uint8_t* bst = smem + bias_off + buf * kBiasStage;  // staged pair-bias tile [query in tile][key in tile]
        const uint32_t qb = sb + buf * 2 * C::TILE_BYTES, dob = qb + C::TILE_BYTES;
        const float* st = stat + buf * 128;
        float s[8][4], dp[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
            dp[j][0] = dp[j][1] = dp[j][2] = dp[j][3] = 0.f;
        }
        mma_a_tileT<T, D>(s, kf, qb, lane);    // S^T  [16 keys x 64 queries]
        mma_a_tileT<T, D>(dp, vf, dob, lane);  // dP^T
        uint32_t pa[4][4], da[4][4];
        // full query tile, full key tile, below the causal diagonal for this warp's keys, every layout block on: no masking
        const bool plain = (qt * kTile + kTile <= p.Lq) && (kt * kTile + kTile <= p.Lk) &&
                           !(p.causal && kt * kTile + warp * 16 + 15 > qt * kTile) && all_sub_on(p, tmask);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float pv[4], dsv[4];
            const int qi0 = j * 8 + 2 * t;
            const float2 l2 = *reinterpret_cast<const float2*>(st + qi0), dlt = *reinterpret_cast<const float2*>(st + 64 + qi0);
            float a_lo[2] = {b1_lo, b1_lo}, a_hi[2] = {b1_hi, b1_hi};
            if (b2 != nullptr) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    if (staged) {
                        const T* brow = reinterpret_cast<const T*>(bst + (qi0 + e) * kBiasPitch);
                        a_lo[e] += Mma<T>::to_f(brow[warp * 16 + g]) * kLog2e;
                        a_hi[e] += Mma<T>::to_f(brow[warp * 16 + g + 8]) * kLog2e;
                    } else {
                        const int64_t ro = static_cast<int64_t>(min(qt * kTile + qi0 + e, p.Lq - 1)) * p.b2_r;
                        a_lo[e] += ldb(b2, ro + min(k_lo, p.Lk - 1)) * kLog2e;
                        a_hi[e] += ldb(b2, ro + min(k_hi, p.Lk - 1)) * kLog2e;
                    }
                }
            }
            if (plain) {
                pv[0] = fast_exp2(fmaf(s[j][0], sc2, a_lo[0]) - l2.x);
                pv[1] = fast_exp2(fmaf(s[j][1], sc2, a_lo[1]) - l2.y);
                pv[2] = fast_exp2(fmaf(s[j][2], sc2, a_hi[0]) - l2.x);
                pv[3] = fast_exp2(fmaf(s[j][3], sc2, a_hi[1]) - l2.y);
            } else {
                const bool on = sub_on(p, tmask, j * 8, warp * 16);
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int qrow = qt * kTile + qi0 + e;
                    const bool qin = qrow < p.Lq && on;
                    const bool v_lo = qin && k_lo < p.Lk && !(p.causal && k_lo > qrow);
                    const bool v_hi = qin && k_hi < p.Lk && !(p.causal && k_hi > qrow);
                    pv[e] = v_lo ? fast_exp2(fmaf(s[j][e], sc2, a_lo[e]) - (e ? l2.y : l2.x)) : 0.f;
                    pv[2 + e] = v_hi ? fast_exp2(fmaf(s[j][2 + e], sc2, a_hi[e]) - (e ? l2.y : l2.x)) : 0.f;
                }
            }
            dsv[0] = pv[0] * (dp[j][0] - dlt.x);
            dsv[1] = pv[1] * (dp[j][1] - dlt.y);
            dsv[2] = pv[2] * (dp[j][2] - dlt.x);
            dsv[3] = pv[3] * (dp[j][3] - dlt.y);
            g1_lo += dsv[0] + dsv[1];
            g1_hi += dsv[2] + dsv[3];
            pa[j >> 1][(j & 1) * 2] = Mma<T>::pack(pv[0], pv[1]);
            pa[j >> 1][(j & 1) * 2 + 1] = Mma<T>::pack(pv[2], pv[3]);
            da[j >> 1][(j & 1) * 2] = Mma<T>::pack(dsv[0], dsv[1]);
            da[j >> 1][(j & 1) * 2 + 1] = Mma<T>::pack(dsv[2], dsv[3]);
        }
        mma_p_tile<T, D>(dv, pa, dob, lane);  // dV += P^T dO
        mma_p_tile<T, D>(dk, da, qb, lane);   // dK += dS^T Q
        __syncthreads();
        buf ^= 1;
    }
    T* dkp = static_cast<T*>(p.dk) + nb * p.k_b + h * p.k_h;
    T* dvp = static_cast<T*>(p.dv) + nb * p.v_b + h * p.v_h;
#pragma unroll
    for (int i = 0; i < C::ON; ++i) {
        const int c = i * 8 + 2 * t;
        if (k_lo < p.Lk) {
            *reinterpret_cast<uint32_t*>(dkp + static_cast<int64_t>(k_lo) * p.k_r + c) = Mma<T>::pack(dk[i][0] * p.scale, dk[i][1] * p.scale);
            *reinterpret_cast<uint32_t*>(dvp + static_cast<int64_t>(k_lo) * p.v_r + c) = Mma<T>::pack(dv[i][0], dv[i][1]);
        }
        if (k_hi < p.Lk) {
            *reinterpret_cast<uint32_t*>(dkp + static_cast<int64_t>(k_hi) * p.k_r + c) = Mma<T>::pack(dk[i][2] * p.scale, dk[i][3] * p.scale);
            *reinterpret_cast<uint32_t*>(dvp + static_cast<int64_t>(k_hi) * p.v_r + c) = Mma<T>::pack(dv[i][2], dv[i][3]);
        }
    }
    if (p.db1 != nullptr) {
        g1_lo += __shfl_xor_sync(0xffffffffu, g1_lo, 1);
        g1_lo += __shfl_xor_sync(0xffffffffu, g1_lo, 2);
        g1_hi += __shfl_xor_sync(0xffffffffu, g1_hi, 1);
        g1_hi += __shfl_xor_sync(0xffffffffu, g1_hi, 2);
        if (t == 0) {
            float* gp = p.db1 + nb * p.b1_b;
            if (k_lo < p.Lk) atomicAdd(gp + k_lo, g1_lo);
            if (k_hi < p.Lk) atomicAdd(gp + k_hi, g1_hi);
        }
    }
}

// ---- backward (B): dQ, d(pair bias) -- one CTA per 64 queries ----------------------------------------------------------------------
template <typename T, int D>
__global__ void __launch_bounds__(kThreads) bwd_dq_kernel(const Params p)
{
    using C = Cfg<D>;
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t sb = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int qt = blockIdx.x, h = blockIdx.y, nb = blockIdx.z;
    const int r_lo = qt * kTile + warp * 16 + g, r_hi = r_lo + 8;

    const T* qp = static_cast<const T*>(p.q) + nb * p.q_b + h * p.q_h;
    const T* kp = static_cast<const T*>(p.k) + nb * p.k_b + h * p.k_h;
    const T* vp = static_cast<const T*>(p.v) + nb * p.v_b + h * p.v_h;
    const T* dop = static_cast<const T*>(p.d_o) + nb * p.o_b + h * p.o_h;
    const T* b1 = p.bias1 ? static_cast<const T*>(p.bias1) + nb * p.b1_b : nullptr;
    const T* b2 = p.bias2 ? static_cast<const T*>(p.bias2) + (nb / p.b2_div) * p.b2_b + h * p.b2_h : nullptr;
    float* g2 = p.db2 ? p.db2 + (nb / p.b2_div) * p.g2_b + h * p.g2_h : nullptr;
    const bool g2_vec = (p.Lk & 1) == 0;
    const uint8_t* lay = p.layout ? p.layout + h * p.lay_h : nullptr;
    const int64_t srow = (static_cast<int64_t>(nb) * p.H + h) * p.Lq;
    const float l2_lo = r_lo < p.Lq ? p.lse[srow + r_lo] * kLog2e : INFINITY, l2_hi = r_hi < p.Lq ? p.lse[srow + r_hi] * kLog2e : INFINITY;
    const float dl_lo = r_lo < p.Lq ? p.delta[srow + r_lo] : 0.f, dl_hi = r_hi < p.Lq ? p.delta[srow + r_hi] : 0.f;

    uint32_t qf[C::KS][4], dof[C::KS][4];
    load_a_frag<T, D>(qf, qp, p.q_r, r_lo, p.Lq, t);
    load_a_frag<T, D>(dof, dop, p.o_r, r_lo, p.Lq, t);

    int n_kt = (p.Lk + kTile - 1) / kTile;
    if (p.causal) n_kt = min(n_kt, qt + 1);
    const bool staged = p.stage_bias && (b1 != nullptr || b2 != nullptr);
    const uint32_t bias_off = 4 * C::TILE_BYTES;
    uint8_t* list_base = smem + bias_off + (staged ? 2 * kBiasStage : 0);
    uint16_t* tl_idx = reinterpret_cast<uint16_t*>(list_base);
    uint16_t* tl_mask = tl_idx + p.list_cap;
    int* tl_count = reinterpret_cast<int*>(tl_mask + p.list_cap);
    const int n_act = build_tile_list(p, lay, true, qt, 0, n_kt, tl_idx, tl_mask, tl_count);
    auto issue = [&](int kt, int buf) {
        load_tile<T, D>(sb + buf * 2 * C::TILE_BYTES, kp, p.k_r, kt * kTile, p.Lk, tid);
        load_tile<T, D>(sb + buf * 2 * C::TILE_BYTES + C::TILE_BYTES, vp, p.v_r, kt * kTile, p.Lk, tid);
        if (staged) load_bias_tile<T>(sb + bias_off + buf * kBiasStage, b2, p.b2_r, qt * kTile, p.Lq, kt * kTile, p.Lk, b1, tid);
        cp_async_commit();
    };
    float dq[C::ON][4];
#pragma unroll
    for (int i = 0; i < C::ON; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;
    const float sc2 = p.scale * kLog2e;

    int buf = 0;
    if (n_act > 0) issue(tl_idx[0], 0);
    for (int it = 0; it < n_act; ++it) {
        const int kt = tl_idx[it];
        const uint32_t tmask = tl_mask[kt];
        if (it + 1 < n_act) {
            issue(tl_idx[it + 1], buf ^ 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const uint8_t* bst = smem + bias_off + buf * kBiasStage;
        const uint32_t kb = sb + buf * 2 * C::TILE_BYTES, vb = kb + C::TILE_BYTES;
        float s[8][4], dp[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
            dp[j][0] = dp[j][1] = dp[j][2] = dp[j][3] = 0.f;
        }
        mma_a_tileT<T, D>(s, qf, kb, lane);
        mma_a_tileT<T, D>(dp, dof, vb, lane);
        uint32_t da[4][4];
        auto bias_pair = [&](int j, float2& lo, float2& hi) {  // (bias1 + bias2) * log2 e for cols (c0, c0 + 1), rows lo / hi
            float2 k1 = make_float2(0.f, 0.f);
            lo = hi = k1;
            if (staged) {
                const int cb = (j * 8 + 2 * t) * 2;
                if (b1) k1 = lds_pair<T>(bst + kTile * kBiasPitch + cb);
                if (b2) {
                    lo = lds_pair<T>(bst + (warp * 16 + g) * kBiasPitch + cb);
                    hi = lds_pair<T>(bst + (warp * 16 + g + 8) * kBiasPitch + cb);
                }
            } else {
                const int ca = min(kt * kTile + j * 8 + 2 * t, p.Lk - 1), cb = min(kt * kTile + j * 8 + 2 * t + 1, p.Lk - 1);
                if (b1) k1 = make_float2(ldb(b1, ca), ldb(b1, cb));
                if (b2) {
                    const int64_t ra = static_cast<int64_t>(min(r_lo, p.Lq - 1)) * p.b2_r, rb = static_cast<int64_t>(min(r_hi, p.Lq - 1)) * p.b2_r;
                    lo = make_float2(ldb(b2, ra + ca), ldb(b2, ra + cb));
                    hi = make_float2(ldb(b2, rb + ca), ldb(b2, rb + cb));
                }
            }
            lo.x = (lo.x + k1.x) * kLog2e;
            lo.y = (lo.y + k1.y) * kLog2e;
            hi.x = (hi.x + k1.x) * kLog2e;
            hi.y = (hi.y + k1.y) * kLog2e;
        };
        const bool has_bias = b1 != nullptr || b2 != nullptr;
        // rows past Lq carry lse = +inf (p = 0), so only columns / causality / layout decide whether masking is needed
        const bool plain = (kt * kTile + kTile <= p.Lk) && !(p.causal && kt * kTile + kTile - 1 > qt * kTile + warp * 16) &&
                           all_sub_on(p, tmask);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c0 = kt * kTile + j * 8 + 2 * t;
            float dsv[4];
            float2 lo = make_float2(0.f, 0.f), hi = lo;
            if (has_bias) bias_pair(j, lo, hi);
            bool on = true;
            if (plain) {
                const float p0 = fast_exp2(fmaf(s[j][0], sc2, lo.x) - l2_lo), p1 = fast_exp2(fmaf(s[j][1], sc2, lo.y) - l2_lo);
                const float p2 = fast_exp2(fmaf(s[j][2], sc2, hi.x) - l2_hi), p3 = fast_exp2(fmaf(s[j][3], sc2, hi.y) - l2_hi);
                dsv[0] = p0 * (dp[j][0] - dl_lo);
                dsv[1] = p1 * (dp[j][1] - dl_lo);
                dsv[2] = p2 * (dp[j][2] - dl_hi);
                dsv[3] = p3 * (dp[j][3] - dl_hi);
            } else {
                on = sub_on(p, tmask, warp * 16, j * 8);
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = c0 + e;
                    const bool in = col < p.Lk && on;
                    const bool v_lo = in && r_lo < p.Lq && !(p.causal && col > r_lo);
                    const bool v_hi = in && r_hi < p.Lq && !(p.causal && col > r_hi);
                    const float p_lo = v_lo ? fast_exp2(fmaf(s[j][e], sc2, e ? lo.y : lo.x) - l2_lo) : 0.f;
                    const float p_hi = v_hi ? fast_exp2(fmaf(s[j][2 + e], sc2, e ? hi.y : hi.x) - l2_hi) : 0.f;
                    dsv[e] = p_lo * (dp[j][e] - dl_lo);
                    dsv[2 + e] = p_hi * (dp[j][2 + e] - dl_hi);
                }
            }
            if (g2 != nullptr && on) {
                if (g2_vec) {
                    if (c0 < p.Lk) {
                        if (r_lo < p.Lq) red_add_v2(g2 + static_cast<int64_t>(r_lo) * p.Lk + c0, dsv[0], dsv[1]);
                        if (r_hi < p.Lq) red_add_v2(g2 + static_cast<int64_t>(r_hi) * p.Lk + c0, dsv[2], dsv[3]);
                    }
                } else {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        if (c0 + e < p.Lk) {
                            if (r_lo < p.Lq) atomicAdd(g2 + static_cast<int64_t>(r_lo) * p.Lk + c0 + e, dsv[e]);
                            if (r_hi < p.Lq) atomicAdd(g2 + static_cast<int64_t>(r_hi) * p.Lk + c0 + e, dsv[2 + e]);
                        }
                    }
                }
            }
            da[j >> 1][(j & 1) * 2] = Mma<T>::pack(dsv[0], dsv[1]);
            da[j >> 1][(j & 1) * 2 + 1] = Mma<T>::pack(dsv[2], dsv[3]);
        }
        mma_p_tile<T, D>(dq, da, kb, lane);  // dQ += dS K
        __syncthreads();
        buf ^= 1;
    }
    T* dqp = static_cast<T*>(p.dq) + nb * p.q_b + h * p.q_h;
#pragma unroll
    for (int i = 0; i < C::ON; ++i) {
        const int c = i * 8 + 2 * t;
        if (r_lo < p.Lq)
            *reinterpret_cast<uint32_t*>(dqp + static_cast<int64_t>(r_lo) * p.q_r + c) = Mma<T>::pack(dq[i][0] * p.scale, dq[i][1] * p.scale);
        if (r_hi < p.Lq)
            *reinterpret_cast<uint32_t*>(dqp + static_cast<int64_t>(r_hi) * p.q_r + c) = Mma<T>::pack(dq[i][2] * p.scale, dq[i][3] * p.scale);
    }
}

// bias staging (two stages) + active-tile list (index + mask per tile) + its counter
static int extra_smem(const Params& p) { return (p.stage_bias ? 2 * kBiasStage : 0) + p.list_cap * 4 + 16; }

template <typename T, int D>
int launch_fwd(const Params& p, cudaStream_t stream)
{
    const int smem = 4 * Cfg<D>::TILE_BYTES + extra_smem(p);
    cudaFuncSetAttribute(fwd_kernel<T, D>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    const dim3 grid((p.Lq + kTile - 1) / kTile, p.H, p.NB);
    fwd_kernel<T, D><<<grid, kThreads, smem, stream>>>(p);
    DSB_CHECK_LAUNCH();
    return 0;
}
template <typename T, int D>
int launch_bwd(const Params& p, cudaStream_t stream)
{
    const int64_t rows = static_cast<int64_t>(p.NB) * p.H * p.Lq * (D / 8);
    delta_kernel<T, D><<<static_cast<unsigned>((rows + 255) / 256), 256, 0, stream>>>(p);
    DSB_CHECK_LAUNCH();
    const int smem_a = 4 * Cfg<D>::TILE_BYTES + 2 * 128 * 4 + extra_smem(p), smem_b = 4 * Cfg<D>::TILE_BYTES + extra_smem(p);
    cudaFuncSetAttribute(bwd_dkdv_kernel<T, D>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_a);
    cudaFuncSetAttribute(bwd_dq_kernel<T, D>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_b);
    bwd_dkdv_kernel<T, D><<<dim3((p.Lk + kTile - 1) / kTile, p.H, p.NB), kThreads, smem_a, stream>>>(p);
    DSB_CHECK_LAUNCH();
    bwd_dq_kernel<T, D><<<dim3((p.Lq + kTile - 1) / kTile, p.H, p.NB), kThreads, smem_b, stream>>>(p);
    DSB_CHECK_LAUNCH();
    return 0;
}

template <typename T>
int dispatch(const Params& p, int D, bool bwd, cudaStream_t s)
{
    switch (D) {
        case 16: return bwd ? launch_bwd<T, 16>(p, s) : launch_fwd<T, 16>(p, s);
        case 32: return bwd ? launch_bwd<T, 32>(p, s) : launch_fwd<T, 32>(p, s);
        case 64: return bwd ? launch_bwd<T, 64>(p, s) : launch_fwd<T, 64>(p, s);
        default: return -2;
    }
}

}  // namespace battn
}  // namespace dsb

// `iparams`: NB, H, Lq, Lk, D, dtype, b2_div, lay_bs, lay_nq, lay_nk, causal, backward
// `strides`: q_b q_h q_r  k_b k_h k_r  v_b v_h v_r  o_b o_h o_r  b1_b  b2_b b2_h b2_r  g2_b g2_h  lay_h
DSB_EXPORT int dsb_attn_bias(const void* q, const void* k, const void* v, void* o, float* lse, const void* bias1, const void* bias2,
                             const uint8_t* layout, const void* d_o, void* dq, void* dk, void* dv, float* delta, float* db1, float* db2,
                             const int32_t* iparams, const int64_t* strides, float scale, cudaStream_t stream)
{
    using namespace dsb::battn;
    Params p{};
    p.q = q; p.k = k; p.v = v; p.o = o; p.lse = lse; p.bias1 = bias1; p.bias2 = bias2; p.layout = layout;
    p.d_o = d_o; p.dq = dq; p.dk = dk; p.dv = dv; p.delta = delta; p.db1 = db1; p.db2 = db2;
    p.NB = iparams[0]; p.H = iparams[1]; p.Lq = iparams[2]; p.Lk = iparams[3];
    const int D = iparams[4], dtype = iparams[5];
    p.b2_div = iparams[6] > 0 ? iparams[6] : 1;
    p.lay_bs = iparams[7]; p.lay_nq = iparams[8]; p.lay_nk = iparams[9]; p.causal = iparams[10];
    const bool bwd = iparams[11] != 0;
    const int64_t* s = strides;
    p.q_b = s[0]; p.q_h = s[1]; p.q_r = s[2]; p.k_b = s[3]; p.k_h = s[4]; p.k_r = s[5];
    p.v_b = s[6]; p.v_h = s[7]; p.v_r = s[8]; p.o_b = s[9]; p.o_h = s[10]; p.o_r = s[11];
    p.b1_b = s[12]; p.b2_b = s[13]; p.b2_h = s[14]; p.b2_r = s[15]; p.g2_b = s[16]; p.g2_h = s[17]; p.lay_h = s[18];
    p.scale = scale;
    if (p.NB <= 0 || p.H <= 0 || p.Lq <= 0 || p.Lk <= 0) return 0;
    if (p.H > 65535 || p.NB > 65535) return -3;
    if (layout != nullptr && (p.lay_bs < 16 || (p.lay_bs & (p.lay_bs - 1)) != 0)) return -4;
    p.lay_sh = 6;  // no layout: one always-active block per tile
    if (layout != nullptr) {
        p.lay_sh = 0;
        while ((1 << p.lay_sh) < p.lay_bs) ++p.lay_sh;
    }
    const int n_tiles = (max(p.Lq, p.Lk) + kTile - 1) / kTile;
    if (n_tiles > 8192) return -2;
    p.list_cap = (n_tiles + 7) & ~7;
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    const bool b1_ok = bias1 == nullptr || ((p.Lk & 7) == 0 && (p.b1_b & 7) == 0 && al16(bias1));
    const bool b2_ok = bias2 == nullptr || ((p.Lk & 7) == 0 && ((p.b2_r | p.b2_b | p.b2_h) & 7) == 0 && al16(bias2));
    p.stage_bias = (bias1 != nullptr || bias2 != nullptr) && b1_ok && b2_ok;
    if (dtype == dsb::kBF16) return dispatch<__nv_bfloat16>(p, D, bwd, stream);
    if (dtype == dsb::kF16) return dispatch<__half>(p, D, bwd, stream);
    return -1;
}
