// MoE routing + ragged-batch (continuous batching) device ops for sm_90a.
//   * top_k_gating         : softmax over experts, top-k selection, optional renormalisation, expert histogram
//   * moe_assign_positions : deterministic slot of every (token, k) assignment inside its expert's segment
//   * moe_scatter          : token rows -> expert-major buffer (the producer side of the EP all-to-all)
//   * moe_gather           : weighted un-permute + combine (the consumer side)
//   * ragged_embed         : embedding lookup (+ positional embedding) for a flat token batch
//   * logits_gather        : pick each sequence's last-token hidden state
//   * kv_rotary_append     : RoPE on q/k + append k/v into a paged (blocked) KV cache
//
// Role parity: reference inference/v2/kernels/ragged_ops/{top_k_gating,moe_scatter,moe_gather,embed,
// logits_gather,linear_blocked_kv_rotary}/*.cu (N9b).  These also serve the training MoE layer
// (parallel/moe) instead of the reference's dense einsum dispatch (moe/sharded_moe.py:609).
#include "dsb_common.cuh"

namespace dsb {
namespace moe {

constexpr int kMaxExperts = 256;
constexpr int kMaxTopK = 8;

// One warp per token.  logits [T, E] (T dtype) -> expert ids [T, K], weights [T, K] (fp32), counts [E] (+=).
template <typename T>
__global__ void __launch_bounds__(256)
top_k_gating_kernel(const T* __restrict__ logits, int32_t* __restrict__ expert_ids, float* __restrict__ weights,
                    int32_t* __restrict__ counts, float* __restrict__ probs_out, int tokens, int E, int K, int normalize)
{
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= tokens) return;
    const T* row = logits + static_cast<int64_t>(warp) * E;
    // each lane holds E/32 (<= 8) logits
    float v[kMaxExperts / 32];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < kMaxExperts / 32; ++j) {
        const int e = lane + j * 32;
        v[j] = e < E ? Elem<T>::to_f(row[e]) : -INFINITY;
        mx = fmaxf(mx, v[j]);
    }
    mx = warp_reduce<MaxOp>(mx);
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxExperts / 32; ++j) {
        v[j] = (lane + j * 32) < E ? __expf(v[j] - mx) : 0.f;
        sum += v[j];
    }
    sum = warp_reduce<SumOp>(sum);
    const float inv = 1.f / sum;
    if (probs_out) {
#pragma unroll
        for (int j = 0; j < kMaxExperts / 32; ++j) {
            const int e = lane + j * 32;
            if (e < E) probs_out[static_cast<int64_t>(warp) * E + e] = v[j] * inv;
        }
    }
    // A NaN or +inf logit, or a row without a finite logit, makes the sum NaN (it is >= 1 otherwise) and leaves nothing to
    // rank: the row routes to experts 0..K-1 with NaN weights, so the NaN reaches the layer output and every id and
    // count index stays in range.  `sum` is the same in every lane, so the whole warp takes this branch.
    if (sum != sum) {
        if (lane == 0) {
            for (int k = 0; k < K; ++k) {
                expert_ids[static_cast<int64_t>(warp) * K + k] = k;
                weights[static_cast<int64_t>(warp) * K + k] = __int_as_float(0x7fffffff);
                atomicAdd(counts + k, 1);
            }
        }
        return;
    }
    float wsum = 0.f;
    float wk[kMaxTopK];
    int ek[kMaxTopK];
    for (int k = 0; k < K; ++k) {
        // arg-max across the warp (ties -> lowest expert index)
        float best = -1.f;
        int bi = 0x7fffffff;
#pragma unroll
        for (int j = 0; j < kMaxExperts / 32; ++j) {
            const int e = lane + j * 32;
            if (e < E && (v[j] > best)) {
                best = v[j];
                bi = e;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ob > best || (ob == best && oi < bi)) {
                best = ob;
                bi = oi;
            }
        }
        ek[k] = bi;
        wk[k] = best * inv;
        wsum += wk[k];
        if ((bi & 31) == lane) v[bi >> 5] = -1.f;  // remove the winner
    }
    if (lane == 0) {
        for (int k = 0; k < K; ++k) {
            expert_ids[static_cast<int64_t>(warp) * K + k] = ek[k];
            weights[static_cast<int64_t>(warp) * K + k] = normalize ? wk[k] / wsum : wk[k];
            atomicAdd(counts + ek[k], 1);
        }
    }
}

// Block e walks all T*K assignments in order and numbers the ones routed to expert e: deterministic
// (token-major) ordering inside every expert segment.  positions[t*K+k] = index within its expert.
__global__ void __launch_bounds__(1024)
moe_assign_positions_kernel(const int32_t* __restrict__ expert_ids, int32_t* __restrict__ positions, int n_assign)
{
    __shared__ int warp_sums[32];
    __shared__ int running;
    const int e = blockIdx.x;
    if (threadIdx.x == 0) running = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int base = 0; base < n_assign; base += blockDim.x) {
        const int i = base + threadIdx.x;
        const bool hit = i < n_assign && expert_ids[i] == e;
        const unsigned ballot = __ballot_sync(0xffffffffu, hit);
        const int within = __popc(ballot & ((1u << lane) - 1u));
        if (lane == 0) warp_sums[warp] = __popc(ballot);
        __syncthreads();
        int prefix = 0;
        for (int w = 0; w < warp; ++w) prefix += warp_sums[w];
        if (hit) positions[i] = running + prefix + within;
        __syncthreads();
        if (threadIdx.x == 0) {
            int tot = 0;
            for (int w = 0; w < nw; ++w) tot += warp_sums[w];
            running += tot;
        }
        __syncthreads();
    }
}

// exclusive scan of counts -> offsets (E <= 256, one block)
__global__ void moe_offsets_kernel(const int32_t* __restrict__ counts, int32_t* __restrict__ offsets, int E)
{
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int e = 0; e < E; ++e) {
            offsets[e] = acc;
            acc += counts[e];
        }
        offsets[E] = acc;
    }
}

// out[offsets[e] + pos] = x[token]; mapped_slots[t*K+k] = destination row.  One block per assignment row.
template <typename T>
__global__ void __launch_bounds__(256)
moe_scatter_kernel(const T* __restrict__ x, T* __restrict__ out, const int32_t* __restrict__ expert_ids,
                   const int32_t* __restrict__ positions, const int32_t* __restrict__ offsets,
                   int32_t* __restrict__ mapped_slots, int n_assign, int K, int hidden, int capacity)
{
    constexpr int kPer = Elem<T>::kPerVec;
    const int a = blockIdx.x;
    if (a >= n_assign) return;
    const int e = expert_ids[a];
    const int pos = positions[a];
    const bool dropped = capacity > 0 && pos >= capacity;
    const int dst = dropped ? -1 : (capacity > 0 ? e * capacity + pos : offsets[e] + pos);
    if (threadIdx.x == 0) mapped_slots[a] = dst;
    if (dropped) return;
    const T* src = x + static_cast<int64_t>(a / K) * hidden;
    T* d = out + static_cast<int64_t>(dst) * hidden;
    for (int v = threadIdx.x; v < hidden / kPer; v += blockDim.x) st_plain(d + v * kPer, ld_stream(src + v * kPer));
}

// y[t] = sum_k weights[t,k] * expert_out[mapped_slots[t*K+k]]  (dropped assignments contribute 0)
template <typename T>
__global__ void __launch_bounds__(256)
moe_gather_kernel(const T* __restrict__ expert_out, T* __restrict__ y, const float* __restrict__ weights,
                  const int32_t* __restrict__ mapped_slots, int tokens, int K, int hidden)
{
    constexpr int kPer = Elem<T>::kPerVec;
    const int t = blockIdx.x;
    if (t >= tokens) return;
    for (int v = threadIdx.x; v < hidden / kPer; v += blockDim.x) {
        float acc[kPer];
#pragma unroll
        for (int e = 0; e < kPer; ++e) acc[e] = 0.f;
        for (int k = 0; k < K; ++k) {
            const int slot = mapped_slots[t * K + k];
            if (slot < 0) continue;
            const float w = weights[t * K + k];
            float f[kPer];
            Elem<T>::unpack(ld_stream(expert_out + static_cast<int64_t>(slot) * hidden + v * kPer), f);
#pragma unroll
            for (int e = 0; e < kPer; ++e) acc[e] = fmaf(w, f[e], acc[e]);
        }
        st_plain(y + static_cast<int64_t>(t) * hidden + v * kPer, Elem<T>::pack(acc));
    }
}

// Backward of gather wrt expert_out: d_expert_out[slot] = w * dy[t]; and wrt weights: dw[t,k] = <dy[t], expert_out[slot]>
template <typename T>
__global__ void __launch_bounds__(256)
moe_gather_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ expert_out, T* __restrict__ d_expert_out,
                      float* __restrict__ dweights, const float* __restrict__ weights,
                      const int32_t* __restrict__ mapped_slots, int n_assign, int K, int hidden)
{
    __shared__ float scratch[32];
    constexpr int kPer = Elem<T>::kPerVec;
    const int a = blockIdx.x;
    if (a >= n_assign) return;
    const int slot = mapped_slots[a];
    if (slot < 0) {
        if (threadIdx.x == 0 && dweights) dweights[a] = 0.f;
        return;
    }
    const float w = weights[a];
    const T* g = dy + static_cast<int64_t>(a / K) * hidden;
    float dot = 0.f;
    for (int v = threadIdx.x; v < hidden / kPer; v += blockDim.x) {
        float gf[kPer], of[kPer], o[kPer];
        Elem<T>::unpack(ld_stream(g + v * kPer), gf);
        Elem<T>::unpack(ld_stream(expert_out + static_cast<int64_t>(slot) * hidden + v * kPer), of);
#pragma unroll
        for (int e = 0; e < kPer; ++e) {
            o[e] = w * gf[e];
            dot = fmaf(gf[e], of[e], dot);
        }
        st_plain(d_expert_out + static_cast<int64_t>(slot) * hidden + v * kPer, Elem<T>::pack(o));
    }
    dot = block_reduce<SumOp>(dot, scratch);
    if (threadIdx.x == 0 && dweights) dweights[a] = dot;
}

// ---- ragged batch ops ----------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
ragged_embed_kernel(const int32_t* __restrict__ ids, const int32_t* __restrict__ pos_ids, const T* __restrict__ wte,
                    const T* __restrict__ wpe, T* __restrict__ out, int tokens, int hidden, int pos_offset)
{
    constexpr int kPer = Elem<T>::kPerVec;
    const int t = blockIdx.x;
    if (t >= tokens) return;
    const T* w = wte + static_cast<int64_t>(ids[t]) * hidden;
    const T* p = wpe ? wpe + static_cast<int64_t>(pos_ids[t] + pos_offset) * hidden : nullptr;
    for (int v = threadIdx.x; v < hidden / kPer; v += blockDim.x) {
        float f[kPer];
        Elem<T>::unpack(ld_plain(w + v * kPer), f);
        if (p) {
            float q[kPer];
            Elem<T>::unpack(ld_plain(p + v * kPer), q);
#pragma unroll
            for (int e = 0; e < kPer; ++e) f[e] += q[e];
        }
        st_plain(out + static_cast<int64_t>(t) * hidden + v * kPer, Elem<T>::pack(f));
    }
}

template <typename T>
__global__ void __launch_bounds__(256)
row_gather_kernel(const T* __restrict__ h, const int32_t* __restrict__ idx, T* __restrict__ out, int rows, int hidden)
{
    constexpr int kPer = Elem<T>::kPerVec;
    const int s = blockIdx.x;
    if (s >= rows) return;
    const T* src = h + static_cast<int64_t>(idx[s]) * hidden;
    for (int v = threadIdx.x; v < hidden / kPer; v += blockDim.x)
        st_plain(out + static_cast<int64_t>(s) * hidden + v * kPer, ld_plain(src + v * kPer));
}

template <typename T>
__global__ void __launch_bounds__(256)
row_scatter_add_kernel(const T* __restrict__ src, const int32_t* __restrict__ idx, T* __restrict__ dst, int rows,
                       int hidden, int accumulate)
{
    constexpr int kPer = Elem<T>::kPerVec;
    const int s = blockIdx.x;
    if (s >= rows) return;
    T* d = dst + static_cast<int64_t>(idx[s]) * hidden;
    for (int v = threadIdx.x; v < hidden / kPer; v += blockDim.x) {
        Vec16 val = ld_plain(src + static_cast<int64_t>(s) * hidden + v * kPer);
        if (accumulate) {
            float a[kPer], b[kPer];
            Elem<T>::unpack(val, a);
            Elem<T>::unpack(ld_plain(d + v * kPer), b);
#pragma unroll
            for (int e = 0; e < kPer; ++e) a[e] += b[e];
            val = Elem<T>::pack(a);
        }
        st_plain(d + v * kPer, val);
    }
}

// qkv: [tokens, (hq + 2 hkv) * d] packed.  For token t (sequence seq_of[t], absolute position pos_of[t]):
//   rotate q heads in place, rotate k heads, then write k and v into the paged cache:
//   cache[block_table[seq * max_blocks + pos / block_size]][pos % block_size][0|1][kv_head][d]
template <typename T>
__global__ void __launch_bounds__(256)
kv_rotary_append_kernel(T* __restrict__ qkv, T* __restrict__ cache, const float* __restrict__ cos_t,
                        const float* __restrict__ sin_t, const int32_t* __restrict__ seq_of,
                        const int32_t* __restrict__ pos_of, const int32_t* __restrict__ block_table, int tokens, int hq,
                        int hkv, int d, int rot_dim, int block_size, int max_blocks)
{
    const int t = blockIdx.x;
    if (t >= tokens) return;
    const int pos = pos_of[t];
    const int seq = seq_of[t];
    const int blk = block_table[seq * max_blocks + pos / block_size];
    const int slot = pos % block_size;
    T* row = qkv + static_cast<int64_t>(t) * (hq + 2 * hkv) * d;
    const int half = rot_dim / 2;
    // rotate q and k heads (pairs i, i+half)
    const int n_rot_heads = hq + hkv;
    for (int i = threadIdx.x; i < n_rot_heads * half; i += blockDim.x) {
        const int h = i / half, j = i % half;
        T* base = row + static_cast<int64_t>(h) * d;
        const float a = Elem<T>::to_f(base[j]), b = Elem<T>::to_f(base[j + half]);
        const float c = cos_t[static_cast<int64_t>(pos) * half + j], s = sin_t[static_cast<int64_t>(pos) * half + j];
        // explicit fmas: the rounding is fixed by the source, not by the compiler's contraction choices
        base[j] = Elem<T>::from_f(fmaf(a, c, -(b * s)));
        base[j + half] = Elem<T>::from_f(fmaf(b, c, a * s));
    }
    __syncthreads();
    // append k, v
    T* cbase = cache + (static_cast<int64_t>(blk) * block_size + slot) * 2 * hkv * d;
    const T* k = row + static_cast<int64_t>(hq) * d;
    for (int i = threadIdx.x; i < 2 * hkv * d; i += blockDim.x) cbase[i] = k[i];  // k heads then v heads, contiguous
}

}  // namespace moe
}  // namespace dsb

using namespace dsb;
using namespace dsb::moe;

#define DISPATCH_MT(code, T, ...)  \
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

DSB_EXPORT int dsb_top_k_gating(const void* logits, int32_t* expert_ids, float* weights, int32_t* counts,
                                float* probs_out, int tokens, int E, int K, int normalize, int dtype,
                                cudaStream_t stream)
{
    if (tokens <= 0) return 0;
    if (E > kMaxExperts || K > kMaxTopK || K > E) return -2;
    const int grid = (tokens * 32 + 255) / 256;
    DISPATCH_MT(dtype, T, {
        top_k_gating_kernel<T><<<grid, 256, 0, stream>>>((const T*)logits, expert_ids, weights, counts, probs_out, tokens, E,
                                                          K, normalize);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_moe_assign_positions(const int32_t* expert_ids, const int32_t* counts, int32_t* positions,
                                        int32_t* offsets, int n_assign, int E, cudaStream_t stream)
{
    if (E > kMaxExperts) return -2;
    if (n_assign > 0) moe_assign_positions_kernel<<<E, 1024, 0, stream>>>(expert_ids, positions, n_assign);
    moe_offsets_kernel<<<1, 32, 0, stream>>>(counts, offsets, E);
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_moe_scatter(const void* x, void* out, const int32_t* expert_ids, const int32_t* positions,
                               const int32_t* offsets, int32_t* mapped_slots, int n_assign, int K, int hidden,
                               int capacity, int dtype, cudaStream_t stream)
{
    if (n_assign <= 0) return 0;
    const int per = dtype == kF32 ? 4 : 8;
    if (hidden % per) return -2;
    DISPATCH_MT(dtype, T, {
        moe_scatter_kernel<T><<<n_assign, 256, 0, stream>>>((const T*)x, (T*)out, expert_ids, positions, offsets,
                                                             mapped_slots, n_assign, K, hidden, capacity);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_moe_gather(const void* expert_out, void* y, const float* weights, const int32_t* mapped_slots,
                              int tokens, int K, int hidden, int dtype, cudaStream_t stream)
{
    if (tokens <= 0) return 0;
    const int per = dtype == kF32 ? 4 : 8;
    if (hidden % per) return -2;
    DISPATCH_MT(dtype, T, {
        moe_gather_kernel<T><<<tokens, 256, 0, stream>>>((const T*)expert_out, (T*)y, weights, mapped_slots, tokens, K,
                                                          hidden);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_moe_gather_bwd(const void* dy, const void* expert_out, void* d_expert_out, float* dweights,
                                  const float* weights, const int32_t* mapped_slots, int n_assign, int K, int hidden,
                                  int dtype, cudaStream_t stream)
{
    if (n_assign <= 0) return 0;
    const int per = dtype == kF32 ? 4 : 8;
    if (hidden % per) return -2;
    DISPATCH_MT(dtype, T, {
        moe_gather_bwd_kernel<T><<<n_assign, 256, 0, stream>>>((const T*)dy, (const T*)expert_out, (T*)d_expert_out,
                                                                dweights, weights, mapped_slots, n_assign, K, hidden);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_ragged_embed(const int32_t* ids, const int32_t* pos_ids, const void* wte, const void* wpe, void* out,
                                int tokens, int hidden, int pos_offset, int dtype, cudaStream_t stream)
{
    if (tokens <= 0) return 0;
    const int per = dtype == kF32 ? 4 : 8;
    if (hidden % per) return -2;
    DISPATCH_MT(dtype, T, {
        ragged_embed_kernel<T><<<tokens, 256, 0, stream>>>(ids, pos_ids, (const T*)wte, (const T*)wpe, (T*)out, tokens,
                                                            hidden, pos_offset);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_row_gather(const void* h, const int32_t* idx, void* out, int rows, int hidden, int dtype,
                              cudaStream_t stream)
{
    if (rows <= 0) return 0;
    const int per = dtype == kF32 ? 4 : 8;
    if (hidden % per) return -2;
    DISPATCH_MT(dtype, T, { row_gather_kernel<T><<<rows, 256, 0, stream>>>((const T*)h, idx, (T*)out, rows, hidden); })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_row_scatter(const void* src, const int32_t* idx, void* dst, int rows, int hidden, int accumulate,
                               int dtype, cudaStream_t stream)
{
    if (rows <= 0) return 0;
    const int per = dtype == kF32 ? 4 : 8;
    if (hidden % per) return -2;
    DISPATCH_MT(dtype, T, {
        row_scatter_add_kernel<T><<<rows, 256, 0, stream>>>((const T*)src, idx, (T*)dst, rows, hidden, accumulate);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}

DSB_EXPORT int dsb_kv_rotary_append(void* qkv, void* cache, const float* cos_t, const float* sin_t, const int32_t* seq_of,
                                    const int32_t* pos_of, const int32_t* block_table, int tokens, int hq, int hkv, int d,
                                    int rot_dim, int block_size, int max_blocks, int dtype, cudaStream_t stream)
{
    if (tokens <= 0) return 0;
    DISPATCH_MT(dtype, T, {
        kv_rotary_append_kernel<T><<<tokens, 256, 0, stream>>>((T*)qkv, (T*)cache, cos_t, sin_t, seq_of, pos_of,
                                                                block_table, tokens, hq, hkv, d, rot_dim, block_size,
                                                                max_blocks);
    })
    DSB_CHECK_LAUNCH();
    return 0;
}
