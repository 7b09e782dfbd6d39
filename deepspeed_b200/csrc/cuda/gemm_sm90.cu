// Hand-written sm_90a GEMM: C[M,N] (bf16) = op(A)[M,K] x op(B)[N,K]^T, bf16 operands, fp32 accumulate.
//
//   * operands staged global -> shared by TMA (cp.async.bulk.tensor, 128-byte swizzle) through a 4-stage mbarrier ring;
//     every operand box is [64 rows x 64 bf16], so K-major ([rows, k]) and MN-major ([k, rows]) operands share one ring
//   * two consumer warpgroups each own 64 rows of the 128 x 256 tile and issue wgmma.m64n256k16 straight from the shared
//     tiles (MN-major operands through the transpose bits), 128 fp32 accumulators per thread; a producer warpgroup hands
//     its registers to the consumers (setmaxnreg) and one of its threads issues the TMA
//   * persistent CTAs (one per SM) walk the tile list; the producer runs ahead into the next tile while the consumers
//     run the epilogue of the current one
//   * fused epilogues: plain store, accumulate into C (dW over micro-batches), SwiGLU (gate and up rows of the same 128
//     features share one tile), dSwiGLU
//   * grouped (MoE) form: the tile list is built on the device from the expert offsets (no host synchronisation)
//   * ragged (dropless MoE training) forms: the grouped form with every epilogue and an MN-major B whose expert offset
//     lies on K, plus a variable-K weight-gradient form whose tile (expert, m, n) sums only its expert's rows
//   * tensorwise- or blockwise-scaled FP8 form (gemm_fp8_kernel, dsb_gemm_fp8 / dsb_gemm_fp8_block): e4m3 / e5m2 K-major
//     operands, 128 x 128 tiles, every 128-product k-block promoted into an fp32 accumulator, the same epilogues; and
//     its ragged forms (dsb_gemm_fp8_ragged / dsb_gemm_fp8_ragged_wgrad) on the same tile walk, with 128-row segments
//   * OPTIONAL fused all-gather: when `ag` is given, the weight matrix B is being assembled in local memory from the
//     other ranks' ZeRO shards *by this same kernel*: `ag.comm_ctas` CTAs pull the peers' shard bytes over NVLink
//     (peer-mapped addresses) chunk by chunk and publish a per-chunk ready flag (st.release.gpu); the producer of each
//     MMA CTA acquires the flag of the chunk(s) backing a B tile before loading it, and tiles are visited starting with
//     the locally owned rows, so transfer and math overlap tile by tile with no NCCL call.
//
// The reference has no tensor-core GEMM of its own for training (cuBLAS via csrc/transformer/
// cublas_wrappers.cu:65 or torch.matmul); this kernel is the framework's native path.
#include "dsb_tc.cuh"

namespace dsb {
namespace gemm {
using namespace dsb::tc;

constexpr int BM = 128, BN = 256, BK = 64;
constexpr int STAGES = 4;
constexpr int kConsumerThreads = 256;                 // two warpgroups, 64 rows each
constexpr int kThreads = kConsumerThreads + 128;      // + the producer warpgroup
constexpr int kProducerRegs = 40, kConsumerRegs = 232;  // 128 x 40 + 256 x 232 <= 64 K registers
constexpr uint32_t BOX = 64 * 64 * 2;                 // one TMA box: 8 KiB
constexpr uint32_t STAGE_BYTES = 6 * BOX;             // A: 2 boxes, B: 4 boxes
constexpr uint32_t SMEM_BAR = STAGES * STAGE_BYTES;   // 192 KiB (also the all-gather ring: 3 x 64 KiB)
constexpr int kMaxGroups = 256;
constexpr uint32_t SMEM_GRP = SMEM_BAR + 256;         // grouped form: int tile_prefix[kMaxGroups + 1]
constexpr uint32_t SMEM_TOTAL = SMEM_GRP + (kMaxGroups + 1) * 4 + 1024;

__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read()
{
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---- fused all-gather descriptor ------------------------------------------------------------------------
struct AgParams {
    // B (= this unit's gathered weights) lives in `local_full`; rank p's shard is `shard_bytes` long and is
    // found at peers[p] (peer-mapped VA).  Chunk c covers bytes [c*chunk_bytes, (c+1)*chunk_bytes) of the
    // unit's flat buffer; flags[c] becomes `epoch` once the chunk is resident in local_full.
    const void* peers[8];
    void* local_full;
    uint32_t* flags;
    int64_t shard_bytes;
    int64_t chunk_bytes;
    int64_t b_offset_bytes;  // byte offset of B's first element inside the unit flat buffer
    int64_t b_bytes;         // extent of B: its chunks are gathered FIRST so the multiply can start while the rest streams
    int n_chunks;
    int world;
    int rank;
    int comm_ctas;  // trailing CTAs of the grid that do the gathering
    uint32_t epoch;
    int enabled;
};

__device__ __forceinline__ uint32_t ld_acquire_gpu_u32(const uint32_t* p)
{
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu_u32(uint32_t* p, uint32_t v)
{
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Gather role: CTA `ci` of `nc` copies chunks ci, ci+nc, ... in the order "own shard first, then rank+1, ...".
// The copy is done by the TMA engine, not by SM load/store instructions: one elected thread streams each chunk through a
// ring of 3 x 64 KiB shared-memory buffers with  cp.async.bulk (peer global -> smem, mbarrier complete_tx)  followed by
// cp.async.bulk (smem -> local global, bulk_group);  192 KiB in flight per CTA hides the NVLink round trip, so a dozen
// gather CTAs saturate the links while leaving their SMs' issue slots idle.
constexpr uint32_t AG_PIECE = 64 * 1024;
constexpr int AG_BUFS = 3;

__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src_smem, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src_smem), "r"(bytes)
                 : "memory");
}

__device__ void ag_gather_role(const AgParams& ag, int ci, int nc, uint8_t* smem)
{
    if (threadIdx.x != 0) return;
    const uint32_t sbase = smem_u32(smem);
    const uint32_t bar0 = sbase + AG_BUFS * AG_PIECE;  // AG_BUFS mbarriers after the ring
    for (int b = 0; b < AG_BUFS; ++b) mbar_init(bar0 + 8 * b, 1);
    fence_barrier_init();
    const int chunks_per_shard = static_cast<int>(ag.shard_bytes / ag.chunk_bytes);
    // chunks holding the matrix this very kernel multiplies by go first (pass 0), the rest of the unit follows (pass 1)
    const int b_c0 = static_cast<int>(ag.b_offset_bytes / ag.chunk_bytes);
    const int b_c1 = static_cast<int>((ag.b_offset_bytes + ag.b_bytes - 1) / ag.chunk_bytes);
    uint32_t issued = 0;           // pieces issued so far (ring position = issued % AG_BUFS)
    for (int pass = 0; pass < 2; ++pass)
    for (int j = ci; j < ag.n_chunks; j += nc) {
        // visit order: shards rotated so that every rank starts pulling from a different peer
        const int k = j / chunks_per_shard;
        const int within = j - k * chunks_per_shard;
        const int peer = (ag.rank + k) % ag.world;
        const int chunk = peer * chunks_per_shard + within;
        if ((chunk >= b_c0 && chunk <= b_c1) != (pass == 0)) continue;
        const int64_t off = static_cast<int64_t>(within) * ag.chunk_bytes;
        const char* src = static_cast<const char*>(ag.peers[peer]) + off;
        char* dst = static_cast<char*>(ag.local_full) + static_cast<int64_t>(peer) * ag.shard_bytes + off;
        const int n_pieces = static_cast<int>((ag.chunk_bytes + AG_PIECE - 1) / AG_PIECE);
        // software pipeline inside the chunk: loads run AG_BUFS-1 pieces ahead of the stores
        int loaded = 0, stored = 0;
        uint32_t first = issued;
        while (stored < n_pieces) {
            while (loaded < n_pieces && loaded - stored < AG_BUFS) {
                const uint32_t slot = (first + loaded) % AG_BUFS;
                // the store that last read this slot must have finished reading shared memory
                if (first + loaded >= static_cast<uint32_t>(AG_BUFS)) tma_store_wait_read<0>();
                const int64_t po = static_cast<int64_t>(loaded) * AG_PIECE;
                const int64_t rem = ag.chunk_bytes - po;
                const uint32_t bytes = static_cast<uint32_t>(rem < static_cast<int64_t>(AG_PIECE) ? rem : AG_PIECE);
                mbar_expect_tx(bar0 + 8 * slot, bytes);
                bulk_g2s(sbase + slot * AG_PIECE, src + po, bytes, bar0 + 8 * slot);
                ++loaded;
            }
            const uint32_t n = first + stored;
            const uint32_t slot = n % AG_BUFS;
            mbar_wait(bar0 + 8 * slot, (n / AG_BUFS) & 1);
            const int64_t po = static_cast<int64_t>(stored) * AG_PIECE;
            const int64_t rem2 = ag.chunk_bytes - po;
            const uint32_t bytes = static_cast<uint32_t>(rem2 < static_cast<int64_t>(AG_PIECE) ? rem2 : AG_PIECE);
            bulk_s2g(dst + po, sbase + slot * AG_PIECE, bytes);
            tma_store_commit();
            ++stored;
        }
        issued = first + n_pieces;
        tma_store_wait_all();  // the chunk's bytes are written before the flag is published
        __threadfence();
        st_release_gpu_u32(ag.flags + chunk, ag.epoch);
    }
}

// Wait until every chunk overlapping B rows [n0, n0+rows) is resident.
__device__ __forceinline__ void ag_wait_rows(const AgParams& ag, int n0, int rows, int K)
{
    const int64_t lo = ag.b_offset_bytes + static_cast<int64_t>(n0) * K * 2;
    const int64_t hi = lo + static_cast<int64_t>(rows) * K * 2;
    int c0 = static_cast<int>(lo / ag.chunk_bytes);
    int c1 = static_cast<int>((hi - 1) / ag.chunk_bytes);
    if (c1 >= ag.n_chunks) c1 = ag.n_chunks - 1;
    for (int c = c0; c <= c1; ++c) {
        while (ld_acquire_gpu_u32(ag.flags + c) != ag.epoch) __nanosleep(64);
    }
    // the chunk was written through the async proxy (bulk copies) and is about to be read through it (TMA loads)
    asm volatile("fence.proxy.async;" ::: "memory");
}

static_assert(AG_BUFS * AG_PIECE + 8 * AG_BUFS <= SMEM_TOTAL, "all-gather ring must fit the GEMM's shared memory");

// ---- fused epilogues ------------------------------------------------------------------------------------------
// EPI_STORE    C = acc
// EPI_ACCUM    C = C + acc                                   (dW accumulation over micro-batches: no addmm, no memset)
// EPI_SWIGLU   B = [gate; up] stacked ([2I, K]); a tile multiplies 128 gate rows and the matching 128 up rows so
//              accumulator columns 0-127 / 128-255 are gate / up of the SAME 128 features:  C[M, I] = silu(gate) * up,
//              optionally gate|up saved to out2 [M, 2I] for backward.
// EPI_DSWIGLU  acc = d_act tile (dY W_down); aux = saved gate|up [M, 2I]:
//              dgate = acc * up * silu'(gate) -> C (the [M, I] left half of dgate_up),  dup = acc * silu(gate) -> out2 + I.
// (cuBLAS cannot express the last two: they remove one full pass over the [tokens, 2I] / [tokens, I] activations each.)
enum : int { EPI_STORE = 0, EPI_ACCUM = 1, EPI_SWIGLU = 2, EPI_DSWIGLU = 3 };
// MODE_GROUPED    m-tiles per expert over expert-sorted rows, K-major B [E, N, K] (inference, offsets trusted)
// MODE_RAGGED     MODE_GROUPED for training: 64-row aligned segments, checked offsets, SwiGLU / dSwiGLU epilogues and an
//                 MN-major B [E, K, N] (the expert's slab starts at K coordinate e * K)
// MODE_RAGGED_K   dW[e] = A_e^T B_e over the rows of expert e only: tiles (e, m, n), k-blocks [off[e] / 64, off[e+1] / 64)
enum : int { MODE_PLAIN = 0, MODE_GROUPED = 1, MODE_ALLGATHER = 2, MODE_RAGGED = 3, MODE_RAGGED_K = 4 };

struct EpiParams {
    const __nv_bfloat16* aux;  // DSWIGLU: saved gate|up
    __nv_bfloat16* out2;       // SWIGLU: gate|up save (nullable); DSWIGLU: dgate_up base (dup goes to + inter)
    __nv_bfloat16* c;          // output
    int ld_aux, ld_out2, ldc;
    int inter;                 // I
    int group_m;               // rasterisation: m-blocks per L2 super-group
    const int* offsets;        // grouped: expert row offsets [E + 1] on the device
    int E;
};

__device__ __forceinline__ float silu_f(float g) { return g / (1.f + __expf(-g)); }
__device__ __forceinline__ float dsilu_f(float g)
{
    const float sg = 1.f / (1.f + __expf(-g));
    return sg * (1.f + g * (1.f - sg));
}

// Grouped rasterisation: tiles are numbered so that `group_m` consecutive m-blocks share every n-block before the next
// group starts -- one wave of CTAs then touches ~group_m A-blocks and ~CTAs/group_m B-blocks instead of all A-blocks
// and a few B-blocks, which keeps the wave's operand set inside L2 for the wide (N = 28672 / 128256) problems.
__device__ __forceinline__ void tile_coords(int tile, int num_m, int num_n, int group_m, int& m_blk, int& n_blk)
{
    const int per_group = group_m * num_n;
    const int g = tile / per_group;
    const int first_m = g * group_m;
    const int gm = (num_m - first_m) < group_m ? (num_m - first_m) : group_m;
    const int local = tile - g * per_group;
    m_blk = first_m + local % gm;
    n_blk = local / gm;
}

__device__ __forceinline__ float2 ld_bf16x2(const __nv_bfloat16* p)
{
    return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p));
}
__device__ __forceinline__ void st_bf16x2(__nv_bfloat16* p, float lo, float hi)
{
    *reinterpret_cast<uint32_t*>(p) = pack_bf16(lo, hi);
}

// Where one tile lives: first row of A / C, rows of C it may write, first B row of each half of the B tile (K-major B:
// each half is two 64-row boxes), first C column (MN-major B: also the first B column).  Ragged forms only: k0 is added
// to the K coordinate of the MN-major operands' loads, nk is the tile's k-block count and crow0 its first C row.
struct Tile {
    int row0, rows, b0, b1, col0;
    int k0, nk, crow0;
};

// Ragged forms: offsets[0..E] must be non-decreasing multiples of the segment granule GRAN (the kernel's k-block: 64 rows
// bf16, 128 rows FP8) inside [0, rows].  Anything else could send a TMA load into another expert's K rows or a store
// past the output, so the kernel refuses it before it does anything.
// kPrefix (m-tiled form): the same pass fills prefix[1..E] with the running count of (m-tile x nn n-tiles).
template <bool kPrefix, int GRAN>
__device__ __forceinline__ bool ragged_walk(const int* off, int E, int rows, int nn, int* prefix)
{
    int prev = off[0];
    if (prev < 0 || (prev & (GRAN - 1))) return false;
    int acc = 0;
    for (int e = 1; e <= E; ++e) {
        const int cur = off[e];
        if (cur < prev || (cur & (GRAN - 1))) return false;
        if (kPrefix) {
            acc += ((cur - prev + BM - 1) / BM) * nn;
            prefix[e] = acc;
        }
        prev = cur;
    }
    return prev <= rows;
}

// TBN: B rows per tile (256 bf16, 128 FP8); KB: rows per k-block of the variable-K form (= the segment granule).
template <int EPI, int MODE, int TBN = BN, int KB = BK>
struct Sched {
    static constexpr bool kGrouped = MODE == MODE_GROUPED || MODE == MODE_RAGGED;  // m-tiles per expert
    static constexpr int TN = (EPI == EPI_SWIGLU) ? TBN / 2 : TBN;  // output columns per tile
    int num_m, num_n, num_tiles, group_m, n_rot, M, N, K;
    const int* offsets;
    const int* prefix;  // grouped: tile_prefix in shared memory
    int e;              // grouped: current expert (tiles are visited in increasing order)

    __device__ void init(const EpiParams& ep, const AgParams& ag, int M_, int N_, int K_, const int* pre)
    {
        M = M_;
        N = N_;
        num_n = (N + TN - 1) / TN;
        offsets = ep.offsets;
        prefix = pre;
        e = 0;
        n_rot = 0;
        if (MODE == MODE_RAGGED) K = K_;
        if (kGrouped) {
            num_m = 0;
            num_tiles = pre[ep.E];
            group_m = 1;
        } else if (MODE == MODE_RAGGED_K) {
            num_m = (M + BM - 1) / BM;
            num_tiles = ep.E * num_m * num_n;
            group_m = num_m;
        } else {
            num_m = (M + BM - 1) / BM;
            num_tiles = num_m * num_n;
            group_m = (MODE == MODE_PLAIN && ep.group_m > 0) ? ep.group_m : num_m;
        }
        if (MODE == MODE_ALLGATHER) {
            // n-blocks are visited starting at the locally owned rows
            const int64_t own_lo = static_cast<int64_t>(ag.rank) * ag.shard_bytes - ag.b_offset_bytes;
            int64_t row = own_lo > 0 ? (own_lo + static_cast<int64_t>(K_) * 2 - 1) / (static_cast<int64_t>(K_) * 2) : 0;
            n_rot = static_cast<int>((row + BN - 1) / BN) % num_n;
        }
    }
    __device__ Tile at(int tile, int inter)
    {
        Tile t;
        int m_blk, n_blk;
        if (kGrouped) {
            while (tile >= prefix[e + 1]) ++e;
            const int lo = offsets[e], cnt = offsets[e + 1] - lo;
            const int nm = (cnt + BM - 1) / BM;
            const int local = tile - prefix[e];
            m_blk = local % nm;
            n_blk = local / nm;
            t.row0 = lo + m_blk * BM;
            t.rows = cnt - m_blk * BM;
            t.col0 = n_blk * TN;
            if (MODE == MODE_RAGGED && EPI == EPI_SWIGLU) {
                // w13 [E, 2I, K]: the expert's gate rows, then its up rows
                t.b0 = e * 2 * inter + t.col0;
                t.b1 = t.b0 + inter;
            } else {
                t.b0 = e * N + t.col0;
                t.b1 = t.b0 + TBN / 2;
            }
            if (MODE == MODE_RAGGED) t.k0 = e * K;  // MN-major B [E, K, N]
            return t;
        }
        if (MODE == MODE_RAGGED_K) {
            const int per_e = num_m * num_n;
            e = tile / per_e;
            const int local = tile - e * per_e;
            m_blk = local % num_m;
            n_blk = local / num_m;
            t.row0 = m_blk * BM;
            t.rows = M - t.row0;
            t.col0 = n_blk * TBN;
            t.crow0 = e * M + t.row0;
            t.k0 = offsets[e];
            t.nk = (offsets[e + 1] - t.k0) / KB;
            return t;
        }
        tile_coords(tile, num_m, num_n, group_m, m_blk, n_blk);
        if (MODE == MODE_ALLGATHER) n_blk = (n_blk + n_rot) % num_n;
        t.row0 = m_blk * BM;
        t.rows = M - t.row0;
        t.col0 = n_blk * TN;
        t.b0 = t.col0;
        t.b1 = (EPI == EPI_SWIGLU) ? inter + t.col0 : t.col0 + TBN / 2;
        return t;
    }
};

template <bool A_MN, bool B_MN, int EPI, int MODE>
__global__ void __launch_bounds__(kThreads, 1)
gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, int M, int N, int K,
            const EpiParams ep, const AgParams ag)
{
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment required by SWIZZLE_128B
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const uint32_t sbase = smem_u32(smem);
    const uint32_t bar_base = sbase + SMEM_BAR;
    auto full_bar = [&](int s) { return bar_base + 8 * s; };
    auto empty_bar = [&](int s) { return bar_base + 8 * (STAGES + s); };
    int* tile_prefix = reinterpret_cast<int*>(smem + SMEM_GRP);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int mma_ctas = MODE == MODE_ALLGATHER ? static_cast<int>(gridDim.x) - ag.comm_ctas : static_cast<int>(gridDim.x);

    if (MODE == MODE_ALLGATHER && static_cast<int>(blockIdx.x) >= mma_ctas) {
        ag_gather_role(ag, static_cast<int>(blockIdx.x) - mma_ctas, ag.comm_ctas, smem);
        return;
    }

    if constexpr (MODE == MODE_RAGGED || MODE == MODE_RAGGED_K) {
        // one pass over the offsets checks them (and, m-tiled, builds the tile prefix); tile_prefix[0] is 0 when they are
        // well formed, -1 when not -- then the whole CTA leaves before any barrier exists and writes nothing
        if (threadIdx.x == kConsumerThreads) {
            const int nn = (N + Sched<EPI, MODE>::TN - 1) / Sched<EPI, MODE>::TN;
            tile_prefix[0] = ragged_walk<MODE == MODE_RAGGED, BK>(ep.offsets, ep.E, MODE == MODE_RAGGED ? M : K, nn,
                                                                  tile_prefix)
                                 ? 0
                                 : -1;
        }
        __syncthreads();
        if (tile_prefix[0] != 0) return;
    }

    if (threadIdx.x == kConsumerThreads) {
        prefetch_map(&map_a);
        prefetch_map(&map_b);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), kConsumerThreads / 32);  // one arrival per consumer warp
        }
        fence_barrier_init();
        if (MODE == MODE_GROUPED) {
            const int nn = (N + Sched<EPI, MODE>::TN - 1) / Sched<EPI, MODE>::TN;
            int acc = 0;
            tile_prefix[0] = 0;
            for (int e = 0; e < ep.E; ++e) {
                const int cnt = ep.offsets[e + 1] - ep.offsets[e];
                acc += ((cnt + BM - 1) / BM) * nn;
                tile_prefix[e + 1] = acc;
            }
        }
    }
    __syncthreads();

    Sched<EPI, MODE> sch;
    sch.init(ep, ag, M, N, K, tile_prefix);
    const int num_k = (K + BK - 1) / BK;

    if (threadIdx.x >= kConsumerThreads) {
        // ===================== TMA producer warpgroup =====================
        setmaxnreg_dec<kProducerRegs>();
        if (threadIdx.x == kConsumerThreads) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < sch.num_tiles; tile += mma_ctas) {
                const Tile t = sch.at(tile, ep.inter);
                if (MODE == MODE_ALLGATHER) ag_wait_rows(ag, t.col0, (N - t.col0) < BN ? (N - t.col0) : BN, K);
                const int nk = MODE == MODE_RAGGED_K ? t.nk : num_k;
                for (int kb = 0; kb < nk; ++kb) {
                    mbar_wait(empty_bar(stage), phase ^ 1);
                    const uint32_t sa = sbase + stage * STAGE_BYTES, sb = sa + 2 * BOX;  // B: 4 boxes of 64 rows
                    const uint32_t fb = full_bar(stage);
                    mbar_expect_tx(fb, STAGE_BYTES);
                    const int ka = kb * BK + (MODE == MODE_RAGGED_K ? t.k0 : 0);
                    const int kbb = kb * BK + (MODE == MODE_RAGGED_K || (MODE == MODE_RAGGED && B_MN) ? t.k0 : 0);
                    if (A_MN) {
                        tma_load_2d(sa, &map_a, fb, t.row0, ka);
                        tma_load_2d(sa + BOX, &map_a, fb, t.row0 + 64, ka);
                    } else {
                        tma_load_2d(sa, &map_a, fb, ka, t.row0);
                        tma_load_2d(sa + BOX, &map_a, fb, ka, t.row0 + 64);
                    }
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        if (B_MN) tma_load_2d(sb + i * BOX, &map_b, fb, t.col0 + 64 * i, kbb);
                        else tma_load_2d(sb + i * BOX, &map_b, fb, kbb, (i < 2 ? t.b0 : t.b1) + 64 * (i & 1));
                    }
                    if (++stage == STAGES) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
        return;
    }

    // ===================== consumers: warpgroup `wg` owns rows [64 wg, 64 wg + 64) of the tile =====================
    setmaxnreg_inc<kConsumerRegs>();
    const int wg = threadIdx.x >> 7;
    const int r_in = 64 * wg + 16 * (warp & 3) + (lane >> 2);  // first of this thread's two rows (+8)
    const int c_in = 2 * (lane & 3);                             // first of this thread's column pairs (+8 j)
    int stage = 0;
    uint32_t phase = 0;
    float acc[128];
    for (int tile = blockIdx.x; tile < sch.num_tiles; tile += mma_ctas) {
        const Tile t = sch.at(tile, ep.inter);
        const int nk = MODE == MODE_RAGGED_K ? t.nk : num_k;
        int prev = -1;
        for (int kb = 0; kb < nk; ++kb) {
            mbar_wait(full_bar(stage), phase);
            const uint32_t sa = sbase + stage * STAGE_BYTES + wg * BOX, sb = sbase + stage * STAGE_BYTES + 2 * BOX;
            const uint64_t da = A_MN ? desc_mnmajor_sw128(sa, BOX) : desc_kmajor_sw128(sa);
            const uint64_t db = B_MN ? desc_mnmajor_sw128(sb, BOX) : desc_kmajor_sw128(sb);
            // per 16-element K step: K-major advances 32 B inside the swizzle row, MN-major 16 k-rows = 2 KiB
            constexpr uint64_t ka = A_MN ? (2048 >> 4) : (32 >> 4);
            constexpr uint64_t kbs = B_MN ? (2048 >> 4) : (32 >> 4);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; ++k)
                wgmma_m64n256k16_ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da + ka * k, db + kbs * k, (kb > 0 || k > 0) ? 1 : 0);
            wgmma_commit();
            wgmma_wait<1>();  // the previous stage's products have retired: hand its buffers back
            if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
            prev = stage;
            if (++stage == STAGES) {
                stage = 0;
                phase ^= 1;
            }
        }
        wgmma_wait<0>();
        fence_regs<128>(acc);
        if (prev >= 0 && lane == 0) mbar_arrive(empty_bar(prev));
        if constexpr (MODE == MODE_RAGGED_K) {
            // an expert without rows: no wgmma initialised the accumulators; its dW is zero (STORE) or unchanged (ACCUM)
            if (nk == 0) {
                if constexpr (EPI == EPI_ACCUM) {
                    continue;
                } else {
#pragma unroll
                    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
                }
            }
        }

        // ---- epilogue straight from the accumulators: thread holds rows r_in (+8), column pairs c_in + 8 j ----
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int lr = r_in + 8 * i;
            if (lr >= t.rows || lr >= BM) continue;
            const int64_t grow = static_cast<int64_t>((MODE == MODE_RAGGED_K ? t.crow0 : t.row0) + lr);
            if constexpr (EPI == EPI_SWIGLU) {
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int col = t.col0 + 8 * j + c_in;
                    if (col >= N) continue;
                    const float g0 = acc[4 * j + 2 * i], g1 = acc[4 * j + 2 * i + 1];
                    const float u0 = acc[4 * (j + 16) + 2 * i], u1 = acc[4 * (j + 16) + 2 * i + 1];
                    st_bf16x2(ep.c + grow * ep.ldc + col, silu_f(g0) * u0, silu_f(g1) * u1);
                    if (ep.out2 != nullptr) {
                        st_bf16x2(ep.out2 + grow * ep.ld_out2 + col, g0, g1);
                        st_bf16x2(ep.out2 + grow * ep.ld_out2 + ep.inter + col, u0, u1);
                    }
                }
            } else {
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    const int col = t.col0 + 8 * j + c_in;
                    if (col >= N) continue;
                    float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
                    __nv_bfloat16* dst = ep.c + grow * ep.ldc + col;
                    if constexpr (EPI == EPI_ACCUM) {
                        const float2 o = ld_bf16x2(dst);
                        v0 += o.x;
                        v1 += o.y;
                    }
                    if constexpr (EPI == EPI_DSWIGLU) {
                        const float2 g = ld_bf16x2(ep.aux + grow * ep.ld_aux + col);
                        const float2 u = ld_bf16x2(ep.aux + grow * ep.ld_aux + ep.inter + col);
                        st_bf16x2(ep.out2 + grow * ep.ld_out2 + ep.inter + col, v0 * silu_f(g.x), v1 * silu_f(g.y));
                        v0 = v0 * u.x * dsilu_f(g.x);
                        v1 = v1 * u.y * dsilu_f(g.y);
                    }
                    st_bf16x2(dst, v0, v1);
                }
            }
        }
    }
}

// ---- FP8 (tensorwise- or blockwise-scaled) GEMM ---------------------------------------------------------------------------------------
// C[M, N] (bf16) = epi(sa_inv * sb_inv * A[M, K] B[N, K]^T) with A e4m3 / e5m2 and B e4m3, both K-major (fp8 wgmma reads
// K-major shared operands only).  A stage is [128 rows x 128 B] of A and of B: the same [64 x 128 B] swizzled boxes, the
// same `desc_kmajor_sw128` and the same 32-byte step per k32 wgmma as the bf16 kernel's.
// Promoted accumulation: Hopper's fp8 wgmma adds into its accumulator with reduced precision (about 14 bits, aligned to
// the largest term), so each k-block's four wgmmas (128 K elements) go into a partial accumulator that ordinary FADDs add
// into the fp32 main accumulator.  The reduced precision then applies to 128 products at a time and never to the running
// sum: a block partial the tensor core holds exactly (e.g. small integers on a common power-of-two grid) gives an exact
// result for any K, where an unpromoted accumulation loses the low bits once the sum outgrows 14 bits.  The two 64-float
// accumulators per thread are why a tile is 128 x 128 (64 x 128 per consumer warpgroup), not the bf16 kernel's 128 x 256.
constexpr int F8_BN = 128, F8_BK = 128;  // BK in fp8 elements (= bytes)
constexpr int F8_STAGES = 6;
constexpr uint32_t F8_BOX = 64 * 128;               // [64 rows x 128 B]
constexpr uint32_t F8_STAGE_BYTES = 4 * F8_BOX;     // A: 2 boxes, B: 2 boxes
static_assert(F8_STAGES * F8_STAGE_BYTES <= SMEM_BAR, "the fp8 ring must fit below the barriers");

// EPI_SWIGLU: a tile's 128 B rows are 64 gate rows and the 64 up rows of the same features (N = inter, inter % 64 == 0)
//
// BLOCK (blockwise scaling): sa_inv [ceil(K/128), M] (row stride ld_sa) holds one scale per row of A and k-block, sb_inv
// [ceil(rows of B / 128), ceil(K/128)] (row stride ld_sb) one per 128 x 128 block of B.  The scale granularity is the
// k-block and the tile the kernel walks anyway, so the promotion's FADD becomes an FFMA with
// sa_inv[kb, row] * sb_inv[n-block, kb] and the epilogue applies no scale.  A SwiGLU tile's gate and up rows lie in two
// different 128-row blocks of B (inter % 64 == 0 keeps each 64-row box inside one), so it carries two B scales.
//
// MODE (the dropless MoE forms; segments are 128-row aligned, so no k-block, strip or block straddles two experts):
//   MODE_PLAIN      one [M, N] product
//   MODE_RAGGED     m-tiles per expert over expert-sorted rows A [M, K].  The A format picks the B addressing: e4m3
//                   (forward) B is the stacked weight viewed [E * Nb, K] and expert e's rows start at e * Nb (SwiGLU:
//                   gate rows at e * 2I + col0, up rows at e * 2I + I + col0); e5m2 (dgrad) B is the transposed cast of
//                   that view, [N, E * K], and expert e's W^T is the column slab at K coordinate e * K.  Blockwise B
//                   scales are indexed the same way: block row (e * Nb + col0) / 128, or block column e * K / 128 + kb.
//   MODE_RAGGED_K   dW[e] = A_e B_e^T over expert e's rows only: A [M, R] and B [N, R] (the transposed casts), tiles
//                   (e, m, n), k-blocks [off[e] / 128, off[e+1] / 128); strip row and block column off[e] / 128 + kb.
template <int AE5M2, int EPI, bool BLOCK = false, int MODE = MODE_PLAIN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_fp8_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, int M, int N, int K,
                const EpiParams ep, const float* sa_inv, const float* sb_inv, int ld_sa = 0, int ld_sb = 0)
{
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const uint32_t sbase = smem_u32(smem);
    const uint32_t bar_base = sbase + SMEM_BAR;
    auto full_bar = [&](int s) { return bar_base + 8 * s; };
    auto empty_bar = [&](int s) { return bar_base + 8 * (F8_STAGES + s); };
    int* tile_prefix = reinterpret_cast<int*>(smem + SMEM_GRP);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    using S = Sched<EPI, MODE, F8_BN, F8_BK>;
    constexpr bool kOff = MODE == MODE_RAGGED && AE5M2;  // dgrad: the expert offset lies on B's K coordinate
    constexpr bool kVarK = MODE == MODE_RAGGED_K;

    if constexpr (MODE == MODE_RAGGED || MODE == MODE_RAGGED_K) {
        // as in gemm_kernel: malformed offsets make every CTA leave before any barrier exists, writing nothing
        if (threadIdx.x == kConsumerThreads) {
            const int nn = (N + S::TN - 1) / S::TN;
            tile_prefix[0] = ragged_walk<MODE == MODE_RAGGED, F8_BK>(ep.offsets, ep.E, kVarK ? K : M, nn, tile_prefix)
                                 ? 0
                                 : -1;
        }
        __syncthreads();
        if (tile_prefix[0] != 0) return;
    }

    if (threadIdx.x == kConsumerThreads) {
        prefetch_map(&map_a);
        prefetch_map(&map_b);
        for (int s = 0; s < F8_STAGES; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), kConsumerThreads / 32);
        }
        fence_barrier_init();
    }
    __syncthreads();

    const AgParams no_ag{};
    S sch;
    sch.init(ep, no_ag, M, N, K, tile_prefix);
    const int num_k = (K + F8_BK - 1) / F8_BK;

    if (threadIdx.x >= kConsumerThreads) {
        setmaxnreg_dec<kProducerRegs>();
        if (threadIdx.x == kConsumerThreads) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < sch.num_tiles; tile += gridDim.x) {
                const Tile t = sch.at(tile, ep.inter);
                const int b0 = kOff || kVarK ? t.col0 : t.b0, b1 = kOff || kVarK ? t.col0 + 64 : t.b1;
                const int ka0 = kVarK ? t.k0 : 0, kb0 = kOff || kVarK ? t.k0 : 0;
                const int nk = kVarK ? t.nk : num_k;
                for (int kb = 0; kb < nk; ++kb) {
                    mbar_wait(empty_bar(stage), phase ^ 1);
                    const uint32_t sa = sbase + stage * F8_STAGE_BYTES, sb = sa + 2 * F8_BOX;
                    const uint32_t fb = full_bar(stage);
                    mbar_expect_tx(fb, F8_STAGE_BYTES);
                    tma_load_2d(sa, &map_a, fb, ka0 + kb * F8_BK, t.row0);
                    tma_load_2d(sa + F8_BOX, &map_a, fb, ka0 + kb * F8_BK, t.row0 + 64);
                    tma_load_2d(sb, &map_b, fb, kb0 + kb * F8_BK, b0);
                    tma_load_2d(sb + F8_BOX, &map_b, fb, kb0 + kb * F8_BK, b1);
                    if (++stage == F8_STAGES) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
            }
        }
        return;
    }

    setmaxnreg_inc<kConsumerRegs>();
    const int wg = threadIdx.x >> 7;
    const int r_in = 64 * wg + 16 * (warp & 3) + (lane >> 2);
    const int c_in = 2 * (lane & 3);
    // both scales are powers of two, so the product and the rescaling below are exact; a NaN scale makes C NaN
    float scale = 1.f;  // BLOCK: the scales are applied in the promotion
    if constexpr (!BLOCK) scale = *sa_inv * *sb_inv;
    int stage = 0;
    uint32_t phase = 0;
    float acc[64], part[64];
    for (int tile = blockIdx.x; tile < sch.num_tiles; tile += gridDim.x) {
        const Tile t = sch.at(tile, ep.inter);
        const int nk = kVarK ? t.nk : num_k;
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        // BLOCK: the thread's two rows of sa_inv (a row past M reads row M - 1; it is never stored) and the tile's
        // n-block(s) of sb_inv
        const float* sa_p = sa_inv;
        const float* sb_p = sb_inv;
        int a_off = 0, b_off = 0;
        if constexpr (BLOCK) {
            const int ra = min(t.row0 + r_in, M - 1);
            sa_p += ra;
            a_off = min(t.row0 + r_in + 8, M - 1) - ra;
            const int brow = kOff || kVarK ? t.col0 : t.b0;
            sb_p += static_cast<int64_t>(brow / F8_BN) * ld_sb;
            if constexpr (EPI == EPI_SWIGLU) b_off = (t.b1 / F8_BN - t.b0 / F8_BN) * ld_sb;
            if constexpr (kVarK) sa_p += static_cast<int64_t>(t.k0 / F8_BK) * ld_sa;
            if constexpr (kOff || kVarK) sb_p += t.k0 / F8_BK;
        }
        for (int kb = 0; kb < nk; ++kb) {
            // s[2 h + i]: the scale of row r_in + 8 i in column half h (the two halves differ for SwiGLU only); loaded
            // before the wait so the loads are not behind the k-block's wgmmas
            float s[4];
            if constexpr (BLOCK) {
                const float* sa_kb = sa_p + static_cast<int64_t>(kb) * ld_sa;
                const float a0 = __ldg(sa_kb), a1 = __ldg(sa_kb + a_off);
                const float b0 = __ldg(sb_p + kb), b1 = EPI == EPI_SWIGLU ? __ldg(sb_p + b_off + kb) : b0;
                s[0] = a0 * b0, s[1] = a1 * b0, s[2] = a0 * b1, s[3] = a1 * b1;
            }
            mbar_wait(full_bar(stage), phase);
            const uint32_t sa = sbase + stage * F8_STAGE_BYTES + wg * F8_BOX, sb = sbase + stage * F8_STAGE_BYTES + 2 * F8_BOX;
            const uint64_t da = desc_kmajor_sw128(sa), db = desc_kmajor_sw128(sb);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < F8_BK / 32; ++k) wgmma_m64n128k32_f8_ss<AE5M2>(part, da + 2 * k, db + 2 * k, k > 0 ? 1 : 0);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs<64>(part);
            if (lane == 0) mbar_arrive(empty_bar(stage));
            if constexpr (BLOCK) {
#pragma unroll
                for (int i = 0; i < 64; ++i) acc[i] = fmaf(part[i], s[2 * (i >> 5) + ((i >> 1) & 1)], acc[i]);
            } else {
#pragma unroll
                for (int i = 0; i < 64; ++i) acc[i] += part[i];
            }
            if (++stage == F8_STAGES) {
                stage = 0;
                phase ^= 1;
            }
        }

        // an expert without rows (variable K): its dW is zero (STORE; acc is, and a NaN scale must not reach it) or unchanged
        float tscale = scale;
        if constexpr (kVarK) {
            if (nk == 0) {
                if constexpr (EPI == EPI_ACCUM) continue;
                tscale = 0.f;
            }
        }

        // ---- epilogue from the accumulators: thread holds rows r_in (+8), column pairs c_in + 8 j ----
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int lr = r_in + 8 * i;
            if (lr >= t.rows) continue;
            const int64_t grow = (kVarK ? t.crow0 : t.row0) + lr;
            if constexpr (EPI == EPI_SWIGLU) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int col = t.col0 + 8 * j + c_in;
                    if (col >= N) continue;
                    const float g0 = acc[4 * j + 2 * i] * tscale, g1 = acc[4 * j + 2 * i + 1] * tscale;
                    const float u0 = acc[4 * (j + 8) + 2 * i] * tscale, u1 = acc[4 * (j + 8) + 2 * i + 1] * tscale;
                    st_bf16x2(ep.c + grow * ep.ldc + col, silu_f(g0) * u0, silu_f(g1) * u1);
                    if (ep.out2 != nullptr) {
                        st_bf16x2(ep.out2 + grow * ep.ld_out2 + col, g0, g1);
                        st_bf16x2(ep.out2 + grow * ep.ld_out2 + ep.inter + col, u0, u1);
                    }
                }
            } else {
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int col = t.col0 + 8 * j + c_in;
                    if (col >= N) continue;
                    float v0 = acc[4 * j + 2 * i] * tscale, v1 = acc[4 * j + 2 * i + 1] * tscale;
                    __nv_bfloat16* dst = ep.c + grow * ep.ldc + col;
                    if constexpr (EPI == EPI_ACCUM) {
                        const float2 o = ld_bf16x2(dst);
                        v0 += o.x;
                        v1 += o.y;
                    }
                    if constexpr (EPI == EPI_DSWIGLU) {
                        const float2 g = ld_bf16x2(ep.aux + grow * ep.ld_aux + col);
                        const float2 u = ld_bf16x2(ep.aux + grow * ep.ld_aux + ep.inter + col);
                        st_bf16x2(ep.out2 + grow * ep.ld_out2 + ep.inter + col, v0 * silu_f(g.x), v1 * silu_f(g.y));
                        v0 = v0 * u.x * dsilu_f(g.x);
                        v1 = v1 * u.y * dsilu_f(g.y);
                    }
                    st_bf16x2(dst, v0, v1);
                }
            }
        }
    }
}

}  // namespace gemm
}  // namespace dsb

using namespace dsb::gemm;

static int g_sm_count = 0;

static int sm_count()
{
    if (!g_sm_count) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&g_sm_count, cudaDevAttrMultiProcessorCount, dev);
    }
    return g_sm_count;
}

template <bool A_MN, bool B_MN, int EPI, int MODE>
static int launch_kernel(const CUtensorMap& ma, const CUtensorMap& mb, int M, int N, int K, int grid, const EpiParams& ep,
                         const AgParams& ag, cudaStream_t stream)
{
    static bool attr = false;
    if (!attr) {
        cudaError_t e = cudaFuncSetAttribute(gemm_kernel<A_MN, B_MN, EPI, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             SMEM_TOTAL);
        if (e != cudaSuccess) return static_cast<int>(e);
        attr = true;
    }
    gemm_kernel<A_MN, B_MN, EPI, MODE><<<grid, kThreads, SMEM_TOTAL, stream>>>(ma, mb, M, N, K, ep, ag);
    DSB_CHECK_LAUNCH();
    return 0;
}

template <int EPI>
static int dispatch_major(int a_mn, int b_mn, const CUtensorMap& ma, const CUtensorMap& mb, int M, int N, int K, int grid,
                          const EpiParams& ep, const AgParams& ag, cudaStream_t stream)
{
    if (a_mn && b_mn) return launch_kernel<true, true, EPI, MODE_PLAIN>(ma, mb, M, N, K, grid, ep, ag, stream);
    if (a_mn) return launch_kernel<true, false, EPI, MODE_PLAIN>(ma, mb, M, N, K, grid, ep, ag, stream);
    if (b_mn) return launch_kernel<false, true, EPI, MODE_PLAIN>(ma, mb, M, N, K, grid, ep, ag, stream);
    return launch_kernel<false, false, EPI, MODE_PLAIN>(ma, mb, M, N, K, grid, ep, ag, stream);
}

// General GEMM with selectable operand majorness and fused epilogue:  C[M,N] = epi(op(A) x op(B)), bf16 in/out, fp32
// accumulate.  (The `_2cta` names are kept for API stability; on sm_90a one CTA computes one 128 x 256 tile.)
//   a_mn == 0: A is stored [M, K] row-major (K-major)      a_mn == 1: A is stored [K, M] row-major (MN-major)
//   b_mn == 0: B is stored [N, K] row-major (K-major)      b_mn == 1: B is stored [K, N] row-major (MN-major)
// so (0,0) = "NT" (y = x W^T), (0,1) = "NN" (dx = dy W), (1,1) = "TN" (dW = dy^T x).  lda/ldb are row strides in elements.
//   epi: 0 store, 1 accumulate into C, 2 SwiGLU (B = [gate; up] stacked [2*inter, K], N = inter, C = [M, inter], out2 =
//   optional gate|up save [M, 2*inter]), 3 dSwiGLU (N = inter, aux = saved gate|up, C = out2 = dgate|dup [M, 2*inter]).
//   group_m: m-blocks (of 128 rows) per rasterisation super-group, <= 0 = column-major tile order.
DSB_EXPORT int dsb_gemm_bf16_2cta_ex(const void* a, const void* b, void* c, int M, int N, int K, int lda, int ldb, int ldc,
                                     int a_mn, int b_mn, int epi, const void* aux, int ld_aux, void* out2, int ld_out2,
                                     int inter, int group_m, int sms, cudaStream_t stream)
{
    if (M <= 0 || N <= 0 || K <= 0) return -2;
    if (lda % 8 || ldb % 8 || ldc % 8) return -2;
    if ((a_mn ? M : K) % 8 || (b_mn ? N : K) % 8 || N % 8) return -2;
    if ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) & 15) return -2;
    if (epi < 0 || epi > 3) return -2;
    if (epi == EPI_SWIGLU && (a_mn || b_mn || inter != N || inter % (BN / 2) || (out2 && (ld_out2 % 8)))) return -2;
    if (epi == EPI_DSWIGLU && (a_mn || !aux || !out2 || inter != N || ld_aux % 8 || ld_out2 % 8)) return -2;
    if ((reinterpret_cast<uintptr_t>(aux) | reinterpret_cast<uintptr_t>(out2)) & 15) return -2;
    CUtensorMap ma, mb;
    int rc;
    if ((rc = a_mn ? make_map(&ma, a, K, M, lda, 64) : make_map(&ma, a, M, K, lda, 64))) return rc;
    const uint64_t b_rows = (epi == EPI_SWIGLU) ? static_cast<uint64_t>(2) * inter : static_cast<uint64_t>(N);
    if ((rc = b_mn ? make_map(&mb, b, K, N, ldb, 64) : make_map(&mb, b, b_rows, K, ldb, 64))) return rc;
    EpiParams ep;
    memset(&ep, 0, sizeof(ep));
    ep.aux = static_cast<const __nv_bfloat16*>(aux);
    ep.out2 = static_cast<__nv_bfloat16*>(out2);
    ep.c = static_cast<__nv_bfloat16*>(c);
    ep.ld_aux = ld_aux;
    ep.ld_out2 = ld_out2;
    ep.ldc = ldc;
    ep.inter = inter;
    ep.group_m = group_m;
    AgParams ag;
    memset(&ag, 0, sizeof(ag));
    int grid = sms > 0 ? sms : sm_count();
    const int tn = (epi == EPI_SWIGLU) ? BN / 2 : BN;
    const int tiles = ((M + BM - 1) / BM) * ((N + tn - 1) / tn);
    if (grid > tiles) grid = tiles;
    switch (epi) {
        case EPI_STORE: return dispatch_major<EPI_STORE>(a_mn, b_mn, ma, mb, M, N, K, grid, ep, ag, stream);
        case EPI_ACCUM: return dispatch_major<EPI_ACCUM>(a_mn, b_mn, ma, mb, M, N, K, grid, ep, ag, stream);
        case EPI_SWIGLU: return launch_kernel<false, false, EPI_SWIGLU, MODE_PLAIN>(ma, mb, M, N, K, grid, ep, ag, stream);
        default:
            return b_mn ? launch_kernel<false, true, EPI_DSWIGLU, MODE_PLAIN>(ma, mb, M, N, K, grid, ep, ag, stream)
                        : launch_kernel<false, false, EPI_DSWIGLU, MODE_PLAIN>(ma, mb, M, N, K, grid, ep, ag, stream);
    }
}

DSB_EXPORT int dsb_gemm_bf16_2cta(const void* a, const void* b, void* c, int M, int N, int K, int lda, int ldb, int ldc,
                                  int a_mn, int b_mn, int sms, cudaStream_t stream)
{
    return dsb_gemm_bf16_2cta_ex(a, b, c, M, N, K, lda, ldb, ldc, a_mn, b_mn, EPI_STORE, nullptr, 0, nullptr, 0, 0, 8, sms,
                                 stream);
}

DSB_EXPORT int dsb_gemm_nt_bf16_2cta(const void* a, const void* b, void* c, int M, int N, int K, int lda, int ldb, int ldc,
                                     int sms, cudaStream_t stream)
{
    return dsb_gemm_bf16_2cta(a, b, c, M, N, K, lda, ldb, ldc, 0, 0, sms, stream);
}

// C[M,N] = A[M,K] @ B[N,K]^T   (bf16 in/out, fp32 accumulate).  sms <= 0 -> all SMs.
DSB_EXPORT int dsb_gemm_nt_bf16(const void* a, const void* b, void* c, int M, int N, int K, int lda, int ldb, int ldc,
                                int sms, cudaStream_t stream)
{
    return dsb_gemm_bf16_2cta_ex(a, b, c, M, N, K, lda, ldb, ldc, 0, 0, EPI_STORE, nullptr, 0, nullptr, 0, 0, 0, sms, stream);
}

// Fused all-gather + GEMM.  `b` points at B inside `local_full` (the unit's gathered buffer); the kernel
// fills local_full from peers[] (each `shard_bytes` long) while multiplying.  `flags` holds n_chunks words.
DSB_EXPORT int dsb_gemm_nt_bf16_allgather(const void* a, const void* b, void* c, int M, int N, int K, int lda, int ldb,
                                          int ldc, void* const* peers, void* local_full, uint32_t* flags,
                                          int64_t shard_bytes, int64_t chunk_bytes, int64_t b_offset_bytes, int world,
                                          int rank, int comm_ctas, uint32_t epoch, int sms, cudaStream_t stream)
{
    if (world > 8 || chunk_bytes <= 0 || shard_bytes % chunk_bytes || chunk_bytes % 16) return -2;
    if (M <= 0 || N <= 0 || K <= 0 || K % 8 || N % 8 || lda % 8 || ldb % 8 || ldc % 8) return -2;
    if ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) & 15) return -2;
    AgParams ag;
    memset(&ag, 0, sizeof(ag));
    for (int i = 0; i < world; ++i) ag.peers[i] = peers[i];
    ag.local_full = local_full;
    ag.flags = flags;
    ag.shard_bytes = shard_bytes;
    ag.chunk_bytes = chunk_bytes;
    ag.b_offset_bytes = b_offset_bytes;
    ag.b_bytes = static_cast<int64_t>(N) * ldb * 2;
    ag.n_chunks = static_cast<int>(shard_bytes / chunk_bytes) * world;
    ag.world = world;
    ag.rank = rank;
    ag.comm_ctas = comm_ctas;
    ag.epoch = epoch;
    ag.enabled = 1;
    CUtensorMap ma, mb;
    int rc;
    if ((rc = make_map(&ma, a, M, K, lda, 64))) return rc;
    if ((rc = make_map(&mb, b, N, K, ldb, 64))) return rc;
    EpiParams ep;
    memset(&ep, 0, sizeof(ep));
    ep.c = static_cast<__nv_bfloat16*>(c);
    ep.ldc = ldc;
    // every CTA (math and gather) must be resident at once: the math CTAs spin on flags the gather CTAs publish
    int grid = sms > 0 ? sms : sm_count();
    const int tiles = ((M + BM - 1) / BM) * ((N + BN - 1) / BN);
    int mma = grid - comm_ctas;
    if (mma < 1) return -2;
    if (mma > tiles) mma = tiles;
    return launch_kernel<false, false, EPI_STORE, MODE_ALLGATHER>(ma, mb, M, N, K, mma + comm_ctas, ep, ag, stream);
}

// Grouped GEMM for expert-sorted rows: c[r, :] = a[r, :] @ w[e]^T for offsets[e] <= r < offsets[e+1].
// a [rows, K] (lda), w [E, N, K] contiguous, c [rows, N] (ldc), offsets int32 [E+1] ON THE DEVICE.
DSB_EXPORT int dsb_gemm_grouped_nt_bf16(const void* a, const void* w, void* c, const int* offsets, int rows, int E, int N, int K,
                                        int lda, int ldc, int sms, cudaStream_t stream)
{
    if (rows <= 0 || E <= 0) return 0;
    if (E > kMaxGroups || K % 8 || N % 8 || lda % 8 || ldc % 8) return -3;
    if ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(w) | reinterpret_cast<uintptr_t>(c)) & 15) return -3;
    CUtensorMap ma, mb;
    int rc;
    if ((rc = make_map(&ma, a, rows, K, lda, 64))) return rc;
    if ((rc = make_map(&mb, w, static_cast<uint64_t>(E) * N, K, K, 64))) return rc;
    EpiParams ep;
    memset(&ep, 0, sizeof(ep));
    ep.c = static_cast<__nv_bfloat16*>(c);
    ep.ldc = ldc;
    ep.offsets = offsets;
    ep.E = E;
    AgParams ag;
    memset(&ag, 0, sizeof(ag));
    int grid = sms > 0 ? sms : sm_count();
    // upper bound of the tile count (each expert adds at most one partial m-tile) so tiny problems do not launch idle CTAs
    const int64_t max_tiles = (static_cast<int64_t>(rows + BM - 1) / BM + E) * ((N + BN - 1) / BN);
    if (grid > max_tiles) grid = static_cast<int>(max_tiles);
    return launch_kernel<false, false, EPI_STORE, MODE_GROUPED>(ma, mb, rows, N, K, grid, ep, ag, stream);
}

// ---- ragged (dropless MoE training) forms ---------------------------------------------------------------------------
// Rows are sorted by expert: expert e owns rows [offsets[e], offsets[e+1]) of every [rows, *] operand; offsets is int32
// [E + 1] ON THE DEVICE (no host synchronisation).  Contract, for both entry points:
//   * segments are 64-row aligned and zero-padded: every offset is a multiple of 64 and the rows of a segment past its
//     expert's true token count are zero.  The variable-K form then reads only its expert's rows and the padding adds
//     exact zeros; the m-tiled forms write the padding rows like any other (SwiGLU(0) = 0, so they stay zero);
//   * rows outside [offsets[0], offsets[E]) are neither read into a result nor written;
//   * malformed device offsets -- decreasing, not multiples of 64, negative or past `rows` -- are not launched into: every
//     CTA checks the whole table first and, if it is malformed, exits before it initialises a barrier, writing nothing;
//   * host-checked (-2, nothing launched): 1 <= E <= 256, K % 64 == 0, N % 8 == 0 (SwiGLU / dSwiGLU: N = inter and
//     N % 128 == 0), row strides % 8, 16-byte aligned pointers.

// m-tiled ragged GEMM: for each expert e and its rows r,
//   b_mn == 0:  b = w [E, Nb, K] (K-major), epi STORE: c[r] = a[r] w[e]^T with Nb = N;
//               epi SWIGLU: Nb = 2N (gate rows, then up rows), c [rows, N] = silu(gate) * up, out2 = gate|up (nullable)
//   b_mn == 1:  b = w [E, K, N] (MN-major), epi STORE: c[r] = a[r] w[e];
//               epi DSWIGLU: aux = saved gate|up [rows, 2N], c = out2 = dgate|dup [rows, 2N] (c the left half)
// a [rows, K] (lda), c [rows, N] (ldc).
DSB_EXPORT int dsb_gemm_ragged_bf16(const void* a, const void* b, void* c, const int* offsets, int rows, int E, int N, int K,
                                    int lda, int ldc, int b_mn, int epi, const void* aux, int ld_aux, void* out2, int ld_out2,
                                    int sms, cudaStream_t stream)
{
    if (rows < 0 || E < 1 || E > kMaxGroups || N <= 0 || K <= 0 || K % BK || N % 8 || lda % 8 || ldc % 8) return -2;
    if ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c) |
         reinterpret_cast<uintptr_t>(aux) | reinterpret_cast<uintptr_t>(out2)) & 15)
        return -2;
    const bool fused = epi == EPI_SWIGLU || epi == EPI_DSWIGLU;
    if (epi == EPI_ACCUM || epi < 0 || epi > 3 || (fused && N % (BN / 2))) return -2;
    if (epi == EPI_SWIGLU && (b_mn || (out2 && ld_out2 % 8))) return -2;
    if (epi == EPI_DSWIGLU && (!b_mn || !aux || !out2 || ld_aux % 8 || ld_out2 % 8)) return -2;
    if (offsets == nullptr) return -2;
    if (rows == 0) return 0;
    CUtensorMap ma, mb;
    int rc;
    if ((rc = make_map(&ma, a, rows, K, lda, 64))) return rc;
    const uint64_t e = static_cast<uint64_t>(E);
    if ((rc = b_mn ? make_map(&mb, b, e * K, N, N, 64) : make_map(&mb, b, e * (epi == EPI_SWIGLU ? 2 * N : N), K, K, 64)))
        return rc;
    EpiParams ep;
    memset(&ep, 0, sizeof(ep));
    ep.aux = static_cast<const __nv_bfloat16*>(aux);
    ep.out2 = static_cast<__nv_bfloat16*>(out2);
    ep.c = static_cast<__nv_bfloat16*>(c);
    ep.ld_aux = ld_aux;
    ep.ld_out2 = ld_out2;
    ep.ldc = ldc;
    ep.inter = N;
    ep.offsets = offsets;
    ep.E = E;
    AgParams ag;
    memset(&ag, 0, sizeof(ag));
    int grid = sms > 0 ? sms : sm_count();
    const int tn = epi == EPI_SWIGLU ? BN / 2 : BN;
    const int64_t max_tiles = (static_cast<int64_t>(rows + BM - 1) / BM + E) * ((N + tn - 1) / tn);
    if (grid > max_tiles) grid = static_cast<int>(max_tiles);
    switch (epi) {
        case EPI_SWIGLU: return launch_kernel<false, false, EPI_SWIGLU, MODE_RAGGED>(ma, mb, rows, N, K, grid, ep, ag, stream);
        case EPI_DSWIGLU: return launch_kernel<false, true, EPI_DSWIGLU, MODE_RAGGED>(ma, mb, rows, N, K, grid, ep, ag, stream);
        default:
            return b_mn ? launch_kernel<false, true, EPI_STORE, MODE_RAGGED>(ma, mb, rows, N, K, grid, ep, ag, stream)
                        : launch_kernel<false, false, EPI_STORE, MODE_RAGGED>(ma, mb, rows, N, K, grid, ep, ag, stream);
    }
}

// Variable-K grouped weight gradient: c[e] (+)= a[rows of e]^T b[rows of e] for every expert, i.e. c [E, M, N] contiguous,
// a [rows, M] (lda), b [rows, N] (ldb), both MN-major.  One launch of E x ceil(M/128) x ceil(N/256) tiles; a tile sums its
// expert's k-blocks only.  An expert without rows gets c[e] = 0, or keeps c[e] with `accumulate`.
// Host-checked (-2): rows >= 1, M % 8 == 0 and N % 8 == 0 besides the contract above.
DSB_EXPORT int dsb_gemm_ragged_wgrad_bf16(const void* a, const void* b, void* c, const int* offsets, int rows, int E, int M,
                                          int N, int lda, int ldb, int accumulate, int sms, cudaStream_t stream)
{
    if (rows < 1 || E < 1 || E > kMaxGroups || M <= 0 || N <= 0 || M % 8 || N % 8 || lda % 8 || ldb % 8) return -2;
    if ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) & 15) return -2;
    if (offsets == nullptr) return -2;
    CUtensorMap ma, mb;
    int rc;
    if ((rc = make_map(&ma, a, rows, M, lda, 64))) return rc;
    if ((rc = make_map(&mb, b, rows, N, ldb, 64))) return rc;
    EpiParams ep;
    memset(&ep, 0, sizeof(ep));
    ep.c = static_cast<__nv_bfloat16*>(c);
    ep.ldc = N;
    ep.offsets = offsets;
    ep.E = E;
    AgParams ag;
    memset(&ag, 0, sizeof(ag));
    int grid = sms > 0 ? sms : sm_count();
    const int64_t tiles = static_cast<int64_t>(E) * ((M + BM - 1) / BM) * ((N + BN - 1) / BN);
    if (grid > tiles) grid = static_cast<int>(tiles);
    return accumulate ? launch_kernel<true, true, EPI_ACCUM, MODE_RAGGED_K>(ma, mb, M, N, rows, grid, ep, ag, stream)
                      : launch_kernel<true, true, EPI_STORE, MODE_RAGGED_K>(ma, mb, M, N, rows, grid, ep, ag, stream);
}

template <int AE5M2, int EPI, bool BLOCK, int MODE = MODE_PLAIN>
static int launch_fp8(const CUtensorMap& ma, const CUtensorMap& mb, int M, int N, int K, int grid, const EpiParams& ep,
                      const float* sa_inv, const float* sb_inv, int ld_sa, int ld_sb, cudaStream_t stream)
{
    static bool attr = false;
    if (!attr) {
        cudaError_t e = cudaFuncSetAttribute(gemm_fp8_kernel<AE5M2, EPI, BLOCK, MODE>,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL);
        if (e != cudaSuccess) return static_cast<int>(e);
        attr = true;
    }
    gemm_fp8_kernel<AE5M2, EPI, BLOCK, MODE>
        <<<grid, kThreads, SMEM_TOTAL, stream>>>(ma, mb, M, N, K, ep, sa_inv, sb_inv, ld_sa, ld_sb);
    DSB_CHECK_LAUNCH();
    return 0;
}

// The checks and the launch the two FP8 entry points share (their contracts are written at the entry points).
template <bool BLOCK>
static int gemm_fp8_host(const void* a, const void* b, void* c, int M, int N, int K, int lda, int ldb, int ldc, int a_fmt,
                         const float* sa_inv, int ld_sa, const float* sb_inv, int ld_sb, int epi, const void* aux, int ld_aux,
                         void* out2, int ld_out2, int group_m, int sms, cudaStream_t stream)
{
    if (M <= 0 || N <= 0 || K <= 0 || K % 16 || N % 8) return -2;
    if (lda % 16 || ldb % 16 || lda < K || ldb < K || ldc % 8 || ldc < N || ld_aux % 8 || ld_out2 % 8) return -2;
    if ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c) |
         reinterpret_cast<uintptr_t>(aux) | reinterpret_cast<uintptr_t>(out2)) & 15)
        return -2;
    if (!sa_inv || !sb_inv || (a_fmt != dsb::kF8E4M3 && a_fmt != dsb::kF8E5M2) || epi < 0 || epi > 3) return -2;
    if (BLOCK && (ld_sa < M || ld_sb < (K + F8_BK - 1) / F8_BK)) return -2;
    const bool e5m2 = a_fmt == dsb::kF8E5M2;
    if (epi == EPI_SWIGLU && (e5m2 || N % 64)) return -2;
    if (epi == EPI_DSWIGLU && (!e5m2 || !aux || !out2)) return -2;
    CUtensorMap ma, mb;
    int rc;
    if ((rc = make_map_fp8(&ma, a, M, K, lda, 64))) return rc;
    if ((rc = make_map_fp8(&mb, b, epi == EPI_SWIGLU ? 2 * static_cast<uint64_t>(N) : N, K, ldb, 64))) return rc;
    EpiParams ep;
    memset(&ep, 0, sizeof(ep));
    ep.aux = static_cast<const __nv_bfloat16*>(aux);
    ep.out2 = static_cast<__nv_bfloat16*>(out2);
    ep.c = static_cast<__nv_bfloat16*>(c);
    ep.ld_aux = ld_aux;
    ep.ld_out2 = ld_out2;
    ep.ldc = ldc;
    ep.inter = N;
    ep.group_m = group_m;
    int grid = sms > 0 ? sms : sm_count();
    const int tn = epi == EPI_SWIGLU ? F8_BN / 2 : F8_BN;
    const int64_t tiles = static_cast<int64_t>((M + BM - 1) / BM) * ((N + tn - 1) / tn);
    if (grid > tiles) grid = static_cast<int>(tiles);
    switch (epi) {
        case EPI_STORE:
            return e5m2 ? launch_fp8<1, EPI_STORE, BLOCK>(ma, mb, M, N, K, grid, ep, sa_inv, sb_inv, ld_sa, ld_sb, stream)
                        : launch_fp8<0, EPI_STORE, BLOCK>(ma, mb, M, N, K, grid, ep, sa_inv, sb_inv, ld_sa, ld_sb, stream);
        case EPI_ACCUM:
            return e5m2 ? launch_fp8<1, EPI_ACCUM, BLOCK>(ma, mb, M, N, K, grid, ep, sa_inv, sb_inv, ld_sa, ld_sb, stream)
                        : launch_fp8<0, EPI_ACCUM, BLOCK>(ma, mb, M, N, K, grid, ep, sa_inv, sb_inv, ld_sa, ld_sb, stream);
        case EPI_SWIGLU: return launch_fp8<0, EPI_SWIGLU, BLOCK>(ma, mb, M, N, K, grid, ep, sa_inv, sb_inv, ld_sa, ld_sb, stream);
        default: return launch_fp8<1, EPI_DSWIGLU, BLOCK>(ma, mb, M, N, K, grid, ep, sa_inv, sb_inv, ld_sa, ld_sb, stream);
    }
}

// Tensorwise-scaled FP8 GEMM:  C[M, N] (bf16) = epi(s * A[M, K] B[N, K]^T),  s = *sa_inv * *sb_inv  (device fp32 scalars,
// read by the kernel: no host synchronisation).  Both operands are row-major and K-major: a [M, K] (lda), b [N, K] (ldb),
// one byte per element.  a_fmt is the A format, 5 = e4m3 or 6 = e5m2 (the dtype codes of dsb_common.cuh); B is e4m3.
// Every k-block of 128 products is added into an fp32 accumulator with ordinary FADDs (see the kernel: a block the tensor
// core sums exactly gives an exact result for any K); the scaled result rounds once to bf16 (ACCUM: C_old + s * sum rounds
// once).  A NaN scale inverse gives NaN outputs.
//   epi 0 STORE   C = s AB^T
//   epi 1 ACCUM   C = C + s AB^T
//   epi 2 SWIGLU  A e4m3; b = [gate; up] [2N, K]; C [M, N] = silu(g) * u of g|u = s AB^T; out2 (nullable) [M, 2N] = g|u
//   epi 3 DSWIGLU A e5m2; d = s AB^T [M, N]; aux = saved gate|up [M, 2N]; out2 [M, 2N] = dgate|dup, C its left half
//                 (c == out2, ldc == ld_out2)
// group_m: 128-row m-blocks per rasterisation super-group (<= 0: column-major tile order); sms <= 0: all SMs.
// Host-checked (-2, nothing launched): M, N, K >= 1; K % 16 == 0; N % 8 == 0 (SWIGLU: N % 64 == 0); lda and ldb
// multiples of 16 and >= K; ldc, ld_aux, ld_out2 multiples of 8 and ldc >= N; a, b, c, aux, out2 16-byte aligned;
// sa_inv and sb_inv not null; a_fmt 5 or 6 and, for SWIGLU, 5, for DSWIGLU, 6; DSWIGLU with aux and out2; epi in 0..3.
DSB_EXPORT int dsb_gemm_fp8(const void* a, const void* b, void* c, int M, int N, int K, int lda, int ldb, int ldc, int a_fmt,
                            const float* sa_inv, const float* sb_inv, int epi, const void* aux, int ld_aux, void* out2,
                            int ld_out2, int group_m, int sms, cudaStream_t stream)
{
    return gemm_fp8_host<false>(a, b, c, M, N, K, lda, ldb, ldc, a_fmt, sa_inv, 0, sb_inv, 0, epi, aux, ld_aux, out2, ld_out2,
                                group_m, sms, stream);
}

// Blockwise-scaled FP8 GEMM:  C[M, N] (bf16) = epi(sum over k-blocks kb of sa_inv[kb, m] * sb_inv[n / 128, kb] *
// A[m, kb-block] B[n, kb-block]^T): dsb_gemm_fp8 with one scale per 1 x 128 strip of A and one per 128 x 128 block of B
// (device fp32, the layouts dsb_fp8_cast_block writes) in place of the two scalars.
//   sa_inv [ceil(K/128), M], row stride ld_sa: row kb holds the scale of every row of A for its columns [128 kb, 128 kb + 128)
//   sb_inv [ceil(rows of b / 128), ceil(K/128)], row stride ld_sb (SWIGLU: b has 2N rows; the gate rows of a tile use
//          block row col / 128, its up rows block row (N + col) / 128)
// A k-block's partial sum is multiplied by its scale as it is added to the fp32 accumulator (one FFMA; exact rescaling,
// the scales being powers of two), so a block the tensor core sums exactly still gives an exact result.  A NaN in sa_inv
// makes its row of C NaN, a NaN in sb_inv the columns of its n-block.  Operands, formats, epilogues, group_m, sms and the
// host checks are those of dsb_gemm_fp8, and (-2, nothing launched) ld_sa >= M and ld_sb >= ceil(K/128).
DSB_EXPORT int dsb_gemm_fp8_block(const void* a, const void* b, void* c, int M, int N, int K, int lda, int ldb, int ldc,
                                  int a_fmt, const float* sa_inv, int ld_sa, const float* sb_inv, int ld_sb, int epi,
                                  const void* aux, int ld_aux, void* out2, int ld_out2, int group_m, int sms,
                                  cudaStream_t stream)
{
    return gemm_fp8_host<true>(a, b, c, M, N, K, lda, ldb, ldc, a_fmt, sa_inv, ld_sa, sb_inv, ld_sb, epi, aux, ld_aux, out2,
                               ld_out2, group_m, sms, stream);
}

// ---- ragged (dropless MoE training) FP8 forms ----------------------------------------------------------------------
// The contract of the bf16 ragged forms (expert-sorted rows, int32 device offsets [E + 1], zero-padded segments, rows
// outside [offsets[0], offsets[E]) neither read into a result nor written, malformed device offsets refused by the
// kernel, which then writes nothing) with a 128-row segment granule: every offset is a multiple of 128, the FP8 k-block,
// so no k-block, scale strip or scale block straddles two experts.  Scales are those of dsb_gemm_fp8 (block == 0: two
// device scalars; a stacked weight is one tensor with one scale) or dsb_gemm_fp8_block (block == 1), indexed by the
// tile's expert as the kernel's MODE comment says.

// m-tiled ragged FP8 GEMM, c [rows, N] (ldc) from a [rows, K] (lda), for each expert e and its rows r:
//   a e4m3 (forward):  b = the stacked weight viewed [E * Nb, K] (ldb), c[r] = epi(a[r] b_e^T) with b_e its rows
//                      [e Nb, (e+1) Nb); epi STORE (Nb = N) or SWIGLU (Nb = 2N: gate rows, then up rows; out2 = gate|up
//                      [rows, 2N], nullable)
//   a e5m2 (dgrad):    b = the transposed cast of that view, [N, E * K] (ldb), c[r] = epi(a[r] b_e^T) with b_e its
//                      columns [e K, (e+1) K); epi STORE or DSWIGLU (aux = saved gate|up [rows, 2N], out2 = dgate|dup
//                      [rows, 2N], c its left half)
// block == 1: sa_inv [ceil(K/128), rows] (ld_sa), sb_inv the block scales of b as dsb_fp8_cast_block writes them (ld_sb).
// Host-checked (-2, nothing launched): 1 <= E <= 256, N >= 1, K >= 16, K % 16 == 0, N % 8 == 0 (SWIGLU: N % 64 == 0),
// dgrad K % 128 == 0, blockwise forward STORE N % 128 == 0; lda, ldb multiples of 16 with lda >= K and ldb >= K
// (dgrad: E * K); ldc, ld_aux, ld_out2 multiples of 8, ldc >= N; 16-byte aligned pointers; offsets, sa_inv and sb_inv
// not null; the epilogue allowed for the A format; block: ld_sa >= rows and ld_sb >= the k-blocks of b.
DSB_EXPORT int dsb_gemm_fp8_ragged(const void* a, const void* b, void* c, const int* offsets, int rows, int E, int N, int K,
                                   int lda, int ldb, int ldc, int a_fmt, const float* sa_inv, int ld_sa,
                                   const float* sb_inv, int ld_sb, int epi, const void* aux, int ld_aux, void* out2,
                                   int ld_out2, int block, int sms, cudaStream_t stream)
{
    if (rows < 0 || E < 1 || E > kMaxGroups || N <= 0 || K <= 0 || K % 16 || N % 8) return -2;
    if (lda % 16 || ldb % 16 || lda < K || ldc % 8 || ldc < N || ld_aux % 8 || ld_out2 % 8) return -2;
    if ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c) |
         reinterpret_cast<uintptr_t>(aux) | reinterpret_cast<uintptr_t>(out2)) & 15)
        return -2;
    if (!offsets || !sa_inv || !sb_inv || (a_fmt != dsb::kF8E4M3 && a_fmt != dsb::kF8E5M2)) return -2;
    const bool dgrad = a_fmt == dsb::kF8E5M2;
    if (dgrad ? (epi != EPI_STORE && epi != EPI_DSWIGLU) : (epi != EPI_STORE && epi != EPI_SWIGLU)) return -2;
    if (epi == EPI_SWIGLU && N % 64) return -2;
    if (epi == EPI_DSWIGLU && (!aux || !out2)) return -2;
    const uint64_t e = static_cast<uint64_t>(E);
    const uint64_t b_rows = dgrad ? N : e * (epi == EPI_SWIGLU ? 2 * N : N), b_cols = dgrad ? e * K : K;
    if (dgrad && K % F8_BK) return -2;
    if (static_cast<uint64_t>(ldb) < b_cols) return -2;
    if (block && (ld_sa < rows || static_cast<uint64_t>(ld_sb) < (b_cols + F8_BK - 1) / F8_BK ||
                  (!dgrad && epi == EPI_STORE && N % F8_BN)))
        return -2;
    if (rows == 0) return 0;
    CUtensorMap ma, mb;
    int rc;
    if ((rc = make_map_fp8(&ma, a, rows, K, lda, 64))) return rc;
    if ((rc = make_map_fp8(&mb, b, b_rows, b_cols, ldb, 64))) return rc;
    EpiParams ep;
    memset(&ep, 0, sizeof(ep));
    ep.aux = static_cast<const __nv_bfloat16*>(aux);
    ep.out2 = static_cast<__nv_bfloat16*>(out2);
    ep.c = static_cast<__nv_bfloat16*>(c);
    ep.ld_aux = ld_aux;
    ep.ld_out2 = ld_out2;
    ep.ldc = ldc;
    ep.inter = N;
    ep.offsets = offsets;
    ep.E = E;
    int grid = sms > 0 ? sms : sm_count();
    const int tn = epi == EPI_SWIGLU ? F8_BN / 2 : F8_BN;
    const int64_t max_tiles = (static_cast<int64_t>(rows + BM - 1) / BM + E) * ((N + tn - 1) / tn);
    if (grid > max_tiles) grid = static_cast<int>(max_tiles);
#define DSB_F8R(AF, EP, BL) \
    launch_fp8<AF, EP, BL, MODE_RAGGED>(ma, mb, rows, N, K, grid, ep, sa_inv, sb_inv, ld_sa, ld_sb, stream)
    if (block) {
        if (dgrad) return epi == EPI_DSWIGLU ? DSB_F8R(1, EPI_DSWIGLU, true) : DSB_F8R(1, EPI_STORE, true);
        return epi == EPI_SWIGLU ? DSB_F8R(0, EPI_SWIGLU, true) : DSB_F8R(0, EPI_STORE, true);
    }
    if (dgrad) return epi == EPI_DSWIGLU ? DSB_F8R(1, EPI_DSWIGLU, false) : DSB_F8R(1, EPI_STORE, false);
    return epi == EPI_SWIGLU ? DSB_F8R(0, EPI_SWIGLU, false) : DSB_F8R(0, EPI_STORE, false);
#undef DSB_F8R
}

// Variable-K FP8 weight gradient: c[e] (+)= a_e b_e^T for every expert, where a_e / b_e are the columns
// [offsets[e], offsets[e+1]) of a [M, rows] (e5m2, lda) and b [N, rows] (e4m3, ldb) -- the transposed casts of the
// gradient and of the input -- and c [E, M, N] is contiguous bf16.  One launch of E x ceil(M/128) x ceil(N/128) tiles;
// a tile sums its expert's k-blocks only.  An expert without rows gets c[e] = 0, or keeps c[e] with `accumulate`.
// block == 1: sa_inv [ceil(rows/128), M] (ld_sa; strips along the rows), sb_inv [ceil(N/128), ceil(rows/128)] (ld_sb).
// Host-checked (-2): rows >= 1, M, N >= 1 with N % 8 == 0, lda and ldb multiples of 16 and >= rows,
// 16-byte aligned pointers, offsets / sa_inv / sb_inv not null, 1 <= E <= 256; block: ld_sa >= M and
// ld_sb >= ceil(rows/128).
DSB_EXPORT int dsb_gemm_fp8_ragged_wgrad(const void* a, const void* b, void* c, const int* offsets, int rows, int E, int M,
                                         int N, int lda, int ldb, const float* sa_inv, int ld_sa, const float* sb_inv,
                                         int ld_sb, int accumulate, int block, int sms, cudaStream_t stream)
{
    if (rows < 1 || E < 1 || E > kMaxGroups || M <= 0 || N <= 0 || N % 8) return -2;
    if (lda % 16 || ldb % 16 || lda < rows || ldb < rows) return -2;
    if ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) & 15) return -2;
    if (!offsets || !sa_inv || !sb_inv) return -2;
    if (block && (ld_sa < M || ld_sb < (rows + F8_BK - 1) / F8_BK)) return -2;
    CUtensorMap ma, mb;
    int rc;
    if ((rc = make_map_fp8(&ma, a, M, rows, lda, 64))) return rc;
    if ((rc = make_map_fp8(&mb, b, N, rows, ldb, 64))) return rc;
    EpiParams ep;
    memset(&ep, 0, sizeof(ep));
    ep.c = static_cast<__nv_bfloat16*>(c);
    ep.ldc = N;
    ep.offsets = offsets;
    ep.E = E;
    int grid = sms > 0 ? sms : sm_count();
    const int64_t tiles = static_cast<int64_t>(E) * ((M + BM - 1) / BM) * ((N + F8_BN - 1) / F8_BN);
    if (grid > tiles) grid = static_cast<int>(tiles);
#define DSB_F8K(EP, BL) \
    launch_fp8<1, EP, BL, MODE_RAGGED_K>(ma, mb, M, N, rows, grid, ep, sa_inv, sb_inv, ld_sa, ld_sb, stream)
    if (block) return accumulate ? DSB_F8K(EPI_ACCUM, true) : DSB_F8K(EPI_STORE, true);
    return accumulate ? DSB_F8K(EPI_ACCUM, false) : DSB_F8K(EPI_STORE, false);
#undef DSB_F8K
}

DSB_EXPORT int dsb_gemm_tile_m() { return BM; }
DSB_EXPORT int dsb_gemm_tile_n() { return BN; }
DSB_EXPORT int dsb_gemm_tile_k() { return BK; }
