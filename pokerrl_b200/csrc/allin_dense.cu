// All-in showdowns before the board is complete, two-hole-card games - sm_90a (wgmma tensor cores, TMA bulk copies, mbarrier).
//
// Reference: ValueFiller.py:160-175 (`_get_call_eq_preflop`, one-card games: the missing board card is enumerated per
// terminal and the per-board showdown rows of ValueFiller.py:127-158 are averaged).  For two-card hands the enumeration is
// C(48,5) boards per terminal and iteration; the sum over boards does not depend on the strategy, so it is done ONCE:
//     E[h][h'] = sum_q sum_b w_b * sign(rank_b(q(h)) - rank_b(q(h')))     (0: a hand blocked by b, or h and h' share a card)
// (q: the suit permutations of the isomorphism contract, holdem_boards.py; w_b = deal probability x weight in the parent's
// sum) and an all-in terminal's value row is  K * pot / 2 * E @ reach_opp  - a dense real 1326 x 1326 contraction, the one
// place of this path where tensor cores are the right tool (BASELINE.json north_star).
//
// Precision: fp32 operands are split into three bf16 planes (8 + 8 + 8 mantissa bits); the six products of total order
// <= 2 (hi*hi, hi*mid, mid*hi, hi*lo, mid*mid, lo*hi) accumulate in fp32 registers: ~2^-22 of the row's mass, the
// level of an fp32 dot product (test: tests/test_gpu_allin.py against float64).
//
// Kernels:
//   allin_accum_kernel   Ec += sum_b w_b S_b over a chunk of boards, 64 x 64 tile per CTA, double accumulators
//   allin_tiles_kernel   symmetrise over q, mask card-sharing pairs, 3-way bf16 split, write wgmma operand tiles
//                        (K-major, no swizzle: 8 x 16-byte core matrices; a 128 x 64 tile is 16 KB contiguous, fetched by
//                        ONE cp.async.bulk)
//   allin_gemm_kernel    CTA (m-tile of 128 hands, k-block of 64 hands): A tiles by TMA bulk copy on an mbarrier, B (the
//                        <= 16 reach rows, split on the fly) built in shared memory; two warpgroups, each 24 wgmma
//                        (M64 N16 K16, bf16 -> fp32 registers) over its 64 rows of the m-tile -> partial sums
//   allin_finish_kernel  fixed-order sum of the 21 k-block partials, scale, write the ev / ev_br rows
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include "pokerrl_b200.h"
#include "prl_common.cuh"

namespace {

constexpr int kTileM = 128, kTileK = 64, kCols = 16;       // m-tile, k-block, wgmma N (reach rows per launch)
constexpr int kSplits = 3;
constexpr int kATileBytes = kTileM * kTileK * 2;           // 16 KB per split plane
constexpr int kBTileBytes = kCols * kTileK * 2;            // 2 KB per split plane
constexpr int kLBO = 128, kSBO = (kTileK / 8) * 128;       // core matrices: adjacent in K / adjacent 8-row groups (bytes)
constexpr int kWgM = 64;                                   // wgmma M: rows of the m-tile per warpgroup
constexpr int kGemmThreads = 128 * (kTileM / kWgM);        // two warpgroups

inline int m_tiles(int R) { return (R + kTileM - 1) / kTileM; }
inline int k_blocks(int R) { return (R + kTileK - 1) / kTileK; }

// ---------------------------------------------------------------------------------------------------------------- PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// bounded wait: a descriptor mistake must trap, not hang the GPU
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok = 0;
    for (long long spin = 0; spin < (1ll << 26); ++spin) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
        if (ok) return;
    }
    __trap();
}
__device__ __forceinline__ void fence_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// d (+)= A[smem] * B[smem], both K-major bf16, fp32 accumulators in registers; issued by the whole warpgroup
__device__ __forceinline__ void wgmma_m64n16k16(float (&d)[8], uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a_desc), "l"(b_desc), "r"(1)
        : "memory");
}

// wgmma shared-memory matrix descriptor, K-major, no swizzle (layout type 0): start address, leading (K-adjacent core
// matrices) and stride (8-row groups) byte offsets, all >> 4
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(kLBO >> 4) << 16) | ((uint64_t)(kSBO >> 4) << 32);
}

// element (row r of the tile, column k of the k-block) inside a K-major no-swizzle operand tile, in bf16 elements
__host__ __device__ __forceinline__ int tile_elem(int r, int k) { return (r >> 3) * (kSBO / 2) + (k >> 3) * (kLBO / 2) + (r & 7) * 8 + (k & 7); }

__device__ __forceinline__ void split3(double x, __nv_bfloat16& b1, __nv_bfloat16& b2, __nv_bfloat16& b3) {
    b1 = __double2bfloat16(x);
    const double r1 = x - (double)__bfloat162float(b1);
    b2 = __double2bfloat16(r1);
    b3 = __double2bfloat16(r1 - (double)__bfloat162float(b2));
}

// ------------------------------------------------------------------------------------------------- equity matrix, step 1
// Ec[h][h'] += sum_b w_b * sign(rank_b[h] - rank_b[h'])  (rank < 0: the hand holds a board card).  CTA = 64 x 64 tile,
// thread = 4 x 4 pairs, boards staged 32 at a time.
constexpr int kAccTile = 64, kAccBoards = 32;
__global__ void __launch_bounds__(256) allin_accum_kernel(const int32_t* __restrict__ ranks, const double* __restrict__ weight,
                                                          int n_boards, int R, double* __restrict__ ec) {
    __shared__ int sr[kAccBoards][kAccTile], sc[kAccBoards][kAccTile];
    __shared__ double sw[kAccBoards];
    const int h0 = blockIdx.y * kAccTile, g0 = blockIdx.x * kAccTile;
    const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
    double acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
    for (int b0 = 0; b0 < n_boards; b0 += kAccBoards) {
        const int nb = min(kAccBoards, n_boards - b0);
        __syncthreads();
        for (int t = threadIdx.x; t < kAccBoards * kAccTile; t += 256) {
            const int b = t / kAccTile, i = t % kAccTile;
            int vr = -1, vc = -1;
            if (b < nb) {
                if (h0 + i < R) vr = ranks[(size_t)(b0 + b) * R + h0 + i];
                if (g0 + i < R) vc = ranks[(size_t)(b0 + b) * R + g0 + i];
            }
            sr[b][i] = vr;
            sc[b][i] = vc;
        }
        if (threadIdx.x < kAccBoards) sw[threadIdx.x] = (threadIdx.x < nb) ? weight[b0 + threadIdx.x] : 0.0;
        __syncthreads();
        for (int b = 0; b < nb; ++b) {
            const double w = sw[b];
            int rr[4], rc[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                rr[i] = sr[b][ty * 4 + i];
                rc[i] = sc[b][tx * 4 + i];
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const bool live = (rr[i] >= 0) && (rc[j] >= 0);
                    const double s = (rr[i] > rc[j]) ? w : ((rr[i] < rc[j]) ? -w : 0.0);
                    acc[i][j] += live ? s : 0.0;
                }
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int h = h0 + ty * 4 + i, g = g0 + tx * 4 + j;
            if (h < R && g < R) ec[(size_t)h * R + g] += acc[i][j];
        }
}

// ------------------------------------------------------------------------------------------------- equity matrix, step 2
// E[h][h'] = sum_q Ec[perm_q[h]][perm_q[h']] (no permutations: Ec), 0 for hands that share a card or lie in the padding; three bf16
// planes into the operand tiles: plane s of tile (mt, kb) starts at ((mt * KB + kb) * 3 + s) * 8192 elements.
__global__ void __launch_bounds__(256) allin_tiles_kernel(const double* __restrict__ ec, int R, const int8_t* __restrict__ hand_cards,
                                                          const int16_t* __restrict__ sym_perm, int n_sym, int KB,
                                                          __nv_bfloat16* __restrict__ tiles) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;  // padded column
    const int h = blockIdx.y;                              // padded row
    if (g >= KB * kTileK) return;
    double e = 0.0;
    if (h < R && g < R) {
        const int a1 = hand_cards[2 * h], a2 = hand_cards[2 * h + 1], b1 = hand_cards[2 * g], b2 = hand_cards[2 * g + 1];
        if (a1 != b1 && a1 != b2 && a2 != b1 && a2 != b2) {
            if (n_sym > 1) {
                for (int q = 0; q < n_sym; ++q) e += ec[(size_t)sym_perm[(size_t)q * R + h] * R + sym_perm[(size_t)q * R + g]];
            } else {
                e = ec[(size_t)h * R + g];
            }
        }
    }
    __nv_bfloat16 p1, p2, p3;
    split3(e, p1, p2, p3);
    const int mt = h / kTileM, kb = g / kTileK;
    const size_t base = ((size_t)(mt * KB + kb) * kSplits) * (kTileM * kTileK) + tile_elem(h % kTileM, g % kTileK);
    tiles[base] = p1;
    tiles[base + (size_t)kTileM * kTileK] = p2;
    tiles[base + (size_t)2 * kTileM * kTileK] = p3;
}

// ------------------------------------------------------------------------------------------------------------ the GEMM
struct GemmArgs {
    const __nv_bfloat16* tiles;
    const float* x[kCols];  // reach rows (NULL: zero column)
    float* partial;         // [KB][kCols][MT * 128]
    int R, KB, MT;
};

__global__ void __launch_bounds__(kGemmThreads) allin_gemm_kernel(const GemmArgs a) {
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char* sA = smem;                                  // 3 planes x 16 KB
    unsigned char* sB = smem + kSplits * kATileBytes;          // 3 planes x 2 KB
    uint64_t* bar = reinterpret_cast<uint64_t*>(sB + kSplits * kBTileBytes);  // A landed
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;
    const int mt = blockIdx.x, kb = blockIdx.y;

    if (tid == 0) {
        mbar_init(bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    if (tid == 0) {  // the three planes of this (m-tile, k-block) are contiguous: one 48 KB bulk copy
        mbar_expect_tx(bar, kSplits * kATileBytes);
        bulk_g2s(sA, a.tiles + (size_t)(mt * a.KB + kb) * kSplits * (kTileM * kTileK), kSplits * kATileBytes, bar);
    }
    // B: thread (n = tid / 8, 8 consecutive k) of the first warpgroup - one 16-byte core-matrix row per plane
    if (tid < kCols * (kTileK / 8)) {
        const int n = tid >> 3, k0 = (tid & 7) * 8;
        const float* xr = a.x[n];
        __align__(16) __nv_bfloat16 p[kSplits][8];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            const int k = kb * kTileK + k0 + c;
            const float v = (xr != nullptr && k < a.R) ? __ldg(xr + k) : 0.0f;
            split3((double)v, p[0][c], p[1][c], p[2][c]);
        }
#pragma unroll
        for (int s = 0; s < kSplits; ++s)
            *reinterpret_cast<uint4*>(sB + s * kBTileBytes + tile_elem(n, k0) * 2) = *reinterpret_cast<const uint4*>(p[s]);
    }
    fence_async_shared();  // generic-proxy writes of B -> visible to the tensor core (async proxy)
    __syncthreads();
    mbar_wait(bar, 0);

    // warpgroup wg: rows 64 wg .. 64 wg + 63 of the m-tile = 8 core-matrix row groups further into each A plane
    float d[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) d[i] = 0.0f;
    const uint32_t a0 = smem_u32(sA) + wg * (kWgM / 8) * kSBO, b0 = smem_u32(sB);
    // (plane of E, plane of x): the six products of total order <= 2, largest last is not required - fp32 accumulation
    const int pa[6] = {2, 0, 1, 1, 0, 0}, pb[6] = {0, 2, 1, 0, 1, 0};
    wgmma_fence();
#pragma unroll
    for (int t = 0; t < 6; ++t)
#pragma unroll
        for (int ks = 0; ks < kTileK / 16; ++ks)  // K = 16 per instruction: two core matrices = 256 bytes along K
            wgmma_m64n16k16(d, smem_desc(a0 + pa[t] * kATileBytes + ks * 2 * kLBO), smem_desc(b0 + pb[t] * kBTileBytes + ks * 2 * kLBO));
    wgmma_commit();
    wgmma_wait_all();
    // epilogue: accumulator i of lane l in warp w holds row 16 w + l / 4 + 8 (i / 2 % 2), column 8 (i / 4) + 2 (l % 4) + i % 2
    float* out = a.partial + (size_t)kb * kCols * (a.MT * kTileM);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int m = mt * kTileM + wg * kWgM + warp * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
        const int n = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        out[(size_t)n * (a.MT * kTileM) + m] = d[i];
    }
}

struct FinishArgs {
    const float* partial;
    float* y[kCols];
    float* y2[kCols];
    float scale[kCols];
    int R, KB, MT;
};

__global__ void __launch_bounds__(256) allin_finish_kernel(const FinishArgs a) {
    const int h = blockIdx.x * blockDim.x + threadIdx.x, n = blockIdx.y;
    if (h >= a.R || a.y[n] == nullptr) return;
    float s = 0.0f;
    for (int kb = 0; kb < a.KB; ++kb) s += a.partial[((size_t)kb * kCols + n) * (a.MT * kTileM) + h];  // fixed order
    s *= a.scale[n];
    a.y[n][h] = s;
    if (a.y2[n] != nullptr) a.y2[n][h] = s;
}

constexpr int kGemmSmem = kSplits * (kATileBytes + kBTileBytes) + 64;

}  // namespace

extern "C" int64_t prl_allin_tiles_bytes(int n_range) {
    return (int64_t)m_tiles(n_range) * k_blocks(n_range) * kSplits * kATileBytes;
}

extern "C" int64_t prl_allin_partial_bytes(int n_range) {
    return (int64_t)k_blocks(n_range) * kCols * m_tiles(n_range) * kTileM * (int64_t)sizeof(float);
}

extern "C" int prl_allin_equity_accumulate(const int32_t* ranks, const double* weight, int n_boards, int n_range, double* ec,
                                           prl_stream_t stream) {
    if (!ranks || !weight || !ec || n_range <= 0) return prl::fail("prl_allin_equity_accumulate: missing arguments");
    if (n_boards <= 0) return 0;
    const dim3 grid((n_range + kAccTile - 1) / kAccTile, (n_range + kAccTile - 1) / kAccTile);
    allin_accum_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(ranks, weight, n_boards, n_range, ec);
    prl::count_launch();
    return prl::check(cudaGetLastError(), "prl_allin_equity_accumulate");
}

extern "C" int prl_allin_equity_finish(const double* ec, int n_range, const int8_t* hand_cards, const int16_t* sym_perm, int n_sym,
                                       void* tiles, prl_stream_t stream) {
    if (!ec || !hand_cards || !tiles || n_range <= 0) return prl::fail("prl_allin_equity_finish: missing arguments");
    if (n_sym > 1 && !sym_perm) return prl::fail("prl_allin_equity_finish: sym_perm missing");
    const int KB = k_blocks(n_range), MT = m_tiles(n_range);
    const dim3 grid((KB * kTileK + 255) / 256, MT * kTileM);
    allin_tiles_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(ec, n_range, hand_cards, sym_perm, n_sym, KB,
                                                              reinterpret_cast<__nv_bfloat16*>(tiles));
    prl::count_launch();
    return prl::check(cudaGetLastError(), "prl_allin_equity_finish");
}

extern "C" int prl_allin_values(const void* tiles, int n_range, const float* const* x_rows, float* const* y_rows, float* const* y2_rows,
                                const float* scale, int n_cols, float* partial, prl_stream_t stream) {
    if (!tiles || !x_rows || !y_rows || !scale || !partial || n_range <= 0) return prl::fail("prl_allin_values: missing arguments");
    cudaStream_t s = (cudaStream_t)stream;
    const int KB = k_blocks(n_range), MT = m_tiles(n_range);
    if (cudaError_t e = cudaFuncSetAttribute(allin_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kGemmSmem))  // per device
        return prl::check(e, "prl_allin_values: shared memory opt-in");
    for (int c0 = 0; c0 < n_cols; c0 += kCols) {
        GemmArgs g;
        FinishArgs f;
        g.tiles = reinterpret_cast<const __nv_bfloat16*>(tiles);
        g.partial = partial;
        g.R = f.R = n_range;
        g.KB = f.KB = KB;
        g.MT = f.MT = MT;
        f.partial = partial;
        for (int n = 0; n < kCols; ++n) {
            const int c = c0 + n;
            g.x[n] = (c < n_cols) ? x_rows[c] : nullptr;
            f.y[n] = (c < n_cols) ? y_rows[c] : nullptr;
            f.y2[n] = (c < n_cols && y2_rows) ? y2_rows[c] : nullptr;
            f.scale[n] = (c < n_cols) ? scale[c] : 0.0f;
        }
        allin_gemm_kernel<<<dim3(MT, KB), kGemmThreads, kGemmSmem, s>>>(g);
        prl::count_launch();
        const int live = min(kCols, n_cols - c0);
        allin_finish_kernel<<<dim3((n_range + 255) / 256, live), 256, 0, s>>>(f);
        prl::count_launch();
    }
    return prl::check(cudaGetLastError(), "prl_allin_values");
}
