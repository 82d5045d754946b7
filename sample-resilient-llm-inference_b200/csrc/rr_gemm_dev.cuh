// rr_gemm_dev.cuh — device-side pieces shared by the wgmma GEMM kernels (rr_gemm.cu) and the persistent
// decode layer kernel (rr_layer.cu): tile configuration, the consumer warpgroup's main loop, the per-CTA work schedule,
// small helpers.
//
// CTA layout of every decode-orientation kernel built on this (the prefill GEMM, gemm_pf_wgmma, has its own): warps 0..3 = ONE consumer warpgroup (wgmma issue + epilogue, thread t owns
// row t of the 128-row tile in the epilogue), warp 4 = TMA producer.  The tile's accumulators live in the warpgroup's
// registers (2 x m64nBN: rows 0..63 and 64..127); after the main loop they are staged row-major in shared memory so
// the epilogues read "row t, 32 consecutive columns" per thread.
#pragma once
#include "rr_ptx.cuh"
#include "rr_launch.cuh"
#include "rr_kernels.h"

namespace rr {

constexpr int BLOCK_A = 128;   // tile rows: two m64 wgmma halves
constexpr int BLOCK_K = 64;    // 64 bf16 = 128 B = one swizzle row
constexpr int GMMA_K = 16;
constexpr int GEMM_CONSUMERS = 128;                // warps 0..3
constexpr int GEMM_THREADS = GEMM_CONSUMERS + 32;  // + the TMA producer warp
constexpr int PRODUCER_WARP = GEMM_CONSUMERS / 32;
constexpr int GROUP_A = 16;    // raster group: 16 A tiles share the streamed B tiles through L2

constexpr int cmax(int a, int b) { return a > b ? a : b; }

// CAP bounds the smem ring.  Shared memory: [ring A][ring B][barriers 256 B][staged accumulators][epilogue staging];
// the ring gets what the 227 KB of an H100 SM leave after the largest epilogue staging of any mode.
template <int BN, int CAP = 8>
struct GemmCfg {
    static_assert(BN >= 16 && BN <= MAX_BN, "tile width");
    static constexpr int kStageBytesA = BLOCK_A * BLOCK_K * 2;
    static constexpr int kStageBytesB = BN * BLOCK_K * 2;
    static constexpr int kStageBytes = kStageBytesA + kStageBytesB;
    static constexpr int kAccPitch = BN + 4;               // fp32 words per staged row: conflict-free 16-byte row reads
    static constexpr int kAccBytes = BLOCK_A * kAccPitch * 4;
    static constexpr int kSiluStageBytes = 2 * 32 * 64 * 4;   // OUT_TRANSPOSED_SILU: up-row exchange, 2 x [32 cols][64 rows] fp32
    static constexpr int kEpiMax = cmax(BN <= 64 ? BN * 512 : 0, kSiluStageBytes + (BN <= 64 ? BN * 128 : 0));
    static constexpr int kStagesRaw = (224 * 1024 - 1024 - 256 - kAccBytes - kEpiMax) / kStageBytes;
    static constexpr int kStages = kStagesRaw > CAP ? CAP : kStagesRaw;
    static constexpr int kAccOff = kStages * kStageBytes + 256;         // staged accumulator tile
    static constexpr int kEpiOff = kAccOff + kAccBytes;                 // epilogue staging (mode dependent)
    static constexpr int kSmemBytes = kEpiOff + 1024 /*align slack*/;
};
// TMA-store epilogues of the decode orientation (BN <= 64): the planes tile [BN][128] fp32 (one 3-D TMA store per item); the
// fused MLP kernel aliases it with the up-row exchange (16 KB) + the act tile [BN][64] bf16 of the SiLU epilogue.
template <int BN>
constexpr int planes_stage_bytes() { return BN <= 64 ? BN * 128 * 4 : 0; }
template <int BN>
constexpr int mlp_stage_bytes() {
    constexpr int a = planes_stage_bytes<BN>(), b = GemmCfg<BN>::kSiluStageBytes + (BN <= 64 ? BN * 64 * 2 : 0);
    return a > b ? a : b;
}
template <int BN, int MODE, int CAP = 8>
constexpr int gemm_smem_bytes() {
    // SILU: up-row exchange; F32: the planes tile of the TMA-store epilogue
    return GemmCfg<BN, CAP>::kSmemBytes +
           (MODE == OUT_TRANSPOSED_SILU ? GemmCfg<BN, CAP>::kSiluStageBytes : MODE == OUT_TRANSPOSED_F32 ? planes_stage_bytes<BN>() : 0);
}
// ---- consumer warpgroup ------------------------------------------------------------------------------------------------
// Accumulate the next `nkb` ring slots into acc (acc[0]: tile rows 0..63, acc[1]: rows 64..127).  The first k step
// overwrites the accumulators.  One k-block stays in flight: a slot is released (one arrival per consumer warp on its
// empty barrier) once the wgmma group that read it has retired.
template <int BN>
__device__ __forceinline__ void gmma_mainloop(float (&acc)[2][BN / 2], uint32_t smemA, uint32_t smemB, uint64_t* full_bar,
                                              uint64_t* empty_bar, int& stage, uint32_t& phase, int nkb, int depth) {
    constexpr int kStageA = BLOCK_A * BLOCK_K * 2, kStageB = BN * BLOCK_K * 2;
    const bool arrive = (threadIdx.x & 31) == 0;
    int prev = -1;
    wgmma_fence_regs(acc[0]);
    wgmma_fence_regs(acc[1]);
    for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint64_t da = gmma_desc_sw128(smemA + stage * kStageA);
        const uint64_t db = gmma_desc_sw128(smemB + stage * kStageB);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / GMMA_K; ++k) {
            const uint32_t accum = (kb > 0 || k > 0) ? 1u : 0u;
            wgmma_ss<BN>(acc[0], da + 2 * k, db + 2 * k, accum);
            wgmma_ss<BN>(acc[1], da + ((64 * 128) >> 4) + 2 * k, db + 2 * k, accum);   // rows 64..127: 8 KB further
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && arrive) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == depth) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc[0]);
    wgmma_fence_regs(acc[1]);
    if (prev >= 0 && arrive) mbar_arrive(&empty_bar[prev]);
}
__device__ __forceinline__ void acc_bar() { asm volatile("bar.sync 1, 128;" ::: "memory"); }
// Registers -> the staged tile [128 rows][BN + 4] fp32.  Call between two acc_bar(): the previous item's epilogue must
// have finished reading the tile, and every row is written by two warps.
template <int BN>
__device__ __forceinline__ void stage_acc(const float (&acc)[2][BN / 2], float* tile) {
    constexpr int P = BN + 4;
    const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float* p0 = tile + (64 * h + 16 * w + (l >> 2)) * P + 2 * (l & 3);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            *reinterpret_cast<float2*>(p0 + 8 * j) = make_float2(acc[h][4 * j], acc[h][4 * j + 1]);
            *reinterpret_cast<float2*>(p0 + 8 * P + 8 * j) = make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
        }
    }
}
// This thread's row of the staged tile, columns [c, c + 32) / [c, c + 16) (p = row start + c).
__device__ __forceinline__ void acc_ld32(const float* p, uint32_t (&v)[32]) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const uint4 q = *reinterpret_cast<const uint4*>(p + 4 * i);
        v[4 * i] = q.x; v[4 * i + 1] = q.y; v[4 * i + 2] = q.z; v[4 * i + 3] = q.w;
    }
}
__device__ __forceinline__ void acc_ld16(const float* p, uint32_t (&v)[16]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const uint4 q = *reinterpret_cast<const uint4*>(p + 4 * i);
        v[4 * i] = q.x; v[4 * i + 1] = q.y; v[4 * i + 2] = q.z; v[4 * i + 3] = q.w;
    }
}

// SiLU(g) * u.  __fdividef, not `/`: the IEEE division compiles to a convergence-barrier region with a slow-path CALL per element,
// which serialises the unrolled epilogue loops (2 ulp of fp32 before the bf16 rounding; 0 instead of -1e-36 for g < -87).
__device__ __forceinline__ float silu_mul(float g, float u) { return __fdividef(g, 1.f + __expf(-g)) * u; }

struct WorkItem {
    int a_tile, b_tile, z, kb0, kb1;
};

// Deterministic per-CTA sequence of work items (uniform split-K); every warp role walks the same sequence.
// (A stream-K split -- k-block units dealt evenly to the SMs regardless of tile boundaries -- was measured in round 1:
// 4.55 -> 4.92 ms per decode step, the consumers read more planes than the better balance returns; removed.)
struct WorkSched {
    int tilesA, tilesB, splits, kblocks, n_work, w;

    __device__ __forceinline__ void init(int rowsA, int rowsB, int K, int splits_, int BN) {
        tilesA = (rowsA + BLOCK_A - 1) / BLOCK_A;
        tilesB = (rowsB + BN - 1) / BN;
        kblocks = (K + BLOCK_K - 1) / BLOCK_K;
        splits = splits_;
        n_work = tilesA * tilesB * splits;
        w = blockIdx.x;
    }
    __device__ __forceinline__ bool next(WorkItem& it) {
        if (w >= n_work) return false;
        it.z = w % splits;
        const int q = w / splits;
        const int per_group = GROUP_A * tilesB;
        const int g = q / per_group;
        const int r = q - g * per_group;
        const int a0 = g * GROUP_A;
        const int ga = min(GROUP_A, tilesA - a0);
        it.a_tile = a0 + r % ga;
        it.b_tile = r / ga;
        it.kb0 = (int)(((long long)kblocks * it.z) / splits);
        it.kb1 = (int)(((long long)kblocks * (it.z + 1)) / splits);
        w += gridDim.x;
        return true;
    }
};

}  // namespace rr
