// rr_gemm.cu — the path's one dense contraction (QKV / O / gate-up / down / lm_head projections)
// on Hopper tensor cores: wgmma (m64nNk16, bf16 in, fp32 accumulators in registers), operands staged by TMA
// into 128B-swizzled shared memory, persistent warp-specialised CTAs.
//
//   D[a, b] = sum_k A[a, k] * B[b, k]          A: [rowsA, K] bf16, B: [rowsB, K] bf16 (both K-major)
//
// Two orientations, two kernels:
//   * prefill  (OUT_ROWMAJOR_*, gemm_pf_wgmma): A = activations [T, K], B = weight [N, K] -> C[T, N] row-major; 128 x 256
//     tiles on two consumer warpgroups, epilogues straight from the accumulator registers
//   * decode   (OUT_TRANSPOSED_*, gemm_bf16_wgmma and the fused MLP kernel): 1 TMA producer warp, 1 consumer warpgroup that
//     issues the wgmma and runs the epilogue from the accumulators staged in shared memory;
//                                    A = weight [N, K] (wgmma M side, streamed once from HBM),
//                                    B = activations [batch<=BN, K]; fp32 partial planes
//                                    P[z][b][n] reduced by the consumer kernel (rr_elementwise.cu).
//     Work split for decode: uniform split-K (splits planes); the wave-quantisation tail of the big gate/up
//     projection is removed by the fused MLP kernel below (per-slice dataflow), not by a stream-K split.
//
// PDL: the weight operand is constant, its first pipeline stages are requested before
// griddepcontrol.wait; only the activation operand and the output wait for the preceding kernel.
//
// FP8 weights (template flag FP8 of the decode kernels): A is e4m3 [N, K] with one power-of-two scale per row (rr_fp8.cu).
// The TMA producer streams 128 x 64-byte e4m3 slices (no swizzle) into a ring of half the bf16 stage size; the consumer
// warpgroup converts each slice exactly into bf16(Q * s), written into one of three 128B-swizzled 16 KB tiles (the layout
// TMA gives a bf16 A stage), fences the generic-proxy writes against the async proxy, and runs the same wgmma sequence,
// k order, split-K planes and epilogues as the bf16 kernel: the output bits equal the bf16 kernel's on D = bf16(Q * s).
//
// Replaces: the remote bedrock:InvokeModel call (reference iam/policy.json:8,
// src/demo_cris.py:233-238) — there is no reference kernel; see DESIGN.md §kernels.
#include "rr_ptx.cuh"
#include "rr_launch.cuh"
#include "rr_kernels.h"

#include <mutex>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

namespace rr {

// ---- decode-orientation tile configuration, the consumer warpgroup's main loop, the per-CTA work schedule, small helpers.
// CTA layout of every decode-orientation kernel (the prefill GEMM, gemm_pf_wgmma, has its own): warps 0..3 = ONE consumer
// warpgroup (wgmma issue + epilogue, thread t owns row t of the 128-row tile in the epilogue), warp 4 = TMA producer.  The
// tile's accumulators live in the warpgroup's registers (2 x m64nBN: rows 0..63 and 64..127); after the main loop they are
// staged row-major in shared memory so the epilogues read "row t, 32 consecutive columns" per thread.

constexpr int BLOCK_A = 128;   // tile rows: two m64 wgmma halves
constexpr int BLOCK_K = 64;    // 64 bf16 = 128 B = one swizzle row
constexpr int GMMA_K = 16;
constexpr int GEMM_CONSUMERS = 128;                // warps 0..3
constexpr int GEMM_THREADS = GEMM_CONSUMERS + 32;  // + the TMA producer warp
constexpr int PRODUCER_WARP = GEMM_CONSUMERS / 32;
constexpr int GROUP_A = 16;    // raster group: 16 A tiles share the streamed B tiles through L2

constexpr int cmax(int a, int b) { return a > b ? a : b; }

// CAP bounds the smem ring.  Shared memory: [converted tiles (FP8)][ring A][ring B][barriers 256 B][staged accumulators]
// [epilogue staging]; the ring gets what the 227 KB of an H100 SM leave after the largest epilogue staging of any mode and,
// with FP8 weights, the three converted bf16 A tiles (48 KB).  An e4m3 A stage is 8 KB instead of 16 KB.  Stages, bf16 ->
// FP8: BN 16: 8 -> 8, BN 32: 8 -> 8, BN 64: 6 -> 6, BN 128: 4 -> 3.
template <int BN, int CAP = 8, bool FP8 = false>
struct GemmCfg {
    static_assert(BN >= 16 && BN <= MAX_BN, "tile width");
    static constexpr int kStageBytesA = BLOCK_A * BLOCK_K * (FP8 ? 1 : 2);
    static constexpr int kStageBytesB = BN * BLOCK_K * 2;
    static constexpr int kStageBytes = kStageBytesA + kStageBytesB;
    static constexpr int kCvtTiles = FP8 ? 3 : 0;          // converted A tiles: wgmma k-block i reads tile i % 3
    static constexpr int kCvtBytes = kCvtTiles * BLOCK_A * BLOCK_K * 2;
    static constexpr int kAccPitch = BN + 4;               // fp32 words per staged row: conflict-free 16-byte row reads
    static constexpr int kAccBytes = BLOCK_A * kAccPitch * 4;
    static constexpr int kSiluStageBytes = 2 * 32 * 64 * 4;   // OUT_TRANSPOSED_SILU: up-row exchange, 2 x [32 cols][64 rows] fp32
    static constexpr int kEpiMax = cmax(BN <= 64 ? BN * 512 : 0, kSiluStageBytes + (BN <= 64 ? BN * 128 : 0));
    static constexpr int kStagesRaw = (224 * 1024 - 1024 - 256 - kAccBytes - kEpiMax - kCvtBytes) / kStageBytes;
    static constexpr int kStages = kStagesRaw > CAP ? CAP : kStagesRaw;
    static constexpr int kRingOff = kCvtBytes;                          // ring A, then ring B
    static constexpr int kBarOff = kRingOff + kStages * kStageBytes;    // full / empty barriers (+ the MLP's item queue)
    static constexpr int kAccOff = kBarOff + 256;                       // staged accumulator tile
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
template <int BN, int MODE, int CAP = 8, bool FP8 = false>
constexpr int gemm_smem_bytes() {
    // SILU: up-row exchange; F32: the planes tile of the TMA-store epilogue
    return GemmCfg<BN, CAP, FP8>::kSmemBytes +
           (MODE == OUT_TRANSPOSED_SILU ? GemmCfg<BN, CAP>::kSiluStageBytes : MODE == OUT_TRANSPOSED_F32 ? planes_stage_bytes<BN>() : 0);
}
// ---- FP8 weights: the consumer warpgroup's converter ------------------------------------------------------------------
// Lane l of warp w converts 16 bytes (k 16 (l % 4) ..) of rows 32 w + l / 4 + 8 i, i < 4: each read instruction of a warp
// covers 512 contiguous bytes of the slice, and the two 16-byte writes per row land on 128B-swizzle chunks that cover all
// eight bank groups of a row block (no bank conflicts either way).
struct Fp8Conv {
    const uint8_t* ring;      // e4m3 ring A
    uint8_t* tiles;           // kCvtTiles converted bf16 tiles, 16 KB each, 1024-byte aligned
    int tile;                 // the tile the next k-block is converted into
    float sc[4];              // scales of this lane's rows for the current item (1 for rows >= rowsA, which TMA zero-fills)
    __device__ __forceinline__ void load_scales(const float* scale, int a_tile, int rowsA) {
        const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int r = a_tile * BLOCK_A + 32 * w + (l >> 2) + 8 * i;
            sc[i] = r < rowsA ? __ldg(scale + r) : 1.f;
        }
    }
    // ring slot -> tile; returns the tile's shared-memory address.  Tile t is rewritten three k-blocks after it was read:
    // every warp has passed the wgmma_wait<1> that retires that read before it reached the barrier of the k-block between.
    __device__ __forceinline__ uint32_t convert(int stage) {
        const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
        const uint8_t* src = ring + stage * (BLOCK_A * BLOCK_K);
        uint8_t* dst = tiles + tile * (BLOCK_A * BLOCK_K * 2);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int r = 32 * w + (l >> 2) + 8 * i;
            const uint4 q = *reinterpret_cast<const uint4*>(src + r * BLOCK_K + 16 * (l & 3));
            const uint2 a = e4m3x4_to_bf16x4(q.x, sc[i]), b = e4m3x4_to_bf16x4(q.y, sc[i]);
            const uint2 c = e4m3x4_to_bf16x4(q.z, sc[i]), d = e4m3x4_to_bf16x4(q.w, sc[i]);
            const int c0 = 2 * (l & 3);                  // 16-byte bf16 chunks c0, c0 + 1 of row r, swizzled by r % 8
            *reinterpret_cast<uint4*>(dst + r * 128 + ((c0 ^ (r & 7)) << 4)) = make_uint4(a.x, a.y, b.x, b.y);
            *reinterpret_cast<uint4*>(dst + r * 128 + (((c0 + 1) ^ (r & 7)) << 4)) = make_uint4(c.x, c.y, d.x, d.y);
        }
        fence_proxy_async();                             // generic-proxy writes -> the wgmma's async-proxy reads
        asm volatile("bar.sync 5, 128;" ::: "memory");
        const uint32_t t = smem_u32(dst);
        tile = tile == 2 ? 0 : tile + 1;
        return t;
    }
};

// ---- consumer warpgroup ------------------------------------------------------------------------------------------------
// Accumulate the next `nkb` ring slots into acc (acc[0]: tile rows 0..63, acc[1]: rows 64..127).  The first k step
// overwrites the accumulators.  One k-block stays in flight: a slot is released (one arrival per consumer warp on its
// empty barrier) once the wgmma group that read it has retired.
// FP8: cv converts each ring slot first and the wgmma read the converted tile.
template <int BN, bool FP8 = false>
__device__ __forceinline__ void gmma_mainloop(float (&acc)[2][BN / 2], uint32_t smemA, uint32_t smemB, uint64_t* full_bar,
                                              uint64_t* empty_bar, int& stage, uint32_t& phase, int nkb, int depth,
                                              Fp8Conv* cv = nullptr) {
    constexpr int kStageA = BLOCK_A * BLOCK_K * 2, kStageB = BN * BLOCK_K * 2;
    const bool arrive = (threadIdx.x & 31) == 0;
    int prev = -1;
    wgmma_fence_regs(acc[0]);
    wgmma_fence_regs(acc[1]);
    for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        uint64_t da;
        if constexpr (FP8) da = gmma_desc_sw128(cv->convert(stage));
        else da = gmma_desc_sw128(smemA + stage * kStageA);
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

// Epilogue of one work item: staged accumulator tile (this thread's row, BN columns at arow) -> global memory, in the
// layout / fusion selected by MODE.  Shared by the GEMM kernel and the fused MLP kernel.
template <int BN, int MODE>
__device__ __forceinline__ void epilogue_item(const float* arow, int a_row, const WorkItem& t, int quarter, int lane,
                                              void* __restrict__ out, int rowsA, int rowsB, int ldo, int ld_rows,
                                              float* silu_stage) {
    constexpr int CH = (BN >= 32) ? 32 : 16;
    if constexpr (MODE == OUT_TRANSPOSED_SILU) {
        // gate/up rows are interleaved in blocks of 64: lanes 0..63 of the tile hold gate rows, lanes 64..127 the
        // matching up rows.  The up warps hand their values over through smem ([col][row] -> conflict-free), the
        // gate warps write act[b][n] = silu(g) * u as bf16.  rowsA = 2 * inter (interleaved), ldo = inter.
        float* stage = silu_stage;
        const bool is_up = quarter >= 2;
        const int r64 = (quarter & 1) * 32 + lane;
        const int n = t.a_tile * 64 + r64;
        __nv_bfloat16* act = reinterpret_cast<__nv_bfloat16*>(out);
#pragma unroll 1
        for (int c = 0; c < BN; c += 32) {
            float* buf = stage + ((c >> 5) & 1) * (32 * 64);
            uint32_t v[32];
            acc_ld32(arow + c, v);
            if (is_up) {
#pragma unroll
                for (int j = 0; j < 32; ++j) buf[j * 64 + r64] = __uint_as_float(v[j]);
            }
            asm volatile("bar.sync 2, 128;" ::: "memory");
            if (!is_up && 2 * n < rowsA) {
                const int b0 = t.b_tile * BN + c;
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    const int b = b0 + j;
                    if (b < rowsB)
                        act[(size_t)b * ldo + n] = __float2bfloat16(silu_mul(__uint_as_float(v[j]), buf[j * 64 + r64]));
                }
            }
        }
    } else {
#pragma unroll 1
    for (int c = 0; c < BN; c += CH) {
        uint32_t v[32];
        if constexpr (CH == 32) {
            acc_ld32(arow + c, v);
        } else {
            uint32_t v16[16];
            acc_ld16(arow + c, v16);
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] = v16[j];
        }
        const int b0 = t.b_tile * BN + c;
        float* dst = reinterpret_cast<float*>(out);
        if (a_row < rowsA) {
#pragma unroll
            for (int j = 0; j < CH; ++j) {
                const int b = b0 + j;
                if (b < rowsB)
                    dst[((size_t)t.z * ld_rows + b) * ldo + a_row] = __uint_as_float(v[j]);
            }
        }
    }
    }
}

// ---- TMA-store epilogues (decode orientation, BN <= 64) ---------------------------------------------------------------------
// Under a saturated weight stream an LSU store costs the issuing warp 75-170 ns (tools/trace_mlp.py: 64 four-byte stores
// per thread = 5 us per planes tile, the 2-byte act stores of the SiLU epilogue + the fence = 14 us from "accumulator
// ready" to "tile published", and the down items of the fused MLP kernel wait exactly for that).  Here the 128 epilogue
// threads transpose the tile through shared memory and ONE thread hands it to the TMA engine as a single bulk store.
__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 4, 128;" ::: "memory"); }

// planes tile: stage[b][n] fp32, b < BN, n < 128 (n = accumulator row = this thread)  ->  P[z][b][a_tile * 128 + n]
template <int BN>
__device__ __forceinline__ void epilogue_planes_tma(const float* arow, const WorkItem& t, int quarter, int lane, int etid,
                                                    const CUtensorMap* tmOut, float* stage) {
    constexpr int CH = (BN >= 32) ? 32 : 16;
    if (etid == 0) bulk_wait_read0();              // the previous item's store has read the staging tile
    epi_bar();
    float* col = stage + quarter * 32 + lane;
#pragma unroll 1
    for (int c = 0; c < BN; c += CH) {
        uint32_t v[32];
        if constexpr (CH == 32) {
            acc_ld32(arow + c, v);
        } else {
            uint32_t v16[16];
            acc_ld16(arow + c, v16);
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] = v16[j];
        }
#pragma unroll
        for (int j = 0; j < CH; ++j) col[(c + j) * 128] = __uint_as_float(v[j]);      // lanes = consecutive n: conflict-free
    }
    fence_proxy_async();                           // generic-proxy smem writes -> the TMA engine's reads
    epi_bar();
    if (etid == 0) {
        tma_store_3d(tmOut, stage, t.a_tile * BLOCK_A, t.b_tile * BN, t.z);
        bulk_commit();
    }
}

// SiLU tile of the gate/up projection: lanes 0..63 of the accumulator = gate rows, 64..127 = the matching up rows.  ALL four
// warps compute: per 32-column chunk the gate thread of a feature hands its columns 16..31 to the up thread and receives the up
// values of columns 0..15 (exch: two [16][64] fp32 halves per chunk, double-buffered), so each thread evaluates 16 SiLUs per
// chunk instead of the gate threads 32.  act_stage[b][n64] bf16  ->  act[b][a_tile * 64 + n64]
template <int BN>
__device__ __forceinline__ void epilogue_silu_tma(const float* arow, const WorkItem& t, int quarter, int lane, int etid,
                                                  const CUtensorMap* tmAct, float* exch, __nv_bfloat16* act_stage) {
    const bool is_up = quarter >= 2;
    const int r64 = (quarter & 1) * 32 + lane;
    if (etid == 0) bulk_wait_read0();
    epi_bar();
#pragma unroll 1
    for (int c = 0; c < BN; c += 32) {
        float* buf = exch + ((c >> 5) & 1) * (32 * 64);     // [0, 16) rows: up values of cols 0..15; [16, 32): gate values of cols 16..31
        uint32_t v[32];
        acc_ld32(arow + c, v);
        if (is_up) {
#pragma unroll
            for (int j = 0; j < 16; ++j) buf[j * 64 + r64] = __uint_as_float(v[j]);
        } else {
#pragma unroll
            for (int j = 16; j < 32; ++j) buf[j * 64 + r64] = __uint_as_float(v[j]);
        }
        asm volatile("bar.sync 2, 128;" ::: "memory");
        float o[16];
        if (is_up) {
#pragma unroll
            for (int j = 0; j < 16; ++j) o[j] = buf[(16 + j) * 64 + r64];          // gate values, cols 16..31
#pragma unroll
            for (int j = 0; j < 16; ++j)
                act_stage[(c + 16 + j) * 64 + r64] = __float2bfloat16(silu_mul(o[j], __uint_as_float(v[16 + j])));
        } else {
#pragma unroll
            for (int j = 0; j < 16; ++j) o[j] = buf[j * 64 + r64];                 // up values, cols 0..15
#pragma unroll
            for (int j = 0; j < 16; ++j)
                act_stage[(c + j) * 64 + r64] = __float2bfloat16(silu_mul(__uint_as_float(v[j]), o[j]));
        }
    }
    fence_proxy_async();
    epi_bar();
    if (etid == 0) {
        tma_store_2d(tmAct, act_stage, t.a_tile * 64, t.b_tile * BN);
        bulk_commit();
    }
}

template <int BN, int MODE, int CAP = 8, bool FP8 = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_wgmma(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                void* __restrict__ out, int rowsA, int rowsB, int K, int splits, int ldo,
                int ld_rows, const __grid_constant__ CUtensorMap tmOut, int tma_epi, const float* __restrict__ scaleA) {
    using Cfg = GemmCfg<BN, CAP, FP8>;
    constexpr int kStages = Cfg::kStages;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align_smem_1024(smem_raw);
    uint8_t* smemA = smem + Cfg::kRingOff;
    uint8_t* smemB = smemA + kStages * Cfg::kStageBytesA;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kBarOff);
    uint64_t* empty_bar = full_bar + kStages;
    float* acc_tile = reinterpret_cast<float*>(smem + Cfg::kAccOff);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    griddep_launch();   // PDL: the next kernel may start its prologue now
    const int tr_slot = trace_begin(TR_GEMM_DEC);

    if (warp == PRODUCER_WARP && elect_one()) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], GEMM_CONSUMERS / 32);   // one arrival per consumer warp
        }
        fence_barrier_init();
    }
    __syncthreads();

    WorkSched sched;
    sched.init(rowsA, rowsB, K, splits, BN);
    WorkItem t;
    // detail trace of a plain decode projection: selected by its split-K factor (rr_debug_trace_detail(10 + splits)), CTAs 0 / 37 / 74 / 111
    const int tsm = (rr_trace_detail == 10 + splits && blockIdx.x % 37 == 0) ? 8 + (int)(blockIdx.x / 37) : -1;

    if (warp == PRODUCER_WARP) {
        // ===================== TMA producer =====================
        if (elect_one()) {
            // Streamed-once operand (decode weights) should not displace the KV cache in L2;
            // the small re-read operand is kept.
            const uint64_t polA = l2_policy_evict_first();
            const uint64_t polB = l2_policy_evict_last();
            int stage = 0;
            uint32_t phase = 0;
            bool have = sched.next(t);
            if (tsm >= 0) trace_mark_at(TR_GEMM_MARK + 0, tsm, 0);
            // PDL prefetch of the constant (weight) operand for the first `pre` k-blocks.
            int pre = 0;
            if (have) {
                pre = min(kStages, t.kb1 - t.kb0);
                for (int i = 0; i < pre; ++i) {
                    mbar_arrive_expect_tx(&full_bar[i], Cfg::kStageBytes);
                    tma_load_2d_hint(smemA + i * Cfg::kStageBytesA, &tmA, &full_bar[i], (t.kb0 + i) * BLOCK_K,
                                     t.a_tile * BLOCK_A, polA);
                }
            }
            griddep_wait();
            trace_dep(tr_slot);
            if (tsm >= 0) trace_mark_at(TR_GEMM_MARK + 1, tsm, 1);
            if (have) {
                for (int i = 0; i < pre; ++i)
                    tma_load_2d_hint(smemB + i * Cfg::kStageBytesB, &tmB, &full_bar[i], (t.kb0 + i) * BLOCK_K,
                                     t.b_tile * BN, polB);
                t.kb0 += pre;                          // already in flight
                stage = pre % kStages;
                phase = (pre == kStages) ? 1u : 0u;
            }
            while (have) {
                for (int kb = t.kb0; kb < t.kb1; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
                    tma_load_2d_hint(smemA + stage * Cfg::kStageBytesA, &tmA, &full_bar[stage],
                                     kb * BLOCK_K, t.a_tile * BLOCK_A, polA);
                    tma_load_2d_hint(smemB + stage * Cfg::kStageBytesB, &tmB, &full_bar[stage],
                                     kb * BLOCK_K, t.b_tile * BN, polB);
                    if (++stage == kStages) {
                        stage = 0;
                        phase ^= 1;
                    }
                }
                have = sched.next(t);
            }
            if (tsm >= 0) trace_mark_at(TR_GEMM_MARK + 2, tsm, 2);
        }
    } else {
        // ===================== consumer warpgroup: wgmma main loop, then the epilogue (warps 0..3) =====================
        const int quarter = warp;                     // rows [32 quarter, 32 quarter + 32) of the tile in the epilogue
        const int row_in_tile = quarter * 32 + lane;
        const int etid = threadIdx.x;
        float* epi_stage = reinterpret_cast<float*>(smem + Cfg::kEpiOff);
        const uint32_t smemA_u = smem_u32(smemA), smemB_u = smem_u32(smemB);
        if (MODE == OUT_TRANSPOSED_F32 && BN <= 64 && tma_epi && etid == 0) tma_prefetch_desc(&tmOut);
        griddep_wait();                               // `out` may still be read by the preceding kernel
        trace_dep(tr_slot);
        int stage = 0;
        uint32_t phase = 0;
        Fp8Conv cv{smemA, smem, 0, {}};
        for (int it = 0; sched.next(t); ++it) {
            float acc[2][BN / 2];
            if constexpr (FP8) cv.load_scales(scaleA, t.a_tile, rowsA);
            gmma_mainloop<BN, FP8>(acc, smemA_u, smemB_u, full_bar, empty_bar, stage, phase, t.kb1 - t.kb0, kStages, &cv);
            if (tsm >= 0 && etid == 0) trace_mark_at(TR_GEMM_MARK + 4, tsm, 16 + 2 * it);
            acc_bar();                                // the previous item's epilogue is done with the staged tile
            stage_acc<BN>(acc, acc_tile);
            acc_bar();
            const int a_row = t.a_tile * BLOCK_A + row_in_tile;
            const float* arow = acc_tile + row_in_tile * Cfg::kAccPitch;
            bool done = false;
            if constexpr (MODE == OUT_TRANSPOSED_F32 && BN <= 64) {
                if (tma_epi) { epilogue_planes_tma<BN>(arow, t, quarter, lane, etid, &tmOut, epi_stage); done = true; }
            }
            if (!done)
                epilogue_item<BN, MODE>(arow, a_row, t, quarter, lane, out, rowsA, rowsB, ldo, ld_rows, epi_stage);
            if (tsm >= 0 && etid == 0) trace_mark_at(TR_GEMM_MARK + 5, tsm, 17 + 2 * it);
        }
        if constexpr (MODE == OUT_TRANSPOSED_F32 && BN <= 64) {
            if (tma_epi && etid == 0) bulk_wait_read0();   // the staging tile must outlive the reads of its stores; grid completion covers the writes
        }
    }

    __syncthreads();
    if (tsm >= 0 && threadIdx.x == 0) trace_mark_at(TR_GEMM_MARK + 6, tsm, 3);
    trace_end(tr_slot);
}

// =================================================================================================
// Prefill orientation: A = activations [T, K], B = weight [N, K], row-major outputs (QKV + RoPE, O / down + residual,
// gate/up + SiLU, plain bf16).  Compute-bound, so the tile is as wide as a warpgroup's registers allow: 128 tokens x 256
// weight rows, two consumer warpgroups (64 token rows each, m64n256k16: 128 fp32 accumulators per thread), one producer
// warpgroup of which one thread issues the TMA loads.  setmaxnreg moves the producer's registers to the consumers.  The
// epilogues run straight from the accumulator fragments: a thread holds rows r and r + 8 at columns 8j + 2(lane % 4) + {0, 1},
// j < 32, so a quad covers 8 consecutive columns (a full 32-byte sector of fp32), a head's columns d and d + 64 (RoPE) and a
// block's gate and up columns (SiLU) sit in the same thread.
struct PfCfg {
    static constexpr int kTileB = 256;
    static constexpr int kStages = 4;
    static constexpr int kStageBytesA = BLOCK_A * BLOCK_K * 2;             // 16 KB
    static constexpr int kStageBytesB = kTileB * BLOCK_K * 2;              // 32 KB
    static constexpr int kStageBytes = kStageBytesA + kStageBytesB;
    static constexpr int kThreads = 384;                                   // warpgroup 0: producer, 1 and 2: consumers
    static constexpr int kConsumerWarps = 8;
    static constexpr int kSmemBytes = kStages * kStageBytes + 256 + 1024 /*align slack*/;
    static constexpr int kProducerRegs = 40, kConsumerRegs = 232;          // 128 x 40 + 256 x 232 <= 64 K registers
};
static_assert(2 * PfCfg::kSmemBytes > 227 * 1024 && PfCfg::kSmemBytes <= 227 * 1024, "one prefill GEMM CTA per SM");
static_assert(2 * PF_NORM_COLS == PfCfg::kTileB, "the residual epilogue writes two sum(x^2) partials per tile");

// Deferred RMSNorm, consumer side: the operand row was bf16(x * gamma); 1 / rms(x) from its partial sums of squares.
__device__ __forceinline__ float pf_rinv(const RopeEpi& rope, int row, int rowsA) {
    if (rope.n_part <= 0 || row >= rowsA) return 1.f;
    const float* ps = rope.rowss + (size_t)row * rope.n_part;
    float ss = 0.f;
    for (int j = 0; j < rope.n_part; ++j) ss += ps[j];
    return rsqrtf(ss * rope.inv_hidden + rope.eps);
}

// acc: this thread's fragment of the consumer warpgroup's 64 x 256 block; row0 = its first token row, cb = first column of the tile
template <int MODE>
__device__ __forceinline__ void pf_epilogue(const float (&acc)[128], int row0, int b_tile, int quad, void* __restrict__ out,
                                            int rowsA, int rowsB, int ldo, const RopeEpi& rope) {
    const int cb = b_tile * PfCfg::kTileB;
    const int cq = 2 * quad;                                   // column offset of this thread inside each group of 8
    if constexpr (MODE == OUT_ROWMAJOR_RESID) {
        float* xres = reinterpret_cast<float*>(out);
        const bool defer = rope.xhat != nullptr;               // also emit bf16(x * gamma) and sum(x^2) per 128 columns
        // sum(x^2) of a row over 128 columns, in one fixed order (the deferred norm of the next GEMM depends on its last bit):
        // columns in groups of 4, g = x0^2 + x1^2 + x2^2 + x3^2; group k of a 32-column chunk accumulated over the 4 chunks
        // into S_k; then ((S0 + S1) + (S2 + S3)) + ((S4 + S5) + (S6 + S7)).  A group is columns 8j + 4(quad / 2) + [0, 4): the
        // even lane of a lane pair sums it with its partner's two values, and holds S_k for k = 2 (j % 4) + quad / 2.
        float ss[2][2][4] = {};                                // [row h][128-column partial][j % 4]
#pragma unroll
        for (int c8 = 0; c8 < 32; c8 += 8) {                   // 64 columns at a time: all residual loads before the stores
            float2 xv[2][8];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = row0 + 8 * h;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int col = cb + 8 * (c8 + j) + cq;
                    const float* src = xres + (size_t)row * ldo + col;
                    xv[h][j] = make_float2(0.f, 0.f);
                    if (row < rowsA) {
                        if (col + 1 < rowsB) xv[h][j] = *reinterpret_cast<const float2*>(src);
                        else if (col < rowsB) xv[h][j].x = *src;
                    }
                }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = row0 + 8 * h;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int jj = c8 + j, col = cb + 8 * jj + cq;
                    const float x0 = xv[h][j].x + acc[4 * jj + 2 * h], x1 = xv[h][j].y + acc[4 * jj + 2 * h + 1];
                    if (defer) {                               // all lanes: the shuffle needs the whole warp
                        const float y0 = __shfl_xor_sync(0xffffffffu, x0, 1), y1 = __shfl_xor_sync(0xffffffffu, x1, 1);
                        ss[h][jj >> 4][jj & 3] += x0 * x0 + x1 * x1 + y0 * y0 + y1 * y1;
                    }
                    if (row >= rowsA || col >= rowsB) continue;
                    float* dst = xres + (size_t)row * ldo + col;
                    const bool pair = col + 1 < rowsB;
                    if (pair) *reinterpret_cast<float2*>(dst) = make_float2(x0, x1);
                    else *dst = x0;
                    if (defer) {
                        __nv_bfloat16* hd = rope.xhat + (size_t)row * ldo + col;
                        if (pair) {
                            const uint32_t gw = *reinterpret_cast<const uint32_t*>(rope.gamma + col);
                            *reinterpret_cast<uint32_t*>(hd) = pack_bf16(x0 * bf16_lo(gw), x1 * bf16_hi(gw));
                        } else {
                            *hd = __float2bfloat16(x0 * __bfloat162float(rope.gamma[col]));
                        }
                    }
                }
            }
        }
        if (defer) {
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int p = 0; p < 2; ++p) {
                    float a[4];                                // lane quad 0: S_2m + S_2m+1 (S_2m+1 from quad 2)
#pragma unroll
                    for (int m = 0; m < 4; ++m) a[m] = ss[h][p][m] + __shfl_xor_sync(0xffffffffu, ss[h][p][m], 2);
                    const float v = (a[0] + a[1]) + (a[2] + a[3]);
                    const int row = row0 + 8 * h, part = 2 * b_tile + p;
                    if (quad == 0 && row < rowsA && part * 128 < rowsB) rope.rowss_out[(size_t)row * rope.n_part_out + part] = v;
                }
        }
    } else {
        const float rinv[2] = {pf_rinv(rope, row0, rowsA), pf_rinv(rope, row0 + 8, rowsA)};
        if constexpr (MODE == OUT_ROWMAJOR_ROPE) {
            // two heads of 128 columns of the fused qkv projection: [q heads | k heads | v heads]
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = row0 + 8 * h;
                const int slot = row < rowsA ? rope.slot[row] : -1;
                if (slot < 0) continue;
                const int pos = rope.pos[row];
                const float2* tab = rope.table + (size_t)pos * 64;
                const int page = kv_page(rope.page_table, rope.pages_per_slot, slot, pos);    // one lookup per token row
#pragma unroll
                for (int hb = 0; hb < 2; ++hb) {
                    const int H = b_tile * 2 + hb;
                    if (H * 128 >= rowsB) continue;
                    if (H < rope.n_heads + rope.n_kv_heads) {
                        __nv_bfloat16* dst = H < rope.n_heads
                            ? rope.q_out + (size_t)row * (rope.n_heads * 128) + H * 128
                            : rope.k_cache + kv_page_row(rope.page_table != nullptr, page, rope.n_kv_heads, rope.ctx_max,
                                                         H - rope.n_heads, pos) * 128;
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const int d = 8 * j + cq;
                            const int jl = 16 * hb + j, jh = jl + 8;     // columns d and d + 64 of the head
                            const float4 cs = *reinterpret_cast<const float4*>(tab + d);   // (cos, sin) of d and d + 1
                            const float l0 = acc[4 * jl + 2 * h] * rinv[h], l1 = acc[4 * jl + 2 * h + 1] * rinv[h];
                            const float h0 = acc[4 * jh + 2 * h] * rinv[h], h1 = acc[4 * jh + 2 * h + 1] * rinv[h];
                            *reinterpret_cast<uint32_t*>(dst + d) = pack_bf16(l0 * cs.x - h0 * cs.y, l1 * cs.z - h1 * cs.w);
                            *reinterpret_cast<uint32_t*>(dst + 64 + d) = pack_bf16(h0 * cs.x + l0 * cs.y, h1 * cs.z + l1 * cs.w);
                        }
                    } else {
                        __nv_bfloat16* dst = rope.v_cache + kv_page_row(rope.page_table != nullptr, page, rope.n_kv_heads,
                                                                        rope.ctx_max, H - rope.n_heads - rope.n_kv_heads, pos) * 128;
#pragma unroll
                        for (int j = 0; j < 16; ++j) {
                            const int jj = 16 * hb + j;
                            *reinterpret_cast<uint32_t*>(dst + 8 * j + cq) =
                                pack_bf16(acc[4 * jj + 2 * h] * rinv[h], acc[4 * jj + 2 * h + 1] * rinv[h]);
                        }
                    }
                }
            }
        } else if constexpr (MODE == OUT_ROWMAJOR_SILU) {
            // weight rows interleaved [gate 64 | up 64] per 128: 2 x 64 output columns per tile, ldo = inter
            __nv_bfloat16* act = reinterpret_cast<__nv_bfloat16*>(out);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = row0 + 8 * h;
                if (row >= rowsA) continue;
#pragma unroll
                for (int hb = 0; hb < 2; ++hb) {
                    if (cb + hb * 128 >= rowsB) continue;
                    __nv_bfloat16* dst = act + (size_t)row * ldo + b_tile * 128 + hb * 64 + cq;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const int jg = 16 * hb + j, ju = jg + 8;
                        const float g0 = acc[4 * jg + 2 * h] * rinv[h], g1 = acc[4 * jg + 2 * h + 1] * rinv[h];
                        const float u0 = acc[4 * ju + 2 * h] * rinv[h], u1 = acc[4 * ju + 2 * h + 1] * rinv[h];
                        *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16(silu_mul(g0, u0), silu_mul(g1, u1));
                    }
                }
            }
        } else if constexpr (MODE == OUT_ROWMAJOR_F32) {
            float* c = reinterpret_cast<float*>(out);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = row0 + 8 * h;
                if (row >= rowsA) continue;
                float* dst = c + (size_t)row * ldo;
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    const int col = cb + 8 * j + cq;
                    const float v0 = acc[4 * j + 2 * h] * rinv[h], v1 = acc[4 * j + 2 * h + 1] * rinv[h];
                    if (col + 1 < rowsB) *reinterpret_cast<float2*>(dst + col) = make_float2(v0, v1);
                    else if (col < rowsB) dst[col] = v0;
                }
            }
        } else {
            static_assert(MODE == OUT_ROWMAJOR_BF16, "row-major modes");
            __nv_bfloat16* c = reinterpret_cast<__nv_bfloat16*>(out);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = row0 + 8 * h;
                if (row >= rowsA) continue;
                __nv_bfloat16* dst = c + (size_t)row * ldo;
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    const int col = cb + 8 * j + cq;
                    const float v0 = acc[4 * j + 2 * h] * rinv[h], v1 = acc[4 * j + 2 * h + 1] * rinv[h];
                    if (col + 1 < rowsB) *reinterpret_cast<uint32_t*>(dst + col) = pack_bf16(v0, v1);
                    else if (col < rowsB) dst[col] = __float2bfloat16(v0);
                }
            }
        }
    }
}

template <int MODE>
__global__ void __launch_bounds__(PfCfg::kThreads, 1)
gemm_pf_wgmma(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, void* __restrict__ out,
              int rowsA, int rowsB, int K, int ldo, const RopeEpi rope) {
    constexpr int kStages = PfCfg::kStages;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align_smem_1024(smem_raw);
    uint8_t* smemA = smem;
    uint8_t* smemB = smem + kStages * PfCfg::kStageBytesA;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * PfCfg::kStageBytes);
    uint64_t* empty_bar = full_bar + kStages;

    const int wg = threadIdx.x >> 7;
    griddep_launch();
    const int tr_slot = trace_begin(TR_GEMM_PF);
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], PfCfg::kConsumerWarps);     // one arrival per consumer warp
        }
        fence_barrier_init();
    }
    __syncthreads();

    WorkSched sched;
    sched.init(rowsA, rowsB, K, 1, PfCfg::kTileB);
    WorkItem t;
    if (wg == 0) {
        // ===================== TMA producer (one thread of warpgroup 0) =====================
        setmaxnreg_dec<PfCfg::kProducerRegs>();
        if (threadIdx.x < 32 && elect_one()) {
            const uint64_t pol = l2_policy_evict_last();     // both operands are re-read by other tiles
            int stage = 0;
            uint32_t phase = 0;
            bool have = sched.next(t);
            // PDL: the weight stages of the first item go out before the activations are known to exist
            int pre = 0;
            if (have) {
                pre = min(kStages, t.kb1 - t.kb0);
                for (int i = 0; i < pre; ++i) {
                    mbar_arrive_expect_tx(&full_bar[i], PfCfg::kStageBytes);
                    tma_load_2d_hint(smemB + i * PfCfg::kStageBytesB, &tmB, &full_bar[i], (t.kb0 + i) * BLOCK_K,
                                     t.b_tile * PfCfg::kTileB, pol);
                }
            }
            griddep_wait();
            trace_dep(tr_slot);
            if (have) {
                for (int i = 0; i < pre; ++i)
                    tma_load_2d_hint(smemA + i * PfCfg::kStageBytesA, &tmA, &full_bar[i], (t.kb0 + i) * BLOCK_K,
                                     t.a_tile * BLOCK_A, pol);
                t.kb0 += pre;
                stage = pre % kStages;
                phase = (pre == kStages) ? 1u : 0u;
            }
            while (have) {
                for (int kb = t.kb0; kb < t.kb1; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_arrive_expect_tx(&full_bar[stage], PfCfg::kStageBytes);
                    tma_load_2d_hint(smemA + stage * PfCfg::kStageBytesA, &tmA, &full_bar[stage], kb * BLOCK_K,
                                     t.a_tile * BLOCK_A, pol);
                    tma_load_2d_hint(smemB + stage * PfCfg::kStageBytesB, &tmB, &full_bar[stage], kb * BLOCK_K,
                                     t.b_tile * PfCfg::kTileB, pol);
                    if (++stage == kStages) { stage = 0; phase ^= 1; }
                }
                have = sched.next(t);
            }
        }
    } else {
        // ===================== consumer warpgroups: rows [64 (wg - 1), 64 wg) of the tile =====================
        setmaxnreg_inc<PfCfg::kConsumerRegs>();
        const int cw = wg - 1;
        const int wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
        const bool arrive = lane == 0;
        const uint32_t smemA_u = smem_u32(smemA) + cw * (64 * BLOCK_K * 2), smemB_u = smem_u32(smemB);
        griddep_wait();                               // `out` may still be read by the preceding kernel
        int stage = 0;
        uint32_t phase = 0;
        while (sched.next(t)) {
            float acc[128];
            int prev = -1;
            wgmma_fence_regs(acc);
            for (int kb = t.kb0; kb < t.kb1; ++kb) {
                mbar_wait(&full_bar[stage], phase);
                const uint64_t da = gmma_desc_sw128(smemA_u + stage * PfCfg::kStageBytesA);
                const uint64_t db = gmma_desc_sw128(smemB_u + stage * PfCfg::kStageBytesB);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BLOCK_K / GMMA_K; ++k)
                    wgmma_ss<256>(acc, da + 2 * k, db + 2 * k, (kb > t.kb0 || k > 0) ? 1u : 0u);
                wgmma_commit();
                wgmma_wait<1>();                      // the group of the previous k-block has retired: release its slot
                if (prev >= 0 && arrive) mbar_arrive(&empty_bar[prev]);
                prev = stage;
                if (++stage == kStages) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            wgmma_fence_regs(acc);
            if (prev >= 0 && arrive) mbar_arrive(&empty_bar[prev]);
            const int row0 = t.a_tile * BLOCK_A + cw * 64 + wq * 16 + (lane >> 2);
            pf_epilogue<MODE>(acc, row0, t.b_tile, lane & 3, out, rowsA, rowsB, ldo, rope);
        }
    }
    __syncthreads();
    trace_end(tr_slot);
}

// =================================================================================================
// Fused decode MLP: act = SiLU(x Wg^T) * (x Wu^T), planes = act Wd^T in ONE persistent launch (decode orientation,
// weights on the wgmma M side).  Same warp roles and smem ring as gemm_bf16_wgmma; the pipeline
// state simply carries from item to item.  Each CTA runs its gate/up tiles from a host-built list, then its down items:
// drawn from a device counter (a.dyn, default) or from the same list (static schedule, RR_MLP_STATIC).
// A down item = (128 output features, one K-slice of `slice_kb` k-blocks); k-block kb of the down GEMM is
// exactly the 64 act columns gate/up tile kb writes, so the item only depends on the tiles of its slice: the gate/up
// epilogue (TMA store of the act tile, completion wait, fence) bumps ready[slice] and the producer of a down item requests
// the WEIGHT tiles of its first stages, then acquires ready[slice] == slice length, then requests the activation tiles.
// No kernel boundary,
// no wave-quantisation tail of the gate/up grid (224 tiles on 132 SMs): CTAs that own one gate/up tile start on the
// early slices while the others finish their second tile.
__device__ __forceinline__ unsigned ld_acquire_gpu_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

template <int BN, bool FP8 = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_mlp_wgmma(const __grid_constant__ MlpArgs a) {
    using Cfg = GemmCfg<BN, 8, FP8>;
    constexpr int kStages = Cfg::kStages;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align_smem_1024(smem_raw);
    uint8_t* smemA = smem + Cfg::kRingOff;
    uint8_t* smemB = smemA + kStages * Cfg::kStageBytesA;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kBarOff);
    uint64_t* empty_bar = full_bar + kStages;
    volatile int* dyn_q = reinterpret_cast<volatile int*>(smem + Cfg::kBarOff + 176);   // [16] dynamic down items of this CTA
    float* acc_tile = reinterpret_cast<float*>(smem + Cfg::kAccOff);
    float* silu_stage = reinterpret_cast<float*>(smem + Cfg::kEpiOff);    // exchange; aliased by the planes tile
    __nv_bfloat16* act_stage = reinterpret_cast<__nv_bfloat16*>(smem + Cfg::kEpiOff + Cfg::kSiluStageBytes);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    griddep_launch();
    const int tr_slot = trace_begin(TR_GEMM_DEC);

    if (warp == PRODUCER_WARP && elect_one()) {
        tma_prefetch_desc(&a.tmA0); tma_prefetch_desc(&a.tmB0);
        tma_prefetch_desc(&a.tmA1); tma_prefetch_desc(&a.tmB1);
        if (a.tma_epi) { tma_prefetch_desc(&a.tmAct); tma_prefetch_desc(&a.tmPlanes); }
        for (int s = 0; s < kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], GEMM_CONSUMERS / 32); }
        for (int s = 0; s < 16; ++s) dyn_q[s] = -2;
        fence_barrier_init();
    }
    __syncthreads();

    const int4* my = reinterpret_cast<const int4*>(a.items) + (size_t)blockIdx.x * a.max_items;   // constant data
    auto get = [&](int i, WorkItem& t, int& ph) -> bool {
        if (i >= a.max_items) return false;
        const int4 v = __ldg(my + i);
        if (v.x < 0) return false;
        ph = v.x >> 16; t.a_tile = v.x & 0xffff; t.b_tile = 0; t.kb0 = v.y; t.kb1 = v.z; t.z = v.w;
        return true;
    };
    // Down items are not in the static lists when a.dyn: after its gate/up tiles a CTA takes the next item q of the slice-major
    // order (z = q / tiles1) from a global counter, so the split follows the real finishing order instead of a host-side time
    // model (the static list schedule left a 10 us tail: CTAs with three down items next to CTAs with one).  The producer thread
    // draws q -- when the last load of the current item is out, so the round trip of the atomic overlaps the drain of the ring and
    // no CTA sits on an item it cannot start -- and publishes it to the consumer warpgroup through dyn_q[] (-2 = not drawn yet,
    // -1 = no more work).  Which CTA computes an item does not change a single bit of its plane tile.
    auto dyn_decode = [&](int q, WorkItem& t, int& ph) {
        const int z = q / a.tiles1;
        t.a_tile = q - z * a.tiles1; t.b_tile = 0; t.kb0 = z * a.slice_kb;
        t.kb1 = min(t.kb0 + a.slice_kb, a.kb1n); t.z = z; ph = 1;
    };
    auto next_consumer = [&](int it, int& nstat, WorkItem& t, int& ph) -> bool {
        if (nstat < 0) {
            if (get(it, t, ph)) return true;
            nstat = it;
        }
        if (!a.dyn) return false;
        const int d = it - nstat;
        if (d >= 16) return false;
        int q;
        do { q = dyn_q[d]; } while (q == -2);
        if (q < 0) return false;
        dyn_decode(q, t, ph);
        return true;
    };
    WorkItem t;
    int ph = 0;

    if (warp == PRODUCER_WARP) {
        // ===================== TMA producer =====================
        if (elect_one()) {
            const uint64_t polA = l2_policy_evict_first(), polB = l2_policy_evict_last();
            int stage = 0;
            uint32_t phase = 0;
            bool first = true;
            int tm_i = 0;
            trace_mark_fixed(TR_MLP_MARK + 0, tm_i++);
            int nstat = -1;
            unsigned q_next = 0;
            bool have_next = false;
            for (int i = 0;; ++i) {
                if (nstat < 0 && !get(i, t, ph)) nstat = i;
                if (nstat >= 0) {
                    if (!a.dyn) break;
                    const int d = i - nstat;
                    if (d >= 16) break;
                    if (first) { griddep_wait(); trace_dep(tr_slot); first = false; }    // the counter is zeroed by the preceding kernel
                    const unsigned q = have_next ? q_next : atomicAdd(a.ready + a.n_slices, 1u);
                    have_next = false;
                    if (q >= (unsigned)a.n_down) { dyn_q[d] = -1; break; }
                    dyn_q[d] = (int)q;
                    dyn_decode((int)q, t, ph);
                }
                const CUtensorMap* tA = ph ? &a.tmA1 : &a.tmA0;
                const CUtensorMap* tB = ph ? &a.tmB1 : &a.tmB0;
                // weight tiles of the first stages go out before the activations are known to exist: at the start
                // of the kernel (PDL: the preceding kernel is still running) and for every down item (its slice of
                // act may still be in flight on other SMs)
                const int pre = (first || ph) ? min(kStages, t.kb1 - t.kb0) : 0;
                const int st0 = stage;
                for (int j = 0; j < pre; ++j) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
                    tma_load_2d_hint(smemA + stage * Cfg::kStageBytesA, tA, &full_bar[stage], (t.kb0 + j) * BLOCK_K,
                                     t.a_tile * BLOCK_A, polA);
                    if (++stage == kStages) { stage = 0; phase ^= 1; }
                }
                if (first) { griddep_wait(); trace_dep(tr_slot); first = false; trace_mark_fixed(TR_MLP_MARK + 1, tm_i++); }
                if (ph) {
                    const unsigned need = (unsigned)(t.kb1 - t.kb0);
                    trace_mark_fixed(TR_MLP_MARK + 2, tm_i++);
                    while (ld_acquire_gpu_u32(a.ready + t.z) < need) {
                    }
                    asm volatile("fence.proxy.async;" ::: "memory");   // other SMs' generic-proxy stores -> our TMA reads
                    trace_mark_fixed(TR_MLP_MARK + 3, tm_i++);
                }
                for (int j = 0, s2 = st0; j < pre; ++j) {
                    tma_load_2d_hint(smemB + s2 * Cfg::kStageBytesB, tB, &full_bar[s2], (t.kb0 + j) * BLOCK_K, 0, polB);
                    if (++s2 == kStages) s2 = 0;
                }
                for (int kb = t.kb0 + pre; kb < t.kb1; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
                    tma_load_2d_hint(smemA + stage * Cfg::kStageBytesA, tA, &full_bar[stage], kb * BLOCK_K, t.a_tile * BLOCK_A, polA);
                    tma_load_2d_hint(smemB + stage * Cfg::kStageBytesB, tB, &full_bar[stage], kb * BLOCK_K, 0, polB);
                    if (++stage == kStages) { stage = 0; phase ^= 1; }
                }
                if (a.dyn) {                       // the next item is a dynamic one: draw it now
                    WorkItem tn; int pn;
                    const bool next_static = nstat < 0 && get(i + 1, tn, pn);
                    const int dn = nstat < 0 ? 0 : i + 1 - nstat;
                    if (!next_static && dn < 16) { q_next = atomicAdd(a.ready + a.n_slices, 1u); have_next = true; }
                }
            }
        }
    } else {
        // ===================== consumer warpgroup: wgmma main loop + epilogue (warps 0..3) =====================
        const int quarter = warp;
        const int row_in_tile = quarter * 32 + lane;
        const int etid = threadIdx.x;
        const uint32_t smemA_u = smem_u32(smemA), smemB_u = smem_u32(smemB);
        int stage = 0;
        uint32_t phase = 0;
        griddep_wait();
        trace_dep(tr_slot);
        int nstat = -1;
        Fp8Conv cv{smemA, smem, 0, {}};
        for (int it = 0; next_consumer(it, nstat, t, ph); ++it) {
            if (etid == 0) trace_mark_fixed(TR_MLP_MARK + 4 + ph, 64 + it);
            float acc[2][BN / 2];
            if constexpr (FP8) cv.load_scales(ph ? a.sc1 : a.sc0, t.a_tile, ph ? a.hidden : 2 * a.inter);
            gmma_mainloop<BN, FP8>(acc, smemA_u, smemB_u, full_bar, empty_bar, stage, phase, t.kb1 - t.kb0, kStages, &cv);
            if (etid == 0) trace_mark_fixed(TR_MLP_MARK + 6 + ph, 128 + 4 * it);
            acc_bar();
            stage_acc<BN>(acc, acc_tile);
            acc_bar();
            const int a_row = t.a_tile * BLOCK_A + row_in_tile;
            const float* arow = acc_tile + row_in_tile * Cfg::kAccPitch;
            bool tma_done = false;
            if constexpr (BN <= 64) {
                if (a.tma_epi) {
                    if (ph == 0) epilogue_silu_tma<BN>(arow, t, quarter, lane, etid, &a.tmAct, silu_stage, act_stage);
                    else epilogue_planes_tma<BN>(arow, t, quarter, lane, etid, &a.tmPlanes, silu_stage);
                    tma_done = true;
                }
            }
            if (tma_done) {
            } else if (ph == 0)
                epilogue_item<BN, OUT_TRANSPOSED_SILU>(arow, a_row, t, quarter, lane, a.act, 2 * a.inter, a.rows, a.inter, 0,
                                                       silu_stage);
            else
                epilogue_item<BN, OUT_TRANSPOSED_F32>(arow, a_row, t, quarter, lane, a.out1, a.hidden, a.rows, a.hidden,
                                                      a.ld_rows, nullptr);
            if (etid == 0) trace_mark_fixed(TR_MLP_MARK + 10, 128 + 4 * it + 1);      // stores issued
            if (ph == 0) {
                // publish this tile's 64 act columns: every epilogue thread's stores, then one release-increment
                if (tma_done) {
                    if (etid == 0) {
                        bulk_wait0();                                                  // the bulk store's writes are performed
                        trace_mark_fixed(TR_MLP_MARK + 11, 128 + 4 * it + 2);
                        asm volatile("fence.proxy.async;" ::: "memory");
                        __threadfence();
                        atomicAdd(a.ready + t.a_tile / a.slice_kb, 1u);
                        trace_mark_fixed(TR_MLP_MARK + 8, 128 + 4 * it + 3);
                    }
                } else {
                    asm volatile("bar.sync 3, 128;" ::: "memory");
                    if (etid == 0) {
                        trace_mark_fixed(TR_MLP_MARK + 11, 128 + 4 * it + 2);          // all epilogue threads past their stores
                        __threadfence();
                        atomicAdd(a.ready + t.a_tile / a.slice_kb, 1u);
                        trace_mark_fixed(TR_MLP_MARK + 8, 128 + 4 * it + 3);
                    }
                }
            }
        }
    }

    if (a.tma_epi && threadIdx.x == 0) bulk_wait_read0();   // epilogue thread 0: the staging tile must outlive the reads of its stores
    __syncthreads();
    trace_end(tr_slot);
}

// ---------------------------------------------------------------- host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
        if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = (PFN_encodeTiled)p;
    });
    return fn;
}

// [rows, K] bf16 row-major (K contiguous, row pitch ld elements) -> TMA map with box {64, box_rows}.
int make_tmap_bf16_2d(CUtensorMap* map, const void* base, int rows, int K, int ld, int box_rows) {
    PFN_encodeTiled enc = get_encode_fn();
    if (!enc) return RR_ERR_CUDA;
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {(cuuint32_t)BLOCK_K, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides,
                     box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? RR_OK : RR_ERR_CUDA;
}

// [rows, K] e4m3 row-major (row pitch ld bytes) -> TMA map with box {64 bytes, box_rows}, no swizzle (the FP8 ring slot).
// The caller has checked fp8_weight_ok and ld % 16 == 0: TMA needs a 16-byte aligned base and pitch, and a box row of 64
// bytes is a multiple of 16.
static int make_tmap_e4m3_2d(CUtensorMap* map, const void* base, int rows, int K, int ld, int box_rows) {
    PFN_encodeTiled enc = get_encode_fn();
    if (!enc) return RR_ERR_CUDA;
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld};
    cuuint32_t box[2] = {(cuuint32_t)BLOCK_K, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? RR_OK : RR_ERR_CUDA;
}

// planes P[z][b][n] fp32 (n contiguous, row pitch ldo, plane pitch ld_rows * ldo), valid n < n_valid, b < rows_valid:
// 3-D map {n, b, z}, box {128, box_rows, 1}, no swizzle -- the destination of epilogue_planes_tma
int make_tmap_planes_f32(CUtensorMap* map, const void* base, int n_valid, int ldo, int rows_valid, int ld_rows, int splits, int box_rows) {
    PFN_encodeTiled enc = get_encode_fn();
    if (!enc) return RR_ERR_CUDA;
    cuuint64_t dims[3] = {(cuuint64_t)n_valid, (cuuint64_t)rows_valid, (cuuint64_t)splits};
    cuuint64_t strides[2] = {(cuuint64_t)ldo * 4, (cuuint64_t)ld_rows * ldo * 4};
    cuuint32_t box[3] = {128, (cuuint32_t)box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? RR_OK : RR_ERR_CUDA;
}
// act[b][n] bf16 (row pitch ld): 2-D map {n, b}, box {64, box_rows}, no swizzle -- the destination of epilogue_silu_tma
int make_tmap_act_store(CUtensorMap* map, const void* base, int rows, int n, int ld, int box_rows) {
    PFN_encodeTiled enc = get_encode_fn();
    if (!enc) return RR_ERR_CUDA;
    cuuint64_t dims[2] = {(cuuint64_t)n, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? RR_OK : RR_ERR_CUDA;
}

static bool rowmajor(int mode) {
    return mode == OUT_ROWMAJOR_BF16 || mode == OUT_ROWMAJOR_SILU || mode == OUT_ROWMAJOR_ROPE || mode == OUT_ROWMAJOR_RESID ||
           mode == OUT_ROWMAJOR_F32;
}

static std::atomic<int> g_num_sms[64];
int num_sms() {                         // of the current device (one process may drive several)
    int dev = 0;
    cudaGetDevice(&dev);
    int n = g_num_sms[dev & 63].load(std::memory_order_relaxed);
    if (!n) {
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        g_num_sms[dev & 63].store(n, std::memory_order_relaxed);
    }
    return n;
}

template <int BN, int MODE, bool FP8 = false>
static int launch_one(const GemmPlan& p, cudaStream_t st) {
    constexpr int CAP = 8;
    auto kern = gemm_bf16_wgmma<BN, MODE, CAP, FP8>;
    static std::atomic<uint64_t> attr_set{0};
    static_assert(gemm_smem_bytes<BN, MODE, CAP, FP8>() <= 227 * 1024, "decode GEMM: shared memory budget");
    if (ensure_dyn_smem(kern, (int)gemm_smem_bytes<BN, MODE, CAP, FP8>(), attr_set) != cudaSuccess) return RR_ERR_CUDA;
    const int tilesA = (p.rowsA + BLOCK_A - 1) / BLOCK_A;
    const int tilesB = (p.rowsB + BN - 1) / BN;
    const int n_work = tilesA * tilesB * p.splits;
    const int grid = n_work < num_sms() ? n_work : num_sms();
    cudaError_t le = launch_pdl(kern, dim3(grid), dim3(GEMM_THREADS), (size_t)gemm_smem_bytes<BN, MODE, CAP, FP8>(), st, p.tmA,
                                p.tmB, p.out, p.rowsA, p.rowsB, p.K, p.splits, p.ldo, p.ld_rows, p.tmOut, p.tma_epi, p.scaleA);
    return (le == cudaSuccess && cudaGetLastError() == cudaSuccess) ? RR_OK : RR_ERR_CUDA;
}

template <int MODE>
static int launch_pf(const GemmPlan& p, cudaStream_t st, bool pdl) {
    auto kern = gemm_pf_wgmma<MODE>;
    static std::atomic<uint64_t> attr_set{0};
    if (ensure_dyn_smem(kern, PfCfg::kSmemBytes, attr_set) != cudaSuccess) return RR_ERR_CUDA;
    const int tilesA = (p.rowsA + BLOCK_A - 1) / BLOCK_A;
    const int tilesB = (p.rowsB + PfCfg::kTileB - 1) / PfCfg::kTileB;
    const int n_work = tilesA * tilesB;
    const int grid = n_work < num_sms() ? n_work : num_sms();
    cudaError_t le = launch_ex(pdl ? g_use_pdl : 0, kern, dim3(grid), dim3(PfCfg::kThreads), (size_t)PfCfg::kSmemBytes, st, p.tmA,
                               p.tmB, p.out, p.rowsA, p.rowsB, p.K, p.ldo, p.rope);
    return (le == cudaSuccess && cudaGetLastError() == cudaSuccess) ? RR_OK : RR_ERR_CUDA;
}

// splits >= 1: uniform split-K with `splits` planes.  Decode orientation: bn = 256 is accepted and runs 128-wide tiles (a
// consumer warpgroup holds at most 128 x 128 fp32 accumulators in registers).  Row-major (prefill) modes always run the
// 128 x 256 tiles of gemm_pf_wgmma; their bn is only validated.
int gemm_plan_init(GemmPlan* p, const void* A, int rowsA, int ldA, const void* B, int rowsB, int ldB,
                   int K, void* out, int ldo, int ld_rows, int splits, int mode, int bn) {
    if (K % 8 != 0 || ldA % 8 != 0 || ldB % 8 != 0) return RR_ERR_ARG;
    if (!(bn == 16 || bn == 32 || bn == 64 || bn == 128 || bn == 256)) return RR_ERR_ARG;
    const int kblocks = (K + BLOCK_K - 1) / BLOCK_K;
    if (splits < 1) return RR_ERR_ARG;
    if (splits > kblocks) splits = kblocks;
    if (mode == OUT_ROWMAJOR_BF16 && (splits != 1 || ldo % 8 != 0)) return RR_ERR_ARG;
    // fused SiLU*mul epilogues: weights row-interleaved in 64-row gate/up blocks, one plane, bf16 act output
    if (mode == OUT_TRANSPOSED_SILU && (splits != 1 || bn < 32 || rowsA % 128 != 0)) return RR_ERR_ARG;
    if (mode == OUT_ROWMAJOR_SILU && (splits != 1 || bn < 128 || rowsB % 128 != 0 || ldo % 8 != 0)) return RR_ERR_ARG;
    if (mode == OUT_ROWMAJOR_ROPE && (splits != 1 || bn < 128 || rowsB % 128 != 0)) return RR_ERR_ARG;
    if (bn > MAX_BN) bn = MAX_BN;
    if (mode == OUT_ROWMAJOR_RESID && (splits != 1 || bn < 32 || ldo % 4 != 0)) return RR_ERR_ARG;
    // fp32 pairs are stored 8-byte aligned
    if (mode == OUT_ROWMAJOR_F32 && (splits != 1 || ldo % 2 != 0 || ((uintptr_t)out & 7) != 0)) return RR_ERR_ARG;
    if (mode < 0 || mode > OUT_ROWMAJOR_F32) return RR_ERR_ARG;
    memset(&p->rope, 0, sizeof(p->rope));
    p->rowsA = rowsA; p->rowsB = rowsB; p->K = K; p->out = out; p->ldo = ldo; p->ld_rows = ld_rows;
    p->splits = splits; p->mode = mode; p->bn = bn; p->max_ctas = 0; p->scaleA = nullptr;
    int rc = make_tmap_bf16_2d(&p->tmA, A, rowsA, K, ldA, BLOCK_A);
    if (rc != RR_OK) return rc;
    // decode planes through one TMA store per item: needs 16-byte pitches and at most 64 batch columns per tile
    p->tma_epi = 0;
    if (mode == OUT_TRANSPOSED_F32 && bn <= 64 && ldo % 4 == 0 && ((uintptr_t)out & 15) == 0 && !getenv("RR_NO_TMA_EPI")) {
        rc = make_tmap_planes_f32(&p->tmOut, out, rowsA, ldo, rowsB, ld_rows > 0 ? ld_rows : rowsB, splits, bn);
        if (rc != RR_OK) return rc;
        p->tma_epi = 1;
    }
    return make_tmap_bf16_2d(&p->tmB, B, rowsB, K, ldB, rowmajor(mode) ? PfCfg::kTileB : bn);
}

int gemm_plan_init_fp8w(GemmPlan* p, const void* A, const float* scale, int rowsA, int ldA, const void* B, int rowsB,
                        int ldB, int K, void* out, int ldo, int ld_rows, int splits, int mode, int bn) {
    if (mode != OUT_TRANSPOSED_F32 && mode != OUT_TRANSPOSED_SILU) return RR_ERR_ARG;
    if (!scale || !fp8_weight_ok(A, K) || ldA < K || ldA % 16 != 0 || rowsA < 1) return RR_ERR_ARG;
    // the bf16 plan on a stand-in A of the same shape, then the e4m3 map of the real one
    int rc = gemm_plan_init(p, A, rowsA, ldA, B, rowsB, ldB, K, out, ldo, ld_rows, splits, mode, bn);
    if (rc != RR_OK) return rc;
    rc = make_tmap_e4m3_2d(&p->tmA, A, rowsA, K, ldA, BLOCK_A);
    if (rc != RR_OK) return rc;
    p->scaleA = scale;
    return RR_OK;
}

int gemm_launch(const GemmPlan& p, cudaStream_t st, bool pdl) {
    switch (p.mode) {
        case OUT_ROWMAJOR_BF16: return launch_pf<OUT_ROWMAJOR_BF16>(p, st, pdl);
        case OUT_ROWMAJOR_SILU: return launch_pf<OUT_ROWMAJOR_SILU>(p, st, pdl);
        case OUT_ROWMAJOR_ROPE: return launch_pf<OUT_ROWMAJOR_ROPE>(p, st, pdl);
        case OUT_ROWMAJOR_RESID: return launch_pf<OUT_ROWMAJOR_RESID>(p, st, pdl);
        case OUT_ROWMAJOR_F32: return launch_pf<OUT_ROWMAJOR_F32>(p, st, pdl);
    }
#define RR_CASE(BN_)                                                                                            \
    case BN_:                                                                                                   \
        if (p.scaleA) {                                                                                         \
            if (p.mode == OUT_TRANSPOSED_F32) return launch_one<BN_, OUT_TRANSPOSED_F32, true>(p, st);           \
            if constexpr (BN_ >= 32) {                                                                          \
                if (p.mode == OUT_TRANSPOSED_SILU) return launch_one<BN_, OUT_TRANSPOSED_SILU, true>(p, st);     \
            }                                                                                                   \
            return RR_ERR_ARG;                                                                                  \
        }                                                                                                       \
        if (p.mode == OUT_TRANSPOSED_F32) return launch_one<BN_, OUT_TRANSPOSED_F32>(p, st);                     \
        if constexpr (BN_ >= 32) {                                                                              \
            if (p.mode == OUT_TRANSPOSED_SILU) return launch_one<BN_, OUT_TRANSPOSED_SILU>(p, st);               \
        }                                                                                                       \
        return RR_ERR_ARG;
    switch (p.bn) {
        RR_CASE(16)
        RR_CASE(32)
        RR_CASE(64)
        RR_CASE(128)
    }
#undef RR_CASE
    return RR_ERR_ARG;
}


int pick_bn(int rows) {
    const int opts[4] = {16, 32, 64, MAX_BN};
    for (int b : opts) if (rows <= b) return b;
    return MAX_BN;
}

int pick_splits(int rows_w, int K) {
    const int tilesA = (rows_w + 127) / 128;
    int s = num_sms() / tilesA;
    const int kblocks = (K + 63) / 64;
    if (s < 1) s = 1;
    if (s > 8) s = 8;
    while (s > 1 && kblocks / s < 8) --s;
    return s;
}

int decode_plan_init(GemmPlan* p, const void* W, const float* scale, int rows_w, int K, const void* X, int rows, void* out,
                     int ldo, int splits, int mode) {
    const int bn = pick_bn(rows);
    return scale ? gemm_plan_init_fp8w(p, W, scale, rows_w, K, X, rows, K, K, out, ldo, rows, splits, mode, bn)
                 : gemm_plan_init(p, W, rows_w, K, X, rows, K, K, out, ldo, rows, splits, mode, bn);
}

// ---- fused decode MLP: host side ------------------------------------------------------------------
int mlp_slices(int inter, int* slice_kb) {
    const int kb1n = inter / BLOCK_K;
    if (kb1n < 1) { *slice_kb = 0; return 0; }
    int n_sl = (kb1n + 15) / 16;
    n_sl = n_sl > 8 ? 8 : n_sl;
    *slice_kb = (kb1n + n_sl - 1) / n_sl;
    return (kb1n + *slice_kb - 1) / *slice_kb;
}

// List schedule on a time line in units of k-blocks (one 16 KB weight tile at a CTA's fair share of the HBM rate, 0.37 us;
// + a fixed per-item cost for pipeline refill / epilogue).  Gate/up tile t goes to CTA t % grid (wave order: tile t is
// finished before tile t + grid).  A slice becomes READY kPublish units after its last gate/up tile finished its mainloop --
// the measured epilogue -> TMA store -> fence -> counter -> acquire chain (tools/trace_mlp.py: ~10 us).  The down items, slice by
// slice, go to the CTA that can START them first, max(CTA free, slice ready); among CTAs that would all wait, the one that
// has been free for the shortest time (best fit).  With the earlier "least loaded CTA" rule every early slice went to the CTAs
// that own one gate/up tile, and the CTAs that own two found only late slices when they finished: they all stalled for one
// publish latency (RR_MLP_SCHED_P=0 restores that rule).
int mlp_schedule(int grid, int inter, int hidden, int slice_kb, std::vector<MlpItem>* items, int dynamic) {
    const int tiles0 = (2 * inter) / BLOCK_A, kb0n = (hidden + BLOCK_K - 1) / BLOCK_K;
    const int tiles1 = (hidden + BLOCK_A - 1) / BLOCK_A, kb1n = inter / BLOCK_K;
    const int n_slices = (kb1n + slice_kb - 1) / slice_kb;
    constexpr int kItemCost = 6;
    const char* pe = getenv("RR_MLP_SCHED_P");
    const long long kPublish = pe ? atoi(pe) : 27;
    std::vector<std::vector<MlpItem>> per(grid);
    std::vector<long long> load(grid, 0);
    std::vector<long long> tile_done(tiles0, 0);
    for (int t = 0; t < tiles0; ++t) {
        MlpItem it; it.tile_phase = t; it.kb0 = 0; it.kb1 = kb0n; it.z = 0;
        per[t % grid].push_back(it);
        load[t % grid] += kb0n + kItemCost;
        tile_done[t] = load[t % grid];
    }
    for (int z = 0; z < (dynamic ? 0 : n_slices); ++z) {          // dynamic: the kernel deals the down items itself
        const int k0 = z * slice_kb, k1 = (k0 + slice_kb < kb1n) ? k0 + slice_kb : kb1n;
        long long ready = 0;
        if (kPublish > 0) {
            for (int t = k0; t < k1 && t < tiles0; ++t) ready = tile_done[t] > ready ? tile_done[t] : ready;
            ready += kPublish;
        }
        for (int tl = 0; tl < tiles1; ++tl) {
            int best = 0;
            for (int c = 1; c < grid; ++c) {
                const long long sc = load[c] > ready ? load[c] : ready, sb = load[best] > ready ? load[best] : ready;
                if (sc < sb || (sc == sb && load[c] > load[best])) best = c;
            }
            MlpItem it; it.tile_phase = tl | (1 << 16); it.kb0 = k0; it.kb1 = k1; it.z = z;
            per[best].push_back(it);
            load[best] = (load[best] > ready ? load[best] : ready) + (k1 - k0) + kItemCost;
        }
    }
    size_t mx = 1;
    for (auto& v : per) mx = v.size() > mx ? v.size() : mx;
    items->assign((size_t)grid * mx, MlpItem{-1, 0, 0, 0});
    for (int c = 0; c < grid; ++c)
        for (size_t i = 0; i < per[c].size(); ++i) (*items)[(size_t)c * mx + i] = per[c][i];
    return (int)mx;
}

int mlp_plan_init(MlpPlan* p, const void* Wgu, const void* Wd, int inter, int hidden, const void* xn, int rows,
                  void* act, void* planes, int ld_rows, int bn, const MlpItem* items_dev, int max_items, int grid,
                  unsigned* ready, int slice_kb, int dynamic, const float* sc_gu, const float* sc_down) {
    if (!p || !Wgu || !Wd || !xn || !act || !planes || !items_dev || !ready) return RR_ERR_ARG;
    if (inter % 64 || (2 * inter) % BLOCK_A || hidden % 8 || rows > bn || bn < 32 || bn > MAX_BN || slice_kb < 1) return RR_ERR_ARG;
    if ((2 * inter) / BLOCK_A > 0xffff || grid < 1 || grid > num_sms()) return RR_ERR_ARG;
    const bool fp8 = sc_gu || sc_down;
    if (fp8 && (!sc_gu || !sc_down || !fp8_weight_ok(Wgu, hidden) || !fp8_weight_ok(Wd, inter))) return RR_ERR_ARG;
    MlpArgs& a = p->args;
    int rc = fp8 ? make_tmap_e4m3_2d(&a.tmA0, Wgu, 2 * inter, hidden, hidden, BLOCK_A)
                 : make_tmap_bf16_2d(&a.tmA0, Wgu, 2 * inter, hidden, hidden, BLOCK_A);
    if (rc == RR_OK) rc = make_tmap_bf16_2d(&a.tmB0, xn, rows, hidden, hidden, bn);
    if (rc == RR_OK) rc = fp8 ? make_tmap_e4m3_2d(&a.tmA1, Wd, hidden, inter, inter, BLOCK_A)
                              : make_tmap_bf16_2d(&a.tmA1, Wd, hidden, inter, inter, BLOCK_A);
    if (rc == RR_OK) rc = make_tmap_bf16_2d(&a.tmB1, act, rows, inter, inter, bn);
    if (rc != RR_OK) return rc;
    a.act = (__nv_bfloat16*)act; a.out1 = (float*)planes; a.inter = inter; a.hidden = hidden; a.rows = rows;
    a.ld_rows = ld_rows; a.items = items_dev; a.max_items = max_items; a.ready = ready; a.slice_kb = slice_kb;
    a.kb1n = inter / BLOCK_K; a.tiles1 = (hidden + BLOCK_A - 1) / BLOCK_A;
    a.n_slices = (a.kb1n + slice_kb - 1) / slice_kb; a.n_down = a.n_slices * a.tiles1; a.dyn = dynamic ? 1 : 0;
    a.sc0 = sc_gu; a.sc1 = sc_down;
    p->grid = grid; p->bn = bn; p->n_slices = (inter / BLOCK_K + slice_kb - 1) / slice_kb; p->fp8 = fp8 ? 1 : 0;
    a.tma_epi = 0;
    if (bn <= 64 && hidden % 4 == 0 && inter % 8 == 0 && ((uintptr_t)planes & 15) == 0 && ((uintptr_t)act & 15) == 0 &&
        !getenv("RR_NO_TMA_EPI")) {
        rc = make_tmap_act_store(&a.tmAct, act, rows, inter, inter, bn);
        if (rc == RR_OK) rc = make_tmap_planes_f32(&a.tmPlanes, planes, hidden, hidden, rows, ld_rows, p->n_slices, bn);
        if (rc != RR_OK) return rc;
        a.tma_epi = 1;
    }
    return RR_OK;
}

template <int BN, bool FP8 = false>
static int launch_mlp_bn(const MlpPlan& p, cudaStream_t st) {
    auto kern = gemm_mlp_wgmma<BN, FP8>;
    static std::atomic<uint64_t> attr_set{0};
    constexpr int smem = GemmCfg<BN, 8, FP8>::kSmemBytes + mlp_stage_bytes<BN>();
    static_assert(smem <= 227 * 1024, "fused MLP kernel: shared memory budget");
    if (ensure_dyn_smem(kern, smem, attr_set) != cudaSuccess) return RR_ERR_CUDA;
    cudaError_t e = launch_pdl(kern, dim3(p.grid), dim3(GEMM_THREADS), (size_t)smem, st, p.args);
    return e == cudaSuccess ? RR_OK : RR_ERR_CUDA;
}
// Requires all CTAs co-resident (grid <= SM count; one CTA per SM by shared memory) and ready[] zero at launch.
int mlp_launch(const MlpPlan& p, cudaStream_t st) {
    if (p.fp8) {
        switch (p.bn) {
            case 32: return launch_mlp_bn<32, true>(p, st);
            case 64: return launch_mlp_bn<64, true>(p, st);
            case 128: return launch_mlp_bn<128, true>(p, st);
        }
        return RR_ERR_ARG;
    }
    switch (p.bn) {
        case 32: return launch_mlp_bn<32>(p, st);
        case 64: return launch_mlp_bn<64>(p, st);
        case 128: return launch_mlp_bn<128>(p, st);
    }
    return RR_ERR_ARG;
}

void rr_trace_set_gemm(unsigned long long* p) { rr_trace_set_local(p); }
void rr_trace_set_gemm_detail(int on) { rr_trace_set_detail_local(on); }

}  // namespace rr
