// rr_layer.cu — decode layer as ONE persistent dataflow launch between two attention kernels:
//
//   phase 0  O projection      attn_out[rows, nq]  x Wo[hidden, nq]      -> split-K planes -> x += ..., xhat, sum(x^2)
//   phase 1  gate/up + SiLU    xhat[rows, hidden]  x Wgu[2 inter, hidden] -> act = silu(g r) * (u r)
//   phase 2  down projection   act[rows, inter]    x Wd[hidden, inter]    -> x += ... (slice by slice), xhat, sum(x^2)
//   phase 3  next projection   xhat[rows, hidden]  x W3[rowsA3, hidden]   -> planes * r   (QKV of layer l + 1, or lm_head)
//
// Same warp roles and smem ring as gemm_bf16_wgmma / gemm_mlp_wgmma (rr_gemm.cu): one TMA producer warp, one consumer
// warpgroup (wgmma with the weights on the M side and the <= BN batch rows on the N side, then the epilogue).  The pipeline state carries from item to item and from phase to phase, so the weight stream never
// drains inside a layer: every CTA walks a host-built list (layer_schedule) and a phase boundary is a dependency
// counter, not a kernel boundary; the weight tiles of an item's first stages are always requested BEFORE its
// dependency is awaited.
//
// The two RMSNorms of a layer would be all-to-all barriers (a row's 1/rms needs every output feature of the
// producing GEMM).  They are DEFERRED instead: the producer of the residual emits the un-normalised operand
// xhat = bf16(x * gamma) and per-(row, 128-feature tile) partial sums of squares; the consuming GEMM is linear, so its
// epilogue multiplies the accumulators of batch row b by r_b = rsqrt(mean(x_b^2) + eps).  What is left of the norm is
// one counter per phase boundary.
//
//   * O -> residual: the s_o split-K CTAs of a 128-feature tile (each the FIRST item of its CTA, so all are running)
//     store their fp32 planes, meet on arr_o[tile], and each reduces rows/s_o of the batch rows: x += sum_z P_z in
//     fixed order, writes x, xhat, rowss_a[row][tile]; then cnt_o++.  Gate/up items wait for cnt_o == #O items.
//   * gate/up -> down: per K-slice counters exactly as in gemm_mlp_wgmma (ready_gu[slice] == tiles of the slice).
//   * down -> residual: every (tile, K-slice) item stores its plane and bumps arr_d[tile]; REDUCE items (consumer warps
//     only, no MMA; tile x row group, placed after the down items in the lists) wait for arr_d[tile] == #slices and do
//     the same fixed-order reduction into x, xhat, rowss_b; then cnt_d++.  (A first version added the slices into x in
//     turn, slice after slice: 8 dependent store->flag->load hops per tile, 63 us per layer instead of 20.)
//   * phase 3 waits for cnt_d == #reduce items, and scales by r from rowss_b.
//   Waiting only ever targets items of an earlier phase, and every list is ordered by phase: no cycles.
//
// Requires all CTAs co-resident (grid <= SM count, one CTA per SM by shared memory) and zeroed counters.
//
// Replaces (with rr_attn_decode.cu) the remote bedrock:InvokeModel call of the reference (iam/policy.json:8,
// src/demo_cris.py:233-238) — there is no reference kernel.
#include "rr_gemm_dev.cuh"

#include <string.h>
#include <algorithm>
#include <atomic>

namespace rr {

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_u32(unsigned* p, unsigned v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void spin_until(const unsigned* p, unsigned target) {
    while (ld_acquire_u32(p) < target) {
    }
}
__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 3, 128;" ::: "memory"); }

constexpr int PH_RED_D = 4;   // item phase ids: 0 O, 1 gate/up, 2 down, 3 next projection, 4 reduce (down planes -> residual)

constexpr int LAYER_EXTRA_SMEM = 1024;   // rinv[256]
template <int BN>
constexpr int layer_smem_bytes() { return gemm_smem_bytes<BN, OUT_TRANSPOSED_SILU>() + LAYER_EXTRA_SMEM; }

template <int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
decode_layer_wgmma(const __grid_constant__ LayerArgs a) {
    using Cfg = GemmCfg<BN>;
    constexpr int kStages = Cfg::kStages;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = align_smem_1024(smem_raw);
    uint8_t* smemA = smem;
    uint8_t* smemB = smem + kStages * Cfg::kStageBytesA;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * Cfg::kStageBytes);
    uint64_t* empty_bar = full_bar + kStages;
    float* acc_tile = reinterpret_cast<float*>(smem + Cfg::kAccOff);
    float* silu_stage = reinterpret_cast<float*>(smem + Cfg::kEpiOff);
    // Ring slots actually used (<= kStages).  Bytes in flight beyond bandwidth x latency only queue inside the memory system
    // and delay everything ELSE this SM asks for (dependency counters, reductions, epilogue stores): see DESIGN.md.
    const int depth = a.ring_depth;
    float* rinv_s = silu_stage + Cfg::kSiluStageBytes / 4;      // [256]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    griddep_launch();
    const int tr_slot = trace_begin(TR_GEMM_DEC);

    if (warp == PRODUCER_WARP && elect_one()) {
        for (int p = 0; p < 4; ++p) {
            tma_prefetch_desc(&a.tmA[p]);
            tma_prefetch_desc(&a.tmB[p]);
        }
        for (int s = 0; s < kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], GEMM_CONSUMERS / 32); }
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
    // counter block (zero at launch): [0] cnt_o, [1] cnt_d, then arr_o[tiles_h], arr_d[tiles_h], ready_gu[n_slices]
    unsigned* cnt_o = a.ctr;
    unsigned* cnt_d = a.ctr + 1;
    unsigned* arr_o = a.ctr + 2;
    unsigned* arr_d = arr_o + a.tiles_h;
    unsigned* ready_gu = arr_d + a.tiles_h;

    WorkItem t;
    int ph = 0;

    if (warp == PRODUCER_WARP) {
        // ===================== TMA producer =====================
        if (elect_one()) {
            const uint64_t polA = l2_policy_evict_first(), polB = l2_policy_evict_last();
            int stage = 0;
            uint32_t phase = 0;
            bool first = true, o_seen = false, d_seen = false;
            for (int i = 0; get(i, t, ph); ++i) {
                if (ph >= PH_RED_D) continue;                  // reduce items: consumer warps only
                const CUtensorMap* tA = &a.tmA[ph];
                const CUtensorMap* tB = &a.tmB[ph];
                const int nkb = t.kb1 - t.kb0;
                // is the activation operand of this item known to exist?
                const unsigned* dep = nullptr;
                unsigned need = 0;
                bool ok = !first;
                if (ph == 1) { dep = cnt_o; need = a.o_target; ok = ok && o_seen; }
                else if (ph == 2) { dep = ready_gu + t.z; need = (unsigned)nkb; ok = false; }
                else if (ph == 3) { dep = cnt_d; need = a.d_target; ok = ok && d_seen; }
                if (!ok && !first && dep != nullptr && ld_acquire_u32(dep) >= need) {
                    ok = true;
                    asm volatile("fence.proxy.async;" ::: "memory");
                }
                // Not yet: the WEIGHT tiles of the first stages go out before the wait (and, optionally, an L2 prefetch of
                // the k-blocks behind them), the activation tiles after it.  Known: plain interleaved A + B issue, so the
                // ring never drains at an item boundary.
                const int pre = ok ? 0 : min(depth, nkb);
                const int st0 = stage;
                for (int j = 0; j < pre; ++j) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
                    tma_load_2d_hint(smemA + stage * Cfg::kStageBytesA, tA, &full_bar[stage], (t.kb0 + j) * BLOCK_K,
                                     t.a_tile * BLOCK_A, polA);
                    if (++stage == depth) { stage = 0; phase ^= 1; }
                }
                if (!ok) {
                    const int ahead = min(t.kb1, t.kb0 + pre + a.l2_ahead);
                    for (int kb = t.kb0 + pre; kb < ahead; ++kb) tma_prefetch_l2_2d(tA, kb * BLOCK_K, t.a_tile * BLOCK_A);
                    if (first) { griddep_wait(); trace_dep(tr_slot); first = false; }
                    if (dep != nullptr) spin_until(dep, need);
                    asm volatile("fence.proxy.async;" ::: "memory");   // other SMs' generic stores -> our TMA reads
                    trace_mark_cta(40 + ph);                           // producer: dependency of an item of phase ph resolved
                }
                if (ph == 1) o_seen = true;
                if (ph == 3) d_seen = true;
                for (int j = 0, s2 = st0; j < pre; ++j) {
                    tma_load_2d_hint(smemB + s2 * Cfg::kStageBytesB, tB, &full_bar[s2], (t.kb0 + j) * BLOCK_K, 0, polB);
                    if (++s2 == depth) s2 = 0;
                }
                for (int kb = t.kb0 + pre; kb < t.kb1; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
                    tma_load_2d_hint(smemA + stage * Cfg::kStageBytesA, tA, &full_bar[stage], kb * BLOCK_K, t.a_tile * BLOCK_A, polA);
                    tma_load_2d_hint(smemB + stage * Cfg::kStageBytesB, tB, &full_bar[stage], kb * BLOCK_K, 0, polB);
                    if (++stage == depth) { stage = 0; phase ^= 1; }
                }
            }
            if (first) { griddep_wait(); trace_dep(tr_slot); }
        }
    } else {
        // ===================== consumer warpgroup: wgmma main loop + epilogue (warps 0..3) =====================
        const int quarter = warp;                     // rows [32 quarter, 32 quarter + 32) of the tile in the epilogue
        const int wq = warp;
        const int row_in_tile = quarter * 32 + lane;
        const int etid = threadIdx.x;
        const uint32_t smemA_u = smem_u32(smemA), smemB_u = smem_u32(smemB);
        int stage = 0;
        uint32_t phase = 0;
        const int rows = a.rows, hidden = a.hidden;
        int rinv_of = -1;                             // which r_b is staged in rinv_s: 1 = after O, 3 = after down
        griddep_wait();                               // outputs may still be read by the preceding kernel
        trace_dep(tr_slot);

        auto publish = [&](unsigned* ctr_add) {
            epi_bar();                                // every epilogue thread's stores
            if (etid == 0) {
                __threadfence();
                atomicAdd(ctr_add, 1u);
            }
        };
        // r_b = rsqrt(mean(x_b^2) + eps) of every batch row from the per-tile partial sums (all loads of a row independent)
        auto stage_rinv = [&](const float* rowss, const unsigned* ctr, unsigned target) {
            if (etid == 0) { spin_until(ctr, target); trace_mark_cta(37); }
            epi_bar();
            for (int b = etid; b < rows; b += 128) {
                const float* ps = rowss + (size_t)b * a.n_part;
                float ss = 0.f;
                for (int j0 = 0; j0 < a.n_part; j0 += 32) {
                    float v[32];
#pragma unroll
                    for (int j = 0; j < 32; ++j) v[j] = (j0 + j < a.n_part) ? __ldcg(ps + j0 + j) : 0.f;
#pragma unroll
                    for (int j = 0; j < 32; ++j) ss += v[j];
                }
                rinv_s[b] = rsqrtf(ss * a.inv_hidden + a.eps);
            }
            epi_bar();
            if (etid == 0) trace_mark_cta(38);
        };
        // planes of this item: P[z][b][f] = acc[f][b]
        auto store_plane = [&](float* planes, int z, const float* arow, int f) {
            float* pl = planes + (size_t)z * a.ld_rows * hidden;
#pragma unroll 1
            for (int c = 0; c < BN; c += 32) {
                uint32_t v[32];
                acc_ld32(arow + c, v);
                if (f < hidden) {
#pragma unroll
                    for (int j = 0; j < 32; ++j)
                        if (c + j < rows) pl[(size_t)(c + j) * hidden + f] = __uint_as_float(v[j]);
                }
            }
        };
        // x[b][tile] += sum_z planes[z][b][tile] (fixed order) for b in [b0, b1); xhat = bf16(x * gamma); rowss[b][tile] = sum x^2.
        // Warp = row (two rows in flight), lane = 4 consecutive features: every load is a 512-byte warp request from L2
        // and all loads of a pass are independent; sum(x^2) is a plain warp reduction.
        auto reduce_rows = [&](int tile, int b0, int b1, const float* planes, int n_planes, const __nv_bfloat16* gamma,
                               float* rowss_out) {
            const int f4 = tile * BLOCK_A + lane * 4;
            const bool fok = f4 < hidden;
            float g0 = 0.f, g1 = 0.f, g2 = 0.f, g3 = 0.f;
            if (fok) {
                const uint2 gw = *reinterpret_cast<const uint2*>(gamma + f4);
                g0 = bf16_lo(gw.x); g1 = bf16_hi(gw.x); g2 = bf16_lo(gw.y); g3 = bf16_hi(gw.y);
            }
            const size_t pstride = (size_t)a.ld_rows * hidden;
#pragma unroll 1
            for (int b = b0 + wq; b < b1; b += 8) {
                const int bb = b + 4;
                const bool two = bb < b1;
                float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
                float4 p0[8], p1[8];
                if (fok) {
                    v0 = __ldcg(reinterpret_cast<const float4*>(a.x + (size_t)b * hidden + f4));
                    if (two) v1 = __ldcg(reinterpret_cast<const float4*>(a.x + (size_t)bb * hidden + f4));
#pragma unroll
                    for (int z = 0; z < 8; ++z) {
                        if (z < n_planes) {
                            p0[z] = __ldcg(reinterpret_cast<const float4*>(planes + z * pstride + (size_t)b * hidden + f4));
                            if (two) p1[z] = __ldcg(reinterpret_cast<const float4*>(planes + z * pstride + (size_t)bb * hidden + f4));
                        }
                    }
#pragma unroll
                    for (int z = 0; z < 8; ++z) {
                        if (z < n_planes) {
                            v0.x += p0[z].x; v0.y += p0[z].y; v0.z += p0[z].z; v0.w += p0[z].w;
                            if (two) { v1.x += p1[z].x; v1.y += p1[z].y; v1.z += p1[z].z; v1.w += p1[z].w; }
                        }
                    }
                    *reinterpret_cast<float4*>(a.x + (size_t)b * hidden + f4) = v0;
                    uint2 h0;
                    h0.x = pack_bf16(v0.x * g0, v0.y * g1); h0.y = pack_bf16(v0.z * g2, v0.w * g3);
                    *reinterpret_cast<uint2*>(a.xhat + (size_t)b * hidden + f4) = h0;
                    if (two) {
                        *reinterpret_cast<float4*>(a.x + (size_t)bb * hidden + f4) = v1;
                        uint2 h1;
                        h1.x = pack_bf16(v1.x * g0, v1.y * g1); h1.y = pack_bf16(v1.z * g2, v1.w * g3);
                        *reinterpret_cast<uint2*>(a.xhat + (size_t)bb * hidden + f4) = h1;
                    }
                }
                float s0 = v0.x * v0.x + v0.y * v0.y + v0.z * v0.z + v0.w * v0.w;
                float s1 = v1.x * v1.x + v1.y * v1.y + v1.z * v1.z + v1.w * v1.w;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    s0 += __shfl_xor_sync(0xffffffffu, s0, o);
                    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
                }
                if (lane == 0) {
                    rowss_out[(size_t)b * a.n_part + tile] = s0;
                    if (two) rowss_out[(size_t)bb * a.n_part + tile] = s1;
                }
            }
        };

        for (int i = 0; get(i, t, ph); ++i) {
            if (ph == PH_RED_D) {
                // ---------------- reduce item: down planes of a tile complete -> residual rows [q R, (q + 1) R)
                if (etid == 0) { trace_mark_cta(34); spin_until(arr_d + t.a_tile, (unsigned)a.n_slices); trace_mark_cta(35); }
                epi_bar();
                reduce_rows(t.a_tile, t.z * a.rows_red_d, min(rows, (t.z + 1) * a.rows_red_d), a.part_d, a.n_slices, a.gamma_b,
                            a.rowss_b);
                if (etid == 0) trace_mark_cta(36);
                publish(cnt_d);
                if (etid == 0) trace_mark_cta(TR_LAYER_PH0 + 3);
                continue;
            }
            float acc[2][BN / 2];
            gmma_mainloop<BN>(acc, smemA_u, smemB_u, full_bar, empty_bar, stage, phase, t.kb1 - t.kb0, depth);
            acc_bar();                                          // the previous item's epilogue is done with the staged tile
            stage_acc<BN>(acc, acc_tile);
            acc_bar();
            if (etid == 0) trace_mark_cta(20 + ph);            // accumulator of an item of phase ph complete
            const int f = t.a_tile * BLOCK_A + row_in_tile;     // output feature of this thread (accumulator row)
            const float* arow = acc_tile + row_in_tile * Cfg::kAccPitch;

            if (ph == 0) {
                // ---------------- O projection: planes, then the tile's split CTAs reduce the batch rows together
                store_plane(a.part_o, t.z, arow, f);
                epi_bar();
                if (etid == 0) {
                    trace_mark_cta(30);
                    __threadfence();
                    atomicAdd(arr_o + t.a_tile, 1u);
                    trace_mark_cta(31);
                    spin_until(arr_o + t.a_tile, (unsigned)a.s_o);
                    trace_mark_cta(32);
                }
                epi_bar();
                const int R = (rows + a.s_o - 1) / a.s_o;
                reduce_rows(t.a_tile, t.z * R, min(rows, (t.z + 1) * R), a.part_o, a.s_o, a.gamma_a, a.rowss_a);
                if (etid == 0) trace_mark_cta(33);
                publish(cnt_o);
            } else if (ph == 1) {
                // ---------------- gate/up: act[b][n] = silu(g r_b) * (u r_b); weights interleaved in 64-row gate/up blocks
                if (rinv_of != 1) { stage_rinv(a.rowss_a, cnt_o, a.o_target); rinv_of = 1; }
                const bool is_up = quarter >= 2;            // accumulator rows 64..127 of the tile hold the up rows
                const int r64 = (quarter & 1) * 32 + lane;
                const int n = t.a_tile * 64 + r64;
#pragma unroll 1
                for (int c = 0; c < BN; c += 32) {
                    float* buf = silu_stage + ((c >> 5) & 1) * (32 * 64);
                    uint32_t v[32];
                    acc_ld32(arow + c, v);
                    if (is_up) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) buf[j * 64 + r64] = __uint_as_float(v[j]);
                    }
                    asm volatile("bar.sync 2, 128;" ::: "memory");
                    if (!is_up && n < a.inter) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            const int b = c + j;
                            if (b < rows) {
                                const float r = rinv_s[b];
                                a.act[(size_t)b * a.inter + n] =
                                    __float2bfloat16(silu_mul(__uint_as_float(v[j]) * r, buf[j * 64 + r64] * r));
                            }
                        }
                    }
                }
                publish(ready_gu + t.a_tile / a.slice_kb);
            } else if (ph == 2) {
                // ---------------- down: plane of this K-slice; the tile's reduce items wait for all of them
                store_plane(a.part_d, t.z, arow, f);
                publish(arr_d + t.a_tile);
            } else {
                // ---------------- next projection (QKV of the next layer / lm_head): planes scaled by r_b
                if (rinv_of != 3) { stage_rinv(a.rowss_b, cnt_d, a.d_target); rinv_of = 3; }
                float* pl = a.out3 + (size_t)t.z * a.ld_rows * a.ldo3;
#pragma unroll 1
                for (int c = 0; c < BN; c += 32) {
                    uint32_t v[32];
                    acc_ld32(arow + c, v);
                    if (f < a.rowsA3) {
#pragma unroll
                        for (int j = 0; j < 32; ++j)
                            if (c + j < rows) pl[(size_t)(c + j) * a.ldo3 + f] = __uint_as_float(v[j]) * rinv_s[c + j];
                    }
                }
            }
            if (etid == 0) trace_mark_cta(TR_LAYER_PH0 + (ph == 3 ? 4 : ph));      // debug timeline: item finished on this CTA
        }
    }

    __syncthreads();
    trace_end(tr_slot);
}

// ---------------------------------------------------------------------------------------------------- host side
// Greedy list schedule in units of k-blocks (+ a fixed per-item cost for pipeline refill / epilogue).  Phases are placed
// in order; inside a phase the items go, in dependency order, to the least-loaded CTA.  O items are pinned one per CTA
// (CTA i gets item i): their epilogues wait for each other, which is only safe when each is its CTA's first item.
int layer_schedule(int grid, const LayerShape& s, std::vector<MlpItem>* items) {
    constexpr int kItemCost = 6, kRedCost = 3;
    std::vector<std::vector<MlpItem>> per(grid);
    std::vector<long long> load(grid, 0);
    auto least = [&]() {
        int best = 0;
        for (int c = 1; c < grid; ++c) if (load[c] < load[best]) best = c;
        return best;
    };
    auto put = [&](int c, int phase, int tile, int k0, int k1, int z) {
        MlpItem it; it.tile_phase = tile | (phase << 16); it.kb0 = k0; it.kb1 = k1; it.z = z;
        per[c].push_back(it);
        load[c] += (k1 - k0) + kItemCost;
    };
    const int tiles_h = (s.hidden + BLOCK_A - 1) / BLOCK_A;
    if (s.has_main) {
        const int kb_o = (s.nq + BLOCK_K - 1) / BLOCK_K;
        if (tiles_h * s.s_o > grid || s.s_o < 1 || s.s_o > kb_o) return -1;
        int c = 0;
        for (int tl = 0; tl < tiles_h; ++tl)
            for (int z = 0; z < s.s_o; ++z, ++c)
                put(c, 0, tl, (int)((long long)kb_o * z / s.s_o), (int)((long long)kb_o * (z + 1) / s.s_o), z);
        const int tiles_gu = (2 * s.inter) / BLOCK_A, kb_h = (s.hidden + BLOCK_K - 1) / BLOCK_K;
        for (int tl = 0; tl < tiles_gu; ++tl) put(least(), 1, tl, 0, kb_h, 0);
        const int kb_d = s.inter / BLOCK_K;
        const int n_slices = (kb_d + s.slice_kb - 1) / s.slice_kb;
        for (int z = 0; z < n_slices; ++z) {
            const int k0 = z * s.slice_kb, k1 = std::min(k0 + s.slice_kb, kb_d);
            for (int tl = 0; tl < tiles_h; ++tl) put(least(), 2, tl, k0, k1, z);
        }
        // reduce items (epilogue only): tile x row group, after every down item of every list
        // (latency-bound work: spread over distinct CTAs, least loaded first, before any CTA gets a second one)
        const int n_rq = layer_red_groups(grid, tiles_h);
        std::vector<int> order(grid);
        for (int c = 0; c < grid; ++c) order[c] = c;
        std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return load[x] < load[y]; });
        int k = 0;
        for (int q = 0; q < n_rq; ++q)
            for (int tl = 0; tl < tiles_h; ++tl, ++k) {
                const int c = order[k % grid];
                put(c, PH_RED_D, tl, 0, 0, q);
                load[c] += kRedCost - kItemCost;
            }
    }
    if (s.rowsA3 > 0) {
        const int tiles3 = (s.rowsA3 + BLOCK_A - 1) / BLOCK_A, kb_h = (s.hidden + BLOCK_K - 1) / BLOCK_K;
        if (s.s3 < 1 || s.s3 > kb_h) return -1;
        for (int tl = 0; tl < tiles3; ++tl)
            for (int z = 0; z < s.s3; ++z)
                put(least(), 3, tl, (int)((long long)kb_h * z / s.s3), (int)((long long)kb_h * (z + 1) / s.s3), z);
    }
    size_t mx = 1;
    for (auto& v : per) mx = std::max(mx, v.size());
    items->assign((size_t)grid * mx, MlpItem{-1, 0, 0, 0});
    for (int c = 0; c < grid; ++c)
        for (size_t i = 0; i < per[c].size(); ++i) (*items)[(size_t)c * mx + i] = per[c][i];
    return (int)mx;
}

// row groups per tile for the reduction of the down planes: as many as there are CTAs to take them, at most 8
int layer_red_groups(int grid, int tiles_h) {
    int n = grid / tiles_h;
    return n < 1 ? 1 : (n > 8 ? 8 : (n >= 4 ? 4 : n));
}

int layer_counter_words(const LayerShape& s) {
    const int tiles_h = (s.hidden + BLOCK_A - 1) / BLOCK_A;
    const int n_slices = s.has_main ? (s.inter / BLOCK_K + s.slice_kb - 1) / s.slice_kb : 0;
    return 2 + 2 * tiles_h + n_slices;
}

int layer_plan_init(LayerPlan* p, const LayerShape& s, const LayerBuffers& b, int bn, const MlpItem* items_dev,
                    int max_items, int grid, unsigned* ctr) {
    if (!p || !items_dev || !ctr || !b.x || !b.xhat || !b.rowss_b) return RR_ERR_ARG;
    if (s.hidden % 64 || b.rows > bn || bn < 32 || bn > MAX_BN || grid < 1 || grid > num_sms()) return RR_ERR_ARG;
    LayerArgs& a = p->args;
    memset(&a, 0, sizeof(a));
    const int tiles_h = (s.hidden + BLOCK_A - 1) / BLOCK_A;
    int rc = RR_OK;
    if (s.has_main) {
        if (!b.wo || !b.wgu || !b.wdown || !b.attn_out || !b.act || !b.part_o || !b.part_d || !b.rowss_a || !b.gamma_a || !b.gamma_b)
            return RR_ERR_ARG;
        if (s.inter % 64 || (2 * s.inter) % BLOCK_A || s.nq % 8 || s.slice_kb < 1 || (2 * s.inter) / BLOCK_A > 0xffff)
            return RR_ERR_ARG;
        rc = make_tmap_bf16_2d(&a.tmA[0], b.wo, s.hidden, s.nq, s.nq, BLOCK_A);
        if (rc == RR_OK) rc = make_tmap_bf16_2d(&a.tmB[0], b.attn_out, b.rows, s.nq, s.nq, bn);
        if (rc == RR_OK) rc = make_tmap_bf16_2d(&a.tmA[1], b.wgu, 2 * s.inter, s.hidden, s.hidden, BLOCK_A);
        if (rc == RR_OK) rc = make_tmap_bf16_2d(&a.tmB[1], b.xhat, b.rows, s.hidden, s.hidden, bn);
        if (rc == RR_OK) rc = make_tmap_bf16_2d(&a.tmA[2], b.wdown, s.hidden, s.inter, s.inter, BLOCK_A);
        if (rc == RR_OK) rc = make_tmap_bf16_2d(&a.tmB[2], b.act, b.rows, s.inter, s.inter, bn);
        if (rc != RR_OK) return rc;
    }
    if (s.rowsA3 > 0) {
        if (!b.w3 || !b.out3) return RR_ERR_ARG;
        rc = make_tmap_bf16_2d(&a.tmA[3], b.w3, s.rowsA3, s.hidden, s.hidden, BLOCK_A);
        if (rc == RR_OK) rc = make_tmap_bf16_2d(&a.tmB[3], b.xhat, b.rows, s.hidden, s.hidden, bn);
        if (rc != RR_OK) return rc;
    }
    // unused phases still get valid descriptors (they are prefetched): alias a live one
    for (int ph = 0; ph < 4; ++ph) {
        const bool live = ph == 3 ? s.rowsA3 > 0 : s.has_main != 0;
        if (!live) { const int src = s.has_main ? 0 : 3; a.tmA[ph] = a.tmA[src]; a.tmB[ph] = a.tmB[src]; }
    }
    a.part_o = b.part_o; a.part_d = b.part_d; a.x = b.x; a.xhat = b.xhat; a.act = b.act; a.out3 = b.out3;
    a.gamma_a = b.gamma_a; a.gamma_b = b.gamma_b; a.rowss_a = b.rowss_a; a.rowss_b = b.rowss_b;
    a.hidden = s.hidden; a.inter = s.inter; a.rows = b.rows; a.ld_rows = b.ld_rows; a.rowsA3 = s.rowsA3; a.ldo3 = b.ldo3;
    a.n_part = tiles_h; a.tiles_h = tiles_h; a.s_o = s.s_o;
    a.slice_kb = s.slice_kb > 0 ? s.slice_kb : 1;
    a.n_slices = s.has_main ? (s.inter / BLOCK_K + s.slice_kb - 1) / s.slice_kb : 0;
    a.inv_hidden = 1.0f / (float)s.hidden; a.eps = b.eps;
    a.items = items_dev; a.max_items = max_items; a.ctr = ctr;
    const int n_rq = layer_red_groups(grid, tiles_h);
    a.rows_red_d = (b.rows + n_rq - 1) / n_rq;
    a.o_target = s.has_main ? (unsigned)(tiles_h * s.s_o) : 0u;
    a.d_target = s.has_main ? (unsigned)(tiles_h * n_rq) : 0u;
    a.l2_ahead = b.l2_ahead;
    a.ring_depth = b.ring_depth;       // clamped to the kernel's stage count at launch
    if (s.has_main && (a.n_slices > 8 || s.s_o > 8 || s.hidden % 4)) return RR_ERR_ARG;
    p->grid = grid; p->bn = bn;
    return RR_OK;
}

template <int BN>
static int launch_layer_bn(const LayerPlan& p, cudaStream_t st) {
    auto kern = decode_layer_wgmma<BN>;
    static std::atomic<uint64_t> attr_set{0};
    if (ensure_dyn_smem(kern, layer_smem_bytes<BN>(), attr_set) != cudaSuccess) return RR_ERR_CUDA;
    LayerArgs args = p.args;
    constexpr int kStages = GemmCfg<BN>::kStages;
    if (args.ring_depth < 2 || args.ring_depth > kStages) args.ring_depth = kStages;
    cudaError_t e = launch_pdl(kern, dim3(p.grid), dim3(GEMM_THREADS), (size_t)layer_smem_bytes<BN>(), st, args);
    return e == cudaSuccess ? RR_OK : RR_ERR_CUDA;
}
int layer_launch(const LayerPlan& p, cudaStream_t st) {
    switch (p.bn) {
        case 32: return launch_layer_bn<32>(p, st);
        case 64: return launch_layer_bn<64>(p, st);
        case 128: return launch_layer_bn<128>(p, st);
    }
    return RR_ERR_ARG;
}

void rr_trace_set_layer(unsigned long long* p) { rr_trace_set_local(p); }
void rr_trace_set_layer_detail(int on) { rr_trace_set_detail_local(on); }

}  // namespace rr
