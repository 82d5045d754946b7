// rr_attn_decode.cu — K8: decode attention over the KV cache, [page][kv_head][P][128] bf16 addressed by kv_row
// (rr_kernels.h): 64-token pages through a page table, or one ctx_max-token page per slot.  One query token per row; the G query heads of a GQA group
// share each KV head, so one CTA = (row, kv_head[, kv split]) streams ctx * 512 B exactly once.
//
// HBM-bound by design (SURVEY.md §8d: 128 KiB/token/step for Llama-3-8B):
//  * K and V tiles (64 tokens x 256 B = 16 KB "units") are staged by TMA (UTMALDG, 128B swizzle,
//    two 64-column boxes per unit) into a 3-slot shared-memory ring fed by a dedicated producer warp
//    through full/empty mbarriers; 4 CTAs/SM are resident, so all 512 CTAs of a 64-row step run in
//    one wave with up to 192 KB of loads in flight per SM.
//  * The math is on mma.sync.m16n8k16 (bf16, fp32 accumulate) in the transposed formulation
//    S^T[tokens x heads] = K Q^T and O^T[d x heads] = V^T P^T (heads padded to n = 8), so K and V
//    feed the A operand straight from ldmatrix / ldmatrix.trans and the accumulators are 32 registers;
//    P^T is re-laid out with movmatrix.  ~70 warp instructions per 16 tokens instead of ~850 for a
//    CUDA-core dot-product loop (profiles/r01_*): the kernel is issue-light and stays HBM-bound.
//  * Each of the 4 consumer warps owns 16 tokens of every tile with a private online-softmax state;
//    states are merged once at the end (and across kv splits by a small combine kernel).
//  * Sliding window (DecodeAttnArgs::window): the tiles start at that of the row's first visible key; keys below it are
//    masked in that tile.
//
// Replaces the remote bedrock:InvokeModel call (reference iam/policy.json:8).
#include <stdlib.h>
#include "rr_ptx.cuh"
#include "rr_launch.cuh"
#include "rr_kernels.h"

namespace rr {

constexpr int HD = 128;
constexpr int DT = 64;                  // tokens per unit
constexpr int UNIT_BYTES = DT * HD * 2; // 16 KB
constexpr int RING = 3;
constexpr int DEC_THREADS = 160;        // 4 consumer warps + 1 producer warp
constexpr int DEC_SMEM = RING * UNIT_BYTES + 1024 /*align*/ + 128 /*barriers*/ + 512 /*new k, v row*/ + 2048 /*q*/;
// + the cache row of each of the CTA's tiles, int32: room for at least DEC_TBL tiles (8192 tokens), so contexts up to that
// run every kv-split count with one shared-memory size and 4 CTAs/SM
constexpr int DEC_TBL = 128;
static_assert(DT == KV_PAGE, "a decode tile never crosses a page");
static int dec_smem(const DecodeAttnArgs& a) {
    const int tiles = (a.ctx_max / DT + a.kv_splits - 1) / a.kv_splits;
    return DEC_SMEM + 4 * (tiles > DEC_TBL ? tiles : DEC_TBL);
}

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ uint32_t movmatrix_t(uint32_t v) {
    uint32_t r;
    asm volatile("movmatrix.sync.aligned.m8n8.trans.b16 %0, %1;" : "=r"(r) : "r"(v));
    return r;
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// byte offset of 16-byte chunk `c` (0..15 across the 256 B row) of row `r` inside a TMA-written unit:
// two [64 rows x 128 B] halves, each with the 128B swizzle (chunk ^ (row & 7)).
__device__ __forceinline__ uint32_t unit_off(int r, int c) {
    return (uint32_t)(((c >> 3) << 13) + (r << 7) + ((((c & 7) ^ (r & 7))) << 4));
}

template <int G>
__global__ void __launch_bounds__(DEC_THREADS, 4)
decode_attn_mma_kernel(const __grid_constant__ DecodeAttnArgs a) {
    extern __shared__ uint8_t dsm_raw[];
    uint8_t* ring = align_smem_1024(dsm_raw);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(ring + RING * UNIT_BYTES);
    uint64_t* empty_bar = full_bar + RING;
    uint64_t* newkv_bar = empty_bar + RING;
    __nv_bfloat16* newkv = reinterpret_cast<__nv_bfloat16*>(ring + RING * UNIT_BYTES + 128);   // [k 128 | v 128]
    __nv_bfloat16* q_s = newkv + 2 * HD;                                                          // [8 heads][128]
    int* tile_row_s = reinterpret_cast<int*>(q_s + 8 * HD);      // [tiles] cache row of tile tile0 + j (dec_smem)

    griddep_launch();
    const int tr_slot = trace_begin(TR_ATTN_DEC);
    const int kvh = blockIdx.x, row = blockIdx.y, split = blockIdx.z;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // detail trace: (row 0 | 21 | 42 | 63, kv head 0); the fixed slots keep the last launch (tools/trace_attn.py)
    const int tsm = (kvh == 0 && split == 0 && row % 21 == 0) ? row / 21 : -1;
    if (tsm >= 0 && tid == 0) trace_mark_at(TR_ATTN_MARK + 0, 4 + tsm, 0);
    if (tid == 0) {
        for (int i = 0; i < RING; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 4); }
        mbar_init(newkv_bar, 1);
        fence_barrier_init();
        tma_prefetch_desc(&a.tmK);
        tma_prefetch_desc(&a.tmV);
        if (a.trim_tail) { tma_prefetch_desc(&a.tmK16); tma_prefetch_desc(&a.tmV16); }
    }
    __syncthreads();
    // Row metadata and the K/V rows of EARLIER tokens are constant for the whole step (written by previous graph
    // launches; argmax bumps pos only at the very end of a step), so they may be read before the PDL wait: the producer
    // gets the first ring of K/V tiles in flight while the QKV GEMM in front of this kernel is still draining.  Only q and
    // the new token's k / v depend on that GEMM.
    const int slot = a.slot[row];
    if (slot < 0) {
        // inactive row.  Still wait: a grid none of whose CTAs executes griddepcontrol.wait would "complete" while its
        // predecessor is running and break the completion chain the later kernels rely on (PDL ordering is transitive
        // only through the waits).
        griddep_wait();
        return;
    }
    const int ctx = a.pos[row] + 1;
    const int pos = ctx - 1;
    // sliding window: keys lo .. pos.  The splits divide tiles lo / DT .. (ctx - 1) / DT; the first of them holds key lo, so
    // every split with a tile has a visible key.  Without a window (or pos < W) lo = 0 and the tiles are today's.
    const int lo = a.window > 0 ? max(0, pos - a.window + 1) : 0;
    const int tile_lo = lo / DT;
    const int n_tiles_all = (ctx + DT - 1) / DT;
    const int tiles_per = (n_tiles_all - tile_lo + a.kv_splits - 1) / a.kv_splits;
    const int tile0 = tile_lo + split * tiles_per;
    const int tile1 = min(n_tiles_all, tile0 + tiles_per);
    const int n_units = 2 * max(0, tile1 - tile0);

    const bool owns_new = a.fuse_rope && tile1 == n_tiles_all && tile1 > tile0;   // this split holds token `pos`

    if (warp == 4) {
        // ===================== producer: TMA units K0 V0 K1 V1 ... =====================
        // The page table, like slot and pos, only changes between steps: the rows of this CTA's tiles are read before the PDL
        // wait, once, so the steady state issues no dependent global load per tile.
        // Row of the first token of tile tile0 + j in the [n_pages*kvh*P, 128] view; a 64-token tile never crosses a page.
        for (int j = lane; j < tile1 - tile0; j += 32)
            tile_row_s[j] = (int)kv_row(a.page_table, a.pages_per_slot, a.n_kv_heads, a.ctx_max, slot, kvh, (tile0 + j) * DT);
        __syncwarp();
        const bool leader = elect_one();
        // The last tile of a row usually holds fewer than 64 tokens: it is requested as 16-row boxes covering only the rows in use
        // (ncu: the kernel read 1.14 x its algorithmic bytes with whole tiles).  The rows of the slot that are not rewritten keep
        // the finite K / V data of the unit staged there before (hence u >= RING); their scores are masked, p = 0.
        auto issue = [&](int u) {
            const int s = u % RING;
            const bool is_v = (u & 1) != 0;
            const int tile = tile0 + (u >> 1);
            const int r0 = tile_row_s[u >> 1];
            const int valid = ctx - tile * DT;                        // > 0; >= DT for all but the last tile
            if (a.trim_tail && valid <= DT - 16 && u >= RING) {
                const int nb = (valid + 15) >> 4;
                const CUtensorMap* tm = is_v ? &a.tmV16 : &a.tmK16;
                mbar_arrive_expect_tx(&full_bar[s], nb * 4096);
                for (int b = 0; b < nb; ++b) {
                    tma_load_2d(ring + s * UNIT_BYTES + b * 2048, tm, &full_bar[s], 0, r0 + 16 * b);
                    tma_load_2d(ring + s * UNIT_BYTES + 8192 + b * 2048, tm, &full_bar[s], 64, r0 + 16 * b);
                }
                return;
            }
            const CUtensorMap* tm = is_v ? &a.tmV : &a.tmK;
            mbar_arrive_expect_tx(&full_bar[s], UNIT_BYTES);
            tma_load_2d(ring + s * UNIT_BYTES, tm, &full_bar[s], 0, r0);
            tma_load_2d(ring + s * UNIT_BYTES + 8192, tm, &full_bar[s], 64, r0);
        };
        const int first = min(RING, n_units);
        if (leader)
            for (int u = 0; u < first; ++u) issue(u);
        griddep_wait();                         // q / new k / new v come from the QKV GEMM
        if (tsm >= 0 && lane == 0) trace_mark_at(TR_ATTN_MARK + 1, 4 + tsm, 1);
        if (a.fuse_rope) {
            // K6 fused.  Rotated queries of the G heads -> smem (lane owns rotation pairs i = 2*lane, 2*lane+1 of
            // every head); if this CTA holds token `pos`: rotate the new key, append k / v (bf16) to the cache and
            // publish the row in smem.  All loads of one split plane are issued together (one latency per plane);
            // the whole block overlaps the flight of the first K/V tiles.
            const int hd = a.head_dim, half = hd >> 1;
            const int i = 2 * lane;
            const bool lane_on = i < half;                            // rotation pairs (i, i + hd/2)
            const bool v_on = 4 * lane < hd;
            const int kcol = a.n_heads * hd + kvh * hd, vcol = (a.n_heads + a.n_kv_heads) * hd + kvh * hd;
            const float4 cs = *reinterpret_cast<const float4*>(a.rope_table + (size_t)pos * 64 + (lane_on ? i : 0));
            float2 lo[G], hi[G];
            float2 klo = make_float2(0.f, 0.f), khi = klo, v0 = klo, v1 = klo;
#pragma unroll
            for (int h = 0; h < G; ++h) lo[h] = hi[h] = make_float2(0.f, 0.f);
            // The split-K planes are summed here.  All loads of up to kPlaneBatch planes are issued before the first add: with
            // one plane per loop iteration the prologue was n_splits dependent L2 round trips (~1.3 us each under load): a
            // no-split QKV experiment (one plane) showed 4 us of the kernel's 34 were exactly that.  In-process A/B on the
            // split-K path: 4.376 vs 4.493 ms per decode step (profiles/r02_layer_kernel_experiment.md).
            constexpr int kPlaneBatch = G <= 2 ? 4 : (G <= 4 ? 3 : 2);
            const float2 z2 = make_float2(0.f, 0.f);
            const int pstep = kPlaneBatch;
            for (int zb = 0; zb < a.qkv.n_splits; zb += pstep) {
                float2 tl[kPlaneBatch][G], th[kPlaneBatch][G], tk[kPlaneBatch][4];
#pragma unroll
                for (int zz = 0; zz < kPlaneBatch; ++zz) {
                    const bool on = zb + zz < a.qkv.n_splits;
                    const float* pl = reinterpret_cast<const float*>(a.qkv.ptr) + (size_t)(on ? zb + zz : 0) * a.qkv.split_stride +
                                      (size_t)row * a.qkv.ld;
#pragma unroll
                    for (int h = 0; h < G; ++h) {
                        tl[zz][h] = (on && lane_on) ? *reinterpret_cast<const float2*>(pl + (kvh * G + h) * hd + i) : z2;
                        th[zz][h] = (on && lane_on) ? *reinterpret_cast<const float2*>(pl + (kvh * G + h) * hd + half + i) : z2;
                    }
                    tk[zz][0] = (on && owns_new && lane_on) ? *reinterpret_cast<const float2*>(pl + kcol + i) : z2;
                    tk[zz][1] = (on && owns_new && lane_on) ? *reinterpret_cast<const float2*>(pl + kcol + half + i) : z2;
                    tk[zz][2] = (on && owns_new && v_on) ? *reinterpret_cast<const float2*>(pl + vcol + 4 * lane) : z2;
                    tk[zz][3] = (on && owns_new && v_on) ? *reinterpret_cast<const float2*>(pl + vcol + 4 * lane + 2) : z2;
                }
#pragma unroll
                for (int zz = 0; zz < kPlaneBatch; ++zz) {            // plane order = the summation order of the unbatched loop
#pragma unroll
                    for (int h = 0; h < G; ++h) {
                        lo[h].x += tl[zz][h].x; lo[h].y += tl[zz][h].y; hi[h].x += th[zz][h].x; hi[h].y += th[zz][h].y;
                    }
                    klo.x += tk[zz][0].x; klo.y += tk[zz][0].y; khi.x += tk[zz][1].x; khi.y += tk[zz][1].y;
                    v0.x += tk[zz][2].x; v0.y += tk[zz][2].y; v1.x += tk[zz][3].x; v1.y += tk[zz][3].y;
                }
            }
            if (tsm >= 0 && lane == 0) trace_mark_at(TR_ATTN_MARK + 2, 4 + tsm, 2);
            // smem rows are 128 wide: zero the padding beyond the true head dim first
            if (hd < HD) {
#pragma unroll
                for (int h = 0; h < G; ++h) *reinterpret_cast<uint2*>(q_s + h * HD + 4 * lane) = make_uint2(0u, 0u);
                *reinterpret_cast<uint2*>(newkv + 4 * lane) = make_uint2(0u, 0u);
                *reinterpret_cast<uint2*>(newkv + HD + 4 * lane) = make_uint2(0u, 0u);
                __syncwarp();
            }
            if (lane_on) {
#pragma unroll
                for (int h = 0; h < G; ++h) {
                    *reinterpret_cast<uint32_t*>(q_s + h * HD + i) =
                        pack_bf16(lo[h].x * cs.x - hi[h].x * cs.y, lo[h].y * cs.z - hi[h].y * cs.w);
                    *reinterpret_cast<uint32_t*>(q_s + h * HD + half + i) =
                        pack_bf16(hi[h].x * cs.x + lo[h].x * cs.y, hi[h].y * cs.z + lo[h].y * cs.w);
                }
            }
            if (owns_new) {
                const uint32_t k_lo = pack_bf16(klo.x * cs.x - khi.x * cs.y, klo.y * cs.z - khi.y * cs.w);
                const uint32_t k_hi = pack_bf16(khi.x * cs.x + klo.x * cs.y, khi.y * cs.z + klo.y * cs.w);
                uint2 vv;
                vv.x = pack_bf16(v0.x, v0.y);
                vv.y = pack_bf16(v1.x, v1.y);
                const size_t prow = (size_t)tile_row_s[pos / DT - tile0] + pos % DT;   // the append goes through the same rule
                __nv_bfloat16* kdst = const_cast<__nv_bfloat16*>(a.k_cache) + prow * HD;
                __nv_bfloat16* vdst = const_cast<__nv_bfloat16*>(a.v_cache) + prow * HD;
                if (lane_on) {
                    *reinterpret_cast<uint32_t*>(kdst + i) = k_lo;
                    *reinterpret_cast<uint32_t*>(kdst + half + i) = k_hi;
                    *reinterpret_cast<uint32_t*>(newkv + i) = k_lo;
                    *reinterpret_cast<uint32_t*>(newkv + half + i) = k_hi;
                }
                if (v_on) {
                    *reinterpret_cast<uint2*>(vdst + 4 * lane) = vv;
                    *reinterpret_cast<uint2*>(newkv + HD + 4 * lane) = vv;
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(newkv_bar);      // q (and the new k / v row) are in smem
            if (tsm >= 0 && lane == 0) trace_mark_at(TR_ATTN_MARK + 3, 4 + tsm, 3);
        }
        if (leader)
            for (int u = first; u < n_units; ++u) {
                mbar_wait(&empty_bar[u % RING], ((u / RING) - 1) & 1);
                issue(u);
                if (tsm >= 0) trace_mark_at(TR_ATTN_MARK + 4, 4 + tsm, 8 + u);
            }
        return;
    }

    // ===================== consumers: warp w owns tokens [16w, 16w+16) of every tile =====================
    griddep_wait();                             // a.q (unfused path) and `out` / `ws` ordering against the previous kernels
    trace_dep(tr_slot);
    const int g = lane >> 2, t = lane & 3;
    // Q^T B-fragments: b0 = Q[head g][16ks + 2t, +1], b1 = Q[head g][16ks + 8 + 2t, +1]; heads >= G are zero
    uint32_t qb[8][2];
    if (a.fuse_rope) {
        mbar_wait(newkv_bar, 0);
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
            qb[ks][0] = g < G ? *reinterpret_cast<const uint32_t*>(q_s + g * HD + ks * 16 + 2 * t) : 0u;
            qb[ks][1] = g < G ? *reinterpret_cast<const uint32_t*>(q_s + g * HD + ks * 16 + 8 + 2 * t) : 0u;
        }
    } else {
        const __nv_bfloat16* qrow = a.q + (size_t)row * a.n_heads * HD + (size_t)(kvh * G + g) * HD;
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
            qb[ks][0] = g < G ? *reinterpret_cast<const uint32_t*>(qrow + ks * 16 + 2 * t) : 0u;
            qb[ks][1] = g < G ? *reinterpret_cast<const uint32_t*>(qrow + ks * 16 + 8 + 2 * t) : 0u;
        }
    }
    const int patch_tile = owns_new ? pos / DT : -1;                  // tile whose staged copy lacks token `pos`
    const bool patch_warp = ((pos % DT) >> 4) == warp;
    const float sc = a.scale * 1.4426950408889634f;
    float o[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;      // heads 2t and 2t+1
    const uint32_t ring_u = smem_u32(ring);

    if (tsm >= 0 && tid == 0) trace_mark_at(TR_ATTN_MARK + 5, 4 + tsm, 4);
    for (int tile = tile0; tile < tile1; ++tile) {
        const int u = 2 * (tile - tile0);
        // ---- S^T = K Q^T for this warp's 16 tokens
        {
            const int s = u % RING;
            mbar_wait(&full_bar[s], (u / RING) & 1);
            if (tsm >= 0 && tid == 0) trace_mark_at(TR_ATTN_MARK + 6, 4 + tsm, 64 + u);
            const uint32_t base = ring_u + s * UNIT_BYTES;
            if (tile == patch_tile && patch_warp) {          // the cache row of `pos` was written after/while TMA read it
                if (lane < 16)
                    *reinterpret_cast<uint4*>(ring + s * UNIT_BYTES + unit_off(pos % DT, lane)) =
                        *reinterpret_cast<const uint4*>(newkv + lane * 8);
                __syncwarp();
            }
            float c[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
                uint32_t ka[4];
                ldsm_x4(ka, base + unit_off(warp * 16 + (lane & 15), ks * 2 + (lane >> 4)));
                mma16816(c, ka, qb[ks][0], qb[ks][1]);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[s]);
            // ---- online softmax over tokens (rows g and g+8 of the fragment), per head column
            const int tok = tile * DT + warp * 16 + g;
            float s00 = c[0] * sc, s01 = c[1] * sc, s10 = c[2] * sc, s11 = c[3] * sc;
            if (tok >= ctx || tok < lo) { s00 = -INFINITY; s01 = -INFINITY; }
            if (tok + 8 >= ctx || tok + 8 < lo) { s10 = -INFINITY; s11 = -INFINITY; }
            float mx0 = fmaxf(s00, s10), mx1 = fmaxf(s01, s11);
#pragma unroll
            for (int of = 4; of < 32; of <<= 1) {
                mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, of));
                mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, of));
            }
            const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
            const float r0 = mn0 == -INFINITY ? 0.f : mn0, r1 = mn1 == -INFINITY ? 0.f : mn1;
            const float al0 = exp2f(m0 - r0), al1 = exp2f(m1 - r1);
            m0 = mn0; m1 = mn1;
            const float p00 = exp2f(s00 - r0), p01 = exp2f(s01 - r1), p10 = exp2f(s10 - r0), p11 = exp2f(s11 - r1);
            float ps0 = p00 + p10, ps1 = p01 + p11;
#pragma unroll
            for (int of = 4; of < 32; of <<= 1) {
                ps0 += __shfl_xor_sync(0xffffffffu, ps0, of);
                ps1 += __shfl_xor_sync(0xffffffffu, ps1, of);
            }
            l0 = l0 * al0 + ps0;
            l1 = l1 * al1 + ps1;
#pragma unroll
            for (int i = 0; i < 8; ++i) { o[i][0] *= al0; o[i][1] *= al1; o[i][2] *= al0; o[i][3] *= al1; }
            // P^T B-fragments via movmatrix: [token x head] 8x8 blocks -> [head-major] operand layout
            const uint32_t pb0 = movmatrix_t(pack_bf16(p00, p01));
            const uint32_t pb1 = movmatrix_t(pack_bf16(p10, p11));
            // ---- O^T += V^T P^T
            const int s2 = (u + 1) % RING;
            mbar_wait(&full_bar[s2], ((u + 1) / RING) & 1);
            const uint32_t vbase = ring_u + s2 * UNIT_BYTES;
            if (tile == patch_tile && patch_warp) {
                if (lane < 16)
                    *reinterpret_cast<uint4*>(ring + s2 * UNIT_BYTES + unit_off(pos % DT, lane)) =
                        *reinterpret_cast<const uint4*>(newkv + HD + lane * 8);
                __syncwarp();
            }
#pragma unroll
            for (int mt = 0; mt < 8; ++mt) {
                uint32_t va[4];
                ldsm_x4_t(va, vbase + unit_off(warp * 16 + (lane & 7) + ((lane >> 4) << 3), mt * 2 + ((lane >> 3) & 1)));
                mma16816(o[mt], va, pb0, pb1);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[s2]);
        }
    }

    // ---- merge the 4 warps' states (ring memory is free: every unit was consumed by every warp)
    if (tsm >= 0 && tid == 0) trace_mark_at(TR_ATTN_MARK + 7, 4 + tsm, 5);
    asm volatile("bar.sync 1, 128;" ::: "memory");          // consumer warps only
    float* red_o = reinterpret_cast<float*>(ring);          // [4 warps][8 heads][128]
    float* red_ml = red_o + 4 * 8 * HD;                     // [4][8][2]
#pragma unroll
    for (int mt = 0; mt < 8; ++mt) {
        const int d = mt * 16 + g;
        red_o[(warp * 8 + 2 * t) * HD + d] = o[mt][0];
        red_o[(warp * 8 + 2 * t + 1) * HD + d] = o[mt][1];
        red_o[(warp * 8 + 2 * t) * HD + d + 8] = o[mt][2];
        red_o[(warp * 8 + 2 * t + 1) * HD + d + 8] = o[mt][3];
    }
    if (g == 0) {
        red_ml[(warp * 8 + 2 * t) * 2] = m0; red_ml[(warp * 8 + 2 * t) * 2 + 1] = l0;
        red_ml[(warp * 8 + 2 * t + 1) * 2] = m1; red_ml[(warp * 8 + 2 * t + 1) * 2 + 1] = l1;
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");
    for (int i = tid; i < G * (HD / 2); i += 128) {
        const int h = i / (HD / 2), dp = (i % (HD / 2)) * 2;
        if (dp >= a.head_dim) continue;                 // padding columns
        float M = -INFINITY;
#pragma unroll
        for (int w = 0; w < 4; ++w) M = fmaxf(M, red_ml[(w * 8 + h) * 2]);
        float L = 0.f, o0 = 0.f, o1 = 0.f;
#pragma unroll
        for (int w = 0; w < 4; ++w) {
            const float mw = red_ml[(w * 8 + h) * 2];
            const float f = mw == -INFINITY ? 0.f : exp2f(mw - M);
            L += red_ml[(w * 8 + h) * 2 + 1] * f;
            o0 += red_o[(w * 8 + h) * HD + dp] * f;
            o1 += red_o[(w * 8 + h) * HD + dp + 1] * f;
        }
        const int head = kvh * G + h;
        if (a.kv_splits == 1) {
            const float inv = L > 0.f ? 1.f / L : 0.f;
            *reinterpret_cast<uint32_t*>(a.out + (size_t)row * a.n_heads * a.head_dim + head * a.head_dim + dp) =
                pack_bf16(o0 * inv, o1 * inv);
        } else {
            float* w = a.ws + (((size_t)row * a.n_heads + head) * a.kv_splits + split) * (HD + 2);
            w[dp] = o0;
            w[dp + 1] = o1;
            if (dp == 0) { w[HD] = M; w[HD + 1] = L; }
        }
    }
    if (tsm >= 0 && tid == 0) trace_mark_at(TR_ATTN_MARK + 8, 4 + tsm, 6);
    trace_end(tr_slot);
}

// combine split-KV partials: grid (n_heads, rows), 64 threads (dim pairs)
__global__ void decode_attn_combine_kernel(const float* __restrict__ ws, __nv_bfloat16* __restrict__ out,
                                           const int32_t* __restrict__ slot, int n_heads, int kv_splits, int head_dim) {
    griddep_launch();
    griddep_wait();
    const int head = blockIdx.x, row = blockIdx.y;
    if (slot[row] < 0) return;
    const float* w = ws + ((size_t)row * n_heads + head) * kv_splits * (HD + 2);
    float m = -INFINITY;
    for (int s = 0; s < kv_splits; ++s) m = fmaxf(m, w[s * (HD + 2) + HD]);
    float l = 0.f, o0 = 0.f, o1 = 0.f;
    const int dp = threadIdx.x;
    if (dp * 2 >= head_dim) return;
    for (int s = 0; s < kv_splits; ++s) {
        const float* p = w + s * (HD + 2);
        const float ms = p[HD];
        if (ms == -INFINITY) continue;                // empty split
        const float f = exp2f(ms - m);
        l += p[HD + 1] * f;
        o0 += p[dp * 2] * f;
        o1 += p[dp * 2 + 1] * f;
    }
    const float inv = l > 0.f ? 1.f / l : 0.f;
    *reinterpret_cast<uint32_t*>(out + (size_t)row * n_heads * head_dim + head * head_dim + dp * 2) = pack_bf16(o0 * inv, o1 * inv);
}

int pick_kv_splits(int rows, int n_kv_heads) {
    int ks = 1;
    while (rows * n_kv_heads * ks < 2 * num_sms() && ks < 8) ks *= 2;
    return ks;
}

size_t decode_attn_ws_bytes(int rows, int n_heads, int kv_splits) {
    return kv_splits > 1 ? (size_t)rows * n_heads * kv_splits * (HD + 2) * sizeof(float) : 0;
}

int decode_attn_make_maps(DecodeAttnArgs* a, int n_pages) {
    const long long rows = (long long)n_pages * a->n_kv_heads * (a->page_table ? KV_PAGE : a->ctx_max);
    if (rows <= 0 || rows > 0x7fffffffLL || a->ctx_max % DT) return RR_ERR_ARG;
    int rc = make_tmap_bf16_2d(&a->tmK, a->k_cache, (int)rows, HD, HD, DT);
    if (rc == RR_OK) rc = make_tmap_bf16_2d(&a->tmV, a->v_cache, (int)rows, HD, HD, DT);
    if (rc == RR_OK) rc = make_tmap_bf16_2d(&a->tmK16, a->k_cache, (int)rows, HD, HD, 16);
    if (rc == RR_OK) rc = make_tmap_bf16_2d(&a->tmV16, a->v_cache, (int)rows, HD, HD, 16);
    a->trim_tail = getenv("RR_ATTN_NO_TRIM") ? 0 : 1;
    return rc;
}

template <int G>
static void launch_dec(const DecodeAttnArgs& a, cudaStream_t st) {
    static std::atomic<uint64_t> attr{0};
    if (ensure_dyn_smem(decode_attn_mma_kernel<G>, 227 * 1024, attr) != cudaSuccess) return;
    dim3 grid(a.n_kv_heads, a.rows, a.kv_splits);
    launch_pdl(decode_attn_mma_kernel<G>, grid, dim3(DEC_THREADS), (size_t)dec_smem(a), st, a);
    if (a.kv_splits > 1)
        launch_pdl(decode_attn_combine_kernel, dim3(a.n_heads, a.rows), dim3(64), 0, st, (const float*)a.ws, a.out,
                   a.slot, a.n_heads, a.kv_splits, a.head_dim);
}

void launch_decode_attn(const DecodeAttnArgs& a, cudaStream_t st) {
    if (a.rows <= 0) return;
    const int G = a.n_heads / a.n_kv_heads;
    switch (G) {
        case 1: launch_dec<1>(a, st); break;
        case 2: launch_dec<2>(a, st); break;
        case 4: launch_dec<4>(a, st); break;
        case 8: launch_dec<8>(a, st); break;
        default: break;
    }
}

void rr_trace_set_attn_decode(unsigned long long* p) { rr_trace_set_local(p); }
void rr_trace_set_attn_decode_detail(int on) { rr_trace_set_detail_local(on); }

}  // namespace rr
