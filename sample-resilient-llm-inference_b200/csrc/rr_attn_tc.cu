// rr_attn_tc.cu — prefill attention (K7) on Hopper tensor cores: causal flash attention with both contractions on
// wgmma, Q / K / V tiles staged by TMA, S, P and the O accumulator in registers.
//
// Persistent kernel, one CTA per SM, 9 warps:
//   warps 0-3   consumer warpgroup 0: query rows  0..63 of the item's 128-row tile
//   warps 4-7   consumer warpgroup 1: query rows 64..127
//   warp 8      TMA producer: the Q tile (128 rows x 128 dims) and a 4-deep ring of K/V tiles (64 keys x 128 dims
//               each) from the KV cache
// Per key tile a consumer warpgroup computes S = Q K^T (m64n64k16 x 8, both operands K-major in shared memory),
// the causal mask and the online softmax on the S registers, then O += P V (m64n128k16 x 4) with P straight from
// registers (the accumulator layout of S is the A-fragment layout of the next wgmma) and V as the MN-major B operand
// exactly as it lies in the cache: 64 dims (128 B) contiguous, 8 keys per 1024 B swizzle atom (SBO), the second
// 64-dim half one TMA box (8192 B) further (LBO).  A key tile that lies wholly above a warpgroup's rows (the last
// tile of warpgroup 0) is only waited for and released.
//
// Work item = (sequence, query head, 128-row query tile), heaviest (last) query tiles first, strided over the CTAs.
// KV addresses follow kv_row (rr_kernels.h): with a page table the producer looks up each key tile's page, else the tiles
// of a slot are consecutive.
// Prefix caching: a sequence's `len` query rows may sit at positions pos0 .. pos0 + len - 1 of its slot (seq_pos0; the
// prefix 0 .. pos0 - 1 is already in the cache).  They attend to positions 0 .. own position; the key tiles, the causal
// mask and the skip test use absolute positions, Q stays at the sequence's rows of q.  A query row visits key tiles
// 0, 1, ... in order whatever its tile, and a fully masked tile leaves m, l and O bit-unchanged (alpha = 1, P = 0 against
// finite V), so a row's output does not depend on pos0: it is the row of a cold run over the whole sequence, bit for bit.
// Sliding window (W > 0): a query tile starts at the key tile of its first row's first visible key, and keys below
// q - W + 1 are masked too; a tile wholly below a row's window leaves its state unchanged as well (also while the row has
// seen no key: m = -inf, l = 0, O = 0), so the same holds with a window.
// Any GQA group size (MHA included): the kv head is head / (n_heads / n_kv_heads).  Head dims below 128 (Phi-3-mini:
// 96) are zero-padded to 128 in q and the caches; only the true head dim is written.
//
// Replaces the remote bedrock:InvokeModel call (reference iam/policy.json:8).
#include "rr_ptx.cuh"
#include "rr_launch.cuh"
#include "rr_kernels.h"
#include <cstdlib>

namespace rr {
namespace {

constexpr int TQ = 128;                 // query rows per work item
constexpr int TKV = 64;                 // keys per tile
constexpr int NS = 4;                   // K/V ring depth
constexpr int TC_CONSUMERS = 256;       // two warpgroups
constexpr int TC_THREADS = TC_CONSUMERS + 32;
constexpr int TC_PRODUCER_WARP = TC_CONSUMERS / 32;
constexpr uint32_t Q_BYTES = 32768;     // [2 dim halves][128 rows][128 B]
constexpr uint32_t KV_BYTES = 16384;    // [2 dim halves][64 keys][128 B]
constexpr uint32_t OFF_Q = 0;
constexpr uint32_t OFF_KV = OFF_Q + Q_BYTES;
constexpr uint32_t OFF_BAR = OFF_KV + NS * 2 * KV_BYTES;
constexpr uint32_t TC_SMEM = OFF_BAR + 256 + 1024;   // + barriers + manual 1024 B alignment slack

struct Bars {
    uint64_t q_full, q_empty;
    uint64_t kv_full[NS], kv_empty[NS];
};
static_assert(sizeof(Bars) <= 256, "barrier block");

__device__ __forceinline__ float ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

struct Work {
    int qt, seq, head, tok0, len, pos0, kt0, n_kt;   // key tiles kt0 .. n_kt - 1
};
// Work item w -> (query tile, sequence, head).  The sequence bounds, its first position (and the slot, for the producer)
// are loaded one item ahead (WorkFetch) so their latency hides under the current item.
struct WorkFetch {
    int tok0 = 0, tok1 = 0, pos0 = 0, slot = 0;
};
__device__ __forceinline__ void fetch_work(const PrefillAttnArgs& a, int w, int n_work, bool want_slot, WorkFetch& f) {
    if (w >= n_work) return;
    const int seq = (w % (a.n_seqs * a.n_heads)) / a.n_heads;
    f.tok0 = __ldg(a.seq_start + seq);
    f.tok1 = __ldg(a.seq_start + seq + 1);
    f.pos0 = a.seq_pos0 ? __ldg(a.seq_pos0 + seq) : 0;
    if (want_slot) f.slot = __ldg(a.seq_slot + seq);
}
__device__ __forceinline__ bool decode_work(const PrefillAttnArgs& a, int w, int max_qt, const WorkFetch& f, Work& k) {
    const int per_qt = a.n_seqs * a.n_heads;
    const int qrev = w / per_qt, rem = w - qrev * per_qt;
    k.qt = max_qt - 1 - qrev;
    k.seq = rem / a.n_heads;
    k.head = rem - k.seq * a.n_heads;
    k.tok0 = f.tok0;
    k.len = f.tok1 - f.tok0;
    k.pos0 = f.pos0;
    if (k.qt * TQ >= k.len) return false;
    // key tiles up to the tile's last query position (absolute: the cached prefix comes first)
    const int rows = (k.qt + 1) * TQ < k.len ? (k.qt + 1) * TQ : k.len;
    k.n_kt = (k.pos0 + rows + TKV - 1) / TKV;
    // sliding window: from the tile of the first row's first visible key (0 while that row is below the window)
    k.kt0 = a.window > 0 ? max(0, k.pos0 + k.qt * TQ - a.window + 1) / TKV : 0;
    return true;
}

__global__ void __launch_bounds__(TC_THREADS, 1)
prefill_attn_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                       const __grid_constant__ CUtensorMap tmV, const PrefillAttnArgs a) {
    extern __shared__ uint8_t tc_smem_raw[];
    uint8_t* smem = align_smem_1024(tc_smem_raw);
    Bars* bars = reinterpret_cast<Bars*>(smem + OFF_BAR);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    griddep_launch();
    const int tr_slot = trace_begin(TR_ATTN_PF);
    if (threadIdx.x == TC_CONSUMERS) {
        tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
        mbar_init(&bars->q_full, 1); mbar_init(&bars->q_empty, TC_CONSUMERS / 32);
        for (int s = 0; s < NS; ++s) { mbar_init(&bars->kv_full[s], 1); mbar_init(&bars->kv_empty[s], TC_CONSUMERS / 32); }
        fence_barrier_init();
    }
    __syncthreads();

    const int G = a.n_heads / a.n_kv_heads;
    const int max_qt = (a.max_len + TQ - 1) / TQ;
    const int n_work = max_qt * a.n_seqs * a.n_heads;

    griddep_wait();
    trace_dep(tr_slot);

    if (warp == TC_PRODUCER_WARP) {
        // ------------------------------------------------------------------ TMA producer
        if (elect_one()) {
            uint32_t kv_it = 0, q_it = 0;
            WorkFetch nf;
            fetch_work(a, blockIdx.x, n_work, true, nf);
            for (int w = blockIdx.x; w < n_work; w += gridDim.x) {
                Work k;
                const WorkFetch f = nf;
                fetch_work(a, w + gridDim.x, n_work, true, nf);
                if (!decode_work(a, w, max_qt, f, k)) continue;
                const int kvh = k.head / G;
                const bool paged = a.page_table != nullptr;
                mbar_wait(&bars->q_empty, (q_it & 1) ^ 1);
                mbar_arrive_expect_tx(&bars->q_full, Q_BYTES);
                for (int c = 0; c < 2; ++c)
                    tma_load_2d(smem + OFF_Q + c * 16384, &tmQ, &bars->q_full, k.head * 128 + c * 64, k.tok0 + k.qt * TQ);
                ++q_it;
                // a 64-key tile never crosses a page: one table lookup per tile, the next tile's issued before this tile's
                // ring-slot wait so that its latency hides under the wait
                auto kv_tile_row = [&](int j) {
                    return (int)kv_page_row(paged, kv_page(a.page_table, a.pages_per_slot, f.slot, j * TKV), a.n_kv_heads,
                                            a.ctx_max, kvh, j * TKV);
                };
                int kv_next = kv_tile_row(k.kt0);
                for (int j = k.kt0; j < k.n_kt; ++j, ++kv_it) {
                    const uint32_t s = kv_it % NS;
                    const int kv_r = kv_next;
                    if (j + 1 < k.n_kt) kv_next = kv_tile_row(j + 1);
                    mbar_wait(&bars->kv_empty[s], ((kv_it / NS) & 1) ^ 1);
                    mbar_arrive_expect_tx(&bars->kv_full[s], 2 * KV_BYTES);
                    uint8_t* dst = smem + OFF_KV + s * 2 * KV_BYTES;
                    for (int c = 0; c < 2; ++c) {
                        tma_load_2d(dst + c * 8192, &tmK, &bars->kv_full[s], c * 64, kv_r);
                        tma_load_2d(dst + KV_BYTES + c * 8192, &tmV, &bars->kv_full[s], c * 64, kv_r);
                    }
                }
            }
        }
    } else {
        // ------------------------------------------------------------------ consumer warpgroups
        const int g = warp >> 2, w4 = warp & 3;
        const int r_in = 64 * g + 16 * w4 + (lane >> 2);            // this thread's rows: r_in and r_in + 8 of the tile
        const int cq = 2 * (lane & 3);                               // first of its two columns in every group of 8
        const float sc = a.scale * 1.4426950408889634f;
        const uint32_t q_u = smem_u32(smem + OFF_Q), kv_u = smem_u32(smem + OFF_KV);
        uint32_t kv_it = 0, q_it = 0;
        WorkFetch nf;
        fetch_work(a, blockIdx.x, n_work, false, nf);
        for (int w = blockIdx.x; w < n_work; w += gridDim.x) {
            Work k;
            const WorkFetch f = nf;
            fetch_work(a, w + gridDim.x, n_work, false, nf);
            if (!decode_work(a, w, max_qt, f, k)) continue;
            const int q0 = k.qt * TQ + r_in;                         // query indices inside the sequence
            // causal / ragged bound (inclusive) and the warpgroup's last row, as absolute positions of the slot
            const int last0 = k.pos0 + min(q0, k.len - 1), last1 = k.pos0 + min(q0 + 8, k.len - 1);
            const int wg_last_row = k.pos0 + k.qt * TQ + 64 * g + 63;
            // sliding window: the first visible key of each row (a lower causal bound), and of the warpgroup's first row.
            // Without a window the bounds lie below every key.
            const int W = a.window > 0 ? a.window : (1 << 30);
            const int first0 = last0 - W + 1, first1 = last1 - W + 1;
            const int wg_first_key = k.pos0 + k.qt * TQ + 64 * g - W + 1;
            float o[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) o[i] = 0.f;
            float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // running max (log2 domain), partial row sums
            mbar_wait(&bars->q_full, q_it & 1);
            ++q_it;
            for (int j = k.kt0; j < k.n_kt; ++j, ++kv_it) {
                const uint32_t s = kv_it % NS;
                mbar_wait(&bars->kv_full[s], (kv_it / NS) & 1);
                const int key0 = j * TKV;
                if (key0 <= wg_last_row && key0 + TKV > wg_first_key) {
                    const uint32_t k_u = kv_u + s * 2 * KV_BYTES, v_u = k_u + KV_BYTES;
                    float sa[32];
                    wgmma_fence_regs(sa);
                    wgmma_fence();
#pragma unroll
                    for (int ks = 0; ks < 8; ++ks)
                        wgmma_ss<64>(sa, gmma_desc_sw128(q_u + (ks >> 2) * 16384 + g * 8192) + (ks & 3) * 2,
                                     gmma_desc_sw128(k_u + (ks >> 2) * 8192) + (ks & 3) * 2, ks > 0 ? 1u : 0u);
                    wgmma_commit();
                    wgmma_wait<0>();
                    wgmma_fence_regs(sa);
                    // ---- causal mask, online softmax (a row lives in the 4 threads of a quad)
                    const int lim0 = last0 - key0, lim1 = last1 - key0;
                    const int low0 = first0 - key0, low1 = first1 - key0;
                    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int col = 8 * jj + cq + e;
                            if (col > lim0 || col < low0) sa[4 * jj + e] = -INFINITY;
                            if (col > lim1 || col < low1) sa[4 * jj + 2 + e] = -INFINITY;
                            mx0 = fmaxf(mx0, sa[4 * jj + e]);
                            mx1 = fmaxf(mx1, sa[4 * jj + 2 + e]);
                        }
                    }
#pragma unroll
                    for (int x = 1; x <= 2; x <<= 1) {
                        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, x));
                        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, x));
                    }
                    // A window can mask a row's whole tile before its first visible key (m = n = -inf): the exponents
                    // then use 0 instead of -inf - (-inf) = NaN, giving alpha = 0 and P = 0, so the row stays empty.
                    const float n0 = fmaxf(m0, mx0 * sc), n1 = fmaxf(m1, mx1 * sc);
                    const float e0n = n0 == -INFINITY ? 0.f : n0, e1n = n1 == -INFINITY ? 0.f : n1;
                    const float al0 = ex2(m0 - e0n), al1 = ex2(m1 - e1n);   // m = -inf on the first tile: 0
                    m0 = n0; m1 = n1;
                    l0 *= al0; l1 *= al1;
#pragma unroll
                    for (int jj = 0; jj < 16; ++jj) {
                        o[4 * jj] *= al0; o[4 * jj + 1] *= al0;
                        o[4 * jj + 2] *= al1; o[4 * jj + 3] *= al1;
                    }
                    uint32_t pa[4][4];                                  // P as the A fragments of the 4 k16 steps
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int b = 8 * kk + 4 * h;
                            const float e0 = ex2(fmaf(sa[b], sc, -e0n)), e1 = ex2(fmaf(sa[b + 1], sc, -e0n));
                            const float e2 = ex2(fmaf(sa[b + 2], sc, -e1n)), e3 = ex2(fmaf(sa[b + 3], sc, -e1n));
                            l0 += e0 + e1;
                            l1 += e2 + e3;
                            pa[kk][2 * h] = pack_bf16(e0, e1);
                            pa[kk][2 * h + 1] = pack_bf16(e2, e3);
                        }
                    }
                    wgmma_fence_regs(o);
                    wgmma_fence();
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk)                      // 16 keys = two 8-key swizzle atoms (2048 B) per step
                        wgmma_rs_n128_tb(o, pa[kk], gmma_desc_sw128(v_u, 8192) + kk * (2048 >> 4), 1u);
                    wgmma_commit();
                    wgmma_wait<0>();
                    wgmma_fence_regs(o);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&bars->kv_empty[s]);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&bars->q_empty);                 // Q may be overwritten by the next item
            // ---- O / l -> bf16, true head dims only
#pragma unroll
            for (int x = 1; x <= 2; x <<= 1) {
                l0 += __shfl_xor_sync(0xffffffffu, l0, x);
                l1 += __shfl_xor_sync(0xffffffffu, l1, x);
            }
            const float inv0 = l0 > 0.f ? 1.f / l0 : 0.f, inv1 = l1 > 0.f ? 1.f / l1 : 0.f;
            const size_t row_pitch = (size_t)a.n_heads * a.head_dim;
            __nv_bfloat16* ob = a.out + (size_t)k.tok0 * row_pitch + (size_t)k.head * a.head_dim;
#pragma unroll
            for (int jj = 0; jj < 16; ++jj) {
                const int d = 8 * jj + cq;
                if (d < a.head_dim) {
                    if (q0 < k.len)
                        *reinterpret_cast<uint32_t*>(ob + (size_t)q0 * row_pitch + d) = pack_bf16(o[4 * jj] * inv0, o[4 * jj + 1] * inv0);
                    if (q0 + 8 < k.len)
                        *reinterpret_cast<uint32_t*>(ob + (size_t)(q0 + 8) * row_pitch + d) =
                            pack_bf16(o[4 * jj + 2] * inv1, o[4 * jj + 3] * inv1);
                }
            }
        }
    }
    __syncthreads();
    trace_end(tr_slot);
}

}  // namespace

bool prefill_attn_tc_eligible(const PrefillAttnArgs& a) {
    const int G = a.n_kv_heads > 0 ? a.n_heads / a.n_kv_heads : 0;
    return a.has_maps && G >= 1 && a.n_heads % a.n_kv_heads == 0 && a.ctx_max % TKV == 0 && a.head_dim % 8 == 0;
}

// q: [q_rows, n_heads*128]; caches: [kv_rows = n_pages*n_kv_heads*P, 128] (kv_row).  Boxes: Q 64 x 128 rows,
// K/V 64 x 64 rows, 128-byte swizzle.
int prefill_attn_make_maps(PrefillAttnArgs* a, long long q_rows, long long kv_rows) {
    a->has_maps = 0;
    if (q_rows <= 0 || kv_rows <= 0 || q_rows > 0x7fffffffLL || kv_rows > 0x7fffffffLL) return RR_ERR_ARG;
    int rc = make_tmap_bf16_2d(&a->tmQ, a->q, (int)q_rows, a->n_heads * 128, a->n_heads * 128, TQ);
    if (rc != RR_OK) return rc;
    rc = make_tmap_bf16_2d(&a->tmK, a->k_cache, (int)kv_rows, 128, 128, TKV);
    if (rc != RR_OK) return rc;
    rc = make_tmap_bf16_2d(&a->tmV, a->v_cache, (int)kv_rows, 128, 128, TKV);
    if (rc != RR_OK) return rc;
    a->has_maps = 1;
    return RR_OK;
}

int launch_prefill_attn_tc(const PrefillAttnArgs& a, cudaStream_t st) {
    static std::atomic<uint64_t> attr{0};
    if (ensure_dyn_smem(prefill_attn_tc_kernel, (int)TC_SMEM, attr) != cudaSuccess) return RR_ERR_CUDA;
    const int n_work = ((a.max_len + TQ - 1) / TQ) * a.n_seqs * a.n_heads;
    const int grid = n_work < num_sms() ? n_work : num_sms();
    cudaError_t e = launch_pdl(prefill_attn_tc_kernel, dim3(grid), dim3(TC_THREADS), (size_t)TC_SMEM, st,
                               a.tmQ, a.tmK, a.tmV, a);
    return e == cudaSuccess ? RR_OK : RR_ERR_CUDA;
}

// The one prefill attention path: the wgmma kernel serves every group size, so there is nothing to fall back to: an
// ineligible call fails.
int launch_prefill_attn(const PrefillAttnArgs& a, cudaStream_t st) {
    if (a.n_seqs <= 0 || a.max_len <= 0) return RR_OK;
    if (!prefill_attn_tc_eligible(a)) return RR_ERR_ARG;
    return launch_prefill_attn_tc(a, st);
}

void rr_trace_set_attn_tc(unsigned long long* p) { rr_trace_set_local(p); }

}  // namespace rr
