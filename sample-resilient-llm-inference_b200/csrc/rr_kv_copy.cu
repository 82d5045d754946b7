// rr_kv_copy.cu — prompt prefix caching: copy the first n positions of one KV slot into another, every layer, every kv
// head, K and V, for a whole list of (src slot, dst slot, n) in one launch.
//
// Each layer's cache is layer_rows rows of 128 bf16; position p of (slot, kv head) is row kv_row(...) (rr_kernels.h).  A
// chunk of 64 positions never crosses a page, so chunk c of a (layer, slot, kv head) is one contiguous run of 64 x 256 B: in
// the slot-contiguous layout a piece of the slot's segment, in the paged one page table[slot][c]; source and destination
// each go through their own table row.  Grid (chunks of 64 positions, layer x kv head, copy); a CTA moves one chunk of K and
// the same chunk of V with 16-byte loads, all issued before the first store.  HBM-bound: 2 x n x 256 B x layers x kv heads
// read and as many written per copy.
#include "rr_kernels.h"
#include "rr_launch.cuh"

namespace rr {
namespace {

constexpr int KC_THREADS = 256;
constexpr int KC_VEC = 4;                                   // uint4 per thread and tensor
constexpr int KC_CHUNK = KC_THREADS * KC_VEC;               // uint4 per CTA and tensor = 64 positions of 256 B

__global__ void __launch_bounds__(KC_THREADS)
kv_copy_prefix_kernel(const __grid_constant__ KvCopyList c, __nv_bfloat16* __restrict__ k_cache,
                      __nv_bfloat16* __restrict__ v_cache, long long layer_rows, int n_kv_heads, int ctx_max,
                      const int32_t* __restrict__ page_table, int pages_per_slot) {
    griddep_launch();
    const int i = blockIdx.z;
    const int l = blockIdx.y / n_kv_heads, h = blockIdx.y - l * n_kv_heads;
    const int n_vec = c.n[i] * 16;                          // 128 bf16 = 16 uint4 per position
    const int v0 = blockIdx.x * KC_CHUNK;
    if (v0 >= n_vec) return;
    const int p0 = blockIdx.x * (KC_CHUNK / 16);            // first position of the chunk
    const size_t layer = (size_t)l * layer_rows;
    const size_t src = (layer + kv_row(page_table, pages_per_slot, n_kv_heads, ctx_max, c.src[i], h, p0)) * 16;
    const size_t dst = (layer + kv_row(page_table, pages_per_slot, n_kv_heads, ctx_max, c.dst[i], h, p0)) * 16;
    const uint4* ks = reinterpret_cast<const uint4*>(k_cache) + src;
    const uint4* vs = reinterpret_cast<const uint4*>(v_cache) + src;
    uint4* kd = reinterpret_cast<uint4*>(k_cache) + dst;
    uint4* vd = reinterpret_cast<uint4*>(v_cache) + dst;
    griddep_wait();                                         // the preceding kernels may still write the source positions
    uint4 kr[KC_VEC], vr[KC_VEC];
#pragma unroll
    for (int j = 0; j < KC_VEC; ++j) {
        const int x = v0 + j * KC_THREADS + threadIdx.x;
        if (x < n_vec) { kr[j] = __ldcs(ks + (x - v0)); vr[j] = __ldcs(vs + (x - v0)); }
    }
#pragma unroll
    for (int j = 0; j < KC_VEC; ++j) {
        const int x = v0 + j * KC_THREADS + threadIdx.x;
        if (x < n_vec) { kd[x - v0] = kr[j]; vd[x - v0] = vr[j]; }
    }
}

}  // namespace

int kv_copy_check(const KvCopyList& c, int n_slots, int ctx_max) {
    if (c.count < 1 || c.count > KV_COPY_MAX) return RR_ERR_ARG;
    for (int i = 0; i < c.count; ++i) {
        if (c.src[i] < 0 || c.src[i] >= n_slots || c.dst[i] < 0 || c.dst[i] >= n_slots) return RR_ERR_ARG;
        if (c.n[i] < 1 || c.n[i] > ctx_max) return RR_ERR_ARG;
        for (int j = 0; j < c.count; ++j)
            if ((j != i && c.dst[j] == c.dst[i]) || c.src[j] == c.dst[i]) return RR_ERR_ARG;
    }
    return RR_OK;
}

int launch_kv_copy(__nv_bfloat16* k_cache, __nv_bfloat16* v_cache, int n_layers, long long layer_rows, int n_kv_heads,
                   int ctx_max, const int32_t* page_table, int pages_per_slot, const KvCopyList& c, cudaStream_t st) {
    int max_n = 0;
    for (int i = 0; i < c.count; ++i) max_n = c.n[i] > max_n ? c.n[i] : max_n;
    const dim3 grid((max_n * 16 + KC_CHUNK - 1) / KC_CHUNK, n_layers * n_kv_heads, c.count);
    const cudaError_t e = launch_pdl(kv_copy_prefix_kernel, grid, dim3(KC_THREADS), 0, st, c, k_cache, v_cache, layer_rows,
                                     n_kv_heads, ctx_max, page_table, pages_per_slot);
    return e == cudaSuccess ? RR_OK : RR_ERR_CUDA;
}

}  // namespace rr
