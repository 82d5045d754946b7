// rr_elementwise.cu — the HBM-bound glue between the projections: embedding gather (K3),
// split-K reduce + residual add + RMSNorm (K4), RoPE + KV-cache append (K6), SiLU*mul,
// greedy argmax (K11 tail).  All are row-parallel, 16-byte vectorised, fp32 math.
// Each consumer reads the producing GEMM's output either as fp32 split-K partials
// P[z][row][col] (decode orientation) or as one bf16 matrix (prefill orientation).
// Every kernel is PDL-aware (rr_launch.cuh): constants may be touched before griddep_wait().
//
// Replaces (together with rr_gemm.cu / rr_attn_tc.cu / rr_attn_decode.cu) the remote bedrock:InvokeModel call
// (reference iam/policy.json:8; src/demo_cris.py:233-238).
#include "rr_ptx.cuh"
#include "rr_launch.cuh"
#include "rr_kernels.h"

namespace rr {

// ---- reading a GEMM output ---------------------------------------------------------------------
// 4 consecutive columns of one row, summed over split planes.
__device__ __forceinline__ float4 part_load4(const PartIn& p, int row, int col) {
    if (p.is_bf16) {
        const uint2 v = *reinterpret_cast<const uint2*>(
            reinterpret_cast<const __nv_bfloat16*>(p.ptr) + (size_t)row * p.ld + col);
        return make_float4(bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y));
    }
    const float* base = reinterpret_cast<const float*>(p.ptr) + (size_t)row * p.ld + col;
    float4 acc = *reinterpret_cast<const float4*>(base);
#pragma unroll 8
    for (int z = 1; z < p.n_splits; ++z) {
        const float4 t = *reinterpret_cast<const float4*>(base + (size_t)z * p.split_stride);
        acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
    }
    return acc;
}

__device__ __forceinline__ float block_sum(float v, float* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = (lane < nw) ? red[lane] : 0.f;
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    __syncthreads();
    return t;
}

// ---- K3 embedding gather -----------------------------------------------------------------------
__global__ void embed_kernel(const int32_t* __restrict__ ids, const __nv_bfloat16* __restrict__ table,
                             float* __restrict__ x, int hidden, const int32_t* __restrict__ row_active) {
    griddep_launch();
    const int tr_slot = trace_begin(TR_EMBED);
    griddep_wait();
    trace_dep(tr_slot);
    const int row = blockIdx.x;
    if (row_active && row_active[row] < 0) return;
    const int id = ids[row];
    const __nv_bfloat16* src = table + (size_t)id * hidden;
    float* dst = x + (size_t)row * hidden;
    for (int c = threadIdx.x * 8; c < hidden; c += blockDim.x * 8) {
        const uint4 v = ldg_nc_v4(src + c);
        float4 a = make_float4(bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y));
        float4 b = make_float4(bf16_lo(v.z), bf16_hi(v.z), bf16_lo(v.w), bf16_hi(v.w));
        *reinterpret_cast<float4*>(dst + c) = a;
        *reinterpret_cast<float4*>(dst + c + 4) = b;
    }
    trace_end(tr_slot);
}

void launch_embed(const int32_t* ids, const __nv_bfloat16* table, float* x, int rows, int hidden,
                  const int32_t* row_active, cudaStream_t st) {
    if (rows <= 0) return;
    launch_pdl(embed_kernel, dim3(rows), dim3(256), 0, st, ids, table, x, hidden, row_active);
}

// ---- K4 residual add + RMSNorm (+ split-K reduce) ------------------------------------------------
// One CTA per row; the row (hidden <= 8192) stays in registers between the sum-of-squares pass and
// the normalise pass: x and the split planes are read exactly once.
// Decode (few rows, latency-bound): 1024 threads, one float4 each, so every load of a thread is independent.
// Prefill (thousands of rows, bandwidth-bound): 256 threads, 4 float4 each.

template <int THREADS, int MAXV>
__global__ void __launch_bounds__(THREADS)
add_rmsnorm_kernel(float* __restrict__ x, PartIn part, const __nv_bfloat16* __restrict__ w,
                   __nv_bfloat16* __restrict__ xn, int hidden, float eps, unsigned* __restrict__ zero, int zero_n,
                   float* __restrict__ rowss_out, int n_part_out) {
    __shared__ float red[32];
    griddep_launch();
    const int tr_slot = trace_begin(TR_NORM);
    const int row = blockIdx.x;
    float* xr = x + (size_t)row * hidden;
    // norm weights are constants: fetch them before waiting for the producer
    uint2 wv[MAXV];
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int c = (threadIdx.x + i * THREADS) * 4;
        if (c < hidden) wv[i] = *reinterpret_cast<const uint2*>(w + c);
    }
    griddep_wait();
    trace_dep(tr_slot);
    // optional: reset the dependency counters of the fused MLP kernel that follows (its previous user has completed)
    for (int i = blockIdx.x * THREADS + threadIdx.x; i < zero_n; i += gridDim.x * THREADS) zero[i] = 0u;
    float4 v[MAXV];
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int c = (threadIdx.x + i * THREADS) * 4;
        if (c < hidden) {
            v[i] = *reinterpret_cast<float4*>(xr + c);
            if (part.ptr) {
                const float4 p = part_load4(part, row, c);
                v[i].x += p.x; v[i].y += p.y; v[i].z += p.z; v[i].w += p.w;
            }
            ss += v[i].x * v[i].x + v[i].y * v[i].y + v[i].z * v[i].z + v[i].w * v[i].w;
        }
    }
    // the residual is written back only after every load of this thread has been issued: a store inside the load
    // loop would fence the following loads (possible aliasing) and turn them into a latency chain
    if (part.ptr) {
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            const int c = (threadIdx.x + i * THREADS) * 4;
            if (c < hidden) *reinterpret_cast<float4*>(xr + c) = v[i];
        }
    }
    ss = block_sum(ss, red);
    // deferred norm: hand sum(x^2) to the consuming GEMM's epilogue and leave the operand un-normalised
    if (rowss_out != nullptr && (int)threadIdx.x < n_part_out)
        rowss_out[(size_t)row * n_part_out + threadIdx.x] = threadIdx.x == 0 ? ss : 0.f;
    const float inv = rowss_out != nullptr ? 1.f : rsqrtf(ss / (float)hidden + eps);
    __nv_bfloat16* out = xn + (size_t)row * hidden;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int c = (threadIdx.x + i * THREADS) * 4;
        if (c < hidden) {
            uint2 o;
            o.x = pack_bf16(v[i].x * inv * bf16_lo(wv[i].x), v[i].y * inv * bf16_hi(wv[i].x));
            o.y = pack_bf16(v[i].z * inv * bf16_lo(wv[i].y), v[i].w * inv * bf16_hi(wv[i].y));
            *reinterpret_cast<uint2*>(out + c) = o;
        }
    }
    trace_end(tr_slot);
}

// Decode variant (<= 256 rows, fp32 planes, <= 8 of them, hidden <= 4096): one memory round trip and a register budget that
// leaves room for the next kernel's CTA.
//  * every load of a thread -- x and ALL split planes of both of its column groups -- is issued before the first add.  The
//    generic kernel sums the planes in a loop whose trip count is a run-time value: the compiler keeps it rolled, the add of
//    plane z stalls on its load and the load of plane z + 1 is only issued after it, i.e. n_splits dependent L2 round trips.
//  * 512 threads x 88 registers: 4 warps x 88 x 32 = 11 K of the 16 K registers of each SM sub-partition, which leaves room for
//    the 2 warps x 80 registers the next GEMM's CTA (6 warps) puts on a sub-partition.  The generic kernel runs 1024 threads x
//    64 registers = the whole register file: on the 64 SMs that host a row, the next GEMM's CTA could not start until the norm
//    had finished, and its weight prefetch before the PDL wait was lost on 43 % of the SMs (tools/trace_gemm.py).
// predicated 16-byte load as a volatile asm: volatile asm statements keep their program order, so a block of these followed by
// pin4() on every result forces "all loads issued, then one wait" (nvcc otherwise sinks each load next to its add to save
// registers, which re-creates the dependent-round-trip chain)
__device__ __forceinline__ float4 ldg_f4_pred(const float* p, bool pred) {
    float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
    asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %5, 0;\n\t@q ld.global.v4.f32 {%0, %1, %2, %3}, [%4];\n\t}"
                 : "+f"(r.x), "+f"(r.y), "+f"(r.z), "+f"(r.w) : "l"(p), "r"((int)pred) : "memory");
    return r;
}
__device__ __forceinline__ void pin4(float4& v) { asm volatile("" : "+f"(v.x), "+f"(v.y), "+f"(v.z), "+f"(v.w)); }

template <int MAXV>
__global__ void __maxnreg__(88)
add_rmsnorm_dec_kernel(float* __restrict__ x, PartIn part, const __nv_bfloat16* __restrict__ w,
                       __nv_bfloat16* __restrict__ xn, int hidden, float eps, unsigned* __restrict__ zero, int zero_n) {
    constexpr int THREADS = 512, NP = 8;
    __shared__ float red[32];
    __shared__ float one_s;
    if (threadIdx.x == 0) one_s = 1.f;
    griddep_launch();
    const int tr_slot = trace_begin(TR_NORM);
    const int row = blockIdx.x;
    float* xr = x + (size_t)row * hidden;
    uint2 wv[MAXV];
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int c = (threadIdx.x + i * THREADS) * 4;
        wv[i] = c < hidden ? *reinterpret_cast<const uint2*>(w + c) : make_uint2(0u, 0u);
    }
    griddep_wait();
    trace_dep(tr_slot);
    for (int i = blockIdx.x * THREADS + threadIdx.x; i < zero_n; i += gridDim.x * THREADS) zero[i] = 0u;
    const int ns = part.ptr ? part.n_splits : 0;
    float4 v[MAXV], t[MAXV][NP];
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int c = (threadIdx.x + i * THREADS) * 4;
        const bool on = c < hidden;
        v[i] = ldg_f4_pred(xr + c, on);
        const float* base = reinterpret_cast<const float*>(part.ptr) + (size_t)row * part.ld + c;
#pragma unroll
        for (int z = 0; z < NP; ++z) t[i][z] = ldg_f4_pred(base + (size_t)z * part.split_stride, on && z < ns);
    }
    // ptxas re-interleaves loads and adds to save registers (even across a barrier or an empty asm), which re-creates the chain.
    // What it cannot move: every add below is an FMA with a factor 1.0f that is read from shared memory AFTER a block barrier
    // that follows the loads -- fma(t, 1, acc) == acc + t exactly, and no add can issue before all 18 loads have.
    __syncthreads();
    const float one = *reinterpret_cast<volatile float*>(&one_s);
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        // same association as part_load4: (((p0 + p1) + p2) + ...) first, then x + that sum
        float4 acc = t[i][0];
#pragma unroll
        for (int z = 1; z < NP; ++z) {
            acc.x = fmaf(t[i][z].x, one, acc.x); acc.y = fmaf(t[i][z].y, one, acc.y);
            acc.z = fmaf(t[i][z].z, one, acc.z); acc.w = fmaf(t[i][z].w, one, acc.w);
        }
        v[i].x += acc.x; v[i].y += acc.y; v[i].z += acc.z; v[i].w += acc.w;
        ss += v[i].x * v[i].x + v[i].y * v[i].y + v[i].z * v[i].z + v[i].w * v[i].w;
    }
    if (ns > 0) {
#pragma unroll
        for (int i = 0; i < MAXV; ++i) {
            const int c = (threadIdx.x + i * THREADS) * 4;
            if (c < hidden) *reinterpret_cast<float4*>(xr + c) = v[i];
        }
    }
    ss = block_sum(ss, red);
    const float inv = rsqrtf(ss / (float)hidden + eps);
    __nv_bfloat16* out = xn + (size_t)row * hidden;
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
        const int c = (threadIdx.x + i * THREADS) * 4;
        if (c < hidden) {
            uint2 o;
            o.x = pack_bf16(v[i].x * inv * bf16_lo(wv[i].x), v[i].y * inv * bf16_hi(wv[i].x));
            o.y = pack_bf16(v[i].z * inv * bf16_lo(wv[i].y), v[i].w * inv * bf16_hi(wv[i].y));
            *reinterpret_cast<uint2*>(out + c) = o;
        }
    }
    trace_end(tr_slot);
}

void launch_add_rmsnorm(float* x, PartIn part, const __nv_bfloat16* w, __nv_bfloat16* xn, int rows,
                        int hidden, float eps, cudaStream_t st, unsigned* zero, int zero_n) {
    if (rows <= 0 || hidden > 8192) return;
    if (rows <= 256 && hidden <= 4096 && (part.ptr == nullptr || (!part.is_bf16 && part.n_splits <= 8)))
        launch_pdl(add_rmsnorm_dec_kernel<2>, dim3(rows), dim3(512), 0, st, x, part, w, xn, hidden, eps, zero, zero_n);
    else if (rows <= 256)
        launch_pdl(add_rmsnorm_kernel<1024, 2>, dim3(rows), dim3(1024), 0, st, x, part, w, xn, hidden, eps, zero, zero_n,
                   (float*)nullptr, 0);
    else if (hidden <= 4096)      // fewer registers -> more rows in flight per SM (HBM-bound at thousands of rows)
        launch_pdl(add_rmsnorm_kernel<256, 4>, dim3(rows), dim3(256), 0, st, x, part, w, xn, hidden, eps, zero, zero_n,
                   (float*)nullptr, 0);
    else
        launch_pdl(add_rmsnorm_kernel<256, 8>, dim3(rows), dim3(256), 0, st, x, part, w, xn, hidden, eps, zero, zero_n,
                   (float*)nullptr, 0);
}

// Prefill chunks: the kernel, and so the order of the sum of squares, depends on the hidden size only, never on the row
// count, so a token's bits do not depend on how many tokens share its chunk (a prefix-cache hit must reproduce a cold
// prefill exactly).  These are the kernels chunks of more than 256 rows always ran.
void launch_add_rmsnorm_pf(float* x, const __nv_bfloat16* w, __nv_bfloat16* xn, int rows, int hidden, float eps,
                           cudaStream_t st, float* rowss_out, int n_part_out) {
    if (rows <= 0 || hidden > 8192) return;
    PartIn none; none.ptr = nullptr; none.is_bf16 = 0; none.n_splits = 1; none.split_stride = 0; none.ld = 0;
    if (hidden <= 4096)
        launch_pdl(add_rmsnorm_kernel<256, 4>, dim3(rows), dim3(256), 0, st, x, none, w, xn, hidden, eps, (unsigned*)nullptr, 0,
                   rowss_out, n_part_out);
    else
        launch_pdl(add_rmsnorm_kernel<256, 8>, dim3(rows), dim3(256), 0, st, x, none, w, xn, hidden, eps, (unsigned*)nullptr, 0,
                   rowss_out, n_part_out);
}

// ---- SiLU(gate) * up -----------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
silu_mul_kernel(PartIn gu, __nv_bfloat16* __restrict__ act, int inter) {
    griddep_launch();
    const int tr_slot = trace_begin(TR_SILU);
    griddep_wait();
    trace_dep(tr_slot);
    const int row = blockIdx.y;
    const int c = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (c >= inter) return;
    const float4 g = part_load4(gu, row, c);
    const float4 u = part_load4(gu, row, inter + c);
    auto f = [](float a, float b) { return __fdividef(a, 1.f + __expf(-a)) * b; };   // same formula as silu_mul (rr_gemm.cu)
    uint2 o;
    o.x = pack_bf16(f(g.x, u.x), f(g.y, u.y));
    o.y = pack_bf16(f(g.z, u.z), f(g.w, u.w));
    *reinterpret_cast<uint2*>(act + (size_t)row * inter + c) = o;
    trace_end(tr_slot);
}

void launch_silu_mul(PartIn gu, __nv_bfloat16* act, int rows, int inter, cudaStream_t st) {
    if (rows <= 0) return;
    dim3 grid((inter / 4 + 255) / 256, rows);
    launch_pdl(silu_mul_kernel, grid, dim3(256), 0, st, gu, act, inter);
}

// ---- K6 RoPE + KV-cache append --------------------------------------------------------------------
// head_dim = 128, HF "rotate_half" convention: pairs (i, i + 64), inv_freq_i = theta^(-i/64).
// cos/sin come from a table [ctx_max][64] (float2) built once per engine in double precision;
// without a table (kernel-level tests) they are computed inline.
__global__ void rope_table_kernel(float2* __restrict__ table, int ctx_max, double theta, int half) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= ctx_max * 64) return;
    const int pos = idx >> 6, i = idx & 63;
    if (i >= half) { table[idx] = make_float2(1.f, 0.f); return; }
    const double inv_freq = pow(theta, -(double)i / (double)half);
    // the oracle (and HF) form the angle in fp32: pos * float(inv_freq)
    const float ang = (float)pos * (float)inv_freq;
    table[idx] = make_float2((float)cos((double)ang), (float)sin((double)ang));
}

void launch_rope_table(float2* table, int ctx_max, float theta, int head_dim, cudaStream_t st) {
    const int n = ctx_max * 64;
    rope_table_kernel<<<(n + 255) / 256, 256, 0, st>>>(table, ctx_max, (double)theta, head_dim / 2);
}

__device__ __forceinline__ float2 part_load2(const PartIn& p, int row, int col) {   // 2 consecutive columns
    if (p.is_bf16) {
        const uint32_t v = *reinterpret_cast<const uint32_t*>(
            reinterpret_cast<const __nv_bfloat16*>(p.ptr) + (size_t)row * p.ld + col);
        return make_float2(bf16_lo(v), bf16_hi(v));
    }
    const float* base = reinterpret_cast<const float*>(p.ptr) + (size_t)row * p.ld + col;
    float2 acc = *reinterpret_cast<const float2*>(base);
    for (int z = 1; z < p.n_splits; ++z) {
        const float2 t = *reinterpret_cast<const float2*>(base + (size_t)z * p.split_stride);
        acc.x += t.x; acc.y += t.y;
    }
    return acc;
}

__global__ void __launch_bounds__(256)
rope_kv_kernel(RopeArgs a) {
    griddep_launch();
    const int tr_slot = trace_begin(TR_ROPE);
    griddep_wait();
    trace_dep(tr_slot);
    const int row = blockIdx.x;
    const int slot = a.slot[row];
    if (slot < 0) return;
    const int pos = a.pos[row];
    const int page = kv_page(a.page_table, a.pages_per_slot, slot, pos);        // one lookup per token row
    const bool paged = a.page_table != nullptr;
    // work items of 2 rotation pairs: (head, i..i+1) for q heads then k heads, then v copies (4 elements).
    // hd = true head dim: rotation pairs (i, i + hd/2); destination rows are padded to 128 (pad stays zero).
    const int hd = a.head_dim, half = hd >> 1, ipw = half >> 1, vpw = hd >> 2;      // items per head
    const int n_q = a.n_heads * ipw, n_k = a.n_kv_heads * ipw;
    const int total = n_q + n_k + a.n_kv_heads * vpw;
    const float l2t = a.table ? 0.f : log2f(a.theta);
    for (int it = threadIdx.x; it < total; it += blockDim.x) {
        if (it < n_q + n_k) {
            const bool is_q = it < n_q;
            const int j = is_q ? it : it - n_q;
            const int head = j / ipw, i = (j % ipw) * 2;
            const int col = (is_q ? 0 : a.n_heads * hd) + head * hd + i;
            const float2 lo = part_load2(a.qkv, row, col);
            const float2 hi = part_load2(a.qkv, row, col + half);
            float c0, s0, c1, s1;
            if (a.table) {
                const float4 t = *reinterpret_cast<const float4*>(a.table + (size_t)pos * 64 + i);
                c0 = t.x; s0 = t.y; c1 = t.z; s1 = t.w;
            } else {
                sincosf((float)pos * exp2f(-l2t * (float)i / (float)half), &s0, &c0);
                sincosf((float)pos * exp2f(-l2t * (float)(i + 1) / (float)half), &s1, &c1);
            }
            const uint32_t o_lo = pack_bf16(lo.x * c0 - hi.x * s0, lo.y * c1 - hi.y * s1);
            const uint32_t o_hi = pack_bf16(hi.x * c0 + lo.x * s0, hi.y * c1 + lo.y * s1);
            __nv_bfloat16* dst = is_q
                ? a.q_out + (size_t)row * (a.n_heads * 128) + head * 128 + i
                : a.k_cache + kv_page_row(paged, page, a.n_kv_heads, a.ctx_max, head, pos) * 128 + i;
            *reinterpret_cast<uint32_t*>(dst) = o_lo;
            *reinterpret_cast<uint32_t*>(dst + half) = o_hi;
        } else {
            const int j = it - n_q - n_k;            // 4 elements each
            const int head = j / vpw, i4 = (j % vpw) * 4;
            const int col = (a.n_heads + a.n_kv_heads) * hd + head * hd + i4;
            const float4 v = part_load4(a.qkv, row, col);
            __nv_bfloat16* dst = a.v_cache + kv_page_row(paged, page, a.n_kv_heads, a.ctx_max, head, pos) * 128 + i4;
            uint2 o;
            o.x = pack_bf16(v.x, v.y);
            o.y = pack_bf16(v.z, v.w);
            *reinterpret_cast<uint2*>(dst) = o;
        }
    }
    trace_end(tr_slot);
}

void launch_rope_kv(const RopeArgs& a, cudaStream_t st) {
    if (a.rows <= 0) return;
    launch_pdl(rope_kv_kernel, dim3(a.rows), dim3(256), 0, st, a);
}

// ---- greedy argmax (lowest index wins ties; NaN never wins; no value above -inf: token 0) -------------
__global__ void __launch_bounds__(1024)
argmax_kernel(PartIn logits, int vocab, int32_t* __restrict__ out_tok, float* __restrict__ out_val,
              const int32_t* __restrict__ row_active, int32_t* __restrict__ pos_inc) {
    __shared__ float s_v[32];
    __shared__ int s_i[32];
    griddep_launch();
    const int tr_slot = trace_begin(TR_ARGMAX);
    griddep_wait();
    trace_dep(tr_slot);
    const int row = blockIdx.x;
    if (row_active && row_active[row] < 0) return;
    const float* r = reinterpret_cast<const float*>(logits.ptr) + (size_t)row * logits.ld;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    const int v4 = vocab & ~3;
    // 8 independent 16-byte loads per round: the compare chain is loop-carried, and with one load per iteration the 31
    // iterations of a 128 k vocabulary were 31 dependent memory round trips (51 us per step; now ~4 rounds)
    constexpr int U = 8;
    const int stride = blockDim.x * 4;
    for (int c0 = threadIdx.x * 4; c0 < v4; c0 += stride * U) {
        float4 v[U];
#pragma unroll
        for (int k = 0; k < U; ++k) {
            const int c = c0 + k * stride;
            v[k] = c < v4 ? *reinterpret_cast<const float4*>(r + c) : make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
        }
#pragma unroll
        for (int k = 0; k < U; ++k) {                      // increasing index order: the lowest index wins ties
            const int c = c0 + k * stride;
            if (v[k].x > best) { best = v[k].x; bi = c; }
            if (v[k].y > best) { best = v[k].y; bi = c + 1; }
            if (v[k].z > best) { best = v[k].z; bi = c + 2; }
            if (v[k].w > best) { best = v[k].w; bi = c + 3; }
        }
    }
    for (int c = v4 + threadIdx.x; c < vocab; c += blockDim.x) {
        const float v = r[c];
        if (v > best) { best = v; bi = c; }
    }
    auto better = [](float v, int i, float bv, int bi_) { return v > bv || (v == bv && i < bi_); };
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (better(ov, oi, best, bi)) { best = ov; bi = oi; }
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { s_v[warp] = best; s_i[warp] = bi; }
    __syncthreads();
    if (warp == 0) {
        const int nw = blockDim.x >> 5;
        best = lane < nw ? s_v[lane] : -INFINITY;
        bi = lane < nw ? s_i[lane] : 0x7fffffff;
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (better(ov, oi, best, bi)) { best = ov; bi = oi; }
        }
        if (lane == 0) {
            // only a value above -inf replaces the start (-inf, 0x7fffffff), and NaN never compares above: a row of -inf
            // and NaN only picks token 0, as torch.argmax does for an all -inf row, so the next step's embedding gather
            // stays inside the table
            out_tok[row] = best > -INFINITY ? bi : 0;
            if (out_val) out_val[row] = best;
            if (pos_inc) pos_inc[row] += 1;
        }
    }
    trace_end(tr_slot);
}

void launch_argmax(PartIn logits, int rows, int vocab, int32_t* out_tok, float* out_val,
                   const int32_t* row_active, int32_t* pos_inc, cudaStream_t st) {
    if (rows <= 0) return;
    launch_pdl(argmax_kernel, dim3(rows), dim3(1024), 0, st, logits, vocab, out_tok, out_val, row_active, pos_inc);
}

// ---- log-softmax + top-k (logprobs) ---------------------------------------------------------------
// One CTA per LP_CHUNK columns of a row (so 64 rows x 128 k vocabulary is 1024 CTAs, not 64 on 132 SMs): it reads its chunk
// from HBM once into shared memory and writes the chunk's max m_c, s_c = sum exp(x - m_c) and its k best (value, id) in the
// argmax order (value descending, id ascending).  k rounds over shared memory each pick the best element strictly after the
// previous pick in that order, so equal values need no special case.  The merge CTA of the row combines the chunks in chunk
// order: m = max m_c, s = sum s_c exp(m_c - m), lse = m + log s, and ranks the chunks' candidates.  Every sum runs in a
// fixed order, so two calls give the same bits.
constexpr int LP_THREADS = 256;
struct LpPart {
    float m, s;
    float v[LP_MAX_TOP];
    int32_t id[LP_MAX_TOP];   // -1: the chunk has fewer than k columns
};

__device__ __forceinline__ bool lp_before(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

__device__ __forceinline__ float block_max(float v, float* red) {
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = (lane < nw) ? red[lane] : -INFINITY;
    for (int o = 16; o > 0; o >>= 1) t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, o));
    __syncthreads();
    return t;
}

// best (value, id) of the block in the argmax order; every thread gets it
__device__ __forceinline__ void block_best(float& v, int& i, float* s_v, int* s_i) {
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (lp_before(ov, oi, v, i)) { v = ov; i = oi; }
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    if (lane == 0) { s_v[warp] = v; s_i[warp] = i; }
    __syncthreads();
    v = lane < nw ? s_v[lane] : -INFINITY;
    i = lane < nw ? s_i[lane] : 0x7fffffff;
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (lp_before(ov, oi, v, i)) { v = ov; i = oi; }
    }
    __syncthreads();
}

__global__ void __launch_bounds__(LP_THREADS)
logprobs_chunk_kernel(const float* __restrict__ logits, int ld, int vocab, const int32_t* __restrict__ top_n, int max_top,
                      LpPart* __restrict__ ws) {
    __shared__ __align__(16) float s_x[LP_CHUNK];
    __shared__ float s_rv[32];
    __shared__ int s_ri[32];
    griddep_launch();
    const int tr_slot = trace_begin(TR_LOGPROBS);
    griddep_wait();
    trace_dep(tr_slot);
    const int row = blockIdx.y, c = blockIdx.x;
    const int tn = top_n[row];
    if (tn < 0) return;
    const int k = min(max(1, tn), max_top);
    const int c0 = c * LP_CHUNK;
    const int n = min(LP_CHUNK, vocab - c0);
    const float* x = logits + (size_t)row * ld + c0;          // 16-byte aligned: ld % 4 == 0, c0 % 4 == 0
    float mx = -INFINITY;
    const int n4 = n & ~3;
#pragma unroll 8
    for (int j = threadIdx.x * 4; j < n4; j += LP_THREADS * 4) {
        const float4 v = __ldcs(reinterpret_cast<const float4*>(x + j));
        *reinterpret_cast<float4*>(s_x + j) = v;
        mx = fmaxf(mx, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
    }
    for (int j = n4 + threadIdx.x; j < n; j += LP_THREADS) {     // scalar tail (vocab % 4 != 0)
        const float v = x[j];
        s_x[j] = v;
        mx = fmaxf(mx, v);
    }
    __syncthreads();
    const float m = block_max(mx, s_rv);
    float s = 0.f;
    // a chunk of -inf columns only (a JSON-mode mask) has m = -inf: it adds s = 0, not expf(-inf - -inf) = NaN
    if (m != -INFINITY)
        for (int j = threadIdx.x; j < n; j += LP_THREADS) s += expf(s_x[j] - m);
    s = block_sum(s, s_rv);
    LpPart* out = ws + (size_t)row * gridDim.x + c;
    if (threadIdx.x == 0) { out->m = m; out->s = s; }
    float pv = INFINITY;                                          // previous pick; (+inf, -1) precedes every element
    int pi = -1;
    for (int r = 0; r < k; ++r) {
        float bv = -INFINITY;
        int bi = 0x7fffffff;
        for (int j = threadIdx.x; j < n; j += LP_THREADS) {
            const float v = s_x[j];
            const int id = c0 + j;
            if (lp_before(pv, pi, v, id) && lp_before(v, id, bv, bi)) { bv = v; bi = id; }
        }
        block_best(bv, bi, s_rv, s_ri);
        if (threadIdx.x == 0) { out->v[r] = bv; out->id[r] = bi == 0x7fffffff ? -1 : bi; }
        pv = bv; pi = bi;
    }
    trace_end(tr_slot);
}

__global__ void __launch_bounds__(LP_THREADS)
logprobs_merge_kernel(const int32_t* __restrict__ top_n, int max_top, int n_chunks, const LpPart* __restrict__ ws,
                      float* __restrict__ lp_out, int32_t* __restrict__ id_out, const float* __restrict__ logits, int ld,
                      const int32_t* __restrict__ tok, float* __restrict__ tok_lp) {
    __shared__ float s_v[LP_MAX_CHUNKS * LP_MAX_TOP];
    __shared__ int s_i[LP_MAX_CHUNKS * LP_MAX_TOP];
    __shared__ float s_lse;
    griddep_launch();
    const int tr_slot = trace_begin(TR_LOGPROBS);
    griddep_wait();
    trace_dep(tr_slot);
    const int row = blockIdx.x;
    const int tn = top_n[row];
    if (tn < 0) return;
    const int k = min(max(1, tn), max_top);
    const LpPart* p = ws + (size_t)row * n_chunks;
    const int nk = n_chunks * k;
    for (int t = threadIdx.x; t < nk; t += blockDim.x) {
        const int c = t / k, j = t - c * k;
        s_v[t] = p[c].v[j];
        s_i[t] = p[c].id[j];
    }
    if (threadIdx.x == 0) {
        float m = -INFINITY;
        for (int c = 0; c < n_chunks; ++c) m = fmaxf(m, p[c].m);
        float s = 0.f;
        for (int c = 0; c < n_chunks; ++c)
            if (p[c].m != -INFINITY) s += p[c].s * expf(p[c].m - m);      // an all -inf chunk adds nothing
        s_lse = m + logf(s);
        // a sampled token may lie outside the top k: its own pair, from the same value and lse as the ranked entries
        if (tok) tok_lp[row] = logits[(size_t)row * ld + tok[row]] - s_lse;
    }
    __syncthreads();
    const float lse = s_lse;
    // the global k best are among the chunks' k best; a candidate's rank is the number of candidates before it
    for (int t = threadIdx.x; t < nk; t += blockDim.x) {
        const int id = s_i[t];
        if (id < 0) continue;
        const float v = s_v[t];
        int rank = 0;
        for (int u = 0; u < nk; ++u) rank += (s_i[u] >= 0 && lp_before(s_v[u], s_i[u], v, id)) ? 1 : 0;
        if (rank < k) {
            lp_out[(size_t)row * max_top + rank] = v - lse;
            id_out[(size_t)row * max_top + rank] = id;
        }
    }
    trace_end(tr_slot);
}

size_t logprobs_ws_bytes(int rows, int vocab) {
    return (size_t)rows * ((vocab + LP_CHUNK - 1) / LP_CHUNK) * sizeof(LpPart);
}

void launch_logprobs(const float* logits, int ld, int rows, int vocab, const int32_t* top_n, int max_top, void* ws,
                     float* lp_out, int32_t* id_out, cudaStream_t st, const int32_t* tok, float* tok_lp) {
    if (rows <= 0) return;
    const int nc = (vocab + LP_CHUNK - 1) / LP_CHUNK;
    launch_pdl(logprobs_chunk_kernel, dim3(nc, rows), dim3(LP_THREADS), 0, st, logits, ld, vocab, top_n, max_top,
               (LpPart*)ws);
    launch_pdl(logprobs_merge_kernel, dim3(rows), dim3(LP_THREADS), 0, st, top_n, max_top, nc, (const LpPart*)ws, lp_out,
               id_out, logits, ld, tok, tok_lp);
}

// ---- seeded temperature / top-p sampling ------------------------------------------------------------
// Contract (include/rr_b200.h, rr_op_sample): for a row with T > 0, tau = the largest logit value whose set {x >= tau}
// holds at least top_p of the mass of softmax(x / T); the token is argmax over {x >= tau} of x / T + G_i (lowest id on
// ties), G_i = -log(-log u_i), u_i from Philox4x32-10 with key = seed and counter = (i, position, 0, 0).
//
// Three launches.  (1) One CTA per row finds tau by a mass-weighted radix select on the order-preserving key of x: the row
// max m, then one pass per key digit (11, 11, 10 bits) building the histogram of w = exp((x - m) / T) over the keys that
// share the digits found so far; the crossing bin's digit is appended.  Weights are summed as 2^-40 fixed-point integers,
// so the shared-memory atomics are order-independent and the result is bit-reproducible; an element lighter than 2^-40 of
// the row max counts as 0.  top_p >= 1 skips the search (tau = -inf).  (2) One CTA per LP_CHUNK columns draws the chunk's
// Gumbel-max candidate over {x >= tau}.  (3) One warp per row merges the chunks' candidates in the argmax order, which is
// a total order, so the result does not depend on the merge order either.  A row without any candidate keeps its token.
constexpr int SP_THREADS = 1024;
constexpr int SP_BINS = 2048;
struct SpPart { float v; int32_t id; };

__device__ __forceinline__ uint32_t sample_key(float x) {
    uint32_t b = __float_as_uint(x);
    if (b == 0x80000000u) b = 0;                             // -0 and +0 are one value
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float sample_key_value(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// First 32-bit word of Philox4x32-10 (Salmon et al., SC'11) for counter (c0, c1, 0, 0) and the 64-bit key `seed`.
__device__ __forceinline__ uint32_t philox_first(uint32_t c0, uint32_t c1, uint64_t seed) {
    uint32_t c2 = 0, c3 = 0, k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return c0;
}

// u = (2 (r >> 9) + 1) / 2^24: 2^23 odd multiples of 2^-24, exact in fp32 and strictly inside (0, 1)
__device__ __forceinline__ float sample_gumbel(uint32_t r) {
    const float u = (float)(((r >> 9) << 1) | 1u) * 5.9604644775390625e-8f;
    return -logf(-logf(u));
}

// f(v) for every value of a row, each thread in increasing column order; U 16-byte loads in flight per thread (the row is
// read once per pass, and a single load per iteration would leave each pass latency-bound)
template <class F>
__device__ __forceinline__ void sample_row_pass(const float* __restrict__ x, int vocab, F&& f) {
    constexpr int U = 4;
    const int v4 = vocab & ~3, stride = SP_THREADS * 4;
    for (int c0 = threadIdx.x * 4; c0 < v4; c0 += stride * U) {
        float4 v[U];
#pragma unroll
        for (int k = 0; k < U; ++k) {
            const int c = c0 + k * stride;
            v[k] = c < v4 ? *reinterpret_cast<const float4*>(x + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int k = 0; k < U; ++k) {
            if (c0 + k * stride >= v4) break;
            f(v[k].x); f(v[k].y); f(v[k].z); f(v[k].w);
        }
    }
    for (int j = v4 + threadIdx.x; j < vocab; j += SP_THREADS) f(x[j]);
}

__device__ __forceinline__ unsigned long long sample_weight(float x, float m, float T) {
    return (unsigned long long)(expf((x - m) / T) * 1099511627776.0f);   // 2^40
}

__global__ void __launch_bounds__(SP_THREADS)
sample_threshold_kernel(const float* __restrict__ logits, int ld, int vocab, const float* __restrict__ temperature,
                        const float* __restrict__ top_p, float* __restrict__ tau_out) {
    __shared__ unsigned long long s_h[SP_BINS];
    __shared__ unsigned long long s_scan[32];
    __shared__ float s_red[32];
    __shared__ unsigned long long s_need, s_above;
    __shared__ uint32_t s_prefix;
    griddep_launch();
    const int tr_slot = trace_begin(TR_SAMPLE);
    griddep_wait();
    trace_dep(tr_slot);
    const int row = blockIdx.x, tid = threadIdx.x;
    const float T = temperature[row], p = top_p[row];
    if (!(T > 0.f)) return;
    if (p >= 1.f) {
        if (tid == 0) tau_out[row] = -INFINITY;
        return;
    }
    const float* x = logits + (size_t)row * ld;
    float mx = -INFINITY;
    sample_row_pass(x, vocab, [&](float v) { mx = fmaxf(mx, v); });
    const float m = block_max(mx, s_red);
    if (tid == 0) { s_prefix = 0; s_above = 0; }
    const int lane = tid & 31, warp = tid >> 5;
    for (int d = 0; d < 3; ++d) {
        const int shift = d == 0 ? 21 : (d == 1 ? 10 : 0);
        const int nbins = d == 2 ? 1024 : 2048;
        for (int b = tid; b < SP_BINS; b += SP_THREADS) s_h[b] = 0;
        __syncthreads();
        const uint32_t prefix = s_prefix;
        const int hi = shift + (d == 2 ? 10 : 11);          // key bits [hi, 32) are already fixed
        // consecutive elements of a thread often share a bin (a flat row sits in a few top-digit bins): add runs, not elements
        int run_bin = -1;
        unsigned long long run = 0;
        sample_row_pass(x, vocab, [&](float v) {
            const uint32_t k = sample_key(v);
            if (d > 0 && (k >> hi) != (prefix >> hi)) return;
            const int b = (int)((k >> shift) & (uint32_t)(nbins - 1));
            if (b != run_bin) {
                if (run) atomicAdd(&s_h[run_bin], run);
                run_bin = b; run = 0;
            }
            run += sample_weight(v, m, T);
        });
        if (run) atomicAdd(&s_h[run_bin], run);
        __syncthreads();
        // bins in descending key order: thread t holds bins nbins-1-2t and nbins-2-2t; inclusive scan over threads
        const int b0 = nbins - 1 - 2 * tid, b1 = b0 - 1;
        const unsigned long long h0 = b0 >= 0 ? s_h[b0] : 0, h1 = b1 >= 0 ? s_h[b1] : 0;
        unsigned long long a = h0 + h1, incl = a;
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) s_scan[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            unsigned long long w = s_scan[lane];
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned long long t = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += t;
            }
            s_scan[lane] = w;                                  // inclusive over warps
        }
        __syncthreads();
        incl += warp > 0 ? s_scan[warp - 1] : 0ull;
        if (d == 0 && tid == SP_THREADS - 1) {               // total mass Z: need = max(1, ceil(top_p Z))
            const double need = ceil((double)p * (double)incl);
            s_need = need < 1.0 ? 1ull : (unsigned long long)need;
        }
        __syncthreads();
        const unsigned long long need = s_need, above = s_above;
        const unsigned long long e0 = above + incl - a;        // mass of every key above bin b0
        // every thread has read s_above before the crossing thread overwrites it: a late reader of the new value would
        // shift its e0 and could find a second crossing
        __syncthreads();
        // the crossing bin is the first, in descending order, whose cumulative mass reaches `need`; exactly one thread has
        // it, because the mass above this prefix is < need and the mass up to the end of it is >= need
        if (e0 < need && e0 + a >= need) {
            const bool first = e0 + h0 >= need;
            s_prefix = prefix | ((uint32_t)(first ? b0 : b1) << shift);
            s_above = first ? e0 : e0 + h0;
        }
        __syncthreads();
    }
    if (tid == 0) tau_out[row] = sample_key_value(s_prefix);
    trace_end(tr_slot);
}

__global__ void __launch_bounds__(LP_THREADS)
sample_chunk_kernel(const float* __restrict__ logits, int ld, int vocab, const float* __restrict__ temperature,
                    const uint64_t* __restrict__ seed, const int32_t* __restrict__ position, const float* __restrict__ tau,
                    SpPart* __restrict__ ws) {
    __shared__ float s_v[32];
    __shared__ int s_i[32];
    griddep_launch();
    const int tr_slot = trace_begin(TR_SAMPLE);
    griddep_wait();
    trace_dep(tr_slot);
    const int row = blockIdx.y, c = blockIdx.x;
    const float T = temperature[row];
    if (!(T > 0.f)) return;
    const float t = tau[row];
    const uint64_t key = seed[row];
    const uint32_t pos = (uint32_t)position[row];
    const int c0 = c * LP_CHUNK;
    const int n = min(LP_CHUNK, vocab - c0);
    const float* x = logits + (size_t)row * ld + c0;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int j = threadIdx.x; j < n; j += LP_THREADS) {
        const float v = x[j];
        if (!(v >= t) || v == -INFINITY) continue;        // with top_p = 1, tau = -inf: a masked column is never drawn
        const int id = c0 + j;
        const float s = v / T + sample_gumbel(philox_first((uint32_t)id, pos, key));
        if (lp_before(s, id, bv, bi)) { bv = s; bi = id; }
    }
    block_best(bv, bi, s_v, s_i);
    if (threadIdx.x == 0) ws[(size_t)row * gridDim.x + c] = SpPart{bv, bi};
    trace_end(tr_slot);
}

__global__ void __launch_bounds__(32)
sample_merge_kernel(const float* __restrict__ temperature, int n_chunks, const SpPart* __restrict__ ws,
                    int32_t* __restrict__ out_tok) {
    griddep_launch();
    const int tr_slot = trace_begin(TR_SAMPLE);
    griddep_wait();
    trace_dep(tr_slot);
    const int row = blockIdx.x;
    if (!(temperature[row] > 0.f)) return;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int c = threadIdx.x; c < n_chunks; c += 32) {
        const SpPart q = ws[(size_t)row * n_chunks + c];
        if (lp_before(q.v, q.id, bv, bi)) { bv = q.v; bi = q.id; }
    }
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (lp_before(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    // no chunk had a candidate (every column -inf or NaN, or a NaN tau): the token the argmax wrote stays
    if (threadIdx.x == 0 && bi != 0x7fffffff) out_tok[row] = bi;
    trace_end(tr_slot);
}

size_t sample_ws_bytes(int rows, int vocab) {
    const size_t tau = ((size_t)rows * sizeof(float) + 15) & ~(size_t)15;
    return tau + (size_t)rows * ((vocab + LP_CHUNK - 1) / LP_CHUNK) * sizeof(SpPart);
}

void launch_sample(const float* logits, int ld, int rows, int vocab, const float* temperature, const float* top_p,
                   const uint64_t* seed, const int32_t* position, int32_t* out_tok, void* ws, cudaStream_t st) {
    if (rows <= 0) return;
    const int nc = (vocab + LP_CHUNK - 1) / LP_CHUNK;
    float* tau = (float*)ws;
    SpPart* part = (SpPart*)((char*)ws + (((size_t)rows * sizeof(float) + 15) & ~(size_t)15));
    launch_pdl(sample_threshold_kernel, dim3(rows), dim3(SP_THREADS), 0, st, logits, ld, vocab, temperature, top_p, tau);
    launch_pdl(sample_chunk_kernel, dim3(nc, rows), dim3(LP_THREADS), 0, st, logits, ld, vocab, temperature, seed, position,
               (const float*)tau, part);
    launch_pdl(sample_merge_kernel, dim3(rows), dim3(32), 0, st, temperature, nc, (const SpPart*)part, out_tok);
}

// ---- frequency / presence penalties and logit bias (rr_op_logit_penalties) ------------------------------------------
// One CTA per row, three phases separated by barriers: (1) x_j += b_j over the row's bias entries (unique ids: no two
// threads write one logit); (2) cnt[t] += 1 for every history token t, integer atomics into the row's [vocab] slice of the
// workspace; (3) per history entry old = atomicExch(&cnt[t], 0): the one thread that sees old > 0 applies the penalty with
// c = old.  Whichever thread wins computes the same value, and the exchange leaves the workspace zeroed for the next call.
// Work per row is O(history + bias entries); nothing is sized by shared memory, so the history has no cap.
constexpr int PEN_THREADS = 256;

__global__ void __launch_bounds__(PEN_THREADS)
logit_penalties_kernel(float* __restrict__ logits, int ld, int vocab, PenaltyArgs a, int32_t* __restrict__ cnt_ws) {
    griddep_launch();
    const int tr_slot = trace_begin(TR_PENALTY);
    griddep_wait();
    trace_dep(tr_slot);
    const int row = blockIdx.x, tid = threadIdx.x;
    const float af = a.freq[row], ap = a.pres[row];
    const int nb = min(max(a.n_bias[row], 0), a.bias_ld);
    const bool pen = af != 0.f || ap != 0.f;
    if (!pen && nb == 0) return;
    float* x = logits + (size_t)row * ld;
    int32_t* h = a.hist ? a.hist + (size_t)row * a.hist_ld : nullptr;
    int len = 0;
    if (h && a.app_tok) {
        // the engine's decode step: the row's input token (its last generated token, at position app_pos) joins the
        // history at index app_pos - gen0 before the logits are processed
        const int i = a.app_pos[row] - a.gen0[row];
        if (i >= 0 && i < a.hist_ld) {
            if (tid == 0) h[i] = a.app_tok[row];
            len = i + 1;
        }
        __syncthreads();
    } else if (h && a.hist_len) {
        len = min(max(a.hist_len[row], 0), a.hist_ld);
    }
    const int32_t* bid = a.bias_ids + (size_t)row * a.bias_ld;
    const float* bv = a.bias_vals + (size_t)row * a.bias_ld;
    for (int k = tid; k < nb; k += PEN_THREADS) {
        const int j = bid[k];
        if (j >= 0 && j < vocab) x[j] = __fadd_rn(x[j], bv[k]);
    }
    if (!pen || len == 0) { trace_end(tr_slot); return; }
    int32_t* cnt = cnt_ws + (size_t)row * vocab;
    __syncthreads();
    for (int k = tid; k < len; k += PEN_THREADS) {
        const int t = h[k];
        if (t >= 0 && t < vocab) atomicAdd(&cnt[t], 1);
    }
    __syncthreads();
    for (int k = tid; k < len; k += PEN_THREADS) {
        const int t = h[k];
        if (t < 0 || t >= vocab) continue;
        const int c = atomicExch(&cnt[t], 0);
        if (c > 0) x[t] = __fsub_rn(x[t], __fadd_rn(__fmul_rn((float)c, af), ap));
    }
    trace_end(tr_slot);
}

void launch_logit_penalties(float* logits, int ld, int rows, int vocab, const PenaltyArgs& a, int32_t* cnt_ws,
                            cudaStream_t st) {
    if (rows <= 0) return;
    launch_pdl(logit_penalties_kernel, dim3(rows), dim3(PEN_THREADS), 0, st, logits, ld, vocab, a, cnt_ws);
}

// ---- stop sequences (rr_op_stop_match) ---------------------------------------------------------------------------------
// One warp per row.  The warp stores the new token in the history, then walks the history back in 32-token steps and
// compacts (ballot + popc) the last <= STOP_MAX_LEN text bytes and the history index of each into shared memory, newest
// first; byteless tokens (< 3) are skipped, so the walk is O(STOP_MAX_LEN) except through runs of them.  Lane k then tests,
// for every sequence, "the last k + 1 (and k + 33) text bytes are the first k + 1 (k + 33) bytes of the sequence": the
// full-length test is a hit, shorter ones are partial matches; warp maxima pick the longest of each.  Integer work only,
// no atomics: the outputs are a function of the inputs.
constexpr int STOP_WARPS = 4;

__global__ void __launch_bounds__(32 * STOP_WARPS) stop_match_kernel(StopArgs a, int rows) {
    griddep_launch();
    griddep_wait();
    __shared__ uint8_t s_txt[STOP_WARPS][STOP_MAX_LEN];
    __shared__ int32_t s_idx[STOP_WARPS][STOP_MAX_LEN];
    __shared__ uint32_t s_stop[STOP_WARPS][STOP_MAX_SEQS * STOP_MAX_LEN / 4];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row = blockIdx.x * STOP_WARPS + warp;
    if (row >= rows) return;
    const int ns = min(a.n_stop[row], STOP_MAX_SEQS);
    if (ns <= 0 || (a.row_active && a.row_active[row] < 0)) return;
    const int i = a.position ? a.position[row] - a.gen0[row] : 0;
    if (i < 0 || i >= a.hist_ld) {
        if (lane == 0) { a.cut[row] = -1; a.hold[row] = 0; }
        return;
    }
    int32_t* h = a.hist + (size_t)(a.hist_row ? a.hist_row[row] : row) * a.hist_ld;
    const int newest = a.tok[row];
    if (lane == 0) h[i] = newest;
    const uint32_t* sb = reinterpret_cast<const uint32_t*>(a.bytes + (size_t)row * STOP_MAX_SEQS * STOP_MAX_LEN);
    s_stop[warp][lane] = sb[lane];
    s_stop[warp][lane + 32] = sb[lane + 32];
    __syncwarp();
    uint8_t* txt = s_txt[warp];
    int32_t* idx = s_idx[warp];
    int nb = 0;                                    // text bytes staged so far: txt[k] = the k-th newest, idx[k] its token
    for (int base = i; base >= 0 && nb < STOP_MAX_LEN; base -= 32) {
        const int j = base - lane;
        const int t = j >= 0 ? h[j] : 0;
        const unsigned m = __ballot_sync(0xffffffffu, t >= 3);
        const int k = nb + __popc(m & ((1u << lane) - 1u));
        if (t >= 3 && k < STOP_MAX_LEN) { txt[k] = (uint8_t)((t - 3) & 255); idx[k] = j; }
        nb += __popc(m);
    }
    nb = min(nb, STOP_MAX_LEN);
    __syncwarp();
    const uint8_t* stop = reinterpret_cast<const uint8_t*>(s_stop[warp]);
    int hit = 0, part = 0;                         // longest full / proper-prefix match this lane found, in bytes
    for (int s = 0; s < ns; ++s) {
        const int L = a.len[row * STOP_MAX_SEQS + s];
        if (L < 1 || L > STOP_MAX_LEN) continue;
        const uint8_t* q = stop + s * STOP_MAX_LEN;
        for (int kl = lane + 1; kl <= min(L, nb); kl += 32) {
            int j = 0;
            while (j < kl && q[j] == txt[kl - 1 - j]) ++j;
            if (j < kl) continue;
            if (kl == L) hit = max(hit, kl);
            else part = max(part, kl);
        }
    }
    hit = __reduce_max_sync(0xffffffffu, hit);
    part = __reduce_max_sync(0xffffffffu, part);
    if (lane != 0) return;
    if (hit > 0 && newest >= 3) { a.cut[row] = idx[hit - 1]; a.hold[row] = 0; }
    else { a.cut[row] = -1; a.hold[row] = part > 0 ? i + 1 - idx[part - 1] : 0; }
}

void launch_stop_match(const StopArgs& a, int rows, cudaStream_t st) {
    if (rows <= 0) return;
    launch_pdl(stop_match_kernel, dim3((rows + STOP_WARPS - 1) / STOP_WARPS), dim3(32 * STOP_WARPS), 0, st, a, rows);
}

// ---- JSON mode (rr_op_json_mask / rr_op_json_advance) -------------------------------------------------------------------
// The automaton both kernels run (tests/json_oracle.py states the same one in Python).  A JsonState holds the node, the
// depth and a bit per open container (array or object), the whitespace run and, in w1, the progress inside a literal, an
// escape, a \u escape or a multi-byte UTF-8 character.  All zero is the initial state (JN_START).
enum JsonNode : uint32_t {
    JN_START = 0,   // before the top-level value: '{'
    JN_OBJ_FIRST,   // after '{': a key or '}'
    JN_OBJ_KEY,     // after ',' in an object: a key
    JN_COLON,       // after a key: ':'
    JN_VALUE,       // after ':', or after ',' in an array: a value
    JN_ARR_FIRST,   // after '[': a value or ']'
    JN_AFTER,       // after a value in a container: ',' or the container's close
    JN_STR,         // in a string (w0 bit 24: it is a key)
    JN_ESC,         // after '\' in a string
    JN_HEX,         // in \uXXXX: w1 = hex digits still due
    JN_UTF8,        // in a multi-byte character: w1 = bytes due | lo << 8 | hi << 16, the next byte's range
    JN_LIT,         // in true / false / null: w1 = literal << 4 | bytes matched
    JN_MINUS,       // number: after '-'
    JN_ZERO,        //         after a leading '0'
    JN_INT,         //         in the integer digits
    JN_DOT,         //         after '.'
    JN_FRAC,        //         in the fraction digits
    JN_EXP,         //         after 'e' / 'E'
    JN_EXP_SIGN,    //         after the exponent's sign
    JN_EXP_DIG,     //         in the exponent digits
    JN_DONE         // the top-level object is closed: only trailing whitespace, which RFC 8259 allows (the choice has ended)
};

__device__ __forceinline__ bool json_ws(int c) { return c == ' ' || c == '\t' || c == '\n' || c == '\r'; }
__device__ __forceinline__ bool json_digit(int c) { return c >= '0' && c <= '9'; }

// One byte c: true and *s advanced when the state allows c, else false and *s unchanged.  Integer work only.
__device__ bool json_step(JsonState* s, int c) {
    uint64_t stack = s->stack;
    uint32_t node = s->w0 & 0xff, depth = (s->w0 >> 8) & 0xff, ws = (s->w0 >> 16) & 0xff, key = (s->w0 >> 24) & 1;
    uint32_t aux = s->w1;
    bool ok = false, structural = false;
    switch (node) {
    case JN_MINUS:
        if (json_digit(c)) { node = c == '0' ? JN_ZERO : JN_INT; ok = true; }
        break;
    case JN_ZERO:           // a byte that does not continue a number ends it and is read as in JN_AFTER
    case JN_INT:
        if (node == JN_INT && json_digit(c)) ok = true;
        else if (c == '.') { node = JN_DOT; ok = true; }
        else if (c == 'e' || c == 'E') { node = JN_EXP; ok = true; }
        else { node = JN_AFTER; structural = true; }
        break;
    case JN_DOT:
        if (json_digit(c)) { node = JN_FRAC; ok = true; }
        break;
    case JN_FRAC:
        if (json_digit(c)) ok = true;
        else if (c == 'e' || c == 'E') { node = JN_EXP; ok = true; }
        else { node = JN_AFTER; structural = true; }
        break;
    case JN_EXP:
        if (c == '+' || c == '-') { node = JN_EXP_SIGN; ok = true; }
        else if (json_digit(c)) { node = JN_EXP_DIG; ok = true; }
        break;
    case JN_EXP_SIGN:
        if (json_digit(c)) { node = JN_EXP_DIG; ok = true; }
        break;
    case JN_EXP_DIG:
        if (json_digit(c)) ok = true;
        else { node = JN_AFTER; structural = true; }
        break;
    case JN_STR:
        if (c == '"') { node = key ? JN_COLON : JN_AFTER; key = 0; ok = true; }
        else if (c == '\\') { node = JN_ESC; ok = true; }
        else if (c >= 0x20 && c < 0x80) ok = true;
        else if (c >= 0xC2 && c <= 0xF4) {   // a lead byte: no overlong (C0, C1, E0 80..9F, F0 80..8F), no surrogate
            const uint32_t n = c < 0xE0 ? 1 : c < 0xF0 ? 2 : 3;                // (ED A0..BF), nothing above U+10FFFF
            const uint32_t lo = c == 0xE0 ? 0xA0 : c == 0xF0 ? 0x90 : 0x80;
            const uint32_t hi = c == 0xED ? 0x9F : c == 0xF4 ? 0x8F : 0xBF;
            node = JN_UTF8; aux = n | lo << 8 | hi << 16; ok = true;
        }
        break;
    case JN_UTF8:
        if ((uint32_t)c >= ((aux >> 8) & 0xff) && (uint32_t)c <= (aux >> 16)) {
            const uint32_t n = (aux & 0xff) - 1;
            if (n == 0) node = JN_STR;
            else aux = n | 0x80u << 8 | 0xBFu << 16;
            ok = true;
        }
        break;
    case JN_ESC:
        if (c == '"' || c == '\\' || c == '/' || c == 'b' || c == 'f' || c == 'n' || c == 'r' || c == 't') {
            node = JN_STR; ok = true;
        } else if (c == 'u') { node = JN_HEX; aux = 4; ok = true; }
        break;
    case JN_HEX:
        if (json_digit(c) || (c >= 'a' && c <= 'f') || (c >= 'A' && c <= 'F')) {
            if (--aux == 0) node = JN_STR;
            ok = true;
        }
        break;
    case JN_LIT: {      // "true", "false", "null", little-endian
        const uint32_t lit = aux >> 4, pos = aux & 15, len = lit == 1 ? 5 : 4;
        const uint64_t w = lit == 0 ? 0x65757274ull : lit == 1 ? 0x65736c6166ull : 0x6c6c756eull;
        if ((uint32_t)c == ((w >> (8 * pos)) & 0xff)) {
            aux = lit << 4 | (pos + 1);
            if (pos + 1 == len) node = JN_AFTER;
            ok = true;
        }
        break;
    }
    case JN_DONE:
        ok = json_ws(c);
        break;
    default:
        structural = true;
    }
    if (structural) {
        if (json_ws(c)) {
            if (ws < JSON_MAX_WS) { ++ws; ok = true; }
        } else {
            const bool arr = depth > 0 && (stack >> (depth - 1) & 1);
            int push = -1;                         // 0: open an object, 1: an array
            bool pop = false;
            switch (node) {
            case JN_START:
                if (c == '{') push = 0;
                break;
            case JN_OBJ_FIRST:
            case JN_OBJ_KEY:
                if (c == '"') { node = JN_STR; key = 1; ok = true; }
                else if (c == '}' && node == JN_OBJ_FIRST) pop = true;
                break;
            case JN_COLON:
                if (c == ':') { node = JN_VALUE; ok = true; }
                break;
            case JN_AFTER:
                if (c == ',') { node = arr ? JN_VALUE : JN_OBJ_KEY; ok = true; }
                else if (c == (arr ? ']' : '}')) pop = true;
                break;
            default:            // JN_VALUE, JN_ARR_FIRST: a value
                if (c == ']' && node == JN_ARR_FIRST) pop = true;
                else if (c == '{' || c == '[') { if (depth < JSON_MAX_DEPTH) push = c == '['; }
                else if (c == '"') { node = JN_STR; key = 0; ok = true; }
                else if (c == '-') { node = JN_MINUS; ok = true; }
                else if (c == '0') { node = JN_ZERO; ok = true; }
                else if (json_digit(c)) { node = JN_INT; ok = true; }
                else if (c == 't' || c == 'f' || c == 'n') { node = JN_LIT; aux = (c == 't' ? 0 : c == 'f' ? 1 : 2) << 4 | 1; ok = true; }
            }
            if (push >= 0) {
                stack = (stack & ~(1ull << depth)) | ((uint64_t)push << depth);
                ++depth;
                node = push ? JN_ARR_FIRST : JN_OBJ_FIRST;
                ok = true;
            } else if (pop) {
                --depth;
                node = depth == 0 ? JN_DONE : JN_AFTER;
                ok = true;
            }
            if (ok) ws = 0;
        }
    }
    if (!ok) return false;
    if (node != JN_HEX && node != JN_UTF8 && node != JN_LIT) aux = 0;
    s->stack = stack;
    s->w0 = node | depth << 8 | ws << 16 | key << 24;
    s->w1 = aux;
    return true;
}

// Mask: LP_CHUNK is a multiple of JSON_THREADS = 256, so the columns of thread j in every chunk all carry the byte
// (j - 3) mod 256: the thread steps a copy of the state by that one byte and, when it is not allowed, writes -inf to all of
// its columns (and to columns 0..2, which carry no byte).  No shared memory, and the logits are never read.
constexpr int JSON_THREADS = 256;
static_assert(LP_CHUNK % JSON_THREADS == 0, "a chunk's columns repeat the byte pattern");

__global__ void __launch_bounds__(JSON_THREADS)
json_mask_kernel(float* __restrict__ logits, int ld, int vocab, const int32_t* __restrict__ fmt,
                 const int32_t* __restrict__ row_active, const JsonState* __restrict__ state) {
    griddep_launch();
    griddep_wait();
    const int row = blockIdx.y;
    if (fmt[row] == 0 || (row_active && row_active[row] < 0)) return;
    JsonState s = {0, 0, 0};
    if (state) s = state[row];
    const bool allowed = json_step(&s, (threadIdx.x + 253) & 255);
    const int c0 = blockIdx.x * LP_CHUNK, n = min(LP_CHUNK, vocab - c0);
    float* x = logits + (size_t)row * ld + c0;
    if (!allowed) {
#pragma unroll 4
        for (int j = threadIdx.x; j < n; j += JSON_THREADS) x[j] = -INFINITY;
    } else if (c0 == 0 && threadIdx.x < 3 && (int)threadIdx.x < n) {
        x[threadIdx.x] = -INFINITY;
    }
}

__global__ void __launch_bounds__(128)
json_advance_kernel(int rows, const int32_t* __restrict__ fmt, const int32_t* __restrict__ row_active,
                    const int32_t* __restrict__ tok, const JsonState* state_in, JsonState* state_out,
                    const int32_t* __restrict__ out_row, int32_t* __restrict__ done) {
    griddep_launch();
    griddep_wait();
    const int r = blockIdx.x * 128 + threadIdx.x;
    if (r >= rows || fmt[r] == 0 || (row_active && row_active[r] < 0)) return;
    JsonState s = {0, 0, 0};
    if (state_in) s = state_in[r];
    const int t = tok[r];
    if (t >= 3) json_step(&s, (t - 3) & 255);
    state_out[out_row ? out_row[r] : r] = s;
    done[r] = (s.w0 & 0xff) == JN_DONE ? 1 : 0;
}

void launch_json_mask(float* logits, int ld, int rows, int vocab, const int32_t* fmt, const int32_t* row_active,
                      const JsonState* state, cudaStream_t st) {
    if (rows <= 0) return;
    launch_pdl(json_mask_kernel, dim3((vocab + LP_CHUNK - 1) / LP_CHUNK, rows), dim3(JSON_THREADS), 0, st, logits, ld,
               vocab, fmt, row_active, state);
}

void launch_json_advance(int rows, const int32_t* fmt, const int32_t* row_active, const int32_t* tok,
                         const JsonState* state_in, JsonState* state_out, const int32_t* out_row, int32_t* done,
                         cudaStream_t st) {
    if (rows <= 0) return;
    launch_pdl(json_advance_kernel, dim3((rows + 127) / 128), dim3(128), 0, st, rows, fmt, row_active, tok, state_in,
               state_out, out_row, done);
}

// ---- embedding pool (rr_op_embed_pool) ------------------------------------------------------------
// One CTA of EMBED_POOL_THREADS per row.  Thread t owns the 8-column groups t, t + 256, ...; it squares its bf16 values in
// fp64 (exact: 8-bit mantissas) and sums them in column order, then a fixed xor tree per warp and warp 0..7 in order:
// the same shape every call, so the same bits.  The normalise pass reads the row again (it is in L1 / L2).
constexpr int EMBED_POOL_THREADS = 256;

__global__ void __launch_bounds__(EMBED_POOL_THREADS)
embed_pool_kernel(const __nv_bfloat16* __restrict__ xn, int ld, const int32_t* __restrict__ rows, int hidden,
                  float* __restrict__ out, int out_ld) {
    __shared__ double red[EMBED_POOL_THREADS / 32];
    griddep_launch();
    griddep_wait();
    const int i = blockIdx.x;
    const __nv_bfloat16* src = xn + (size_t)(rows ? rows[i] : i) * ld;
    double s = 0.0;
    for (int c = threadIdx.x * 8; c < hidden; c += EMBED_POOL_THREADS * 8) {
        const uint4 v = *reinterpret_cast<const uint4*>(src + c);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const double a = (double)bf16_lo(w[j]), b = (double)bf16_hi(w[j]);
            s += a * a;
            s += b * b;
        }
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    double S = 0.0;
#pragma unroll
    for (int w = 0; w < EMBED_POOL_THREADS / 32; ++w) S += red[w];
    const double norm = sqrt(S);
    float* dst = out + (size_t)i * out_ld;
    for (int c = threadIdx.x * 8; c < hidden; c += EMBED_POOL_THREADS * 8) {
        const uint4 v = *reinterpret_cast<const uint4*>(src + c);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            dst[c + 2 * j] = S > 0.0 ? (float)((double)bf16_lo(w[j]) / norm) : 0.f;
            dst[c + 2 * j + 1] = S > 0.0 ? (float)((double)bf16_hi(w[j]) / norm) : 0.f;
        }
    }
}

void launch_embed_pool(const __nv_bfloat16* xn, int ld, const int32_t* rows, int n, int hidden, float* out, int out_ld,
                       cudaStream_t st) {
    if (n <= 0) return;
    launch_pdl(embed_pool_kernel, dim3(n), dim3(EMBED_POOL_THREADS), 0, st, xn, ld, rows, hidden, out, out_ld);
}

void rr_trace_set_elementwise(unsigned long long* p) { rr_trace_set_local(p); }

}  // namespace rr
