// rr_api.cu — extern "C" surface of librr_b200.so for the kernel-level entry points
// (include/rr_b200.h §2, §3).  Router: rr_router.cu.  Engine: rr_engine.cu.
#include "rr_kernels.h"
#include <vector>

#include <string.h>

#define RR_API extern "C" __attribute__((visibility("default")))

#include <stdlib.h>

namespace rr {
int g_use_pdl = getenv("RR_NO_PDL") ? 0 : 1;
thread_local char g_last_cuda_error[256] = "";
void note_cuda_error(cudaError_t e) {
    if (e != cudaSuccess) {
        strncpy(g_last_cuda_error, cudaGetErrorString(e), sizeof(g_last_cuda_error) - 1);
    }
}
int check_last(void) {
    cudaError_t e = cudaGetLastError();
    note_cuda_error(e);
    return e == cudaSuccess ? RR_OK : RR_CUDA_ERROR;
}
}  // namespace rr

using namespace rr;

RR_API const char* rr_version(void) { return "rr_b200 0.1 (sm_90a)"; }

RR_API const char* rr_strerror(int rc) {
    switch (rc) {
        case RR_OK: return "ok";
        case RR_RATE_LIMITED: return "rate limited (429)";
        case RR_NO_GROUP: return "unknown model group";
        case RR_INTERNAL: return "internal error";
        case RR_INVALID_ARGUMENT: return "invalid argument";
        case RR_CUDA_ERROR: return "CUDA error";
        case RR_TIMEOUT: return "timeout";
        case RR_BACKEND_FAILED: return "backend failed";
        case RR_CANCELLED: return "cancelled";
    }
    return "unknown";
}

RR_API const char* rr_last_cuda_error(void) { return g_last_cuda_error; }

namespace rr {
void rr_trace_set_gemm(unsigned long long*);
void rr_trace_set_attn_decode(unsigned long long*);
void rr_trace_set_attn_tc(unsigned long long*);
void rr_trace_set_elementwise(unsigned long long*);
void rr_trace_set_gemm_detail(int);
void rr_trace_set_attn_decode_detail(int);
}
static unsigned long long* g_trace_dev = nullptr;
static int g_trace_cap = 0;
static int g_trace_detail_on = 0;

// Debug timeline: (kernel id, start ns, dependency-resolved ns, end ns) of CTA 0 of every library kernel (globaltimer).
RR_API int rr_debug_trace_start(int max_entries) {
    if (max_entries < 1) return RR_INVALID_ARGUMENT;
    if (g_trace_dev) cudaFree(g_trace_dev);
    const size_t n = 2 + 4 * (size_t)max_entries;
    if (cudaMalloc(&g_trace_dev, n * 8) != cudaSuccess) return RR_CUDA_ERROR;
    cudaMemset(g_trace_dev, 0, n * 8);
    unsigned long long cap = (unsigned long long)max_entries;
    cudaMemcpy(g_trace_dev + 1, &cap, 8, cudaMemcpyHostToDevice);
    g_trace_cap = max_entries;
    rr_trace_set_gemm(g_trace_dev); rr_trace_set_attn_decode(g_trace_dev);
    rr_trace_set_attn_tc(g_trace_dev);
    rr_trace_set_elementwise(g_trace_dev);
    return check_last();
}
// Stops tracing and copies up to max_entries (id, start, dep, end) records; returns the number recorded via *n.
RR_API int rr_debug_trace_stop(unsigned long long* out, int max_entries, int* n) {
    if (!g_trace_dev || !out || !n) return RR_INVALID_ARGUMENT;
    cudaDeviceSynchronize();
    rr_trace_set_gemm(nullptr); rr_trace_set_attn_decode(nullptr);
    rr_trace_set_attn_tc(nullptr);
    rr_trace_set_elementwise(nullptr);
    unsigned long long cnt = 0;
    cudaMemcpy(&cnt, g_trace_dev, 8, cudaMemcpyDeviceToHost);
    int m = (int)(cnt < (unsigned long long)g_trace_cap ? cnt : g_trace_cap);
    if (g_trace_detail_on) m = g_trace_cap;       // fixed-slot detail marks live at the end of the buffer; empty rows are zero
    if (m > max_entries) m = max_entries;
    cudaMemcpy(out, g_trace_dev + 2, (size_t)m * 32, cudaMemcpyDeviceToHost);
    *n = m;
    cudaFree(g_trace_dev);
    g_trace_dev = nullptr;
    return check_last();
}

// Per-phase marks of sample CTAs inside the fused MLP kernel, one plain decode projection and decode attention
// (tools/trace_mlp.py, trace_gemm.py, trace_attn.py); off by default.
RR_API int rr_debug_trace_detail(int on) {
    g_trace_detail_on = on ? 1 : 0;
    rr_trace_set_gemm_detail(on);      // 1: fused MLP kernel; 10 + s: the plain decode projection with split-K factor s
    rr_trace_set_attn_decode_detail(on ? 1 : 0);
    return check_last();
}

RR_API int rr_set_pdl(int enabled) {
    int old = g_use_pdl;
    g_use_pdl = enabled ? 1 : 0;
    return old;
}

// ---------------------------------------------------------------- tokenizer (K2)
// Byte-level: id 1 = BOS, then 3 + byte value (0/1/2 reserved: pad/bos/eos), folded into the
// model's vocabulary by modulo when vocab < 259.
RR_API int rr_count_tokens(const uint8_t* text, size_t n_bytes, int32_t* n_tokens) {
    if (!n_tokens || (!text && n_bytes)) return RR_INVALID_ARGUMENT;
    *n_tokens = (int32_t)n_bytes + 1;
    return RR_OK;
}

RR_API int rr_tokenize(const uint8_t* text, size_t n_bytes, int32_t vocab, int32_t* ids,
                       int32_t max_ids, int32_t* n_ids) {
    if (!ids || !n_ids || vocab < 4 || (!text && n_bytes)) return RR_INVALID_ARGUMENT;
    if ((size_t)max_ids < n_bytes + 1) return RR_INVALID_ARGUMENT;
    ids[0] = 1;
    for (size_t i = 0; i < n_bytes; ++i) {
        int32_t t = 3 + (int32_t)text[i];
        ids[i + 1] = t < vocab ? t : 3 + (t - 3) % (vocab - 3);
    }
    *n_ids = (int32_t)n_bytes + 1;
    return RR_OK;
}

// ---------------------------------------------------------------- kernels
RR_API int rr_gemm_bf16(const void* A, int rowsA, int ldA, const void* B, int rowsB, int ldB, int K,
                        void* out, int ldo, int ld_rows, int splits, int mode, int bn,
                        void* stream) {
    GemmPlan p;
    int rc = gemm_plan_init(&p, A, rowsA, ldA, B, rowsB, ldB, K, out, ldo, ld_rows, splits, mode, bn);
    if (rc != RR_OK) return rc;
    rc = gemm_launch(p, (cudaStream_t)stream);
    if (rc != RR_OK) note_cuda_error(cudaPeekAtLastError());
    return rc;
}

RR_API int rr_gemm_fp8w(const void* A, const float* scale, int rowsA, int ldA, const void* B, int rowsB, int ldB, int K,
                        void* out, int ldo, int ld_rows, int splits, int mode, int bn, void* stream) {
    GemmPlan p;
    int rc = gemm_plan_init_fp8w(&p, A, scale, rowsA, ldA, B, rowsB, ldB, K, out, ldo, ld_rows, splits, mode, bn);
    if (rc != RR_OK) return rc;
    rc = gemm_launch(p, (cudaStream_t)stream);
    if (rc != RR_OK) note_cuda_error(cudaPeekAtLastError());
    return rc;
}

// One decode projection as rr_engine_create plans it for max_batch = rows (decode_plan_init) and the decode step launches it.
RR_API int rr_op_decode_proj(const void* w, const float* w_scale, int rows_w, int K, const void* xn, int rows, void* out,
                             int mode, int lm_head, int* n_splits, void* stream) {
    if (!w || !xn || !out || !n_splits) return RR_INVALID_ARGUMENT;
    if (rows < 1 || rows > MAX_BATCH || rows_w < 1 || K < 8 || K % 8) return RR_INVALID_ARGUMENT;
    if (mode != OUT_TRANSPOSED_F32 && mode != OUT_TRANSPOSED_SILU) return RR_INVALID_ARGUMENT;
    if (lm_head && (mode != OUT_TRANSPOSED_F32 || w_scale)) return RR_INVALID_ARGUMENT;
    if (w_scale && !fp8_weight_ok(w, K)) return RR_INVALID_ARGUMENT;
    // the engine fuses SiLU * up into the gate/up epilogue only on batch tiles of 32 rows or more and whole 128-row
    // gate/up tiles (rr_engine_create: fuse_silu) ...
    if (mode == OUT_TRANSPOSED_SILU && (pick_bn(rows) < 32 || rows_w % 128)) return RR_INVALID_ARGUMENT;
    const int splits = lm_head ? 1 : pick_splits(rows_w, K);
    if (mode == OUT_TRANSPOSED_SILU && splits != 1) return RR_INVALID_ARGUMENT;      // ... and one gate/up plane
    GemmPlan p;
    int rc = decode_plan_init(&p, w, w_scale, rows_w, K, xn, rows, out, mode == OUT_TRANSPOSED_SILU ? rows_w / 2 : rows_w,
                              splits, mode);
    if (rc != RR_OK) return rc;
    rc = gemm_launch(p, (cudaStream_t)stream);
    if (rc != RR_OK) { note_cuda_error(cudaPeekAtLastError()); return rc; }
    *n_splits = p.splits;
    return check_last();
}

RR_API int rr_op_quantize_fp8_weight(const void* w, int rows, int K, int ld, void* q_out, float* scale_out, void* stream) {
    if (!w || !scale_out || rows < 1 || ld < K || ld % 8 || ((uintptr_t)w & 15) || !fp8_weight_ok(q_out, K))
        return RR_INVALID_ARGUMENT;
    cudaStream_t st = (cudaStream_t)stream;
    int* bad = nullptr;
    int h_bad = 0;
    cudaError_t e = cudaMallocAsync(&bad, sizeof(int), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(bad, 0, sizeof(int), st);
    int rc = RR_CUDA_ERROR;
    if (e == cudaSuccess)
        rc = launch_quantize_fp8((const __nv_bfloat16*)w, rows, K, ld, (uint8_t*)q_out, scale_out, bad, st);
    if (rc == RR_OK) e = cudaMemcpyAsync(&h_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, st);
    if (bad) cudaFreeAsync(bad, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { note_cuda_error(e); return RR_CUDA_ERROR; }
    if (rc != RR_OK) { note_cuda_error(cudaPeekAtLastError()); return rc; }
    return h_bad ? RR_INVALID_ARGUMENT : check_last();
}

RR_API int rr_op_dequantize_fp8_weight(const void* q, const float* scale, int rows, int K, void* out, int ld_out, void* stream) {
    if (!scale || !out || rows < 1 || !fp8_weight_ok(q, K) || ld_out < K || ld_out % 8 || ((uintptr_t)out & 15))
        return RR_INVALID_ARGUMENT;
    Fp8DequantJobs J;
    fp8_dequant_job(&J, q, scale, rows, K, (__nv_bfloat16*)out, ld_out);
    const int rc = launch_dequantize_fp8(J, (cudaStream_t)stream);
    if (rc != RR_OK) { note_cuda_error(cudaPeekAtLastError()); return rc; }
    return check_last();
}

// A layer's dequantize as the engine runs it before each prefill layer: up to four jobs in one launch (launch_dequant_layer).
RR_API int rr_op_dequantize_fp8_jobs(const void* const* q, const float* const* scale, const int32_t* rows, const int32_t* K,
                                     void* const* out, const int32_t* ld_out, int n_jobs, void* stream) {
    if (!q || !scale || !rows || !K || !out || !ld_out || n_jobs < 1 || n_jobs > 4) return RR_INVALID_ARGUMENT;
    Fp8DequantJobs J;
    for (int i = 0; i < n_jobs; ++i) {
        if (!scale[i] || !out[i] || rows[i] < 1 || !fp8_weight_ok(q[i], K[i]) || ld_out[i] < K[i] || ld_out[i] % 8 ||
            ((uintptr_t)out[i] & 15))
            return RR_INVALID_ARGUMENT;
        fp8_dequant_job(&J, q[i], scale[i], rows[i], K[i], (__nv_bfloat16*)out[i], ld_out[i]);
    }
    const int rc = launch_dequantize_fp8(J, (cudaStream_t)stream);
    if (rc != RR_OK) { note_cuda_error(cudaPeekAtLastError()); return rc; }
    return check_last();
}

static PartIn mk_part(const void* p, int is_bf16, int n_splits, long long split_stride, int ld) {
    PartIn r;
    r.ptr = p; r.is_bf16 = is_bf16; r.n_splits = n_splits < 1 ? 1 : n_splits;
    r.split_stride = split_stride; r.ld = ld;
    return r;
}

// The embedding gather as the engine runs it at the start of a step; ids are trusted, as slot indices are.
RR_API int rr_op_embed(const int32_t* ids, const void* table, float* x, int rows, int hidden,
                       const int32_t* row_active, void* stream) {
    if (!ids || !table || !x || rows < 1 || hidden < 8 || hidden % 8) return RR_INVALID_ARGUMENT;
    if (((uintptr_t)table & 15) || ((uintptr_t)x & 15)) return RR_INVALID_ARGUMENT;     // 16-byte loads and stores
    launch_embed(ids, (const __nv_bfloat16*)table, x, rows, hidden, row_active, (cudaStream_t)stream);
    return check_last();
}

// The embedding pool as the engine runs it over a prefill chunk's embedding rows; row indices are trusted, as ids are.
RR_API int rr_op_embed_pool(const void* xn, int ld, const int32_t* rows, int n, int hidden, float* out, int out_ld,
                            void* stream) {
    if (!xn || !out || n < 1 || n > 65535 || hidden < 8 || hidden > 16384 || hidden % 8 || ld < hidden || out_ld < hidden)
        return RR_INVALID_ARGUMENT;
    if (((uintptr_t)xn & 15) || ld % 8) return RR_INVALID_ARGUMENT;         // 16-byte loads of every row
    launch_embed_pool((const __nv_bfloat16*)xn, ld, rows, n, hidden, out, out_ld, (cudaStream_t)stream);
    return check_last();
}

RR_API int rr_op_add_rmsnorm(float* x, const void* part, int part_is_bf16, int n_splits,
                             long long split_stride, int part_ld, const void* w, void* xn, int rows,
                             int hidden, float eps, void* stream) {
    if (!x || !w || !xn || hidden % 4) return RR_INVALID_ARGUMENT;
    launch_add_rmsnorm(x, mk_part(part, part_is_bf16, n_splits, split_stride, part_ld),
                       (const __nv_bfloat16*)w, (__nv_bfloat16*)xn, rows, hidden, eps, (cudaStream_t)stream);
    return check_last();
}

RR_API int rr_op_silu_mul(const void* gu, int is_bf16, int n_splits, long long split_stride, int ld,
                          void* act, int rows, int inter, void* stream) {
    if (!gu || !act || inter % 4) return RR_INVALID_ARGUMENT;
    launch_silu_mul(mk_part(gu, is_bf16, n_splits, split_stride, ld), (__nv_bfloat16*)act, rows, inter,
                    (cudaStream_t)stream);
    return check_last();
}

RR_API int rr_op_rope_kv(const void* qkv, int is_bf16, int n_splits, long long split_stride, int ld,
                         void* q_out, void* k_cache, void* v_cache, const int32_t* slot,
                         const int32_t* pos, int rows, int n_heads, int n_kv_heads, int ctx_max,
                         float theta, void* stream) {
    if (!qkv || !q_out || !k_cache || !v_cache || !slot || !pos) return RR_INVALID_ARGUMENT;
    RopeArgs a;
    a.qkv = mk_part(qkv, is_bf16, n_splits, split_stride, ld);
    a.q_out = (__nv_bfloat16*)q_out; a.k_cache = (__nv_bfloat16*)k_cache; a.v_cache = (__nv_bfloat16*)v_cache;
    a.slot = slot; a.pos = pos; a.rows = rows; a.n_heads = n_heads; a.n_kv_heads = n_kv_heads;
    a.ctx_max = ctx_max; a.theta = theta; a.table = nullptr; a.head_dim = 128;
    launch_rope_kv(a, (cudaStream_t)stream);
    return check_last();
}

// The greedy pick as the engine runs it first in the logits tail.
RR_API int rr_op_argmax(const float* logits, int ld, int rows, int vocab, int32_t* out_tok,
                        float* out_val, const int32_t* row_active, int32_t* pos_inc, void* stream) {
    if (!logits || !out_tok || rows < 1 || vocab < 1 || vocab > ld || ld % 4) return RR_INVALID_ARGUMENT;
    if ((uintptr_t)logits & 15) return RR_INVALID_ARGUMENT;                              // 16-byte loads of each row
    launch_argmax(mk_part(logits, 0, 1, 0, ld), rows, vocab, out_tok, out_val, row_active, pos_inc,
                  (cudaStream_t)stream);
    return check_last();
}

// Log-softmax + top-k as the engine runs it after the argmax; the chunk workspace is stream-ordered scratch memory.
RR_API int rr_op_logprobs(const float* logits, int ld, int rows, int vocab, const int32_t* top_n, int max_top,
                          float* lp_out, int32_t* id_out, void* stream) {
    if (!logits || !top_n || !lp_out || !id_out) return RR_INVALID_ARGUMENT;
    if (rows < 1 || rows > 65535 || vocab < 1 || vocab > ld || ld % 4 || max_top < 1 || max_top > LP_MAX_TOP)
        return RR_INVALID_ARGUMENT;
    if (vocab > LP_MAX_CHUNKS * LP_CHUNK) return RR_INVALID_ARGUMENT;
    cudaStream_t st = (cudaStream_t)stream;
    void* ws = nullptr;
    cudaError_t e = cudaMallocAsync(&ws, logprobs_ws_bytes(rows, vocab), st);
    if (e != cudaSuccess) { note_cuda_error(e); return RR_CUDA_ERROR; }
    launch_logprobs(logits, ld, rows, vocab, top_n, max_top, ws, lp_out, id_out, st);
    cudaFreeAsync(ws, st);
    return check_last();
}

// Seeded temperature / top-p draw as the engine runs it after the argmax; the workspace is stream-ordered scratch memory.
RR_API int rr_op_sample(const float* logits, int ld, int rows, int vocab, const float* temperature, const float* top_p,
                        const uint64_t* seed, const int32_t* position, int32_t* out_tok, void* stream) {
    if (!logits || !temperature || !top_p || !seed || !position || !out_tok) return RR_INVALID_ARGUMENT;
    if (rows < 1 || rows > 65535 || vocab < 1 || vocab > ld || ld % 4 || vocab > LP_MAX_CHUNKS * LP_CHUNK)
        return RR_INVALID_ARGUMENT;
    cudaStream_t st = (cudaStream_t)stream;
    void* ws = nullptr;
    cudaError_t e = cudaMallocAsync(&ws, sample_ws_bytes(rows, vocab), st);
    if (e != cudaSuccess) { note_cuda_error(e); return RR_CUDA_ERROR; }
    launch_sample(logits, ld, rows, vocab, temperature, top_p, seed, position, out_tok, ws, st);
    cudaFreeAsync(ws, st);
    return check_last();
}

// Penalties and logit bias in place, as the engine applies them before the argmax.  hist_len and n_bias are device data:
// the kernel clamps them to [0, hist_ld] and [0, bias_ld] and skips ids outside [0, vocab).  The count workspace is
// stream-ordered scratch memory, zeroed here; the kernel leaves it zero.
RR_API int rr_op_logit_penalties(float* logits, int ld, int rows, int vocab, const int32_t* hist, int hist_ld,
                                 const int32_t* hist_len, const float* frequency_penalty, const float* presence_penalty,
                                 const int32_t* bias_ids, const float* bias_vals, int bias_ld, const int32_t* n_bias,
                                 void* stream) {
    if (!logits || !hist || !hist_len || !frequency_penalty || !presence_penalty || !bias_ids || !bias_vals || !n_bias)
        return RR_INVALID_ARGUMENT;
    if (rows < 1 || rows > 65535 || vocab < 1 || vocab > ld || ld % 4 || vocab > LP_MAX_CHUNKS * LP_CHUNK)
        return RR_INVALID_ARGUMENT;
    if (hist_ld < 0 || bias_ld < 0 || bias_ld > PEN_MAX_BIAS) return RR_INVALID_ARGUMENT;
    cudaStream_t st = (cudaStream_t)stream;
    void* ws = nullptr;
    const size_t ws_bytes = sizeof(int32_t) * (size_t)rows * vocab;
    cudaError_t e = cudaMallocAsync(&ws, ws_bytes, st);
    if (e != cudaSuccess) { note_cuda_error(e); return RR_CUDA_ERROR; }
    e = cudaMemsetAsync(ws, 0, ws_bytes, st);
    if (e != cudaSuccess) { cudaFreeAsync(ws, st); note_cuda_error(e); return RR_CUDA_ERROR; }
    PenaltyArgs a;
    a.freq = frequency_penalty; a.pres = presence_penalty; a.bias_ids = bias_ids; a.n_bias = n_bias; a.bias_vals = bias_vals;
    a.bias_ld = bias_ld; a.hist = const_cast<int32_t*>(hist); a.hist_ld = hist_ld; a.hist_len = hist_len;
    a.app_tok = nullptr; a.app_pos = nullptr; a.gen0 = nullptr;
    launch_logit_penalties(logits, ld, rows, vocab, a, (int32_t*)ws, st);
    cudaFreeAsync(ws, st);
    return check_last();
}

// Stop-sequence matching as the engine runs it at the end of the logits tail (StopArgs, rr_kernels.h), on caller buffers.
RR_API int rr_op_stop_match(int32_t* hist, int hist_ld, const int32_t* tok, const int32_t* position,
                            const int32_t* row_active, const int32_t* n_stop, const int32_t* gen0, const uint8_t* stop_len,
                            const uint8_t* stop_bytes, int32_t* cut_out, int32_t* hold_out, int rows, void* stream) {
    if (!hist || !tok || !position || !n_stop || !gen0 || !stop_len || !stop_bytes || !cut_out || !hold_out)
        return RR_INVALID_ARGUMENT;
    if (rows < 1 || rows > 65535 || hist_ld < 1 || ((uintptr_t)stop_bytes & 3)) return RR_INVALID_ARGUMENT;
    StopArgs a;
    a.n_stop = n_stop; a.gen0 = gen0; a.len = stop_len; a.bytes = stop_bytes; a.hist = hist; a.hist_ld = hist_ld;
    a.hist_row = nullptr; a.tok = tok; a.position = position; a.row_active = row_active; a.cut = cut_out; a.hold = hold_out;
    launch_stop_match(a, rows, (cudaStream_t)stream);
    return check_last();
}

// JSON mode as the engine runs it in the logits tail (rr_kernels.h, JsonState), on caller buffers.
RR_API int rr_op_json_mask(float* logits, int ld, int rows, int vocab, const int32_t* fmt, const int32_t* row_active,
                           const void* state, void* stream) {
    if (!logits || !fmt) return RR_INVALID_ARGUMENT;
    if (rows < 1 || rows > 65535 || vocab < 1 || vocab > ld || ld % 4 || vocab > LP_MAX_CHUNKS * LP_CHUNK)
        return RR_INVALID_ARGUMENT;
    launch_json_mask(logits, ld, rows, vocab, fmt, row_active, (const JsonState*)state, (cudaStream_t)stream);
    return check_last();
}

RR_API int rr_op_json_advance(int rows, const int32_t* fmt, const int32_t* row_active, const int32_t* tok,
                              const void* state_in, void* state_out, const int32_t* out_row, int32_t* done, void* stream) {
    if (!fmt || !tok || !state_out || !done || rows < 1 || rows > 65535) return RR_INVALID_ARGUMENT;
    launch_json_advance(rows, fmt, row_active, tok, (const JsonState*)state_in, (JsonState*)state_out, out_row, done,
                        (cudaStream_t)stream);
    return check_last();
}

RR_API int rr_op_decode_attn(const void* q,const void* k_cache, const void* v_cache, void* out,
                             const int32_t* slot, const int32_t* pos, int rows, int n_heads,
                             int n_kv_heads, int ctx_max, int n_slots, float scale, int kv_splits, void* stream) {
    if (!q || !k_cache || !v_cache || !out || !slot || !pos || n_slots < 1) return RR_INVALID_ARGUMENT;
    if (n_kv_heads <= 0 || n_heads % n_kv_heads) return RR_INVALID_ARGUMENT;
    const int G = n_heads / n_kv_heads;
    if (!(G == 1 || G == 2 || G == 4 || G == 8)) return RR_INVALID_ARGUMENT;
    DecodeAttnArgs a;
    a.q = (const __nv_bfloat16*)q; a.k_cache = (const __nv_bfloat16*)k_cache;
    a.v_cache = (const __nv_bfloat16*)v_cache; a.out = (__nv_bfloat16*)out; a.slot = slot; a.pos = pos;
    a.rows = rows; a.n_heads = n_heads; a.n_kv_heads = n_kv_heads; a.ctx_max = ctx_max; a.scale = scale;
    a.kv_splits = kv_splits < 1 ? 1 : kv_splits; a.ws = nullptr;
    a.fuse_rope = 0; a.qkv.ptr = nullptr; a.rope_table = nullptr; a.head_dim = 128;
    { int rcm = decode_attn_make_maps(&a, n_slots); if (rcm != RR_OK) return rcm; }
    float* ws = nullptr;
    if (a.kv_splits > 1) {
        cudaError_t e = cudaMallocAsync(&ws, decode_attn_ws_bytes(rows, n_heads, a.kv_splits), (cudaStream_t)stream);
        if (e != cudaSuccess) { note_cuda_error(e); return RR_CUDA_ERROR; }
        a.ws = ws;
    }
    launch_decode_attn(a, (cudaStream_t)stream);
    if (ws) cudaFreeAsync(ws, (cudaStream_t)stream);
    return check_last();
}

// Decode attention as the engine runs it (rr_engine_create): RoPE and the KV append fused in, q / k / v summed from the QKV
// GEMM's fp32 split-K planes, the engine's scale, kv-split rule and RoPE table; RR_ATTN_NO_TRIM is read per call.  The
// table and the split-KV workspace live in stream-ordered scratch memory.
// page_table == nullptr: the slot-contiguous cache of n_slots slots; else n_pages 64-token pages (kv_row).
static int decode_attn_qkv(const float* qkv, int n_splits, long long split_stride, int ld, void* k_cache, void* v_cache,
                           void* out, const int32_t* slot, const int32_t* pos, int rows, int n_heads, int n_kv_heads,
                           int head_dim, int ctx_max, int n_slots, float theta, int* kv_splits, const int32_t* page_table,
                           int pages_per_slot, int n_pages, int window, void* stream) {
    if (!qkv || !k_cache || !v_cache || !out || !slot || !pos || !kv_splits || window < 0) return RR_INVALID_ARGUMENT;
    if (rows < 1 || n_slots < 1 || n_splits < 1) return RR_INVALID_ARGUMENT;
    if (n_kv_heads <= 0 || n_heads % n_kv_heads) return RR_INVALID_ARGUMENT;
    const int G = n_heads / n_kv_heads;
    if (!(G == 1 || G == 2 || G == 4 || G == 8)) return RR_INVALID_ARGUMENT;
    if (head_dim < 64 || head_dim > 128 || head_dim % 16 || ctx_max < 64 || ctx_max % 64) return RR_INVALID_ARGUMENT;
    // the kernel reads the planes as float2
    if (ld < (n_heads + 2 * n_kv_heads) * head_dim || ld % 2 || split_stride % 2) return RR_INVALID_ARGUMENT;
    DecodeAttnArgs a;
    a.q = nullptr; a.k_cache = (const __nv_bfloat16*)k_cache; a.v_cache = (const __nv_bfloat16*)v_cache;
    a.out = (__nv_bfloat16*)out; a.slot = slot; a.pos = pos;
    a.rows = rows; a.n_heads = n_heads; a.n_kv_heads = n_kv_heads; a.ctx_max = ctx_max;
    a.scale = 1.0f / sqrtf((float)head_dim);
    a.kv_splits = pick_kv_splits(rows, n_kv_heads); a.ws = nullptr;
    a.fuse_rope = 1; a.qkv = mk_part(qkv, 0, n_splits, split_stride, ld); a.head_dim = head_dim;
    a.page_table = page_table; a.pages_per_slot = pages_per_slot; a.window = window;
    { int rcm = decode_attn_make_maps(&a, page_table ? n_pages : n_slots); if (rcm != RR_OK) return rcm; }
    cudaStream_t st = (cudaStream_t)stream;
    float2* table = nullptr;
    float* ws = nullptr;
    cudaError_t e = cudaMallocAsync(&table, (size_t)ctx_max * 64 * sizeof(float2), st);
    if (e == cudaSuccess && a.kv_splits > 1) e = cudaMallocAsync(&ws, decode_attn_ws_bytes(rows, n_heads, a.kv_splits), st);
    if (e == cudaSuccess) {
        launch_rope_table(table, ctx_max, theta, head_dim, st);
        a.rope_table = table; a.ws = ws;
        launch_decode_attn(a, st);
    } else {
        note_cuda_error(e);
    }
    if (table) cudaFreeAsync(table, st);
    if (ws) cudaFreeAsync(ws, st);
    if (e != cudaSuccess) return RR_CUDA_ERROR;
    *kv_splits = a.kv_splits;
    return check_last();
}

RR_API int rr_op_decode_attn_qkv(const float* qkv, int n_splits, long long split_stride, int ld, void* k_cache,
                                 void* v_cache, void* out, const int32_t* slot, const int32_t* pos, int rows, int n_heads,
                                 int n_kv_heads, int head_dim, int ctx_max, int n_slots, float theta, int* kv_splits,
                                 void* stream) {
    return decode_attn_qkv(qkv, n_splits, split_stride, ld, k_cache, v_cache, out, slot, pos, rows, n_heads, n_kv_heads,
                           head_dim, ctx_max, n_slots, theta, kv_splits, nullptr, 0, 0, 0, stream);
}

// The paged entry points' own checks, made before their counterpart's: a page table, at least one page per slot and in the
// pool, and ctx_max = KV_PAGE x pages_per_slot.
static bool paged_ok(const int32_t* page_table, int pages_per_slot, int n_pages, int ctx_max) {
    return page_table && pages_per_slot >= 1 && n_pages >= 1 && (long long)ctx_max == (long long)KV_PAGE * pages_per_slot;
}

RR_API int rr_op_decode_attn_qkv_window(const float* qkv, int n_splits, long long split_stride, int ld, void* k_cache,
                                        void* v_cache, void* out, const int32_t* slot, const int32_t* pos, int rows,
                                        int n_heads, int n_kv_heads, int head_dim, int ctx_max, int n_slots, float theta,
                                        int* kv_splits, const int32_t* page_table, int pages_per_slot, int n_pages,
                                        int window, void* stream) {
    if (!paged_ok(page_table, pages_per_slot, n_pages, ctx_max)) return RR_INVALID_ARGUMENT;
    return decode_attn_qkv(qkv, n_splits, split_stride, ld, k_cache, v_cache, out, slot, pos, rows, n_heads, n_kv_heads,
                           head_dim, ctx_max, n_slots, theta, kv_splits, page_table, pages_per_slot, n_pages, window, stream);
}

RR_API int rr_op_decode_attn_qkv_paged(const float* qkv, int n_splits, long long split_stride, int ld, void* k_cache,
                                       void* v_cache, void* out, const int32_t* slot, const int32_t* pos, int rows,
                                       int n_heads, int n_kv_heads, int head_dim, int ctx_max, int n_slots, float theta,
                                       int* kv_splits, const int32_t* page_table, int pages_per_slot, int n_pages,
                                       void* stream) {
    return rr_op_decode_attn_qkv_window(qkv, n_splits, split_stride, ld, k_cache, v_cache, out, slot, pos, rows, n_heads,
                                        n_kv_heads, head_dim, ctx_max, n_slots, theta, kv_splits, page_table, pages_per_slot,
                                        n_pages, 0, stream);
}

// Layer 0's RMSNorm of a prefill chunk in the deferred form, the only form run_prefill launches.
RR_API int rr_op_add_rmsnorm_pf(float* x, const void* w, void* xn, int rows, int hidden, float eps, float* rowss_out,
                                int n_part_out, void* stream) {
    if (!x || !w || !xn || !rowss_out) return RR_INVALID_ARGUMENT;
    if (rows < 1 || hidden < 64 || hidden % 64 || hidden > 8192 || n_part_out != pf_norm_parts(hidden)) return RR_INVALID_ARGUMENT;
    launch_add_rmsnorm_pf(x, (const __nv_bfloat16*)w, (__nv_bfloat16*)xn, rows, hidden, eps, (cudaStream_t)stream, rowss_out,
                          n_part_out);
    return check_last();
}

// The prefill QKV projection as run_prefill runs it: the plan is made for plan_rows rows and launched for T, the deferred
// norm scale comes from rowss, and RoPE + KV append run in the epilogue (head_dim 128) or in rope_kv_kernel from a bf16
// qkv matrix.  The RoPE table and that matrix live in stream-ordered scratch memory.
static int prefill_qkv(const void* xhat, const float* rowss, int plan_rows, int T, int hidden, const void* wqkv,
                       int n_heads, int n_kv_heads, int head_dim, int ctx_max, float theta, float eps, const int32_t* slot,
                       const int32_t* pos, void* q_out, void* k_cache, void* v_cache, int* fused,
                       const int32_t* page_table, int pages_per_slot, void* stream) {
    if (!xhat || !rowss || !wqkv || !slot || !pos || !q_out || !k_cache || !v_cache || !fused) return RR_INVALID_ARGUMENT;
    if (T < 1 || T > plan_rows || hidden < 64 || hidden % 64 || hidden > 8192) return RR_INVALID_ARGUMENT;
    if (n_heads < 1 || n_kv_heads < 1 || n_heads % n_kv_heads) return RR_INVALID_ARGUMENT;
    const int G = n_heads / n_kv_heads;
    if (!(G == 1 || G == 2 || G == 4 || G == 8)) return RR_INVALID_ARGUMENT;
    if (head_dim < 64 || head_dim > 128 || head_dim % 16 || ctx_max < 64 || ctx_max % 64) return RR_INVALID_ARGUMENT;
    const int nqkv = (n_heads + 2 * n_kv_heads) * head_dim;
    const bool fuse = pf_rope_fused(head_dim);
    GemmPlan p;
    int rc = gemm_plan_init(&p, xhat, plan_rows, hidden, wqkv, nqkv, hidden, hidden, nullptr, nqkv, 0, 1,
                            fuse ? OUT_ROWMAJOR_ROPE : OUT_ROWMAJOR_BF16, MAX_BN);
    if (rc != RR_OK) return rc;
    pf_norm_consumer(&p.rope, rowss, hidden, eps);
    p.rowsA = T;
    cudaStream_t st = (cudaStream_t)stream;
    float2* table = nullptr;
    __nv_bfloat16* qkv = nullptr;
    cudaError_t e = cudaMallocAsync(&table, (size_t)ctx_max * 64 * sizeof(float2), st);
    if (e == cudaSuccess && !fuse) e = cudaMallocAsync(&qkv, (size_t)plan_rows * nqkv * sizeof(__nv_bfloat16), st);
    rc = RR_CUDA_ERROR;
    if (e == cudaSuccess) {
        launch_rope_table(table, ctx_max, theta, head_dim, st);
        if (fuse) {
            RopeEpi& r = p.rope;
            r.q_out = (__nv_bfloat16*)q_out; r.k_cache = (__nv_bfloat16*)k_cache; r.v_cache = (__nv_bfloat16*)v_cache;
            r.slot = slot; r.pos = pos; r.table = table; r.n_heads = n_heads; r.n_kv_heads = n_kv_heads; r.ctx_max = ctx_max;
            r.page_table = page_table; r.pages_per_slot = pages_per_slot;
        } else {
            p.out = qkv;
        }
        rc = gemm_launch(p, st);
        if (rc == RR_OK && !fuse) {
            RopeArgs ra;
            ra.qkv = mk_part(qkv, 1, 1, 0, nqkv);
            ra.q_out = (__nv_bfloat16*)q_out; ra.k_cache = (__nv_bfloat16*)k_cache; ra.v_cache = (__nv_bfloat16*)v_cache;
            ra.slot = slot; ra.pos = pos; ra.rows = T; ra.n_heads = n_heads; ra.n_kv_heads = n_kv_heads; ra.ctx_max = ctx_max;
            ra.theta = theta; ra.table = table; ra.head_dim = head_dim;
            ra.page_table = page_table; ra.pages_per_slot = pages_per_slot;
            launch_rope_kv(ra, st);
        }
        if (rc != RR_OK) note_cuda_error(cudaPeekAtLastError());
    } else {
        note_cuda_error(e);
    }
    if (table) cudaFreeAsync(table, st);
    if (qkv) cudaFreeAsync(qkv, st);
    if (rc != RR_OK) return rc;
    *fused = fuse ? 1 : 0;
    return check_last();
}

RR_API int rr_op_prefill_qkv(const void* xhat, const float* rowss, int plan_rows, int T, int hidden, const void* wqkv,
                             int n_heads, int n_kv_heads, int head_dim, int ctx_max, float theta, float eps,
                             const int32_t* slot, const int32_t* pos, void* q_out, void* k_cache, void* v_cache, int* fused,
                             void* stream) {
    return prefill_qkv(xhat, rowss, plan_rows, T, hidden, wqkv, n_heads, n_kv_heads, head_dim, ctx_max, theta, eps, slot, pos,
                       q_out, k_cache, v_cache, fused, nullptr, 0, stream);
}

RR_API int rr_op_prefill_qkv_paged(const void* xhat, const float* rowss, int plan_rows, int T, int hidden, const void* wqkv,
                                   int n_heads, int n_kv_heads, int head_dim, int ctx_max, float theta, float eps,
                                   const int32_t* slot, const int32_t* pos, void* q_out, void* k_cache, void* v_cache,
                                   int* fused, const int32_t* page_table, int pages_per_slot, int n_pages, void* stream) {
    if (!paged_ok(page_table, pages_per_slot, n_pages, ctx_max)) return RR_INVALID_ARGUMENT;
    return prefill_qkv(xhat, rowss, plan_rows, T, hidden, wqkv, n_heads, n_kv_heads, head_dim, ctx_max, theta, eps, slot, pos,
                       q_out, k_cache, v_cache, fused, page_table, pages_per_slot, stream);
}

// The O, gate/up and down projections of a prefill chunk as run_prefill runs them: planned for plan_rows rows, launched
// for T, with the deferred-norm fields of the epilogue filled by the engine's helpers.
RR_API int rr_op_prefill_gemm(const void* A, int plan_rows, int T, int ldA, const void* W, int rowsW, int K, void* out,
                              int ldo, int mode, const float* rowss, int n_part, int hidden, float eps, const void* gamma,
                              void* xhat, float* rowss_out, int n_part_out, void* stream) {
    if (!A || !W || !out) return RR_INVALID_ARGUMENT;
    if (T < 1 || T > plan_rows || rowsW < 1) return RR_INVALID_ARGUMENT;
    if (mode != OUT_ROWMAJOR_BF16 && mode != OUT_ROWMAJOR_SILU && mode != OUT_ROWMAJOR_RESID && mode != OUT_ROWMAJOR_F32)
        return RR_INVALID_ARGUMENT;
    if (n_part < 0 || (n_part > 0 && (!rowss || mode == OUT_ROWMAJOR_RESID || hidden < 1 || n_part != pf_norm_parts(hidden))))
        return RR_INVALID_ARGUMENT;
    if (xhat && (mode != OUT_ROWMAJOR_RESID || !gamma || !rowss_out || n_part_out != pf_norm_parts(rowsW)))
        return RR_INVALID_ARGUMENT;
    GemmPlan p;
    const int rc = gemm_plan_init(&p, A, plan_rows, ldA, W, rowsW, K, K, out, ldo, 0, 1, mode, MAX_BN);
    if (rc != RR_OK) return rc;
    if (n_part > 0) pf_norm_consumer(&p.rope, rowss, hidden, eps);
    if (xhat) pf_norm_producer(&p.rope, (const __nv_bfloat16*)gamma, (__nv_bfloat16*)xhat, rowss_out, rowsW);
    p.rowsA = T;
    if (gemm_launch(p, (cudaStream_t)stream) != RR_OK) {
        note_cuda_error(cudaPeekAtLastError());
        return RR_CUDA_ERROR;
    }
    return check_last();
}

// The fused decode MLP as the engine runs it (rr_engine_create): tile width, K slices, grid and schedule come from the same
// helpers and environment switches; the schedule and the dependency counters live in stream-ordered scratch memory.
static int decode_mlp(const void* wgu_il, const float* sc_gu, const void* wdown, const float* sc_down, const void* xn, int rows,
                      int hidden, int inter, void* act, void* planes, int ld_rows, int* n_slices, int* slice_kb, void* stream) {
    if (!wgu_il || !wdown || !xn || !act || !planes || !n_slices || !slice_kb) return RR_INVALID_ARGUMENT;
    // the engine fuses the MLP for batches of 17..MAX_BN rows (tile width >= 32, one batch tile)
    if (rows <= 16 || rows > MAX_BN || ld_rows < rows) return RR_INVALID_ARGUMENT;
    if (hidden < 64 || hidden % 64 || hidden > 8192 || inter < 64 || inter % 64) return RR_INVALID_ARGUMENT;
    int skb = 0;
    const int ns = mlp_slices(inter, &skb);
    const int grid = num_sms();
    const int dyn = getenv("RR_MLP_STATIC") ? 0 : 1;
    std::vector<MlpItem> sched;
    const int max_items = mlp_schedule(grid, inter, hidden, skb, &sched, dyn);
    cudaStream_t st = (cudaStream_t)stream;
    MlpItem* items = nullptr;
    unsigned* ready = nullptr;
    cudaError_t e = cudaMallocAsync(&items, sched.size() * sizeof(MlpItem), st);
    if (e == cudaSuccess) e = cudaMallocAsync(&ready, (size_t)(ns + 1) * sizeof(unsigned), st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(items, sched.data(), sched.size() * sizeof(MlpItem), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(ready, 0, (size_t)(ns + 1) * sizeof(unsigned), st);
    int rc = RR_CUDA_ERROR;
    if (e == cudaSuccess) {
        MlpPlan p;
        rc = mlp_plan_init(&p, wgu_il, wdown, inter, hidden, xn, rows, act, planes, ld_rows, pick_bn(rows), items, max_items,
                           grid, ready, skb, dyn, sc_gu, sc_down);
        if (rc == RR_OK) rc = mlp_launch(p, st);
    }
    if (e != cudaSuccess) note_cuda_error(e);
    else if (rc != RR_OK) note_cuda_error(cudaPeekAtLastError());
    if (items) cudaFreeAsync(items, st);
    if (ready) cudaFreeAsync(ready, st);
    if (rc != RR_OK) return rc;
    *n_slices = ns;
    *slice_kb = skb;
    return check_last();
}

RR_API int rr_op_decode_mlp(const void* wgu_il, const void* wdown, const void* xn, int rows, int hidden, int inter,
                            void* act, void* planes, int ld_rows, int* n_slices, int* slice_kb, void* stream) {
    return decode_mlp(wgu_il, nullptr, wdown, nullptr, xn, rows, hidden, inter, act, planes, ld_rows, n_slices, slice_kb, stream);
}

RR_API int rr_op_decode_mlp_fp8(const void* wgu_il, const float* wgu_scale, const void* wdown, const float* wdown_scale,
                                const void* xn, int rows, int hidden, int inter, void* act, void* planes, int ld_rows,
                                int* n_slices, int* slice_kb, void* stream) {
    if (!wgu_scale || !wdown_scale || !fp8_weight_ok(wgu_il, hidden) || !fp8_weight_ok(wdown, inter)) return RR_INVALID_ARGUMENT;
    return decode_mlp(wgu_il, wgu_scale, wdown, wdown_scale, xn, rows, hidden, inter, act, planes, ld_rows, n_slices,
                      slice_kb, stream);
}

RR_API int rr_debug_mlp_schedule(int grid, int inter, int hidden, int slice_kb, int32_t* items_out, int capacity,
                                 int* max_items) {
    if (grid < 1 || inter < 64 || inter % 64 || hidden < 8 || slice_kb < 1 || !max_items) return RR_INVALID_ARGUMENT;
    std::vector<MlpItem> items;
    *max_items = mlp_schedule(grid, inter, hidden, slice_kb, &items);
    if (!items_out || (size_t)capacity < items.size()) return RR_INVALID_ARGUMENT;
    static_assert(sizeof(MlpItem) == 4 * sizeof(int32_t), "MlpItem layout");
    memcpy(items_out, items.data(), items.size() * sizeof(MlpItem));
    return RR_OK;
}

RR_API int rr_op_prefill_attn(const void* q, const void* k_cache, const void* v_cache, void* out,
                              const int32_t* seq_start, const int32_t* seq_slot, int n_seqs,
                              int max_len, int n_heads, int n_kv_heads, int ctx_max, float scale,
                              void* stream) {
    if (!q || !k_cache || !v_cache || !out || !seq_start || !seq_slot) return RR_INVALID_ARGUMENT;
    if (n_kv_heads <= 0 || n_heads % n_kv_heads) return RR_INVALID_ARGUMENT;
    PrefillAttnArgs a;
    a.q = (const __nv_bfloat16*)q; a.k_cache = (const __nv_bfloat16*)k_cache;
    a.v_cache = (const __nv_bfloat16*)v_cache; a.out = (__nv_bfloat16*)out; a.seq_start = seq_start;
    a.seq_slot = seq_slot; a.n_seqs = n_seqs; a.max_len = max_len; a.n_heads = n_heads;
    a.n_kv_heads = n_kv_heads; a.ctx_max = ctx_max; a.scale = scale; a.head_dim = 128;
    if (n_seqs > 0) {
        // the TMA maps need the extents of q and of the caches, which this entry point
        // does not take -- read them back from the caller's index arrays (standalone op, not the engine path).
        std::vector<int32_t> h(n_seqs + 1);
        cudaError_t e = cudaMemcpyAsync(h.data(), seq_slot, sizeof(int32_t) * n_seqs, cudaMemcpyDeviceToHost, (cudaStream_t)stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(&h[n_seqs], seq_start + n_seqs, sizeof(int32_t), cudaMemcpyDeviceToHost, (cudaStream_t)stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize((cudaStream_t)stream);
        if (e != cudaSuccess) { note_cuda_error(e); return RR_CUDA_ERROR; }
        int max_slot = 0;
        for (int i = 0; i < n_seqs; ++i) max_slot = h[i] > max_slot ? h[i] : max_slot;
        (void)prefill_attn_make_maps(&a, h[n_seqs], (long long)(max_slot + 1) * n_kv_heads * ctx_max);
    }
    const int rcl = launch_prefill_attn(a, (cudaStream_t)stream);
    if (rcl != RR_OK) return rcl;
    return check_last();
}

// Prefill attention with a cached prefix per sequence (seq_pos0): the engine's launch, through the engine's helpers
// (pf_attn_layer, pf_attn_chunk).  Like rr_op_prefill_attn, the TMA maps need the extents of the caches, and q_rows = 0
// those of q (T rows), read back from the caller's index arrays; the positions are checked against ctx_max on the way.
// scale null: the engine's, 1 / sqrt(head_dim).
static int prefill_attn_cached(const void* q, const void* k_cache, const void* v_cache, void* out, const int32_t* seq_start,
                               const int32_t* seq_slot, const int32_t* seq_pos0, int n_seqs, int max_len, int n_heads,
                               int n_kv_heads, int ctx_max, const float* scale, int head_dim, int q_rows,
                               const int32_t* page_table, int pages_per_slot, int n_pages, int window, void* stream) {
    if (!q || !k_cache || !v_cache || !out || !seq_start || !seq_slot || !seq_pos0 || window < 0) return RR_INVALID_ARGUMENT;
    if (n_seqs < 1 || max_len < 1 || n_heads < 1 || n_kv_heads < 1 || n_heads % n_kv_heads) return RR_INVALID_ARGUMENT;
    if (ctx_max < 64 || ctx_max % 64 || q_rows < 0) return RR_INVALID_ARGUMENT;
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<int32_t> h(3 * (size_t)n_seqs + 1);         // seq_start[n + 1] | seq_slot[n] | seq_pos0[n]
    cudaError_t e = cudaMemcpyAsync(h.data(), seq_start, sizeof(int32_t) * (n_seqs + 1), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&h[n_seqs + 1], seq_slot, sizeof(int32_t) * n_seqs, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&h[2 * n_seqs + 1], seq_pos0, sizeof(int32_t) * n_seqs, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { note_cuda_error(e); return RR_CUDA_ERROR; }
    int max_slot = 0;
    for (int i = 0; i < n_seqs; ++i) {
        const int len = h[i + 1] - h[i], slot = h[n_seqs + 1 + i], p0 = h[2 * n_seqs + 1 + i];
        if (len < 0 || len > max_len || slot < 0 || p0 < 0 || p0 + len > ctx_max) return RR_INVALID_ARGUMENT;
        max_slot = slot > max_slot ? slot : max_slot;
    }
    if (q_rows > 0 && q_rows < h[n_seqs]) return RR_INVALID_ARGUMENT;
    PrefillAttnArgs a;
    (void)pf_attn_layer(&a, (const __nv_bfloat16*)q, (const __nv_bfloat16*)k_cache, (const __nv_bfloat16*)v_cache, n_heads,
                        n_kv_heads, head_dim, ctx_max, page_table, pages_per_slot, page_table ? n_pages : max_slot + 1,
                        window, q_rows > 0 ? q_rows : h[n_seqs]);
    if (scale) a.scale = *scale;
    pf_attn_chunk(&a, (__nv_bfloat16*)out, seq_start, seq_slot, seq_pos0, n_seqs, max_len);
    const int rcl = launch_prefill_attn(a, st);
    if (rcl != RR_OK) return rcl;
    return check_last();
}

RR_API int rr_op_prefill_attn_cached(const void* q, const void* k_cache, const void* v_cache, void* out,
                                     const int32_t* seq_start, const int32_t* seq_slot, const int32_t* seq_pos0, int n_seqs,
                                     int max_len, int n_heads, int n_kv_heads, int ctx_max, float scale, void* stream) {
    return prefill_attn_cached(q, k_cache, v_cache, out, seq_start, seq_slot, seq_pos0, n_seqs, max_len, n_heads, n_kv_heads,
                               ctx_max, &scale, 128, 0, nullptr, 0, 0, 0, stream);
}

RR_API int rr_op_prefill_attn_window(const void* q, const void* k_cache, const void* v_cache, void* out,
                                     const int32_t* seq_start, const int32_t* seq_slot, const int32_t* seq_pos0, int n_seqs,
                                     int max_len, int n_heads, int n_kv_heads, int ctx_max, float scale,
                                     const int32_t* page_table, int pages_per_slot, int n_pages, int window, void* stream) {
    if (!paged_ok(page_table, pages_per_slot, n_pages, ctx_max)) return RR_INVALID_ARGUMENT;
    return prefill_attn_cached(q, k_cache, v_cache, out, seq_start, seq_slot, seq_pos0, n_seqs, max_len, n_heads, n_kv_heads,
                               ctx_max, &scale, 128, 0, page_table, pages_per_slot, n_pages, window, stream);
}

// Prefill attention exactly as run_prefill launches it: the true head dim, its compact output and the engine's scale, the
// page table and window, q mapped over q_rows rows.  Refuses whatever rr_engine_create would not build.
RR_API int rr_op_prefill_attn_hd(const void* q, const void* k_cache, const void* v_cache, void* out, const int32_t* seq_start,
                                 const int32_t* seq_slot, const int32_t* seq_pos0, int n_seqs, int max_len, int n_heads,
                                 int n_kv_heads, int head_dim, int ctx_max, const int32_t* page_table, int pages_per_slot,
                                 int n_pages, int window, int q_rows, void* stream) {
    if (!paged_ok(page_table, pages_per_slot, n_pages, ctx_max)) return RR_INVALID_ARGUMENT;
    if (head_dim < 64 || head_dim > 128 || head_dim % 16) return RR_INVALID_ARGUMENT;
    if (n_kv_heads < 1 || n_heads < 1 || n_heads % n_kv_heads) return RR_INVALID_ARGUMENT;
    const int G = n_heads / n_kv_heads;
    if (!(G == 1 || G == 2 || G == 4 || G == 8)) return RR_INVALID_ARGUMENT;
    if (max_len < 1 || q_rows < max_len) return RR_INVALID_ARGUMENT;     // q_rows >= T >= max_len; T is checked on read-back
    return prefill_attn_cached(q, k_cache, v_cache, out, seq_start, seq_slot, seq_pos0, n_seqs, max_len, n_heads, n_kv_heads,
                               ctx_max, nullptr, head_dim, q_rows, page_table, pages_per_slot, n_pages, window, stream);
}

RR_API int rr_op_prefill_attn_cached_paged(const void* q, const void* k_cache, const void* v_cache, void* out,
                                           const int32_t* seq_start, const int32_t* seq_slot, const int32_t* seq_pos0,
                                           int n_seqs, int max_len, int n_heads, int n_kv_heads, int ctx_max, float scale,
                                           const int32_t* page_table, int pages_per_slot, int n_pages, void* stream) {
    return rr_op_prefill_attn_window(q, k_cache, v_cache, out, seq_start, seq_slot, seq_pos0, n_seqs, max_len, n_heads,
                                     n_kv_heads, ctx_max, scale, page_table, pages_per_slot, n_pages, 0, stream);
}

// Prefix copy between KV slots as the engine runs it at the start of a prefill chunk.  The lists are host arrays, checked
// before the device is touched.
static int kv_copy_prefix(void* k_cache, void* v_cache, int n_layers, int n_slots, int n_kv_heads, int ctx_max,
                          const int32_t* src, const int32_t* dst, const int32_t* n_tok, int n_copies,
                          const int32_t* page_table, int pages_per_slot, int n_pages, void* stream) {
    if (!k_cache || !v_cache || !src || !dst || !n_tok) return RR_INVALID_ARGUMENT;
    if (n_layers < 1 || n_slots < 1 || n_kv_heads < 1 || ctx_max < 1 || n_copies < 1 || n_copies > KV_COPY_MAX)
        return RR_INVALID_ARGUMENT;
    KvCopyList c;
    c.count = n_copies;
    for (int i = 0; i < n_copies; ++i) { c.src[i] = src[i]; c.dst[i] = dst[i]; c.n[i] = n_tok[i]; }
    if (kv_copy_check(c, n_slots, ctx_max) != RR_OK) return RR_INVALID_ARGUMENT;
    const long long layer_rows = page_table ? (long long)n_pages * n_kv_heads * KV_PAGE : (long long)n_slots * n_kv_heads * ctx_max;
    if (launch_kv_copy((__nv_bfloat16*)k_cache, (__nv_bfloat16*)v_cache, n_layers, layer_rows, n_kv_heads, ctx_max, page_table,
                       pages_per_slot, c, (cudaStream_t)stream) != RR_OK)
        note_cuda_error(cudaPeekAtLastError());
    return check_last();
}

RR_API int rr_op_kv_copy_prefix(void* k_cache, void* v_cache, int n_layers, int n_slots, int n_kv_heads, int ctx_max,
                                const int32_t* src, const int32_t* dst, const int32_t* n_tok, int n_copies, void* stream) {
    return kv_copy_prefix(k_cache, v_cache, n_layers, n_slots, n_kv_heads, ctx_max, src, dst, n_tok, n_copies, nullptr, 0, 0,
                          stream);
}

RR_API int rr_op_kv_copy_prefix_paged(void* k_cache, void* v_cache, int n_layers, int n_slots, int n_kv_heads, int ctx_max,
                                      const int32_t* src, const int32_t* dst, const int32_t* n_tok, int n_copies,
                                      const int32_t* page_table, int pages_per_slot, int n_pages, void* stream) {
    if (!paged_ok(page_table, pages_per_slot, n_pages, ctx_max)) return RR_INVALID_ARGUMENT;
    return kv_copy_prefix(k_cache, v_cache, n_layers, n_slots, n_kv_heads, ctx_max, src, dst, n_tok, n_copies, page_table,
                          pages_per_slot, n_pages, stream);
}

// The hand-off of a prefill chunk to decode, as run_prefill launches it; row, slot and index arrays are trusted, as slot
// indices are.
RR_API int rr_op_gather_last(const void* attn, const float* x, const int32_t* last, int n_rows, int nq, int hidden,
                             void* attn_out, float* x_out, void* stream) {
    if (!attn || !x || !last || !attn_out || !x_out) return RR_INVALID_ARGUMENT;
    if (n_rows < 1 || nq < 8 || nq % 8 || hidden < 4 || hidden % 4) return RR_INVALID_ARGUMENT;
    if ((((uintptr_t)attn | (uintptr_t)x | (uintptr_t)attn_out | (uintptr_t)x_out) & 15)) return RR_INVALID_ARGUMENT;
    launch_gather_last((const __nv_bfloat16*)attn, x, last, n_rows, nq, hidden, (__nv_bfloat16*)attn_out, x_out,
                       (cudaStream_t)stream);
    return check_last();
}

RR_API int rr_op_activate_rows(const int32_t* seq_slot, const int32_t* first_tok, const int32_t* tok_pos, const int32_t* last,
                               int n, int32_t* d_tok, int32_t* d_pos, int32_t* d_slot, void* stream) {
    if (!seq_slot || !first_tok || !tok_pos || !last || !d_tok || !d_pos || !d_slot || n < 1) return RR_INVALID_ARGUMENT;
    launch_activate_rows(seq_slot, first_tok, tok_pos, last, n, d_tok, d_pos, d_slot, (cudaStream_t)stream);
    return check_last();
}
