/* rr_b200.h — public C-ABI of librr_b200.so, the GPU-native (H100, sm_90a) replacement for the request-router
 * hot path of aws-samples/sample-resilient-llm-inference.
 *
 * The reference has NO native/FFI boundary: its hot path is `litellm.Router` (un-vendored
 * dependency, reference pyproject.toml:8) configured by reference config/config.yaml:35-108,
 * launched by reference bin/start-gateway.sh:54 and called over HTTP from
 * reference src/demo_load_balancing.py:106-110, src/demo_fallback.py:143-147 and
 * src/demo_quota_isolation.py:52-56; tokens are produced by the remote bedrock:InvokeModel call
 * (reference iam/policy.json:8, src/demo_cris.py:233-238).  Every entry point below names the
 * reference interface it replaces.  INTEGRATION.md shows the ctypes binding a maintainer of the
 * reference would add.
 *
 * Conventions: plain C types only; integer return codes (no exceptions cross the ABI);
 * caller-owned buffers; `stream` arguments are cudaStream_t passed as void* (NULL = legacy
 * default stream).  All functions return RR_OK (0) on success.
 */
#ifndef RR_B200_H
#define RR_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * Return codes.  RR_RATE_LIMITED is what the Python host maps to HTTP 429 / RateLimitError
 * (reference src/demo_quota_isolation.py:80, src/demo_fallback.py:184). */
enum {
    RR_OK = 0,
    RR_RATE_LIMITED = 1,      /* no deployment admitted the request (rpm/tpm/cooldown) -> 429 */
    RR_NO_GROUP = 2,          /* unknown model group -> 400 */
    RR_INTERNAL = 3,          /* -> 500 */
    RR_INVALID_ARGUMENT = 4,
    RR_CUDA_ERROR = 5,
    RR_TIMEOUT = 6,
    RR_BACKEND_FAILED = 7,    /* injected/real backend failure with no fallback left -> 500 */
    RR_CANCELLED = 8          /* the request was abandoned by its owner (rr_engine_cancel / rr_gateway_cancel) */
};

const char* rr_version(void);
const char* rr_strerror(int rc);
/* Last CUDA error string seen by the library on this thread (diagnostics). */
const char* rr_last_cuda_error(void);
/* Programmatic dependent launch between the library's kernels (default on; env RR_NO_PDL=1 turns it
 * off).  Returns the previous setting.  Must not change between capture and replay of an engine graph. */
int rr_set_pdl(int enabled);
/* Debug timeline: CTA 0 of every library kernel records (kernel id, start ns, ns when griddepcontrol.wait
 * returned, end ns) with %globaltimer.  start allocates a device buffer; stop copies `*n` records
 * (4 x uint64 each) to `out`. */
int rr_debug_trace_start(int max_entries);
int rr_debug_trace_stop(unsigned long long* out, int max_entries, int* n);
/* on != 0: sample CTAs of the fused decode MLP kernel, of decode attention and of one plain decode projection also record
 * per-phase marks (kernel ids 50 +, 80 +, 100 +) into fixed slots at the end of the buffer. */
int rr_debug_trace_detail(int on);
/* Host-side work schedule of the fused decode MLP kernel (gate/up + down GEMMs in one launch, DESIGN.md section 3), for
 * inspection and tests; no device is touched.  items_out receives grid * (*max_items) entries of 4 x int32
 * {tile | phase << 16 (phase 0 gate/up, 1 down; -1 = end of the CTA's list), kb0, kb1, slice}, CTA-major;
 * returns RR_INVALID_ARGUMENT when `capacity` (in entries) is too small (*max_items is still set). */
int rr_debug_mlp_schedule(int grid, int inter, int hidden, int slice_kb, int32_t* items_out, int capacity,
                          int* max_items);

/* ================================================================================================
 * 1. Router: admission + rpm/tpm bucket debit + backend pick + cooldown + fallback chain (K1).
 *    Replaces litellm.Router as configured by reference config/config.yaml:35-108
 *    (model_list[].{model_name,litellm_params,rpm,tpm}; router_settings.{routing_strategy,
 *    enable_pre_call_checks,allowed_fails,cooldown_time,fallbacks}).
 *    State lives in HBM; one kernel launch processes an ordered trace of events with the same
 *    result as processing them one at a time (serialised-trace semantics, DESIGN.md §router). */

enum {                       /* router_settings.routing_strategy (reference config.yaml:101) */
    RR_STRATEGY_SIMPLE_SHUFFLE = 0,
    RR_STRATEGY_LEAST_BUSY = 1,
    /* client-side distribution strategies of reference src/demo_account_sharding.py:335-343: */
    RR_STRATEGY_ROUND_ROBIN = 2,  /* req_id % n */
    RR_STRATEGY_SPLIT = 3,        /* first share of the burst to backend 0, next to backend 1, ... (req_id < N / 2) */
    RR_STRATEGY_RANDOM = 4,       /* random.choice, weights ignored */
    /* litellm's latency-based-routing: random.choice among the eligible deployments whose mean latency per output token
     * is within (1 + buffer) of the lowest; latency samples arrive on DONE / FAIL events (rr_event.chain_start) */
    RR_STRATEGY_LATENCY_BASED = 5
};

/* RR_EV_BURST(target = group, tokens = N) declares the size of the next burst for RR_STRATEGY_SPLIT. */
enum { RR_EV_ADMIT = 0, RR_EV_DONE = 1, RR_EV_FAIL = 2, RR_EV_BURST = 3 };

typedef struct rr_deployment_desc {
    int32_t group;           /* index of model_name (reference config.yaml:36,44,...) */
    int32_t rpm;             /* requests / minute, <0 = unlimited (config.yaml:41) */
    int32_t tpm;             /* tokens / minute, <0 = unlimited (config.yaml:42) */
    int32_t weight;          /* simple-shuffle weight, <0 = unset */
    int32_t replica;         /* GPU / engine index that serves this deployment */
    int32_t reserved;
} rr_deployment_desc;

typedef struct rr_router_settings {
    int32_t strategy;               /* RR_STRATEGY_* */
    int32_t enable_pre_call_checks; /* config.yaml:102 */
    int32_t allowed_fails;          /* config.yaml:103 */
    int32_t cooldown_ms;            /* config.yaml:104 (seconds * 1000) */
    int32_t weight_by;              /* 0 = uniform, 1 = weight, 2 = rpm, 3 = tpm (simple-shuffle) */
    /* RR_STRATEGY_LATENCY_BASED (router_settings.routing_strategy_args); ignored by the other strategies: */
    int32_t latency_list_size;      /* max_latency_list_size: samples kept per deployment, 1..32 (0 = 10) */
    int32_t latency_buffer_ppm;     /* lowest_latency_buffer in millionths, >= 0 (0.5 -> 500000) */
    int32_t latency_ttl_ms;         /* ttl: a model group's samples are dropped this long after its last write (0 = 1 h) */
} rr_router_settings;

typedef struct rr_event {
    int32_t type;            /* RR_EV_* */
    int32_t target;          /* ADMIT: group index; DONE/FAIL: deployment index */
    int32_t tokens;          /* ADMIT: prompt tokens; DONE: completion tokens */
    int32_t chain_start;     /* ADMIT: 0 = try the group itself first, k = start at k-th fallback;
                                DONE: measured request latency in microseconds (<= 0: no sample);
                                FAIL: 1 = the request timed out (penalty sample), 0 = any other failure.
                                Only RR_STRATEGY_LATENCY_BASED reads it on DONE / FAIL. */
    int64_t now_ms;          /* injectable clock, milliseconds */
} rr_event;

typedef struct rr_decision {
    int32_t status;          /* RR_OK / RR_RATE_LIMITED / RR_NO_GROUP */
    int32_t deployment;      /* picked deployment, -1 if none */
    int32_t served_group;    /* group that served (differs from target when fell back) */
    int32_t chain_pos;       /* 0 = primary, k = k-th fallback */
} rr_decision;

typedef struct rr_deployment_state {
    int64_t window;          /* minute index of the rpm/tpm window */
    int32_t req_count;
    int32_t tok_count;
    int64_t fail_window;
    int32_t fail_count;
    int32_t inflight;
    int64_t cooldown_until_ms;
    int64_t total_admitted;
} rr_deployment_state;

typedef struct rr_router rr_router;

/* fallback chains in CSR form: group g falls back to fb_groups[fb_offsets[g] .. fb_offsets[g+1])
 * (reference config.yaml:105-108). */
int rr_router_create(const rr_deployment_desc* deployments, int n_deployments, int n_groups,
                     const int32_t* fb_offsets, const int32_t* fb_groups,
                     const rr_router_settings* settings, uint64_t seed, int device,
                     rr_router** out);
void rr_router_destroy(rr_router* r);
/* Host buffers: copies events H2D, runs the admission kernel, copies decisions D2H. Thread-safe. */
int rr_router_process(rr_router* r, const rr_event* events, int n_events, rr_decision* decisions);
/* Device buffers already resident in HBM; asynchronous on `stream`. */
int rr_router_process_device(rr_router* r, const rr_event* d_events, int n_events,
                             rr_decision* d_decisions, void* stream);
int rr_router_snapshot(rr_router* r, rr_deployment_state* out /* [n_deployments] */);
/* RR_STRATEGY_LATENCY_BASED state as stored (a TTL expiry is applied at the next write or pick of the group):
 * per deployment the mean of its latency samples in microseconds per output token (0.0 without samples) and the
 * sample count.  All zeros for the other strategies. */
int rr_router_latency_snapshot(rr_router* r, double* mean_out /* [n_deployments] */,
                               int32_t* n_samples_out /* [n_deployments] */);
/* Re-seed the MT19937 stream exactly like CPython random.seed(int). */
int rr_router_seed(rr_router* r, uint64_t seed);
/* Host-only: the MT19937 state (624 words + index) CPython's random.seed(seed) produces. */
int rr_mt_seed_state(uint64_t seed, uint32_t* out625);

/* ================================================================================================
 * 2. Prompt token count (K2).  Replaces litellm.token_counter as used for tpm accounting
 *    (no call site in the reference tree; tpm values at reference config.yaml:42).
 *    Counts tokens of the library's byte-level tokenizer: n_tokens = n_utf8_bytes + 1 (BOS).
 *    rr_count_tokens / rr_tokenize are the host forms (one message); the request path uses the batch kernel below. */
int rr_count_tokens(const uint8_t* text, size_t n_bytes, int32_t* n_tokens);
int rr_tokenize(const uint8_t* text, size_t n_bytes, int32_t vocab, int32_t* ids, int32_t max_ids,
                int32_t* n_ids);
/* The same tokenizer as a CUDA kernel over a batch of messages (csrc/rr_tokenizer.cu): n_texts messages back to back in
 * `text`, text_off[n_texts + 1] byte offsets.  counts[i] = tokens of message i (what an ADMIT event carries into the tpm
 * check); ids (optional) = the packed token ids, message i at ids_off[i] = text_off[i] - text_off[0] + i.
 * rr_tokenize_batch: host buffers (H2D copy, kernel, D2H copies inside; thread-safe).
 * rr_tokenize_batch_device: device buffers, asynchronous on `stream`; max_text_bytes bounds the longest message. */
int rr_tokenize_batch(const uint8_t* text, const int64_t* text_off, int n_texts, int32_t vocab, int32_t* counts_out,
                      int32_t* ids_out, int64_t ids_capacity, int64_t* ids_off_out);
int rr_tokenize_batch_device(const uint8_t* d_text, const int64_t* d_text_off, int n_texts, int64_t max_text_bytes,
                             int32_t vocab, int32_t* d_counts, int32_t* d_ids, int64_t* d_ids_off, void* stream);

/* ================================================================================================
 * 3. Kernel-level entry points (used by the parity tests and the engine).
 *    Replaces the remote bedrock:InvokeModel prefill/decode (reference iam/policy.json:8,
 *    src/demo_cris.py:233-238).  All pointers are device pointers. */

enum { RR_OUT_ROWMAJOR_BF16 = 0, RR_OUT_TRANSPOSED_F32 = 1,
       /* fused SiLU(gate)*up epilogues; the weight operand holds gate/up rows interleaved in 64-row blocks
        * [g0..g63, u0..u63, g64..g127, u64..u127, ...] and the output is bf16 act[.., inter]: */
       RR_OUT_TRANSPOSED_SILU = 2,   /* decode: A = interleaved weight [2*inter, K], out[b*ldo + n], splits = 1 */
       RR_OUT_ROWMAJOR_SILU = 3,     /* prefill: B = interleaved weight, bn >= 128, out[a*ldo + n] */
       RR_OUT_ROWMAJOR_ROPE = 4,     /* engine-internal (prefill QKV epilogue with RoPE + KV scatter) */
       RR_OUT_ROWMAJOR_RESID = 5,    /* out = fp32 residual [rowsA, ldo]: out[a*ldo + b] += acc (bn >= 32) */
       RR_OUT_ROWMAJOR_F32 = 6 };    /* out fp32 [rowsA, ldo]: out[a*ldo + b] = acc (ldo even, out 8-byte aligned) */

/* D[a,b] = sum_k A[a,k] B[b,k] on wgmma tensor cores (bf16 in, fp32 accumulate).
 * mode RR_OUT_ROWMAJOR_BF16:  out bf16 [rowsA, ldo], out[a*ldo + b]         (splits must be 1)
 * mode RR_OUT_TRANSPOSED_F32: out fp32 [splits, ld_rows, ldo], out[(z*ld_rows + b)*ldo + a]
 * bn = tile width along B rows of the transposed modes: 16/32/64/128 (256 is accepted and runs 128-wide tiles).  The
 * row-major modes always run 128 x 256 tiles; their bn is only validated.  splits >= 1. */
int rr_gemm_bf16(const void* A, int rowsA, int ldA, const void* B, int rowsB, int ldB, int K,
                 void* out, int ldo, int ld_rows, int splits, int mode, int bn, void* stream);

/* FP8 weights.  A weight W [rows, K] bf16 is stored as Q [rows, K] e4m3 (row pitch K bytes) and one fp32 scale per row,
 * scale[n] = 2^e[n], e[n] = the smallest integer with max_k |W[n, k]| <= 448 * 2^e, clamped to [-117, 127] (0 for an
 * all-zero row); Q = e4m3 round-to-nearest-even of W / 2^e[n], subnormals included (it never saturates).
 * D = bf16(Q * scale) is exact for every row the quantizer accepts.  Q pointers must be 16-byte aligned and K a positive
 * multiple of 16.
 * quantize: w bf16 [rows, ld] (16-byte aligned, ld % 8 == 0, ld >= K).  Synchronises the stream.  RR_INVALID_ARGUMENT
 *   before touching the device for a bad argument, and after the kernel when a row holds Inf or NaN, or has a largest
 *   magnitude within 2^-4 of bf16's largest finite value (its e4m3 code times 2^e would be inf); those rows of q_out and
 *   scale_out are not written.
 * dequantize: out bf16 [rows, ld_out] = bf16(Q * scale) exactly (16-byte aligned, ld_out % 8 == 0, ld_out >= K). */
int rr_op_quantize_fp8_weight(const void* w, int rows, int K, int ld, void* q_out, float* scale_out, void* stream);
int rr_op_dequantize_fp8_weight(const void* q, const float* scale, int rows, int K, void* out, int ld_out, void* stream);
/* The dequantize of n_jobs (1..4) weights in one launch, as the engine runs it before each prefill layer of an FP8 model
 * (QKV, O, gate/up and down; the last layer QKV only): job i is rr_op_dequantize_fp8_weight(q[i], scale[i], rows[i], K[i],
 * out[i], ld_out[i]), with the same result bit for bit.  The arguments are host arrays of n_jobs entries.  Nothing outside
 * the jobs' rows [0, rows[i]) x columns [0, K[i]) of out[i] is written.  RR_INVALID_ARGUMENT before touching the device
 * for a null array, n_jobs outside 1..4, or a job rr_op_dequantize_fp8_weight would refuse. */
int rr_op_dequantize_fp8_jobs(const void* const* q, const float* const* scale, const int32_t* rows, const int32_t* K,
                              void* const* out, const int32_t* ld_out, int n_jobs, void* stream);
/* rr_gemm_bf16's decode modes (RR_OUT_TRANSPOSED_F32 / _SILU) with A an e4m3 weight [rowsA, K] (pitch ldA bytes, a
 * multiple of 16) and its row scales: the same tiles, splits, summation order and epilogues as rr_gemm_bf16 on
 * D = bf16(A * scale), so the same output bits.  RR_INVALID_ARGUMENT for a row-major mode or a null scale. */
int rr_gemm_fp8w(const void* A, const float* scale, int rowsA, int ldA, const void* B, int rowsB, int ldB, int K,
                 void* out, int ldo, int ld_rows, int splits, int mode, int bn, void* stream);
/* One decode projection (QKV, O, gate/up, down or lm_head) exactly as the engine plans and launches it for a decode working
 * set of `rows` rows (its max_batch): xn bf16 [rows, K], tile width 16 / 32 / 64 / 128 (the narrowest that holds rows;
 * 129..256 rows run two 128-row batch tiles per weight tile), plane pitch rows, the engine's split-K rule for (rows_w, K)
 * on this device (lm_head = 1: one plane, as the engine's lm_head), TMA-store epilogue where the engine uses one
 * (RR_NO_TMA_EPI is read per call).  *n_splits gets the planes used.
 *   RR_OUT_TRANSPOSED_F32:  w [rows_w, K]; out fp32 [n_splits][rows][rows_w]; plane z = sum over the k-blocks
 *                           [kb*z/n, kb*(z+1)/n) of xn[b,k] * w[n,k], kb = ceil(K / 64), n = n_splits
 *   RR_OUT_TRANSPOSED_SILU: w = gate/up rows interleaved in 64-row blocks [2*inter, K], rows_w = 2*inter; out bf16 act
 *                           [rows][inter] = SiLU(gate) * up; refused where the engine does not fuse it (rows <= 16, or
 *                           the split rule gives gate/up more than one plane)
 *   w_scale non-NULL: w is e4m3 with row scales (FP8 weights, rr_op_quantize_fp8_weight): bit for bit the bf16 call on
 *   the dequantized weight.  Not with lm_head.
 * RR_INVALID_ARGUMENT, *n_splits unchanged, for a null pointer, rows outside 1..256, another mode and whatever
 * rr_gemm_bf16 / rr_gemm_fp8w reject; all of these but the SiLU plane count before touching the device. */
int rr_op_decode_proj(const void* w, const float* w_scale, int rows_w, int K, const void* xn, int rows, void* out,
                      int mode, int lm_head, int* n_splits, void* stream);

/* Embedding gather, as the engine starts a step: x[r][c] = float(table[ids[r]][c]) exactly, for every row r < rows with
 * row_active NULL or row_active[r] >= 0; other rows of x are not written.  table bf16 [vocab][hidden], x fp32
 * [rows][hidden], ids / row_active int32 [rows] (device).  Ids are trusted, as slot indices are: each must be in
 * [0, vocab).  RR_INVALID_ARGUMENT before touching the device for a null ids, table or x, rows < 1, hidden not a positive
 * multiple of 8, and a table or x that is not 16-byte aligned. */
int rr_op_embed(const int32_t* ids, const void* table, float* x, int rows, int hidden,
                const int32_t* row_active, void* stream);
/* Embedding pool, as the engine pools a prefill chunk's embedding rows: for i < n, v = float(xn[rows ? rows[i] : i][0..hidden))
 * (bf16, row pitch ld elements), S = sum_c v_c^2 accumulated in fp64 in a fixed order (each square is exact),
 * out[i * out_ld + c] = fp32(v_c / sqrt(S)) computed in fp64 and rounded once, for c < hidden; S == 0 gives zeros.
 * Columns >= hidden of out and rows not listed are not written.  Deterministic: two calls agree bit for bit.  Row indices
 * are trusted, as ids are.  RR_INVALID_ARGUMENT before touching the device for a null xn or out, n outside 1..65535,
 * hidden not a positive multiple of 8 up to 16384, ld < hidden, out_ld < hidden, or a misaligned xn (16 B: xn itself and
 * ld % 8, every row). */
int rr_op_embed_pool(const void* xn, int ld, const int32_t* rows, int n, int hidden, float* out, int out_ld, void* stream);
int rr_op_add_rmsnorm(float* x, const void* part, int part_is_bf16, int n_splits,
                      long long split_stride, int part_ld, const void* w, void* xn, int rows,
                      int hidden, float eps, void* stream);
int rr_op_silu_mul(const void* gu, int is_bf16, int n_splits, long long split_stride, int ld,
                   void* act, int rows, int inter, void* stream);
int rr_op_rope_kv(const void* qkv, int is_bf16, int n_splits, long long split_stride, int ld,
                  void* q_out, void* k_cache, void* v_cache, const int32_t* slot,
                  const int32_t* pos, int rows, int n_heads, int n_kv_heads, int ctx_max,
                  float theta, void* stream);
/* Greedy pick over fp32 logits rows x (row r at logits + r * ld), as the engine picks a token: for every row r < rows with
 * row_active NULL or row_active[r] >= 0, m = the largest value of x[0 .. vocab) that is not NaN, and
 *   out_tok[r] = the lowest index i with x_i == m (-0 == +0), or 0 when m is -inf (every value -inf or NaN);
 *   out_val[r] = x_i of that index (m, or -inf), when out_val is non-NULL;
 *   pos_inc[r] += 1, when pos_inc is non-NULL.
 * So NaN never wins and the token is always in [0, vocab).  Inactive rows keep out_tok, out_val and pos_inc; columns
 * >= vocab are not read.  All arrays are device memory [rows].  RR_INVALID_ARGUMENT before touching the device unless
 * logits and out_tok are non-null, rows >= 1, 1 <= vocab <= ld, ld % 4 == 0 and logits is 16-byte aligned. */
int rr_op_argmax(const float* logits, int ld, int rows, int vocab, int32_t* out_tok,
                 float* out_val, const int32_t* row_active, int32_t* pos_inc, void* stream);
/* Log-probabilities of the best tokens of fp32 logits rows (row r at logits + r * ld), as the engine computes them for
 * `top_logprobs`: a row with top_n[r] >= 0 gets k = min(max(1, top_n[r]), max_top) entries, the k largest logits ordered by
 * value descending then token id ascending (entry 0 is rr_op_argmax's token), lp_out[r][j] = x - logsumexp(row) in fp32
 * and id_out[r][j] = the token id.
 * lp_out fp32 / id_out int32 [rows][max_top]; row r gets k = min(max(1, top_n[r]), max_top) entries, the rest of its
 * row and every row with top_n[r] < 0 untouched.  RR_INVALID_ARGUMENT before touching the device unless no pointer is
 * null, 1 <= rows <= 65535, 1 <= vocab <= ld, vocab <= 524288, ld % 4 == 0 and 1 <= max_top <= 20.  Deterministic: every
 * reduction runs in a fixed order. */
int rr_op_logprobs(const float* logits, int ld, int rows, int vocab, const int32_t* top_n, int max_top,
                   float* lp_out, int32_t* id_out, void* stream);
/* Seeded temperature / top-p draw from fp32 logits rows x (row r at logits + r * ld), as the engine samples a token.  All
 * per-row arrays are device memory [rows].  A row with temperature[r] = T > 0 gets out_tok[r] =
 *   argmax over {i : x_i >= tau} of x_i / T + G_i, ties to the lowest id, where
 *   tau = the largest logit value such that {j : x_j >= tau} holds at least top_p[r] of the mass of softmax(x / T)
 *         (top_p >= 1: every token; tokens tied at tau are all inside),
 *   G_i = -log(-log u_i), u_i = (2 (r_i >> 9) + 1) / 2^24, r_i = word 0 of Philox4x32-10 with key seed[r] (low word first)
 *         and counter (i, position[r], 0, 0).
 * Rows with temperature[r] <= 0 are not touched, nor are rows with no candidate i (every x_i -inf or NaN, or a tau that
 * is NaN): in the engine, out_tok[r] then keeps the greedy token rr_op_argmax wrote.  The draw is a pure function of (row,
 * T, top_p, seed, position).
 * RR_INVALID_ARGUMENT before touching the device unless no pointer is null, 1 <= rows <= 65535, 1 <= vocab <= ld,
 * vocab <= 524288 and ld % 4 == 0.  Deterministic: every sum is exact (fixed point) or runs in a fixed order. */
int rr_op_sample(const float* logits, int ld, int rows, int vocab, const float* temperature, const float* top_p,
                 const uint64_t* seed, const int32_t* position, int32_t* out_tok, void* stream);
/* Frequency / presence penalties and logit bias, in place over fp32 logits rows x (row r at logits + r * ld), as the
 * engine applies them before the argmax, the sampler and logprobs.  All per-row arrays are device memory.  With c_j the
 * number of times token j occurs in row r's history (hist + r * hist_ld, hist_len[r] tokens: the tokens generated so far)
 * and b_j the bias of token j (the n_bias[r] entries of bias_ids / bias_vals + r * bias_ld; ids unique), every processed
 * logit becomes
 *   x'_j = (x_j + b_j) - (c_j * frequency_penalty[r] + [c_j > 0] * presence_penalty[r]),
 * each operation one fp32 round-to-nearest op without FMA contraction.  A token without a bias entry skips the addition, one
 * with c_j = 0 the subtraction; a row with both penalties 0 and no bias entries is not touched.  Deterministic: the counts
 * are integer atomics and exactly one thread writes each logit.  History ids outside [0, vocab) are ignored; hist_len[r] is
 * clamped to [0, hist_ld] and n_bias[r] to [0, bias_ld].  RR_INVALID_ARGUMENT before touching the device unless no pointer
 * is null, 1 <= rows <= 65535, 1 <= vocab <= ld, vocab <= 524288, ld % 4 == 0, hist_ld >= 0 and 0 <= bias_ld <= 300. */
int rr_op_logit_penalties(float* logits, int ld, int rows, int vocab, const int32_t* hist, int hist_ld,
                          const int32_t* hist_len, const float* frequency_penalty, const float* presence_penalty,
                          const int32_t* bias_ids, const float* bias_vals, int bias_ld, const int32_t* n_bias, void* stream);
/* Stop sequences, as the engine matches them after a token is picked.  All arrays are device memory.  Row r has n_stop[r]
 * (0..4) sequences, sequence s the stop_len[r * 4 + s] (1..64) bytes at stop_bytes + (r * 4 + s) * 64 (stop_bytes 4-byte
 * aligned).  The reply text of a row is its history tokens mapped like the byte tokenizer maps them back: a token t >= 3 is
 * the byte (t - 3) % 256, a token < 3 is no text.  For every row with n_stop[r] > 0 and (row_active NULL or
 * row_active[r] >= 0) the kernel stores tok[r] at hist[r * hist_ld + i], i = position[r] - gen0[r], and over the text of
 * hist[r][0 .. i] writes
 *   cut_out[r]  = -1, or when tok[r] has a byte and the text ends in a sequence: the index in the history of the first
 *                 token of the longest such sequence, which is the number of tokens that come before the match;
 *   hold_out[r] = 0 on a hit, else the number of newest tokens from the first token of the longest suffix of the text that
 *                 is a proper prefix of a sequence (0 when there is none): what a streaming reader must not be shown yet.
 * Other rows are not touched; i outside [0, hist_ld) gives (-1, 0) and no store.  No other history cell is written.  Work
 * per row is O(64 x 4) plus the length of any run of byteless tokens; integer only, so two calls agree bit for bit.
 * RR_INVALID_ARGUMENT before touching the device for a null pointer other than row_active, rows outside 1..65535,
 * hist_ld < 1 or a misaligned stop_bytes. */
int rr_op_stop_match(int32_t* hist, int hist_ld, const int32_t* tok, const int32_t* position, const int32_t* row_active,
                     const int32_t* n_stop, const int32_t* gen0, const uint8_t* stop_len, const uint8_t* stop_bytes,
                     int32_t* cut_out, int32_t* hold_out, int rows, void* stream);
/* JSON mode, as the engine masks and advances a json_object row.  All arrays are device memory.  state is [rows] opaque
 * 16-byte automaton states (all zero: the initial state, before the top-level '{'); the caller never interprets them.
 * Token t >= 3 is the byte (t - 3) % 256; tokens 0..2 are never allowed.  The automaton accepts exactly the prefixes of JSON
 * texts (RFC 8259) whose top-level value is an object, with strict UTF-8 in strings (no overlongs, no surrogates, nothing
 * above U+10FFFF), no raw bytes < 0x20 in strings, at most 64 open containers ('{' and '[' are not allowed at 64) and runs
 * of insignificant whitespace of at most 64 bytes; after the closing '}' it allows whitespace only.  No state allows no byte.
 * Rows with fmt[r] == 0 or (row_active non-NULL and row_active[r] < 0) are skipped by both calls.
 * mask: writes -inf to every column c < vocab of row r (logits + r * ld) that the row's state (state NULL: the initial
 *   state) does not allow: c < 3, or byte (c - 3) % 256 not allowed.  It never reads the logits; allowed columns and
 *   columns >= vocab are not touched.  Grid: one CTA per 8192 columns of a row.
 * advance: state_out[out_row ? out_row[r] : r] = the state of row r (state_in NULL: the initial state) after tok[r], and
 *   done[r] = 1 when that state is past the top-level object's closing '}', else 0.  A token the state does not allow
 *   leaves the state as it was.  Integer work only: two calls agree bit for bit.
 * RR_INVALID_ARGUMENT before touching the device for a null logits / fmt / tok / state_out / done pointer, rows outside
 * 1..65535, or (mask) unless 1 <= vocab <= ld, vocab <= 524288 and ld % 4 == 0. */
int rr_op_json_mask(float* logits, int ld, int rows, int vocab, const int32_t* fmt, const int32_t* row_active,
                    const void* state, void* stream);
int rr_op_json_advance(int rows, const int32_t* fmt, const int32_t* row_active, const int32_t* tok, const void* state_in,
                       void* state_out, const int32_t* out_row, int32_t* done, void* stream);
int rr_op_decode_attn(const void* q, const void* k_cache, const void* v_cache, void* out,
                      const int32_t* slot, const int32_t* pos, int rows, int n_heads,
                      int n_kv_heads, int ctx_max /* % 64 == 0 */, int n_slots, float scale,
                      int kv_splits, void* stream);
int rr_op_prefill_attn(const void* q, const void* k_cache, const void* v_cache, void* out,
                       const int32_t* seq_start, const int32_t* seq_slot, int n_seqs, int max_len,
                       int n_heads, int n_kv_heads, int ctx_max, float scale, void* stream);
/* Prefill attention over a cached prompt prefix, as the engine runs it with prefix caching on (rr_engine_opts.prefix_cache):
 * sequence i's seq_start[i + 1] - seq_start[i] query rows sit at positions seq_pos0[i] .. seq_pos0[i] + len - 1 of slot
 * seq_slot[i] and attend to positions 0 .. own position of that slot's cache (positions < seq_pos0[i] hold the prefix).
 * max_len = the longest len.  Caches [n_slots][n_kv_heads][ctx_max][128], q / out [T][n_heads * 128] bf16.  Row r of a
 * sequence equals, bit for bit, row seq_pos0[i] + r of rr_op_prefill_attn over the whole sequence.  Returns
 * RR_INVALID_ARGUMENT before touching the device for a null pointer, n_seqs or max_len below 1, a group size that does not
 * divide, or ctx_max not a positive multiple of 64; and after reading the index arrays back, for a negative pos0, a
 * sequence longer than max_len or pos0 + len > ctx_max. */
int rr_op_prefill_attn_cached(const void* q, const void* k_cache, const void* v_cache, void* out,
                              const int32_t* seq_start, const int32_t* seq_slot, const int32_t* seq_pos0, int n_seqs,
                              int max_len, int n_heads, int n_kv_heads, int ctx_max, float scale, void* stream);
/* KV prefix copy, one launch for a list of n_copies (src[i], dst[i], n_tok[i]) (host arrays): positions [0, n_tok[i]) of
 * slot src[i] are copied to slot dst[i] in K and V, for every layer and kv head.  Caches [n_layers][n_slots][n_kv_heads]
 * [ctx_max][128] bf16 (device).  No other byte changes.  Returns RR_INVALID_ARGUMENT before touching the device for a null
 * pointer, n_copies outside 1..256, a slot outside [0, n_slots), n_tok outside 1..ctx_max, a destination listed twice, or a
 * destination that is also a source in the same call. */
int rr_op_kv_copy_prefix(void* k_cache, void* v_cache, int n_layers, int n_slots, int n_kv_heads, int ctx_max,
                         const int32_t* src, const int32_t* dst, const int32_t* n_tok, int n_copies, void* stream);
/* Paged KV cache, as the engine runs it: the four entry points below take the arguments of rr_op_decode_attn_qkv,
 * rr_op_prefill_qkv, rr_op_prefill_attn_cached and rr_op_kv_copy_prefix plus a page table.  The caches are
 * [n_pages][n_kv_heads][64][128] bf16 (per layer for the copy), and position p of slot s lives on page
 * page_table[s * pages_per_slot + p / 64] (device int32 [n_slots][pages_per_slot]), at row p % 64 of the page.  ctx_max
 * must be 64 x pages_per_slot.  Table entries are trusted, as slot indices are: each must be in [0, n_pages).  Only the
 * table rows of the slots named (slot >= 0, seq_slot, src / dst) are read, so the table needs n_slots rows.  Returns
 * RR_INVALID_ARGUMENT before touching the device for a null page_table, pages_per_slot or n_pages below 1, or ctx_max
 * other than 64 x pages_per_slot; otherwise for whatever the counterpart rejects.  Results, bit for bit: the
 * counterpart's over the cache gathered through the table. */
int rr_op_decode_attn_qkv_paged(const float* qkv, int n_splits, long long split_stride, int ld, void* k_cache,
                                void* v_cache, void* out, const int32_t* slot, const int32_t* pos, int rows, int n_heads,
                                int n_kv_heads, int head_dim, int ctx_max, int n_slots, float theta, int* kv_splits,
                                const int32_t* page_table, int pages_per_slot, int n_pages, void* stream);
int rr_op_prefill_qkv_paged(const void* xhat, const float* rowss, int plan_rows, int T, int hidden, const void* wqkv,
                            int n_heads, int n_kv_heads, int head_dim, int ctx_max, float theta, float eps,
                            const int32_t* slot, const int32_t* pos, void* q_out, void* k_cache, void* v_cache, int* fused,
                            const int32_t* page_table, int pages_per_slot, int n_pages, void* stream);
int rr_op_prefill_attn_cached_paged(const void* q, const void* k_cache, const void* v_cache, void* out,
                                    const int32_t* seq_start, const int32_t* seq_slot, const int32_t* seq_pos0, int n_seqs,
                                    int max_len, int n_heads, int n_kv_heads, int ctx_max, float scale,
                                    const int32_t* page_table, int pages_per_slot, int n_pages, void* stream);
int rr_op_kv_copy_prefix_paged(void* k_cache, void* v_cache, int n_layers, int n_slots, int n_kv_heads, int ctx_max,
                               const int32_t* src, const int32_t* dst, const int32_t* n_tok, int n_copies,
                               const int32_t* page_table, int pages_per_slot, int n_pages, void* stream);
/* The hand-off of a prefill chunk to decode, as the engine runs it after the chunk's last layer (device arrays).
 * gather_last: for r < n_rows, attn_out[r][0..nq) = attn[last[r]][0..nq) (bf16) and x_out[r][0..hidden) =
 *   x[last[r]][0..hidden) (fp32), bit for bit; the rows of the tail and embedding rows of a chunk, several of them may name
 *   the same last[r].  Rows >= n_rows of the outputs are not written.  RR_INVALID_ARGUMENT before touching the device for a
 *   null pointer, n_rows < 1, nq not a positive multiple of 8, hidden not a positive multiple of 4, or a buffer that is not
 *   16-byte aligned.
 * activate_rows: for i < n, slot s = seq_slot[i] becomes a live decode row: d_tok[s] = first_tok[i],
 *   d_pos[s] = tok_pos[last[i]] + 1 (the position after the prompt's last token, a cached prefix included), d_slot[s] = s.
 *   No other entry is written; the slots must be distinct.  RR_INVALID_ARGUMENT before touching the device for a null
 *   pointer or n < 1.
 * Indices are trusted, as slot indices are. */
int rr_op_gather_last(const void* attn, const float* x, const int32_t* last, int n_rows, int nq, int hidden, void* attn_out,
                      float* x_out, void* stream);
int rr_op_activate_rows(const int32_t* seq_slot, const int32_t* first_tok, const int32_t* tok_pos, const int32_t* last, int n,
                        int32_t* d_tok, int32_t* d_pos, int32_t* d_slot, void* stream);
/* Decode attention with a sliding window W = window: the arguments of rr_op_decode_attn_qkv_paged plus window.  The row
 * at position pos attends to positions max(0, pos - W + 1) .. pos of its slot; window 0 is full causal attention, and
 * rr_op_decode_attn_qkv_paged is this call with window 0.  The kv splits divide the key tiles from the tile of
 * max(0, pos - W + 1) on, so a row whose every key lies inside the window (pos < W) gets rr_op_decode_attn_qkv_paged's
 * result bit for bit.  Table entries are read only for the pages of the window's tiles, so a table may map logical page p
 * to pages[p mod R] (a ring of R pages) when no window spans more than R pages.  Returns RR_INVALID_ARGUMENT before touching the device
 * for a negative window, and otherwise for whatever rr_op_decode_attn_qkv_paged rejects. */
int rr_op_decode_attn_qkv_window(const float* qkv, int n_splits, long long split_stride, int ld, void* k_cache,
                                 void* v_cache, void* out, const int32_t* slot, const int32_t* pos, int rows, int n_heads,
                                 int n_kv_heads, int head_dim, int ctx_max, int n_slots, float theta, int* kv_splits,
                                 const int32_t* page_table, int pages_per_slot, int n_pages, int window, void* stream);
/* Prefill attention with a sliding window W = window: the arguments of rr_op_prefill_attn_cached_paged plus window.  The
 * query row at absolute position q (seq_pos0 + its row) attends to positions max(0, q - W + 1) .. q of its slot; window 0
 * is full causal attention, and rr_op_prefill_attn_cached_paged is this call with window 0.  Each 128-row query tile reads
 * key tiles from the tile of max(0, q0 - W + 1) on, q0 its first row's position; key tiles wholly outside a row's window
 * leave its softmax state unchanged, so rows whose every key lies inside the window (q < W) get
 * rr_op_prefill_attn_cached_paged's result bit for bit, and each row is the softmax over exactly its visible keys.
 * Returns RR_INVALID_ARGUMENT before touching the device for a negative window, and otherwise for whatever
 * rr_op_prefill_attn_cached_paged rejects. */
int rr_op_prefill_attn_window(const void* q, const void* k_cache, const void* v_cache, void* out,
                              const int32_t* seq_start, const int32_t* seq_slot, const int32_t* seq_pos0, int n_seqs,
                              int max_len, int n_heads, int n_kv_heads, int ctx_max, float scale,
                              const int32_t* page_table, int pages_per_slot, int n_pages, int window, void* stream);
/* Prefill attention exactly as the engine launches it for one chunk: the arguments of rr_op_prefill_attn_window with the
 * true head_dim in place of scale, plus q_rows.  The scale is the engine's, 1 / sqrtf(head_dim).  q is [q_rows][n_heads *
 * 128] bf16 with columns [head_dim, 128) of each head zero, mapped over all q_rows rows as the engine maps its prefill
 * buffer (q_rows >= T = seq_start[n_seqs]; rows T.. may hold anything and are never written out).  Caches are paged
 * [n_pages][n_kv_heads][64][128] bf16, columns [head_dim, 128) ignored.  out is [T][n_heads * head_dim] bf16: element
 * (t, h * head_dim + d) for d < head_dim; nothing else is written.  With head_dim 128 the result equals
 * rr_op_prefill_attn_window's at scale 1 / sqrtf(128), bit for bit.  Returns RR_INVALID_ARGUMENT before touching the
 * device for a null pointer, head_dim outside 64..128 or not a multiple of 16, n_heads / n_kv_heads not in {1, 2, 4, 8},
 * a page table rr_op_prefill_attn_window rejects, max_len below 1, q_rows < max_len or a negative window; and after
 * reading the index arrays back, for what rr_op_prefill_attn_cached rejects there or q_rows < T. */
int rr_op_prefill_attn_hd(const void* q, const void* k_cache, const void* v_cache, void* out, const int32_t* seq_start,
                          const int32_t* seq_slot, const int32_t* seq_pos0, int n_seqs, int max_len, int n_heads,
                          int n_kv_heads, int head_dim, int ctx_max, const int32_t* page_table, int pages_per_slot,
                          int n_pages, int window, int q_rows, void* stream);
/* Fused decode MLP, one launch exactly as the engine runs it for a batch of `rows` (tile width, K slices, grid and
 * schedule from the engine's rules; env RR_MLP_STATIC / RR_NO_TMA_EPI are read per call):
 *   act[b, n]       = bf16(SiLU(xn[b] . gate[n]) * (xn[b] . up[n]))                        bf16 [rows, inter]
 *   planes[z][b][h] = sum over k in slice z of act[b, k] * wdown[h, k]                       fp32 [n_slices][ld_rows][hidden]
 * Slice z covers the k-blocks (64 act columns each) [z * slice_kb, min((z + 1) * slice_kb, inter / 64)); the sum of the
 * planes is the down projection.  Plane rows >= rows are not written.  wgu_il = [gate; up] rows interleaved in 64-row
 * blocks [2*inter, hidden].  Returns RR_INVALID_ARGUMENT before touching the device unless 17 <= rows <= 128,
 * ld_rows >= rows, hidden and inter are positive multiples of 64, hidden <= 8192 and no pointer is null. */
int rr_op_decode_mlp(const void* wgu_il, const void* wdown, const void* xn, int rows, int hidden, int inter,
                     void* act, void* planes, int ld_rows, int* n_slices, int* slice_kb, void* stream);
/* The same with e4m3 weights (rr_op_quantize_fp8_weight) and their row scales (wgu_scale interleaved like the rows):
 * bit for bit rr_op_decode_mlp on the dequantized weights.  Also RR_INVALID_ARGUMENT for a null scale. */
int rr_op_decode_mlp_fp8(const void* wgu_il, const float* wgu_scale, const void* wdown, const float* wdown_scale,
                         const void* xn, int rows, int hidden, int inter, void* act, void* planes, int ld_rows,
                         int* n_slices, int* slice_kb, void* stream);
/* Decode attention, one step exactly as the engine runs it: RoPE and the KV append fused in, scale 1 / sqrt(head_dim), the
 * engine's kv-split rule (returned in *kv_splits) and RoPE table (theta); env RR_ATTN_NO_TRIM is read per call.
 *   qkv      fp32 split-K planes [n_splits][..][ld], plane z of row b at qkv + z * split_stride + b * ld; columns are the
 *            q heads, then the k heads, then the v heads, head_dim each (unpadded); q / k / v = the sum of the planes
 *   k_cache, v_cache  bf16 [n_slots][n_kv_heads][ctx_max][128]; row b (slot[b] >= 0) appends its rotated k and its v at
 *            position pos[b] of slot[b] (columns [0, head_dim)) and attends over positions 0..pos[b]; rows with
 *            slot[b] < 0 are skipped
 *   out      bf16 [rows][n_heads * head_dim]
 * Returns RR_INVALID_ARGUMENT before touching the device, *kv_splits unchanged, unless no pointer is null, rows >= 1,
 * n_slots >= 1, n_splits >= 1, n_heads / n_kv_heads is 1, 2, 4 or 8, head_dim is a multiple of 16 in 64..128, ctx_max is
 * a positive multiple of 64, ld >= (n_heads + 2 * n_kv_heads) * head_dim and ld and split_stride are even. */
int rr_op_decode_attn_qkv(const float* qkv, int n_splits, long long split_stride, int ld, void* k_cache, void* v_cache,
                          void* out, const int32_t* slot, const int32_t* pos, int rows, int n_heads, int n_kv_heads,
                          int head_dim, int ctx_max, int n_slots, float theta, int* kv_splits, void* stream);
/* Prefill, deferred RMSNorm.  The engine does not normalise the operands of a prefill chunk's projections: the operand row
 * is xhat = bf16(x * gamma) and comes with n_part = ceil(hidden / 128) partial sums of squares rowss[row][p]; the consuming
 * GEMM scales its fp32 accumulators by rsqrt(sum_p rowss[row][p] / hidden + eps) before its epilogue.  The entry points
 * below run the prefill kernels exactly as the engine does (plans made for plan_rows rows and launched for the first T,
 * deferred-norm fields filled by the engine's helpers).  Each returns RR_INVALID_ARGUMENT before touching the device, with
 * its out-parameters unchanged, for the arguments listed.
 *
 * Layer 0's norm of a prefill chunk: xn[r] = bf16(x[r] * w) (not normalised), rowss_out[r][0] = sum(x[r]^2) in fp32,
 * rowss_out[r][1 .. n_part_out) = 0, for rows r < rows; x is not written.  Rejects a null pointer, rows < 1, hidden not a
 * multiple of 64 in 64..8192, and n_part_out != ceil(hidden / 128). */
int rr_op_add_rmsnorm_pf(float* x, const void* w, void* xn, int rows, int hidden, float eps, float* rowss_out,
                         int n_part_out, void* stream);
/* The QKV projection of a prefill chunk with RoPE and the KV append (theta: the engine's RoPE table):
 *   xhat     bf16 [plan_rows][hidden], rowss fp32 [plan_rows][ceil(hidden / 128)]; rows >= T are not read into any output
 *   wqkv     bf16 [(n_heads + 2 n_kv_heads) head_dim][hidden]: q heads, then k heads, then v heads
 *   q_out    bf16 [T][n_heads * 128]: rotated q, columns [0, head_dim) of each head
 *   k_cache, v_cache  bf16 [..][n_kv_heads][ctx_max][128]: token t writes its rotated k and its v to columns [0, head_dim)
 *            of position pos[t] of slot slot[t] (slot[t] >= 0)
 * *fused = 1 when the GEMM epilogue did RoPE and the append (head_dim 128), 0 when rope_kv_kernel did them from a bf16 qkv
 * matrix.  Rejects a null pointer, T outside 1..plan_rows, hidden not a multiple of 64 in 64..8192, n_heads / n_kv_heads
 * not 1, 2, 4 or 8, head_dim not a multiple of 16 in 64..128, and ctx_max not a positive multiple of 64. */
int rr_op_prefill_qkv(const void* xhat, const float* rowss, int plan_rows, int T, int hidden, const void* wqkv,
                      int n_heads, int n_kv_heads, int head_dim, int ctx_max, float theta, float eps,
                      const int32_t* slot, const int32_t* pos, void* q_out, void* k_cache, void* v_cache, int* fused,
                      void* stream);
/* The O, gate/up and down projections of a prefill chunk: rr_gemm_bf16's row-major modes on A [plan_rows][K] (pitch ldA),
 * launched for rows < T.
 *   mode RR_OUT_ROWMAJOR_BF16 / RR_OUT_ROWMAJOR_SILU / RR_OUT_ROWMAJOR_F32 with n_part > 0: deferred-norm consumer (rowss
 *        [plan_rows][n_part], n_part = ceil(hidden / 128)); n_part = 0: A is used as it is
 *   mode RR_OUT_ROWMAJOR_F32: out fp32 [T][ldo], out[t][n] = acc * rinv(t) for n < rowsW (ldo even, out 8-byte aligned);
 *        rinv(t) = 1 / sqrt(sum(rowss[t][..]) / hidden + eps) with n_part > 0, else 1.  Rows >= T and columns >= rowsW are
 *        not written.  lm_head over the prompt rows of a scoring prefill chunk (rr_engine_submit_scored).
 *   mode RR_OUT_ROWMAJOR_RESID: out is the fp32 residual [..][ldo], out[t][n] += acc.  With xhat: deferred-norm producer,
 *        xhat[t][n] = bf16(out[t][n] * gamma[n]) (pitch ldo) and rowss_out[t][p] = sum of out[t][n]^2 over n in
 *        [128 p, 128 p + 128), n_part_out = ceil(rowsW / 128)
 * Rejects a null A, W or out, T outside 1..plan_rows, rowsW < 1, another mode, a consumer with a null rowss, mode RESID or
 * the wrong n_part, a producer outside mode RESID, with a null gamma or rowss_out, or the wrong n_part_out, and whatever
 * rr_gemm_bf16 rejects. */
int rr_op_prefill_gemm(const void* A, int plan_rows, int T, int ldA, const void* W, int rowsW, int K, void* out, int ldo,
                       int mode, const float* rowss, int n_part, int hidden, float eps, const void* gamma, void* xhat,
                       float* rowss_out, int n_part_out, void* stream);

/* ================================================================================================
 * 4. Engine: one model replica on one GPU (prefill + continuous-batching greedy decode).
 *    Replaces one `litellm_params.model: bedrock/...` deployment (reference config.yaml:39,47,54,
 *    62,69,77,84,91). */

/* vocab: a multiple of 4, >= 4 (each row of the [rows][vocab] fp32 logits is read with 16-byte loads); rr_engine_create
 * returns RR_INVALID_ARGUMENT before any CUDA call otherwise. */
typedef struct rr_model_desc {
    int32_t vocab, hidden, inter, n_layers, n_heads, n_kv_heads, head_dim;
    float rope_theta, rms_eps;
} rr_model_desc;

/* Device pointers to bf16 weights, row-major [out_features, in_features] like torch nn.Linear.
 * wqkv = concat(q_proj, k_proj, v_proj) rows; wgu = concat(gate_proj, up_proj) rows. */
typedef struct rr_model_weights {
    const void* embed;            /* [vocab, hidden] */
    const void* lm_head;          /* [vocab, hidden] */
    const void* final_norm;       /* [hidden] */
    const void* const* wqkv;      /* n_layers x [(n_heads + 2 n_kv_heads) * head_dim, hidden] */
    const void* const* wo;        /* n_layers x [hidden, n_heads * head_dim] */
    const void* const* wgu;       /* n_layers x [2 * inter, hidden] */
    const void* const* wdown;     /* n_layers x [hidden, inter] */
    const void* const* norm_attn; /* n_layers x [hidden] */
    const void* const* norm_mlp;  /* n_layers x [hidden] */
    int32_t flags;                /* RR_WEIGHTS_* */
    /* Sliding-window attention W >= 0 (0: full causal): position q attends to positions max(0, q - W + 1) .. q.  A model
     * property, not a deployment one; rr_engine_create refuses a negative value.  See rr_engine_submit for the KV ring. */
    int32_t sliding_window;
    /* RR_WEIGHTS_FP8_E4M3 only (ignored otherwise): n_layers x fp32 [out_features] row scales of wqkv / wo / wgu / wdown */
    const void* const* wqkv_scale;
    const void* const* wo_scale;
    const void* const* wgu_scale;
    const void* const* wdown_scale;
} rr_model_weights;
/* wgu rows are interleaved in 64-row gate/up blocks [g0..g63, u0..u63, g64.., u64.., ...] instead of
 * [gate; up]: enables the fused SiLU*mul GEMM epilogues (no separate activation kernel). */
#define RR_WEIGHTS_WGU_INTERLEAVED64 1
/* wqkv / wo / wgu / wdown are e4m3 [out_features, in_features] (rr_op_quantize_fp8_weight: 16-byte aligned) with the row
 * scales above (with RR_WEIGHTS_WGU_INTERLEAVED64 the wgu rows and their scales are interleaved alike); embed, lm_head
 * and the norms stay bf16.  The engine computes exactly what a bf16 engine computes on D = bf16(Q * scale): decode
 * converts the e4m3 tiles in its GEMMs, prefill dequantizes each layer into an engine-owned bf16 scratch of one layer's
 * four projections (2 x (nqkv + nq + 3 inter) x hidden bytes) before the layer's GEMMs.  rr_engine_create returns
 * RR_INVALID_ARGUMENT before any CUDA call for a null or misaligned e4m3 pointer or a null scale pointer. */
#define RR_WEIGHTS_FP8_E4M3 2

typedef struct rr_engine rr_engine;

typedef struct rr_engine_opts {
    int32_t device;
    int32_t max_batch;            /* decode rows / KV slots (<= 256) */
    int32_t ctx_max;              /* tokens per request (prompt + max_new_tokens), a multiple of 64 */
    int32_t max_prefill_tokens;   /* tokens per prefill chunk.  A prompt whose uncached part does not fit the room left in a
                                     chunk is prefilled in pieces: its first piece fills that room, each later piece
                                     (up to this many tokens) leads the next chunk, and after every chunk that leaves it
                                     in progress the worker runs one decode step for the rows already decoding.  One
                                     prompt is in progress at a time, and nothing overtakes it. */
    int32_t use_cuda_graph;       /* capture the decode step */
    int32_t fail_seed;            /* fault injection: seed of the Bernoulli failure mask */
    float fail_prob;              /* fault injection: P(request fails) (BASELINE config #4) */
    int32_t kv_cache_tokens;      /* offset 28: the KV cache, a pool of 64-token pages shared by the decode rows.  0 =
                                     max_batch x ctx_max (every row can hold ctx_max tokens at once, the pool never binds);
                                     otherwise a multiple of 64 in [ctx_max, max_batch x ctx_max], else rr_engine_create
                                     returns RR_INVALID_ARGUMENT before any CUDA call.  Each choice of a request reserves
                                     ceil((n_prompt + max_new_tokens) / 64) pages when it is admitted, at most the ring of
                                     a windowed model (rr_engine_submit); a request that does
                                     not fit waits at the head of the queue (nothing overtakes it).  Memory: 2 x n_layers x
                                     kv_cache_tokens x n_kv_heads x 256 B. */
    int32_t reserved[3];          /* ignored (pass zeros); keeps prefix_cache at offset 44 */
    int32_t prefix_cache;         /* 1: prompt prefix caching.  A slot keeps the prompt KV its last prefill wrote; a new prompt
                                     sharing >= 64 leading tokens with one is prefilled from there on (the prefix is copied
                                     when that slot is busy).  Tokens and logits are bit-identical to a cold prefill.  Off
                                     by default: a resident prefix is a timing side channel between the engine's users. */
} rr_engine_opts;

int rr_engine_create(const rr_model_desc* desc, const rr_model_weights* w,
                     const rr_engine_opts* opts, rr_engine** out);
void rr_engine_destroy(rr_engine* e);

/* Low-level synchronous steps (parity tests).  Host buffers.  Both forget every retained prompt prefix (prefix_cache), and
 * both first give each named slot the KV pages of the positions they write (positions [0, prompt length) / [0, pos]); they
 * return RR_INVALID_ARGUMENT when the free pages do not cover that.  A slot keeps those pages until a request takes it.
 * prefill: n_seqs prompts concatenated in `ids`; seq_start[n_seqs+1]; slots[n_seqs] = KV slots.
 *          Writes first generated token per prompt to first_tok[n_seqs].
 *          If logits_out != NULL: fp32 [n_seqs, vocab] last-position logits. */
int rr_engine_prefill(rr_engine* e, const int32_t* ids, const int32_t* seq_start,
                      const int32_t* slots, int n_seqs, int32_t* first_tok, float* logits_out);
/* One decode step for the given slots, feeding tok[i] at position pos[i]; returns next tokens and
 * optionally fp32 logits [n, vocab]. */
int rr_engine_decode_step(rr_engine* e, const int32_t* slots, const int32_t* tok,
                          const int32_t* pos, int n, int32_t* next_tok, float* logits_out);

/* Asynchronous serving interface (the call shape of chat.completions.create: reference
 * src/demo_load_balancing.py:106-110).  submit is thread-safe and non-blocking; wait blocks
 * (release the GIL around it). */
typedef struct rr_completion {
    uint64_t ticket;
    int32_t status;               /* RR_OK / RR_BACKEND_FAILED / RR_TIMEOUT */
    int32_t n_prompt;
    int32_t n_generated;
    int32_t n_cached;             /* prompt tokens whose KV came from the prefix cache (prefix_cache; 0 otherwise) */
    double t_submit_s, t_first_token_s, t_done_s;   /* engine monotonic clock */
} rr_completion;

/* Generation parameters of one request: the fields of chat.completions.create that steer decoding.  rr_engine_submit
 * states what each does; the field comments give the encodings.  A NULL rr_gen_params* is a plain greedy request of one
 * choice.  A non-NULL struct is read in full: zero is a value, never "use the default". */
typedef struct rr_gen_params {
    int32_t n_choices;                   /* 1..max_batch (OpenAI n) */
    int32_t top_logprobs;                /* -1: off; 0..20 */
    float temperature, top_p;            /* temperature 0: greedy (top_p and seed unused) */
    uint64_t seed;
    float frequency_penalty, presence_penalty;
    int32_t n_bias, n_stop;
    const int32_t* bias_ids;  const float* bias_vals;      /* [n_bias] */
    const uint8_t* stop_bytes; const int32_t* stop_off;    /* sequence i = stop_bytes[stop_off[i] .. stop_off[i+1]) */
    int32_t response_format;             /* 0 text, 1 json_object */
    int32_t reserved;                    /* pass 0 */
} rr_gen_params;                         /* 80 bytes; the offsets are pinned by tests/test_abi.py */

/* Queue one request and write its ticket to *ticket; finish it with rr_engine_wait or rr_engine_cancel.  p = NULL is a
 * greedy request of one choice.  The tokens depend only on the prompt, the weights and p: not on the batch, the slot, the
 * prefix cache or the replica.
 * - top_logprobs (OpenAI `logprobs` / `top_logprobs`) 0..20: for every generated token the engine records K =
 *   max(1, top_logprobs) (logprob, token id) pairs, the K most likely tokens of that step ordered by logprob descending then
 *   id ascending (pair 0 is the greedy token), computed on the GPU from the same fp32 logits the pick reads
 *   (rr_op_logprobs).  With temperature > 0 a token has K + 1 pairs, the last being (the generated token's logprob, its
 *   id).  Logprobs change no token.
 * - temperature > 0 (seeded sampling, OpenAI `temperature` / `top_p` / `seed`): every token is drawn by rr_op_sample with
 *   (temperature, top_p, seed) at its own position (n_prompt for the first generated token, n_prompt + j for the j-th after
 *   it).  temperature = 0 is greedy.
 * - frequency_penalty / presence_penalty / logit bias (bias_ids[i] gets bias_vals[i]): before every token is picked
 *   (argmax, or the draw), its logits go through rr_op_logit_penalties with the tokens the choice generated so far as the
 *   history (prompt tokens do not count, so the first token gets the bias only).  Logprobs describe the processed logits.
 *   Penalties 0 and n_bias = 0 change nothing.
 * - n_choices (OpenAI `n`): completions of the same prompt.  The prompt is prefilled once; its KV is then copied into
 *   n_choices - 1 further KV slots, and every choice decodes in a row of its own.  Choice i is exactly what the request of
 *   one choice gives with seed (seed + i) mod 2^64 and the same other parameters (greedy: every choice is the greedy
 *   completion); penalties count the choice's own tokens.  The choices run in lockstep: they are admitted together (a
 *   request waits at the head of the queue until n_choices rows are free; nothing overtakes it) and get one token each per
 *   step.  Without stop sequences or JSON mode they end together.  Cancellation, an injected failure or an internal error
 *   ends every choice.
 * - stop sequences (OpenAI `stop`): n_stop sequences, sequence i = stop_bytes[stop_off[i] .. stop_off[i + 1]).  They are
 *   matched on the reply text (a generated token t >= 3 is the byte (t - 3) % 256, a token < 3 is no text) by
 *   rr_op_stop_match after every generated token, the first included.  A choice whose text comes to end in a sequence
 *   finishes with reason 1 (stop): it returns the tokens before the first token of the match (of the longest sequence when
 *   several end there), its logprob pairs likewise, and its decode row is free from the next step on, while the request's
 *   other choices go on.  Stop sequences change no logit and no draw: the tokens returned are a prefix of those of the
 *   same request without them.
 * - response_format 1 (JSON mode, OpenAI `response_format: {"type": "json_object"}`): before every token is picked (after
 *   penalties and logit bias, before the argmax, the sampler and logprobs) rr_op_json_mask sets the logit of every token
 *   the JSON grammar does not allow next to -inf, so the reply's bytes are always a prefix of a JSON text whose top-level
 *   value is an object (rr_op_json_mask states the grammar), and logprobs describe the masked distribution (a masked
 *   token's logprob is -inf).  The choice whose token closes the top-level object finishes with reason 1 (stop), that token
 *   included, and frees its decode row at once; a stop-sequence cut on the same token wins.
 * A choice that reaches max_new_tokens first finishes with reason 0 (length), in JSON mode with a valid prefix.  The
 * request is done when every choice has finished.
 * Sliding window (rr_model_weights.sliding_window = W > 0): with Tmax = max_prefill_tokens, a choice reserves at most
 * R = ceil((W + Tmax - 2) / 64) + 1 pages, the most any prefill piece or decode step reads and writes at once.  A request
 * whose reach (n_prompt + max_new_tokens) needs more is a ring request: each of its slots holds R pages and its page-table
 * row maps logical page p to the slot's page p mod R, so positions more than W - 1 behind every query still to come are
 * overwritten.  A ring request takes no prefix-cache hit and its slots retain nothing; every other request pages and
 * caches as without a window.
 * RR_INVALID_ARGUMENT, before anything is queued and with *ticket untouched, for a NULL engine, prompt or ticket,
 * n_prompt or max_new_tokens below 1, n_prompt + max_new_tokens above ctx_max,
 * n_choices x min(ceil((n_prompt + max_new_tokens) / 64), R) x 64 above kv_cache_tokens (the request could never be
 * admitted; R as above, no limit without a window), a
 * prompt token outside [0, vocab), and for parameters outside these ranges (NaN is outside every range):
 * 1 <= n_choices <= max_batch; -1 <= top_logprobs <= 20; 0 <= temperature <= 2; 0 <= top_p <= 1; -2 <= penalties <= 2;
 * 0 <= n_bias <= 300 with non-null arrays when n_bias > 0, unique bias ids in [0, vocab) and -100 <= bias values <= 100;
 * 0 <= n_stop <= 4 sequences of 1..64 bytes with non-null arrays when n_stop > 0; response_format 0 or 1, and 1 only with
 * vocab >= 259 (some bytes have no token otherwise).  top_logprobs >= 0 and temperature > 0 need vocab <= 524288.
 * Stats: prefill_tokens counts the prompt once (over all its pieces), kv_copy_tokens grows by (n_choices - 1) x the prompt length,
 * generated_tokens counts every token produced, the ones a stop sequence cut included. */
int rr_engine_submit(rr_engine* e, const int32_t* prompt_ids, int n_prompt, int max_new_tokens, const rr_gen_params* p,
                     uint64_t* ticket);
/* rr_engine_submit that also scores the prompt when prompt_top >= 0 (-1: exactly rr_engine_submit).  Prompt logprobs
 * (OpenAI /v1/completions `echo` with `logprobs`): for every prompt position t >= 1 the logprob of prompt[t] given
 * prompt[0..t), and K = max(1, prompt_top) (logprob, id) pairs of the most likely tokens at t, ordered as rr_op_logprobs
 * orders them.  Position 0 has none.  The prefill chunks that hold the prompt run the last layer and lm_head
 * (RR_OUT_ROWMAJOR_F32) over its rows in prefill orientation, S = 1024 rows of fp32 logits at a time, then rr_op_logprobs'
 * kernels with the next prompt token as the target.  A long prompt scores each piece as it runs.  The generated tokens
 * and their logprobs are bit-identical to the request without scoring; with n_choices > 1 the prompt is scored once.  A
 * scoring request takes no prefix-cache hit (every row must reach lm_head), so rr_completion.n_cached is 0; it retains
 * its prompt like any other request.  The engine allocates the scoring buffers (S x vocab x 4 B of logits, about
 * 525 MB at vocab 128256, and 96 B per max_prefill_tokens row) with its first scoring request; if that fails, the scoring
 * requests end with RR_INTERNAL and the engine serves on.  Read the scores with rr_engine_prompt_logprobs before
 * rr_engine_wait.  RR_INVALID_ARGUMENT, before anything is queued, for whatever rr_engine_submit rejects, prompt_top
 * outside -1..20, and prompt_top >= 0 with vocab above 524288. */
int rr_engine_submit_scored(rr_engine* e, const int32_t* prompt_ids, int n_prompt, int max_new_tokens,
                            const rr_gen_params* p, int prompt_top, uint64_t* ticket);
/* Blocks like rr_engine_wait until the request is done, then copies its prompt logprobs WITHOUT consuming the ticket
 * (finish with rr_engine_wait): target_lp_out [n_prompt - 1] (entry t - 1: position t), lp_out / id_out
 * [n_prompt - 1][K] (each may be NULL).  Returns RR_OK, RR_TIMEOUT while in flight, the request's status when it did not
 * end RR_OK (a cancel, a failure: nothing is written), and RR_INVALID_ARGUMENT for a NULL engine, an unknown, consumed or
 * cancelled ticket and a request submitted without scoring. */
int rr_engine_prompt_logprobs(rr_engine* e, uint64_t ticket, double timeout_s, float* target_lp_out, float* lp_out,
                              int32_t* id_out);
/* Queue an embedding request (OpenAI /v1/embeddings): prefill the prompt, pool its last position's final-norm row
 * (rr_op_embed_pool: L2-normalised, fp32 [hidden]) and finish.  No decode row, no token.
 * - Admission: as a prompt.  It waits at the head of the queue for a free row and ceil(n_prompt / 64) pages (or the ring
 *   R of a windowed model, as in rr_engine_submit), goes into the chunk as one sequence, and a long prompt is prefilled in
 *   pieces with the usual decode step between them.  It takes prefix-cache hits and, on success, leaves its prompt
 *   retained, exactly as a generation request does.
 * - The chunk that holds its last piece gives it one embedding row after the chunk's tail rows: the trimmed last layer
 *   runs over both, lm_head and the logits tail over the tail rows only (a chunk of embedding rows only launches neither).
 *   Every kernel of the trimmed layer is row-independent, so generation requests in the same chunk get bit-identical
 *   tokens, logprobs and stop / JSON results, and the embedding does not depend on the chunk, the pieces, the prefix
 *   cache or the slot.
 * - After that chunk the request is done and its row free: it never enters the decode working set or changes the decode
 *   graph.  generated_tokens does not grow; prefill_tokens counts its prompt.  Cancellation, fail_prob and internal errors
 *   behave as for any request; the done hook reports 0 tokens.
 * - The engine allocates the embedding buffers (4 B x max_batch x hidden, device and pinned) with its first embedding row:
 *   an engine that never embeds allocates nothing for them.
 * Read the embedding with rr_engine_embedding, then finish with rr_engine_wait (0 tokens) or rr_engine_cancel.
 * RR_INVALID_ARGUMENT, before anything is queued, for a NULL engine / prompt / ticket, n_prompt below 1 or above ctx_max,
 * min(ceil(n_prompt / 64), R) x 64 above kv_cache_tokens and a prompt token outside [0, vocab). */
int rr_engine_submit_embed(rr_engine* e, const int32_t* prompt_ids, int n_prompt, uint64_t* ticket);
/* Blocks like rr_engine_prompt_logprobs until the request is done, then copies its embedding (fp32 [hidden]) into out
 * WITHOUT consuming the ticket (finish with rr_engine_wait, which reports 0 tokens); *dim_out = hidden (dim_out may be
 * NULL).  Same returns as rr_engine_prompt_logprobs; RR_INVALID_ARGUMENT also for a NULL out, capacity < hidden and a
 * request that is not an embedding. */
int rr_engine_embedding(rr_engine* e, uint64_t ticket, double timeout_s, float* out, int capacity, int* dim_out);
/* Block (release the GIL) until the request is done, or timeout_s (<= 0: no limit) elapses.  RR_TIMEOUT: still in flight
 * (out->status = RR_TIMEOUT), wait again or rr_engine_cancel.  Otherwise the ticket is consumed and the request's status
 * returned (RR_OK / RR_BACKEND_FAILED / ...), with `out` filled and for every choice c of its n_choices:
 *   n_tokens_out[c] = the tokens choice c returned, finish_out[c] = its finish reason (0 length, 1 stop);
 *   row c of tokens_out [n_choices][max_tokens_out] = its first min(n_tokens_out[c], max_tokens_out) tokens;
 *   with top_logprobs >= 0, row c of lp_out / id_out [n_choices][max_tokens_out][K] = their pairs (K as rr_engine_submit
 *   describes); nothing is written there for a request without logprobs.
 * tokens_out, lp_out, id_out, n_tokens_out and finish_out may each be NULL.  rr_completion.n_generated is the longest
 * choice's count.  RR_INVALID_ARGUMENT for a NULL engine or out, and for an unknown, consumed or cancelled ticket. */
int rr_engine_wait(rr_engine* e, uint64_t ticket, double timeout_s, rr_completion* out, int32_t* tokens_out,
                   int max_tokens_out, float* lp_out, int32_t* id_out, int32_t* n_tokens_out /* [n_choices] */,
                   int32_t* finish_out /* [n_choices] */);
/* Abandon a request: queued -> dropped; running -> its decode row is freed at the next step; finished -> freed.
 * Consumes the ticket (do not wait on it afterwards).  Replaces the client-side `timeout=` of the reference's
 * chat.completions.create calls (reference src/demo_fallback.py:146) as seen from the backend. */
int rr_engine_cancel(rr_engine* e, uint64_t ticket);
/* Streaming (SSE): block until the request shows more than `have` tokens, is done, or `timeout_s` elapses; then
 * *n_generated = the tokens shown, *done = 1 once the request is done, *t_first_token_s = its time to the first token, and
 * the first min(*n_generated, max_tokens_out) tokens go to tokens_out, with top_logprobs >= 0 their pairs to lp_out /
 * id_out [max_tokens_out][K] (tokens_out, t_first_token_s, lp_out and id_out may each be NULL).  Does not consume the
 * request: finish with rr_engine_wait.  While a request runs, a token is shown only once no stop sequence can take it back
 * (hold_out of rr_op_stop_match), so *n_generated never shrinks; a request that ends by length releases the held tokens
 * with its last ones.  After a cancel, an injected failure or an internal error the tokens shown so far are what is kept.
 * RR_INVALID_ARGUMENT for a NULL engine, n_generated or done, for a request of n_choices > 1 (it stays in flight) and for
 * an unknown or consumed ticket. */
int rr_engine_peek(rr_engine* e, uint64_t ticket, int have, double timeout_s, int32_t* tokens_out, int max_tokens_out,
                   int32_t* n_generated, int32_t* done, double* t_first_token_s, float* lp_out, int32_t* id_out);
/* Closed-batch convenience used by bench.py: submit all, wait all. prompts are host buffers
 * (pinned or pageable); the H2D copies happen inside. */
int rr_engine_run_batch(rr_engine* e, const int32_t* prompt_ids, const int32_t* prompt_start,
                        int n_requests, int max_new_tokens, rr_completion* out,
                        int32_t* tokens_out /* [n_requests, max_new_tokens] */);
double rr_engine_now(rr_engine* e);

typedef struct rr_engine_stats {
    uint64_t kernel_launches;     /* library kernels launched (graph replays count their nodes) */
    uint64_t decode_steps, prefill_chunks, prefill_tokens, generated_tokens;
    double decode_ms_total, prefill_ms_total;   /* CUDA-event time on the engine stream */
    int32_t active_rows, queued;
    uint64_t h2d_bytes, d2h_bytes;
    /* prefix_cache: requests that hit, prompt tokens they did not prefill, tokens copied between slots */
    uint64_t prefix_hits, prefix_cached_tokens, kv_copy_tokens;
} rr_engine_stats;
int rr_engine_get_stats(rr_engine* e, rr_engine_stats* out);
/* The KV page pool: *pages_total = kv_cache_tokens / 64, *pages_free = pages no slot holds.  A slot keeps the pages of its
 * retained prompt prefix (prefix_cache) after its request; otherwise every page is free once the engine is idle.
 * RR_INVALID_ARGUMENT for a NULL argument. */
int rr_engine_kv_usage(rr_engine* e, int32_t* pages_total, int32_t* pages_free);
int rr_engine_reset_stats(rr_engine* e);

/* ================================================================================================
 * 5. Gateway: the whole per-request path behind one submit / wait pair, in native code.
 *    Replaces the reference's gateway process as its clients see it: N concurrent blocking
 *    chat.completions.create calls (reference src/demo_load_balancing.py:195-203,
 *    src/demo_quota_isolation.py:135-139) into litellm's single worker (reference bin/start-gateway.sh:54).
 *    rr_gateway_submit is thread-safe and non-blocking: the request enters an admission queue; a dispatcher
 *    thread coalesces everything pending (ADMIT / DONE / FAIL / fallback re-ADMIT) into ONE ordered trace per
 *    K1 launch (rr_router_process) and hands admitted prompts straight to the engine of the picked
 *    deployment, or serves them itself on a mock replica (rr_stub_desc).  A backend failure walks the fallback chain
 *    inside the library. */

typedef struct rr_gateway rr_gateway;

typedef struct rr_gateway_opts {
    int32_t manual_clock;      /* 0: events are stamped with the wall clock (ms); 1: with rr_gateway_set_now() */
    int32_t record_trace;      /* keep the last N (event, decision) pairs for replay through an oracle; 0 = off */
    int32_t max_batch_events;  /* events per K1 launch, 0 = 4096 */
    int32_t reserved[5];
} rr_gateway_opts;

typedef struct rr_gateway_result {
    uint64_t ticket;
    int32_t status;            /* RR_OK / RR_RATE_LIMITED (429) / RR_NO_GROUP / RR_BACKEND_FAILED / RR_TIMEOUT / RR_CANCELLED / ...;
                                  -1 while in flight (rr_gateway_peek) */
    int32_t deployment, served_group, chain_pos, replica;   /* the admission decision (valid once admitted) */
    int32_t n_prompt, n_generated;
    int32_t attempts;          /* admissions this request went through (1 + backends that failed under it) */
    double t_submit_s, t_admit_s, t_first_token_s, t_done_s;   /* gateway monotonic clock, seconds */
    int32_t n_cached;          /* rr_completion.n_cached of the engine that served the request */
    int32_t finish;            /* choice 0's finish reason once finished: 0 length, 1 stop (rr_engine_wait) */
} rr_gateway_result;

typedef struct rr_gateway_stats {
    uint64_t submitted, admitted, completed, rate_limited, failed, failed_over;
    uint64_t launches;         /* K1 launches */
    uint64_t events;           /* events those launches processed */
    uint64_t max_batch;        /* largest trace of one launch */
    uint64_t in_flight;
    double admit_wait_s;       /* sum over admissions of (decision time - submit time) */
} rr_gateway_stats;

/* A mock-completion replica, served by the gateway itself in place of an engine.  The n-th request handed to it (n from 1,
 * per replica and gateway) fails without tokens when fail_every > 0 and n % fail_every == 0; any other completes with
 * min(max_new_tokens, reply_tokens) tokens 3 + (i % 200).  Generation parameters are ignored. */
typedef struct rr_stub_desc {
    int32_t reply_tokens, fail_every, vocab, reserved;
} rr_stub_desc;

/* engines[i] serves the deployments whose rr_deployment_desc.replica == replica_ids[i]; engines[i] == NULL makes that
 * replica a mock one described by stubs[i] (stubs is read only there and may be NULL when no engine is NULL).
 * RR_INVALID_ARGUMENT, with nothing created, for a NULL engine without a descriptor, reply_tokens < 0, fail_every < 0 or
 * vocab < 1.  A mock replica's vocab counts toward the smallest vocabulary; it sets no context or prefill limit.  A
 * gateway with a mock replica refuses logprobs, stop sequences and JSON mode at submit (rr_gateway_submit).  The router and
 * the engines must outlive the gateway; the engines' completion hooks are taken by the gateway until it is destroyed. */
int rr_gateway_create(rr_router* router, rr_engine* const* engines, const int32_t* replica_ids, int n_engines,
                      const rr_stub_desc* stubs, const rr_gateway_opts* opts, rr_gateway** out);
void rr_gateway_destroy(rr_gateway* g);
int rr_gateway_set_now(rr_gateway* g, int64_t now_ms);
/* Queue one request for model group `group` (index of the model_name the client asked for) and write its ticket to
 * *ticket.  p as rr_engine_submit describes it (NULL: greedy, one choice).  The parameters are stored with the request and
 * handed to every engine it is admitted to, a fallback re-admission included (all choices restart there), so a
 * re-admitted sampled request draws the same tokens on a replica with the same weights.  The request is one ADMIT event
 * (the prompt's tokens) and one DONE event carrying the tokens its choices return, whatever p holds.
 * Refusals, before anything is debited and with *ticket untouched, in this order: RR_INVALID_ARGUMENT for a NULL gateway
 * or for parameters rr_engine_submit rejects, bias ids and JSON mode judged against the smallest vocabulary of the
 * gateway's replicas (stop bytes need no vocabulary check); RR_INVALID_ARGUMENT when a mock replica is attached and p asks
 * for logprobs (top_logprobs >= 0), stop sequences (n_stop > 0) or JSON mode (response_format 1): a mock replica has no
 * logits to fill pairs from or to mask and no decode loop to cut; RR_INVALID_ARGUMENT for a NULL prompt or ticket;
 * RR_NO_GROUP for an unknown group; RR_INVALID_ARGUMENT (HTTP 400) for n_prompt or max_new_tokens below 1, n_choices
 * outside 1..the smallest max_batch of the gateway's engines (a mock replica sets no limit and replies with n_choices
 * copies of its reply), prompt + max_new_tokens beyond a replica's context,
 * n_choices x min(ceil((prompt + max_new_tokens) / 64), R) x 64 beyond the KV pool of any of the gateway's engines, R
 * that engine's ring (rr_engine_submit; no limit without a window; a mock replica sets no KV limit), and a bad token id. */
int rr_gateway_submit(rr_gateway* g, int group, const int32_t* prompt_ids, int n_prompt, int max_new_tokens,
                      const rr_gen_params* p, uint64_t* ticket);
/* rr_gateway_submit with prompt logprobs (rr_engine_submit_scored; prompt_top -1: exactly rr_gateway_submit).  Also
 * RR_INVALID_ARGUMENT, before anything is debited, for prompt_top outside -1..20, prompt_top >= 0 with a smallest
 * vocabulary that is not a multiple of 4, and prompt_top >= 0 with a mock replica attached.  A fallback re-admission
 * scores the prompt again on the new replica. */
int rr_gateway_submit_scored(rr_gateway* g, int group, const int32_t* prompt_ids, int n_prompt, int max_new_tokens,
                             const rr_gen_params* p, int prompt_top, uint64_t* ticket);
/* rr_engine_prompt_logprobs for a gateway ticket: blocks until the request is finished and copies the scores of the
 * replica that served it without consuming the ticket (finish with rr_gateway_wait).  Same buffers and returns. */
int rr_gateway_prompt_logprobs(rr_gateway* g, uint64_t ticket, double timeout_s, float* target_lp_out, float* lp_out,
                               int32_t* id_out);
/* An embedding request (rr_engine_submit_embed) through the gateway: one ADMIT event carrying its n_prompt tokens (the tpm
 * debit), and on success one DONE event with 0 completion tokens and the usual latency sample.  A backend failure walks
 * the fallback chain and the new replica prefills the prompt again.  Refusals in rr_gateway_submit's order and codes (a
 * prompt of up to the smallest context window, ceil(n_prompt / 64) pages per engine pool); RR_INVALID_ARGUMENT also with a
 * mock replica attached, which has no hidden state. */
int rr_gateway_submit_embed(rr_gateway* g, int group, const int32_t* prompt_ids, int n_prompt, uint64_t* ticket);
/* rr_engine_embedding for a gateway ticket: blocks until the request is finished and copies the embedding of the replica
 * that served it without consuming the ticket (finish with rr_gateway_wait); *dim_out = that replica's hidden size.  Same
 * returns as rr_gateway_prompt_logprobs; RR_INVALID_ARGUMENT also for a NULL out, capacity below the served embedding's
 * size and a request that is not an embedding. */
int rr_gateway_embedding(rr_gateway* g, uint64_t ticket, double timeout_s, float* out, int capacity, int* dim_out);
/* A closed burst of plain requests (greedy, one choice) as one contiguous block of the admission trace (declare_burst != 0
 * prepends RR_EV_BURST). */
int rr_gateway_submit_batch(rr_gateway* g, int group, const int32_t* prompt_ids, const int32_t* prompt_start, int n,
                            int max_new_tokens, int declare_burst, uint64_t* tickets);
/* Blocks (release the GIL) until the request is finished; returns its status and consumes the ticket.
 * RR_TIMEOUT: still in flight -- wait again or rr_gateway_cancel.  The buffers as rr_engine_wait fills them (each may be
 * NULL); a request that never reached a replica reports 0 tokens and reason 0 for every choice.
 * rr_gateway_result.n_generated is the longest choice's count and .finish choice 0's reason. */
int rr_gateway_wait(rr_gateway* g, uint64_t ticket, double timeout_s, rr_gateway_result* out, int32_t* tokens_out,
                    int max_tokens_out, float* lp_out, int32_t* id_out, int32_t* n_tokens_out /* [n_choices] */,
                    int32_t* finish_out /* [n_choices] */);
/* Streaming: returns once more than `have` tokens are shown, the request is finished, or timeout_s elapsed; the tokens
 * and pairs as rr_engine_peek shows them (a token a stop sequence may still take back is held), and `out` (may be NULL)
 * gets the request's record so far (status -1 while in flight).  RR_INVALID_ARGUMENT for a request of n_choices > 1. */
int rr_gateway_peek(rr_gateway* g, uint64_t ticket, int have, double timeout_s, int32_t* tokens_out, int max_tokens_out,
                    int32_t* n_generated, int32_t* done, rr_gateway_result* out, float* lp_out, int32_t* id_out);
/* Abandon a request (consumes the ticket).  count_as_failure != 0: a client-side timeout -- the deployment gets a FAIL
 * event (allowed_fails / cooldown, reference config/config.yaml:103-104); 0: a disconnect -- a DONE event. */
int rr_gateway_cancel(rr_gateway* g, uint64_t ticket, int count_as_failure);
/* Block until every event queued so far (the DONE / FAIL reports of finished requests included) has been through K1:
 * call before rr_router_snapshot when the counters must reflect all completed requests. */
int rr_gateway_quiesce(rr_gateway* g, double timeout_s);
int rr_gateway_get_stats(rr_gateway* g, rr_gateway_stats* out);
/* The recorded trace (opts.record_trace): *n pairs, oldest first. */
int rr_gateway_trace(rr_gateway* g, rr_event* events, rr_decision* decisions, int capacity, int* n);

#ifdef __cplusplus
}
#endif
#endif /* RR_B200_H */
