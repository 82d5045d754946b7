// rr_kernels.h — internal (C++) declarations shared by the .cu files of librr_b200.so.
// The public C-ABI is include/rr_b200.h; nothing here crosses the library boundary.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <vector>

#include "../../include/rr_b200.h"

namespace rr {

#define RR_ERR_ARG RR_INVALID_ARGUMENT
#define RR_ERR_CUDA RR_CUDA_ERROR

// ---- the KV cache address rule, the one formula every kernel that reads or writes the cache goes through.  A page holds P
// consecutive positions of one slot for every kv head, [page][kv_head][P][128] bf16 per layer for K and for V.  With a page
// table ([n_slots][pages_per_slot], the engine's layout) P = KV_PAGE and position pos of slot s lies on page
// table[s * pages_per_slot + pos / KV_PAGE]; without one (table == nullptr) P = ctx_max and the page is the slot, which is
// the slot-contiguous layout [slot][kv_head][ctx_max][128].  Table entries are trusted, like slot indices.
constexpr int KV_PAGE = 64;
__host__ __device__ __forceinline__ int kv_page(const int32_t* table, int pages_per_slot, int slot, int pos) {
    return table ? table[slot * pages_per_slot + pos / KV_PAGE] : slot;
}
// Row of (page, kv head, pos) in the [n_pages * n_kv_heads * P, 128] view of one layer's cache.
__host__ __device__ __forceinline__ long long kv_page_row(bool paged, int page, int n_kv_heads, int ctx_max, int kvh, int pos) {
    return paged ? ((long long)page * n_kv_heads + kvh) * KV_PAGE + (pos & (KV_PAGE - 1))
                 : ((long long)page * n_kv_heads + kvh) * ctx_max + pos;
}
__host__ __device__ __forceinline__ long long kv_row(const int32_t* table, int pages_per_slot, int n_kv_heads, int ctx_max,
                                                     int slot, int kvh, int pos) {
    return kv_page_row(table != nullptr, kv_page(table, pages_per_slot, slot, pos), n_kv_heads, ctx_max, kvh, pos);
}

enum GemmOutMode { OUT_ROWMAJOR_BF16 = 0, OUT_TRANSPOSED_F32 = 1, OUT_TRANSPOSED_SILU = 2, OUT_ROWMAJOR_SILU = 3,
                   OUT_ROWMAJOR_ROPE = 4, OUT_ROWMAJOR_RESID = 5, OUT_ROWMAJOR_F32 = 6 };
// OUT_ROWMAJOR_F32 (lm_head over the prompt rows of a scoring prefill chunk): out[a*ldo + b] = acc * rinv(a) as fp32, the
// deferred-norm consumer factor included.  fp32 because a logprob needs more than bf16's 8 bits near a logit of 20.
// OUT_ROWMAJOR_RESID (prefill O / down projections): out is the fp32 residual stream, out[a*ldo + b] += acc —
// the following norm kernel then only reads x and writes xn (half its bytes).

// OUT_ROWMAJOR_ROPE (prefill QKV projection, head_dim 128): the epilogue rotates q and k (RoPE table), writes q to q_out
// and appends k / v to the KV cache — no intermediate qkv matrix, no separate rope_kv launch.
struct RopeEpi {
    __nv_bfloat16* q_out;     // [T, n_heads*128]
    __nv_bfloat16* k_cache;   // [slot][kv_head][ctx_max][128]
    __nv_bfloat16* v_cache;
    const int32_t* slot;      // per token row
    const int32_t* pos;
    const float2* table;      // [ctx_max][64] (cos, sin)
    int n_heads, n_kv_heads, ctx_max;
    const int32_t* page_table = nullptr;   // KV address rule (kv_row): null = [slot][kv_head][ctx_max][128]
    int pages_per_slot = 0;
    // ---- deferred RMSNorm (prefill): the GEMM that writes the residual also emits the next GEMM's operand
    // xhat = bf16(x * gamma) (NOT normalised) and per-row partial sums of squares; the next GEMM scales its
    // accumulators by rsqrt(mean(x^2) + eps) of the row in its epilogue (the projection is linear).  No norm kernel,
    // no second pass over the fp32 residual.
    // consumer side (OUT_ROWMAJOR_ROPE / _SILU / _BF16):
    const float* rowss;       // [rowsA][n_part] partial sum(x^2) of the operand rows; n_part = 0: operand is normalised
    int n_part;
    float inv_hidden, eps;
    // producer side (OUT_ROWMAJOR_RESID): xhat = nullptr -> plain residual add
    const __nv_bfloat16* gamma;   // [rowsB] norm weight of the NEXT norm
    __nv_bfloat16* xhat;          // [rowsA][ldo]
    float* rowss_out;             // [rowsA][n_part_out], column = this item's b_tile
    int n_part_out;
};

// Widest GEMM tile along B rows: a consumer warpgroup holds 128 x MAX_BN fp32 accumulators in registers, 2 x 64 per thread
// at 128.  Wider decode batches (up to MAX_BATCH rows, rr_engine_opts.max_batch) run several batch tiles per weight tile.
constexpr int MAX_BN = 128;
constexpr int MAX_BATCH = 256;

struct GemmPlan {
    CUtensorMap tmA, tmB;
    void* out;
    int rowsA, rowsB, K, splits, ldo, ld_rows, mode, bn, max_ctas;
    RopeEpi rope;             // OUT_ROWMAJOR_ROPE only
    CUtensorMap tmOut;        // OUT_TRANSPOSED_F32: planes [splits][rowsB][rowsA] (3-D, box {128, bn, 1}) for the TMA-store epilogue
    int tma_epi;              // 1: the epilogue stages the tile in shared memory and issues ONE TMA store per item
    const float* scaleA;      // FP8 weights (gemm_plan_init_fp8w): A is e4m3 [rowsA, K] with one power-of-two scale per row
};

// ---- prefill decisions shared by the engine (init_pf_plans, run_prefill) and the kernel-level entry points (rr_api.cu)
// RoPE and the KV append run in the QKV GEMM's epilogue (OUT_ROWMAJOR_ROPE) only at head_dim 128, where a head is half of a
// 256-wide tile; other head dims take OUT_ROWMAJOR_BF16 into a qkv matrix, then rope_kv_kernel.
inline bool pf_rope_fused(int head_dim) { return head_dim == 128; }
// Deferred RMSNorm: the OUT_ROWMAJOR_RESID epilogue writes one partial sum(x^2) per 128 columns of the residual.
constexpr int PF_NORM_COLS = 128;
inline int pf_norm_parts(int hidden) { return (hidden + PF_NORM_COLS - 1) / PF_NORM_COLS; }
// Consumer side (QKV, gate/up): scale the accumulators of row r by rsqrt(sum(rowss[r][0..n_part)) / hidden + eps).
inline void pf_norm_consumer(RopeEpi* r, const float* rowss, int hidden, float eps) {
    r->rowss = rowss; r->n_part = pf_norm_parts(hidden); r->inv_hidden = 1.0f / (float)hidden; r->eps = eps;
}
// Producer side (O, down): also write xhat = bf16(x * gamma) and rowss_out[r][0..pf_norm_parts(hidden)).
inline void pf_norm_producer(RopeEpi* r, const __nv_bfloat16* gamma, __nv_bfloat16* xhat, float* rowss_out, int hidden) {
    r->gamma = gamma; r->xhat = xhat; r->rowss_out = rowss_out; r->n_part_out = pf_norm_parts(hidden);
}

int num_sms();

// ---- engine / router internals used by the native gateway (rr_gateway.cu)
typedef void (*EngineDoneHook)(void* ctx, uint64_t tag, uint64_t ticket, int status, int n_generated);
// What a request asks the decoder to do (an rr_gen_params of rr_engine_submit / rr_gateway_submit, less n_choices; the
// defaults are a plain greedy request).  The gateway hands it unchanged to every engine the request is admitted to.
struct GenParams {
    int top_lp = -1;                  // -1: no logprobs, else max(1, top_lp) (logprob, id) pairs per token
    float temp = 0.f, top_p = 1.f;    // temp > 0 draws every token with rr_op_sample
    uint64_t seed = 0;
    float fpen = 0.f, ppen = 0.f;     // frequency / presence penalties over the generated tokens, and a logit bias, applied
    std::vector<int32_t> bias_id;     // to the logits before the token is picked (rr_op_logit_penalties)
    std::vector<float> bias_val;
    bool logprobs() const { return top_lp >= 0; }
    bool sampled() const { return temp > 0.f; }
    bool processed() const { return fpen != 0.f || ppen != 0.f || !bias_id.empty(); }
    // stop sequences (rr_op_stop_match): n_stop of them, sequence i = stop[i][0 .. stop_len[i]) bytes of reply text
    int n_stop = 0;
    uint8_t stop_len[4] = {};
    uint8_t stop[4][64] = {};
    bool stops() const { return n_stop > 0; }
    // response format: 0 text, 1 json_object (every token is masked to the JSON grammar, rr_op_json_mask)
    int fmt = 0;
    bool json() const { return fmt == 1; }
    // pairs per token of a logprobs request: max(1, top_lp), plus the sampled token's own pair in the last column
    int lp_width() const { return (top_lp > 1 ? top_lp : 1) + (sampled() ? 1 : 0); }
    // prompt logprobs (rr_engine_submit_scored): -1 off, else every prompt token t >= 1 gets its own logprob given the
    // tokens before it and max(1, prompt_top) (logprob, id) pairs.  Not part of rr_gen_params: set() leaves it at -1.
    int prompt_top = -1;
    bool scores() const { return prompt_top >= 0; }
    int score_width() const { return prompt_top > 1 ? prompt_top : 1; }
    // The raw C struct (NULL: the defaults), checked before anything is stored: -1 <= top_logprobs <= LP_MAX_TOP and
    // OpenAI's ranges 0 <= temperature <= 2, 0 <= top_p <= 1, -2 <= penalties <= 2, 0 <= n_bias <= PEN_MAX_BIAS (non-null
    // arrays when n_bias > 0), bias ids unique and in [0, vocab), -100 <= bias values <= 100; NaN fails; 0 <= n_stop <=
    // STOP_MAX_SEQS sequences of 1..STOP_MAX_LEN bytes each, sequence i = stop_bytes[stop_off[i] .. stop_off[i + 1])
    // (non-null arrays when n_stop > 0); response_format 0 or 1, and 1 only with vocab >= JSON_MIN_VOCAB.  n_choices is
    // the caller's to check.  A greedy request keeps the default top_p and seed, an unprocessed one the default penalties.
    // RR_INVALID_ARGUMENT (nothing stored) or RR_OK.
    int set(int vocab, const rr_gen_params* p);
};
// n_choices (1..max_batch): choices of the request (rr_gen_params.n_choices); the done hook's n_generated is the total of
// the tokens the choices return (a choice cut by a stop sequence counts what is left of it).
int engine_submit_tagged(rr_engine* e, const int32_t* prompt_ids, int n_prompt, int max_new_tokens, uint64_t tag,
                         uint64_t* ticket, const GenParams& p, int n_choices);
// An embedding request (rr_engine_submit_embed) with the done hook's `tag`; the hook reports 0 tokens.
int engine_submit_embed_tagged(rr_engine* e, const int32_t* prompt_ids, int n_prompt, uint64_t tag, uint64_t* ticket);
void engine_set_done_hook(rr_engine* e, EngineDoneHook fn, void* ctx);
// kv_tokens: the KV pool (rr_engine_opts.kv_cache_tokens after its default is applied)
// ring: the pages a windowed engine's ring request reserves per choice (0: no window, every choice reserves its reach)
// hidden: the model's hidden size, the length of its embeddings
int engine_limits(const rr_engine* e, int* ctx_max, int* vocab, int* max_batch, int* kv_tokens = nullptr,
                  int* ring = nullptr, int* hidden = nullptr);
int router_shape(const rr_router* r, int* n_deployments, int* n_groups);
int router_dep_replica(const rr_router* r, int deployment);
int router_strategy(const rr_router* r);
int make_tmap_bf16_2d(CUtensorMap* map, const void* base, int rows, int K, int ld, int box_rows);
int gemm_plan_init(GemmPlan* p, const void* A, int rowsA, int ldA, const void* B, int rowsB, int ldB,
                   int K, void* out, int ldo, int ld_rows, int splits, int mode, int bn);
// Decode orientation (OUT_TRANSPOSED_F32 / _SILU) on an e4m3 weight A [rowsA, K] (row pitch ldA bytes) with scale[rowsA]:
// the same tiles, splits, k order and epilogues as gemm_plan_init on D = bf16(A * scale), so the same bits.  RR_ERR_ARG
// for another mode, a null scale, or an A the TMA cannot stream (16-byte aligned base and pitch, K % 16 == 0).
int gemm_plan_init_fp8w(GemmPlan* p, const void* A, const float* scale, int rowsA, int ldA, const void* B, int rowsB,
                        int ldB, int K, void* out, int ldo, int ld_rows, int splits, int mode, int bn);
// pdl = false: a plain stream-ordered launch (the first GEMM after the prefill dequantize, rr_fp8.cu)
int gemm_launch(const GemmPlan& p, cudaStream_t st, bool pdl = true);

// ---- FP8 weights (rr_fp8.cu)
// An e4m3 weight the decode GEMMs can stream: non-null, 16-byte aligned, K a positive multiple of 16.
bool fp8_weight_ok(const void* q, int K);
// Per-row quantizer (rr_op_quantize_fp8_weight); a row with Inf or NaN sets *bad and writes nothing.
int launch_quantize_fp8(const __nv_bfloat16* w, int rows, int K, int ld, uint8_t* q, float* scale, int* bad, cudaStream_t st);
struct Fp8DequantJob {
    const uint8_t* q;         // [rows, K] e4m3
    const float* scale;       // [rows]
    __nv_bfloat16* out;       // [rows, ld_out]
    int rows, K, ld_out;
};
struct Fp8DequantJobs {       // up to four matrices in one launch (a layer's wqkv, wo, wgu, wdown)
    Fp8DequantJob job[4];
    long long end[4];         // cumulative 16-byte chunks
    int n = 0;
};
void fp8_dequant_job(Fp8DequantJobs* J, const void* q, const float* scale, int rows, int K, __nv_bfloat16* out, int ld_out);
// out = bf16(q * scale) for every job, as a plain stream-ordered launch that does not trigger its dependents.
int launch_dequantize_fp8(const Fp8DequantJobs& J, cudaStream_t st);

// ---- fused decode MLP (rr_gemm.cu): gate/up GEMM (+SiLU*mul) and down GEMM in one persistent launch.
// Per-CTA work lists (built once on the host) replace the kernel boundary: a down item covers one K-slice of
// `slice_kb` k-blocks = the act columns written by `slice_kb` gate/up tiles, and waits for `ready[slice]` to reach
// that count instead of for the whole gate/up grid.
struct MlpItem {             // 16 bytes, read as int4
    int tile_phase;           // a_tile | phase << 16 (phase 0 = gate/up, 1 = down); -1 terminates the list
    int kb0, kb1;             // k-block range
    int z;                    // down: output plane = K-slice index (also the index into `ready`)
};
struct MlpArgs {
    CUtensorMap tmA0, tmB0;   // gate/up: weights [2*inter, hidden] (64-row interleaved), activations xn [rows, hidden]
    CUtensorMap tmA1, tmB1;   // down: weights [hidden, inter], activations act [rows, inter]
    __nv_bfloat16* act;       // [rows, inter]
    float* out1;              // planes [n_slices][ld_rows][hidden]
    int inter, hidden, rows, ld_rows;
    const MlpItem* items;     // [grid][max_items]
    int max_items;
    unsigned* ready;          // [n_slices + 1], zero at launch; the last word is the dynamic down-item counter
    int slice_kb;
    int dyn, n_down, tiles1, kb1n, n_slices;   // dyn: down items drawn from ready[n_slices] in slice-major order (not in `items`)
    CUtensorMap tmAct, tmPlanes;   // TMA-store epilogues: act [rows][inter] bf16 (box {64, bn}), planes (3-D, box {128, bn, 1})
    int tma_epi;
    const float* sc0;         // FP8 weights: the e4m3 rows' scales of Wgu (interleaved like its rows) and of Wd
    const float* sc1;
};
struct MlpPlan {
    MlpArgs args;
    int grid, bn, n_slices, fp8;
};
// Decode tile width along the batch rows: the narrowest of 16 / 32 / 64 / MAX_BN that holds `rows`; wider batches run
// several MAX_BN tiles per weight tile.
int pick_bn(int rows);
// Split-K planes of a decode projection W [rows_w, K]: enough (128-row weight tile, plane) items for one per SM, at most 8
// planes and at least 8 k-blocks of 64 in each (engine.py mirrors this rule to decide the gate/up layout).
int pick_splits(int rows_w, int K);
// One decode projection as the engine plans it for a working set of `rows` decode rows (its max_batch): out = W . X^T in
// `mode` (OUT_TRANSPOSED_F32 / _SILU), X [rows, K] bf16, W [rows_w, K] bf16 or, with scale, e4m3 (gemm_plan_init_fp8w);
// tile width pick_bn(rows), plane pitch rows, `splits` planes of row pitch ldo.
int decode_plan_init(GemmPlan* p, const void* W, const float* scale, int rows_w, int K, const void* X, int rows, void* out,
                     int ldo, int splits, int mode);
// K slices of the fused MLP's down GEMM: its inter / 64 k-blocks in at most 8 slices of about 16 (one output plane each;
// 8 x 28 k-blocks for Llama-3-8B balances the per-CTA lists to within 5 %, see mlp_schedule).  Sets *slice_kb and
// returns the number of slices (0 when inter < 64).
int mlp_slices(int inter, int* slice_kb);
// KV splits of decode attention (rr_attn_decode.cu): one CTA per (row, kv head) as long as that grid fills the GPU twice;
// otherwise each row's KV range is split over 2, 4 or 8 CTAs, merged by decode_attn_combine_kernel.
int pick_kv_splits(int rows, int n_kv_heads);
// Host schedule: `items` gets grid * max_items entries (CTA-major); returns max_items.
int mlp_schedule(int grid, int inter, int hidden, int slice_kb, std::vector<MlpItem>* items, int dynamic = 0);
int mlp_plan_init(MlpPlan* p, const void* Wgu, const void* Wd, int inter, int hidden, const void* xn, int rows,
                  void* act, void* planes, int ld_rows, int bn, const MlpItem* items_dev, int max_items, int grid,
                  unsigned* ready, int slice_kb, int dynamic = 0, const float* sc_gu = nullptr, const float* sc_down = nullptr);
int mlp_launch(const MlpPlan& p, cudaStream_t st);

// ---- elementwise / normalisation (rr_elementwise.cu) -------------------------------------------
// `part` inputs are the GEMM outputs: either fp32 split-K partials P[z][row][col] (n_splits >= 1,
// part_is_bf16 = 0, split stride = split_stride elements) or a single bf16 matrix.
struct PartIn {
    const void* ptr;
    int is_bf16;
    int n_splits;
    long long split_stride;   // elements between split planes
    int ld;                   // row pitch in elements
};

void launch_embed(const int32_t* ids, const __nv_bfloat16* table, float* x, int rows, int hidden,
                  const int32_t* row_active, cudaStream_t st);
// Embedding pool (rr_op_embed_pool): for i < n, out[i][0..hidden) = v / ||v||_2 with v = float(xn[rows ? rows[i] : i]),
// the sum of squares in fp64 in a fixed order, each quotient in fp64 rounded once to fp32; a zero row gives zeros.  One CTA
// per row, 16-byte loads (xn 16-byte aligned, ld % 8 == 0, hidden % 8 == 0).
void launch_embed_pool(const __nv_bfloat16* xn, int ld, const int32_t* rows, int n, int hidden, float* out, int out_ld,
                       cudaStream_t st);
// x[row] (+)= sum_z part[z][row]; xn[row] = rmsnorm(x[row]) * w   (part.ptr may be null: norm only)
// `zero` (optional): zero_n dependency counters reset by the kernel (the fused MLP kernel that follows it).
void launch_add_rmsnorm(float* x, PartIn part, const __nv_bfloat16* w, __nv_bfloat16* xn, int rows,
                        int hidden, float eps, cudaStream_t st, unsigned* zero = nullptr, int zero_n = 0);
// The same in place over the rows of a prefill chunk (no partials), with a kernel chosen by the hidden size only: the row
// count never changes a row's bits.
// `rowss_out` (optional, deferred norm): write xn = bf16(x * w) UN-normalised and rowss_out[row][0] = sum(x^2),
// rowss_out[row][1 .. n_part_out) = 0 -- the layout the OUT_ROWMAJOR_RESID epilogue produces (RopeEpi).
void launch_add_rmsnorm_pf(float* x, const __nv_bfloat16* w, __nv_bfloat16* xn, int rows, int hidden, float eps,
                           cudaStream_t st, float* rowss_out = nullptr, int n_part_out = 0);
// act[row, j] = silu(gate[row, j]) * up[row, j]; gate = cols [0, inter), up = cols [inter, 2*inter)
void launch_silu_mul(PartIn gu, __nv_bfloat16* act, int rows, int inter, cudaStream_t st);
// qkv (partials) -> RoPE(q), RoPE(k); q -> q_out [rows, n_heads*128] bf16; k, v -> KV cache.
struct RopeArgs {
    PartIn qkv;
    __nv_bfloat16* q_out;
    __nv_bfloat16* k_cache;   // [slot][kv_head][ctx_max][128]
    __nv_bfloat16* v_cache;
    const int32_t* slot;      // per row: KV slot (or -1 = skip)
    const int32_t* pos;       // per row: position
    int rows, n_heads, n_kv_heads, ctx_max;
    float theta;
    const float2* table;      // [ctx_max][64] (cos, sin) or null: compute inline
    int head_dim;             // true head dim (<= 128, % 8 == 0): column stride inside qkv; q_out / caches are padded to 128
    const int32_t* page_table = nullptr;   // KV address rule (kv_row)
    int pages_per_slot = 0;
};
void launch_rope_kv(const RopeArgs& a, cudaStream_t st);
void launch_rope_table(float2* table, int ctx_max, float theta, int head_dim, cudaStream_t st);
// argmax over fp32 logits [rows, vocab] (partials with n_splits = 1); writes next token, and if
// advance != 0: pos[row]++ (decode bookkeeping folded into the same launch).
void launch_argmax(PartIn logits, int rows, int vocab, int32_t* out_tok, float* out_val,
                   const int32_t* row_active, int32_t* pos_inc, cudaStream_t st);
// log-softmax + top-k over fp32 logits [rows][ld] (ld % 4 == 0, vocab <= ld): rows with top_n[r] >= 0 get
// k = min(max(1, top_n[r]), max_top) entries lp_out[r][j] = x - logsumexp(x), id_out[r][j], ordered by (value desc, id asc);
// other rows and entries j >= k are not written.  Two launches: LP_CHUNK-column chunks of every row in parallel, then one
// merge CTA per row.  ws = logprobs_ws_bytes(rows, vocab) of scratch, no initialisation needed.
constexpr int LP_MAX_TOP = 20;        // OpenAI's limit for top_logprobs
constexpr int LP_CHUNK = 8192;        // columns per chunk CTA (staged in 32 KB of shared memory)
constexpr int LP_MAX_CHUNKS = 64;     // vocab <= 64 * 8192 = 524288
constexpr int LP_LAUNCHES = 2;
size_t logprobs_ws_bytes(int rows, int vocab);
// tok (optional): also tok_lp[r] = x[tok[r]] - logsumexp(x) for those rows (a sampled token's own logprob).
void launch_logprobs(const float* logits, int ld, int rows, int vocab, const int32_t* top_n, int max_top, void* ws,
                     float* lp_out, int32_t* id_out, cudaStream_t st, const int32_t* tok = nullptr,
                     float* tok_lp = nullptr);
// Seeded temperature / top-p draw (rr_op_sample) over fp32 logits [rows][ld], same shape limits as launch_logprobs: rows
// with temperature[r] > 0 get out_tok[r], the others are not touched.  ws = sample_ws_bytes(rows, vocab) of scratch.
constexpr int SAMPLE_LAUNCHES = 3;
size_t sample_ws_bytes(int rows, int vocab);
void launch_sample(const float* logits, int ld, int rows, int vocab, const float* temperature, const float* top_p,
                   const uint64_t* seed, const int32_t* position, int32_t* out_tok, void* ws, cudaStream_t st);
// Frequency / presence penalties and logit bias (rr_op_logit_penalties), in place over fp32 logits [rows][ld], one launch.
// Per row r: freq[r], pres[r], n_bias[r] entries of bias_ids / bias_vals (row stride bias_ld, ids unique).  History: row r's
// generated tokens at hist + r * hist_ld, hist_len[r] of them; or, in the engine's decode step (app_tok set), the kernel
// first stores app_tok[r] at index app_pos[r] - gen0[r] and takes that index + 1 as the length.  A row with both penalties
// 0 and no bias entries is not touched.  cnt_ws: [rows][vocab] int32, all zero on entry and left all zero.
constexpr int PEN_MAX_BIAS = 300;
struct PenaltyArgs {
    const float *freq, *pres;
    const int32_t *bias_ids, *n_bias;
    const float* bias_vals;
    int bias_ld;
    int32_t* hist;                   // nullptr: no history (prefill: c = 0 for every token)
    int hist_ld;
    const int32_t* hist_len;
    const int32_t *app_tok, *app_pos, *gen0;
};
void launch_logit_penalties(float* logits, int ld, int rows, int vocab, const PenaltyArgs& a, int32_t* cnt_ws,
                            cudaStream_t st);
// Stop sequences (rr_op_stop_match), one launch, one warp per row.  Row r has n_stop[r] sequences (0: the row is skipped and
// its outputs are not written), sequence s = bytes[r][s][0 .. len[r][s]).  The kernel stores tok[r] (the token just picked)
// in the row's history (hist + (hist_row ? hist_row[r] : r) * hist_ld) at index i = position[r] - gen0[r] (position null:
// i = 0) and matches the reply text of history[0 .. i] (token t >= 3 is the byte (t - 3) % 256, t < 3 is no text):
//   cut[r]  = -1, or when the text now ends in a sequence and tok[r] has a byte: the history index of the first token of the
//             longest such sequence (= the tokens to keep)
//   hold[r] = 0 on a hit, else the tokens from the first token of the longest text suffix that is a proper prefix of some
//             sequence up to tok[r] (0: no such suffix)
// Rows with row_active[r] < 0 (row_active optional) are skipped like rows without sequences.
constexpr int STOP_MAX_SEQS = 4;
constexpr int STOP_MAX_LEN = 64;
struct StopArgs {
    const int32_t *n_stop, *gen0;
    const uint8_t* len;              // [rows][STOP_MAX_SEQS]
    const uint8_t* bytes;            // [rows][STOP_MAX_SEQS][STOP_MAX_LEN]
    int32_t* hist;
    int hist_ld;
    const int32_t *hist_row, *tok, *position, *row_active;
    int32_t *cut, *hold;
};
void launch_stop_match(const StopArgs& a, int rows, cudaStream_t st);
// JSON mode (response_format json_object, rr_op_json_mask / rr_op_json_advance).  Each row has an opaque 16-byte state of
// a byte-level automaton for a JSON text whose top-level value is an object (RFC 8259, strict UTF-8 in strings, at most
// JSON_MAX_DEPTH open containers, whitespace runs of at most JSON_MAX_WS bytes); all zero is the initial state.  Token
// t >= 3 is the byte (t - 3) % 256; tokens 0..2 are never allowed.  Rows with fmt[r] == 0 or row_active[r] < 0
// (row_active optional) are skipped by both kernels.
//   mask:    one CTA per (LP_CHUNK columns, row): tests each byte against state[r] (null: the initial state) and writes
//            -inf to every disallowed column of the chunk; it never reads the logits.
//   advance: one thread per row: next = step(state[r] (null: initial), byte of tok[r]) into state_out[out_row ? out_row[r]
//            : r], and done[r] = 1 when the new state is past the top-level object's close, else 0.  A token the state
//            does not allow leaves it unchanged.
constexpr int JSON_MAX_DEPTH = 64;
constexpr int JSON_MAX_WS = 64;
constexpr int JSON_MIN_VOCAB = 259;   // every byte has a token
struct JsonState {
    uint64_t stack;                   // bit l: container at level l is an array (1) or an object (0)
    uint32_t w0;                      // node | depth << 8 | whitespace run << 16 | string-is-a-key << 24
    uint32_t w1;                      // literal / escape / \u-hex / UTF-8 progress of the node
};
static_assert(sizeof(JsonState) == 16, "JsonState is 16 bytes");
constexpr int JSON_LAUNCHES = 2;
void launch_json_mask(float* logits, int ld, int rows, int vocab, const int32_t* fmt, const int32_t* row_active,
                      const JsonState* state, cudaStream_t st);
void launch_json_advance(int rows, const int32_t* fmt, const int32_t* row_active, const int32_t* tok,
                         const JsonState* state_in, JsonState* state_out, const int32_t* out_row, int32_t* done,
                         cudaStream_t st);

// ---- attention (rr_attn_decode.cu, rr_attn_tc.cu) ---------------------------------------------------
struct DecodeAttnArgs {
    const __nv_bfloat16* q;   // [rows, n_heads*128]
    const __nv_bfloat16* k_cache;
    const __nv_bfloat16* v_cache;
    __nv_bfloat16* out;       // [rows, n_heads*128]
    const int32_t* slot;      // per row
    const int32_t* pos;       // per row: position of the current token (ctx = pos + 1)
    int rows, n_heads, n_kv_heads, ctx_max;
    float scale;
    float* ws;                // split-KV workspace (may be null when kv_splits == 1)
    int kv_splits;
    CUtensorMap tmK, tmV;     // [n_slots*n_kv_heads*ctx_max, 128] views of the caches, box {64, 64}, SW128
    CUtensorMap tmK16, tmV16; // same views, box {64, 16}: the last tile of a row is requested in 16-row pieces
    int trim_tail;
    // fused RoPE + KV append (decode): q/k/v of the current token come straight from the QKV GEMM's
    // split-K planes; q is rotated into the MMA fragments, k/v are rotated, appended to the cache and
    // patched into the staged tile.  fuse_rope == 0: `q` holds rotated bf16 queries (rope_kv_kernel ran).
    int fuse_rope;
    PartIn qkv;
    const float2* rope_table;
    int head_dim;             // true head dim: qkv column stride and `out` head stride; q / caches padded to 128
    // KV address rule (kv_row).  The page table changes only between launches, like slot and pos: the producer reads the
    // pages of its tiles before the PDL wait.
    const int32_t* page_table = nullptr;
    int pages_per_slot = 0;
    // sliding window W (0: full causal): the row at pos attends to max(0, pos - W + 1) .. pos, its tiles split from that
    // key's tile on
    int window = 0;
};
// Fills tmK / tmV (ctx_max % 64 == 0) over n_pages pages: n_slots without a page table.
int decode_attn_make_maps(DecodeAttnArgs* a, int n_pages);
void launch_decode_attn(const DecodeAttnArgs& a, cudaStream_t st);
size_t decode_attn_ws_bytes(int rows, int n_heads, int kv_splits);

struct PrefillAttnArgs {
    const __nv_bfloat16* q;   // [T, n_heads*128] (RoPE applied)
    const __nv_bfloat16* k_cache;
    const __nv_bfloat16* v_cache;
    __nv_bfloat16* out;       // [T, n_heads*head_dim]
    const int32_t* seq_start; // [n_seqs+1] token offsets into T
    const int32_t* seq_slot;  // [n_seqs]
    const int32_t* seq_pos0 = nullptr;   // [n_seqs] position of each sequence's first query row (cached prefix); null: all 0
    int n_seqs, max_len, n_heads, n_kv_heads, ctx_max;   // max_len: longest sequence (suffix) in rows
    float scale;
    int head_dim;             // true head dim: `out` head stride; q / caches padded to 128
    int has_maps = 0;         // tmQ/tmK/tmV valid (prefill_attn_make_maps): required
    CUtensorMap tmQ, tmK, tmV;
    const int32_t* page_table = nullptr;   // KV address rule (kv_row): the producer looks up the page of each key tile
    int pages_per_slot = 0;
    int window = 0;           // sliding window W (0: full causal): query position q attends to max(0, q - W + 1) .. q
};
int launch_prefill_attn(const PrefillAttnArgs& a, cudaStream_t st);   // RR_ERR_ARG when the maps are missing / shape unsupported
// wgmma kernel (rr_attn_tc.cu): one (sequence, head, 128-row query tile) per work item.
int prefill_attn_make_maps(PrefillAttnArgs* a, long long q_rows, long long kv_rows);
bool prefill_attn_tc_eligible(const PrefillAttnArgs& a);
int launch_prefill_attn_tc(const PrefillAttnArgs& a, cudaStream_t st);
// Prefill attention as the engine launches it, in two parts.  Per layer (rr_engine_create): the operands, the true head
// dim and its scale 1 / sqrt(head_dim), the page table, the window, and the TMA maps: q over q_rows rows (the engine's Tmax,
// so a chunk of T < q_rows rows loads stale q rows into its last query tile; their outputs are never written) and each
// cache over n_pages pages (slots without a page table).  Per chunk (run_prefill): `out` [T][n_heads * head_dim] and the
// chunk's sequences.
inline int pf_attn_layer(PrefillAttnArgs* a, const __nv_bfloat16* q, const __nv_bfloat16* k_cache, const __nv_bfloat16* v_cache,
                         int n_heads, int n_kv_heads, int head_dim, int ctx_max, const int32_t* page_table, int pages_per_slot,
                         int n_pages, int window, long long q_rows) {
    a->q = q; a->k_cache = k_cache; a->v_cache = v_cache;
    a->n_heads = n_heads; a->n_kv_heads = n_kv_heads; a->ctx_max = ctx_max;
    a->head_dim = head_dim; a->scale = 1.0f / sqrtf((float)head_dim);
    a->page_table = page_table; a->pages_per_slot = pages_per_slot; a->window = window;
    return prefill_attn_make_maps(a, q_rows, (long long)n_pages * n_kv_heads * (page_table ? KV_PAGE : ctx_max));
}
inline void pf_attn_chunk(PrefillAttnArgs* a, __nv_bfloat16* out, const int32_t* seq_start, const int32_t* seq_slot,
                          const int32_t* seq_pos0, int n_seqs, int max_len) {
    a->out = out; a->seq_start = seq_start; a->seq_slot = seq_slot; a->seq_pos0 = seq_pos0;
    a->n_seqs = n_seqs; a->max_len = max_len;
}

// ---- the prefill chunk's hand-off to decode (rr_engine.cu, run_prefill; rr_op_gather_last / rr_op_activate_rows)
// Rows of the trimmed last layer: attn_out[r][0..nq) = attn[last[r]][..] and x_out[r][0..hidden) = x[last[r]][..] for
// r < n_rows, one CTA per row, 16-byte loads and stores (nq % 8 == 0, hidden % 4 == 0, 16-byte aligned buffers).
void launch_gather_last(const __nv_bfloat16* attn, const float* x, const int32_t* last, int n_rows, int nq, int hidden,
                        __nv_bfloat16* attn_out, float* x_out, cudaStream_t st);
// Tail row i < n becomes a live decode row in slot s = seq_slot[i]: d_tok[s] = first_tok[i], d_pos[s] = tok_pos[last[i]] + 1,
// d_slot[s] = s.  Nothing else of d_tok / d_pos / d_slot is written.
void launch_activate_rows(const int32_t* seq_slot, const int32_t* first_tok, const int32_t* tok_pos, const int32_t* last,
                          int n, int32_t* d_tok, int32_t* d_pos, int32_t* d_slot, cudaStream_t st);

// ---- prompt prefix caching (rr_kv_copy.cu): positions [0, n[i]) of slot src[i] -> slot dst[i], every layer and kv head,
// K and V, one launch for the whole list (passed by value as a kernel parameter).  Each layer's cache is layer_rows rows of
// 128 (n_pages * n_kv_heads * P); positions are addressed by kv_row through page_table (null: slot-contiguous).
constexpr int KV_COPY_MAX = 256;      // = the largest max_batch
struct KvCopyList {
    int32_t src[KV_COPY_MAX], dst[KV_COPY_MAX], n[KV_COPY_MAX];
    int count;
};
// RR_ERR_ARG unless 1 <= count <= KV_COPY_MAX, every slot is in [0, n_slots), every n in [1, ctx_max], no destination
// repeats and no destination is also a source.
int kv_copy_check(const KvCopyList& c, int n_slots, int ctx_max);
int launch_kv_copy(__nv_bfloat16* k_cache, __nv_bfloat16* v_cache, int n_layers, long long layer_rows, int n_kv_heads,
                   int ctx_max, const int32_t* page_table, int pages_per_slot, const KvCopyList& c, cudaStream_t st);

}  // namespace rr
