// rr_engine.cu — one model replica on one GPU: chunked prefill + continuous-batching greedy decode.
//
// Replaces one `litellm_params.model: bedrock/...` deployment of the reference
// (config/config.yaml:39,47,54,62,69,77,84,91) and the remote bedrock:InvokeModel call behind it
// (iam/policy.json:8, src/demo_cris.py:233-238).  The request-facing call shape
// (submit -> wait -> tokens + timestamps) is what chat.completions.create needs
// (src/demo_load_balancing.py:106-116).
//
// Layout in HBM (one replica): bf16 weights (caller-owned), a paged KV cache [layer][page][kv_head][64][128] bf16 for K and
// for V (a pool of kv_cache_tokens / 64 pages, addressed through the page table [slot][ctx_max / 64], kv_row), a decode
// working set of max_batch rows (row b == KV slot b) and a prefill working set of max_prefill_tokens rows.
// The decode step is a fixed sequence of 6 launches per layer + 4, captured once in a CUDA graph
// and replayed; per-row metadata (token, position, active flag) lives on the device so replays
// need no parameter changes.
#include "rr_kernels.h"
#include "rr_launch.cuh"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <new>
#include <string.h>
#include <thread>
#include <unordered_map>
#include <vector>

#define RR_API extern "C" __attribute__((visibility("default")))

namespace rr {
void note_cuda_error(cudaError_t e);

// Last layer of a prefill chunk: only the last token of every prompt still matters after attention.  Gather those
// rows (attention output bf16, residual fp32) into the decode working set; the rest of the layer and lm_head then run
// on n_seqs rows with the weight-streaming (decode-orientation) kernels instead of on all T tokens.
__global__ void gather_last_kernel(const __nv_bfloat16* __restrict__ attn, const float* __restrict__ x,
                                   const int32_t* __restrict__ last, __nv_bfloat16* __restrict__ attn_out,
                                   float* __restrict__ x_out, int nq, int hidden) {
    griddep_launch();
    griddep_wait();
    const int r = blockIdx.x;
    const size_t src = (size_t)last[r];
    const uint4* a = reinterpret_cast<const uint4*>(attn + src * nq);
    uint4* ao = reinterpret_cast<uint4*>(attn_out + (size_t)r * nq);
    for (int c = threadIdx.x; c < nq / 8; c += blockDim.x) ao[c] = a[c];
    const float4* xs = reinterpret_cast<const float4*>(x + src * hidden);
    float4* xo = reinterpret_cast<float4*>(x_out + (size_t)r * hidden);
    for (int c = threadIdx.x; c < hidden / 4; c += blockDim.x) xo[c] = xs[c];
}

// After a prefill chunk: row/slot s becomes an active decode row fed with its first token, at the position after the
// prompt's last (a cached prefix included).
__global__ void activate_rows_kernel(const int32_t* __restrict__ seq_slot, const int32_t* __restrict__ first_tok,
                                     const int32_t* __restrict__ tok_pos, const int32_t* __restrict__ last, int n,
                                     int32_t* __restrict__ d_tok, int32_t* __restrict__ d_pos, int32_t* __restrict__ d_slot) {
    griddep_launch();
    griddep_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = seq_slot[i];
    d_tok[s] = first_tok[i];
    d_pos[s] = tok_pos[last[i]] + 1;
    d_slot[s] = s;
}

void launch_gather_last(const __nv_bfloat16* attn, const float* x, const int32_t* last, int n_rows, int nq, int hidden,
                        __nv_bfloat16* attn_out, float* x_out, cudaStream_t st) {
    if (n_rows <= 0) return;
    launch_pdl(gather_last_kernel, dim3(n_rows), dim3(256), 0, st, attn, x, last, attn_out, x_out, nq, hidden);
}

void launch_activate_rows(const int32_t* seq_slot, const int32_t* first_tok, const int32_t* tok_pos, const int32_t* last,
                          int n, int32_t* d_tok, int32_t* d_pos, int32_t* d_slot, cudaStream_t st) {
    if (n <= 0) return;
    launch_pdl(activate_rows_kernel, dim3((n + 127) / 128), dim3(128), 0, st, seq_slot, first_tok, tok_pos, last, n, d_tok,
               d_pos, d_slot);
}

// One request of n_choices choices.  Choice c decodes in row rows[c] (== its KV slot); the prompt is prefilled once, into
// rows[0], and its KV copied to the other rows.  The choices are admitted together and get one token each per step.  A
// choice finishes when it holds max_new tokens, a stop sequence cuts it or (JSON mode) its top-level object closes, and
// gives its row back at once; the request finishes with its last choice.  Without stop sequences or JSON mode that is one
// step for all of them.  A prompt whose uncached part does not fit the room in a chunk is prefilled in pieces over several
// chunks (rr_engine::in_progress); its rows are held but do not decode until its last piece has run.
struct Request {
    uint64_t ticket;
    std::vector<int32_t> prompt;
    int max_new;
    int n_choices = 1;
    std::vector<std::vector<int32_t>> out;     // [n_choices][tokens generated so far]
    int status = RR_OK;
    bool done = false;
    double t_submit = 0, t_first = 0, t_done = 0;
    std::vector<int> rows;     // [n_choices] while admitted (-1: the choice finished and freed its row), else empty
    std::vector<int> finish;   // [n_choices] -1 running, else why the choice finished: 0 length, 1 stop
    std::vector<int> hold;     // [n_choices] newest tokens of a running choice that a stop sequence may still take back
    uint64_t tag = 0;          // opaque caller value handed to the done hook (the gateway's request id)
    bool cancel = false;       // rr_engine_cancel: the worker drops the rows at the next step
    bool detached = false;     // nobody will call rr_engine_wait: the worker frees the request when it finishes
    GenParams gen;
    std::vector<std::vector<float>> lp;        // [n_choices][out[c].size()][gen.lp_width()]
    std::vector<std::vector<int32_t>> lp_id;
    int n_cached = 0;          // prefix caching: prompt tokens taken from the cache (prefill starts at this position)
    int n_done = 0;            // prompt tokens whose KV is in its slot (cached or prefilled), while it is admitted
    uint64_t epoch = 0;        // prefix caching: rr_engine::index_epoch when its first piece was admitted
    // prompt logprobs (gen.scores()), written as the pieces run: ptgt[t - 1] = the logprob of prompt[t] given prompt[0..t),
    // plp / plp_id [n_prompt - 1][gen.score_width()] the best pairs at position t
    std::vector<float> ptgt, plp;
    std::vector<int32_t> plp_id;
    // an embedding request (rr_engine_submit_embed): max_new 0, one choice that never decodes; emb = the pooled,
    // L2-normalised final-norm row of its last prompt position [hidden], written when its last piece has run
    bool embed = false;
    std::vector<float> emb;

    // Tokens of choice c a reader may see: all of a finished choice, else those no stop sequence can take back.
    int visible(int c) const { return (int)out[c].size() - (finish[c] < 0 ? hold[c] : 0); }
    int n_generated() const {          // the longest choice's visible tokens
        int n = 0;
        for (int c = 0; c < n_choices; ++c) n = std::max(n, visible(c));
        return n;
    }
    int n_returned() const {           // over all choices
        int n = 0;
        for (int c = 0; c < n_choices; ++c) n += visible(c);
        return n;
    }
    bool all_finished() const { return std::find(finish.begin(), finish.end(), -1) == finish.end(); }
};

// Prefix caching: the shortest shared prefix that counts as a hit -- one key tile of prefill attention.  Trivial shared
// prefixes (a BOS and a role tag) stay misses.
constexpr int PREFIX_MIN = 64;

// The per-row parameter blocks of n rows, one per step_mode bit, each a structure of arrays at stride n:
//   0 top_n  top_lp i32[n] (-1: no logprobs)
//   1 samp   seed u64[n] | temperature f32[n] (0: greedy) | top_p f32[n], with a position column also | position i32[n]
//   2 pen    frequency_penalty f32[n] | presence_penalty f32[n] | gen0 i32[n] (the position of the first generated token)
//            | n_bias i32[n] | bias ids i32[n][bias_ld] | bias values f32[n][bias_ld]
//   3 stop   n_stop i32[n] | gen0 i32[n] | len u8[n][STOP_MAX_SEQS] | bytes u8[n][STOP_MAX_SEQS][STOP_MAX_LEN]
//   4 json   fmt i32[n] (0 text, 1 json_object)
// The decode rows use n = Bm and bias_ld = PEN_MAX_BIAS (fixed: the graphs hold it).  A prefill chunk uses n = n_seqs, the
// largest bias count among its sequences and a position column, in buffers sized for Bm rows and PEN_MAX_BIAS.
struct ParamBlocks {
    char* blk[5] = {};            // pen / stop / json stay null until the first request that uses them
                                  // (ensure_pen_buffers / ensure_stop_buffers / ensure_json_buffers)
    int n = 0, bias_ld = 0;
    bool has_pos = false;

    ParamBlocks at(int rows, int ld) const { ParamBlocks p = *this; p.n = rows; p.bias_ld = ld; return p; }
    static constexpr size_t STOP_ROW = 12 + STOP_MAX_SEQS * STOP_MAX_LEN;      // 268 B per row
    size_t bytes(int i) const {
        return (size_t)n * (i == 0 || i == 4 ? 4 : i == 1 ? (has_pos ? 20 : 16) : i == 2 ? 16 + 8 * (size_t)bias_ld
                                                                                          : STOP_ROW);
    }
    int32_t* top_n() const { return (int32_t*)blk[0]; }
    uint64_t* seed() const { return (uint64_t*)blk[1]; }
    float* temp() const { return (float*)(blk[1] + 8 * (size_t)n); }
    float* top_p() const { return (float*)(blk[1] + 12 * (size_t)n); }
    int32_t* pos() const { return (int32_t*)(blk[1] + 16 * (size_t)n); }
    float* freq() const { return (float*)blk[2]; }
    float* pres() const { return (float*)(blk[2] + 4 * (size_t)n); }
    int32_t* gen0() const { return (int32_t*)(blk[2] + 8 * (size_t)n); }
    int32_t* n_bias() const { return (int32_t*)(blk[2] + 12 * (size_t)n); }
    int32_t* bias_ids() const { return (int32_t*)(blk[2] + 16 * (size_t)n); }
    float* bias_vals() const { return (float*)(bias_ids() + (size_t)n * bias_ld); }
    int32_t* n_stop() const { return (int32_t*)blk[3]; }
    int32_t* stop_gen0() const { return (int32_t*)(blk[3] + 4 * (size_t)n); }
    uint8_t* stop_len() const { return (uint8_t*)(blk[3] + 8 * (size_t)n); }
    uint8_t* stop_bytes() const { return (uint8_t*)(blk[3] + 12 * (size_t)n); }
    int32_t* fmt() const { return (int32_t*)blk[4]; }

    PenaltyArgs pen_args() const {
        PenaltyArgs a;
        a.freq = freq(); a.pres = pres(); a.gen0 = gen0(); a.n_bias = n_bias();
        a.bias_ids = bias_ids(); a.bias_vals = bias_vals(); a.bias_ld = bias_ld;
        a.hist = nullptr; a.hist_ld = 0; a.hist_len = nullptr; a.app_tok = nullptr; a.app_pos = nullptr;
        return a;
    }
    StopArgs stop_args() const {
        StopArgs a = {};
        a.n_stop = n_stop(); a.gen0 = stop_gen0(); a.len = stop_len(); a.bytes = stop_bytes();
        return a;
    }
    // The step_mode bits of the blocks whose row i differs from the defaults.
    int row_mode(int i) const {
        return (top_n()[i] >= 0 ? 1 : 0) | (temp()[i] > 0.f ? 2 : 0) |
               (blk[2] && (freq()[i] != 0.f || pres()[i] != 0.f || n_bias()[i] != 0) ? 4 : 0) |
               (blk[3] && n_stop()[i] != 0 ? 8 : 0) | (blk[4] && fmt()[i] != 0 ? 16 : 0);
    }
    // Row i from p for its choice `choice`: drawn at `position` (with a position column) with seed p.seed + choice, p's
    // bias, penalties f / pr and p's stop sequences; g0 = the position of the row's first generated token (penalty history
    // and stop matching start there).
    void put_row(int i, const GenParams& p, int choice, int position, float f, float pr, int g0) const {
        top_n()[i] = p.top_lp;
        seed()[i] = p.sampled() ? p.seed + (uint64_t)choice : p.seed; temp()[i] = p.temp; top_p()[i] = p.top_p;
        if (has_pos) pos()[i] = position;
        if (blk[3]) {
            n_stop()[i] = p.n_stop; stop_gen0()[i] = p.stops() ? g0 : 0;
            memcpy(stop_len() + (size_t)i * STOP_MAX_SEQS, p.stop_len, STOP_MAX_SEQS);
            if (p.stops()) memcpy(stop_bytes() + (size_t)i * STOP_MAX_SEQS * STOP_MAX_LEN, p.stop, sizeof(p.stop));
        }
        if (blk[4]) fmt()[i] = p.fmt;
        if (!blk[2]) return;
        const int nb = (int)p.bias_id.size();
        freq()[i] = f; pres()[i] = pr; gen0()[i] = p.processed() ? g0 : 0; n_bias()[i] = nb;
        if (nb) {
            memcpy(bias_ids() + (size_t)i * bias_ld, p.bias_id.data(), 4 * (size_t)nb);
            memcpy(bias_vals() + (size_t)i * bias_ld, p.bias_val.data(), 4 * (size_t)nb);
        }
    }
    // Copies the blocks whose bit is in `mask` from these (pinned) blocks to d, of the same n and bias_ld.
    cudaError_t upload(const ParamBlocks& d, int mask, cudaStream_t s, uint64_t* h2d_bytes) const {
        for (int i = 0; i < 5; ++i) {
            if (!(mask >> i & 1)) continue;
            const cudaError_t err = cudaMemcpyAsync(d.blk[i], blk[i], bytes(i), cudaMemcpyHostToDevice, s);
            if (err != cudaSuccess) return err;
            *h2d_bytes += bytes(i);
        }
        return cudaSuccess;
    }
};

static_assert(sizeof(rr_gen_params) == 80 && offsetof(rr_gen_params, seed) == 16 && offsetof(rr_gen_params, bias_ids) == 40 &&
                  offsetof(rr_gen_params, response_format) == 72,
              "rr_gen_params layout: _lib.GenParams and tests/test_abi.py mirror it");
int GenParams::set(int vocab, const rr_gen_params* p) {
    if (!p) { *this = GenParams(); return RR_OK; }
    if (p->top_logprobs < -1 || p->top_logprobs > LP_MAX_TOP) return RR_INVALID_ARGUMENT;
    if (p->response_format < 0 || p->response_format > 1 || (p->response_format == 1 && vocab < JSON_MIN_VOCAB))
        return RR_INVALID_ARGUMENT;
    if (!(p->temperature >= 0.f && p->temperature <= 2.f && p->top_p >= 0.f && p->top_p <= 1.f)) return RR_INVALID_ARGUMENT;
    if (!(p->frequency_penalty >= -2.f && p->frequency_penalty <= 2.f && p->presence_penalty >= -2.f &&
          p->presence_penalty <= 2.f))
        return RR_INVALID_ARGUMENT;
    const int n_bias = p->n_bias;
    if (n_bias < 0 || n_bias > PEN_MAX_BIAS || (n_bias > 0 && (!p->bias_ids || !p->bias_vals))) return RR_INVALID_ARGUMENT;
    for (int i = 0; i < n_bias; ++i)
        if (p->bias_ids[i] < 0 || p->bias_ids[i] >= vocab || !(p->bias_vals[i] >= -100.f && p->bias_vals[i] <= 100.f))
            return RR_INVALID_ARGUMENT;
    std::vector<int32_t> ids(p->bias_ids, p->bias_ids + n_bias);
    std::sort(ids.begin(), ids.end());
    if (std::adjacent_find(ids.begin(), ids.end()) != ids.end()) return RR_INVALID_ARGUMENT;
    const int32_t* off = p->stop_off;
    if (p->n_stop < 0 || p->n_stop > STOP_MAX_SEQS || (p->n_stop > 0 && (!p->stop_bytes || !off))) return RR_INVALID_ARGUMENT;
    for (int i = 0; i < p->n_stop; ++i)
        if (off[i] < 0 || off[i + 1] - off[i] < 1 || off[i + 1] - off[i] > STOP_MAX_LEN) return RR_INVALID_ARGUMENT;
    *this = GenParams();
    top_lp = p->top_logprobs;
    if (p->temperature > 0.f) { temp = p->temperature; top_p = p->top_p; seed = p->seed; }
    if (p->frequency_penalty != 0.f || p->presence_penalty != 0.f || n_bias > 0) {
        fpen = p->frequency_penalty; ppen = p->presence_penalty;
        bias_id.assign(p->bias_ids, p->bias_ids + n_bias); bias_val.assign(p->bias_vals, p->bias_vals + n_bias);
    }
    n_stop = p->n_stop;
    for (int i = 0; i < n_stop; ++i) {
        stop_len[i] = (uint8_t)(off[i + 1] - off[i]);
        memcpy(stop[i], p->stop_bytes + off[i], stop_len[i]);
    }
    fmt = p->response_format;
    return RR_OK;
}

}  // namespace rr

using namespace rr;

#define CK(x)                                   \
    do {                                        \
        cudaError_t e__ = (x);                  \
        if (e__ != cudaSuccess) {               \
            rr::note_cuda_error(e__);           \
            return RR_CUDA_ERROR;               \
        }                                       \
    } while (0)

struct rr_engine {
    rr_model_desc d;
    rr_engine_opts o;
    int Bm, bn_dec, nq, nkv_dim, nqkv;
    std::vector<const void*> wqkv, wo, wgu, wdown, norm_attn, norm_mlp;
    const void *embed, *lm_head, *final_norm;
    // RR_WEIGHTS_FP8_E4M3: the projections are e4m3 with these row scales; prefill dequantizes layer l into deq (one layer's
    // wqkv | wo | wgu | wdown, bf16) before its GEMMs, and the prefill plans read deq
    bool fp8 = false;
    std::vector<const float*> sqkv, so, sgu, sdown;
    __nv_bfloat16* deq = nullptr;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    std::vector<void*> allocs;

    // decode working set
    int32_t *d_tok, *d_pos, *d_slot;
    float* x;
    __nv_bfloat16 *xn, *qbuf, *attn_out, *act;
    float *part_qkv, *part_o, *part_gu, *part_down, *logits, *attn_ws;   // split-K partial planes
    float2* rope_table;
    __nv_bfloat16 *kcache, *vcache;
    size_t kv_layer_stride;
    // The KV page pool, under mu: n_pages pages of KV_PAGE positions.  slot_pages[b] = the pages slot b holds, in position
    // order (a slot keeps them after its request; see take_pages / trim_pages / reclaim_pages); free_pages = a stack.  The
    // device table d_table [Bm][pps] has a fixed address (the decode graphs hold it); h_table is its pinned mirror, and
    // table_dirty[b] marks the rows upload_table copies before the next prefill chunk or decode step.
    int n_pages = 0, pps = 0;
    // Sliding window (rr_model_weights.sliding_window, 0: none) and the ring a windowed request reserves instead of its whole
    // reach (ring_pages; 0 without a window).  A ring request's table row maps logical page p to slot_pages[b][p % ring].
    int window = 0, ring = 0;
    int32_t *d_table = nullptr, *h_table = nullptr;
    std::vector<std::vector<int32_t>> slot_pages;
    std::vector<int32_t> free_pages;
    std::vector<char> table_dirty;
    int kv_splits;
    std::vector<GemmPlan> pl_qkv, pl_o, pl_gu, pl_down;
    std::vector<DecodeAttnArgs> attn_args;   // per layer (TMA maps of that layer's K / V cache)
    std::vector<PrefillAttnArgs> pf_attn;    // per layer (TMA maps of q and of that layer's K / V cache)
    GemmPlan pl_head;
    int s_qkv, s_o, s_gu, s_down;
    bool fuse_rope_pf = false;        // prefill: RoPE + KV append live in the QKV GEMM epilogue (head_dim 128)
    // prefill defers RMSNorm: no norm kernels inside the layers -- RESID epilogues emit bf16(x * gamma) + sum(x^2), the next
    // GEMM's epilogue applies 1 / rms (RopeEpi)
    float* p_rowss = nullptr;         // [Tmax][pf_parts]
    int pf_parts = 0;
    bool fuse_silu = false;           // wgu interleaved + one gate/up plane: SiLU*mul lives in the GEMM epilogue
    bool fuse_mlp = false;            // decode: gate/up and down GEMMs in one persistent launch (gemm_mlp_wgmma)
    std::vector<MlpPlan> mlp;         // per layer
    MlpItem* mlp_items = nullptr;     // device copy of the schedule (shared by all layers)
    unsigned* mlp_ready = nullptr;    // [n_slices] dependency counters, reset by the norm kernel before each launch
    int mlp_slices = 0, mlp_slice_kb = 0;
    // decode step graphs by step_mode(): bit 0 + launch_logprobs, bit 1 + launch_sample, bit 2 + launch_logit_penalties,
    // bit 3 + launch_stop_match, bit 4 + launch_json_mask / launch_json_advance.  [0] (plain) is captured after the warm-up
    // step, the others on first use: a step without logprobs, sampled, processed, stop or JSON rows replays the plain graph.
    cudaGraphExec_t graph[32] = {};
    bool warmed = false;
    // The decode rows' parameter blocks (d_rows) and their pinned host mirror (h_rows), which set_row_params keeps in step
    // with row_req, marking the blocks it changes in rows_dirty (step_mode bits); upload_row_params copies a dirty block
    // before a step that reads it.  A prefill chunk packs its sequences' parameters into staging (h_pf) and blocks of its
    // own (d_pf).
    ParamBlocks d_rows, h_rows, d_pf, h_pf;
    int rows_dirty = 0;
    void* lp_ws = nullptr;
    float* d_lp = nullptr;                             // [Bm][LP_MAX_TOP]
    int32_t* d_lp_id = nullptr;
    void* sample_ws = nullptr;
    float* d_tok_lp = nullptr;                         // [Bm] the sampled token's logprob (sampled logprobs rows)
    // the generated-token history [Bm][ctx_max], shared by the penalty and the stop kernels and allocated with the first
    // of their buffers (ensure_hist); penalties (ensure_pen_buffers): the count workspace [Bm][vocab] (all zero between
    // launches); stop sequences (ensure_stop_buffers): cut[Bm] | hold[Bm] of rr_op_stop_match and their pinned copy
    int32_t *d_hist = nullptr, *pen_ws = nullptr, *d_stop = nullptr, *h_stop = nullptr;
    // JSON mode (ensure_json_buffers): each slot's automaton state [Bm], and done[Bm] of rr_op_json_advance with its pinned
    // copy
    JsonState* d_json = nullptr;
    int32_t *d_json_done = nullptr, *h_json_done = nullptr;
    // prompt logprobs (ensure_score_buffers, on the first scoring request): the fp32 logits of SCORE_ROWS prompt rows, the
    // logprobs workspace, and per chunk row targets | prompt_top (d_sc_in / h_sc_in [2][Tmax]), the target's logprob
    // [Tmax] and the best pairs [Tmax][LP_MAX_TOP], device and pinned
    float* sc_logits = nullptr;
    void* sc_ws = nullptr;
    int32_t *d_sc_in = nullptr, *h_sc_in = nullptr, *d_sc_id = nullptr, *h_sc_id = nullptr;
    float *d_sc_tlp = nullptr, *h_sc_tlp = nullptr, *d_sc_lp = nullptr, *h_sc_lp = nullptr;
    // embeddings (ensure_embed_buffers, on the first chunk with an embedding row): the pooled rows [Bm][hidden] fp32,
    // device and pinned
    float *d_emb = nullptr, *h_emb = nullptr;

    // prefill working set
    int Tmax;
    int32_t *p_ids, *p_pos, *p_slot, *p_seq_start, *p_seq_slot, *p_last, *p_first;
    float* px;
    __nv_bfloat16 *pxn, *pqkv, *pq, *pattn, *pgu, *pact;
    // prefill GEMM plans (4 L TMA descriptors), built at create for Tmax rows
    struct PfPlans { std::vector<GemmPlan> qkv, o, gu, down; } pf;

    // pinned staging
    int32_t* h_stage;     // ids | pos | slot | seq_start | seq_slot | last   (prefill) / rows meta (decode)
    int32_t* h_tok;       // [Bm] tokens read back each step
    float* h_lp = nullptr;        // [Bm][LP_MAX_TOP] logprobs read back on steps that computed them
    int32_t* h_lp_id = nullptr;
    float* h_tok_lp = nullptr;    // [Bm]

    // serving state
    std::mutex mu;                       // queues + request table
    std::condition_variable cv_work, cv_done;
    std::mutex gpu_mu;                   // serialises GPU work between worker and low-level API
    std::deque<Request*> waiting;
    std::unordered_map<uint64_t, Request*> table;
    std::vector<Request*> row_req;       // [Bm]
    std::vector<int> row_choice;         // [Bm] the choice of row_req[b] that row b decodes
    std::vector<int32_t> h_slot_mirror;  // host mirror of d_slot
    bool slots_dirty = false;
    // The request whose prompt will still be in progress after the chunk being built (some pieces done, no token yet), or
    // null.  At most one: it holds its rows and pages, and its next piece leads the next chunk.
    Request* in_progress = nullptr;
    // prefix caching (o.prefix_cache), under mu: retained[b] = the prompt tokens whose KV the last successful prefill into
    // slot b wrote (computed or copied; never a position decode wrote, since decode rounds differently), kept after the
    // request ends; retained_used[b] = LRU stamp.  index_epoch counts the low-level calls that cleared every list.
    std::vector<std::vector<int32_t>> retained;
    std::vector<uint64_t> retained_used;
    uint64_t lru_clock = 0, index_epoch = 0;
    std::thread worker;
    std::atomic<bool> stop{false};
    uint64_t next_ticket = 1;
    std::chrono::steady_clock::time_point t0;

    rr_engine_stats st;                  // written under gpu_mu (launch / timing counters) or mu (queued, active_rows)
    uint64_t step_launches[32] = {};              // launches of one decode step, by step_mode()
    // completion hook (the native gateway, rr_gateway.cu): called on the worker / submitting thread, outside `mu`
    rr::EngineDoneHook hook = nullptr;
    void* hook_ctx = nullptr;
};

static double now_s(rr_engine* e) {
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - e->t0).count();
}

template <typename T>
static int dalloc(rr_engine* e, T** p, size_t n, bool zero = true) {
    void* q = nullptr;
    cudaError_t err = cudaMalloc(&q, n * sizeof(T) ? n * sizeof(T) : 16);
    if (err != cudaSuccess) { rr::note_cuda_error(err); return RR_CUDA_ERROR; }
    if (zero) cudaMemset(q, 0, n * sizeof(T));
    e->allocs.push_back(q);
    *p = (T*)q;
    return RR_OK;
}

// Tile width argument of the prefill plans (row-major modes only validate it; their tiles are 128 x 256).
constexpr int PF_BN = MAX_BN;

// One engine at a time per device.  The fused MLP kernel is a persistent grid whose CTAs spin on work of sibling CTAs;
// two such grids interleaved on one GPU (two engines, two streams) could each hold SMs the other's not-yet-resident CTAs
// need.  Every path below synchronises its stream before it releases this lock, so engines that share a device alternate
// at prefill-chunk / decode-step granularity.  (The gateway creates one engine per GPU, so this lock is uncontended there.)
static std::mutex& device_mutex(int dev) {
    static std::mutex mu[64];
    return mu[dev & 63];
}

static PartIn part_f32(const float* p, int splits, int rows, int ld) {
    PartIn r; r.ptr = p; r.is_bf16 = 0; r.n_splits = splits; r.split_stride = (long long)rows * ld; r.ld = ld;
    return r;
}
static PartIn part_bf16(const __nv_bfloat16* p, int ld) {
    PartIn r; r.ptr = p; r.is_bf16 = 1; r.n_splits = 1; r.split_stride = 0; r.ld = ld;
    return r;
}
static PartIn part_none() { PartIn r; r.ptr = nullptr; r.is_bf16 = 0; r.n_splits = 1; r.split_stride = 0; r.ld = 0; return r; }

// ---------------------------------------------------------------- decode step (enqueue only)
// The step_mode bits a request needs: 1 logprobs, 2 sampling, 4 penalties / logit bias, 8 stop sequences, 16 JSON mode.
// Over a step's rows or a chunk's sequences they pick the parameter blocks to upload, the kernels of the logits tail and
// the decode graph.
static int step_mode(const GenParams& p) {
    return (p.logprobs() ? 1 : 0) | (p.sampled() ? 2 : 0) | (p.processed() ? 4 : 0) | (p.stops() ? 8 : 0) |
           (p.json() ? 16 : 0);
}

// Caller holds gpu_mu.  The generated-token history, which the decode graphs of modes 4 and 8 hold: allocated once.
static int ensure_hist(rr_engine* e) {
    return e->d_hist ? RR_OK : dalloc(e, &e->d_hist, (size_t)e->Bm * e->o.ctx_max, false);
}

// Caller holds gpu_mu.  Decode rows' and prefill blocks of parameter block i (2, 3 or 4), device and pinned, all zero: the
// defaults of a row that does not use the block.
static int ensure_block(rr_engine* e, int i) {
    const size_t blk = e->d_rows.bytes(i);            // also the prefill blocks' size: Bm rows (of PEN_MAX_BIAS)
    char *dp = nullptr, *dpf = nullptr, *hp = nullptr, *hpf = nullptr;
    int rc = dalloc(e, &dp, blk, false);
    if (rc == RR_OK) rc = dalloc(e, &dpf, blk, false);
    if (rc != RR_OK) return rc;
    CK(cudaMemsetAsync(dp, 0, blk, e->stream));       // on the engine's stream: ordered before the step that reads it
    CK(cudaMallocHost(&hp, blk));
    cudaError_t ce = cudaMallocHost(&hpf, blk);
    if (ce != cudaSuccess) { cudaFreeHost(hp); rr::note_cuda_error(ce); return RR_CUDA_ERROR; }
    memset(hp, 0, blk);
    e->d_pf.blk[i] = dpf; e->h_rows.blk[i] = hp; e->h_pf.blk[i] = hpf; e->d_rows.blk[i] = dp;
    return RR_OK;
}

// Caller holds gpu_mu.  The stop-sequence buffers, allocated on the first request with stop sequences: 2 x 268 B x Bm of
// parameter blocks, the history and 8 B x Bm of results.  An engine that never sees one allocates nothing.
static int ensure_stop_buffers(rr_engine* e) {
    if (e->d_rows.blk[3]) return RR_OK;
    int rc = ensure_hist(e);
    if (rc == RR_OK && !e->d_stop) rc = dalloc(e, &e->d_stop, 2 * (size_t)e->Bm);
    if (rc != RR_OK) return rc;
    if (!e->h_stop) CK(cudaMallocHost(&e->h_stop, sizeof(int32_t) * 2 * e->Bm));
    return ensure_block(e, 3);
}

// Caller holds gpu_mu.  The JSON-mode buffers, allocated on the first JSON request: 2 x 4 B x Bm of parameter blocks,
// 16 B x Bm of automaton state and 4 B x Bm of done flags.  An engine that never sees one allocates nothing.
static int ensure_json_buffers(rr_engine* e) {
    if (e->d_rows.blk[4]) return RR_OK;
    int rc = RR_OK;
    if (!e->d_json) rc = dalloc(e, &e->d_json, (size_t)e->Bm);
    if (rc == RR_OK && !e->d_json_done) rc = dalloc(e, &e->d_json_done, (size_t)e->Bm);
    if (rc != RR_OK) return rc;
    if (!e->h_json_done) CK(cudaMallocHost(&e->h_json_done, sizeof(int32_t) * e->Bm));
    return ensure_block(e, 4);
}

// Caller holds gpu_mu.  The penalty buffers, allocated on the first processed request, so an engine that never sees one
// keeps its footprint.
static int ensure_pen_buffers(rr_engine* e) {
    if (e->d_rows.blk[2]) return RR_OK;
    int rc = ensure_hist(e);
    if (rc == RR_OK && !e->pen_ws) {
        rc = dalloc(e, &e->pen_ws, (size_t)e->Bm * e->d.vocab, false);
        if (rc == RR_OK) CK(cudaMemsetAsync(e->pen_ws, 0, sizeof(int32_t) * e->Bm * (size_t)e->d.vocab, e->stream));
    }
    return rc != RR_OK ? rc : ensure_block(e, 2);
}

// Prompt rows per lm_head block of a scoring chunk: the fp32 logits block is SCORE_ROWS x vocab (525 MB at 128256).
constexpr int SCORE_ROWS = 1024;

// Caller holds gpu_mu.  The prompt-logprob buffers, allocated on the first scoring request: SCORE_ROWS x vocab x 4 B of
// logits, their logprobs workspace and 96 B x Tmax of inputs and results on the device and pinned.  All or nothing: on a
// failure nothing stays allocated and the error is cleared, so the engine serves on without them.
static int ensure_score_buffers(rr_engine* e) {
    if (e->sc_logits) return RR_OK;
    const size_t S = (size_t)std::min(SCORE_ROWS, e->Tmax), T = (size_t)e->Tmax, V = (size_t)e->d.vocab;
    const size_t dev_bytes[5] = {S * V * 4, logprobs_ws_bytes((int)S, (int)V), 2 * T * 4, T * 4, 2 * T * LP_MAX_TOP * 4};
    const size_t host_bytes[3] = {2 * T * 4, T * 4, 2 * T * LP_MAX_TOP * 4};
    void* d[5] = {};
    void* h[3] = {};
    cudaError_t err = cudaSuccess;
    for (int i = 0; i < 5 && err == cudaSuccess; ++i) err = cudaMalloc(&d[i], dev_bytes[i]);
    for (int i = 0; i < 3 && err == cudaSuccess; ++i) err = cudaMallocHost(&h[i], host_bytes[i]);
    if (err != cudaSuccess) {
        rr::note_cuda_error(err);
        for (void* p : d) if (p) cudaFree(p);
        for (void* p : h) if (p) cudaFreeHost(p);
        cudaGetLastError();                // an allocation failure is not sticky: later launches must not report it
        return RR_CUDA_ERROR;
    }
    for (void* p : d) e->allocs.push_back(p);
    e->sc_ws = d[1]; e->d_sc_in = (int32_t*)d[2]; e->d_sc_tlp = (float*)d[3];
    e->d_sc_lp = (float*)d[4]; e->d_sc_id = (int32_t*)(e->d_sc_lp + T * LP_MAX_TOP);
    e->h_sc_in = (int32_t*)h[0]; e->h_sc_tlp = (float*)h[1];
    e->h_sc_lp = (float*)h[2]; e->h_sc_id = (int32_t*)(e->h_sc_lp + T * LP_MAX_TOP);
    e->sc_logits = (float*)d[0];
    return RR_OK;
}

// Caller holds gpu_mu.  The embedding buffers, allocated on the first chunk with an embedding row: 4 B x Bm x hidden on the
// device and pinned.  An engine that never embeds allocates nothing.
static int ensure_embed_buffers(rr_engine* e) {
    if (e->h_emb) return RR_OK;
    if (!e->d_emb) {
        const int rc = dalloc(e, &e->d_emb, (size_t)e->Bm * e->d.hidden, false);
        if (rc != RR_OK) return rc;
    }
    CK(cudaMallocHost(&e->h_emb, sizeof(float) * e->Bm * e->d.hidden));
    return RR_OK;
}

// The rest of layer l after attention on `rows` rows of the decode working set, with the unfused kernels: O GEMM,
// add_rmsnorm, gate/up GEMM (SiLU), down GEMM, add_rmsnorm with the next layer's (or the final) norm weight.
static int enqueue_o_mlp(rr_engine* e, int l, int rows, cudaStream_t s, uint64_t* nl) {
    const rr_model_desc& d = e->d;
    const int B = e->Bm;
    const void* nw = (l + 1 < d.n_layers) ? e->norm_attn[l + 1] : e->final_norm;
    if (gemm_launch(e->pl_o[l], s) != RR_OK) return RR_CUDA_ERROR; ++*nl;
    launch_add_rmsnorm(e->x, part_f32(e->part_o, e->s_o, B, d.hidden), (const __nv_bfloat16*)e->norm_mlp[l], e->xn, rows,
                       d.hidden, d.rms_eps, s); ++*nl;
    if (gemm_launch(e->pl_gu[l], s) != RR_OK) return RR_CUDA_ERROR; ++*nl;
    if (!e->fuse_silu) { launch_silu_mul(part_f32(e->part_gu, e->s_gu, B, 2 * d.inter), e->act, rows, d.inter, s); ++*nl; }
    if (gemm_launch(e->pl_down[l], s) != RR_OK) return RR_CUDA_ERROR; ++*nl;
    launch_add_rmsnorm(e->x, part_f32(e->part_down, e->s_down, B, d.hidden), (const __nv_bfloat16*)nw, e->xn, rows,
                       d.hidden, d.rms_eps, s); ++*nl;
    return RR_OK;
}

// The logits tail over `rows` rows of e->logits (lm_head's output), reading the parameter blocks p; returns its launches.
//   mode & 4: penalties and logit bias, applied to the logits that everything after reads.  With hist (decode) each row
//             first appends its input token tok[r] (the last generated one, at `position`) to its history.
//   argmax into tok; decode passes row_active (d_slot) and pos_inc (d_pos, advanced to the generated token's position).
//   mode & 2: rows with temperature > 0 replace the argmax token by rr_op_sample's draw at `position`.
//   mode & 1: logprobs of the rows with top_n >= 0 (the logits are left as they were), with mode & 2 also the logprob of
//             the token in tok into d_tok_lp.
//   mode & 8: stop sequences over the picked token, into d_stop (cut[Bm] | hold[Bm]).  Decode: the token joins history row
//             r at its position (pos_inc has advanced `position` to it) - gen0.  Prefill (hist null): it is token 0 of the
//             history of its slot, stop_row[r].
//   mode & 16: JSON mode.  After penalties and before the argmax, rr_op_json_mask sets the logits the grammar does not
//             allow next to -inf, so everything after reads the masked logits; last of all rr_op_json_advance steps the
//             state by the picked token into d_json and writes d_json_done.  Decode: row r's state is d_json[r] (row ==
//             slot).  Prefill (pos_inc null): every tail row starts from the initial state and leaves its state in its
//             slot, stop_row[r].
static uint64_t enqueue_tail(rr_engine* e, const ParamBlocks& p, int rows, int mode, int32_t* tok,
                             const int32_t* row_active, int32_t* pos_inc, const int32_t* position, int32_t* hist,
                             cudaStream_t s, const int32_t* stop_row = nullptr) {
    const int V = e->d.vocab;
    uint64_t nl = 0;
    if (mode & 4) {
        PenaltyArgs a = p.pen_args();
        if (hist) { a.hist = hist; a.hist_ld = e->o.ctx_max; a.app_tok = tok; a.app_pos = position; }
        launch_logit_penalties(e->logits, V, rows, V, a, e->pen_ws, s); ++nl;
    }
    // decode (pos_inc set) steps each row's own state; prefill starts every tail row from the initial state.  (hist does not
    // tell them apart: the history exists only once a penalty or stop request allocated it.)
    const JsonState* json_in = pos_inc ? e->d_json : nullptr;
    if (mode & 16) { launch_json_mask(e->logits, V, rows, V, p.fmt(), row_active, json_in, s); ++nl; }
    launch_argmax(part_f32(e->logits, 1, e->Bm, V), rows, V, tok, nullptr, row_active, pos_inc, s); ++nl;
    if (mode & 2) {
        launch_sample(e->logits, V, rows, V, p.temp(), p.top_p(), p.seed(), position, tok, e->sample_ws, s);
        nl += SAMPLE_LAUNCHES;
    }
    if (mode & 1) {
        launch_logprobs(e->logits, V, rows, V, p.top_n(), LP_MAX_TOP, e->lp_ws, e->d_lp, e->d_lp_id, s,
                        mode & 2 ? tok : nullptr, mode & 2 ? e->d_tok_lp : nullptr);
        nl += LP_LAUNCHES;
    }
    if (mode & 8) {
        StopArgs a = p.stop_args();
        a.hist = e->d_hist; a.hist_ld = e->o.ctx_max; a.hist_row = stop_row; a.tok = tok;
        a.position = hist ? position : nullptr; a.row_active = row_active;
        a.cut = e->d_stop; a.hold = e->d_stop + e->Bm;
        launch_stop_match(a, rows, s); ++nl;
    }
    if (mode & 16) {
        launch_json_advance(rows, p.fmt(), row_active, tok, json_in, e->d_json, pos_inc ? nullptr : stop_row, e->d_json_done,
                            s);
        ++nl;
    }
    return nl;
}

// Reads a tail's results for `rows` rows back to the host: the tokens (h_tok), with mode & 1 the [rows][LP_MAX_TOP]
// logprobs and ids (h_lp, h_lp_id), with mode & 3 == 3 the drawn tokens' logprobs (h_tok_lp), with mode & 8 the stop
// results (h_stop: cut[Bm] | hold[Bm]) and with mode & 16 the JSON done flags (h_json_done).
static int enqueue_readback(rr_engine* e, const int32_t* tok, int rows, int mode, cudaStream_t s) {
    CK(cudaMemcpyAsync(e->h_tok, tok, sizeof(int32_t) * rows, cudaMemcpyDeviceToHost, s));
    e->st.d2h_bytes += sizeof(int32_t) * rows;
    if (mode & 16) {
        CK(cudaMemcpyAsync(e->h_json_done, e->d_json_done, sizeof(int32_t) * rows, cudaMemcpyDeviceToHost, s));
        e->st.d2h_bytes += sizeof(int32_t) * rows;
    }
    if (mode & 8) {
        for (int i = 0; i < 2; ++i)
            CK(cudaMemcpyAsync(e->h_stop + i * e->Bm, e->d_stop + i * e->Bm, sizeof(int32_t) * rows, cudaMemcpyDeviceToHost, s));
        e->st.d2h_bytes += 2 * sizeof(int32_t) * rows;
    }
    if (!(mode & 1)) return RR_OK;
    const size_t n = (size_t)rows * LP_MAX_TOP;
    CK(cudaMemcpyAsync(e->h_lp, e->d_lp, sizeof(float) * n, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(e->h_lp_id, e->d_lp_id, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, s));
    e->st.d2h_bytes += (sizeof(float) + sizeof(int32_t)) * n;
    if (mode & 2) {
        CK(cudaMemcpyAsync(e->h_tok_lp, e->d_tok_lp, sizeof(float) * rows, cudaMemcpyDeviceToHost, s));
        e->st.d2h_bytes += sizeof(float) * rows;
    }
    return RR_OK;
}

// The decode step over all Bm rows; mode (step_mode bits) selects the kernels of the logits tail.
static int enqueue_decode_step(rr_engine* e, cudaStream_t s, uint64_t* n_launch, int mode = 0) {
    const rr_model_desc& d = e->d;
    const int B = e->Bm, L = d.n_layers;
    uint64_t nl = 0;
    launch_embed(e->d_tok, (const __nv_bfloat16*)e->embed, e->x, B, d.hidden, e->d_slot, s); ++nl;
    launch_add_rmsnorm(e->x, part_none(), (const __nv_bfloat16*)e->norm_attn[0], e->xn, B, d.hidden, d.rms_eps, s); ++nl;
    for (int l = 0; l < L; ++l) {
        if (gemm_launch(e->pl_qkv[l], s) != RR_OK) return RR_CUDA_ERROR; ++nl;
        // RoPE + KV append are fused into the attention kernel (reads the QKV split-K planes directly)
        launch_decode_attn(e->attn_args[l], s); nl += e->kv_splits > 1 ? 2 : 1;
        if (!e->fuse_mlp) {
            if (enqueue_o_mlp(e, l, B, s, &nl) != RR_OK) return RR_CUDA_ERROR;
            continue;
        }
        const void* nw = (l + 1 < L) ? e->norm_attn[l + 1] : e->final_norm;
        if (gemm_launch(e->pl_o[l], s) != RR_OK) return RR_CUDA_ERROR; ++nl;
        launch_add_rmsnorm(e->x, part_f32(e->part_o, e->s_o, B, d.hidden), (const __nv_bfloat16*)e->norm_mlp[l],
                           e->xn, B, d.hidden, d.rms_eps, s, e->mlp_ready, e->mlp_slices + 1); ++nl;
        if (mlp_launch(e->mlp[l], s) != RR_OK) return RR_CUDA_ERROR; ++nl;
        launch_add_rmsnorm(e->x, part_f32(e->part_down, e->mlp_slices, B, d.hidden), (const __nv_bfloat16*)nw, e->xn, B,
                           d.hidden, d.rms_eps, s); ++nl;
    }
    if (gemm_launch(e->pl_head, s) != RR_OK) return RR_CUDA_ERROR; ++nl;
    nl += enqueue_tail(e, e->d_rows, B, mode, e->d_tok, e->d_slot, e->d_pos, e->d_pos, e->d_hist, s);
    if (n_launch) *n_launch = nl;
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) { rr::note_cuda_error(err); return RR_CUDA_ERROR; }
    return RR_OK;
}

static int capture_decode_step(rr_engine* e, int mode, cudaGraphExec_t* out, uint64_t* n_launch) {
    cudaStream_t s = e->stream;
    cudaGraph_t g = nullptr;
    CK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    int rc = enqueue_decode_step(e, s, n_launch, mode);
    cudaError_t ce = cudaStreamEndCapture(s, &g);
    if (rc != RR_OK || ce != cudaSuccess) { rr::note_cuda_error(ce); return RR_CUDA_ERROR; }
    CK(cudaGraphInstantiate(out, g, 0));
    cudaGraphDestroy(g);
    return RR_OK;
}

// mode: the step_mode bits of the active rows (enqueue_tail).  Each combination has its own graph, captured on first use;
// a step without logprobs, sampled, processed or stop rows replays the plain graph.
static int run_decode_step(rr_engine* e, int mode) {
    cudaStream_t s = e->stream;
    if (!e->warmed || !e->o.use_cuda_graph) {
        uint64_t nl = 0;
        int rc = enqueue_decode_step(e, s, &nl, mode);
        if (rc != RR_OK) return rc;
        e->step_launches[mode] = nl;
        e->st.kernel_launches += nl;
        // NOTE: the warm-up step is a real step (it advances positions); graph capture follows.
        if (!e->warmed) {
            e->warmed = true;
            if (e->o.use_cuda_graph) {
                CK(cudaStreamSynchronize(s));
                // capture for subsequent steps
                rc = capture_decode_step(e, 0, &e->graph[0], &e->step_launches[0]);
                if (rc != RR_OK) return rc;
            }
        }
        return RR_OK;
    }
    if (!e->graph[mode]) {
        const int rc = capture_decode_step(e, mode, &e->graph[mode], &e->step_launches[mode]);
        if (rc != RR_OK) return rc;
    }
    CK(cudaGraphLaunch(e->graph[mode], s));
    e->st.kernel_launches += e->step_launches[mode];
    return RR_OK;
}

// ---------------------------------------------------------------- prefill chunk
// FP8 weights: layer l's four projections dequantized into the prefill scratch (the layout init_pf_plans reads), one launch.
// The last layer needs wqkv only: its O projection and MLP run on the chunk's tail rows through the decode kernels, which
// read the e4m3 weights themselves -- unless the chunk scores (scoring: the last layer also runs over every row).
static int launch_dequant_layer(rr_engine* e, int l, bool scoring, cudaStream_t s) {
    const rr_model_desc& d = e->d;
    Fp8DequantJobs J;
    __nv_bfloat16* p = e->deq;
    fp8_dequant_job(&J, e->wqkv[l], e->sqkv[l], e->nqkv, d.hidden, p, d.hidden); p += (size_t)e->nqkv * d.hidden;
    if (l + 1 == d.n_layers && !scoring) return launch_dequantize_fp8(J, s);
    fp8_dequant_job(&J, e->wo[l], e->so[l], d.hidden, e->nq, p, e->nq); p += (size_t)d.hidden * e->nq;
    fp8_dequant_job(&J, e->wgu[l], e->sgu[l], 2 * d.inter, d.hidden, p, d.hidden); p += (size_t)2 * d.inter * d.hidden;
    fp8_dequant_job(&J, e->wdown[l], e->sdown[l], d.hidden, d.inter, p, d.inter);
    return launch_dequantize_fp8(J, s);
}

// One set of plans (4 L TMA descriptors) built for Tmax rows; the live row count is a launch argument: TMA reads of
// rows >= T stay inside the Tmax-row buffers and every store is guarded by rowsA.
static int init_pf_plans(rr_engine* e) {
    const rr_model_desc& d = e->d;
    rr_engine::PfPlans& P = e->pf;
    const int L = d.n_layers, T = e->Tmax;
    P.qkv.resize(L); P.o.resize(L); P.gu.resize(L); P.down.resize(L);
    for (int l = 0; l < L; ++l) {
        const void *wqkv = e->wqkv[l], *wo = e->wo[l], *wgu = e->wgu[l], *wdown = e->wdown[l];
        if (e->fp8) {
            const __nv_bfloat16* base = e->deq;
            wqkv = base; wo = base + (size_t)e->nqkv * d.hidden; wgu = (const __nv_bfloat16*)wo + (size_t)d.hidden * e->nq;
            wdown = (const __nv_bfloat16*)wgu + (size_t)2 * d.inter * d.hidden;
        }
        int rc = gemm_plan_init(&P.qkv[l], e->pxn, T, d.hidden, wqkv, e->nqkv, d.hidden, d.hidden, e->pqkv,
                                e->nqkv, 0, 1, e->fuse_rope_pf ? OUT_ROWMAJOR_ROPE : OUT_ROWMAJOR_BF16, PF_BN);
        if (rc) return rc;
        if (e->fuse_rope_pf) {
            RopeEpi& r = P.qkv[l].rope;
            r.q_out = e->pq; r.k_cache = e->kcache + (size_t)l * e->kv_layer_stride;
            r.v_cache = e->vcache + (size_t)l * e->kv_layer_stride;
            r.slot = nullptr; r.pos = nullptr;                     // set per chunk (offsets inside the staging buffer)
            r.table = e->rope_table; r.n_heads = d.n_heads; r.n_kv_heads = d.n_kv_heads; r.ctx_max = e->o.ctx_max;
            r.page_table = e->d_table; r.pages_per_slot = e->pps;
        }
        rc = gemm_plan_init(&P.o[l], e->pattn, T, e->nq, wo, d.hidden, e->nq, e->nq, e->px, d.hidden, 0, 1,
                            OUT_ROWMAJOR_RESID, PF_BN);                // residual add in the epilogue
        if (rc) return rc;
        // deferred RMSNorm: the residual GEMMs (O, down) produce the next operand and its sum(x^2); QKV and gate/up apply 1 / rms
        pf_norm_consumer(&P.qkv[l].rope, e->p_rowss, d.hidden, d.rms_eps);
        pf_norm_producer(&P.o[l].rope, (const __nv_bfloat16*)e->norm_mlp[l], e->pxn, e->p_rowss, d.hidden);
        if (e->fuse_silu)
            rc = gemm_plan_init(&P.gu[l], e->pxn, T, d.hidden, wgu, 2 * d.inter, d.hidden, d.hidden, e->pact,
                                d.inter, 0, 1, OUT_ROWMAJOR_SILU, PF_BN);
        else
            rc = gemm_plan_init(&P.gu[l], e->pxn, T, d.hidden, wgu, 2 * d.inter, d.hidden, d.hidden, e->pgu,
                                2 * d.inter, 0, 1, OUT_ROWMAJOR_BF16, PF_BN);
        if (rc) return rc;
        rc = gemm_plan_init(&P.down[l], e->pact, T, d.inter, wdown, d.hidden, d.inter, d.inter, e->px,
                            d.hidden, 0, 1, OUT_ROWMAJOR_RESID, PF_BN);
        if (rc) return rc;
        pf_norm_consumer(&P.gu[l].rope, e->p_rowss, d.hidden, d.rms_eps);
        pf_norm_producer(&P.down[l].rope, (const __nv_bfloat16*)(l + 1 < L ? e->norm_attn[l + 1] : e->final_norm), e->pxn,
                         e->p_rowss, d.hidden);
    }
    return RR_OK;
}

// One prefill chunk: the tokens of its sequences back to back, one record per sequence, the cached prefixes to copy
// between slots before its first layer (prefix caching) and the index epoch it was admitted under.  A sequence is the
// piece [pos0, pos0 + len) of a prompt, prefilled into its slot, which holds positions [0, pos0) already.  The rows after
// attention follow from the records; add() numbers them in sequence order:
//   tail rows: one per choice of a last piece, row `row` + c for choice c, decoding in r->rows[c] (a sequence without a
//              request: one plain greedy row in its own slot);
//   embedding rows: one per last piece of an embedding request (it has no tail rows), after every tail row: n_tail + `row`;
//   scoring rows (prompt logprobs): the rows of a scoring request's piece that predict a prompt token, from `score_row` on.
struct Chunk {
    struct Seq {
        Request* r;                    // null: a sequence of rr_engine_prefill
        int slot, pos0, start, len;    // its tokens are ids[start, start + len)
        bool last;                     // the prompt's last piece
        int row, score_row;
        bool embeds() const { return last && r && r->embed; }
        int n_tail() const { return !last || embeds() ? 0 : r ? r->n_choices : 1; }
        int score_rows() const {
            return r && r->gen.scores() ? std::max(0, std::min(len, (int)r->prompt.size() - 1 - pos0)) : 0;
        }
        const GenParams& gen() const { static const GenParams plain; return r ? r->gen : plain; }
    };
    std::vector<int32_t> ids;
    std::vector<Seq> seqs;
    KvCopyList copies;
    uint64_t epoch = 0;
    bool has_pos0 = false;             // attention reads seq_pos0: prefix caching is on or the chunk continues a prompt
    int n_tail = 0, n_emb = 0, n_score = 0;
    int mode = 0;                      // the step_mode bits of the last pieces' requests

    void reset(uint64_t ep, bool pos0) {
        ids.clear(); seqs.clear(); copies.count = 0;
        epoch = ep; has_pos0 = pos0;
        n_tail = n_emb = n_score = mode = 0;
    }
    void add(Request* r, int slot, int pos0, const int32_t* tok, int n, bool last) {
        Seq q{r, slot, pos0, (int)ids.size(), n, last, 0, n_score};
        ids.insert(ids.end(), tok, tok + std::max(n, 0));      // n < 1: run_prefill refuses the chunk
        if (q.embeds()) q.row = n_emb++;
        else if (last) { q.row = n_tail; n_tail += q.n_tail(); }
        n_score += q.score_rows();
        if (last && r) mode |= step_mode(r->gen);
        seqs.push_back(q);
    }
};

// Runs chunk c.  Caller holds gpu_mu.  Leaves first tokens in e->p_first (device) and activates the tail rows.
// Prefix caching: sequence i's tokens are the prompt from position pos0 on; c.copies run first, in one launch.
// Tail rows: stop sequences are matched over the first token (needs ensure_stop_buffers; results in e->h_stop row j).  A
// JSON-mode row picks its first token from the initial state's mask and leaves its state in its slot (needs
// ensure_json_buffers; done in e->h_json_done row j).  Only a logit bias applies (penalties count generated tokens only, so
// the first token has none; needs ensure_pen_buffers).  A sampled row draws its first token at position pos0 + the
// sequence's length (the prompt length) with its choice's seed.  A logprobs row j also gets its first token's logprobs in
// e->h_lp / e->h_lp_id row j, and if sampled its own logprob in h_tok_lp.  When a sequence has rows in other slots, one
// launch after the last layer copies positions [0, pos0 + its length) of its slot to each of them.
// A chunk without tail or embedding rows stops after the last layer's QKV projection and KV append: nothing after reads
// its other outputs, and nothing is read back -- unless it scores.
// Scoring rows (needs ensure_score_buffers): after the tail rows are gathered and have run through the decode kernels, the
// last layer's O, gate/up and down GEMMs run over all T rows in prefill orientation (its down GEMM leaves
// bf16(x * final_norm) and the partial sums of squares in pxn / p_rowss), then lm_head (OUT_ROWMAJOR_F32) and
// launch_logprobs over the scoring rows only, in blocks of SCORE_ROWS rows of one sequence.  The tail rows were copied
// before the full layer rewrites px, so what they compute does not change.  Scoring row o's results are left in
// h_sc_tlp[o] and h_sc_lp / h_sc_id [o][LP_MAX_TOP].
// Embedding rows (needs ensure_embed_buffers) follow the tail rows through the trimmed last layer, each in its sequence's
// slot, and rr_op_embed_pool turns their final-norm rows in e->xn into e->h_emb row `row`; lm_head, the logits tail,
// activate_rows_kernel and the readback see the tail rows only.  Such a sequence needs no position after its prompt, so
// its prompt may reach ctx_max.
static int run_prefill(rr_engine* e, const Chunk& c, int32_t* first_tok_host, float* logits_host) {
    const rr_model_desc& d = e->d;
    const int T = (int)c.ids.size(), n_seqs = (int)c.seqs.size();
    const int nt = c.n_tail, ne = c.n_emb, nr = nt + ne;       // rows through the trimmed last layer
    const int n_score = c.n_score;
    const bool scoring = n_score > 0;
    if (scoring && !e->sc_logits) return RR_INTERNAL;
    if (ne > 0 && !e->h_emb) return RR_INTERNAL;
    if (T <= 0 || T > e->Tmax || n_seqs > e->Bm || nr > e->Bm) return RR_INVALID_ARGUMENT;
    cudaStream_t s = e->stream;
    // pinned staging: ids[T] | pos[T] | slot_tok[T] | seq_start[n+1] | seq_slot[n] | last[n] (| pos0[n])
    //                 | tail_slot[nr] | tail_last[nr] (the tail rows, then the embedding rows)
    // The last two are uploaded only with fan-out: unless row i is sequence i in its own slot.
    int32_t* h = e->h_stage;
    int32_t *h_ids = h, *h_pos = h + T, *h_slt = h + 2 * T, *h_ss = h + 3 * T, *h_sl = h_ss + n_seqs + 1,
            *h_last = h_sl + n_seqs, *h_p0 = h_last + n_seqs, *h_tsl = h_p0 + (c.has_pos0 ? n_seqs : 0),
            *h_tlast = h_tsl + nr;
    bool fan = nr != n_seqs;
    int max_len = 0, max_bias = 0;
    uint64_t copy_tokens = 0;
    KvCopyList fan_copies;                             // the fan-out: source slot -> the slot of each further tail row
    fan_copies.count = 0;
    memcpy(h_ids, c.ids.data(), sizeof(int32_t) * T);
    for (int i = 0; i < n_seqs; ++i) {
        const Chunk::Seq& q = c.seqs[i];
        const int a = q.start, b = q.start + q.len;
        const int reach = q.pos0 + q.len + (q.embeds() ? 0 : 1);       // + the first generated token's position
        if (q.len < 1 || q.pos0 < 0 || reach > e->o.ctx_max || q.slot < 0 || q.slot >= e->Bm) return RR_INVALID_ARGUMENT;
        for (int t = a; t < b; ++t) { h_pos[t] = q.pos0 + t - a; h_slt[t] = q.slot; }
        h_ss[i] = a; h_sl[i] = q.slot; h_last[i] = b - 1;
        if (c.has_pos0) h_p0[i] = q.pos0;
        max_len = std::max(max_len, q.len);
        if (q.embeds()) {
            h_tsl[nt + q.row] = q.slot; h_tlast[nt + q.row] = b - 1;
            fan = fan || nt + q.row != i;
        }
        for (int ch = 0; ch < q.n_tail(); ++ch) {
            const int j = q.row + ch, sl = q.r ? q.r->rows[ch] : q.slot;
            h_tsl[j] = sl; h_tlast[j] = b - 1;
            fan = fan || j != i || sl != q.slot;
            max_bias = std::max(max_bias, (int)q.gen().bias_id.size());
            if (sl == q.slot) continue;
            const int k = fan_copies.count++;          // < nt <= Bm <= KV_COPY_MAX
            fan_copies.src[k] = q.slot; fan_copies.dst[k] = sl; fan_copies.n[k] = q.pos0 + q.len;
            copy_tokens += fan_copies.n[k];
        }
    }
    h_ss[n_seqs] = T;
    const size_t n_ints = (size_t)3 * T + (c.has_pos0 ? 4 : 3) * n_seqs + 1 + (fan ? 2 * nr : 0);
    if (c.copies.count > 0) {
        if (kv_copy_check(c.copies, e->Bm, e->o.ctx_max) != RR_OK) return RR_INVALID_ARGUMENT;
        for (int i = 0; i < c.copies.count; ++i) copy_tokens += c.copies.n[i];
    }
    if (fan_copies.count && kv_copy_check(fan_copies, e->Bm, e->o.ctx_max) != RR_OK) return RR_INVALID_ARGUMENT;
    // the chunk's parameter blocks, at the stride of its tail rows and of its largest bias count
    int mode = c.mode;
    if (max_bias == 0) mode &= ~4;
    else if (!e->d_pf.blk[2]) return RR_INTERNAL;
    if ((mode & 8) && !e->d_pf.blk[3]) return RR_INTERNAL;
    if ((mode & 16) && !e->d_pf.blk[4]) return RR_INTERNAL;
    const ParamBlocks hp = e->h_pf.at(nt, max_bias), dp = e->d_pf.at(nt, max_bias);
    for (const Chunk::Seq& q : c.seqs)
        for (int ch = 0; mode && ch < q.n_tail(); ++ch) hp.put_row(q.row + ch, q.gen(), ch, q.pos0 + q.len, 0.f, 0.f, 0);
    CK(cudaEventRecord(e->ev0, s));
    CK(cudaMemcpyAsync(e->p_ids, h, n_ints * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    e->st.h2d_bytes += n_ints * sizeof(int32_t);
    CK(hp.upload(dp, mode, s, &e->st.h2d_bytes));
    if (scoring) {              // targets | prompt_top per scoring row
        for (const Chunk::Seq& q : c.seqs)
            for (int j = 0; j < q.score_rows(); ++j) {
                e->h_sc_in[q.score_row + j] = q.r->prompt[q.pos0 + 1 + j];
                e->h_sc_in[e->Tmax + q.score_row + j] = q.r->gen.prompt_top;
            }
        for (int half = 0; half < 2; ++half)
            CK(cudaMemcpyAsync(e->d_sc_in + half * e->Tmax, e->h_sc_in + half * e->Tmax, sizeof(int32_t) * n_score,
                               cudaMemcpyHostToDevice, s));
        e->st.h2d_bytes += 2 * sizeof(int32_t) * n_score;
    }
    int32_t *p_ids = e->p_ids, *p_pos = p_ids + T, *p_slt = p_ids + 2 * T, *p_ss = p_ids + 3 * T,
            *p_sl = p_ss + n_seqs + 1, *p_last = p_sl + n_seqs, *p_p0 = p_last + n_seqs;
    const int32_t* p_tsl = fan ? p_ids + (h_tsl - h) : p_sl;       // the tail rows' slots and last-token indices
    const int32_t* p_tlast = fan ? p_ids + (h_tlast - h) : p_last;

    rr_engine::PfPlans& P = e->pf;
    auto launch_rows = [&](const GemmPlan& pl, bool pdl = true) { GemmPlan q = pl; q.rowsA = T; return gemm_launch(q, s, pdl); };
    uint64_t nl = 0;
    if (c.copies.count > 0) {   // cached prefixes of busy slots into this chunk's slots, before any layer reads them
        if (launch_kv_copy(e->kcache, e->vcache, d.n_layers, (long long)e->n_pages * d.n_kv_heads * KV_PAGE, d.n_kv_heads,
                           e->o.ctx_max, e->d_table, e->pps, c.copies, s) != RR_OK)
            return RR_CUDA_ERROR;
        ++nl;
    }
    launch_embed(p_ids, (const __nv_bfloat16*)e->embed, e->px, T, d.hidden, nullptr, s); ++nl;
    // layer 0's operand in the deferred form: bf16(x * gamma), sum(x^2) in partial 0
    launch_add_rmsnorm_pf(e->px, (const __nv_bfloat16*)e->norm_attn[0], e->pxn, T, d.hidden, d.rms_eps, s, e->p_rowss,
                          e->pf_parts); ++nl;
    for (int l = 0; l < d.n_layers; ++l) {
        __nv_bfloat16* kc = e->kcache + (size_t)l * e->kv_layer_stride;
        __nv_bfloat16* vc = e->vcache + (size_t)l * e->kv_layer_stride;
        if (e->fuse_rope_pf) {
            P.qkv[l].rope.slot = p_slt; P.qkv[l].rope.pos = p_pos;
        }
        // FP8: layer l's weights into the scratch.  The dequantize and the QKV GEMM after it are plain launches: the
        // dequantize starts after the previous layer's GEMMs have finished reading the scratch, and the QKV GEMM (and so
        // every later kernel, whose PDL weight prefetch runs before griddepcontrol.wait) after the scratch is complete.
        if (e->fp8) {
            if (launch_dequant_layer(e, l, scoring, s) != RR_OK) return RR_CUDA_ERROR; ++nl;
        }
        if (launch_rows(P.qkv[l], !e->fp8) != RR_OK) return RR_CUDA_ERROR; ++nl;
        RopeArgs ra;
        ra.qkv = part_bf16(e->pqkv, e->nqkv);
        ra.q_out = e->pq; ra.k_cache = kc; ra.v_cache = vc; ra.slot = p_slt; ra.pos = p_pos; ra.rows = T;
        ra.n_heads = d.n_heads; ra.n_kv_heads = d.n_kv_heads; ra.ctx_max = e->o.ctx_max; ra.theta = d.rope_theta;
        ra.table = e->rope_table; ra.head_dim = d.head_dim; ra.page_table = e->d_table; ra.pages_per_slot = e->pps;
        if (!e->fuse_rope_pf) { launch_rope_kv(ra, s); ++nl; }
        if (nr == 0 && !scoring && l + 1 == d.n_layers) break;    // every layer's KV is written
        PrefillAttnArgs pa = e->pf_attn[l];          // per-layer operands, scale and TMA maps made at create (pf_attn_layer)
        pf_attn_chunk(&pa, e->pattn, p_ss, p_sl, c.has_pos0 ? p_p0 : nullptr, n_seqs, max_len);
        if (launch_prefill_attn(pa, s) != RR_OK) return RR_CUDA_ERROR; ++nl;
        if (l + 1 == d.n_layers && nr > 0) {
            // ---- trimmed tail: the tail and embedding rows through O, MLP, final norm (decode-orientation kernels, decode
            // buffers; every kernel is row-independent, so a row's bits do not depend on the others).  The unfused kernels
            // even with fuse_mlp: the fused kernel's down GEMM sums in a different order.
            launch_gather_last(e->pattn, e->px, p_tlast, nr, e->nq, d.hidden, e->attn_out, e->x, s); ++nl;
            if (enqueue_o_mlp(e, l, nr, s, &nl) != RR_OK) return RR_CUDA_ERROR;
        }
        if (l + 1 == d.n_layers && !scoring) break;    // a scoring chunk runs the whole last layer as well
        if (launch_rows(P.o[l]) != RR_OK) return RR_CUDA_ERROR; ++nl;
        if (launch_rows(P.gu[l]) != RR_OK) return RR_CUDA_ERROR; ++nl;
        if (!e->fuse_silu) { launch_silu_mul(part_bf16(e->pgu, 2 * d.inter), e->pact, T, d.inter, s); ++nl; }
        if (launch_rows(P.down[l]) != RR_OK) return RR_CUDA_ERROR; ++nl;
    }
    if (scoring) {              // lm_head and log-softmax over the scoring rows, SCORE_ROWS rows of one sequence at a time
        const int S = std::min(SCORE_ROWS, e->Tmax), V = d.vocab;
        for (const Chunk::Seq& q : c.seqs) {
            const int r0 = q.start;
            for (int b = 0; b < q.score_rows(); b += S) {
                const int nb = std::min(S, q.score_rows() - b), o = q.score_row + b;
                GemmPlan hd;
                if (gemm_plan_init(&hd, e->pxn + (size_t)(r0 + b) * d.hidden, nb, d.hidden, e->lm_head, V, d.hidden, d.hidden,
                                   e->sc_logits, V, 0, 1, OUT_ROWMAJOR_F32, PF_BN) != RR_OK)
                    return RR_INVALID_ARGUMENT;
                pf_norm_consumer(&hd.rope, e->p_rowss + (size_t)(r0 + b) * e->pf_parts, d.hidden, d.rms_eps);
                if (gemm_launch(hd, s) != RR_OK) return RR_CUDA_ERROR; ++nl;
                launch_logprobs(e->sc_logits, V, nb, V, e->d_sc_in + e->Tmax + o, LP_MAX_TOP, e->sc_ws,
                                e->d_sc_lp + (size_t)o * LP_MAX_TOP, e->d_sc_id + (size_t)o * LP_MAX_TOP, s, e->d_sc_in + o,
                                e->d_sc_tlp + o);
                nl += LP_LAUNCHES;
            }
        }
        const size_t n = (size_t)n_score * LP_MAX_TOP;
        CK(cudaMemcpyAsync(e->h_sc_tlp, e->d_sc_tlp, sizeof(float) * n_score, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(e->h_sc_lp, e->d_sc_lp, sizeof(float) * n, cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(e->h_sc_id, e->d_sc_id, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, s));
        e->st.d2h_bytes += sizeof(float) * n_score + (sizeof(float) + sizeof(int32_t)) * n;
    }
    if (fan_copies.count) {     // every layer's KV of the prompts is written: fan it out before any decode step reads it
        if (launch_kv_copy(e->kcache, e->vcache, d.n_layers, (long long)e->n_pages * d.n_kv_heads * KV_PAGE, d.n_kv_heads,
                           e->o.ctx_max, e->d_table, e->pps, fan_copies, s) != RR_OK)
            return RR_CUDA_ERROR;
        ++nl;
    }
    if (nt > 0) {
        if (gemm_launch(e->pl_head, s) != RR_OK) return RR_CUDA_ERROR; ++nl;      // B = e->xn (rows 0..nt-1)
        nl += enqueue_tail(e, dp, nt, mode, e->p_first, nullptr, nullptr, dp.pos(), nullptr, s, p_tsl);
        launch_activate_rows(p_tsl, e->p_first, p_pos, p_tlast, nt, e->d_tok, e->d_pos, e->d_slot, s); ++nl;
        const int rc = enqueue_readback(e, e->p_first, nt, mode, s);
        if (rc != RR_OK) return rc;
    }
    if (ne > 0) {               // the embedding rows' final-norm rows, pooled and read back
        launch_embed_pool(e->xn + (size_t)nt * d.hidden, d.hidden, nullptr, ne, d.hidden, e->d_emb, d.hidden, s); ++nl;
        CK(cudaMemcpyAsync(e->h_emb, e->d_emb, sizeof(float) * (size_t)ne * d.hidden, cudaMemcpyDeviceToHost, s));
        e->st.d2h_bytes += sizeof(float) * (size_t)ne * d.hidden;
    }
    if (logits_host) {
        CK(cudaMemcpyAsync(logits_host, e->logits, sizeof(float) * (size_t)n_seqs * d.vocab, cudaMemcpyDeviceToHost, s));
    }
    CK(cudaEventRecord(e->ev1, s));
    CK(cudaStreamSynchronize(s));
    float ms = 0;
    cudaEventElapsedTime(&ms, e->ev0, e->ev1);
    e->st.prefill_ms_total += ms;
    e->st.prefill_chunks += 1;
    e->st.prefill_tokens += T;
    e->st.kv_copy_tokens += copy_tokens;
    e->st.kernel_launches += nl;
    for (int j = 0; j < nt; ++j) {
        if (first_tok_host) first_tok_host[j] = e->h_tok[j];
        e->h_slot_mirror[h_tsl[j]] = h_tsl[j];
    }
    return RR_OK;
}

// ---------------------------------------------------------------- KV page pool (caller holds e->mu)
static int pages_for(int tokens) { return (tokens + KV_PAGE - 1) / KV_PAGE; }

// The ring of a windowed engine: R = ceil((W + Tmax - 2) / 64) + 1 pages.  A prefill piece of len <= Tmax rows at positions
// pos0 .. pos0 + len - 1 reads keys from pos0 - W + 1 on and writes its own rows in the QKV epilogue before attention reads
// them, so the positions live at once are the W + len - 1 <= W + Tmax - 1 from pos0 - W + 1 to pos0 + len - 1, and n
// consecutive positions touch at most ceil((n - 1) / 64) + 1 pages: R pages, which are distinct mod R.  A decode step
// needs the pages of W positions, fewer.  So mapping logical page p to pages[p mod R] never lets a write land on a page
// still read, and R - 1 pages fail for the alignment that touches R pages (tests/test_sliding_window_cpu.py).
static int ring_pages(int window, int tmax) { return window > 0 ? pages_for(window + tmax - 2) + 1 : 0; }

// Pages one choice reaching `reach` positions reserves: ceil(reach / 64), or the ring when that is smaller.
static int choice_pages(const rr_engine* e, int reach) {
    const int n = pages_for(reach);
    return e->ring > 0 && n > e->ring ? e->ring : n;
}
static bool ring_request(const rr_engine* e, const Request* r) {
    return e->ring > 0 && pages_for((int)r->prompt.size() + r->max_new) > e->ring;
}

// Slot b holds exactly n pages: it keeps its first ones, returns extra ones from the end and takes missing ones from the free
// stack (the caller made sure there are enough).  Pages go back in the reverse of the order they were taken, so a slot
// that returns its pages and takes as many again gets the same ones: its table row does not change and is not copied.
static void resize_pages(rr_engine* e, int b, int n) {
    std::vector<int32_t>& P = e->slot_pages[b];
    while ((int)P.size() > n) { e->free_pages.push_back(P.back()); P.pop_back(); }
    while ((int)P.size() < n) {
        const int32_t pg = e->free_pages.back();
        e->free_pages.pop_back();
        int32_t& t = e->h_table[(size_t)b * e->pps + P.size()];
        if (t != pg) { t = pg; e->table_dirty[b] = 1; }
        P.push_back(pg);
    }
}

// Pages a request could get now: the free ones and those of the free slots.
static int pages_available(const rr_engine* e) {
    int n = (int)e->free_pages.size();
    for (int b = 0; b < e->Bm; ++b)
        if (!e->row_req[b]) n += (int)e->slot_pages[b].size();
    return n;
}

// Until `need` pages are free: take back every page of a free slot, first of slots with no retained prefix (lowest index
// first), then least recently used by retained_used, and forget each such slot's prefix.
static void reclaim_pages(rr_engine* e, int need) {
    while ((int)e->free_pages.size() < need) {
        int pick = -1;
        for (int b = 0; b < e->Bm; ++b) {
            if (e->row_req[b] || e->slot_pages[b].empty()) continue;
            const bool empty = !e->o.prefix_cache || e->retained[b].empty();
            if (empty) { pick = b; break; }
            if (pick < 0 || e->retained_used[b] < e->retained_used[pick]) pick = b;
        }
        if (pick < 0) return;                              // cannot happen: the caller checked pages_available
        if (e->o.prefix_cache) e->retained[pick].clear();
        resize_pages(e, pick, 0);
    }
}

// The request just took the slots r->rows: give each choice_pages pages, shrinking before growing so the pages a slot
// returns serve the others first.  Entries [0, pages) of a slot's table row always name its pages in order; a ring
// request's row also maps every later logical page p to pages[p % ring] (rewritten, and so uploaded, only where it changes).
static void take_pages(rr_engine* e, const Request* r) {
    const int need = choice_pages(e, (int)r->prompt.size() + r->max_new);
    int missing = 0;
    for (int b : r->rows) {
        if ((int)e->slot_pages[b].size() > need) resize_pages(e, b, need);
        missing += need - (int)e->slot_pages[b].size();
    }
    reclaim_pages(e, missing);
    const bool ring = ring_request(e, r);
    for (int b : r->rows) {
        resize_pages(e, b, need);
        for (int p = need; ring && p < e->pps; ++p) {
            int32_t& t = e->h_table[(size_t)b * e->pps + p];
            const int32_t pg = e->slot_pages[b][p % need];
            if (t != pg) { t = pg; e->table_dirty[b] = 1; }
        }
    }
}

// Slot b's request is done with it: keep the pages of its retained prefix (none without prefix caching), return the rest.
static void trim_pages(rr_engine* e, int b) {
    resize_pages(e, b, e->o.prefix_cache ? pages_for((int)e->retained[b].size()) : 0);
}

// Caller holds gpu_mu.  Copies the changed rows of the page table to the device on the engine stream, ahead of the work
// that reads them.
static int upload_table(rr_engine* e) {
    std::lock_guard<std::mutex> lk(e->mu);
    for (int b = 0; b < e->Bm; ++b) {
        if (!e->table_dirty[b]) continue;
        const size_t off = (size_t)b * e->pps, bytes = sizeof(int32_t) * e->pps;
        CK(cudaMemcpyAsync(e->d_table + off, e->h_table + off, bytes, cudaMemcpyHostToDevice, e->stream));
        e->st.h2d_bytes += bytes;
        e->table_dirty[b] = 0;
    }
    return RR_OK;
}

// Caller holds gpu_mu.  Low-level calls: slot slots[i] must hold the pages of positions [0, n_pos[i]).  RR_INVALID_ARGUMENT,
// nothing changed, when the free pages do not cover that.
static int grow_pages(rr_engine* e, const int32_t* slots, const int* n_pos, int n) {
    std::lock_guard<std::mutex> lk(e->mu);
    std::vector<int> want(e->Bm, 0);
    for (int i = 0; i < n; ++i) want[slots[i]] = std::max(want[slots[i]], pages_for(n_pos[i]));
    int missing = 0;
    for (int b = 0; b < e->Bm; ++b) missing += std::max(0, want[b] - (int)e->slot_pages[b].size());
    if (missing > (int)e->free_pages.size()) return RR_INVALID_ARGUMENT;
    for (int b = 0; b < e->Bm; ++b)
        if (want[b] > (int)e->slot_pages[b].size()) resize_pages(e, b, want[b]);
    return RR_OK;
}

// ---------------------------------------------------------------- worker (continuous batching)
struct DoneNote { uint64_t tag, ticket; int status, n_gen; };

// Caller holds e->mu.  Decode row b is taken (r) or freed (nullptr): write row b of the mirror from r's parameters or the
// defaults.  A block is marked dirty only when the row uses it before or after: the other rows of a mirror hold the
// defaults, as a request that does not use the block does (GenParams::set), so they never need a copy.  A freed row's
// mirror row holds the defaults, so freeing a row that never held parameters changes nothing.
static void set_row_params(rr_engine* e, int b, const Request* r, int choice = 0) {
    static const GenParams plain;
    const GenParams& p = r ? r->gen : plain;
    e->rows_dirty |= e->h_rows.row_mode(b) | step_mode(p);
    e->h_rows.put_row(b, p, choice, 0, p.fpen, p.ppen, r ? (int)r->prompt.size() : 0);
}

// Before a decode step: copy each parameter block the step reads (step_mode bits) whose mirror changed.
static void upload_row_params(rr_engine* e, int mode) {
    e->h_rows.upload(e->d_rows, mode & e->rows_dirty, e->stream, &e->st.h2d_bytes);
    e->rows_dirty &= ~mode;
}

// Caller holds e->mu.  Returns the hook call to make once the lock is released (tag == 0 and no hook: nothing).
static void finish_request(rr_engine* e, Request* r, int status, std::vector<DoneNote>* notes = nullptr) {
    for (int c = 0; c < r->n_choices; ++c) {      // ended from outside: a running choice keeps what a reader may have seen
        if (r->finish[c] >= 0) continue;
        const size_t n = (size_t)r->visible(c);
        r->out[c].resize(n);
        if (r->gen.logprobs()) { r->lp[c].resize(n * r->gen.lp_width()); r->lp_id[c].resize(n * r->gen.lp_width()); }
        r->hold[c] = 0;
    }
    r->status = status;
    r->t_done = now_s(e);
    r->done = true;
    if (notes && e->hook) notes->push_back(DoneNote{r->tag, r->ticket, status, r->n_returned()});
    if (r->detached) {                   // cancelled by its owner: nobody waits for it
        e->table.erase(r->ticket);
        delete r;
    }
}
static void run_hooks(rr_engine* e, std::vector<DoneNote>& notes) {
    for (const DoneNote& n : notes) e->hook(e->hook_ctx, n.tag, n.ticket, n.status, n.n_gen);
    notes.clear();
}

// Caller holds e->mu.  Frees the decode row of choice c of r, if it still has one: inactive from the next step, parameters
// back to the defaults, free for the next waiting prompt.
static void release_row(rr_engine* e, Request* r, int c) {
    const int b = r->rows[c];
    if (b < 0) return;
    e->row_req[b] = nullptr; e->h_slot_mirror[b] = -1;
    trim_pages(e, b);
    set_row_params(e, b, nullptr);
    e->slots_dirty = true;
    r->rows[c] = -1;
}

// Caller holds e->mu.  Frees every decode row r still has and finishes r with `status`.
static void release_request(rr_engine* e, Request* r, int status, std::vector<DoneNote>* notes) {
    for (int c = 0; c < (int)r->rows.size(); ++c) release_row(e, r, c);
    r->rows.clear();
    if (e->in_progress == r) e->in_progress = nullptr;
    finish_request(e, r, status, notes);
}

// Caller holds e->mu.  Prefix caching: a low-level call cleared the index after r was admitted, so its match and the KV of
// its done pieces may be stale.  r gives its rows and pages back (nothing retained) and goes back to the head of the queue,
// to start again from position 0.
static void requeue(rr_engine* e, Request* r) {
    for (int b : r->rows) { e->row_req[b] = nullptr; resize_pages(e, b, 0); }
    r->rows.clear(); r->n_cached = 0; r->n_done = 0;
    if (e->in_progress == r) e->in_progress = nullptr;
    e->waiting.push_front(r);
}

// Caller holds e->mu.  Appends the token read back for row `row` to choice c of r, with its pairs (h_lp / h_lp_id row
// `row`, and for a sampled request the drawn token's own pair from h_tok_lp) if r asked for logprobs.  With stop sequences
// it takes the row's cut / hold (h_stop): a hit finishes the choice with reason stop, its tokens and pairs truncated to the
// cut.  Otherwise, in JSON mode, the token that closed the top-level object (h_json_done) finishes it with reason stop, and
// otherwise max_new tokens finish it with reason length.  True when the choice finished.
static bool take_token(rr_engine* e, Request* r, int c, int row) {
    r->out[c].push_back(e->h_tok[row]);
    if (r->gen.logprobs()) {
        const int k = r->gen.top_lp > 1 ? r->gen.top_lp : 1;
        const float* v = e->h_lp + (size_t)row * LP_MAX_TOP;
        const int32_t* id = e->h_lp_id + (size_t)row * LP_MAX_TOP;
        r->lp[c].insert(r->lp[c].end(), v, v + k);
        r->lp_id[c].insert(r->lp_id[c].end(), id, id + k);
        if (r->gen.sampled()) { r->lp[c].push_back(e->h_tok_lp[row]); r->lp_id[c].push_back(r->out[c].back()); }
    }
    e->st.generated_tokens += 1;
    const int cut = r->gen.stops() ? e->h_stop[row] : -1;
    if (cut >= 0 && cut < (int)r->out[c].size()) {
        r->out[c].resize(cut);
        if (r->gen.logprobs()) {
            r->lp[c].resize((size_t)cut * r->gen.lp_width()); r->lp_id[c].resize((size_t)cut * r->gen.lp_width());
        }
        r->finish[c] = 1;
    } else if (r->gen.json() && e->h_json_done[row]) {
        r->finish[c] = 1;
    } else if ((int)r->out[c].size() >= r->max_new) {
        r->finish[c] = 0;
    } else if (r->gen.stops()) {
        r->hold[c] = std::min(std::max(e->h_stop[e->Bm + row], 0), (int)r->out[c].size());
    }
    return r->finish[c] >= 0;
}

// Caller holds e->mu.  Prefix caching: the slot a prompt p is admitted into and how many of its tokens are cached there.
// m_b = the longest common prefix of retained[b] and p, capped at |p| - 1 (the last prompt token is always prefilled: its
// logits give the first token); a hit needs m_b >= PREFIX_MIN.  The best m wins, then a free slot, then the lower index.
// A hit on a free slot takes that slot as it is; a hit on a busy slot (*src = it) copies m tokens into the slot a miss
// takes: the lowest free slot with nothing retained, else the free slot whose prefix was used least recently.  Slots taken
// in the current chunk have nothing retained, so requests of one chunk never share.  false: no free slot.
// pick_slot_miss: the slot a miss takes (-1: none free); the further choices of a request take their slots by it.
static int pick_slot_miss(const rr_engine* e) {
    int fresh = -1;
    for (int b = 0; b < e->Bm; ++b) {
        if (e->row_req[b]) continue;
        if (e->retained[b].empty()) return b;
        if (fresh < 0 || e->retained_used[b] < e->retained_used[fresh]) fresh = b;
    }
    return fresh;
}
static bool pick_slot_cached(const rr_engine* e, const std::vector<int32_t>& p, int* slot, int* m, int* src) {
    const int cap = (int)p.size() - 1;
    int best = -1, best_m = 0;
    bool best_free = false;
    for (int b = 0; b < e->Bm; ++b) {
        const std::vector<int32_t>& R = e->retained[b];
        const int lim = (int)R.size() < cap ? (int)R.size() : cap;
        int k = 0;
        while (k < lim && R[k] == p[k]) ++k;
        if (k < PREFIX_MIN) continue;
        const bool fr = e->row_req[b] == nullptr;
        if (k > best_m || (k == best_m && fr && !best_free)) { best = b; best_m = k; best_free = fr; }
    }
    *m = best >= 0 ? best_m : 0;
    *src = -1;
    if (best >= 0 && best_free) { *slot = best; return true; }
    const int fresh = pick_slot_miss(e);
    if (fresh < 0) return false;
    *slot = fresh;
    *src = best;
    return true;
}

// Caller holds gpu_mu.  A low-level call writes slots behind the index's back: forget every retained prefix.
static void forget_prefixes(rr_engine* e) {
    if (!e->o.prefix_cache) return;
    std::lock_guard<std::mutex> lk(e->mu);
    for (auto& R : e->retained) R.clear();
    ++e->index_epoch;
}

// Caller holds no lock.  The first scoring request gets its buffers before it is admitted.  If they cannot be had, the
// waiting scoring requests fail, the engine serves on, and this returns false.
static bool alloc_scoring(rr_engine* e, std::vector<DoneNote>* notes) {
    if (e->sc_logits) return true;
    {
        std::lock_guard<std::mutex> lk(e->mu);
        if (std::none_of(e->waiting.begin(), e->waiting.end(), [](const Request* r) { return r->gen.scores(); })) return true;
    }
    int rc;
    {
        std::lock_guard<std::mutex> gl(e->gpu_mu);
        std::lock_guard<std::mutex> dl(device_mutex(e->o.device));
        rc = ensure_score_buffers(e);
    }
    if (rc == RR_OK) return true;
    std::lock_guard<std::mutex> lk(e->mu);
    for (auto it = e->waiting.begin(); it != e->waiting.end();) {
        Request* r = *it;
        if (!r->gen.scores()) { ++it; continue; }
        it = e->waiting.erase(it);
        finish_request(e, r, RR_INTERNAL, notes);
    }
    e->cv_done.notify_all();
    return false;
}

// The rows at the start of a round: held, decoding (not the prompt in progress's), and the step_mode bits of the decoding.
struct RowCount { int active = 0, decoding = 0, step = 0; };

// Caller holds e->mu.  Sends the prompt in progress back to the queue if a low-level call cleared the index since its
// admission, frees the rows of cancelled requests and counts the rest.
static RowCount sweep_rows(rr_engine* e, std::vector<DoneNote>* notes) {
    Request* ip = e->in_progress;
    if (ip && !ip->cancel && e->o.prefix_cache && ip->epoch != e->index_epoch) requeue(e, ip);
    RowCount n;
    for (int b = 0; b < e->Bm; ++b) {
        Request* r = e->row_req[b];
        if (!r) continue;
        if (r->cancel) {                               // rr_engine_cancel: free the rows, keep what was generated
            release_request(e, r, RR_CANCELLED, notes);
            continue;
        }
        ++n.active;
        if (r == e->in_progress) continue;             // held for its next piece: no token yet
        ++n.decoding;
        n.step |= step_mode(r->gen);
    }
    return n;
}

// Caller holds e->mu.  Fills chunk c: the next piece of the prompt in progress first, then waiting requests in FIFO
// order while the head fits; nothing overtakes it.  Returns the rows held after admission (`active` before).
static int admit(rr_engine* e, Chunk* c, int active) {
    if (Request* ip = e->in_progress) {               // its next piece goes first: min(Tmax, remaining) tokens
        const int n = std::min(e->Tmax, (int)ip->prompt.size() - ip->n_done);
        const bool last = ip->n_done + n == (int)ip->prompt.size();
        c->add(ip, ip->rows[0], ip->n_done, ip->prompt.data() + ip->n_done, n, last);
        c->has_pos0 = true;
        if (last) e->in_progress = nullptr;
    }
    int b = 0;
    while (!e->waiting.empty()) {
        Request* r = e->waiting.front();
        if (r->n_choices > e->Bm - active) break;      // its choices take that many free rows, all at its admission
        if (r->gen.scores() && !e->sc_logits) break;   // submitted since alloc_scoring: the next round allocates
        int m = 0, src = -1;
        const bool ring = ring_request(e, r);           // the ring overwrites its prompt: no prefix hit, nothing kept
        if (e->o.prefix_cache && (ring || r->gen.scores())) {     // scoring: every prompt row goes through lm_head
            if ((b = pick_slot_miss(e)) < 0) break;
        } else if (e->o.prefix_cache) {
            if (!pick_slot_cached(e, r->prompt, &b, &m, &src)) break;
        } else {
            while (b < e->Bm && e->row_req[b] != nullptr) ++b;
            if (b >= e->Bm) break;
        }
        // a chunk holds Tmax uncached tokens; with no prompt in progress, one that does not fit the room left starts with a
        // piece that fills it
        int n = (int)r->prompt.size() - m;
        const int room = e->Tmax - (int)c->ids.size();
        if (n > room) {
            if (e->in_progress || room == 0) break;
            n = room;
        }
        // every choice reserves its pages now; a request that does not fit waits at the head of the queue
        if (r->n_choices * choice_pages(e, (int)r->prompt.size() + r->max_new) > pages_available(e)) break;
        e->waiting.pop_front();
        r->n_cached = m;
        r->n_done = m;
        if (e->o.prefix_cache) {
            if (m > 0) e->retained_used[src >= 0 ? src : b] = ++e->lru_clock;
            if (src >= 0) {
                const int k = c->copies.count++;
                c->copies.src[k] = src; c->copies.dst[k] = b; c->copies.n[k] = m;
            }
        }
        for (int ch = 0; ch < r->n_choices; ++ch) {    // choice 0 in the prompt's slot, the others in free ones
            if (ch > 0) {
                if (e->o.prefix_cache) b = pick_slot_miss(e);
                else while (e->row_req[b] != nullptr) ++b;
            }
            e->row_req[b] = r;
            e->row_choice[b] = ch;
            r->rows.push_back(b);
            if (e->o.prefix_cache) e->retained[b].clear();   // rewritten by this prompt; set again once it succeeds
        }
        take_pages(e, r);
        const bool last = m + n == (int)r->prompt.size();
        c->add(r, r->rows[0], m, r->prompt.data() + m, n, last);
        if (!last) { e->in_progress = r; r->epoch = c->epoch; }
        active += r->n_choices;
    }
    return active;
}

// Caller holds gpu_mu.  The lazily allocated buffers that the tail rows of step_mode bits `mode` read, and the embedding
// rows' if there are any.
static int ensure_chunk_buffers(rr_engine* e, int mode, bool embeds) {
    int rc = (mode & 4) ? ensure_pen_buffers(e) : RR_OK;
    if (rc == RR_OK && (mode & 8)) rc = ensure_stop_buffers(e);
    if (rc == RR_OK && (mode & 16)) rc = ensure_json_buffers(e);
    return rc == RR_OK && embeds ? ensure_embed_buffers(e) : rc;
}

// Caller holds gpu_mu and the device lock.  Runs chunk c and hands its results to its requests: scores, embeddings,
// first tokens, retained prefixes; a request whose prompt is done and has nothing left to decode is released, and every
// request of a failed chunk ends with RR_INTERNAL.  Returns whether a prompt is still in progress.
static bool run_chunk(rr_engine* e, const Chunk& c, std::vector<DoneNote>* notes) {
    if (e->o.prefix_cache) {
        // a low-level call took the GPU between admission and here and cleared the index: its matches may be stale, so
        // the chunk goes back to the head of the queue and is admitted again (a prompt in progress from position 0)
        std::lock_guard<std::mutex> lk(e->mu);
        if (e->index_epoch != c.epoch) {
            for (size_t i = c.seqs.size(); i-- > 0;) requeue(e, c.seqs[i].r);
            return false;
        }
    }
    int rc = upload_table(e);
    if (rc == RR_OK) rc = ensure_chunk_buffers(e, c.mode, c.n_emb > 0);
    if (rc == RR_OK) rc = run_prefill(e, c, nullptr, nullptr);
    const double t = now_s(e);
    std::lock_guard<std::mutex> lk(e->mu);
    for (const Chunk::Seq& q : c.seqs) {
        Request* r = q.r;
        if (rc != RR_OK) {
            release_request(e, r, RR_INTERNAL, notes);
            continue;
        }
        const size_t k = (size_t)r->gen.score_width();
        for (int j = 0; j < q.score_rows(); ++j) {
            const size_t p = (size_t)q.pos0 + j, o = (size_t)q.score_row + j;
            r->ptgt[p] = e->h_sc_tlp[o];
            memcpy(&r->plp[p * k], e->h_sc_lp + o * LP_MAX_TOP, sizeof(float) * k);
            memcpy(&r->plp_id[p * k], e->h_sc_id + o * LP_MAX_TOP, sizeof(int32_t) * k);
        }
        r->n_done = q.pos0 + q.len;
        if (!q.last) continue;                         // the prompt in progress: its next piece leads the next chunk
        if (e->o.prefix_cache && !ring_request(e, r)) {   // every choice's slot holds the prompt's prefill-written KV
            for (int b : r->rows) { e->retained[b] = r->prompt; e->retained_used[b] = ++e->lru_clock; }
            if (r->n_cached > 0) { e->st.prefix_hits += 1; e->st.prefix_cached_tokens += r->n_cached; }
        }
        r->t_first = t;
        if (r->embed) {                                // done: its row is free at once, it never decodes
            const float* v = e->h_emb + (size_t)q.row * e->d.hidden;
            r->emb.assign(v, v + e->d.hidden);
            r->finish[0] = 0;
            release_request(e, r, RR_OK, notes);
            continue;
        }
        for (int ch = 0; ch < r->n_choices; ++ch) {
            if (take_token(e, r, ch, q.row + ch)) release_row(e, r, ch);
            else set_row_params(e, r->rows[ch], r, ch);
        }
        if (r->all_finished()) release_request(e, r, RR_OK, notes);
    }
    e->cv_done.notify_all();
    return e->in_progress != nullptr;
}

// Caller holds gpu_mu and the device lock.  One decode step for every active row, of step_mode bits `step`, and its
// tokens taken; a row whose choice finished is free for the next waiting prompt at once.
static void run_step(rr_engine* e, int step, std::vector<DoneNote>* notes) {
    cudaStream_t s = e->stream;
    if (e->slots_dirty) {
        memcpy(e->h_stage, e->h_slot_mirror.data(), sizeof(int32_t) * e->Bm);
        cudaMemcpyAsync(e->d_slot, e->h_stage, sizeof(int32_t) * e->Bm, cudaMemcpyHostToDevice, s);
        e->st.h2d_bytes += sizeof(int32_t) * e->Bm;
        e->slots_dirty = false;
    }
    upload_row_params(e, step);
    int rc = upload_table(e);
    cudaEventRecord(e->ev0, s);
    if (rc == RR_OK) rc = run_decode_step(e, step);
    cudaEventRecord(e->ev1, s);
    const int rb = enqueue_readback(e, e->d_tok, e->Bm, step, s);     // outside ev0 .. ev1: decode_ms_total excludes it
    if (rc == RR_OK) rc = rb;
    cudaError_t se = cudaStreamSynchronize(s);
    if (se != cudaSuccess) { rr::note_cuda_error(se); rc = RR_CUDA_ERROR; }
    float ms = 0;
    cudaEventElapsedTime(&ms, e->ev0, e->ev1);
    e->st.decode_ms_total += ms;
    e->st.decode_steps += 1;
    {
        std::lock_guard<std::mutex> lk(e->mu);
        for (int b = 0; b < e->Bm; ++b) {              // a released request's later rows are already free
            Request* r = e->row_req[b];
            if (!r) continue;
            if (rc != RR_OK) { release_request(e, r, RR_INTERNAL, notes); continue; }
            if (r == e->in_progress) continue;         // its rows are inactive on the device
            const int c = e->row_choice[b];
            if (!take_token(e, r, c, b)) continue;
            release_row(e, r, c);
            if (r->all_finished()) release_request(e, r, RR_OK, notes);
        }
    }
    e->cv_done.notify_all();
}

// Prefill first (best TTFT): a round that admits a chunk runs it and looks for more waiting prompts before decoding.  But
// a running reply waits at most one chunk between tokens, however many pieces a long prompt takes.  Done hooks run outside
// e->mu, before the worker idles.
static void worker_main(rr_engine* e) {
    cudaSetDevice(e->o.device);
    std::vector<DoneNote> notes;
    Chunk chunk;
    bool decode_due = false;         // the last chunk left a prompt in progress: one decode step goes before the next chunk
    while (!e->stop.load()) {
        run_hooks(e, notes);
        if (!alloc_scoring(e, &notes)) continue;
        RowCount rows;
        {
            std::unique_lock<std::mutex> lk(e->mu);
            rows = sweep_rows(e, &notes);
            if (e->waiting.empty() && rows.active == 0) {
                if (!notes.empty()) continue;              // report the requests a cancel just ended before idling
                e->st.queued = 0; e->st.active_rows = 0;   // idle: every row is free and every done hook has run
                e->cv_work.wait_for(lk, std::chrono::milliseconds(50));
                continue;
            }
            const bool decode_first = decode_due && rows.decoding > 0;
            decode_due = false;
            chunk.reset(e->index_epoch, e->o.prefix_cache);
            e->st.active_rows = decode_first ? rows.active : admit(e, &chunk, rows.active);
            e->st.queued = (int)e->waiting.size();
        }
        std::lock_guard<std::mutex> gl(e->gpu_mu);
        std::lock_guard<std::mutex> dl(device_mutex(e->o.device));
        if (!chunk.seqs.empty()) decode_due = run_chunk(e, chunk, &notes);
        else if (rows.decoding > 0) run_step(e, rows.step, &notes);
    }
    run_hooks(e, notes);
}

// ---------------------------------------------------------------- C-ABI
RR_API int rr_engine_create(const rr_model_desc* desc, const rr_model_weights* w, const rr_engine_opts* opts,
                            rr_engine** out) {
    if (!desc || !w || !opts || !out) return RR_INVALID_ARGUMENT;
    const rr_model_desc& d = *desc;
    // head_dim: 64..128, multiple of 16; attention operands (q, KV cache rows) are zero-padded to 128
    if (d.head_dim < 64 || d.head_dim > 128 || d.head_dim % 16 || d.n_heads % d.n_kv_heads || d.hidden % 64 ||
        d.inter % 64 || d.n_layers < 1)
        return RR_INVALID_ARGUMENT;
    const int G = d.n_heads / d.n_kv_heads;
    if (!(G == 1 || G == 2 || G == 4 || G == 8)) return RR_INVALID_ARGUMENT;
    if (d.hidden > 8192) return RR_INVALID_ARGUMENT;      // add_rmsnorm_kernel keeps one row in registers (rr_elementwise.cu)
    // the logits tail reads each row of [rows][vocab] fp32 logits with 16-byte loads: every row must start 16-byte aligned
    if (d.vocab < 4 || d.vocab % 4) return RR_INVALID_ARGUMENT;
    if (opts->max_batch < 1 || opts->max_batch > MAX_BATCH || opts->ctx_max < 64 || opts->ctx_max % 64)
        return RR_INVALID_ARGUMENT;
    // the KV pool: 0 = one ctx_max per decode row, else a multiple of 64 in [ctx_max, max_batch x ctx_max]
    const long long kv_full = (long long)opts->max_batch * opts->ctx_max;
    const long long kv_tokens = opts->kv_cache_tokens == 0 ? kv_full : opts->kv_cache_tokens;
    if (kv_tokens % KV_PAGE || kv_tokens < opts->ctx_max || kv_tokens > kv_full) return RR_INVALID_ARGUMENT;
    if (w->sliding_window < 0) return RR_INVALID_ARGUMENT;
    const bool fp8 = (w->flags & RR_WEIGHTS_FP8_E4M3) != 0;
    if (fp8) {      // e4m3 projections the decode GEMMs can stream, and their scales
        if (!w->wqkv_scale || !w->wo_scale || !w->wgu_scale || !w->wdown_scale) return RR_INVALID_ARGUMENT;
        const int nq = d.n_heads * d.head_dim;
        for (int l = 0; l < d.n_layers; ++l) {
            if (!fp8_weight_ok(w->wqkv[l], d.hidden) || !fp8_weight_ok(w->wo[l], nq) || !fp8_weight_ok(w->wgu[l], d.hidden) ||
                !fp8_weight_ok(w->wdown[l], d.inter))
                return RR_INVALID_ARGUMENT;
            if (!w->wqkv_scale[l] || !w->wo_scale[l] || !w->wgu_scale[l] || !w->wdown_scale[l]) return RR_INVALID_ARGUMENT;
        }
    }
    CK(cudaSetDevice(opts->device));
    rr_engine* e = new (std::nothrow) rr_engine();
    if (!e) return RR_INTERNAL;
    e->d = d; e->o = *opts;
    e->Bm = opts->max_batch;
    e->bn_dec = pick_bn(e->Bm);
    e->nq = d.n_heads * d.head_dim; e->nkv_dim = d.n_kv_heads * d.head_dim; e->nqkv = e->nq + 2 * e->nkv_dim;
    e->Tmax = opts->max_prefill_tokens > 0 ? opts->max_prefill_tokens : 8192;
    if (e->Tmax < 16) e->Tmax = 16;
    e->window = w->sliding_window;
    e->ring = ring_pages(e->window, e->Tmax);
    e->embed = w->embed; e->lm_head = w->lm_head; e->final_norm = w->final_norm;
    const int L = d.n_layers;
    for (int l = 0; l < L; ++l) {
        e->wqkv.push_back(w->wqkv[l]); e->wo.push_back(w->wo[l]); e->wgu.push_back(w->wgu[l]);
        e->wdown.push_back(w->wdown[l]); e->norm_attn.push_back(w->norm_attn[l]); e->norm_mlp.push_back(w->norm_mlp[l]);
        if (fp8) {
            e->sqkv.push_back((const float*)w->wqkv_scale[l]); e->so.push_back((const float*)w->wo_scale[l]);
            e->sgu.push_back((const float*)w->wgu_scale[l]); e->sdown.push_back((const float*)w->wdown_scale[l]);
        }
    }
    e->fp8 = fp8;
    memset(&e->st, 0, sizeof(e->st));
    e->t0 = std::chrono::steady_clock::now();
    int rc = RR_OK;
#define TRY(x) do { rc = (x); if (rc != RR_OK) { rr_engine_destroy(e); return rc; } } while (0)
#define TRYC(x) do { cudaError_t e__ = (x); if (e__ != cudaSuccess) { rr::note_cuda_error(e__); rr_engine_destroy(e); return RR_CUDA_ERROR; } } while (0)
    TRYC(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
    TRYC(cudaEventCreate(&e->ev0));
    TRYC(cudaEventCreate(&e->ev1));
    const int B = e->Bm;
    // Uniform split-K planes.
    e->s_qkv = pick_splits(e->nqkv, d.hidden); e->s_o = pick_splits(d.hidden, e->nq);
    e->s_gu = pick_splits(2 * d.inter, d.hidden); e->s_down = pick_splits(d.hidden, d.inter);
    e->fuse_silu = (w->flags & RR_WEIGHTS_WGU_INTERLEAVED64) && e->s_gu == 1 && e->bn_dec >= 32 &&
                   (2 * d.inter) % 128 == 0;
    if ((w->flags & RR_WEIGHTS_WGU_INTERLEAVED64) && !e->fuse_silu) { rr_engine_destroy(e); return RR_INVALID_ARGUMENT; }
    TRY(dalloc(e, &e->d_tok, B)); TRY(dalloc(e, &e->d_pos, B)); TRY(dalloc(e, &e->d_slot, B));
    TRYC(cudaMemset(e->d_slot, 0xff, sizeof(int32_t) * B));
    TRY(dalloc(e, &e->x, (size_t)B * d.hidden));
    TRY(dalloc(e, &e->xn, (size_t)B * d.hidden));
    TRY(dalloc(e, &e->qbuf, (size_t)B * d.n_heads * 128));
    TRY(dalloc(e, &e->attn_out, (size_t)B * e->nq));
    TRY(dalloc(e, &e->act, (size_t)B * d.inter));
    TRY(dalloc(e, &e->part_qkv, (size_t)e->s_qkv * B * e->nqkv));
    TRY(dalloc(e, &e->part_o, (size_t)e->s_o * B * d.hidden));
    TRY(dalloc(e, &e->part_gu, (size_t)e->s_gu * B * 2 * d.inter));
    // fused decode MLP: the down GEMM's K range in <= 8 slices, one output plane each (mlp_slices)
    {
        const int n_sl = mlp_slices(d.inter, &e->mlp_slice_kb);
        e->fuse_mlp = e->fuse_silu && e->Bm <= e->bn_dec && n_sl > 0;
        e->mlp_slices = e->fuse_mlp ? n_sl : 0;
    }
    TRY(dalloc(e, &e->part_down, (size_t)(e->s_down > e->mlp_slices ? e->s_down : e->mlp_slices) * B * d.hidden));
    TRY(dalloc(e, &e->logits, (size_t)B * d.vocab));
    TRY(dalloc(e, &e->rope_table, (size_t)opts->ctx_max * 64));
    launch_rope_table(e->rope_table, opts->ctx_max, d.rope_theta, d.head_dim, e->stream);
    // zeroed like the rest: decode attention reads stale rows of a partly used tile, whose masked scores must meet finite K/V
    e->n_pages = (int)(kv_tokens / KV_PAGE); e->pps = opts->ctx_max / KV_PAGE;
    e->o.kv_cache_tokens = (int32_t)kv_tokens;
    e->kv_layer_stride = (size_t)e->n_pages * d.n_kv_heads * KV_PAGE * 128;
    TRY(dalloc(e, &e->kcache, e->kv_layer_stride * L));
    TRY(dalloc(e, &e->vcache, e->kv_layer_stride * L));
    TRY(dalloc(e, &e->d_table, (size_t)B * e->pps));
    TRYC(cudaMallocHost(&e->h_table, sizeof(int32_t) * B * e->pps));
    memset(e->h_table, 0, sizeof(int32_t) * B * e->pps);
    {   // split-KV only when the grid would not fill the GPU
        const int ks = pick_kv_splits(B, d.n_kv_heads);
        e->kv_splits = ks;
        e->attn_ws = nullptr;
        if (ks > 1) TRY(dalloc(e, &e->attn_ws, decode_attn_ws_bytes(B, d.n_heads, ks) / sizeof(float)));
    }
    const int T = e->Tmax;
    TRY(dalloc(e, &e->p_ids, (size_t)3 * T + 6 * B + 8));
    TRY(dalloc(e, &e->p_first, B));
    TRY(dalloc(e, &e->px, (size_t)T * d.hidden, false));
    TRY(dalloc(e, &e->pxn, (size_t)T * d.hidden, false));
    TRY(dalloc(e, &e->pqkv, (size_t)T * e->nqkv, false));
    TRY(dalloc(e, &e->pq, (size_t)T * d.n_heads * 128));                 // zeroed: columns beyond head_dim stay 0
    TRY(dalloc(e, &e->pattn, (size_t)T * e->nq, false));
    TRY(dalloc(e, &e->pgu, (size_t)T * 2 * d.inter, false));
    TRY(dalloc(e, &e->pact, (size_t)T * d.inter, false));
    TRYC(cudaMallocHost(&e->h_stage, ((size_t)3 * T + 6 * B + 8) * sizeof(int32_t)));
    TRYC(cudaMallocHost(&e->h_tok, sizeof(int32_t) * (B > 16 ? B : 16)));
    TRY(dalloc(e, (char**)&e->lp_ws, logprobs_ws_bytes(B, d.vocab), false));
    TRY(dalloc(e, &e->d_lp, (size_t)B * LP_MAX_TOP)); TRY(dalloc(e, &e->d_lp_id, (size_t)B * LP_MAX_TOP));
    TRYC(cudaMallocHost(&e->h_lp, sizeof(float) * B * LP_MAX_TOP));
    TRYC(cudaMallocHost(&e->h_lp_id, sizeof(int32_t) * B * LP_MAX_TOP));
    TRY(dalloc(e, (char**)&e->sample_ws, sample_ws_bytes(B, d.vocab), false));
    TRY(dalloc(e, &e->d_tok_lp, B));
    TRYC(cudaMallocHost(&e->h_tok_lp, sizeof(float) * B));
    // top_n and samp blocks (pen: ensure_pen_buffers), all zero but the decode rows' top_n and its mirror, which start at -1:
    // every row plain (no logprobs, greedy), as the mirror is
    e->d_rows.n = B; e->d_rows.bias_ld = PEN_MAX_BIAS;
    e->d_pf = e->d_rows; e->d_pf.has_pos = true;
    e->h_rows = e->d_rows; e->h_pf = e->d_pf;
    for (ParamBlocks* p : {&e->d_rows, &e->d_pf})
        for (int i = 0; i < 2; ++i) TRY(dalloc(e, &p->blk[i], p->bytes(i)));
    for (ParamBlocks* p : {&e->h_rows, &e->h_pf})
        for (int i = 0; i < 2; ++i) { TRYC(cudaMallocHost(&p->blk[i], p->bytes(i))); memset(p->blk[i], 0, p->bytes(i)); }
    TRYC(cudaMemset(e->d_rows.top_n(), 0xff, e->d_rows.bytes(0)));
    memset(e->h_rows.top_n(), 0xff, e->h_rows.bytes(0));

    e->pl_qkv.resize(L); e->pl_o.resize(L); e->pl_gu.resize(L); e->pl_down.resize(L);
    e->attn_args.resize(L);
    e->pf_attn.resize(L);
    for (int l = 0; l < L; ++l) {
        TRY(pf_attn_layer(&e->pf_attn[l], e->pq, e->kcache + (size_t)l * e->kv_layer_stride,
                          e->vcache + (size_t)l * e->kv_layer_stride, d.n_heads, d.n_kv_heads, d.head_dim, opts->ctx_max,
                          e->d_table, e->pps, e->n_pages, e->window, T));
        DecodeAttnArgs& da = e->attn_args[l];
        da.q = e->qbuf; da.k_cache = e->kcache + (size_t)l * e->kv_layer_stride;
        da.v_cache = e->vcache + (size_t)l * e->kv_layer_stride; da.out = e->attn_out; da.slot = e->d_slot;
        da.pos = e->d_pos; da.rows = B; da.n_heads = d.n_heads; da.n_kv_heads = d.n_kv_heads;
        da.ctx_max = opts->ctx_max; da.scale = 1.0f / sqrtf((float)d.head_dim); da.ws = e->attn_ws;
        da.kv_splits = e->kv_splits;
        da.fuse_rope = 1; da.qkv = part_f32(e->part_qkv, e->s_qkv, B, e->nqkv); da.rope_table = e->rope_table;
        da.head_dim = d.head_dim; da.page_table = e->d_table; da.pages_per_slot = e->pps; da.window = e->window;
        TRY(decode_attn_make_maps(&da, e->n_pages));
        // the decode projections: the same plans on e4m3 weights with FP8 (gemm_plan_init_fp8w)
        TRY(decode_plan_init(&e->pl_qkv[l], e->wqkv[l], fp8 ? e->sqkv[l] : nullptr, e->nqkv, d.hidden, e->xn, B,
                             e->part_qkv, e->nqkv, e->s_qkv, OUT_TRANSPOSED_F32));
        TRY(decode_plan_init(&e->pl_o[l], e->wo[l], fp8 ? e->so[l] : nullptr, d.hidden, e->nq, e->attn_out, B, e->part_o,
                             d.hidden, e->s_o, OUT_TRANSPOSED_F32));
        if (e->fuse_silu)
            TRY(decode_plan_init(&e->pl_gu[l], e->wgu[l], fp8 ? e->sgu[l] : nullptr, 2 * d.inter, d.hidden, e->xn, B, e->act,
                                 d.inter, 1, OUT_TRANSPOSED_SILU));
        else
            TRY(decode_plan_init(&e->pl_gu[l], e->wgu[l], fp8 ? e->sgu[l] : nullptr, 2 * d.inter, d.hidden, e->xn, B,
                                 e->part_gu, 2 * d.inter, e->s_gu, OUT_TRANSPOSED_F32));
        TRY(decode_plan_init(&e->pl_down[l], e->wdown[l], fp8 ? e->sdown[l] : nullptr, d.hidden, d.inter, e->act, B,
                             e->part_down, d.hidden, e->s_down, OUT_TRANSPOSED_F32));
    }
    TRY(decode_plan_init(&e->pl_head, e->lm_head, nullptr, d.vocab, d.hidden, e->xn, B, e->logits, d.vocab, 1,
                         OUT_TRANSPOSED_F32));
    e->fuse_rope_pf = pf_rope_fused(d.head_dim);
    // deferred prefill RMSNorm: hidden % 64 == 0 and hidden <= 8192 (checked above) give the 16-byte rows and the <= 64 partial
    // sums per row that the residual epilogue writes
    e->pf_parts = pf_norm_parts(d.hidden);
    TRY(dalloc(e, &e->p_rowss, (size_t)e->Tmax * e->pf_parts));
    if (fp8) TRY(dalloc(e, &e->deq, (size_t)(e->nqkv + e->nq + 3 * d.inter) * d.hidden, false));
    TRY(init_pf_plans(e));
    if (e->fuse_mlp) {
        std::vector<MlpItem> sched;
        const int grid = num_sms();
        const int dyn = getenv("RR_MLP_STATIC") ? 0 : 1;      // down items dealt by the kernel (default) or by the host list schedule
        const int max_items = mlp_schedule(grid, d.inter, d.hidden, e->mlp_slice_kb, &sched, dyn);
        TRY(dalloc(e, &e->mlp_items, sched.size()));
        TRYC(cudaMemcpy(e->mlp_items, sched.data(), sched.size() * sizeof(MlpItem), cudaMemcpyHostToDevice));
        TRY(dalloc(e, &e->mlp_ready, 16));
        e->mlp.resize(L);
        for (int l = 0; l < L; ++l) {
            TRY(mlp_plan_init(&e->mlp[l], e->wgu[l], e->wdown[l], d.inter, d.hidden, e->xn, B, e->act, e->part_down, B,
                              e->bn_dec, e->mlp_items, max_items, grid, e->mlp_ready, e->mlp_slice_kb, dyn,
                              fp8 ? e->sgu[l] : nullptr, fp8 ? e->sdown[l] : nullptr));
        }
    }
    TRYC(cudaDeviceSynchronize());
    e->row_req.assign(B, nullptr);
    e->row_choice.assign(B, 0);
    e->h_slot_mirror.assign(B, -1);
    e->slot_pages.assign(B, {});
    e->table_dirty.assign(B, 0);
    for (int pg = e->n_pages; pg-- > 0;) e->free_pages.push_back(pg);      // pages 0, 1, ... come off the stack first
    if (e->o.prefix_cache) { e->retained.assign(B, {}); e->retained_used.assign(B, 0); }
    e->worker = std::thread(worker_main, e);
    *out = e;
    return RR_OK;
#undef TRY
#undef TRYC
}

RR_API void rr_engine_destroy(rr_engine* e) {
    if (!e) return;
    e->stop.store(true);
    e->cv_work.notify_all();
    if (e->worker.joinable()) e->worker.join();
    cudaSetDevice(e->o.device);
    if (e->stream) cudaStreamSynchronize(e->stream);
    for (cudaGraphExec_t g : e->graph)
        if (g) cudaGraphExecDestroy(g);
    for (void* p : e->allocs) cudaFree(p);
    if (e->h_stage) cudaFreeHost(e->h_stage);
    if (e->h_table) cudaFreeHost(e->h_table);
    if (e->h_tok) cudaFreeHost(e->h_tok);
    if (e->h_lp) cudaFreeHost(e->h_lp);
    if (e->h_lp_id) cudaFreeHost(e->h_lp_id);
    if (e->h_tok_lp) cudaFreeHost(e->h_tok_lp);
    if (e->h_stop) cudaFreeHost(e->h_stop);
    if (e->h_json_done) cudaFreeHost(e->h_json_done);
    for (void* p : {(void*)e->h_sc_in, (void*)e->h_sc_tlp, (void*)e->h_sc_lp, (void*)e->h_emb})
        if (p) cudaFreeHost(p);
    for (const ParamBlocks* p : {&e->h_rows, &e->h_pf})
        for (char* b : p->blk)
            if (b) cudaFreeHost(b);
    if (e->ev0) cudaEventDestroy(e->ev0);
    if (e->ev1) cudaEventDestroy(e->ev1);
    if (e->stream) cudaStreamDestroy(e->stream);
    for (auto& kv : e->table) delete kv.second;
    delete e;
}

RR_API int rr_engine_prefill(rr_engine* e, const int32_t* ids, const int32_t* seq_start, const int32_t* slots,
                             int n_seqs, int32_t* first_tok, float* logits_out) {
    if (!e || !ids || !seq_start || !slots || n_seqs < 1) return RR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> gl(e->gpu_mu);
    std::lock_guard<std::mutex> dl(device_mutex(e->o.device));
    forget_prefixes(e);
    CK(cudaSetDevice(e->o.device));
    std::vector<int> n_pos(n_seqs);
    for (int i = 0; i < n_seqs; ++i) {                 // run_prefill checks the rest
        if (slots[i] < 0 || slots[i] >= e->Bm || seq_start[i + 1] - seq_start[i] > e->o.ctx_max) return RR_INVALID_ARGUMENT;
        n_pos[i] = std::max(0, seq_start[i + 1] - seq_start[i]);
    }
    int rc = grow_pages(e, slots, n_pos.data(), n_seqs);
    if (rc == RR_OK) rc = upload_table(e);
    if (rc != RR_OK) return rc;
    Chunk c;                                           // plain last pieces: one greedy tail row per sequence, in its slot
    c.reset(0, false);
    for (int i = 0; i < n_seqs; ++i) c.add(nullptr, slots[i], 0, ids + seq_start[i], seq_start[i + 1] - seq_start[i], true);
    return run_prefill(e, c, first_tok, logits_out);
}

RR_API int rr_engine_decode_step(rr_engine* e, const int32_t* slots, const int32_t* tok, const int32_t* pos, int n,
                                 int32_t* next_tok, float* logits_out) {
    if (!e || !slots || !tok || !pos || n < 1 || n > e->Bm || !next_tok) return RR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> gl(e->gpu_mu);
    std::lock_guard<std::mutex> dl(device_mutex(e->o.device));
    forget_prefixes(e);
    CK(cudaSetDevice(e->o.device));
    const int B = e->Bm;
    int32_t* h = e->h_stage;                 // tok[B] | pos[B] | slot[B]
    for (int b = 0; b < B; ++b) { h[b] = 0; h[B + b] = 0; h[2 * B + b] = -1; }
    for (int i = 0; i < n; ++i) {
        const int s = slots[i];
        if (s < 0 || s >= B || pos[i] < 0 || pos[i] >= e->o.ctx_max) return RR_INVALID_ARGUMENT;
        h[s] = tok[i]; h[B + s] = pos[i]; h[2 * B + s] = s;
    }
    {
        std::vector<int> n_pos(n);
        for (int i = 0; i < n; ++i) n_pos[i] = pos[i] + 1;
        int rc = grow_pages(e, slots, n_pos.data(), n);
        if (rc == RR_OK) rc = upload_table(e);
        if (rc != RR_OK) return rc;
    }
    cudaStream_t st = e->stream;
    CK(cudaMemcpyAsync(e->d_tok, h, sizeof(int32_t) * B, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(e->d_pos, h + B, sizeof(int32_t) * B, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(e->d_slot, h + 2 * B, sizeof(int32_t) * B, cudaMemcpyHostToDevice, st));
    uint64_t nl = 0;
    int rc = enqueue_decode_step(e, st, &nl);
    if (rc != RR_OK) return rc;
    e->st.kernel_launches += nl;
    CK(cudaMemcpyAsync(e->h_tok, e->d_tok, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (int i = 0; i < n; ++i) {
        next_tok[i] = e->h_tok[slots[i]];
        if (logits_out)
            CK(cudaMemcpy(logits_out + (size_t)i * e->d.vocab, e->logits + (size_t)slots[i] * e->d.vocab,
                          sizeof(float) * e->d.vocab, cudaMemcpyDeviceToHost));
    }
    // leave the rows inactive for the serving loop
    CK(cudaMemsetAsync(e->d_slot, 0xff, sizeof(int32_t) * B, st));
    CK(cudaStreamSynchronize(st));
    for (int b = 0; b < B; ++b) e->h_slot_mirror[b] = -1;
    return RR_OK;
}

static bool injected_failure(const rr_engine* e, uint64_t ticket) {
    if (e->o.fail_prob <= 0.f) return false;
    uint64_t z = ticket + 0x9E3779B97F4A7C15ull * (uint64_t)(uint32_t)(e->o.fail_seed + 1);   // splitmix64
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    return (double)(z >> 11) * (1.0 / 9007199254740992.0) < (double)e->o.fail_prob;
}

// Gives r its ticket and queues it (or fails it at once: fail_prob), then wakes the worker and runs the done hook.
static void enqueue_request(rr_engine* e, Request* r, uint64_t* ticket) {
    std::vector<DoneNote> notes;
    {
        std::lock_guard<std::mutex> lk(e->mu);
        r->ticket = e->next_ticket++;
        r->t_submit = now_s(e);
        e->table[r->ticket] = r;
        *ticket = r->ticket;
        if (injected_failure(e, r->ticket)) {
            r->t_first = r->t_submit;
            finish_request(e, r, RR_BACKEND_FAILED, &notes);
        } else {
            e->waiting.push_back(r);
        }
    }
    e->cv_work.notify_one();
    e->cv_done.notify_all();
    run_hooks(e, notes);
}

namespace rr {
int engine_submit_embed_tagged(rr_engine* e, const int32_t* prompt_ids, int n_prompt, uint64_t tag, uint64_t* ticket) {
    if (!e || !prompt_ids || !ticket || n_prompt < 1 || n_prompt > e->o.ctx_max) return RR_INVALID_ARGUMENT;
    if (choice_pages(e, n_prompt) > e->n_pages) return RR_INVALID_ARGUMENT;
    for (int i = 0; i < n_prompt; ++i)
        if (prompt_ids[i] < 0 || prompt_ids[i] >= e->d.vocab) return RR_INVALID_ARGUMENT;
    Request* r = new (std::nothrow) Request();
    if (!r) return RR_INTERNAL;
    r->prompt.assign(prompt_ids, prompt_ids + n_prompt);
    r->max_new = 0;
    r->embed = true;
    r->out.resize(1); r->finish.assign(1, -1); r->hold.assign(1, 0); r->lp.resize(1); r->lp_id.resize(1);
    r->tag = tag;
    enqueue_request(e, r, ticket);
    return RR_OK;
}

int engine_submit_tagged(rr_engine* e, const int32_t* prompt_ids, int n_prompt, int max_new_tokens, uint64_t tag,
                         uint64_t* ticket, const GenParams& p, int n_choices) {
    if (!e || !prompt_ids || !ticket || n_prompt < 1 || max_new_tokens < 1) return RR_INVALID_ARGUMENT;
    if (n_choices < 1 || n_choices > e->Bm) return RR_INVALID_ARGUMENT;      // the choices decode side by side
    // the vocabularies the logprobs / sampling kernels handle (rr_engine_create refused vocab % 4 != 0)
    if ((p.logprobs() || p.sampled() || p.scores()) && e->d.vocab > LP_MAX_CHUNKS * LP_CHUNK)
        return RR_INVALID_ARGUMENT;
    if (p.prompt_top < -1 || p.prompt_top > LP_MAX_TOP) return RR_INVALID_ARGUMENT;
    if (n_prompt + max_new_tokens > e->o.ctx_max) return RR_INVALID_ARGUMENT;
    if ((long long)n_choices * choice_pages(e, n_prompt + max_new_tokens) > e->n_pages) return RR_INVALID_ARGUMENT;
    for (int i = 0; i < n_prompt; ++i)
        if (prompt_ids[i] < 0 || prompt_ids[i] >= e->d.vocab) return RR_INVALID_ARGUMENT;
    Request* r = new (std::nothrow) Request();
    if (!r) return RR_INTERNAL;
    r->prompt.assign(prompt_ids, prompt_ids + n_prompt);
    r->max_new = max_new_tokens;
    r->n_choices = n_choices;
    r->out.resize(n_choices);
    r->finish.assign(n_choices, -1); r->hold.assign(n_choices, 0);
    r->lp.resize(n_choices); r->lp_id.resize(n_choices);
    for (int c = 0; c < n_choices; ++c) {
        r->out[c].reserve(max_new_tokens);
        if (p.logprobs()) {
            const size_t k = p.lp_width();
            r->lp[c].reserve(k * max_new_tokens); r->lp_id[c].reserve(k * max_new_tokens);
        }
    }
    r->tag = tag;
    r->gen = p;
    if (p.scores()) {
        const size_t n = (size_t)n_prompt - 1, k = (size_t)p.score_width();
        r->ptgt.assign(n, 0.f); r->plp.assign(n * k, 0.f); r->plp_id.assign(n * k, 0);
    }
    enqueue_request(e, r, ticket);
    return RR_OK;
}
void engine_set_done_hook(rr_engine* e, EngineDoneHook fn, void* ctx) {
    std::lock_guard<std::mutex> lk(e->mu);
    e->hook = fn; e->hook_ctx = ctx;
}
int engine_limits(const rr_engine* e, int* ctx_max, int* vocab, int* max_batch, int* kv_tokens, int* ring, int* hidden) {
    if (!e) return RR_INVALID_ARGUMENT;
    if (hidden) *hidden = e->d.hidden;
    if (kv_tokens) *kv_tokens = e->n_pages * KV_PAGE;
    if (ring) *ring = e->ring;
    if (max_batch) *max_batch = e->Bm;
    if (ctx_max) *ctx_max = e->o.ctx_max;
    if (vocab) *vocab = e->d.vocab;
    return RR_OK;
}
}  // namespace rr

RR_API int rr_engine_submit(rr_engine* e, const int32_t* prompt_ids, int n_prompt, int max_new_tokens,
                            const rr_gen_params* params, uint64_t* ticket) {
    if (!e) return RR_INVALID_ARGUMENT;
    rr::GenParams p;
    const int rc = p.set(e->d.vocab, params);
    return rc != RR_OK ? rc : rr::engine_submit_tagged(e, prompt_ids, n_prompt, max_new_tokens, 0, ticket, p,
                                                       params ? params->n_choices : 1);
}

RR_API int rr_engine_submit_scored(rr_engine* e, const int32_t* prompt_ids, int n_prompt, int max_new_tokens,
                                   const rr_gen_params* params, int prompt_top, uint64_t* ticket) {
    if (!e) return RR_INVALID_ARGUMENT;
    rr::GenParams p;
    const int rc = p.set(e->d.vocab, params);
    if (rc != RR_OK) return rc;
    p.prompt_top = prompt_top;
    return rr::engine_submit_tagged(e, prompt_ids, n_prompt, max_new_tokens, 0, ticket, p, params ? params->n_choices : 1);
}

// Caller holds lk on e->mu.  The request of `ticket` once ready(r) holds, else as it is at the deadline (timeout_s <= 0:
// none); null when the ticket is unknown or consumed.  It is looked up again after every wake-up: another thread may have
// consumed (wait) or cancelled the ticket meanwhile.  A caller that reads one kind of request makes ready() true for the
// other kinds, and refuses them.
template <typename Ready>
static Request* await_request(rr_engine* e, std::unique_lock<std::mutex>& lk, uint64_t ticket, double timeout_s,
                              Ready ready) {
    const auto deadline = std::chrono::steady_clock::now() +
                          std::chrono::duration<double>(timeout_s > 0 ? timeout_s : 1e9);
    for (bool late = false;; late = e->cv_done.wait_until(lk, deadline) == std::cv_status::timeout) {
        auto it = e->table.find(ticket);
        if (it == e->table.end()) return nullptr;
        if (late || ready(it->second)) return it->second;
    }
}

RR_API int rr_engine_prompt_logprobs(rr_engine* e, uint64_t ticket, double timeout_s, float* target_lp_out, float* lp_out,
                                     int32_t* id_out) {
    if (!e) return RR_INVALID_ARGUMENT;
    std::unique_lock<std::mutex> lk(e->mu);
    const Request* r = await_request(e, lk, ticket, timeout_s, [](const Request* q) { return !q->gen.scores() || q->done; });
    if (!r || !r->gen.scores()) return RR_INVALID_ARGUMENT;
    if (!r->done) return RR_TIMEOUT;
    if (r->status != RR_OK) return r->status;
    if (target_lp_out) memcpy(target_lp_out, r->ptgt.data(), sizeof(float) * r->ptgt.size());
    if (lp_out) memcpy(lp_out, r->plp.data(), sizeof(float) * r->plp.size());
    if (id_out) memcpy(id_out, r->plp_id.data(), sizeof(int32_t) * r->plp_id.size());
    return RR_OK;
}

RR_API int rr_engine_submit_embed(rr_engine* e, const int32_t* prompt_ids, int n_prompt, uint64_t* ticket) {
    return rr::engine_submit_embed_tagged(e, prompt_ids, n_prompt, 0, ticket);
}

RR_API int rr_engine_embedding(rr_engine* e, uint64_t ticket, double timeout_s, float* out, int capacity, int* dim_out) {
    if (!e || !out || capacity < e->d.hidden) return RR_INVALID_ARGUMENT;
    std::unique_lock<std::mutex> lk(e->mu);
    const Request* r = await_request(e, lk, ticket, timeout_s, [](const Request* q) { return !q->embed || q->done; });
    if (!r || !r->embed) return RR_INVALID_ARGUMENT;
    if (!r->done) return RR_TIMEOUT;
    if (r->status != RR_OK) return r->status;
    memcpy(out, r->emb.data(), sizeof(float) * r->emb.size());
    if (dim_out) *dim_out = (int)r->emb.size();
    return RR_OK;
}

// Caller holds e->mu.  The first min(n, max_tokens_out) visible tokens of each choice of r (fewer for a shorter choice)
// into tokens_out [n_choices][max_tokens_out], and of a logprobs request their pairs into lp_out / id_out [n_choices]
// [max_tokens_out][K] (any may be null).
static void copy_choices(const Request* r, int n, int max_tokens_out, int32_t* tokens_out, float* lp_out, int32_t* id_out) {
    const size_t k = (size_t)r->gen.lp_width();
    for (int c = 0; c < r->n_choices; ++c) {
        const int t = std::min(std::min(n, max_tokens_out), r->visible(c));
        if (t <= 0) continue;
        const size_t o = (size_t)c * max_tokens_out;
        if (tokens_out) memcpy(tokens_out + o, r->out[c].data(), sizeof(int32_t) * t);
        if (!r->gen.logprobs()) continue;
        if (lp_out) memcpy(lp_out + o * k, r->lp[c].data(), sizeof(float) * t * k);
        if (id_out) memcpy(id_out + o * k, r->lp_id[c].data(), sizeof(int32_t) * t * k);
    }
}

// Abandon a request (client gone / timed out): a queued request is dropped, a running one gives up its decode rows at the
// next step; a finished one is just freed.  The ticket is consumed: do not wait on it afterwards.
RR_API int rr_engine_cancel(rr_engine* e, uint64_t ticket) {
    if (!e) return RR_INVALID_ARGUMENT;
    std::vector<DoneNote> notes;
    {
        std::lock_guard<std::mutex> lk(e->mu);
        auto it = e->table.find(ticket);
        if (it == e->table.end()) return RR_INVALID_ARGUMENT;
        Request* r = it->second;
        if (r->done) {
            e->table.erase(it);
            delete r;
        } else {
            r->detached = true;
            bool queued = false;
            for (auto q = e->waiting.begin(); q != e->waiting.end(); ++q)
                if (*q == r) { e->waiting.erase(q); queued = true; break; }
            if (queued) finish_request(e, r, RR_CANCELLED, &notes);      // frees it (detached)
            else r->cancel = true;                                       // active rows: the worker drops them
        }
    }
    e->cv_work.notify_one();
    e->cv_done.notify_all();
    run_hooks(e, notes);
    return RR_OK;
}

// Streaming support: block until the request has more than `have` tokens (or is done / the wait times out), then
// copy the tokens generated so far.  Does not consume the request; finish with rr_engine_wait.  A request of several
// choices gets RR_INVALID_ARGUMENT.
RR_API int rr_engine_peek(rr_engine* e, uint64_t ticket, int have, double timeout_s, int32_t* tokens_out,
                          int max_tokens_out, int32_t* n_generated, int32_t* done, double* t_first_token_s, float* lp_out,
                          int32_t* id_out) {
    if (!e || !n_generated || !done) return RR_INVALID_ARGUMENT;
    std::unique_lock<std::mutex> lk(e->mu);
    const Request* r = await_request(e, lk, ticket, timeout_s, [have](const Request* q) {
        return q->n_choices > 1 || q->done || q->n_generated() > have;
    });
    if (!r || r->n_choices > 1) return RR_INVALID_ARGUMENT;
    const int n = r->n_generated();
    *n_generated = n;
    *done = r->done ? 1 : 0;
    if (t_first_token_s) *t_first_token_s = r->t_first - r->t_submit;
    copy_choices(r, n, max_tokens_out, tokens_out, lp_out, id_out);
    return RR_OK;
}

RR_API int rr_engine_wait(rr_engine* e, uint64_t ticket, double timeout_s, rr_completion* out, int32_t* tokens_out,
                          int max_tokens_out, float* lp_out, int32_t* id_out, int32_t* n_tokens_out, int32_t* finish_out) {
    if (!e || !out) return RR_INVALID_ARGUMENT;
    std::unique_lock<std::mutex> lk(e->mu);
    Request* r = await_request(e, lk, ticket, timeout_s, [](const Request* q) { return q->done; });
    if (!r) return RR_INVALID_ARGUMENT;                // unknown, already consumed, or cancelled
    if (!r->done) {
        out->ticket = ticket; out->status = RR_TIMEOUT;
        return RR_TIMEOUT;   // the request stays in flight: wait again, or rr_engine_cancel
    }
    out->ticket = ticket; out->status = r->status; out->n_prompt = (int)r->prompt.size();
    out->n_generated = r->n_generated(); out->n_cached = r->n_cached;
    out->t_submit_s = r->t_submit; out->t_first_token_s = r->t_first; out->t_done_s = r->t_done;
    copy_choices(r, r->n_generated(), max_tokens_out, tokens_out, lp_out, id_out);
    for (int c = 0; c < r->n_choices; ++c) {
        if (n_tokens_out) n_tokens_out[c] = r->visible(c);
        if (finish_out) finish_out[c] = r->finish[c] > 0 ? 1 : 0;
    }
    const int status = r->status;
    e->table.erase(ticket);
    delete r;
    return status == RR_OK ? RR_OK : status;
}

RR_API int rr_engine_run_batch(rr_engine* e, const int32_t* prompt_ids, const int32_t* prompt_start, int n_requests,
                               int max_new_tokens, rr_completion* out, int32_t* tokens_out) {
    if (!e || !prompt_ids || !prompt_start || n_requests < 1 || !out) return RR_INVALID_ARGUMENT;
    std::vector<uint64_t> tk(n_requests);
    for (int i = 0; i < n_requests; ++i) {
        int rc = rr_engine_submit(e, prompt_ids + prompt_start[i], prompt_start[i + 1] - prompt_start[i],
                                  max_new_tokens, nullptr, &tk[i]);
        if (rc != RR_OK) return rc;
    }
    int worst = RR_OK;
    for (int i = 0; i < n_requests; ++i) {
        int rc = rr_engine_wait(e, tk[i], 0, &out[i], tokens_out ? tokens_out + (size_t)i * max_new_tokens : nullptr,
                                max_new_tokens, nullptr, nullptr, nullptr, nullptr);
        if (rc != RR_OK) worst = rc;
    }
    return worst;
}

RR_API double rr_engine_now(rr_engine* e) { return e ? now_s(e) : 0.0; }

RR_API int rr_engine_kv_usage(rr_engine* e, int32_t* pages_total, int32_t* pages_free) {
    if (!e || !pages_total || !pages_free) return RR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> lk(e->mu);
    *pages_total = e->n_pages;
    *pages_free = (int32_t)e->free_pages.size();
    return RR_OK;
}

RR_API int rr_engine_get_stats(rr_engine* e, rr_engine_stats* out) {
    if (!e || !out) return RR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> gl(e->gpu_mu);      // the worker updates the counters while it holds gpu_mu (then mu)
    std::lock_guard<std::mutex> lk(e->mu);
    *out = e->st;
    return RR_OK;
}

RR_API int rr_engine_reset_stats(rr_engine* e) {
    if (!e) return RR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> gl(e->gpu_mu);
    std::lock_guard<std::mutex> lk(e->mu);
    memset(&e->st, 0, sizeof(e->st));
    return RR_OK;
}
