// rr_gateway.cu — the per-request path in native code: concurrent admission -> K1 -> engine hand-off, no Python hop.
//
// The reference's concurrency is N blocked client threads into a single-worker gateway process
// (reference src/demo_load_balancing.py:195-203, bin/start-gateway.sh:54).  Here every client thread calls
// rr_gateway_submit (non-blocking, any thread): the request goes into an admission queue; ONE dispatcher thread
// drains the queue, turns everything that is pending — ADMITs of new requests, DONE / FAIL reports of finished ones,
// re-ADMITs of requests whose backend failed (the fallback walk) — into one ordered event trace, stages it in pinned
// memory, and processes it with ONE launch of the K1 router kernel (rr_router.cu: events and decisions live in the
// router's HBM-resident rings); decisions come back in one D2H copy and admitted requests go straight into the queue
// of the engine that serves the picked deployment (engine_submit_tagged), whose worker thread reports completion
// through a hook.  Concurrent admissions are therefore COALESCED: under a burst of N callers the path costs
// ~N / batch launches instead of 2 N, and the serialised-trace semantics of K1 are unchanged (the trace is the
// arrival order at the queue; it can be recorded and replayed through the oracle, tests/test_gateway_gpu.py).
// A mock replica (rr_stub_desc) is served by the dispatcher itself at hand-off and settles through the same code as
// the hook (gw_settle), so failure, fallback and cancellation are one path for both kinds of replica.
//
// Replaces: litellm.Router's async request handling behind the proxy (reference pyproject.toml:8,
// config/config.yaml:100-108) for the call shape of reference src/demo_fallback.py:143-147.
#include "rr_kernels.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <new>
#include <string.h>
#include <thread>
#include <unordered_map>
#include <vector>

#define RR_API extern "C" __attribute__((visibility("default")))

namespace {

enum ReqState { Q_ADMIT = 0, RUNNING = 1, FINISHED = 2 };

struct GwReq {
    uint64_t id = 0;
    int group = 0, max_new = 0;
    int n_choices = 1;                // handed with gen to every engine the request is admitted to
    std::vector<int32_t> prompt;
    int chain_start = 0, attempts = 0;
    ReqState state = Q_ADMIT;
    int status = RR_OK;
    int deployment = -1, served_group = -1, chain_pos = 0, replica = -1;
    rr_engine* eng = nullptr;
    uint64_t eng_ticket = 0;
    std::vector<int32_t> tokens;      // the choices' returned tokens, one after the other: n_tok[c] of choice c
    std::vector<int32_t> n_tok, fin;  // [n_choices] tokens returned and finish reason (0 length, 1 stop); empty until settled
    rr::GenParams gen;                // handed to every engine the request is admitted to
    std::vector<float> lp;            // tokens' pairs, [gen.lp_width()] each
    std::vector<int32_t> lp_id;
    // prompt logprobs (gen.scores()) of the engine that served it, read before its record was consumed
    // (rr_engine_prompt_logprobs): [n_prompt - 1] and [n_prompt - 1][gen.score_width()]
    std::vector<float> ptgt, plp;
    std::vector<int32_t> plp_id;
    // an embedding request (rr_gateway_submit_embed, max_new 0): the embedding of the engine that served it, read before
    // its record was consumed (rr_engine_embedding), [that engine's hidden size]
    bool embed = false;
    std::vector<float> emb;
    int n_cached = 0;                 // rr_completion.n_cached of the engine that served it
    double t_submit = 0, t_admit = 0, t_first = 0, t_done = 0, t_eng_submit = 0;   // t_eng_submit: hand-off to the replica
    bool cancelled = false, cancel_as_failure = false, abandoned = false;

    int n_gen() const {               // tokens of the longest choice
        int n = 0;
        for (int32_t t : n_tok) n = t > n ? t : n;
        return n;
    }
};

struct Pending {
    int type;          // RR_EV_*
    GwReq* req;        // ADMIT
    int target;        // DONE / FAIL: deployment; BURST: group
    int tokens;        // DONE: completion tokens; BURST: burst size
    int aux = 0;       // rr_event.chain_start of a DONE (latency, us) / FAIL (1 = timeout): latency-based routers only
};

}  // namespace

struct rr_gateway {
    rr_router* router = nullptr;
    std::vector<rr_engine*> engines;        // index = position in the create() arrays; nullptr: a mock replica
    std::vector<rr_stub_desc> stubs;        // same index: the mock replicas' descriptors
    std::vector<uint64_t> stub_handed;      // same index: requests handed to each mock replica so far
    bool has_stub = false;
    std::unordered_map<int, int> by_replica;   // replica id -> index into engines
    int n_deps = 0, n_groups = 0;
    bool latency = false;                   // the router is latency-based: DONE / FAIL events carry samples
    int min_ctx = 0, min_vocab = 0, min_rows = 0;     // min_rows: decode rows, the limit of n_choices
    // each engine's KV pool in pages and the pages a choice reserves at most (its ring; 0: no window), by engine_limits
    std::vector<std::pair<int, int>> kv_pools;
    rr_gateway_opts opts;

    std::mutex mu;
    std::condition_variable cv_work, cv_done;
    std::deque<Pending> pending;
    std::unordered_map<uint64_t, GwReq*> table;
    uint64_t next_id = 1;
    std::thread dispatcher;
    bool stop = false;
    bool busy = false;                     // the dispatcher is between taking a batch and publishing its decisions
    std::atomic<int64_t> manual_now_ms{0};
    std::chrono::steady_clock::time_point t0;

    // trace recording (ring of the last `record_trace` events)
    std::vector<rr_event> tr_ev;
    std::vector<rr_decision> tr_dec;
    size_t tr_count = 0;

    rr_gateway_stats st;
};

static double gw_now_s(rr_gateway* g) {
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - g->t0).count();
}
static int64_t gw_clock_ms(rr_gateway* g) {
    if (g->opts.manual_clock) return g->manual_now_ms.load(std::memory_order_relaxed);
    return std::chrono::duration_cast<std::chrono::milliseconds>(std::chrono::system_clock::now().time_since_epoch()).count();
}

// caller holds g->mu
static void gw_finish(rr_gateway* g, GwReq* r, int status) {
    r->status = status;
    r->state = FINISHED;
    r->t_done = gw_now_s(g);
    if (status == RR_OK) g->st.completed++;
    else if (status == RR_RATE_LIMITED) g->st.rate_limited++;
    else g->st.failed++;
    if (r->abandoned) {
        g->table.erase(r->id);
        delete r;
    }
}

// caller holds g->mu.  Request r ended on the replica it was handed to with `status` (n_generated tokens by then, over all
// choices).  When the replica's record of it was read (wrc RR_OK / RR_BACKEND_FAILED: comp, toks [n_choices][max_new],
// each choice's token count n_toks and finish reason fins, and with logprobs lps / lp_ids [n_choices][max_new][K]), the
// result is stored.  Then DONE (with the latency sample) / FAIL / the cancel report is posted and the request finishes,
// or after a backend failure goes back into the queue one step further down its fallback chain.
static void gw_settle(rr_gateway* g, GwReq* r, int status, int n_generated, int wrc, const rr_completion& comp,
                      const int32_t* toks, const int32_t* n_toks, const int32_t* fins, const float* lps,
                      const int32_t* lp_ids) {
    const int dep = r->deployment;
    if (wrc == RR_OK || wrc == RR_BACKEND_FAILED) {
        const size_t k = (size_t)r->gen.lp_width();
        r->tokens.clear(); r->lp.clear(); r->lp_id.clear(); r->n_tok.clear(); r->fin.clear();
        for (int c = 0; c < r->n_choices; ++c) {
            int n = n_toks[c] < r->max_new ? n_toks[c] : r->max_new;
            n = n > 0 ? n : 0;
            r->n_tok.push_back(n); r->fin.push_back(fins[c]);
            const size_t o = (size_t)c * r->max_new;
            r->tokens.insert(r->tokens.end(), toks + o, toks + o + n);
            if (r->gen.logprobs()) {
                r->lp.insert(r->lp.end(), lps + o * k, lps + (o + n) * k);
                r->lp_id.insert(r->lp_id.end(), lp_ids + o * k, lp_ids + (o + n) * k);
            }
        }
        r->t_first = r->t_eng_submit + (comp.t_first_token_s - comp.t_submit_s);
        r->n_cached = comp.n_cached;
    }
    if (status == RR_OK) {
        // latency sample: the replica's submit -> done time of the request, in microseconds
        int lat_us = 0;
        if (g->latency && wrc == RR_OK) {
            const double us = std::round((comp.t_done_s - comp.t_submit_s) * 1e6);
            lat_us = us < 1.0 ? 1 : (us > 2147483647.0 ? 2147483647 : (int)us);
        }
        g->pending.push_back(Pending{RR_EV_DONE, nullptr, dep, (int)r->tokens.size(), lat_us});
        gw_finish(g, r, RR_OK);
    } else if (status == RR_CANCELLED) {
        // the owner gave up: a client-side timeout counts as a backend failure (cooldown), a disconnect does not;
        // a latency-based router also records the timeout penalty for the deployment
        g->pending.push_back(Pending{r->cancel_as_failure ? RR_EV_FAIL : RR_EV_DONE, nullptr, dep, n_generated,
                                     g->latency && r->cancel_as_failure ? 1 : 0});
        gw_finish(g, r, r->cancel_as_failure ? RR_TIMEOUT : RR_CANCELLED);
    } else {
        // backend failure: report it, then walk on down the fallback chain with the same request
        g->pending.push_back(Pending{RR_EV_FAIL, nullptr, dep, 0});
        if (r->cancelled) {
            gw_finish(g, r, r->cancel_as_failure ? RR_TIMEOUT : RR_CANCELLED);
        } else {
            r->chain_start = r->chain_pos + 1;
            r->state = Q_ADMIT;
            r->eng = nullptr;
            r->tokens.clear(); r->n_tok.clear(); r->fin.clear();
            r->lp.clear(); r->lp_id.clear();
            r->ptgt.clear(); r->plp.clear(); r->plp_id.clear();     // the next replica scores the prompt again
            r->emb.clear();                                          // and embeds it again
            r->n_cached = 0;
            g->st.failed_over++;
            g->pending.push_back(Pending{RR_EV_ADMIT, r, 0, 0});
        }
    }
}

// Engine worker thread (or the submitting thread for an injected failure): a request of ours finished on `eng`.
static void gw_on_done(void* ctx, uint64_t tag, uint64_t eng_ticket, int status, int n_generated) {
    rr_gateway* g = (rr_gateway*)ctx;
    if (tag == 0) return;                                    // not submitted through this gateway
    GwReq* r = nullptr;
    rr_engine* eng = nullptr;
    int max_new = 0;
    bool logprobs = false;
    size_t k = 1, n_ch = 1, n_score = 0, ks = 1;
    bool embed = false;
    {
        std::lock_guard<std::mutex> lk(g->mu);
        auto it = g->table.find(tag);
        if (it == g->table.end()) return;
        r = it->second;
        eng = r->eng;
        max_new = r->max_new;
        logprobs = r->gen.logprobs();
        k = (size_t)r->gen.lp_width();
        n_ch = (size_t)r->n_choices;
        if (r->gen.scores()) n_score = r->prompt.size() - 1;
        ks = (size_t)r->gen.score_width();
        embed = r->embed;
    }
    // the prompt logprobs first: rr_engine_wait consumes the record
    std::vector<float> ptgt, plp;
    std::vector<int32_t> plp_id;
    int prc = RR_INVALID_ARGUMENT;
    if (eng && status == RR_OK && n_score > 0) {
        ptgt.resize(n_score); plp.resize(n_score * ks); plp_id.resize(n_score * ks);
        prc = rr_engine_prompt_logprobs(eng, eng_ticket, 0.001, ptgt.data(), plp.data(), plp_id.data());
    }
    std::vector<float> emb;
    int erc = RR_INVALID_ARGUMENT;
    if (eng && status == RR_OK && embed) {
        int hidden = 0, dim = 0;
        rr::engine_limits(eng, nullptr, nullptr, nullptr, nullptr, nullptr, &hidden);
        emb.resize((size_t)hidden);
        erc = rr_engine_embedding(eng, eng_ticket, 0.001, emb.data(), hidden, &dim);
    }
    // consume the engine's record (tokens, logprobs, timestamps); a cancelled request has none left
    rr_completion comp;
    memset(&comp, 0, sizeof(comp));
    std::vector<int32_t> toks(n_ch * (size_t)(max_new > 0 ? max_new : 1));
    std::vector<float> lps(logprobs ? toks.size() * k : 0);
    std::vector<int32_t> lp_ids(lps.size());
    std::vector<int32_t> n_toks(n_ch, 0), fins(n_ch, 0);
    int wrc = RR_INVALID_ARGUMENT;
    if (eng && status != RR_CANCELLED)
        wrc = rr_engine_wait(eng, eng_ticket, 0.001, &comp, toks.data(), max_new, logprobs ? lps.data() : nullptr,
                             logprobs ? lp_ids.data() : nullptr, n_toks.data(), fins.data());
    {
        std::lock_guard<std::mutex> lk(g->mu);
        auto it = g->table.find(tag);
        if (it == g->table.end()) return;
        if (prc == RR_OK && wrc == RR_OK) {
            it->second->ptgt.swap(ptgt); it->second->plp.swap(plp); it->second->plp_id.swap(plp_id);
        }
        if (erc == RR_OK && wrc == RR_OK) it->second->emb.swap(emb);
        gw_settle(g, it->second, status, n_generated, wrc, comp, toks.data(), n_toks.data(), fins.data(), lps.data(),
                  lp_ids.data());
    }
    g->cv_work.notify_one();
    g->cv_done.notify_all();
}

// Dispatcher thread, caller holds g->mu: mock replica `rep` serves request r (handed to it at r->t_eng_submit) at once,
// with the same reply for every choice.  Its latency sample is the gateway's hand-off -> settle time.
static void gw_serve_stub(rr_gateway* g, GwReq* r, int rep) {
    const rr_stub_desc& s = g->stubs[(size_t)rep];
    const uint64_t n = ++g->stub_handed[(size_t)rep];
    const bool failed = s.fail_every > 0 && n % (uint64_t)s.fail_every == 0;
    rr_completion comp;
    memset(&comp, 0, sizeof(comp));
    comp.n_generated = failed ? 0 : (r->max_new < s.reply_tokens ? r->max_new : s.reply_tokens);
    std::vector<int32_t> toks((size_t)r->n_choices * r->max_new);
    for (int c = 0; c < r->n_choices; ++c)
        for (int i = 0; i < comp.n_generated; ++i) toks[(size_t)c * r->max_new + i] = 3 + (i % 200);
    comp.t_submit_s = r->t_eng_submit;
    comp.t_first_token_s = comp.t_done_s = gw_now_s(g);
    const int status = failed ? RR_BACKEND_FAILED : RR_OK;
    const std::vector<int32_t> n_toks((size_t)r->n_choices, comp.n_generated), fins((size_t)r->n_choices, 0);
    gw_settle(g, r, status, comp.n_generated * r->n_choices, status, comp, toks.data(), n_toks.data(), fins.data(), nullptr,
              nullptr);
}

static void gw_dispatch(rr_gateway* g) {
    std::vector<Pending> batch;
    std::vector<rr_event> ev;
    std::vector<rr_decision> dec;
    std::vector<GwReq*> to_submit;
    const int cap = g->opts.max_batch_events > 0 ? g->opts.max_batch_events : 4096;
    for (;;) {
        batch.clear();
        {
            std::unique_lock<std::mutex> lk(g->mu);
            g->cv_work.wait(lk, [&] { return g->stop || !g->pending.empty(); });
            if (g->stop && g->pending.empty()) return;
            while (!g->pending.empty() && (int)batch.size() < cap) {
                const Pending p = g->pending.front();
                g->pending.pop_front();
                if (p.type == RR_EV_ADMIT && p.req->cancelled) {     // given up before admission: no event, no debit
                    gw_finish(g, p.req, p.req->cancel_as_failure ? RR_TIMEOUT : RR_CANCELLED);
                    continue;
                }
                batch.push_back(p);
            }
            if (batch.empty()) { g->cv_done.notify_all(); continue; }
            g->busy = true;
        }
        const int64_t now = gw_clock_ms(g);
        ev.clear();
        for (const Pending& p : batch) {
            rr_event e;
            e.type = p.type; e.now_ms = now; e.chain_start = 0;
            if (p.type == RR_EV_ADMIT) {
                // (fields of a queued request are only touched by this thread until the decision is published)
                e.target = p.req->group; e.tokens = (int32_t)p.req->prompt.size(); e.chain_start = p.req->chain_start;
            } else {
                e.target = p.target; e.tokens = p.tokens; e.chain_start = p.aux;
            }
            ev.push_back(e);
        }
        dec.assign(ev.size(), rr_decision{RR_INTERNAL, -1, -1, 0});
        const int rc = rr_router_process(g->router, ev.data(), (int)ev.size(), dec.data());
        to_submit.clear();
        {
            std::lock_guard<std::mutex> lk(g->mu);
            g->st.launches++;
            g->st.events += ev.size();
            if ((uint64_t)ev.size() > g->st.max_batch) g->st.max_batch = ev.size();
            if (g->opts.record_trace > 0) {
                for (size_t i = 0; i < ev.size(); ++i) {
                    const size_t slot = g->tr_count % (size_t)g->opts.record_trace;
                    g->tr_ev[slot] = ev[i]; g->tr_dec[slot] = dec[i];
                    g->tr_count++;
                }
            }
            const double t = gw_now_s(g);
            for (size_t i = 0; i < batch.size(); ++i) {
                if (batch[i].type != RR_EV_ADMIT) continue;
                GwReq* r = batch[i].req;
                r->attempts++;
                r->t_admit = t;
                g->st.admit_wait_s += t - r->t_submit;
                const rr_decision& d = dec[i];
                if (rc != RR_OK) { gw_finish(g, r, RR_INTERNAL); continue; }
                r->deployment = d.deployment; r->served_group = d.served_group; r->chain_pos = d.chain_pos;
                if (d.status == RR_OK) {
                    g->st.admitted++;
                    r->replica = rr::router_dep_replica(g->router, d.deployment);
                    to_submit.push_back(r);
                } else if (d.status == RR_RATE_LIMITED && r->attempts > 1) {
                    gw_finish(g, r, RR_BACKEND_FAILED);      // a backend failed and nothing is left on the chain
                } else {
                    gw_finish(g, r, d.status);
                }
            }
        }
        for (GwReq* r : to_submit) {
            auto it = g->by_replica.find(r->replica);
            const int rep = it == g->by_replica.end() ? -1 : it->second;
            rr_engine* eng = rep < 0 ? nullptr : g->engines[rep];
            const uint64_t id = r->id;           // `r` may be finished and freed by the done hook once it is submitted
            bool cancelled;
            {
                std::lock_guard<std::mutex> lk(g->mu);
                cancelled = r->cancelled;
                if (!cancelled) { r->eng = eng; r->eng_ticket = 0; r->t_eng_submit = gw_now_s(g); }
                if (!cancelled && rep >= 0 && !eng) { gw_serve_stub(g, r, rep); continue; }
            }
            uint64_t tk = 0;
            int src = RR_INTERNAL;
            if (!cancelled && eng && r->embed)
                src = rr::engine_submit_embed_tagged(eng, r->prompt.data(), (int)r->prompt.size(), id, &tk);
            else if (!cancelled && eng)
                src = rr::engine_submit_tagged(eng, r->prompt.data(), (int)r->prompt.size(), r->max_new, id, &tk, r->gen,
                                               r->n_choices);
            bool cancel_now = false;
            std::unique_lock<std::mutex> lk(g->mu);
            if (src == RR_OK) {
                // (the done hook may already have run and finished / re-queued the request: only a still-admitted
                // request becomes RUNNING)
                auto f = g->table.find(id);
                if (f != g->table.end() && f->second->state == Q_ADMIT && f->second->eng == eng && f->second->eng_ticket == 0) {
                    f->second->eng_ticket = tk;
                    f->second->state = RUNNING;
                    cancel_now = f->second->cancelled;       // rr_gateway_cancel raced with the submit: drop the row now
                }
            } else {
                // never reached the backend: give the in-flight slot back (DONE with 0 tokens), fail the request
                g->pending.push_back(Pending{RR_EV_DONE, nullptr, r->deployment, 0});
                gw_finish(g, r, cancelled ? (r->cancel_as_failure ? RR_TIMEOUT : RR_CANCELLED)
                                          : (eng ? src : RR_BACKEND_FAILED));
            }
            lk.unlock();
            if (cancel_now) rr_engine_cancel(eng, tk);
        }
        {
            std::lock_guard<std::mutex> lk(g->mu);
            g->busy = false;
        }
        g->cv_done.notify_all();
    }
}

// ---------------------------------------------------------------------------------------------------- C-ABI
RR_API int rr_gateway_create(rr_router* router, rr_engine* const* engines, const int32_t* replica_ids, int n_engines,
                             const rr_stub_desc* stubs, const rr_gateway_opts* opts, rr_gateway** out) {
    if (!router || !engines || !replica_ids || n_engines < 1 || !out) return RR_INVALID_ARGUMENT;
    rr_gateway* g = new (std::nothrow) rr_gateway();
    if (!g) return RR_INTERNAL;
    g->router = router;
    memset(&g->opts, 0, sizeof(g->opts));
    if (opts) g->opts = *opts;
    memset(&g->st, 0, sizeof(g->st));
    rr::router_shape(router, &g->n_deps, &g->n_groups);
    g->latency = rr::router_strategy(router) == RR_STRATEGY_LATENCY_BASED;
    g->min_ctx = g->min_vocab = g->min_rows = 0x7fffffff;
    g->stubs.assign((size_t)n_engines, rr_stub_desc{0, 0, 0, 0});
    g->stub_handed.assign((size_t)n_engines, 0);
    for (int i = 0; i < n_engines; ++i) {
        g->engines.push_back(engines[i]);
        g->by_replica[replica_ids[i]] = i;
        int c = 0x7fffffff, v = 0, rows = 0x7fffffff, kv = 0, ring = 0;   // a mock replica: no KV limit
        if (engines[i]) {
            rr::engine_limits(engines[i], &c, &v, &rows, &kv, &ring);
            g->kv_pools.emplace_back(kv / rr::KV_PAGE, ring);
        } else {
            if (!stubs || stubs[i].reply_tokens < 0 || stubs[i].fail_every < 0 || stubs[i].vocab < 1) {
                delete g;
                return RR_INVALID_ARGUMENT;
            }
            g->stubs[(size_t)i] = stubs[i];
            g->has_stub = true;
            v = stubs[i].vocab;
        }
        if (c < g->min_ctx) g->min_ctx = c;
        if (v < g->min_vocab) g->min_vocab = v;
        if (rows < g->min_rows) g->min_rows = rows;
    }
    if (g->opts.record_trace > 0) {
        g->tr_ev.resize((size_t)g->opts.record_trace);
        g->tr_dec.resize((size_t)g->opts.record_trace);
    }
    g->t0 = std::chrono::steady_clock::now();
    for (rr_engine* e : g->engines)
        if (e) rr::engine_set_done_hook(e, gw_on_done, g);
    g->dispatcher = std::thread(gw_dispatch, g);
    *out = g;
    return RR_OK;
}

RR_API void rr_gateway_destroy(rr_gateway* g) {
    if (!g) return;
    {
        std::lock_guard<std::mutex> lk(g->mu);
        g->stop = true;
    }
    g->cv_work.notify_all();
    if (g->dispatcher.joinable()) g->dispatcher.join();
    for (rr_engine* e : g->engines)
        if (e) rr::engine_set_done_hook(e, nullptr, nullptr);
    for (auto& kv : g->table) delete kv.second;
    delete g;
}

RR_API int rr_gateway_set_now(rr_gateway* g, int64_t now_ms) {
    if (!g) return RR_INVALID_ARGUMENT;
    g->manual_now_ms.store(now_ms, std::memory_order_relaxed);
    return RR_OK;
}

// embed: an embedding request, max_new 0 (its prompt may fill the context window)
static int gw_check(rr_gateway* g, int group, const int32_t* ids, int n_prompt, int max_new, int n_choices, bool embed) {
    if (group < 0 || group >= g->n_groups) return RR_NO_GROUP;
    if (!ids || n_prompt < 1 || max_new < (embed ? 0 : 1)) return RR_INVALID_ARGUMENT;
    if (n_choices < 1 || n_choices > g->min_rows) return RR_INVALID_ARGUMENT;     // every choice takes a decode row
    if (n_prompt + max_new > g->min_ctx) return RR_INVALID_ARGUMENT;   // -> HTTP 400, before any debit
    // every choice reserves whole 64-token KV pages, at most a windowed engine's ring, in each engine's pool
    // (rr_engine_submit): a request some engine could never fit is refused
    const int pages = (n_prompt + max_new + rr::KV_PAGE - 1) / rr::KV_PAGE;
    for (const auto& kp : g->kv_pools) {
        const int per_choice = kp.second > 0 && pages > kp.second ? kp.second : pages;
        if ((long long)n_choices * per_choice > kp.first) return RR_INVALID_ARGUMENT;
    }
    for (int i = 0; i < n_prompt; ++i)
        if (ids[i] < 0 || ids[i] >= g->min_vocab) return RR_INVALID_ARGUMENT;
    return RR_OK;
}

// p is checked (GenParams::set) against the smallest vocabulary, as prompt ids are: any engine of a fallback accepts it.
static int gw_submit(rr_gateway* g, int group, const int32_t* prompt_ids, const int32_t* prompt_start, int n,
                     int max_new_tokens, int declare_burst, const rr::GenParams& p, int n_choices, uint64_t* tickets,
                     bool embed = false) {
    if (!g || !prompt_ids || !prompt_start || n < 1 || !tickets) return RR_INVALID_ARGUMENT;
    for (int i = 0; i < n; ++i) {
        const int rc = gw_check(g, group, prompt_ids + prompt_start[i], prompt_start[i + 1] - prompt_start[i], max_new_tokens,
                                n_choices, embed);
        if (rc != RR_OK) return rc;
    }
    std::vector<GwReq*> reqs((size_t)n);
    for (int i = 0; i < n; ++i) {
        GwReq* r = new (std::nothrow) GwReq();
        if (!r) { for (int j = 0; j < i; ++j) delete reqs[j]; return RR_INTERNAL; }
        r->group = group; r->max_new = max_new_tokens; r->gen = p; r->n_choices = n_choices; r->embed = embed;
        r->prompt.assign(prompt_ids + prompt_start[i], prompt_ids + prompt_start[i + 1]);
        reqs[i] = r;
    }
    {
        std::lock_guard<std::mutex> lk(g->mu);
        const double t = gw_now_s(g);
        if (declare_burst) g->pending.push_back(Pending{RR_EV_BURST, nullptr, group, n});
        for (int i = 0; i < n; ++i) {                         // one contiguous block of the trace, in request order
            GwReq* r = reqs[i];
            r->id = g->next_id++;
            r->t_submit = t;
            g->table[r->id] = r;
            g->pending.push_back(Pending{RR_EV_ADMIT, r, 0, 0});
            tickets[i] = r->id;
        }
        g->st.submitted += (uint64_t)n;
    }
    g->cv_work.notify_one();
    return RR_OK;
}

RR_API int rr_gateway_submit_batch(rr_gateway* g, int group, const int32_t* prompt_ids, const int32_t* prompt_start, int n,
                                   int max_new_tokens, int declare_burst, uint64_t* tickets) {
    return gw_submit(g, group, prompt_ids, prompt_start, n, max_new_tokens, declare_burst, rr::GenParams(), 1, tickets);
}

// The parameters are checked before the group and the prompt: a request with an unknown group and invalid parameters
// gets RR_INVALID_ARGUMENT.
static int gw_submit_one(rr_gateway* g, int group, const int32_t* prompt_ids, int n_prompt, int max_new_tokens,
                         const rr_gen_params* params, int prompt_top, uint64_t* ticket) {
    if (!g) return RR_INVALID_ARGUMENT;
    rr::GenParams p;
    // the format is checked against the smallest vocabulary: a fallback re-admission may take the request to any replica
    const int rc = p.set(g->min_vocab, params);
    if (rc != RR_OK) return rc;
    if (prompt_top < -1 || prompt_top > rr::LP_MAX_TOP || (prompt_top >= 0 && g->min_vocab % 4)) return RR_INVALID_ARGUMENT;
    p.prompt_top = prompt_top;
    // a mock replica has no logits to fill the pairs from or to mask, and no decode loop to cut
    if ((p.logprobs() || p.stops() || p.json() || p.scores()) && g->has_stub) return RR_INVALID_ARGUMENT;
    const int32_t start[2] = {0, n_prompt};
    return gw_submit(g, group, prompt_ids, start, 1, max_new_tokens, 0, p, params ? params->n_choices : 1, ticket);
}

RR_API int rr_gateway_submit(rr_gateway* g, int group, const int32_t* prompt_ids, int n_prompt, int max_new_tokens,
                             const rr_gen_params* params, uint64_t* ticket) {
    return gw_submit_one(g, group, prompt_ids, n_prompt, max_new_tokens, params, -1, ticket);
}

RR_API int rr_gateway_submit_scored(rr_gateway* g, int group, const int32_t* prompt_ids, int n_prompt, int max_new_tokens,
                                    const rr_gen_params* params, int prompt_top, uint64_t* ticket) {
    return gw_submit_one(g, group, prompt_ids, n_prompt, max_new_tokens, params, prompt_top, ticket);
}

RR_API int rr_gateway_prompt_logprobs(rr_gateway* g, uint64_t ticket, double timeout_s, float* target_lp_out, float* lp_out,
                                      int32_t* id_out) {
    if (!g) return RR_INVALID_ARGUMENT;
    std::unique_lock<std::mutex> lk(g->mu);
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::duration<double>(timeout_s > 0 ? timeout_s : 1e9);
    for (;;) {
        auto it = g->table.find(ticket);
        if (it == g->table.end() || !it->second->gen.scores()) return RR_INVALID_ARGUMENT;
        const GwReq* r = it->second;
        if (r->state == FINISHED) {
            if (r->status != RR_OK) return r->status;
            if (target_lp_out) memcpy(target_lp_out, r->ptgt.data(), sizeof(float) * r->ptgt.size());
            if (lp_out) memcpy(lp_out, r->plp.data(), sizeof(float) * r->plp.size());
            if (id_out) memcpy(id_out, r->plp_id.data(), sizeof(int32_t) * r->plp_id.size());
            return RR_OK;
        }
        if (g->cv_done.wait_until(lk, deadline) == std::cv_status::timeout) {
            it = g->table.find(ticket);
            if (it == g->table.end()) return RR_INVALID_ARGUMENT;
            if (it->second->state != FINISHED) return RR_TIMEOUT;
        }
    }
}

RR_API int rr_gateway_submit_embed(rr_gateway* g, int group, const int32_t* prompt_ids, int n_prompt, uint64_t* ticket) {
    if (!g) return RR_INVALID_ARGUMENT;
    if (g->has_stub) return RR_INVALID_ARGUMENT;       // a mock replica has no hidden state to pool
    const int32_t start[2] = {0, n_prompt};
    return gw_submit(g, group, prompt_ids, start, 1, 0, 0, rr::GenParams(), 1, ticket, true);
}

RR_API int rr_gateway_embedding(rr_gateway* g, uint64_t ticket, double timeout_s, float* out, int capacity, int* dim_out) {
    if (!g || !out) return RR_INVALID_ARGUMENT;
    std::unique_lock<std::mutex> lk(g->mu);
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::duration<double>(timeout_s > 0 ? timeout_s : 1e9);
    for (;;) {
        auto it = g->table.find(ticket);
        if (it == g->table.end() || !it->second->embed) return RR_INVALID_ARGUMENT;
        const GwReq* r = it->second;
        if (r->state == FINISHED) {
            if (r->status != RR_OK) return r->status;
            if ((size_t)capacity < r->emb.size()) return RR_INVALID_ARGUMENT;
            memcpy(out, r->emb.data(), sizeof(float) * r->emb.size());
            if (dim_out) *dim_out = (int)r->emb.size();
            return RR_OK;
        }
        if (g->cv_done.wait_until(lk, deadline) == std::cv_status::timeout) {
            it = g->table.find(ticket);
            if (it == g->table.end()) return RR_INVALID_ARGUMENT;
            if (it->second->state != FINISHED) return RR_TIMEOUT;
        }
    }
}

// caller holds g->mu.  The first min(n, max_tokens_out) tokens of each choice (fewer for a shorter choice) into tokens_out
// [n_choices][max_tokens_out], and of a logprobs request their pairs into lp_out / id_out [n_choices][max_tokens_out]
// [r->gen.lp_width()] (any may be null).
static void gw_copy_choices(const GwReq* r, int n, int max_tokens_out, int32_t* tokens_out, float* lp_out, int32_t* id_out) {
    const size_t k = (size_t)r->gen.lp_width();
    size_t src = 0;
    for (size_t c = 0; c < r->n_tok.size(); src += (size_t)r->n_tok[c], ++c) {
        const int t = std::min(std::min(n, max_tokens_out), (int)r->n_tok[c]);
        if (t <= 0) continue;
        const size_t o = c * (size_t)max_tokens_out;
        if (tokens_out) memcpy(tokens_out + o, r->tokens.data() + src, sizeof(int32_t) * (size_t)t);
        if (!r->gen.logprobs()) continue;
        if (lp_out) memcpy(lp_out + o * k, r->lp.data() + src * k, sizeof(float) * t * k);
        if (id_out) memcpy(id_out + o * k, r->lp_id.data() + src * k, sizeof(int32_t) * t * k);
    }
}

static void gw_fill(const GwReq* r, rr_gateway_result* out) {
    out->ticket = r->id; out->status = r->state == FINISHED ? r->status : -1;
    out->deployment = r->deployment; out->served_group = r->served_group; out->chain_pos = r->chain_pos;
    out->replica = r->replica; out->n_prompt = (int32_t)r->prompt.size(); out->n_generated = (int32_t)r->n_gen();
    out->attempts = r->attempts;
    out->t_submit_s = r->t_submit; out->t_admit_s = r->t_admit; out->t_first_token_s = r->t_first; out->t_done_s = r->t_done;
    out->n_cached = r->n_cached; out->finish = r->fin.empty() ? 0 : r->fin[0];
}

RR_API int rr_gateway_wait(rr_gateway* g, uint64_t ticket, double timeout_s, rr_gateway_result* out, int32_t* tokens_out,
                           int max_tokens_out, float* lp_out, int32_t* id_out, int32_t* n_tokens_out, int32_t* finish_out) {
    if (!g || !out) return RR_INVALID_ARGUMENT;
    std::unique_lock<std::mutex> lk(g->mu);
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::duration<double>(timeout_s > 0 ? timeout_s : 1e9);
    GwReq* r = nullptr;
    for (;;) {
        auto it = g->table.find(ticket);
        if (it == g->table.end()) return RR_INVALID_ARGUMENT;
        r = it->second;
        if (r->state == FINISHED) break;
        if (g->cv_done.wait_until(lk, deadline) == std::cv_status::timeout) {
            it = g->table.find(ticket);
            if (it == g->table.end()) return RR_INVALID_ARGUMENT;
            r = it->second;
            if (r->state == FINISHED) break;
            gw_fill(r, out);
            out->status = RR_TIMEOUT;
            return RR_TIMEOUT;                                // still in flight: wait again or rr_gateway_cancel
        }
    }
    gw_fill(r, out);
    gw_copy_choices(r, r->n_gen(), max_tokens_out, tokens_out, lp_out, id_out);
    for (int c = 0; c < r->n_choices; ++c) {      // a request that never reached a replica has no per-choice record
        if (n_tokens_out) n_tokens_out[c] = (size_t)c < r->n_tok.size() ? r->n_tok[c] : 0;
        if (finish_out) finish_out[c] = (size_t)c < r->fin.size() ? r->fin[c] : 0;
    }
    const int status = r->status;
    g->table.erase(ticket);
    delete r;
    return status;
}

RR_API int rr_gateway_peek(rr_gateway* g, uint64_t ticket, int have, double timeout_s, int32_t* tokens_out, int max_tokens_out,
                           int32_t* n_generated, int32_t* done, rr_gateway_result* out, float* lp_out, int32_t* id_out) {
    if (!g || !n_generated || !done) return RR_INVALID_ARGUMENT;
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::duration<double>(timeout_s > 0 ? timeout_s : 1e9);
    for (;;) {
        rr_engine* eng = nullptr;
        uint64_t tk = 0;
        {
            std::unique_lock<std::mutex> lk(g->mu);
            for (;;) {
                auto it = g->table.find(ticket);
                if (it == g->table.end()) return RR_INVALID_ARGUMENT;
                GwReq* r = it->second;
                if (r->n_choices > 1) return RR_INVALID_ARGUMENT;
                if (out) gw_fill(r, out);
                if (r->state == FINISHED) {
                    const int n = r->n_gen();
                    *n_generated = n; *done = 1;
                    gw_copy_choices(r, n, max_tokens_out, tokens_out, lp_out, id_out);
                    return RR_OK;
                }
                if (r->state == RUNNING) { eng = r->eng; tk = r->eng_ticket; break; }
                if (g->cv_done.wait_until(lk, deadline) == std::cv_status::timeout) { *n_generated = 0; *done = 0; return RR_OK; }
            }
        }
        const double left = std::chrono::duration<double>(deadline - std::chrono::steady_clock::now()).count();
        int32_t n = 0, d = 0;
        const int rc = rr_engine_peek(eng, tk, have, left > 0.001 ? left : 0.001, tokens_out, max_tokens_out, &n, &d, nullptr,
                                      lp_out, id_out);
        if (rc == RR_OK && !d) { *n_generated = n; *done = 0; return RR_OK; }
        // finished (the hook is consuming / has consumed the engine's record) or failed over: look at our own record again
        if (std::chrono::steady_clock::now() >= deadline) { *n_generated = rc == RR_OK ? n : 0; *done = 0; return RR_OK; }
        std::unique_lock<std::mutex> lk(g->mu);
        g->cv_done.wait_for(lk, std::chrono::milliseconds(1));
    }
}

RR_API int rr_gateway_cancel(rr_gateway* g, uint64_t ticket, int count_as_failure) {
    if (!g) return RR_INVALID_ARGUMENT;
    rr_engine* eng = nullptr;
    uint64_t tk = 0;
    {
        std::lock_guard<std::mutex> lk(g->mu);
        auto it = g->table.find(ticket);
        if (it == g->table.end()) return RR_INVALID_ARGUMENT;
        GwReq* r = it->second;
        if (r->state == FINISHED) { g->table.erase(it); delete r; return RR_OK; }
        r->cancelled = true; r->cancel_as_failure = count_as_failure != 0; r->abandoned = true;
        if (r->state == RUNNING) { eng = r->eng; tk = r->eng_ticket; }
        // Q_ADMIT: the dispatcher / done hook sees `cancelled` when it gets to the request
    }
    if (eng) rr_engine_cancel(eng, tk);          // the done hook reports RR_CANCELLED and posts the DONE / FAIL event
    return RR_OK;
}

// Block until every event queued so far (DONE / FAIL reports of finished requests included) has been through K1.
RR_API int rr_gateway_quiesce(rr_gateway* g, double timeout_s) {
    if (!g) return RR_INVALID_ARGUMENT;
    std::unique_lock<std::mutex> lk(g->mu);
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::duration<double>(timeout_s > 0 ? timeout_s : 1e9);
    while (!g->pending.empty() || g->busy) {
        g->cv_work.notify_one();
        if (g->cv_done.wait_until(lk, deadline) == std::cv_status::timeout) return RR_TIMEOUT;
    }
    return RR_OK;
}

RR_API int rr_gateway_get_stats(rr_gateway* g, rr_gateway_stats* out) {
    if (!g || !out) return RR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> lk(g->mu);
    *out = g->st;
    out->in_flight = (uint64_t)g->table.size();
    return RR_OK;
}

RR_API int rr_gateway_trace(rr_gateway* g, rr_event* events, rr_decision* decisions, int capacity, int* n) {
    if (!g || !n) return RR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> lk(g->mu);
    const size_t cap = (size_t)(g->opts.record_trace > 0 ? g->opts.record_trace : 0);
    const size_t have = g->tr_count < cap ? g->tr_count : cap;
    *n = (int)have;
    if (!events || !decisions || (size_t)capacity < have) return have ? RR_INVALID_ARGUMENT : RR_OK;
    const size_t first = g->tr_count - have;
    for (size_t i = 0; i < have; ++i) {
        events[i] = g->tr_ev[(first + i) % cap];
        decisions[i] = g->tr_dec[(first + i) % cap];
    }
    return RR_OK;
}
