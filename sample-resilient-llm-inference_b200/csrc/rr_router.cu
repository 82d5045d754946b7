// rr_router.cu — K1: admission + rpm/tpm bucket debit + backend pick + cooldown + fallback chain.
//
// Replaces litellm.Router as configured by reference config/config.yaml:35-108 and called from
// reference src/demo_load_balancing.py:106-110, src/demo_fallback.py:143-147,
// src/demo_quota_isolation.py:52-56.  Semantics are those of oracle/router.py (latency-based routing:
// oracle/latency_router.py) (serialised-trace: the result of one launch over an ordered event trace equals processing
// the events one by one).
//
// Design: router state (per-deployment window counters, in-flight counts, cooldown deadlines,
// MT19937 stream, round-robin cursors) is resident in HBM between launches and staged in shared memory for the
// duration of one (router_kernel_smem; router_kernel keeps it in HBM for topologies that do not fit).  The picks of one trace depend on each
// other through the RNG stream and the counters, so the trace is consumed by ONE warp in order;
// the parallelism is across the <=32 candidate deployments of a model group: lane l owns
// candidate l — eligibility is a ballot, the weighted pick is a rank-ordered scan + ballot
// bisect, least-busy is a warp min-reduction, latency-based a warp min over per-lane mean latencies + a ballot of the
// lanes within the buffer + a rank under (mean, lane).  Launches on one router are serialised (rr_router_process_device).
// The RNG is CPython's: MT19937 with init_by_array seeding, random() = (a>>5, b>>6) 53-bit
// doubles, _randbelow = getrandbits rejection loop (Lib/random.py:242-250, 454-489).
// Latency/atomic-bound: not a roofline kernel (SURVEY.md §8d); reported as ns/event.
#include "rr_kernels.h"
#include "rr_launch.cuh"

#include <mutex>
#include <new>
#include <stdlib.h>
#include <string.h>
#include <vector>

#define RR_API extern "C" __attribute__((visibility("default")))

namespace rr {
void note_cuda_error(cudaError_t e);

struct RouterDev {
    int n_deps, n_groups;
    int strategy, pre_call, allowed_fails, cooldown_ms;
    // config (read-only)
    const int32_t* group_off;   // [n_groups+1]
    const int32_t* group_deps;  // [n_deps] deployment ids grouped, config order inside a group
    const int32_t* fb_off;      // [n_groups+1]
    const int32_t* fb_groups;
    const int32_t* dep_group;   // [n_deps]
    const int32_t* rpm;
    const int32_t* tpm;
    const int32_t* weight;
    // state
    long long* window;
    int* req_count;
    int* tok_count;
    long long* fail_window;
    int* fail_count;
    int* inflight;
    long long* cooldown_until;
    long long* total_admitted;
    int* rr_next;               // [n_groups] round-robin cursor
    int* burst_size;            // [n_groups] split strategy: size of the declared burst (RR_EV_BURST)
    int* burst_pos;             // [n_groups] split strategy: requests of the burst seen so far
    uint32_t* mt;               // [624] + index at [624]
    // latency-based strategy only (nullptr otherwise).  The per-deployment sample list is stored in O(1) form: the list
    // rule freezes its first N-1 entries and only ever replaces the last one, so Python's in-order sum of the list is
    // exactly  n < N ? lat_head : lat_head + lat_last.
    int lat_cap;                // N = max_latency_list_size
    long long lat_ttl_ms;
    double lat_buf;             // lowest_latency_buffer = ppm / 1e6
    int* lat_n;                 // [n_deps] samples held, <= N
    double* lat_head;           // [n_deps] in-order sum (from 0.0) of the first min(n, N-1) samples
    double* lat_last;           // [n_deps] the N-th sample (valid when n == N)
    long long* lat_stamp;       // [n_groups] now_ms of the group's last write, -1 = never
};

// ---------------------------------------------------------------- device MT19937 (one warp)
struct WarpMT {
    uint32_t* mt;   // shared memory, 624 words
    int mti;

    __device__ __forceinline__ void regenerate() {
        const uint32_t UPPER = 0x80000000u, LOWER = 0x7fffffffu, MAG = 0x9908b0dfu;
        const int lane = threadIdx.x & 31;
        for (int base = 0; base < 227; base += 32) {
            int kk = base + lane;
            uint32_t v = 0;
            bool on = kk < 227;
            if (on) {
                uint32_t y = (mt[kk] & UPPER) | (mt[kk + 1] & LOWER);
                v = mt[kk + 397] ^ (y >> 1) ^ ((y & 1u) ? MAG : 0u);
            }
            __syncwarp();
            if (on) mt[kk] = v;
            __syncwarp();
        }
        for (int base = 227; base < 623; base += 32) {
            int kk = base + lane;
            uint32_t v = 0;
            bool on = kk < 623;
            if (on) {
                uint32_t y = (mt[kk] & UPPER) | (mt[kk + 1] & LOWER);
                v = mt[kk - 227] ^ (y >> 1) ^ ((y & 1u) ? MAG : 0u);
            }
            __syncwarp();
            if (on) mt[kk] = v;
            __syncwarp();
        }
        if (lane == 0) {
            uint32_t y = (mt[623] & UPPER) | (mt[0] & LOWER);
            mt[623] = mt[396] ^ (y >> 1) ^ ((y & 1u) ? MAG : 0u);
        }
        __syncwarp();
        mti = 0;
    }
    // warp-uniform: every lane returns the same value
    __device__ __forceinline__ uint32_t next_u32() {
        if (mti >= 624) regenerate();
        uint32_t y = mt[mti++];
        y ^= (y >> 11);
        y ^= (y << 7) & 0x9d2c5680u;
        y ^= (y << 15) & 0xefc60000u;
        y ^= (y >> 18);
        return y;
    }
    __device__ __forceinline__ double next_double() {   // random.random()
        uint32_t a = next_u32() >> 5, b = next_u32() >> 6;
        return __dmul_rn(__dadd_rn(__dmul_rn((double)a, 67108864.0), (double)b),
                         1.0 / 9007199254740992.0);
    }
    __device__ __forceinline__ uint32_t randbelow(uint32_t n) {   // Random._randbelow_with_getrandbits
        int k = 32 - __clz(n);                                  // n.bit_length()
        uint32_t r = next_u32() >> (32 - k);
        while (r >= n) r = next_u32() >> (32 - k);
        return r;
    }
};

// position of the n-th (0-based) set bit of `mask`; the caller guarantees n < popc(mask).  Five popc steps instead of
// __fns (a software loop): this sits on the dependent chain of every pick.
__device__ __forceinline__ int nth_set_lane(uint32_t mask, int n) {
    int pos = 0;
    uint32_t m = mask;
    int c = __popc(m & 0xFFFFu); if (n >= c) { n -= c; pos += 16; m >>= 16; }
    c = __popc(m & 0xFFu);       if (n >= c) { n -= c; pos += 8;  m >>= 8; }
    c = __popc(m & 0xFu);        if (n >= c) { n -= c; pos += 4;  m >>= 4; }
    c = __popc(m & 0x3u);        if (n >= c) { n -= c; pos += 2;  m >>= 2; }
    if (n >= (int)(m & 1u)) pos += 1;
    return pos;
}

// State accessors: LOCAL = the arrays live in this CTA's shared memory for the duration of the launch (plain accesses);
// otherwise they are in HBM (L2-coherent loads / stores, atomics for the debits).
template <bool LOCAL, typename T> __device__ __forceinline__ T st_ld(const T* p) { return LOCAL ? *p : __ldcg(p); }
template <bool LOCAL, typename T> __device__ __forceinline__ void st_st(T* p, T v) { if (LOCAL) *p = v; else __stcg(p, v); }
template <bool LOCAL> __device__ __forceinline__ int st_add(int* p, int v) {
    if (LOCAL) { const int o = *p; *p = o + v; return o; }
    return atomicAdd(p, v);
}

// Latency-based strategy: one sample for deployment d (one lane).  An expired model group drops every list first; the
// list rule is litellm's: append while shorter than N, otherwise list[:N-1] + [sample].
template <bool LOCAL>
__device__ __forceinline__ void lat_record(const RouterDev& S, int d, double sample, long long now) {
    const int g = S.dep_group[d];
    if (now - st_ld<LOCAL>(&S.lat_stamp[g]) > S.lat_ttl_ms) {
        for (int j = S.group_off[g]; j < S.group_off[g + 1]; ++j) {
            const int k = S.group_deps[j];
            st_st<LOCAL>(&S.lat_n[k], 0);
            st_st<LOCAL>(&S.lat_head[k], 0.0);
            st_st<LOCAL>(&S.lat_last[k], 0.0);
        }
    }
    const int n = st_ld<LOCAL>(&S.lat_n[d]);
    if (n < S.lat_cap - 1) st_st<LOCAL>(&S.lat_head[d], __dadd_rn(st_ld<LOCAL>(&S.lat_head[d]), sample));
    else st_st<LOCAL>(&S.lat_last[d], sample);
    if (n < S.lat_cap) st_st<LOCAL>(&S.lat_n[d], n + 1);
    st_st<LOCAL>(&S.lat_stamp[g], now);
}

// Walks events[0, n_events) in order (one warp).  `events` / `decisions` may be global or shared memory.
// LAT: the router is latency-based (its state arrays exist); the other strategies run the LAT = false instantiation,
// which carries none of the latency code.
template <bool LOCAL, bool LAT>
__device__ __forceinline__ void run_trace(const RouterDev& S, WarpMT& rng, const rr_event* events, int n_events,
                                          rr_decision* decisions) {
    const int lane = threadIdx.x;
    const uint32_t lt_mask = (1u << lane) - 1u;

    for (int e = 0; e < n_events; ++e) {
        const rr_event ev = events[e];
        rr_decision dec;
        dec.status = RR_NO_GROUP;
        dec.deployment = -1;
        dec.served_group = -1;
        dec.chain_pos = 0;
        const long long now = ev.now_ms;
        const long long minute = now / 60000;

        if (ev.type == RR_EV_ADMIT) {
            const int g = ev.target;
            if (g >= 0 && g < S.n_groups) {
                dec.status = RR_RATE_LIMITED;
                const int fb0 = S.fb_off[g];
                const int chain_len = 1 + (S.fb_off[g + 1] - fb0);
                for (int pos = ev.chain_start < 0 ? 0 : ev.chain_start; pos < chain_len; ++pos) {
                    const int grp = pos == 0 ? g : S.fb_groups[fb0 + pos - 1];
                    const int off = S.group_off[grp];
                    const int cnt = S.group_off[grp + 1] - off;
                    const bool valid = lane < cnt;
                    const int d = valid ? S.group_deps[off + lane] : 0;
                    int req = 0, tok = 0, infl = 0x7fffffff, w = -1;
                    bool healthy = false;
                    if (valid) {
                        // roll the fixed one-minute window (bucket refill)
                        if (st_ld<LOCAL>(&S.window[d]) != minute) {
                            st_st<LOCAL>(&S.window[d], (long long)minute);
                            st_st<LOCAL>(&S.req_count[d], 0);
                            st_st<LOCAL>(&S.tok_count[d], 0);
                        } else {
                            req = st_ld<LOCAL>(&S.req_count[d]);
                            tok = st_ld<LOCAL>(&S.tok_count[d]);
                        }
                        infl = st_ld<LOCAL>(&S.inflight[d]);
                        w = S.weight[d];
                        healthy = now >= st_ld<LOCAL>(&S.cooldown_until[d]);
                        if (healthy && S.pre_call) {
                            const int rpm = S.rpm[d], tpm = S.tpm[d];
                            if (rpm >= 0 && req >= rpm) healthy = false;
                            if (tpm >= 0 && (long long)tok + ev.tokens > tpm) healthy = false;
                        }
                    }
                    const uint32_t mask = __ballot_sync(0xffffffffu, healthy);
                    if (mask == 0) continue;
                    const int nh = __popc(mask);
                    const int rank = __popc(mask & lt_mask);
                    int pick_lane = -1;
                    bool uniform = false;
                    if (S.strategy == RR_STRATEGY_SIMPLE_SHUFFLE) {
                        const int first = __ffs(mask) - 1;
                        const int w0 = __shfl_sync(0xffffffffu, w, first);
                        long long total = 0;
                        const int wc = healthy ? (w > 0 ? w : 0) : 0;
                        if (w0 >= 0) {
                            total = wc;
                            for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
                        }
                        if (w0 >= 0 && total > 0) {
                            const double norm = __ddiv_rn((double)wc, (double)total);
                            // sequential (rank-ordered) accumulate == itertools.accumulate
                            double cum = 0.0, prev = 0.0;
                            for (int r = 0; r < nh; ++r) {
                                const int src = nth_set_lane(mask, r);
                                if (lane == src) cum = (r == 0) ? norm : __dadd_rn(prev, norm);
                                prev = __shfl_sync(0xffffffffu, cum, src);
                            }
                            const double tot = __dadd_rn(prev, 0.0);
                            const double x = __dmul_rn(rng.next_double(), tot);
                            // bisect_right(cum, x, 0, nh-1)
                            const uint32_t le =
                                __ballot_sync(0xffffffffu, healthy && rank < nh - 1 && cum <= x);
                            pick_lane = nth_set_lane(mask, __popc(le));
                        } else {
                            uniform = true;
                        }
                    } else if (S.strategy == RR_STRATEGY_LEAST_BUSY) {
                        // first candidate (config order) with minimum in-flight count
                        unsigned long long key =
                            valid ? (((unsigned long long)(unsigned)infl) << 8) | (unsigned)lane
                                  : ~0ull;
                        for (int o = 16; o > 0; o >>= 1) {
                            unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
                            key = other < key ? other : key;
                        }
                        const int best = (int)(key & 0xff);
                        if ((mask >> best) & 1u) pick_lane = best;
                        else uniform = true;
                    } else if (S.strategy == RR_STRATEGY_ROUND_ROBIN) {
                        int k = st_ld<LOCAL>(&S.rr_next[grp]);
                        __syncwarp();
                        if (lane == 0) st_st<LOCAL>(&S.rr_next[grp], k + 1);
                        pick_lane = nth_set_lane(mask, k % nh);
                    } else if (S.strategy == RR_STRATEGY_SPLIT) {
                        // contiguous shares of the declared burst: request i of N -> healthy[i * nh / N]
                        const int n = st_ld<LOCAL>(&S.burst_size[grp]);
                        const int i = st_ld<LOCAL>(&S.burst_pos[grp]);
                        __syncwarp();
                        if (lane == 0) st_st<LOCAL>(&S.burst_pos[grp], i + 1);
                        int idx = n > 0 ? (int)(((long long)i * nh) / n) : 0;
                        if (idx > nh - 1) idx = nh - 1;
                        pick_lane = nth_set_lane(mask, idx);
                    } else if (LAT) {   // RR_STRATEGY_LATENCY_BASED
                        // drop an expired group's samples, then mean = total / len per healthy lane (0.0 unmeasured)
                        const bool expired = now - st_ld<LOCAL>(&S.lat_stamp[grp]) > S.lat_ttl_ms;   // warp-uniform
                        double mean = 0.0;
                        if (valid) {
                            if (expired) {
                                st_st<LOCAL>(&S.lat_n[d], 0);
                                st_st<LOCAL>(&S.lat_head[d], 0.0);
                                st_st<LOCAL>(&S.lat_last[d], 0.0);
                            } else {
                                const int n = st_ld<LOCAL>(&S.lat_n[d]);
                                if (n > 0) {
                                    const double head = st_ld<LOCAL>(&S.lat_head[d]);
                                    const double tot = n < S.lat_cap ? head : __dadd_rn(head, st_ld<LOCAL>(&S.lat_last[d]));
                                    mean = __ddiv_rn(tot, (double)n);
                                }
                            }
                        }
                        double lowest = healthy ? mean : __longlong_as_double(0x7ff0000000000000ll);   // +inf
                        for (int o = 16; o > 0; o >>= 1) {
                            const double other = __shfl_xor_sync(0xffffffffu, lowest, o);
                            lowest = other < lowest ? other : lowest;
                        }
                        // two roundings, as Python computes lowest + (buf * lowest): no FMA
                        const double threshold = __dadd_rn(lowest, __dmul_rn(S.lat_buf, lowest));
                        const bool in = healthy && mean <= threshold;
                        const uint32_t vmask = __ballot_sync(0xffffffffu, in);
                        // random.choice(sorted(valid, key=mean)): rank of each valid lane under (mean, lane)
                        const int r = (int)rng.randbelow((uint32_t)__popc(vmask));
                        int rk = 0;
                        for (uint32_t m = vmask; m; m &= m - 1) {
                            const int k = __ffs(m) - 1;
                            const double mk = __shfl_sync(0xffffffffu, mean, k);
                            rk += (mk < mean || (mk == mean && k < lane)) ? 1 : 0;
                        }
                        pick_lane = __ffs(__ballot_sync(0xffffffffu, in && rk == r)) - 1;
                    } else {   // RR_STRATEGY_RANDOM: uniform, weights ignored
                        uniform = true;
                    }
                    if (uniform) pick_lane = nth_set_lane(mask, (int)rng.randbelow((uint32_t)nh));
                    if (lane == pick_lane) {
                        st_add<LOCAL>(&S.req_count[d], 1);
                        st_add<LOCAL>(&S.tok_count[d], ev.tokens);
                        st_add<LOCAL>(&S.inflight[d], 1);
                        st_st<LOCAL>(&S.total_admitted[d], st_ld<LOCAL>(&S.total_admitted[d]) + 1ll);
                    }
                    dec.status = RR_OK;
                    dec.deployment = __shfl_sync(0xffffffffu, d, pick_lane);
                    dec.served_group = grp;
                    dec.chain_pos = pos;
                    break;
                }
                if (dec.status != RR_OK) {
                    dec.deployment = -1;
                    dec.served_group = -1;
                    dec.chain_pos = 0;
                }
            }
        } else if (ev.type == RR_EV_BURST) {
            const int g = ev.target;
            if (g >= 0 && g < S.n_groups) {
                if (lane == 0) { st_st<LOCAL>(&S.burst_size[g], ev.tokens); st_st<LOCAL>(&S.burst_pos[g], 0); }
                dec.status = RR_OK;
                dec.served_group = g;
            }
        } else if (ev.type == RR_EV_DONE || ev.type == RR_EV_FAIL) {
            const int d = ev.target;
            if (d >= 0 && d < S.n_deps) {
                int cooled = 0;
                if (lane == 0) {
                    int old = atomicSub(&S.inflight[d], 1);
                    if (old <= 0) st_add<LOCAL>(&S.inflight[d], 1);   // clamp at 0
                    if (ev.type == RR_EV_DONE) {
                        if (st_ld<LOCAL>(&S.window[d]) != minute) {
                            st_st<LOCAL>(&S.window[d], (long long)minute);
                            st_st<LOCAL>(&S.req_count[d], 0);
                            st_st<LOCAL>(&S.tok_count[d], 0);
                        }
                        st_add<LOCAL>(&S.tok_count[d], ev.tokens);
                    } else {
                        if (st_ld<LOCAL>(&S.fail_window[d]) != minute) {
                            st_st<LOCAL>(&S.fail_window[d], (long long)minute);
                            st_st<LOCAL>(&S.fail_count[d], 0);
                        }
                        int fc = st_ld<LOCAL>(&S.fail_count[d]) + 1;
                        st_st<LOCAL>(&S.fail_count[d], fc);
                        if (fc > S.allowed_fails) {
                            st_st<LOCAL>(&S.cooldown_until[d], now + (long long)S.cooldown_ms);
                            cooled = 1;
                        }
                    }
                    if (LAT) {
                        // DONE: chain_start = latency in us -> us per output token; FAIL: chain_start 1 = timeout -> 1e9
                        if (ev.type == RR_EV_DONE && ev.chain_start > 0)
                            lat_record<LOCAL>(S, d, ev.tokens > 0 ? __ddiv_rn((double)ev.chain_start, (double)ev.tokens)
                                                                  : (double)ev.chain_start, now);
                        else if (ev.type == RR_EV_FAIL && ev.chain_start == 1)
                            lat_record<LOCAL>(S, d, 1e9, now);
                    }
                }
                cooled = __shfl_sync(0xffffffffu, cooled, 0);
                dec.status = RR_OK;
                dec.deployment = d;
                dec.served_group = S.dep_group[d];
                dec.chain_pos = cooled;
            }
        }
        if (lane == 0) decisions[e] = dec;
        __syncwarp();
        if (!LOCAL) __threadfence_block();
    }
    __syncwarp();
}


// ---- kernel, state in HBM (any topology) ----------------------------------------------------------
template <bool LAT>
__global__ void __launch_bounds__(32, 1)
router_kernel(RouterDev S, const rr_event* __restrict__ events, int n_events,
              rr_decision* __restrict__ decisions) {
    __shared__ uint32_t s_mt[624];
    const int lane = threadIdx.x;
    for (int i = lane; i < 624; i += 32) s_mt[i] = S.mt[i];
    WarpMT rng;
    rng.mt = s_mt;
    rng.mti = (int)S.mt[624];
    __syncwarp();
    run_trace<false, LAT>(S, rng, events, n_events, decisions);
    for (int i = lane; i < 624; i += 32) S.mt[i] = s_mt[i];
    if (lane == 0) S.mt[624] = (uint32_t)rng.mti;
}

// ---- kernel, state staged in shared memory ---------------------------------------------------------
// A trace is a chain of dependent decisions, so what bounds it is the latency of every state access.  All mutable state
// of a router is a few dozen bytes per deployment: this variant copies config + state into shared memory once, walks the
// trace there (events and decisions move through shared memory in chunks of 128, loaded / stored by all lanes), and
// writes the state back at the end.  Launches on one router are serialised by the library (stream order + an event
// chain), which the MT19937 stream required anyway.
constexpr int RT_CHUNK = 128;
struct RouterSmemLayout {
    uint32_t o_window, o_failw, o_cool, o_total, o_req, o_tok, o_failc, o_infl, o_rpm, o_tpm, o_wt, o_dgrp, o_gdeps,
        o_goff, o_fboff, o_fbg, o_rr, o_bs, o_bp, o_mt, o_ev, o_dec, o_lat_n, o_lat_head, o_lat_last, o_lat_stamp, total;
};
// `latency`: the latency-based strategy's arrays follow the common ones (zero bytes for every other strategy)
__host__ __device__ inline RouterSmemLayout router_smem_layout(int n_deps, int n_groups, int n_fb, bool latency) {
    RouterSmemLayout L;
    uint32_t off = 0;
    auto take = [&](uint32_t bytes) { uint32_t o = off; off += (bytes + 15u) & ~15u; return o; };
    L.o_window = take(8 * n_deps); L.o_failw = take(8 * n_deps); L.o_cool = take(8 * n_deps); L.o_total = take(8 * n_deps);
    L.o_req = take(4 * n_deps); L.o_tok = take(4 * n_deps); L.o_failc = take(4 * n_deps); L.o_infl = take(4 * n_deps);
    L.o_rpm = take(4 * n_deps); L.o_tpm = take(4 * n_deps); L.o_wt = take(4 * n_deps); L.o_dgrp = take(4 * n_deps);
    L.o_gdeps = take(4 * n_deps);
    L.o_goff = take(4 * (n_groups + 1)); L.o_fboff = take(4 * (n_groups + 1)); L.o_fbg = take(4 * (n_fb > 0 ? n_fb : 1));
    L.o_rr = take(4 * n_groups); L.o_bs = take(4 * n_groups); L.o_bp = take(4 * n_groups);
    L.o_mt = take(4 * 624);
    L.o_ev = take(sizeof(rr_event) * RT_CHUNK); L.o_dec = take(sizeof(rr_decision) * RT_CHUNK);
    const int ld = latency ? n_deps : 0, lg = latency ? n_groups : 0;
    L.o_lat_n = take(4 * ld); L.o_lat_head = take(8 * ld); L.o_lat_last = take(8 * ld); L.o_lat_stamp = take(8 * lg);
    L.total = off;
    return L;
}

template <typename T>
__device__ __forceinline__ void warp_copy(T* dst, const T* src, int n) {
    for (int i = threadIdx.x; i < n; i += 32) dst[i] = src[i];
}

template <bool LAT>
__global__ void __launch_bounds__(32, 1)
router_kernel_smem(RouterDev G, int n_fb, const rr_event* __restrict__ events, int n_events,
                   rr_decision* __restrict__ decisions) {
    extern __shared__ __align__(16) uint8_t rt_smem[];
    constexpr bool lat = LAT;
    const RouterSmemLayout L = router_smem_layout(G.n_deps, G.n_groups, n_fb, lat);
    const int lane = threadIdx.x, nd = G.n_deps, ng = G.n_groups;
    RouterDev S = G;                                       // same scalars, pointers redirected into shared memory
    long long* window = (long long*)(rt_smem + L.o_window); long long* failw = (long long*)(rt_smem + L.o_failw);
    long long* cool = (long long*)(rt_smem + L.o_cool);     long long* total = (long long*)(rt_smem + L.o_total);
    int* req = (int*)(rt_smem + L.o_req);   int* tok = (int*)(rt_smem + L.o_tok);
    int* failc = (int*)(rt_smem + L.o_failc); int* infl = (int*)(rt_smem + L.o_infl);
    int32_t* rpm = (int32_t*)(rt_smem + L.o_rpm); int32_t* tpm = (int32_t*)(rt_smem + L.o_tpm);
    int32_t* wt = (int32_t*)(rt_smem + L.o_wt);   int32_t* dgrp = (int32_t*)(rt_smem + L.o_dgrp);
    int32_t* gdeps = (int32_t*)(rt_smem + L.o_gdeps); int32_t* goff = (int32_t*)(rt_smem + L.o_goff);
    int32_t* fboff = (int32_t*)(rt_smem + L.o_fboff); int32_t* fbg = (int32_t*)(rt_smem + L.o_fbg);
    int* rrn = (int*)(rt_smem + L.o_rr); int* bs = (int*)(rt_smem + L.o_bs); int* bp = (int*)(rt_smem + L.o_bp);
    uint32_t* s_mt = (uint32_t*)(rt_smem + L.o_mt);
    rr_event* s_ev = (rr_event*)(rt_smem + L.o_ev); rr_decision* s_dec = (rr_decision*)(rt_smem + L.o_dec);

    warp_copy(window, (const long long*)G.window, nd); warp_copy(failw, (const long long*)G.fail_window, nd);
    warp_copy(cool, (const long long*)G.cooldown_until, nd); warp_copy(total, (const long long*)G.total_admitted, nd);
    warp_copy(req, (const int*)G.req_count, nd); warp_copy(tok, (const int*)G.tok_count, nd);
    warp_copy(failc, (const int*)G.fail_count, nd); warp_copy(infl, (const int*)G.inflight, nd);
    warp_copy(rpm, G.rpm, nd); warp_copy(tpm, G.tpm, nd); warp_copy(wt, G.weight, nd); warp_copy(dgrp, G.dep_group, nd);
    warp_copy(gdeps, G.group_deps, nd); warp_copy(goff, G.group_off, ng + 1); warp_copy(fboff, G.fb_off, ng + 1);
    warp_copy(fbg, G.fb_groups, n_fb);
    warp_copy(rrn, (const int*)G.rr_next, ng); warp_copy(bs, (const int*)G.burst_size, ng); warp_copy(bp, (const int*)G.burst_pos, ng);
    warp_copy(s_mt, (const uint32_t*)G.mt, 624);
    S.window = window; S.fail_window = failw; S.cooldown_until = cool; S.total_admitted = total;
    S.req_count = req; S.tok_count = tok; S.fail_count = failc; S.inflight = infl;
    S.rpm = rpm; S.tpm = tpm; S.weight = wt; S.dep_group = dgrp; S.group_deps = gdeps; S.group_off = goff;
    S.fb_off = fboff; S.fb_groups = fbg; S.rr_next = rrn; S.burst_size = bs; S.burst_pos = bp;
    if (lat) {
        S.lat_n = (int*)(rt_smem + L.o_lat_n); S.lat_head = (double*)(rt_smem + L.o_lat_head);
        S.lat_last = (double*)(rt_smem + L.o_lat_last); S.lat_stamp = (long long*)(rt_smem + L.o_lat_stamp);
        warp_copy(S.lat_n, (const int*)G.lat_n, nd); warp_copy(S.lat_head, (const double*)G.lat_head, nd);
        warp_copy(S.lat_last, (const double*)G.lat_last, nd); warp_copy(S.lat_stamp, (const long long*)G.lat_stamp, ng);
    }
    WarpMT rng;
    rng.mt = s_mt;
    rng.mti = (int)G.mt[624];
    __syncwarp();

    constexpr int EW = sizeof(rr_event) / 4, DW = sizeof(rr_decision) / 4;
    for (int base = 0; base < n_events; base += RT_CHUNK) {
        const int n = min(RT_CHUNK, n_events - base);
        warp_copy((uint32_t*)s_ev, (const uint32_t*)(events + base), n * EW);
        __syncwarp();
        run_trace<true, LAT>(S, rng, s_ev, n, s_dec);
        warp_copy((uint32_t*)(decisions + base), (const uint32_t*)s_dec, n * DW);
        __syncwarp();
    }

    warp_copy(G.window, (const long long*)window, nd); warp_copy(G.fail_window, (const long long*)failw, nd);
    warp_copy(G.cooldown_until, (const long long*)cool, nd); warp_copy(G.total_admitted, (const long long*)total, nd);
    warp_copy(G.req_count, (const int*)req, nd); warp_copy(G.tok_count, (const int*)tok, nd);
    warp_copy(G.fail_count, (const int*)failc, nd); warp_copy(G.inflight, (const int*)infl, nd);
    warp_copy(G.rr_next, (const int*)rrn, ng); warp_copy(G.burst_size, (const int*)bs, ng); warp_copy(G.burst_pos, (const int*)bp, ng);
    warp_copy(G.mt, (const uint32_t*)s_mt, 624);
    if (lat) {
        warp_copy(G.lat_n, (const int*)S.lat_n, nd); warp_copy(G.lat_head, (const double*)S.lat_head, nd);
        warp_copy(G.lat_last, (const double*)S.lat_last, nd); warp_copy(G.lat_stamp, (const long long*)S.lat_stamp, ng);
    }
    if (lane == 0) G.mt[624] = (uint32_t)rng.mti;
}

// ---------------------------------------------------------------- host side
static void mt_seed_like_cpython(uint64_t seed, uint32_t* mt /*625*/) {
    uint32_t key[2] = {(uint32_t)(seed & 0xffffffffu), (uint32_t)(seed >> 32)};
    const int klen = key[1] ? 2 : 1;
    mt[0] = 19650218u;
    for (int i = 1; i < 624; ++i) mt[i] = 1812433253u * (mt[i - 1] ^ (mt[i - 1] >> 30)) + (uint32_t)i;
    int i = 1, j = 0;
    for (int k = (624 > klen ? 624 : klen); k; --k) {
        mt[i] = (mt[i] ^ ((mt[i - 1] ^ (mt[i - 1] >> 30)) * 1664525u)) + key[j] + (uint32_t)j;
        ++i; ++j;
        if (i >= 624) { mt[0] = mt[623]; i = 1; }
        if (j >= klen) j = 0;
    }
    for (int k = 623; k; --k) {
        mt[i] = (mt[i] ^ ((mt[i - 1] ^ (mt[i - 1] >> 30)) * 1566083941u)) - (uint32_t)i;
        ++i;
        if (i >= 624) { mt[0] = mt[623]; i = 1; }
    }
    mt[0] = 0x80000000u;
    mt[624] = 624;
}

}  // namespace rr

using namespace rr;

struct rr_router {
    RouterDev dev;
    int device;
    int n_deps, n_groups;
    void* arena;            // one device allocation holding every array
    cudaStream_t stream;
    rr_event* h_events;     // pinned staging
    rr_decision* h_dec;
    rr_event* d_events;
    rr_decision* d_dec;
    int cap;
    int n_fb;               // fallback entries (layout of the shared-memory variant)
    int smem_bytes;         // > 0: router_kernel_smem is usable (state fits in one CTA's shared memory)
    cudaEvent_t last;       // completion of the latest launch: launches on one router are serialised across streams
    std::mutex mu;
    std::vector<int32_t> replica;   // per deployment: engine / GPU that serves it (rr_deployment_desc.replica)
};

#define CK(x)                                   \
    do {                                        \
        cudaError_t e__ = (x);                  \
        if (e__ != cudaSuccess) {               \
            rr::note_cuda_error(e__);           \
            return RR_CUDA_ERROR;               \
        }                                       \
    } while (0)

static int ensure_cap(rr_router* r, int n) {
    if (n <= r->cap) return RR_OK;
    int cap = r->cap ? r->cap : 1024;
    while (cap < n) cap *= 2;
    if (r->h_events) cudaFreeHost(r->h_events);
    if (r->h_dec) cudaFreeHost(r->h_dec);
    if (r->d_events) cudaFree(r->d_events);
    if (r->d_dec) cudaFree(r->d_dec);
    r->cap = 0;
    CK(cudaMallocHost(&r->h_events, sizeof(rr_event) * cap));
    CK(cudaMallocHost(&r->h_dec, sizeof(rr_decision) * cap));
    CK(cudaMalloc(&r->d_events, sizeof(rr_event) * cap));
    CK(cudaMalloc(&r->d_dec, sizeof(rr_decision) * cap));
    r->cap = cap;
    return RR_OK;
}

RR_API int rr_router_create(const rr_deployment_desc* deps, int n_deps, int n_groups,
                            const int32_t* fb_offsets, const int32_t* fb_groups,
                            const rr_router_settings* st, uint64_t seed, int device,
                            rr_router** out) {
    if (!deps || !st || !out || n_deps <= 0 || n_groups <= 0 || !fb_offsets) return RR_INVALID_ARGUMENT;
    if (st->strategy < 0 || st->strategy > RR_STRATEGY_LATENCY_BASED) return RR_INVALID_ARGUMENT;
    const int lat_cap = st->latency_list_size ? st->latency_list_size : 10;
    const int lat_ttl = st->latency_ttl_ms ? st->latency_ttl_ms : 3600000;
    if (lat_cap < 1 || lat_cap > 32 || st->latency_buffer_ppm < 0 || lat_ttl < 0) return RR_INVALID_ARGUMENT;
    const bool lat = st->strategy == RR_STRATEGY_LATENCY_BASED;
    std::vector<int32_t> goff(n_groups + 1, 0), gdeps(n_deps), dgrp(n_deps), rpm(n_deps), tpm(n_deps), wt(n_deps);
    for (int i = 0; i < n_deps; ++i) {
        if (deps[i].group < 0 || deps[i].group >= n_groups) return RR_INVALID_ARGUMENT;
        goff[deps[i].group + 1]++;
    }
    for (int g = 0; g < n_groups; ++g) {
        if (goff[g + 1] > 32) return RR_INVALID_ARGUMENT;   // one lane per candidate
        goff[g + 1] += goff[g];
    }
    {
        std::vector<int32_t> cur(goff.begin(), goff.end() - 1);
        for (int i = 0; i < n_deps; ++i) {
            gdeps[cur[deps[i].group]++] = i;
            dgrp[i] = deps[i].group; rpm[i] = deps[i].rpm; tpm[i] = deps[i].tpm; wt[i] = deps[i].weight;
        }
    }
    const int n_fb = fb_offsets[n_groups];
    for (int i = 0; i < n_fb; ++i)
        if (!fb_groups || fb_groups[i] < 0 || fb_groups[i] >= n_groups) return RR_INVALID_ARGUMENT;

    CK(cudaSetDevice(device));
    rr_router* r = new (std::nothrow) rr_router();
    if (!r) return RR_INTERNAL;
    memset(&r->dev, 0, sizeof(r->dev));
    r->device = device; r->n_deps = n_deps; r->n_groups = n_groups;
    for (int i = 0; i < n_deps; ++i) r->replica.push_back(deps[i].replica);
    r->h_events = nullptr; r->h_dec = nullptr; r->d_events = nullptr; r->d_dec = nullptr; r->cap = 0;

    // arena layout (8-byte aligned pieces first)
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 15) & ~size_t(15); return o; };
    size_t o_window = take(8 * n_deps), o_failw = take(8 * n_deps), o_cool = take(8 * n_deps),
           o_total = take(8 * n_deps);
    size_t o_req = take(4 * n_deps), o_tok = take(4 * n_deps), o_failc = take(4 * n_deps),
           o_infl = take(4 * n_deps), o_rr = take(4 * n_groups), o_bs = take(4 * n_groups), o_bp = take(4 * n_groups),
           o_mt = take(4 * 625);
    size_t o_goff = take(4 * (n_groups + 1)), o_gdeps = take(4 * n_deps),
           o_fboff = take(4 * (n_groups + 1)), o_fbg = take(4 * (n_fb > 0 ? n_fb : 1)),
           o_dgrp = take(4 * n_deps), o_rpm = take(4 * n_deps), o_tpm = take(4 * n_deps),
           o_wt = take(4 * n_deps);
    const int lat_d = lat ? n_deps : 0, lat_g = lat ? n_groups : 0;   // latency state: latency-based routers only
    size_t o_lat_n = take(4 * lat_d), o_lat_head = take(8 * lat_d), o_lat_last = take(8 * lat_d),
           o_lat_stamp = take(8 * lat_g);
    cudaError_t e = cudaMalloc(&r->arena, off);
    if (e != cudaSuccess) { rr::note_cuda_error(e); delete r; return RR_CUDA_ERROR; }
    char* base = (char*)r->arena;
    std::vector<char> host(off, 0);
    {
        long long* w = (long long*)(host.data() + o_window);
        long long* fw = (long long*)(host.data() + o_failw);
        for (int i = 0; i < n_deps; ++i) { w[i] = -1; fw[i] = -1; }
        long long* ls = (long long*)(host.data() + o_lat_stamp);
        for (int g = 0; g < lat_g; ++g) ls[g] = -1;
        mt_seed_like_cpython(seed, (uint32_t*)(host.data() + o_mt));
        memcpy(host.data() + o_goff, goff.data(), 4 * (n_groups + 1));
        memcpy(host.data() + o_gdeps, gdeps.data(), 4 * n_deps);
        memcpy(host.data() + o_fboff, fb_offsets, 4 * (n_groups + 1));
        if (n_fb > 0) memcpy(host.data() + o_fbg, fb_groups, 4 * n_fb);
        memcpy(host.data() + o_dgrp, dgrp.data(), 4 * n_deps);
        memcpy(host.data() + o_rpm, rpm.data(), 4 * n_deps);
        memcpy(host.data() + o_tpm, tpm.data(), 4 * n_deps);
        memcpy(host.data() + o_wt, wt.data(), 4 * n_deps);
    }
    e = cudaMemcpy(base, host.data(), off, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { rr::note_cuda_error(e); cudaFree(r->arena); delete r; return RR_CUDA_ERROR; }

    RouterDev& D = r->dev;
    D.n_deps = n_deps; D.n_groups = n_groups;
    D.strategy = st->strategy; D.pre_call = st->enable_pre_call_checks ? 1 : 0;
    D.allowed_fails = st->allowed_fails; D.cooldown_ms = st->cooldown_ms;
    D.group_off = (const int32_t*)(base + o_goff); D.group_deps = (const int32_t*)(base + o_gdeps);
    D.fb_off = (const int32_t*)(base + o_fboff); D.fb_groups = (const int32_t*)(base + o_fbg);
    D.dep_group = (const int32_t*)(base + o_dgrp);
    D.rpm = (const int32_t*)(base + o_rpm); D.tpm = (const int32_t*)(base + o_tpm);
    D.weight = (const int32_t*)(base + o_wt);
    D.window = (long long*)(base + o_window); D.req_count = (int*)(base + o_req);
    D.tok_count = (int*)(base + o_tok); D.fail_window = (long long*)(base + o_failw);
    D.fail_count = (int*)(base + o_failc); D.inflight = (int*)(base + o_infl);
    D.cooldown_until = (long long*)(base + o_cool); D.total_admitted = (long long*)(base + o_total);
    D.rr_next = (int*)(base + o_rr); D.mt = (uint32_t*)(base + o_mt);
    D.burst_size = (int*)(base + o_bs); D.burst_pos = (int*)(base + o_bp);
    D.lat_cap = lat_cap; D.lat_ttl_ms = lat_ttl;
    D.lat_buf = (double)st->latency_buffer_ppm / 1e6;
    if (lat) {
        D.lat_n = (int*)(base + o_lat_n); D.lat_head = (double*)(base + o_lat_head);
        D.lat_last = (double*)(base + o_lat_last); D.lat_stamp = (long long*)(base + o_lat_stamp);
    }

    e = cudaStreamCreateWithFlags(&r->stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) { rr::note_cuda_error(e); cudaFree(r->arena); delete r; return RR_CUDA_ERROR; }
    e = cudaEventCreateWithFlags(&r->last, cudaEventDisableTiming);
    if (e != cudaSuccess) { rr::note_cuda_error(e); cudaStreamDestroy(r->stream); cudaFree(r->arena); delete r; return RR_CUDA_ERROR; }
    r->n_fb = n_fb;
    r->smem_bytes = 0;
    {
        const RouterSmemLayout L = router_smem_layout(n_deps, n_groups, n_fb, lat);
        // The attribute is per function AND per device: raise it once per device to the cap every router may need (a later,
        // smaller router must not lower it under an earlier one); a launch then only states its own size.
        static std::atomic<uint64_t> attr_set{0}, attr_set_lat{0};
        if (L.total <= 200 * 1024 && !getenv("RR_ROUTER_GLOBAL_STATE") &&
            (lat ? rr::ensure_dyn_smem(router_kernel_smem<true>, 200 * 1024, attr_set_lat)
                 : rr::ensure_dyn_smem(router_kernel_smem<false>, 200 * 1024, attr_set)) == cudaSuccess)
            r->smem_bytes = (int)L.total;
    }
    int rc = ensure_cap(r, 1024);
    if (rc != RR_OK) { cudaStreamDestroy(r->stream); cudaFree(r->arena); delete r; return rc; }
    *out = r;
    return RR_OK;
}

namespace rr {
int router_shape(const rr_router* r, int* n_deployments, int* n_groups) {
    if (!r) return RR_INVALID_ARGUMENT;
    if (n_deployments) *n_deployments = r->n_deps;
    if (n_groups) *n_groups = r->n_groups;
    return RR_OK;
}
int router_dep_replica(const rr_router* r, int deployment) {
    return (r && deployment >= 0 && deployment < r->n_deps) ? r->replica[deployment] : -1;
}
int router_strategy(const rr_router* r) { return r ? r->dev.strategy : -1; }
}  // namespace rr

RR_API void rr_router_destroy(rr_router* r) {
    if (!r) return;
    cudaSetDevice(r->device);
    cudaStreamSynchronize(r->stream);
    if (r->h_events) cudaFreeHost(r->h_events);
    if (r->h_dec) cudaFreeHost(r->h_dec);
    if (r->d_events) cudaFree(r->d_events);
    if (r->d_dec) cudaFree(r->d_dec);
    cudaFree(r->arena);
    cudaEventDestroy(r->last);
    cudaStreamDestroy(r->stream);
    delete r;
}

RR_API int rr_router_process_device(rr_router* r, const rr_event* d_events, int n_events,
                                    rr_decision* d_decisions, void* stream) {
    if (!r || n_events < 0 || (n_events && (!d_events || !d_decisions))) return RR_INVALID_ARGUMENT;
    if (n_events == 0) return RR_OK;
    // one trace at a time per router: the RNG stream and (shared-memory variant) the staged state make launches
    // order-dependent, so a launch on any stream first waits for the previous one
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaStreamWaitEvent(st, r->last, 0);
    if (e != cudaSuccess) { rr::note_cuda_error(e); return RR_CUDA_ERROR; }
    const bool lat = r->dev.strategy == RR_STRATEGY_LATENCY_BASED;
    if (r->smem_bytes > 0 && lat)
        router_kernel_smem<true><<<1, 32, r->smem_bytes, st>>>(r->dev, r->n_fb, d_events, n_events, d_decisions);
    else if (r->smem_bytes > 0)
        router_kernel_smem<false><<<1, 32, r->smem_bytes, st>>>(r->dev, r->n_fb, d_events, n_events, d_decisions);
    else if (lat)
        router_kernel<true><<<1, 32, 0, st>>>(r->dev, d_events, n_events, d_decisions);
    else
        router_kernel<false><<<1, 32, 0, st>>>(r->dev, d_events, n_events, d_decisions);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaEventRecord(r->last, st);
    if (e != cudaSuccess) { rr::note_cuda_error(e); return RR_CUDA_ERROR; }
    return RR_OK;
}

RR_API int rr_router_process(rr_router* r, const rr_event* events, int n_events,
                             rr_decision* decisions) {
    if (!r || n_events < 0 || (n_events && (!events || !decisions))) return RR_INVALID_ARGUMENT;
    if (n_events == 0) return RR_OK;
    std::lock_guard<std::mutex> lk(r->mu);
    CK(cudaSetDevice(r->device));
    int rc = ensure_cap(r, n_events);
    if (rc != RR_OK) return rc;
    memcpy(r->h_events, events, sizeof(rr_event) * n_events);
    CK(cudaMemcpyAsync(r->d_events, r->h_events, sizeof(rr_event) * n_events, cudaMemcpyHostToDevice, r->stream));
    rc = rr_router_process_device(r, r->d_events, n_events, r->d_dec, r->stream);
    if (rc != RR_OK) return rc;
    CK(cudaMemcpyAsync(r->h_dec, r->d_dec, sizeof(rr_decision) * n_events, cudaMemcpyDeviceToHost, r->stream));
    CK(cudaStreamSynchronize(r->stream));
    memcpy(decisions, r->h_dec, sizeof(rr_decision) * n_events);
    return RR_OK;
}

RR_API int rr_router_snapshot(rr_router* r, rr_deployment_state* out) {
    if (!r || !out) return RR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> lk(r->mu);
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    const int n = r->n_deps;
    std::vector<long long> w(n), fw(n), cu(n), tot(n);
    std::vector<int> rq(n), tk(n), fc(n), inf(n);
    CK(cudaMemcpy(w.data(), r->dev.window, 8 * n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(fw.data(), r->dev.fail_window, 8 * n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(cu.data(), r->dev.cooldown_until, 8 * n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(tot.data(), r->dev.total_admitted, 8 * n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(rq.data(), r->dev.req_count, 4 * n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(tk.data(), r->dev.tok_count, 4 * n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(fc.data(), r->dev.fail_count, 4 * n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(inf.data(), r->dev.inflight, 4 * n, cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; ++i) {
        out[i].window = w[i]; out[i].req_count = rq[i]; out[i].tok_count = tk[i];
        out[i].fail_window = fw[i]; out[i].fail_count = fc[i]; out[i].inflight = inf[i];
        out[i].cooldown_until_ms = cu[i]; out[i].total_admitted = tot[i];
    }
    return RR_OK;
}

RR_API int rr_router_latency_snapshot(rr_router* r, double* mean_out, int32_t* n_samples_out) {
    if (!r || !mean_out || !n_samples_out) return RR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> lk(r->mu);
    const int n = r->n_deps;
    if (!r->dev.lat_n) {
        for (int i = 0; i < n; ++i) { mean_out[i] = 0.0; n_samples_out[i] = 0; }
        return RR_OK;
    }
    CK(cudaSetDevice(r->device));
    CK(cudaStreamSynchronize(r->stream));
    std::vector<int> cnt(n);
    std::vector<double> head(n), last(n);
    CK(cudaMemcpy(cnt.data(), r->dev.lat_n, 4 * n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(head.data(), r->dev.lat_head, 8 * n, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(last.data(), r->dev.lat_last, 8 * n, cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; ++i) {   // the kernel's mean: total / len, total = head (+ last once the list is full)
        const double tot = cnt[i] < r->dev.lat_cap ? head[i] : head[i] + last[i];
        mean_out[i] = cnt[i] > 0 ? tot / (double)cnt[i] : 0.0;
        n_samples_out[i] = cnt[i];
    }
    return RR_OK;
}

RR_API int rr_mt_seed_state(uint64_t seed, uint32_t* out625) {
    if (!out625) return RR_INVALID_ARGUMENT;
    mt_seed_like_cpython(seed, out625);
    return RR_OK;
}

RR_API int rr_router_seed(rr_router* r, uint64_t seed) {
    if (!r) return RR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> lk(r->mu);
    CK(cudaSetDevice(r->device));
    uint32_t mt[625];
    mt_seed_like_cpython(seed, mt);
    CK(cudaStreamSynchronize(r->stream));
    CK(cudaMemcpy(r->dev.mt, mt, sizeof(mt), cudaMemcpyHostToDevice));
    return RR_OK;
}
