// Device library shared by the fused kernels: symmetric-block accessors, block scan, grid-wide
// radix select (exact k-th largest magnitude) and the TMA chunk puller.
#pragma once
#include "common.cuh"
#include "oktopk.cuh"

namespace okt {

// ------------------------------------------------------------------------------------------
// symmetric-block accessors
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t* rs_mbox(char* b, const SymmLayout& L, int par, int src) {
    return reinterpret_cast<uint64_t*>(b + L.rs_mbox) + par * OKT_MAXP + src;
}
__device__ __forceinline__ float* rs_thr(char* b, const SymmLayout& L, int par, int src) {
    return reinterpret_cast<float*>(b + L.rs_thr) + par * OKT_MAXP + src;
}
__device__ __forceinline__ uint64_t* ag_mbox(char* b, const SymmLayout& L, int par, int src) {
    return reinterpret_cast<uint64_t*>(b + L.ag_mbox) + par * OKT_MAXP + src;
}
__device__ __forceinline__ uint64_t* cut_mbox(char* b, const SymmLayout& L, int par, int src) {
    return reinterpret_cast<uint64_t*>(b + L.cut_mbox) + par * OKT_MAXP + src;
}
__device__ __forceinline__ int* cut_data(char* b, const SymmLayout& L, int par, int src) {
    return reinterpret_cast<int*>(b + L.cut_data) + (par * OKT_MAXP + src) * OKT_MAXP;
}
__device__ __forceinline__ uint64_t* done_mbox(char* b, const SymmLayout& L, int par, int src) {
    return reinterpret_cast<uint64_t*>(b + L.done_mbox) + par * OKT_MAXP + src;
}
__device__ __forceinline__ uint64_t* tree_mbox(char* b, const SymmLayout& L, int par, int src) {
    return reinterpret_cast<uint64_t*>(b + L.tree_mbox) + par * OKT_MAXP + src;
}
// send slots: base of the (single-buffered) send buffer; destination d's slot starts at slot_off(d) entries
__device__ __forceinline__ int* send_idx_base(char* b, const SymmLayout& L) { return reinterpret_cast<int*>(b + L.send_idx); }
__device__ __forceinline__ float* send_val_base(char* b, const SymmLayout& L) { return reinterpret_cast<float*>(b + L.send_val); }
// lossless layout: the slot of region d starts at align4(edges[d]) + 4 d (16-byte aligned for TMA, capacity >= the
// region's length); bounded layout: d * cap
__device__ __forceinline__ int slot_off(const SymmLayout& L, const int* edges, int d) {
    return L.cap > 0 ? d * L.cap : ((edges[d] + 3) & ~3) + 4 * d;
}
__device__ __forceinline__ int* gat_idx(char* b, const SymmLayout& L, int par) {
    return reinterpret_cast<int*>(b + L.gat_idx) + (size_t)par * L.gcap;
}
__device__ __forceinline__ float* gat_val(char* b, const SymmLayout& L, int par) {
    return reinterpret_cast<float*>(b + L.gat_val) + (size_t)par * L.gcap;
}

// ------------------------------------------------------------------------------------------
// block-wide exclusive scan of one int per thread (kThreads threads); returns exclusive prefix,
// *total gets the block sum.  s_w: kWarps + 1 ints of shared scratch.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int block_excl_scan(int v, int* s_w, int* total) {
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    __syncthreads();
    if (lane == 31) s_w[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        int w = (lane < kWarps) ? s_w[lane] : 0;
        int winc = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, winc, o);
            if (lane >= o) winc += t;
        }
        if (lane < kWarps) s_w[lane] = winc - w;
        if (lane == kWarps - 1) s_w[kWarps] = winc;
    }
    __syncthreads();
    *total = s_w[kWarps];
    return s_w[warp] + inc - v;
}

// ------------------------------------------------------------------------------------------
// Exact k-th largest magnitude over a set of segments: 3-pass radix select (11+10+10 bits of the
// magnitude bit pattern), grid-wide.  The per-pass digit histogram is built in shared memory,
// merged into st->hist, and block 0 picks the digit; state travels in st->sel_prefix/sel_krem.
// ------------------------------------------------------------------------------------------
struct Seg { const float* ptr; int count; const int* idx; };   // idx != nullptr: the values are ptr[idx[i]]

__device__ __forceinline__ void digit_of_pass(int pass, int& shift, int& nbits) {
    shift = (pass == 0) ? 20 : (pass == 1 ? 10 : 0);
    nbits = (pass == 0) ? 11 : 10;
}

static __device__ void radix_pick_digit(OktState* st, int pass, uint32_t k_in, int* s_w) {
    // block 0 only; all kThreads threads
    int shift, nbits;
    digit_of_pass(pass, shift, nbits);
    const int bins = 1 << nbits;
    const int per = (bins + kThreads - 1) / kThreads;
    uint32_t prefix = (pass == 0) ? 0u : st->sel_prefix;
    uint32_t krem = (pass == 0) ? k_in : st->sel_krem;
    // thread t owns reversed bins [t*per, (t+1)*per)  (reversed: rb = bins-1-b, so ascending rb = descending magnitude)
    int mysum = 0;
    for (int j = 0; j < per; ++j) {
        int rb = threadIdx.x * per + j;
        if (rb < bins) mysum += (int)st->hist[bins - 1 - rb];
    }
    int total;
    int excl = block_excl_scan(mysum, s_w, &total);
    if (krem > (uint32_t)total) krem = (uint32_t)total;       // fewer candidates than k: take the smallest
    __shared__ uint32_t s_pick[2];
    if (threadIdx.x == 0) { s_pick[0] = 0; s_pick[1] = 0; }
    __syncthreads();
    if (total > 0) {
        int run = excl;
        for (int j = 0; j < per; ++j) {
            int rb = threadIdx.x * per + j;
            if (rb < bins) {
                int c = (int)st->hist[bins - 1 - rb];
                if ((uint32_t)run < krem && krem <= (uint32_t)(run + c)) {
                    s_pick[0] = (uint32_t)(bins - 1 - rb);
                    s_pick[1] = krem - (uint32_t)run;
                }
                run += c;
            }
        }
    }
    __syncthreads();
    for (int b = threadIdx.x; b < kHistBins; b += kThreads) st->hist[b] = 0;
    if (threadIdx.x == 0) {
        st->sel_prefix = (prefix << nbits) | s_pick[0];
        st->sel_krem = s_pick[1];
    }
    __syncthreads();
}

__device__ __forceinline__ void hist_add(uint32_t* s_hist, float v, int pass, uint32_t prefix) {
    uint32_t key = abs_bits(v);
    int shift, nbits;
    digit_of_pass(pass, shift, nbits);
    if (pass == 0 || (key >> (shift + nbits)) == prefix)
        atomicAdd(&s_hist[(key >> shift) & ((1u << nbits) - 1u)], 1u);
}

__device__ __forceinline__ void hist_flush(OktState* st, uint32_t* s_hist) {
    __syncthreads();
    for (int b = threadIdx.x; b < kHistBins; b += kThreads) {
        uint32_t c = s_hist[b];
        if (c) atomicAdd(&st->hist[b], c);
        s_hist[b] = 0;
    }
    __syncthreads();
}

// returns the bit pattern of the k-th largest |v| (0 if there are no candidates)
static __device__ float grid_kth_abs(const Seg* segs, int nseg, bool remote, uint32_t k, OktState* st,
                              uint32_t* s_hist, int* s_w, int first_pass) {
    const int gtid = blockIdx.x * blockDim.x + threadIdx.x;
    const int gthreads = gridDim.x * blockDim.x;
    for (int pass = 0; pass < 3; ++pass) {
        if (pass >= first_pass) {
            uint32_t prefix = (pass == 0) ? 0u : st->sel_prefix;
            for (int s = 0; s < nseg; ++s) {
                const float* ptr = segs[s].ptr;
                const int cnt = segs[s].count;
                const int* idx = segs[s].idx;
                for (int i = gtid; i < cnt; i += gthreads) {
                    const int j = idx ? __ldcg(idx + i) : i;
                    float v = remote ? ld_peer_f32(ptr + j) : __ldcg(ptr + j);
                    hist_add(s_hist, v, pass, prefix);
                }
            }
            hist_flush(st, s_hist);
        }
        grid_sync(&st->bar);
        if (blockIdx.x == 0) radix_pick_digit(st, pass, k, s_w);
        grid_sync(&st->bar);
    }
    return __uint_as_float(st->sel_prefix);
}

// ------------------------------------------------------------------------------------------
// over-selection ladder (see OktParams): shared-memory thresholds + per-rung tallies
// ------------------------------------------------------------------------------------------
struct LadderCfg { int n_fine, n_total; float f_fine, f_coarse; };

__device__ __forceinline__ LadderCfg ladder_cfg(const OktParams& p, bool on) {
    LadderCfg c;
    c.n_fine = on ? min(p.guard_loops, kGuardFineMax) : 0;
    const int coarse = (on && p.cap_limit > 0) ? min(p.cap_rungs, kGuardMax - 1 - c.n_fine) : 0;
    c.n_total = 1 + c.n_fine + coarse;           // rungs 0 .. n_total-1
    c.f_fine = p.guard_factor;
    c.f_coarse = p.cap_factor;
    return c;
}
// thread 0 fills thr[0..n_total) (plain fp32 multiplications: the oracle reproduces them bit for bit), all zero tallies
__device__ __forceinline__ void ladder_build(float* s_thr, int* s_cnt, const LadderCfg& c, float thr0) {
    if (threadIdx.x == 0) {
        float t = thr0;
        s_thr[0] = t;
        for (int j = 1; j < c.n_total; ++j) { t *= (j <= c.n_fine) ? c.f_fine : c.f_coarse; s_thr[j] = t; }
    }
    for (int j = threadIdx.x; j < kGuardMax; j += blockDim.x) s_cnt[j] = 0;
    __syncthreads();
}
// highest rung j with ax > T_j (ax > T_0 is given)
__device__ __forceinline__ int ladder_rung(const float* s_thr, int n_total, float ax) {
    int lo = 0, hi = n_total - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (ax > s_thr[mid]) lo = mid; else hi = mid - 1;
    }
    return lo;
}
__device__ __forceinline__ void ladder_flush(OktState* st, int* s_cnt) {
    __syncthreads();
    if (threadIdx.x < kGuardMax) {
        const int c = s_cnt[threadIdx.x];
        if (c) atomicAdd(&st->guard_counts[threadIdx.x], c);
    }
    __syncthreads();
}
// one thread: choose the rung from the global tallies; returns the threshold, *count = #(|acc| > threshold);
// zeroes the tallies for the next call
__device__ __forceinline__ float ladder_pick(OktState* st, const LadderCfg& c, float thr0, int guard_limit, int cap_limit,
                                             int* count) {
    int suffix[kGuardMax];
    int run = 0;
    for (int j = kGuardMax - 1; j >= 0; --j) { run += __ldcg(&st->guard_counts[j]); suffix[j] = run; }
    int j = 0;
    float t = thr0;
    while (j < c.n_fine && suffix[j] > guard_limit) { ++j; t *= c.f_fine; }
    if (cap_limit > 0)
        while (j < c.n_total - 1 && suffix[j] > cap_limit) { ++j; t *= (j <= c.n_fine) ? c.f_fine : c.f_coarse; }
    *count = suffix[j];
    for (int q = 0; q < kGuardMax; ++q) st->guard_counts[q] = 0;
    return t;
}

// ------------------------------------------------------------------------------------------
// TMA-fed streaming read: the CTA walks its share of `nvec` float4 (tiles of kTileV float4 dealt round-robin to
// CTAs) through a STAGES-deep shared-memory ring.  One elected thread arms a stage's mbarrier and issues the
// cp.async.bulk load STAGES-1 tiles ahead; all threads consume the landed tile from shared memory through
// body(tile_smem, first_vec_of_tile).  `bars` must be STAGES freshly initialised mbarriers used by nobody else.
// ------------------------------------------------------------------------------------------
constexpr int kTileV = kPackTile * kThreads;      // float4 per tile

template <int STAGES, class Body>
__device__ __forceinline__ void tma_stream_tiles(const float4* src, int nvec, float4* ring, uint64_t* bars, Body&& body) {
    const int ntiles = (nvec + kTileV - 1) / kTileV;
    const int G = gridDim.x;
    const int nmine = (ntiles > (int)blockIdx.x) ? (ntiles - (int)blockIdx.x + G - 1) / G : 0;
    auto arm = [&](int j) {                       // thread 0 only
        const int tile = blockIdx.x + j * G;
        const int stg = j % STAGES;
        const uint32_t bytes = (uint32_t)min(kTileV, nvec - tile * kTileV) * 16u;
        fence_proxy_async_all();
        mbar_expect_tx(&bars[stg], bytes);
        tma_load_1d(ring + stg * kTileV, src + (size_t)tile * kTileV, bytes, &bars[stg]);
    };
    if (threadIdx.x == 0)
        for (int j = 0; j < min(nmine, STAGES - 1); ++j) arm(j);
    for (int j = 0; j < nmine; ++j) {
        __syncthreads();                          // the stage consumed last iteration is drained: re-arm it
        if (threadIdx.x == 0 && j + STAGES - 1 < nmine) arm(j + STAGES - 1);
        const int stg = j % STAGES;
        mbar_wait(&bars[stg], (uint32_t)(j / STAGES) & 1u);
        body(ring + stg * kTileV, (blockIdx.x + j * G) * kTileV);
    }
    __syncthreads();
}

// ------------------------------------------------------------------------------------------
// chunk puller: double-buffered TMA bulk copies of (idx,val) chunks from (possibly remote) slots
// ------------------------------------------------------------------------------------------
struct PullSmem {
    int idx[2][kChunk];
    float val[2][kChunk];
    uint64_t bar[2];
};

struct ChunkSrc { const int* idx; const float* val; int count; };

// Calls fn(src_index, entry_idx, entry_val) for every valid entry of the chunks this CTA owns.
// The chunk list is the concatenation over sources (in the order given) of ceil(count/kChunk) chunks,
// dealt round-robin to CTAs.  pipe_it carries the mbarrier phase across calls.
template <class F>
__device__ __forceinline__ void pull_chunks(const ChunkSrc* srcs, int nsrc, bool use_tma, PullSmem* sm,
                                            uint32_t& pipe_it, F&& fn) {
    int total = 0;
    for (int s = 0; s < nsrc; ++s) total += (srcs[s].count + kChunk - 1) / kChunk;
    const int G = gridDim.x, c0 = blockIdx.x;
    const int nmine = (total > c0) ? (total - c0 + G - 1) / G : 0;
    if (nmine == 0) return;

    auto locate = [&](int cid, int& s, int& off) {
        int acc = 0;
        for (s = 0; s < nsrc; ++s) {
            int nc = (srcs[s].count + kChunk - 1) / kChunk;
            if (cid < acc + nc) { off = (cid - acc) * kChunk; return; }
            acc += nc;
        }
        s = nsrc - 1; off = 0;
    };

    if (use_tma) {
        auto issue = [&](int j) {
            int s, off;
            locate(c0 + j * G, s, off);
            uint32_t it = pipe_it + j;
            int stg = it & 1;
            fence_proxy_async_all();
            mbar_expect_tx(&sm->bar[stg], 2u * kChunk * 4u);
            tma_load_1d(sm->idx[stg], srcs[s].idx + off, kChunk * 4u, &sm->bar[stg]);
            tma_load_1d(sm->val[stg], srcs[s].val + off, kChunk * 4u, &sm->bar[stg]);
        };
        if (threadIdx.x == 0) issue(0);
        for (int j = 0; j < nmine; ++j) {
            if (threadIdx.x == 0 && j + 1 < nmine) issue(j + 1);
            uint32_t it = pipe_it + j;
            int stg = it & 1;
            mbar_wait(&sm->bar[stg], (it >> 1) & 1u);
            int s, off;
            locate(c0 + j * G, s, off);
            const int valid = min(kChunk, srcs[s].count - off);
            for (int e = threadIdx.x; e < valid; e += kThreads) fn(s, sm->idx[stg][e], sm->val[stg][e]);
            __syncthreads();
        }
        pipe_it += nmine;
    } else {
        for (int j = 0; j < nmine; ++j) {
            int s, off;
            locate(c0 + j * G, s, off);
            const int valid = min(kChunk, srcs[s].count - off);
            for (int e = threadIdx.x; e < valid; e += kThreads)
                fn(s, ld_peer_s32(srcs[s].idx + off + e), ld_peer_f32(srcs[s].val + off + e));
        }
    }
}

// ------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al., SC'11, with Random123's constants and round order): four 32-bit words from a 128-bit
// counter and a 64-bit key.  Counter 0 and key 0 give 6627e8d5 e169c58d bc57ac4c 9b00dbd8.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r > 0) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    }
    return c;
}

// ------------------------------------------------------------------------------------------
// Dropout keep bits of the fused LayerNorm and embedding kernels: flat element i is kept iff word i % 4 of
// Philox4x32-10(counter (i/4 low, i/4 high, 0, 0), key (seed low, seed high)) is below keep_thr = floor((1-p) 2^32);
// keep_thr >= 2^32 (p = 0) keeps everything and never reads the seed.
// ------------------------------------------------------------------------------------------
constexpr long long kLnKeepAll = 1LL << 32;

struct LnDrop {
    bool on;
    uint32_t thr, k0, k1;
    float s;
};

__device__ __forceinline__ LnDrop ln_drop(const unsigned long long* seed, long long keep_thr, float scale) {
    LnDrop d;
    d.on = keep_thr < kLnKeepAll;
    d.thr = (uint32_t)keep_thr;
    const unsigned long long k = d.on ? __ldg(seed) : 0ull;
    d.k0 = (uint32_t)k;
    d.k1 = (uint32_t)(k >> 32);
    d.s = scale;
    return d;
}

// The keep bits of the four elements from flat index i (i % 4 == 0), element k in bit k.
__device__ __forceinline__ uint32_t ln_keep(const LnDrop& d, unsigned long long i) {
    if (!d.on) return 0xfu;
    const unsigned long long q = i >> 2;
    const uint4 r = philox4x32_10(make_uint4((uint32_t)q, (uint32_t)(q >> 32), 0u, 0u), d.k0, d.k1);
    return (uint32_t)(r.x < d.thr) | ((uint32_t)(r.y < d.thr) << 1) | ((uint32_t)(r.z < d.thr) << 2) |
           ((uint32_t)(r.w < d.thr) << 3);
}

// The multiplier at those four elements: s where kept, 0 where dropped.
__device__ __forceinline__ float4 ln_mult(const LnDrop& d, uint32_t keep) {
    return make_float4((keep & 1u) ? d.s : 0.f, (keep & 2u) ? d.s : 0.f, (keep & 4u) ? d.s : 0.f, (keep & 8u) ? d.s : 0.f);
}

}  // namespace okt
