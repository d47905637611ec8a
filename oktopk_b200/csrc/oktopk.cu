// The fused Ok-Topk sparse allreduce: ONE persistent cooperative kernel per bucket per step.
//
//   error-feedback accumulate -> threshold select -> pack per destination region
//   -> publish counts to the region owners (st.release.sys into their mailboxes over NVLink)
//   -> pull every source's (idx,val) chunks for my region with TMA bulk copies (cp.async.bulk,
//      global(peer) -> shared, mbarrier completion) and scatter-add (red.global.add.f32)
//   -> global selection on my region, pack my allgather slot, publish
//   -> pull all slots, write result/P in place, clear residual where locally selected AND
//      globally kept, adapt both thresholds on the device.
//
// No NCCL, no host round trip, no host-visible counts.  Behavioural spec: SURVEY 3.3
// (reference: VGG/allreducer.py:575-1098, BERT/bert/allreducer.py:357-743,
// VGG/compression.py:370-415,467-471) -- the data flow here is a redesign, not a translation:
// the reference sizes every receive buffer from host Alltoall/Allgather handshakes and stages
// all payloads through NumPy; here slots are peer-visible buffers whose capacity covers the whole
// destination region (lossless layout, oktopk.cuh) or, in the bounded layout, are protected by an
// in-kernel overflow policy (raise the threshold, redo the pack pass: nothing selected is ever
// lost), counts travel as release/acquire flags, and the over-selection guard is applied
// receiver-side so that the common iteration is a single streaming pass (12 B/element when the gradient is read from
// autograd's tensors, 16 B/element when it was landed in the bucket; see OktParams::src).
// Grid-wide synchronisation: ONE grid barrier per call (reduce -> global selection); "everybody
// finished packing / selecting" is a last-CTA ticket whose winner publishes the counts, and the
// rank's own mailbox doubles as the local barrier of the next phase.
#include "devlib.cuh"

namespace okt {

// ------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int region_of(const int* s_edges, int P, int i) {
    int d = 0;
#pragma unroll 1
    for (int r = 1; r < P; ++r) d += (i >= s_edges[r]) ? 1 : 0;
    return d;
}

// ---- gradient sources (OktParams::src*): a shared-memory copy of the segment table -----------------------------
struct SrcSeg { const float* src; int off, len; };

// last segment that starts at or before element e (-1: none)
__device__ __forceinline__ int seg_find(const SrcSeg* s, int ns, int e) {
    int lo = 0, hi = ns - 1, r = -1;
    while (lo <= hi) {
        const int mid = (lo + hi) >> 1;
        if (s[mid].off <= e) { r = mid; lo = mid + 1; } else { hi = mid - 1; }
    }
    return r;
}

__device__ __forceinline__ float grad_at(const SrcSeg* s, int ns, int i) {
    const int q = seg_find(s, ns, i);
    return (q >= 0 && i - s[q].off < s[q].len) ? s[q].src[i - s[q].off] : 0.f;
}

// elements 4v .. 4v+3 of the gradient (plain loads: the exact-threshold pass runs once per recompute interval)
__device__ __forceinline__ float4 grad4_at(const SrcSeg* s, int ns, int v) {
    float4 out = make_float4(0.f, 0.f, 0.f, 0.f);
    const int q = seg_find(s, ns, 4 * v);
    if (q < 0) return out;
    const int r = 4 * v - s[q].off, len = s[q].len;
    const float* src = s[q].src + r;
    if (r + 4 <= len) return ld_stream_f4(reinterpret_cast<const float4*>(src));
    if (r < len) out.x = src[0];
    if (r + 1 < len) out.y = src[1];
    if (r + 2 < len) out.z = src[2];
    return out;
}

// shared-memory copy of the gradient-source table and the list of its partial last vectors (length % 4 != 0), which the
// streaming pass patches from global memory.  Ends with a block barrier.
__device__ __forceinline__ void load_src_table(const OktParams& p, SrcSeg* s_src, int* s_tail_v, int* s_tail_q, int* s_ntail) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nsrc = p.nsrc, n4 = p.n >> 2;
    for (int q = tid; q < nsrc; q += blockDim.x) s_src[q] = SrcSeg{p.src[q], p.src_off[q], p.src_len[q]};
    if (warp == 0) {
        int cnt = 0;
        for (int q0 = 0; q0 < nsrc; q0 += 32) {
            const int q = q0 + lane;
            const int end = q < nsrc ? p.src_off[q] + p.src_len[q] : 0;
            const bool part = q < nsrc && (end & 3) != 0 && (end >> 2) < n4;
            const unsigned m = __ballot_sync(0xffffffffu, part);
            if (part) { const int t = cnt + __popc(m & ((1u << lane) - 1u)); s_tail_v[t] = end >> 2; s_tail_q[t] = q; }
            cnt += __popc(m);
        }
        if (lane == 0) *s_ntail = cnt;
    }
    __syncthreads();
}

// The tiles of the streaming pass: float4 ranges [lo[r], hi[r]) cut into tiles of kTileV vectors from each range's start;
// range r holds tiles first[r] .. first[r + 1] - 1.  One range [0, n4) is the whole bucket.
struct TileMap { const int* lo; const int* hi; const int* first; int nr; };

// thread 0: ranges -> tile prefix (shared arrays of kPackRangeMax / kPackRangeMax + 1 entries); ends with a block barrier
__device__ __forceinline__ TileMap tile_map_build(int nr, const int* lo_in, const int* hi_in, int* lo, int* hi, int* first) {
    if (threadIdx.x == 0) {
        int t = 0;
        for (int r = 0; r < nr; ++r) {
            lo[r] = lo_in[r]; hi[r] = hi_in[r]; first[r] = t;
            t += (hi[r] - lo[r] + kTileV - 1) / kTileV;
        }
        first[nr] = t;
    }
    __syncthreads();
    return TileMap{lo, hi, first, nr};
}

// first vector and end of tile t
__device__ __forceinline__ void tile_at(const TileMap& m, int t, int* base, int* end) {
    int r = 0;
    while (t >= m.first[r + 1]) ++r;
    *base = m.lo[r] + (t - m.first[r]) * kTileV;
    *end = min(*base + kTileV, m.hi[r]);
}

struct PackRing { float4* r; float4* g; uint64_t* full; uint64_t* empty; };   // [STAGES][kTileV] each; STAGES barriers each
struct PackSrc { const SrcSeg* seg; int nseg; const int* tail_v; const int* tail_q; int ntail; };
struct PackSel {                  // selection: threshold, ladder, region edges, send-slot offsets and buffers
    float thr; LadderCfg lc; const float* lthr; int* lcnt;
    const int* edges; const int* soff; int* sidx; float* sval; int P;
};

// The streaming pack pass over this CTA's tiles of `tm` (tile = blockIdx.x + j * gridDim.x): acc = g + residual ->
// residual (the gradient assembled from the source segments), |acc| > thr appended to the destination's send slot
// through st->send_cursor, ladder tallies into sel.lcnt.  res_only: the accumulator is already in the residual buffer.
// clear_g: write zeros over the bucket (the gradient was landed there).  ring_it counts the tiles ever pushed through the
// ring (its mbarrier phases run on across calls of the same CTA).  Returns the number of tiles this CTA consumed.
//
// Fed by TMA: the CTA walks its tiles (kPackTile x 512 float4 = 16 KB of the gradient + 16 KB of the residual each)
// through a STAGES-deep shared-memory ring.  One elected thread arms the stage's mbarrier (expect_tx) and issues the bulk
// loads STAGES-1 tiles ahead, so the reads in flight per SM do not depend on occupancy or the register budget; consumers
// read the tile with conflict-free LDS.128, write the accumulator (and, when the gradient was landed in the bucket, zeros
// over it) back with streaming 128-bit stores (posted), and run the selection.  HBM traffic: 12 B/element when the
// gradient is read from autograd's tensors (gradient + residual in, residual out), 16 B/element when it was landed (+ the
// bucket cleared).  The gradient half of a tile is assembled from the source segments that overlap it, one bulk copy per
// piece; what no segment covers (padding, parameters without a gradient, the last 1-3 elements of a segment whose length
// is not a multiple of 4) is copied from the bucket, which is all-zero in that mode, and the partial last vector of a
// segment is patched by the consumer from global memory (never read past a source's end).
template <int STAGES>
__device__ __forceinline__ int pack_stream(const OktParams& p, const TileMap& tm, const PackRing& ring, int ring_it,
                                           bool res_only, bool clear_g, const PackSrc& src, const PackSel& sel,
                                           int& dropped) {
    OktState* st = p.st;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = p.n;
    float4* g4 = reinterpret_cast<float4*>(p.g);
    float4* r4 = reinterpret_cast<float4*>(p.res);
    const int ntiles = tm.first[tm.nr];
    const int G = gridDim.x;
    const int nmine = (ntiles > (int)blockIdx.x) ? (ntiles - (int)blockIdx.x + G - 1) / G : 0;
    const SrcSeg* s_src = src.seg;
    const int nsrc = src.nseg;
    const float thr_sel = sel.thr;
    const LadderCfg& lc = sel.lc;

    auto arm = [&](int j) {                                         // thread 0 only; j = tile number of THIS pass
        int base, end;
        tile_at(tm, blockIdx.x + j * G, &base, &end);
        const int stg = (ring_it + j) % STAGES;
        const uint32_t bytes = (uint32_t)(end - base) * 16u;
        fence_proxy_async_all();
        mbar_expect_tx(&ring.full[stg], res_only ? bytes : 2u * bytes);
        tma_load_1d(ring.r + stg * kTileV, r4 + (size_t)base, bytes, &ring.full[stg]);
        if (res_only) return;
        float4* dst = ring.g + stg * kTileV;
        const int e0 = base * 4, e1 = e0 + (int)(bytes >> 2);
        // first segment whose whole vectors reach past e0
        int lo = 0, hi = nsrc;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (s_src[mid].off + (s_src[mid].len & ~3) <= e0) lo = mid + 1; else hi = mid;
        }
        int q = lo, e = e0;
        while (e < e1) {
            if (q < nsrc && s_src[q].off <= e) {                    // inside segment q
                const int stop = min(e1, s_src[q].off + (s_src[q].len & ~3));
                if (stop > e) {
                    tma_load_1d(dst + ((e - e0) >> 2), s_src[q].src + (e - s_src[q].off), (uint32_t)(stop - e) * 4u,
                                &ring.full[stg]);
                    e = stop;
                }
                ++q;
            } else {                                                // not covered: zeros from the bucket
                const int stop = q < nsrc ? min(e1, s_src[q].off) : e1;
                tma_load_1d(dst + ((e - e0) >> 2), p.g + e, (uint32_t)(stop - e) * 4u, &ring.full[stg]);
                e = stop;
            }
        }
    };
    if (tid == 0)
        for (int j = 0; j < min(nmine, STAGES - 1); ++j) {
            // a stage used by the previous pass must have been released by all warps before it is re-armed
            const int q = ring_it + j;
            if (q >= STAGES) mbar_wait(&ring.empty[q % STAGES], (uint32_t)(q / STAGES - 1) & 1u);
            arm(j);
        }
    for (int j = 0; j < nmine; ++j) {
        // Producer (thread 0): re-arm the stage tile j-1 used, once all kWarps warps have released it (per-stage
        // "empty" mbarrier; no block-wide barrier per tile, so a warp waiting for its slot reservation does not
        // hold up the other 15 -- they may run up to STAGES-1 tiles ahead).
        if (tid == 0 && j + STAGES - 1 < nmine) {
            const int q = ring_it + j + STAGES - 1;                 // ring slot sequence number being armed
            if (q >= STAGES) mbar_wait(&ring.empty[q % STAGES], (uint32_t)(q / STAGES - 1) & 1u);
            arm(j + STAGES - 1);
        }
        const int qj = ring_it + j;
        const int stg = qj % STAGES;
        mbar_wait(&ring.full[stg], (uint32_t)(qj / STAGES) & 1u);
        int base, tend;
        tile_at(tm, blockIdx.x + j * G, &base, &tend);
        float4 a[kPackTile];
        bool in[kPackTile];
#pragma unroll
        for (int u = 0; u < kPackTile; ++u) {
            const int v = base + u * kThreads + tid;
            in[u] = v < tend;
            a[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (in[u]) {
                a[u] = ring.r[stg * kTileV + u * kThreads + tid];
                if (!res_only) {
                    float4 gq = ring.g[stg * kTileV + u * kThreads + tid];
                    for (int t = 0; t < src.ntail; ++t)
                        if (src.tail_v[t] == v) {                   // a segment ends inside this vector
                            const SrcSeg sg = s_src[src.tail_q[t]];
                            const float* sp = sg.src + (sg.len & ~3);
                            const int c = sg.len & 3;
                            gq.x = sp[0];
                            if (c > 1) gq.y = sp[1];
                            if (c > 2) gq.z = sp[2];
                        }
                    a[u].x += gq.x; a[u].y += gq.y; a[u].z += gq.z; a[u].w += gq.w;
                    st_stream_f4(r4 + v, a[u]);
                }
                if (clear_g) st_stream_f4(g4 + v, make_float4(0.f, 0.f, 0.f, 0.f));
            }
        }
        __syncwarp();                                               // the warp's part of the tile is in registers:
        if (lane == 0) mbar_arrive(&ring.empty[stg]);               // release the stage (1 of kWarps arrivals)
        // ---- selection: one slot reservation per (warp, trip, destination) ------------------------------
        // 16 element flags per lane -> 16 ballots; the warp's trip covers 4 windows of 128 consecutive elements,
        // which (regions being contiguous ranges) almost always belong to ONE destination, so the append costs
        // one global atomic per trip instead of one per selected vector component.
        unsigned msk[kPackTile * 4];
        unsigned mybits = 0u;
        int tot = 0;
#pragma unroll
        for (int u = 0; u < kPackTile; ++u) {
            const float xs[4] = {a[u].x, a[u].y, a[u].z, a[u].w};
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const bool pred = in[u] && fabsf(xs[c]) > thr_sel;
                // TopkDSA zeroes the residual at the exact top-k INCLUDING the k-th element itself, which the
                // strict '>' select does not send (reference quirk, SURVEY B.4-3).  On a tie at the k-th
                // magnitude the top-k holds only k - #(|x| > thr) of the tied elements -- the radix select's
                // remaining rank, sel_krem -- so a ticket bounds the clears to that many (which ones is unspecified)
                if (p.residual_mode == RES_LOCAL_GE && in[u] && xs[c] != 0.f && fabsf(xs[c]) == thr_sel &&
                    atomicAdd(&st->tie_cursor, 1) < (int)__ldcg(&st->sel_krem))
                    p.res[4 * (base + u * kThreads + tid) + c] = 0.f;
                const unsigned m = __ballot_sync(0xffffffffu, pred);
                msk[u * 4 + c] = m;
                tot += __popc(m);
                if (pred) mybits |= 1u << (u * 4 + c);
            }
        }
        if (tot == 0) continue;
        // ladder tallies of my selected elements (shared-memory atomics: only selected elements get here)
        if (lc.n_total > 1) {
#pragma unroll
            for (int u = 0; u < kPackTile; ++u) {
                const float xs[4] = {a[u].x, a[u].y, a[u].z, a[u].w};
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    if (mybits & (1u << (u * 4 + c)))
                        atomicAdd(&sel.lcnt[ladder_rung(sel.lthr, lc.n_total, fabsf(xs[c]))], 1);
            }
        } else if (lane == 0) {
            atomicAdd(&sel.lcnt[0], tot);                          // one rung: the warp's count in one go
        }
        const int e_first = 4 * (base + (warp << 5));
        const int e_last = min(n - 1, 4 * (base + (kPackTile - 1) * kThreads + (warp << 5) + 31) + 3);
        const int dlo = region_of(sel.edges, sel.P, e_first), dhi = region_of(sel.edges, sel.P, e_last);
        for (int d = dlo; d <= dhi; ++d) {
            unsigned md[kPackTile * 4];
            unsigned mine = mybits;
            int cnt = 0;
            if (dlo == dhi) {
#pragma unroll
                for (int q = 0; q < kPackTile * 4; ++q) { md[q] = msk[q]; cnt += __popc(md[q]); }
            } else {
                const int lo_d = sel.edges[d], hi_d = sel.edges[d + 1];
                mine = 0u;
#pragma unroll
                for (int u = 0; u < kPackTile; ++u) {
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const int i = 4 * (base + u * kThreads + tid) + c;
                        const bool pd = ((mybits >> (u * 4 + c)) & 1u) && i >= lo_d && i < hi_d;
                        md[u * 4 + c] = __ballot_sync(0xffffffffu, pd);
                        cnt += __popc(md[u * 4 + c]);
                        if (pd) mine |= 1u << (u * 4 + c);
                    }
                }
            }
            if (cnt == 0) continue;
            int run = 0;
            if (lane == 0) run = atomicAdd(&st->send_cursor[d], cnt);
            run = __shfl_sync(0xffffffffu, run, 0);
            const int scap_d = sel.soff[d + 1] - sel.soff[d];
            int* sidx = sel.sidx + sel.soff[d];
            float* sval = sel.sval + sel.soff[d];
            const int off_d = sel.edges[d];
            const unsigned lt = (1u << lane) - 1u;
#pragma unroll
            for (int u = 0; u < kPackTile; ++u) {
                const float xs[4] = {a[u].x, a[u].y, a[u].z, a[u].w};
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const int q = u * 4 + c;
                    if ((mine >> q) & 1u) {
                        const int pos = run + __popc(md[q] & lt);
                        const int i = 4 * (base + u * kThreads + tid) + c;
                        if (pos < scap_d) {
                            sidx[pos] = i - off_d;
                            sval[pos] = xs[c];
                            if (p.residual_mode != RES_OKTOPK) p.res[i] = 0.f;   // sent => cleared (classic rule)
                        } else {
                            dropped++;                                           // stays in the residual
                        }
                    }
                    run += __popc(md[q]);
                }
            }
        }
    }
    return nmine;
}

__global__ void __launch_bounds__(kThreads, kCtasPerSm) oktopk_fused_kernel(const OktParams p) {
    __shared__ uint32_t s_hist[kHistBins];
    __shared__ int s_w[kWarps + 1];
    __shared__ int s_edges[OKT_MAXP + 1];
    __shared__ int s_cnt[OKT_MAXP];
    __shared__ float s_thr[OKT_MAXP];
    __shared__ int s_misc[OKT_MAXP * 2 + 4];
    __shared__ int s_soff[OKT_MAXP + 1];            // send-slot offsets (entries) per destination, see slot_off()
    __shared__ float s_lthr[kGuardMax];             // over-selection ladder: thresholds ...
    __shared__ int s_lcnt[kGuardMax];               // ... and this CTA's per-rung tallies
    __shared__ ChunkSrc s_srcs[OKT_MAXP];
    __shared__ float s_sthr[OKT_MAXP];
    __shared__ Seg s_segs[OKT_MAXP];
    __shared__ __align__(128) PullSmem s_pull;
    __shared__ __align__(8) uint64_t s_pk_bar[kPackStages];
    __shared__ __align__(8) uint64_t s_pk_empty[kPackStages];
    __shared__ __align__(8) uint64_t s_sc_bar[kScanStages];
    __shared__ SrcSeg s_src[kSrcSegMax];                    // gradient-source table
    __shared__ int s_tail_v[kSrcSegMax], s_tail_q[kSrcSegMax];   // vectors where a segment ends mid-way (length % 4 != 0)
    __shared__ int s_ntail;
    __shared__ int s_rlo[kPackRangeMax], s_rhi[kPackRangeMax], s_rfirst[kPackRangeMax + 1];   // tiles of the pack pass
    extern __shared__ __align__(128) float4 dyn_pk[];       // TMA ring of the streaming pass (kPackSmemBytes)

    if (verdict_set(p.skip)) return;
    OktState* st = p.st;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int gtid = blockIdx.x * kThreads + tid;
    const int gthreads = gridDim.x * kThreads;
    const int P = p.P, rank = p.rank, n = p.n;
    char* me = p.peers[rank];
    const uint32_t epoch = st->epoch + 1u;     // every CTA reads it before anybody can bump it (see PH_FINAL)
    const int par = epoch & 1u;
    // Carried threshold: every CTA reads it before the pack publisher can rewrite it.  A threshold-reuse call that finds
    // it at 0 (the last exact call saw fewer than k non-zeros) recomputes the exact threshold: at 0 every non-zero would
    // be selected and no ladder rung (0 * f = 0) could cap the volume.  Decided here, not on the host, so that a
    // captured graph stays valid whatever the threshold.
    const float thr_in = st->local_thr;
    const bool exact_local = p.exact_local || thr_in == 0.f;
    const bool two_pass = exact_local || p.repartition;
    uint32_t pipe_it = 0;

    for (int b = tid; b < kHistBins; b += kThreads) s_hist[b] = 0;
    if (blockIdx.x == 0 && tid == 0) st->t_phase[5] = globaltimer_ns();
    const SpinGuard sg_rs{&st->fault, p.timeout_ns, FAULT_RS_TIMEOUT, p.host_fault};
    const SpinGuard sg_ag{&st->fault, p.timeout_ns, FAULT_AG_TIMEOUT, p.host_fault};
    const SpinGuard sg_cut{&st->fault, p.timeout_ns, FAULT_CUT_TIMEOUT, p.host_fault};
    const SpinGuard sg_done{&st->fault, p.timeout_ns, FAULT_DONE_TIMEOUT, p.host_fault};
    if (tid == 0) {
        mbar_init(&s_pull.bar[0], 1);
        mbar_init(&s_pull.bar[1], 1);
        for (int q = 0; q < kPackStages; ++q) { mbar_init(&s_pk_bar[q], 1); mbar_init(&s_pk_empty[q], kWarps); }
        for (int q = 0; q < kScanStages; ++q) mbar_init(&s_sc_bar[q], 1);
        mbar_fence_init();
    }
    const int n4 = n >> 2;
    const int nsrc = p.nsrc;
    load_src_table(p, s_src, s_tail_v, s_tail_q, &s_ntail);
    const int ntail = s_ntail;
    // what the pack pass streams: the whole bucket, or (a threshold-reuse call after segment launches) what they left
    const int whole[2] = {0, n4};
    const bool ranged = p.pk_mode && !two_pass;
    const TileMap tmap = tile_map_build(ranged ? p.pk_nr : 1, ranged ? p.pk_lo : whole, ranged ? p.pk_hi : whole + 1,
                                        s_rlo, s_rhi, s_rfirst);

    float4* r4 = reinterpret_cast<float4*>(p.res);

    // ======================================================================== PH_LOCAL
    if (p.phase_begin <= PH_LOCAL && PH_LOCAL < p.phase_end && two_pass) {
        // (1) acc = g + residual -> residual; exact iterations histogram the top digit on the fly,
        //     threshold-reuse iterations count the guard ladder.
        const float thr0 = thr_in;
        const LadderCfg lcl = ladder_cfg(p, !exact_local);
        ladder_build(s_lthr, s_lcnt, lcl, thr0);

        auto visit = [&](float x) {
            if (exact_local) {
                hist_add(s_hist, x, 0, 0u);
            } else {
                float ax = fabsf(x);
                if (ax > thr0) atomicAdd(&s_lcnt[ladder_rung(s_lthr, lcl.n_total, ax)], 1);
            }
        };
        // Exact iterations: instead of histogramming all n magnitudes (shared-memory atomics on a handful of hot
        // exponent bins), only the elements above a cut derived from the carried threshold become candidates for the
        // radix select -- a few k of them.  The k-th largest of the candidates IS the k-th largest overall as long as
        // at least k elements pass the cut; otherwise (first call, or the gradient scale collapsed) fall back to the
        // full three-pass select.
        const float cut = (exact_local && thr0 > 0.f) ? thr0 * p.prefilter : -1.f;
        const bool prefilter = cut > 0.f;
        constexpr int kLocTile = 4;
        for (int base = blockIdx.x * kThreads * kLocTile; base < n4; base += gridDim.x * kThreads * kLocTile) {
            float4 a[kLocTile], r[kLocTile];
            bool in[kLocTile];
#pragma unroll
            for (int u = 0; u < kLocTile; ++u) {
                const int v = base + u * kThreads + tid;
                in[u] = v < n4;
                if (in[u]) { a[u] = grad4_at(s_src, nsrc, v); r[u] = ld_stream_f4(r4 + v); }
                else { a[u] = make_float4(0.f, 0.f, 0.f, 0.f); r[u] = a[u]; }
            }
#pragma unroll
            for (int u = 0; u < kLocTile; ++u) {
                const int v = base + u * kThreads + tid;
                a[u].x += r[u].x; a[u].y += r[u].y; a[u].z += r[u].z; a[u].w += r[u].w;
                if (in[u]) st_stream_f4(r4 + v, a[u]);
                const float xs[4] = {a[u].x, a[u].y, a[u].z, a[u].w};
                if (!prefilter) {
                    if (in[u]) { visit(xs[0]); visit(xs[1]); visit(xs[2]); visit(xs[3]); }
                    continue;
                }
                unsigned bits = 0u;
                int tot = 0;
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const bool pd = in[u] && fabsf(xs[c]) > cut;
                    if (pd) bits |= 1u << c;
                    tot += __popc(__ballot_sync(0xffffffffu, pd));
                }
                if (tot == 0) continue;
                int run = 0;
                if (lane == 0) run = atomicAdd(&st->cand_cursor, tot);
                run = __shfl_sync(0xffffffffu, run, 0);
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const bool pd = (bits >> c) & 1u;
                    const unsigned m = __ballot_sync(0xffffffffu, pd);
                    if (pd) {
                        const int pos = run + __popc(m & ((1u << lane) - 1u));
                        if (pos < p.ccap) p.cand[pos] = 4 * v + c;
                    }
                    run += __popc(m);
                }
            }
        }
        if (blockIdx.x == 0) {
            for (int i = n4 * 4 + tid; i < n; i += kThreads) {
                float a = grad_at(s_src, nsrc, i) + p.res[i];
                p.res[i] = a;
                if (prefilter) {
                    if (fabsf(a) > cut) { int pos = atomicAdd(&st->cand_cursor, 1); if (pos < p.ccap) p.cand[pos] = i; }
                } else {
                    visit(a);
                }
            }
        }
        if (exact_local) {
            float thr;
            bool done = false;
            if (prefilter) {
                grid_sync(&st->bar);
                const int ncand = *reinterpret_cast<volatile int*>(&st->cand_cursor);
                if (ncand >= p.k && ncand <= p.ccap) {
                    Seg seg{p.res, ncand, p.cand};
                    thr = grid_kth_abs(&seg, 1, false, (uint32_t)p.k, st, s_hist, s_w, 0);
                    done = true;
                }
            }
            if (!done) {
                if (!prefilter) hist_flush(st, s_hist);
                Seg seg{p.res, n, nullptr};
                thr = grid_kth_abs(&seg, 1, false, (uint32_t)p.k, st, s_hist, s_w, /*first_pass=*/prefilter ? 0 : 1);
            }
            if (blockIdx.x == 0 && tid == 0) { st->local_thr_used = thr; st->cand_cursor = 0; }
        } else {
            ladder_flush(st, s_lcnt);
            grid_sync(&st->bar);
            if (blockIdx.x == 0 && tid == 0) {
                int cnt;
                st->local_thr_used = ladder_pick(st, lcl, thr0, p.guard_limit, p.cap_limit, &cnt);
            }
        }
        grid_sync(&st->bar);

        // (2) balanced region re-partition: local quantile cut points of the selected set, averaged
        //     over ranks through the cut mailboxes (replaces nonzero() + host Allreduce, B4).
        if (p.repartition) {
            const float thr = st->local_thr_used;
            const int W = gridDim.x * kWarps;
            const int Lw = (((n + W - 1) / W) + 31) / 32 * 32;
            {
                const int gw = blockIdx.x * kWarps + warp;
                const long long lo = (long long)gw * Lw;
                const long long hi = min((long long)n, lo + Lw);
                int cnt = 0;
                for (long long base = lo; base < hi; base += 32) {
                    long long i = base + lane;
                    float x = (i < hi) ? __ldcg(p.res + i) : 0.f;
                    cnt += __popc(__ballot_sync(0xffffffffu, fabsf(x) > thr));
                }
                if (lane == 0) st->wcounts[gw] = cnt;
            }
            grid_sync(&st->bar);
            if (blockIdx.x == 0) {
                const int per = (W + kThreads - 1) / kThreads;
                int mysum = 0;
                for (int j = 0; j < per; ++j) {
                    int w = tid * per + j;
                    if (w < W) mysum += st->wcounts[w];
                }
                int M;
                int excl = block_excl_scan(mysum, s_w, &M);
                const int chunkM = M / P;
                // s_misc[2*j], s_misc[2*j+1] = (warp id, rank inside that warp's range) of cut j
                if (M > 0) {
                    for (int j = 1; j < P; ++j) {
                        int target = chunkM * j;
                        if (excl <= target && target < excl + mysum) {
                            int run = excl;
                            for (int q = 0; q < per; ++q) {
                                int w = tid * per + q;
                                int c = (w < W) ? st->wcounts[w] : 0;
                                if (target < run + c) { s_misc[2 * j] = w; s_misc[2 * j + 1] = target - run; break; }
                                run += c;
                            }
                        }
                    }
                }
                __syncthreads();
                if (warp >= 1 && warp < P) {
                    const int j = warp;
                    int cut;
                    if (M > 0) {
                        const int gw = s_misc[2 * j];
                        int want = s_misc[2 * j + 1];
                        const long long lo = (long long)gw * Lw;
                        const long long hi = min((long long)n, lo + Lw);
                        cut = (int)lo;
                        for (long long base = lo; base < hi; base += 32) {
                            long long i = base + lane;
                            float x = (i < hi) ? __ldcg(p.res + i) : 0.f;
                            unsigned m = __ballot_sync(0xffffffffu, fabsf(x) > thr);
                            int c = __popc(m);
                            if (want < c) { cut = (int)base + (int)__fns(m, 0, want + 1); break; }
                            want -= c;
                        }
                    } else {
                        cut = (n / P) * j;
                    }
                    if (lane == 0) st->cuts[j - 1] = cut;
                }
                __syncthreads();
                if (tid < P) {               // push my cut points to peer `tid`, then raise its flag
                    int* dst = cut_data(p.peers[tid], p.L, par, rank);
                    for (int j = 0; j < P - 1; ++j) st_relaxed_sys_u32(reinterpret_cast<uint32_t*>(dst + j), (uint32_t)st->cuts[j]);
                    st_release_sys_u64(cut_mbox(p.peers[tid], p.L, par, rank), make_mail(epoch, 1u));
                }
                if (tid < P) wait_mailbox(cut_mbox(me, p.L, par, tid), epoch, sg_cut);
                __syncthreads();
                if (tid < P - 1) {
                    long long sum = 0;
                    for (int s = 0; s < P; ++s)
                        sum += (long long)ld_relaxed_sys_u32(reinterpret_cast<uint32_t*>(cut_data(me, p.L, par, s) + tid));
                    s_misc[tid] = (int)(sum / P);
                }
                __syncthreads();
                if (tid == 0) {
                    int prev = 0;
                    st->edges[0] = 0;
                    for (int j = 0; j < P - 1; ++j) {
                        int c = s_misc[j];
                        c = max(prev, min(c, n));
                        st->edges[j + 1] = c;
                        prev = c;
                    }
                    st->edges[P] = n;
                }
            }
            grid_sync(&st->bar);
        }
    }

    // region edges and send-slot offsets for this call
    if (tid <= P) s_edges[tid] = st->edges[tid];
    __syncthreads();
    if (tid <= P) s_soff[tid] = (tid < P) ? slot_off(p.L, s_edges, tid) : (p.L.cap > 0 ? P * p.L.cap : slot_off(p.L, s_edges, P));
    __syncthreads();
    int* const my_sidx = send_idx_base(me, p.L);
    float* const my_sval = send_val_base(me, p.L);
    // per-phase device timestamps (observability: the reference's _compression/_allreduce wall-clock timers, SURVEY 5.1)
    auto stamp = [&](int slot) { if (blockIdx.x == 0 && tid == 0) st->t_phase[slot] = globaltimer_ns(); };
    stamp(0);

    // ======================================================================== PH_PACK (+ publish to the region owners)
    if (p.phase_begin <= PH_PACK && PH_PACK < p.phase_end) {
        float thr_sel = two_pass ? st->local_thr_used : thr_in;
        const bool bounded = p.L.cap > 0;
        // Overflow policy of the bounded layout (Ok-Topk residual rule): if a destination's slot is full, raise the threshold
        // and redo the pack pass from the accumulator (already in the residual buffer).  Everything above the final
        // threshold is then in the slots, everything below stays in the residual: nothing selected is lost.  The decision
        // is taken identically by every CTA from the slot cursors after a grid barrier.  Classic-residual schemes
        // (TopkDSA / gaussiankSA) zero the residual only for entries that found room, so an unsent entry stays put.
        const bool can_redo = bounded && p.residual_mode == RES_OKTOPK && p.max_redo > 0;
        float redo_f = p.redo_factor > 1.f ? p.redo_factor : 1.5f;
        int attempt = 0;
        int dropped = 0;
        if (blockIdx.x == 0 && tid == 0) { st->stat_global_count = 0; st->stat_recv_total = 0; st->stat_dense_fallback = 0; }

        const PackRing ring{dyn_pk, dyn_pk + kPackStages * kTileV, s_pk_bar, s_pk_empty};   // [kPackStages][kTileV] each
        int ring_it = 0;                                                // tiles this CTA has pushed through the ring so far

        while (true) {
            const bool res_only = two_pass || attempt > 0;              // the accumulator is already in the residual buffer
            const bool ladder_on = !two_pass;                           // count the over-selection ladder in this pass
            const LadderCfg lc = ladder_cfg(p, ladder_on);
            ladder_build(s_lthr, s_lcnt, lc, thr_sel);
            dropped = 0;

            // one element per lane; every lane of the warp calls this (converged) -- scalar tail only
            auto emit = [&](int i, float x, bool inrange) {
                const float ax = fabsf(x);
                const bool pred = inrange && ax > thr_sel;
                unsigned todo = __ballot_sync(0xffffffffu, pred);
                if (todo == 0) return;
                int d = 0;
                if (pred) {
                    d = region_of(s_edges, P, i);
                    atomicAdd(&s_lcnt[lc.n_total > 1 ? ladder_rung(s_lthr, lc.n_total, ax) : 0], 1);
                }
                while (todo) {
                    const int leader = __ffs(todo) - 1;
                    const int dl = __shfl_sync(0xffffffffu, d, leader);
                    const bool mine = pred && d == dl;
                    const unsigned m = __ballot_sync(0xffffffffu, mine);
                    int base = 0;
                    if (lane == leader) base = atomicAdd(&st->send_cursor[dl], __popc(m));
                    base = __shfl_sync(0xffffffffu, base, leader);
                    if (mine) {
                        const int pos = base + __popc(m & ((1u << lane) - 1u));
                        if (pos < s_soff[dl + 1] - s_soff[dl]) {
                            my_sidx[s_soff[dl] + pos] = i - s_edges[dl];
                            my_sval[s_soff[dl] + pos] = x;
                            if (p.residual_mode != RES_OKTOPK) p.res[i] = 0.f;   // classic local error feedback: sent => cleared
                        } else {
                            dropped++;                                           // no room: the entry stays in the residual
                        }
                    }
                    todo &= ~m;
                }
            };

            const PackSrc src{s_src, nsrc, s_tail_v, s_tail_q, ntail};
            const PackSel sel{thr_sel, lc, s_lthr, s_lcnt, s_edges, s_soff, my_sidx, my_sval, P};
            ring_it += pack_stream<kPackStages>(p, tmap, ring, ring_it, res_only, attempt == 0 && p.zero_g, src, sel, dropped);
            if (blockIdx.x == 0 && warp == 0 && (n & 3)) {
                int i = n4 * 4 + lane;
                bool in = i < n;
                float a = 0.f;
                if (in) {
                    a = res_only ? p.res[i] : (grad_at(s_src, nsrc, i) + p.res[i]);
                    if (!res_only) p.res[i] = a;
                    if (p.zero_g) p.g[i] = 0.f;
                }
                emit(i, a, in);
            }
            if (p.residual_mode == RES_LOCAL_GE && blockIdx.x == 0 && (n & 3)) {      // scalar tail of the same rule
                for (int i = n4 * 4 + tid; i < n; i += kThreads) {
                    float x = p.res[i];
                    if (x != 0.f && fabsf(x) == thr_sel && atomicAdd(&st->tie_cursor, 1) < (int)__ldcg(&st->sel_krem))
                        p.res[i] = 0.f;
                }
            }
            ladder_flush(st, s_lcnt);
            if (!can_redo) break;
            grid_sync(&st->bar);
            bool over = false;
            for (int d = 0; d < P; ++d) over = over || (__ldcg(&st->send_cursor[d]) > s_soff[d + 1] - s_soff[d]);
            if (!over || attempt >= p.max_redo) break;
            grid_sync(&st->bar);                                            // every CTA has read the cursors
            if (blockIdx.x == 0 && tid == 0) {
                for (int d = 0; d < P; ++d) st->send_cursor[d] = 0;
                for (int q = 0; q < kGuardMax; ++q) st->guard_counts[q] = 0;
                st->cum_redo += 1ULL;
            }
            thr_sel = fmaxf(thr_sel, 1e-30f) * redo_f;                      // identical on every CTA
            redo_f = fminf(redo_f * redo_f, 1e6f);
            ++attempt;
            grid_sync(&st->bar);
        }
        {
            int dsum = warp_sum(dropped);
            if (lane == 0 && dsum) atomicAdd(&st->cum_overflow_send, (unsigned long long)dsum);
        }
        // ---- publish: final (guarded) threshold + per-destination counts into the owners' mailboxes.  Done by the LAST CTA
        //      to finish packing (ticket), or by block 0 when the redo policy's grid barrier has already run.
        const bool publisher = can_redo ? (blockIdx.x == 0) : last_cta_ticket(&st->tick[0]);
        if (publisher) {
            if (tid == 0) {
                int cnt;
                const float t = ladder_pick(st, ladder_cfg(p, !two_pass), thr_sel, p.guard_limit, p.cap_limit, &cnt);
                st->local_thr_used = t;
                st->pack_thr = thr_sel;
                st->stat_local_count = cnt;
                st->tie_cursor = 0;
                float nt = t;
                if ((double)cnt < p.l_low_cnt) nt = t / p.l_factor;
                else if ((double)cnt > p.l_high_cnt) nt = t * p.l_factor;
                st->local_thr = nt;
                s_thr[0] = t;
                __threadfence();
            }
            __syncthreads();
            if (tid < P) {
                const int c = min(__ldcg(&st->send_cursor[tid]), s_soff[tid + 1] - s_soff[tid]);
                st_relaxed_sys_u32(reinterpret_cast<uint32_t*>(rs_thr(p.peers[tid], p.L, par, rank)), __float_as_uint(s_thr[0]));
                st_release_sys_u64(rs_mbox(p.peers[tid], p.L, par, rank), make_mail(epoch, (uint32_t)c));
            }
            __syncthreads();
        }
        stamp(1);
    }

    // ======================================================================== PH_REDUCE
    if (p.phase_begin <= PH_REDUCE && PH_REDUCE < p.phase_end) {
        // All P mailboxes, my own included: the local publisher raises my own flag only after EVERY local CTA has finished
        // packing (ticket), so this wait is also the local barrier between "bucket zeroed" and "contributions added".
        if (tid < P) {
            s_cnt[tid] = (int)wait_mailbox(rs_mbox(me, p.L, par, tid), epoch, sg_rs);
            s_thr[tid] = __uint_as_float(ld_relaxed_sys_u32(reinterpret_cast<uint32_t*>(rs_thr(me, p.L, par, tid))));
        }
        __syncthreads();
        stamp(6);
        const int off_me = s_edges[rank];
        const int len_me = s_edges[rank + 1] - off_me;
        float* greg = p.g + off_me;
        int pulled = 0;
        // Scatter-add with first-touch detection: the bucket is all-zero here (cleared by the pack pass, or already zero
        // when the gradient was read from its sources), so the contribution that finds
        // 0.0 is the first one of its index; that index goes on the candidate list the global selection walks, which
        // makes the selection O(#entries) instead of a scan of the whole region (4n/P bytes).  (A sum that passes
        // through exactly 0.0 can list an index twice; the selection claims each index with an exchange, so a
        // duplicate is seen as empty.)
        auto add = [&](int s_local, int idx, float val, const float* thr_of) {
            const bool ok = fabsf(val) > thr_of[s_local] && (unsigned)idx < (unsigned)len_me;
            if (p.cand_mode) {
                float old = 1.f;
                if (ok) old = atomicAdd(greg + idx, val);
                const bool first = ok && old == 0.f;
                const int pos = warp_append_active(&st->cand_cursor, first);
                if (first && pos < p.ccap) p.cand[pos] = idx;
            } else if (ok) {
                red_add_f32(greg + idx, val);               // high density: fire-and-forget reduction, region scanned later
            }
            pulled++;
        };
        const int my_soff = s_soff[rank];
        if (!p.deterministic) {
            if (tid < P) {                           // staggered start: spread the pulls over the switch ports
                const int s = (rank + tid) % P;
                s_srcs[tid].idx = send_idx_base(p.peers[s], p.L) + my_soff;
                s_srcs[tid].val = send_val_base(p.peers[s], p.L) + my_soff;
                s_srcs[tid].count = s_cnt[s];
                s_sthr[tid] = s_thr[s];
            }
            __syncthreads();
            pull_chunks(s_srcs, P, p.pull_tma != 0, &s_pull, pipe_it,
                        [&](int sl, int idx, float val) { add(sl, idx, val, s_sthr); });
        } else {
            for (int s = 0; s < P; ++s) {            // fixed source order => bitwise reproducible sums
                ChunkSrc src{send_idx_base(p.peers[s], p.L) + my_soff, send_val_base(p.peers[s], p.L) + my_soff, s_cnt[s]};
                float thr1 = s_thr[s];
                pull_chunks(&src, 1, p.pull_tma != 0, &s_pull, pipe_it,
                            [&](int, int idx, float val) { add(0, idx, val, &thr1); });
                grid_sync(&st->bar);
            }
        }
        int psum = warp_sum(pulled);
        if (lane == 0 && psum) atomicAdd(&st->stat_recv_total, psum);
        if (PH_REDUCE + 1 < p.phase_end) grid_sync(&st->bar);
        stamp(2);
    }

    // ======================================================================== PH_GSELECT (+ publish my gather count)
    if (p.phase_begin <= PH_GSELECT && PH_GSELECT < p.phase_end) {
        const float gthr = st->global_thr;
        const int lo = s_edges[rank], hi = s_edges[rank + 1];
        const int gcap = p.L.gcap;
        int* gi = gat_idx(me, p.L, par);
        float* gv = gat_val(me, p.L, par);
        // GLB_ALL_NONZERO (TopkDSA): everything non-zero is gathered, so the reduced region is left IN PLACE (the final
        // phase overwrites every entry with val/P; the dense-fallback path reads the regions directly).  The threshold
        // modes claim the value and leave the bucket all-zero for the final phase.
        const bool keep_in_place = p.global_mode == GLB_ALL_NONZERO;
        int dropped = 0;
        if (p.cand_mode) {
            // Low density: walk the candidate list of the reduce phase (every index of my region that received a
            // contribution): claim the reduced value (exchange with 0: the bucket stays all-zero until the final phase
            // writes the kept entries), select, append to my gather slot.  No scan of the region.
            const int ncand = min(*reinterpret_cast<volatile int*>(&st->cand_cursor), p.ccap);
            const int ncr = (ncand + 31) / 32 * 32;
            for (int c = gtid; c < ncr; c += gthreads) {
                const bool in = c < ncand;
                const int i = in ? __ldcg(p.cand + c) : 0;
                const float v = in ? (keep_in_place ? __ldcg(p.g + lo + i) : atomicExch(p.g + lo + i, 0.f)) : 0.f;
                const bool nz = in && v != 0.f;
                const bool sel = (p.global_mode == GLB_THRESHOLD) ? (nz && fabsf(v) > gthr) : nz;
                const int pos = warp_append(&st->gather_cursor, sel);
                if (sel) {
                    if (pos < gcap) { gi[pos] = lo + i; gv[pos] = v; }
                    else { dropped++; if (keep_in_place) p.g[lo + i] = 0.f; }
                }
            }
        } else {
            // High density (a large fraction of the region is non-zero): stream the region through the TMA ring, one
            // gather-slot reservation per warp per tile, and zero what was read (the final phase writes the kept
            // entries).  Scalar head / tail so that the body is 16-byte aligned (region edges are arbitrary).
            auto visit1 = [&](int i, bool in) {
                const float v = in ? __ldcg(p.g + i) : 0.f;
                const bool nz = in && v != 0.f;
                const bool sel = (p.global_mode == GLB_THRESHOLD) ? (nz && fabsf(v) > gthr) : nz;
                const int pos = warp_append(&st->gather_cursor, sel);
                bool lost = false;
                if (sel) {
                    if (pos < gcap) { gi[pos] = i; gv[pos] = v; }
                    else { dropped++; lost = true; }
                }
                if (nz && (!keep_in_place || lost)) p.g[i] = 0.f;
            };
            const int first = min(hi, (lo + 3) & ~3), last = max(first, hi & ~3);
            if (blockIdx.x == 0 && warp == 0) {
                visit1(lo + lane, lo + lane < first);
                visit1(last + lane, last + lane < hi);
            }
            const int nv = (last - first) >> 2;
            const float4* gv4 = reinterpret_cast<const float4*>(p.g + first);
            tma_stream_tiles<kScanStages>(gv4, nv, dyn_pk, s_sc_bar, [&](const float4* tile, int q0) {
                float4 a[kPackTile];
                unsigned nzbits = 0u, selbits = 0u, lostbits = 0u;
                int tot = 0;
#pragma unroll
                for (int u = 0; u < kPackTile; ++u) {
                    const bool in = q0 + u * kThreads + tid < nv;
                    a[u] = in ? tile[u * kThreads + tid] : make_float4(0.f, 0.f, 0.f, 0.f);
                    const float xs[4] = {a[u].x, a[u].y, a[u].z, a[u].w};
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const bool nz = in && xs[c] != 0.f;
                        const bool sel = (p.global_mode == GLB_THRESHOLD) ? (nz && fabsf(xs[c]) > gthr) : nz;
                        if (nz) nzbits |= 1u << (u * 4 + c);
                        if (sel) selbits |= 1u << (u * 4 + c);
                        tot += __popc(__ballot_sync(0xffffffffu, sel));
                    }
                }
                if (__ballot_sync(0xffffffffu, nzbits != 0u) == 0u) return;       // nothing landed in this span
                int run = 0;
                if (tot != 0) {
                    if (lane == 0) run = atomicAdd(&st->gather_cursor, tot);
                    run = __shfl_sync(0xffffffffu, run, 0);
                }
                const unsigned lt = (1u << lane) - 1u;
#pragma unroll
                for (int u = 0; u < kPackTile; ++u) {
                    const float xs[4] = {a[u].x, a[u].y, a[u].z, a[u].w};
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const bool sel = (selbits >> (u * 4 + c)) & 1u;
                        const unsigned m = __ballot_sync(0xffffffffu, sel);
                        if (sel) {
                            const int pos = run + __popc(m & lt);
                            if (pos < gcap) {
                                gi[pos] = first + 4 * (q0 + u * kThreads + tid) + c;
                                gv[pos] = xs[c];
                            } else {
                                dropped++;
                                lostbits |= 1u << (u * 4 + c);
                            }
                        }
                        run += __popc(m);
                    }
                    if (!keep_in_place) {
                        if ((nzbits >> (u * 4)) & 0xfu)
                            *reinterpret_cast<float4*>(p.g + first + 4 * (q0 + u * kThreads + tid)) = make_float4(0.f, 0.f, 0.f, 0.f);
                    } else if ((lostbits >> (u * 4)) & 0xfu) {
#pragma unroll
                        for (int c = 0; c < 4; ++c)
                            if ((lostbits >> (u * 4 + c)) & 1u) p.g[first + 4 * (q0 + u * kThreads + tid) + c] = 0.f;
                    }
                }
            });
        }
        int dsum = warp_sum(dropped);
        if (lane == 0 && dsum) atomicAdd(&st->cum_overflow_gather, (unsigned long long)dsum);
        stamp(3);
        // publish my gather count: the last CTA to finish the selection does it (no grid barrier)
        if (last_cta_ticket(&st->tick[1])) {
            if (tid == 0) s_misc[0] = min(__ldcg(&st->gather_cursor), p.L.gcap);
            __syncthreads();
            if (tid < P) st_release_sys_u64(ag_mbox(p.peers[tid], p.L, par, rank), make_mail(epoch, (uint32_t)s_misc[0]));
            __syncthreads();
        }
    }

    // ======================================================================== PH_FINAL
    if (p.phase_begin <= PH_FINAL && PH_FINAL < p.phase_end) {
        // (again all P flags including my own = local barrier: every local CTA has finished the global selection)
        if (tid < P) s_cnt[tid] = (int)wait_mailbox(ag_mbox(me, p.L, par, tid), epoch, sg_ag);
        __syncthreads();
        stamp(7);
        int T = 0;
        for (int s = 0; s < P; ++s) T += s_cnt[s];
        const float fP = (float)P;
        const bool dense_path = p.global_mode == GLB_ALL_NONZERO && p.dense_nnz_limit > 0 && T >= p.dense_nnz_limit &&
                                P > 1 && p.peer_g[0] != nullptr;
        int kept_cnt = 0;
        if (dense_path) {
            // TopkDSA's dynamic dense fallback (reference VGG/allreducer.py:1311-1353: when the reduced regions hold
            // >= n/3 non-zeros the index/value lists would be bigger than the regions themselves): every rank copies
            // every peer's reduced region straight out of that peer's bucket (128-bit peer loads), scaled by 1/P.
            // My own region must stay un-scaled until every peer has read it: "done reading" flags, then scale in place.
            const float inv = 1.f / fP;
            for (int t = 1; t < P; ++t) {
                const int s = (rank + t) % P;
                const int lo_s = s_edges[s], hi_s = s_edges[s + 1];
                const float* src = p.peer_g[s];
                const int first = min(hi_s, (lo_s + 3) & ~3), last = max(first, hi_s & ~3);
                for (int i = lo_s + gtid; i < first; i += gthreads) p.g[i] = ld_peer_f32(src + i) * inv;
                for (int i = last + gtid; i < hi_s; i += gthreads) p.g[i] = ld_peer_f32(src + i) * inv;
                const int nv = (last - first) >> 2;
                const int4* s4 = reinterpret_cast<const int4*>(src + first);
                float4* d4 = reinterpret_cast<float4*>(p.g + first);
                for (int v = gtid; v < nv; v += gthreads) {
                    const int4 r = ld_peer_i4(s4 + v);
                    st_stream_f4(d4 + v, make_float4(__int_as_float(r.x) * inv, __int_as_float(r.y) * inv,
                                                     __int_as_float(r.z) * inv, __int_as_float(r.w) * inv));
                }
            }
            grid_sync(&st->bar);                     // all my peer reads have returned
            if (blockIdx.x == 0 && tid < P) st_release_sys_u64(done_mbox(p.peers[tid], p.L, par, rank), make_mail(epoch, 1u));
            if (tid < P) wait_mailbox(done_mbox(me, p.L, par, tid), epoch, sg_done);
            __syncthreads();
            const int lo = s_edges[rank], hi = s_edges[rank + 1];
            for (int i = lo + gtid; i < hi; i += gthreads) p.g[i] = __ldcg(p.g + i) * inv;
            if (blockIdx.x == 0 && tid == 0) { st->stat_dense_fallback = 1; st->stat_global_count = T; }
        } else {
            float gsel = 0.f;
            if (p.global_mode == GLB_EXACT_TOPK) {
                if (tid < P) { s_segs[tid].ptr = gat_val(p.peers[tid], p.L, par); s_segs[tid].count = s_cnt[tid]; s_segs[tid].idx = nullptr; }
                __syncthreads();
                const uint32_t kk = (uint32_t)min(T, p.k);
                gsel = (kk > 0) ? grid_kth_abs(s_segs, P, true, kk, st, s_hist, s_w, 0) : 0.f;
                if (blockIdx.x == 0 && tid == 0) st->global_thr = gsel;
            } else if (p.global_mode == GLB_THRESHOLD && blockIdx.x == 0 && tid == 0) {
                float gt = st->global_thr;
                if ((double)T < p.g_low_cnt) gt = gt / p.g_inc;
                else if ((double)T > p.g_high_cnt) gt = gt * p.g_dec;
                st->global_thr = gt;
            }
            const float thr_used = st->local_thr_used;
            if (tid < P) {
                const int s = (rank + tid) % P;
                s_srcs[tid].idx = gat_idx(p.peers[s], p.L, par);
                s_srcs[tid].val = gat_val(p.peers[s], p.L, par);
                s_srcs[tid].count = s_cnt[s];
            }
            __syncthreads();
            const bool exact = p.global_mode == GLB_EXACT_TOPK;
            pull_chunks(s_srcs, P, p.pull_tma != 0, &s_pull, pipe_it, [&](int sl, int idx, float val) {
                if ((unsigned)idx >= (unsigned)n) return;
                bool keep = exact ? (fabsf(val) >= gsel) : true;
                if (!keep) return;
                kept_cnt++;
                p.g[idx] = val / fP;             // the bucket is all-zero here: every kept entry (own region included) lands now
                if (p.residual_mode == RES_OKTOPK) {
                    float r = p.res[idx];
                    if (fabsf(r) > thr_used) p.res[idx] = 0.f;
                }
            });
            int ksum = warp_sum(kept_cnt);
            if (lane == 0 && ksum) atomicAdd(&st->stat_global_count, ksum);
        }
        // end of call: the last CTA to get here closes the books (no grid barrier: everybody else just exits)
        if (last_cta_ticket(&st->tick[2]) && tid == 0) {
            const unsigned long long t_end = globaltimer_ns();
            st->epoch = epoch;
            st->t_phase[4] = t_end;
            st->stat_gather_total = T;
            for (int d = 0; d < P; ++d) st->send_cursor[d] = 0;
            st->gather_cursor = 0;
            st->cand_cursor = 0;
            const unsigned long long os = *reinterpret_cast<volatile unsigned long long*>(&st->cum_overflow_send);
            const unsigned long long og = *reinterpret_cast<volatile unsigned long long*>(&st->cum_overflow_gather);
            const unsigned long long rd = *reinterpret_cast<volatile unsigned long long*>(&st->cum_redo);
            st->stat_overflow_send = (int)min(os - st->snap_overflow_send, 0x7fffffffULL);
            st->stat_overflow_gather = (int)min(og - st->snap_overflow_gather, 0x7fffffffULL);
            st->stat_redo = (int)(rd - st->snap_redo);
            st->snap_overflow_send = os; st->snap_overflow_gather = og; st->snap_redo = rd;
            TraceRec& tr = st->trace[epoch % kTraceLen];
            auto us = [&](int a, int b) {
                const unsigned long long ta = *reinterpret_cast<volatile unsigned long long*>(&st->t_phase[a]);
                const unsigned long long tb = *reinterpret_cast<volatile unsigned long long*>(&st->t_phase[b]);
                return tb >= ta ? (float)(tb - ta) * 1e-3f : 0.f;
            };
            tr.epoch = epoch;
            tr.local_count = st->stat_local_count;
            tr.global_count = *reinterpret_cast<volatile int*>(&st->stat_global_count);
            tr.recv_total = *reinterpret_cast<volatile int*>(&st->stat_recv_total);
            tr.gather_total = T;
            tr.overflow_send = st->stat_overflow_send;
            tr.overflow_gather = st->stat_overflow_gather;
            tr.redo = st->stat_redo;
            tr.local_thr = st->local_thr_used;
            tr.global_thr = st->global_thr;
            tr.us_local = us(5, 0); tr.us_pack = us(0, 1); tr.us_wait_rs = us(1, 6); tr.us_reduce = us(6, 2);
            tr.us_gselect = us(2, 3); tr.us_wait_ag = us(3, 7); tr.us_final = us(7, 4);
            tr.t_begin = st->t_phase[5];
        }
    }
}

// ------------------------------------------------------------------------------------------
// Early pack: the threshold-reuse pack pass over some ranges of the bucket, launched while backward is still running
// (their gradients exist; the rest of the bucket's may not).  It does exactly the per-element work of the call's pack
// pass (pack_stream) with the carried threshold, appends to the same send slots through st->send_cursor and adds its
// ladder tallies to st->guard_counts; the call that follows packs only what no segment covered and publishes.  It must
// co-run with backward without holding it up: an ordinary (non-cooperative) grid of a few dozen CTAs with a 64 KB ring
// leaves most SMs to the backward kernels (cuDNN's take far more shared memory, so an SM that hosts a segment CTA hosts
// none of theirs).  A carried threshold of 0 makes the call recompute the exact threshold over the whole bucket: the
// segment then does nothing.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) oktopk_segment_kernel(const OktParams p) {
    __shared__ int s_edges[OKT_MAXP + 1];
    __shared__ int s_soff[OKT_MAXP + 1];
    __shared__ float s_lthr[kGuardMax];
    __shared__ int s_lcnt[kGuardMax];
    __shared__ __align__(8) uint64_t s_full[kSegStages];
    __shared__ __align__(8) uint64_t s_empty[kSegStages];
    __shared__ SrcSeg s_src[kSrcSegMax];
    __shared__ int s_tail_v[kSrcSegMax], s_tail_q[kSrcSegMax];
    __shared__ int s_ntail;
    __shared__ int s_rlo[kPackRangeMax], s_rhi[kPackRangeMax], s_rfirst[kPackRangeMax + 1];
    extern __shared__ __align__(128) float4 dyn_seg[];      // [2][kSegStages][kTileV]

    if (verdict_set(p.skip)) return;
    OktState* st = p.st;
    const float thr = st->local_thr;
    if (thr == 0.f) return;
    const int tid = threadIdx.x, P = p.P;
    if (tid == 0) {
        for (int q = 0; q < kSegStages; ++q) { mbar_init(&s_full[q], 1); mbar_init(&s_empty[q], kWarps); }
        mbar_fence_init();
    }
    if (tid <= P) s_edges[tid] = st->edges[tid];
    load_src_table(p, s_src, s_tail_v, s_tail_q, &s_ntail);
    if (tid <= P) s_soff[tid] = (tid < P) ? slot_off(p.L, s_edges, tid) : slot_off(p.L, s_edges, P);
    const TileMap tmap = tile_map_build(p.pk_nr, p.pk_lo, p.pk_hi, s_rlo, s_rhi, s_rfirst);
    const LadderCfg lc = ladder_cfg(p, true);
    ladder_build(s_lthr, s_lcnt, lc, thr);
    char* me = p.peers[p.rank];
    const PackRing ring{dyn_seg, dyn_seg + kSegStages * kTileV, s_full, s_empty};
    const PackSrc src{s_src, p.nsrc, s_tail_v, s_tail_q, s_ntail};
    const PackSel sel{thr, lc, s_lthr, s_lcnt, s_edges, s_soff, send_idx_base(me, p.L), send_val_base(me, p.L), P};
    int dropped = 0;
    pack_stream<kSegStages>(p, tmap, ring, 0, false, false, src, sel, dropped);
    ladder_flush(st, s_lcnt);
}

// ------------------------------------------------------------------------------------------
// standalone exact k-th |x| (used by tests and by the dist/NCCL baseline on CUDA tensors)
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads, 2) kth_abs_kernel(const float* x, int n, int k, OktState* st, float* out) {
    __shared__ uint32_t s_hist[kHistBins];
    __shared__ int s_w[kWarps + 1];
    for (int b = threadIdx.x; b < kHistBins; b += kThreads) s_hist[b] = 0;
    __syncthreads();
    Seg seg{x, n, nullptr};
    float t = grid_kth_abs(&seg, 1, false, (uint32_t)k, st, s_hist, s_w, 0);
    if (blockIdx.x == 0 && threadIdx.x == 0) *out = t;
}

// ------------------------------------------------------------------------------------------
// host launchers
// ------------------------------------------------------------------------------------------
int okt_max_coop_grid(int device) {
    int sms = 0, per = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    cudaFuncSetAttribute(oktopk_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPackSmemBytes);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, oktopk_fused_kernel, kThreads, kPackSmemBytes);
    if (per < 1) per = 1;
    if (per > kCtasPerSm) per = kCtasPerSm;
    return sms * per;
}

cudaError_t launch_oktopk(const OktParams& p, int grid, cudaStream_t stream) {
    static bool attr_set[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < 64 && !attr_set[dev]) {
        cudaError_t e = cudaFuncSetAttribute(oktopk_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPackSmemBytes);
        if (e != cudaSuccess) return e;
        attr_set[dev] = true;
    }
    void* args[] = {(void*)&p};
    return cudaLaunchCooperativeKernel((void*)oktopk_fused_kernel, dim3(grid), dim3(kThreads), args, kPackSmemBytes, stream);
}

cudaError_t launch_oktopk_segment(const OktParams& p, int max_ctas, cudaStream_t stream) {
    constexpr int kSmem = kSegStages * 2 * kTileV * 16;
    static bool attr_set[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev >= 0 && dev < 64 && !attr_set[dev]) {
        cudaError_t e = cudaFuncSetAttribute(oktopk_segment_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
        if (e != cudaSuccess) return e;
        attr_set[dev] = true;
    }
    int ntiles = 0;
    for (int r = 0; r < p.pk_nr; ++r) ntiles += (p.pk_hi[r] - p.pk_lo[r] + kTileV - 1) / kTileV;
    if (ntiles <= 0) return cudaSuccess;
    const int grid = std::min((ntiles + kSegTiles - 1) / kSegTiles, std::max(max_ctas, 1));
    oktopk_segment_kernel<<<grid, kThreads, kSmem, stream>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_kth_abs(const float* x, int n, int k, OktState* st, float* out_thr, int grid, cudaStream_t stream) {
    void* args[] = {(void*)&x, (void*)&n, (void*)&k, (void*)&st, (void*)&out_thr};
    return cudaLaunchCooperativeKernel((void*)kth_abs_kernel, dim3(grid), dim3(kThreads), args, 0, stream);
}

}  // namespace okt
