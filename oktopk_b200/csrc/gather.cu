// Gather-type sparse allreduce schemes as one persistent kernel: TopkA (exact local top-k),
// TopkAopt (threshold reuse) and Gaussiank (threshold from a normal fit + bounded count
// correction).  Each rank selects, packs (global idx, val) into its peer-visible slot, raises a
// flag in every peer's mailbox, and then every rank pulls all P slots with TMA bulk copies and
// adds val/P into its dense bucket (red.global.add.f32).
//
// Behaviour: SURVEY Appendix B.1 / B.3 / B.6 (reference VGG/allreducer.py:34-69,1100-1150,
// 1420-1465; VGG/compression.py:37-62,220-266).  The reference's <=20 rescans of Gaussiank are
// replaced by ONE ladder-histogram pass that yields the count at every candidate threshold.
//
// TopkA2 (reselect, VGG/allreducer.py:519-525 + VGG/compression.py:151-160): after the P slots have been added, the
// union of the gathered indices (exact first-touch detection through a bitmap) is re-selected down to the global
// top-k with the grid-wide radix select, the losers are zeroed, and every rank puts its own non-surviving picks back
// into its residual.  norm_clip (VGG/allreducer.py:1372-1379): one extra L2-norm pass scales the incoming gradient.
#include "devlib.cuh"

namespace okt {

constexpr int kLadMax = 128;   // thresholds thr * f^j, j in [-loops, +loops], loops <= 63

__global__ void __launch_bounds__(kThreads, 2) gather_scheme_kernel(const GatherParams p) {
    __shared__ uint32_t s_hist[kHistBins];
    __shared__ int s_w[kWarps + 1];
    __shared__ int s_cnt[OKT_MAXP];
    __shared__ float s_lad[kLadMax];
    __shared__ float s_thr;
    __shared__ __align__(128) PullSmem s_pull;

    if (verdict_set(p.skip)) return;
    OktState* st = p.st;
    const int tid = threadIdx.x, lane = tid & 31;
    const int gtid = blockIdx.x * kThreads + tid;
    const int gthreads = gridDim.x * kThreads;
    const int P = p.P, rank = p.rank, n = p.n;
    char* me = p.peers[rank];
    const uint32_t epoch = st->epoch + 1u;
    const int par = epoch & 1u;
    uint32_t pipe_it = 0;

    for (int b = tid; b < kHistBins; b += kThreads) s_hist[b] = 0;
    if (tid == 0) {
        mbar_init(&s_pull.bar[0], 1);
        mbar_init(&s_pull.bar[1], 1);
        mbar_fence_init();
    }
    __syncthreads();

    const int n4 = n >> 2;
    float4* g4 = reinterpret_cast<float4*>(p.g);
    float4* r4 = reinterpret_cast<float4*>(p.res);

    // ---------------------------------------------------------------- norm_clip: ||g||_2 <= clip_max_norm
    float gscale = 1.f;
    if (p.clip_max_norm > 0.f) {
        double ss = 0.0;
        for (int v = gtid; v < n4; v += gthreads) {
            const float4 a = ld_stream_f4(g4 + v);
            ss += (double)a.x * a.x + (double)a.y * a.y + (double)a.z * a.z + (double)a.w * a.w;
        }
        if (blockIdx.x == 0)
            for (int i = n4 * 4 + tid; i < n; i += kThreads) ss += (double)p.g[i] * p.g[i];
        ss = warp_sum_d(ss);
        if (lane == 0 && ss != 0.0) atomicAdd(&st->clip_sumsq, ss);
        grid_sync(&st->bar);
        const double nrm = sqrt(*reinterpret_cast<volatile double*>(&st->clip_sumsq));
        if (nrm > (double)p.clip_max_norm && nrm > 0.0) gscale = (float)((double)p.clip_max_norm / nrm);
    }
    const bool single_pass = (p.select_mode == GS_THRESHOLD_REUSE) && !p.exact_now;
    const bool need_kth = (p.select_mode == GS_EXACT_TOPK) || (p.select_mode == GS_THRESHOLD_REUSE && p.exact_now);
    const bool inclusive = p.select_mode == GS_EXACT_TOPK;     // exact top-k keeps the k-th element itself

    // ---------------------------------------------------------------- pass A (multi-pass modes)
    if (!single_pass) {
        double sum = 0.0, sumsq = 0.0;
        auto visit = [&](float x) {
            if (need_kth) hist_add(s_hist, x, 0, 0u);
            else { sum += (double)x; sumsq += (double)x * (double)x; }
        };
        for (int v = gtid; v < n4; v += gthreads) {
            float4 a = ld_stream_f4(g4 + v);
            float4 r = ld_stream_f4(r4 + v);
            a.x = a.x * gscale + r.x; a.y = a.y * gscale + r.y; a.z = a.z * gscale + r.z; a.w = a.w * gscale + r.w;
            st_stream_f4(r4 + v, a);
            st_stream_f4(g4 + v, make_float4(0.f, 0.f, 0.f, 0.f));
            visit(a.x); visit(a.y); visit(a.z); visit(a.w);
        }
        if (blockIdx.x == 0)
            for (int i = n4 * 4 + tid; i < n; i += kThreads) {
                float a = p.g[i] * gscale + p.res[i];
                p.res[i] = a;
                p.g[i] = 0.f;
                visit(a);
            }
        if (need_kth) {
            hist_flush(st, s_hist);
            Seg seg{p.res, n, nullptr};
            float thr = grid_kth_abs(&seg, 1, false, (uint32_t)p.k, st, s_hist, s_w, 1);
            if (blockIdx.x == 0 && tid == 0) { st->local_thr = thr; st->local_thr_used = thr; }
            grid_sync(&st->bar);
        } else {
            sum = warp_sum_d(sum);
            sumsq = warp_sum_d(sumsq);
            if (lane == 0) { atomicAdd(&st->gs_sum, sum); atomicAdd(&st->gs_sumsq, sumsq); }
            grid_sync(&st->bar);
            // Gaussian threshold: mean - z*std with z = ndtri(rho/2) < 0 (host passes |z| in gauss_factor? no: density)
            const double mean = st->gs_sum / (double)n;
            double var = (n > 1) ? (st->gs_sumsq - (double)n * mean * mean) / (double)(n - 1) : 0.0;
            if (var < 0.0) var = 0.0;
            // |z| for the two-sided tail mass rho: z = -normcdfinv(rho / 2)
            const double z = -normcdfinv((double)p.density * 0.5);
            const float thr0 = (float)(mean + z * sqrt(var));
            const int L = min(p.gauss_loops, (kLadMax - 1) / 2);
            // ladder: s_lad[L + j] = thr0 * f^j
            if (tid == 0) {
                s_lad[L] = thr0;
                float t = thr0;
                for (int j = 1; j <= L; ++j) { t *= p.gauss_factor; s_lad[L + j] = t; }
                t = thr0;
                for (int j = 1; j <= L; ++j) { t /= p.gauss_factor; s_lad[L - j] = t; }
            }
            __syncthreads();
            const int NL = 2 * L + 1;
            const float tmin = s_lad[0];
            // count, for every rung, how many |acc| exceed it: bucket each candidate at its highest rung
            for (int i = gtid; i < n; i += gthreads) {
                float ax = fabsf(__ldcg(p.res + i));
                if (ax > tmin) {
                    int lo = 0, hi = NL - 1;            // largest j with ax > s_lad[j]
                    while (lo < hi) {
                        int mid = (lo + hi + 1) >> 1;
                        if (ax > s_lad[mid]) lo = mid; else hi = mid - 1;
                    }
                    atomicAdd(&s_hist[lo], 1u);
                }
            }
            hist_flush(st, s_hist);
            grid_sync(&st->bar);
            if (blockIdx.x == 0 && tid == 0) {
                // suffix sums: c[j] = #(|acc| > s_lad[j])
                int c[kLadMax];
                int run = 0;
                for (int j = NL - 1; j >= 0; --j) { run += (int)st->hist[j]; c[j] = run; }
                const int k = p.k;
                int j = L;
                const int init = c[L];
                if (p.gauss_mode == 0) {                  // VGG: both directions
                    const int lo = 3 * k / 4, hi = 5 * k / 4;
                    if (init < lo) { int it = 0; while (it < L && c[j] < lo) { --j; ++it; } }
                    else if (init > hi) { int it = 0; while (it < L && c[j] > hi) { ++j; ++it; } }
                } else if (p.gauss_mode == 1) {           // LSTM: only downward
                    const int lo = 3 * k / 4;
                    int it = 0; while (it < L && c[j] < lo) { --j; ++it; }
                } else {                                  // BERT
                    if (init < 3 * k / 4) { const int tgt = 5 * k / 6; int it = 0; while (it < L && c[j] < tgt) { --j; ++it; } }
                }
                st->local_thr = s_lad[j];
                st->local_thr_used = s_lad[j];
                for (int q = 0; q < NL; ++q) st->hist[q] = 0;
                st->gs_sum = 0.0;
                st->gs_sumsq = 0.0;
            }
            grid_sync(&st->bar);
        }
    }

    // ---------------------------------------------------------------- pack into my slot
    {
        const float thr = st->local_thr;
        const int gcap = p.L.gcap;
        int* gi = gat_idx(me, p.L, par);
        float* gv = gat_val(me, p.L, par);
        int selected = 0, dropped = 0;
        auto emit = [&](int i, float x, bool in) {
            const float ax = fabsf(x);
            const bool pred = in && (inclusive ? (ax >= thr && ax > 0.f) : (ax > thr));
            int pos = warp_append(&st->gather_cursor, pred);
            if (pred) {
                selected++;
                if (pos < gcap) { gi[pos] = i; gv[pos] = x; p.res[i] = 0.f; }   // residual zeroed at the selection
                else dropped++;                                              // slot full: stays in the residual
            }
        };
        const int n4r = (n4 + 31) / 32 * 32;
        for (int v = gtid; v < n4r; v += gthreads) {
            const bool in = v < n4;
            float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
            if (in) {
                if (single_pass) {
                    a = ld_stream_f4(g4 + v);
                    float4 r = ld_stream_f4(r4 + v);
                    a.x = a.x * gscale + r.x; a.y = a.y * gscale + r.y; a.z = a.z * gscale + r.z; a.w = a.w * gscale + r.w;
                    st_stream_f4(r4 + v, a);
                    st_stream_f4(g4 + v, make_float4(0.f, 0.f, 0.f, 0.f));
                } else {
                    a = ld_stream_f4(r4 + v);
                }
            }
            const float m4 = fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w)));
            if (__ballot_sync(0xffffffffu, in && m4 >= thr) == 0) continue;
            emit(4 * v + 0, a.x, in);
            emit(4 * v + 1, a.y, in);
            emit(4 * v + 2, a.z, in);
            emit(4 * v + 3, a.w, in);
        }
        if (blockIdx.x == 0 && (tid >> 5) == 0 && (n & 3)) {
            int i = n4 * 4 + lane;
            bool in = i < n;
            float a = 0.f;
            if (in) {
                if (single_pass) { a = p.g[i] * gscale + p.res[i]; p.res[i] = a; p.g[i] = 0.f; }
                else a = p.res[i];
            }
            emit(i, a, in);
        }
        int ssum = warp_sum(selected), dsum = warp_sum(dropped);
        if (lane == 0 && ssum) atomicAdd(&st->guard_counts[0], ssum);
        if (lane == 0 && dsum) atomicAdd(&st->cum_overflow_gather, (unsigned long long)dsum);
        grid_sync(&st->bar);
    }

    // ---------------------------------------------------------------- publish + pull + add
    if (blockIdx.x == 0) {
        if (tid == 0) {
            s_w[0] = min(st->gather_cursor, p.L.gcap);
            st->stat_local_count = st->guard_counts[0];
            st->guard_counts[0] = 0;
            st->stat_global_count = 0;
        }
        __syncthreads();
        if (tid < P) st_release_sys_u64(ag_mbox(p.peers[tid], p.L, par, rank), make_mail(epoch, (uint32_t)s_w[0]));
        __syncthreads();
        if (tid == 0) st->gather_cursor = 0;
    }
    if (tid < P) s_cnt[tid] = (int)wait_mailbox(ag_mbox(me, p.L, par, tid), epoch, SpinGuard{&st->fault, p.timeout_ns, FAULT_AG_TIMEOUT, p.host_fault});
    __syncthreads();
    {
        // Every rank reduces all P slots itself (no owner), so the order of the floating-point additions must be the
        // same on every rank or the replicas drift apart by rounding: sources are processed in rank order with a grid
        // barrier between them (indices are unique inside one slot, so there are no intra-source conflicts) -- the
        // reference's P sequential scatter-adds (VGG/allreducer.py:510-518), bitwise identical on all ranks.
        int T = 0;
        const float fP = (float)P;
        for (int s = 0; s < P; ++s) {
            ChunkSrc src{gat_idx(p.peers[s], p.L, par), gat_val(p.peers[s], p.L, par), s_cnt[s]};
            T += s_cnt[s];
            if (!p.reselect) {
                pull_chunks(&src, 1, p.pull_tma != 0, &s_pull, pipe_it, [&](int, int idx, float val) {
                    if ((unsigned)idx < (unsigned)n) red_add_f32(p.g + idx, val / fP);
                });
            } else {
                // TopkA2: also build the list of DISTINCT gathered indices (bitmap = exact first-touch detection)
                pull_chunks(&src, 1, p.pull_tma != 0, &s_pull, pipe_it, [&](int, int idx, float val) {
                    const bool ok = (unsigned)idx < (unsigned)n;
                    bool first = false;
                    if (ok) {
                        red_add_f32(p.g + idx, val / fP);
                        const unsigned bit = 1u << (idx & 31);
                        first = (atomicOr(p.bitmap + (idx >> 5), bit) & bit) == 0u;
                    }
                    const int pos = warp_append_active(&st->cand_cursor, first);
                    if (first && pos < p.ccap) p.cand[pos] = idx;
                });
            }
            grid_sync(&st->bar);
        }
        int kept_total = T;
        if (p.reselect) {
            const int ncand = min(*reinterpret_cast<volatile int*>(&st->cand_cursor), p.ccap);
            float thr2 = 0.f;
            if (ncand > p.k) {                               // more than k distinct indices: keep the global top-k
                Seg seg{p.g, ncand, p.cand};
                thr2 = grid_kth_abs(&seg, 1, false, (uint32_t)p.k, st, s_hist, s_w, 0);
            }
            // put my own non-surviving picks back into my residual (it was zeroed at the selection)
            {
                const int* mi = gat_idx(me, p.L, par);
                const float* mv = gat_val(me, p.L, par);
                const int mine = s_cnt[rank];
                for (int e = gtid; e < mine; e += gthreads) {
                    const int idx = mi[e];
                    if ((unsigned)idx < (unsigned)n && fabsf(__ldcg(p.g + idx)) < thr2) p.res[idx] += mv[e];
                }
            }
            grid_sync(&st->bar);
            int kept = 0;
            for (int c = gtid; c < ncand; c += gthreads) {
                const int idx = __ldcg(p.cand + c);
                if (fabsf(__ldcg(p.g + idx)) < thr2) p.g[idx] = 0.f; else kept++;
                p.bitmap[idx >> 5] = 0u;                     // leave the bitmap all-zero for the next call
            }
            kept = warp_sum(kept);
            if (lane == 0 && kept) atomicAdd(&st->stat_global_count, kept);
            grid_sync(&st->bar);
            kept_total = *reinterpret_cast<volatile int*>(&st->stat_global_count);
        }
        if (blockIdx.x == 0 && tid == 0) {
            st->epoch = epoch;
            st->stat_gather_total = T;
            st->stat_global_count = kept_total;
            st->cand_cursor = 0;
            st->clip_sumsq = 0.0;
            const unsigned long long og = *reinterpret_cast<volatile unsigned long long*>(&st->cum_overflow_gather);
            st->stat_overflow_gather = (int)min(og - st->snap_overflow_gather, 0x7fffffffULL);
            st->snap_overflow_gather = og;
            st->stat_overflow_send = 0;
        }
    }
}

int gather_max_coop_grid(int device) {
    int sms = 0, per = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, gather_scheme_kernel, kThreads, 0);
    if (per < 1) per = 1;
    if (per > 2) per = 2;
    return sms * per;
}

cudaError_t launch_gather_scheme(const GatherParams& p, int grid, cudaStream_t stream) {
    void* args[] = {(void*)&p};
    return cudaLaunchCooperativeKernel((void*)gather_scheme_kernel, dim3(grid), dim3(kThreads), args, 0, stream);
}

}  // namespace okt
