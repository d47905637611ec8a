// gTopk as ONE persistent cooperative kernel (K9): log2(P) rounds of pairwise sparse merges toward rank 0
// followed by a broadcast of the surviving global top-k, all over peer memory.
//
// Behaviour: SURVEY Appendix B.2 (reference VGG/allreducer.py:76-172: tree rounds :113-152, merge = sum the
// coincident indices and keep the k largest magnitudes of the union :129-138, broadcast :154-162, the local
// picks that did not survive go back into the residual :170-172).  The reference drives the tree from the
// host with mpi4py Send/Recv of NumPy buffers and merges on the CPU; here
//   * every rank's current list lives in its peer-visible slot; a sender only raises a flag
//     (st.release.sys carrying epoch, round and count) in the receiver's mailbox,
//   * the receiver pulls the list with TMA bulk copies over NVLink and merges it into its (all-zero) dense
//     bucket, which doubles as the index -> value map: atomicAdd sums coincident indices, a bitmap gives exact
//     first-touch detection, so the union list is built in the same pass,
//   * the top-k of the union is the grid-wide radix select over that list (no sort),
//   * the final list is pulled by all ranks from rank 0's slot; the bitmap then answers "did my pick
//     survive?" for the residual put-back.
// No host round trip, CUDA-graph capturable, no NCCL.
#include "devlib.cuh"

namespace okt {

__device__ __forceinline__ uint32_t tree_tag(uint32_t epoch, int round) { return (epoch << 5) | (uint32_t)round; }
constexpr int kBcastRound = 31;

__global__ void __launch_bounds__(kThreads, 2) gtopk_kernel(const TreeParams p) {
    __shared__ uint32_t s_hist[kHistBins];
    __shared__ int s_w[kWarps + 1];
    __shared__ int s_cnt;
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
    const SpinGuard sg{&st->fault, p.timeout_ns, FAULT_TREE_TIMEOUT, p.host_fault};

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
    int* const wc = st->wcounts;                 // per-round counters: wc[2r] = new union entries, wc[2r+1] = winners

    // ---------------------------------------------------------------- norm_clip
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

    // ---------------------------------------------------------------- acc = g + residual -> residual, bucket zeroed
    for (int v = gtid; v < n4; v += gthreads) {
        float4 a = ld_stream_f4(g4 + v);
        const float4 r = ld_stream_f4(r4 + v);
        a.x = a.x * gscale + r.x; a.y = a.y * gscale + r.y; a.z = a.z * gscale + r.z; a.w = a.w * gscale + r.w;
        st_stream_f4(r4 + v, a);
        st_stream_f4(g4 + v, make_float4(0.f, 0.f, 0.f, 0.f));
        hist_add(s_hist, a.x, 0, 0u); hist_add(s_hist, a.y, 0, 0u); hist_add(s_hist, a.z, 0, 0u); hist_add(s_hist, a.w, 0, 0u);
    }
    if (blockIdx.x == 0)
        for (int i = n4 * 4 + tid; i < n; i += kThreads) {
            const float a = p.g[i] * gscale + p.res[i];
            p.res[i] = a;
            p.g[i] = 0.f;
            hist_add(s_hist, a, 0, 0u);
        }
    hist_flush(st, s_hist);
    float thr;
    {
        Seg seg{p.res, n, nullptr};
        thr = grid_kth_abs(&seg, 1, false, (uint32_t)p.k, st, s_hist, s_w, 1);
    }

    // ---------------------------------------------------------------- my local top-k -> my slot (+ a private copy)
    int* gi = gat_idx(me, p.L, par);
    float* gv = gat_val(me, p.L, par);
    const int lcap = min(p.L.gcap, p.selcap);
    {
        int dropped = 0;
        auto emit = [&](int i, float x, bool in) {
            const float ax = fabsf(x);
            const bool pred = in && ax >= thr && ax > 0.f;
            const int pos = warp_append(&st->gather_cursor, pred);
            if (pred) {
                if (pos < lcap) { gi[pos] = i; gv[pos] = x; p.sel_idx[pos] = i; p.sel_val[pos] = x; p.res[i] = 0.f; }
                else dropped++;                               // no room: stays in the residual
            }
        };
        const int n4r = (n4 + 31) / 32 * 32;
        for (int v = gtid; v < n4r; v += gthreads) {
            const bool in = v < n4;
            const float4 a = in ? ld_stream_f4(r4 + v) : make_float4(0.f, 0.f, 0.f, 0.f);
            const float m4 = fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w)));
            if (__ballot_sync(0xffffffffu, in && m4 >= thr && m4 > 0.f) == 0) continue;
            emit(4 * v + 0, a.x, in); emit(4 * v + 1, a.y, in); emit(4 * v + 2, a.z, in); emit(4 * v + 3, a.w, in);
        }
        if (blockIdx.x == 0 && (tid >> 5) == 0 && (n & 3)) {
            const int i = n4 * 4 + lane;
            const bool in = i < n;
            emit(i, in ? p.res[i] : 0.f, in);
        }
        const int dsum = warp_sum(dropped);
        if (lane == 0 && dsum) atomicAdd(&st->cum_overflow_gather, (unsigned long long)dsum);
    }
    grid_sync(&st->bar);
    const int m0 = min(__ldcg(&st->gather_cursor), lcap);      // my original picks (put-back list)
    int m = m0;                                                  // length of my current list

    // ---------------------------------------------------------------- tree rounds
    const int chalf = p.ccap >> 1;
    int* candA = p.cand;                                         // union list of the running merge
    int* candB = p.cand + chalf;
    bool scattered = false;
    int recv_total = 0;
    int round = 0;
    for (int step = 1; step < P; step <<= 1, ++round) {
        if ((rank % (2 * step)) == step) {
            // sender: my list is final; raise the receiver's flag and leave the tree
            if (blockIdx.x == 0 && tid == 0)
                st_release_sys_u64(tree_mbox(p.peers[rank - step], p.L, par, rank), make_mail(tree_tag(epoch, round), (uint32_t)m));
            break;
        }
        // receiver (rank % (2 step) == 0)
        if (!scattered) {
            // first merge: my own list goes into the all-zero bucket (index -> value map) and seeds the union list
            for (int e = gtid; e < m; e += gthreads) {
                const int idx = gi[e];
                p.g[idx] = gv[e];
                atomicOr(p.bitmap + (idx >> 5), 1u << (idx & 31));
                candA[e] = idx;
            }
            scattered = true;
            grid_sync(&st->bar);
        }
        if (tid == 0) s_cnt = (int)wait_mailbox(tree_mbox(me, p.L, par, rank + step), tree_tag(epoch, round), sg);
        __syncthreads();
        const int mp = s_cnt;
        recv_total += mp;
        {
            char* peer = p.peers[rank + step];
            ChunkSrc src{gat_idx(peer, p.L, par), gat_val(peer, p.L, par), mp};
            const int room = chalf - m;
            pull_chunks(&src, 1, p.pull_tma != 0, &s_pull, pipe_it, [&](int, int idx, float val) {
                const bool ok = (unsigned)idx < (unsigned)n;
                bool first = false;
                if (ok) {
                    atomicAdd(p.g + idx, val);                  // own value + the sender's: two terms, order-independent
                    const unsigned bit = 1u << (idx & 31);
                    first = (atomicOr(p.bitmap + (idx >> 5), bit) & bit) == 0u;
                }
                const int pos = warp_append_active(&wc[2 * round], first);
                if (first && pos < room) candA[m + pos] = idx;
            });
        }
        grid_sync(&st->bar);
        const int nu = m + min(__ldcg(&wc[2 * round]), chalf - m);   // distinct indices of the union
        float thr2 = 0.f;
        if (nu > p.k) {
            Seg seg{p.g, nu, candA};
            thr2 = grid_kth_abs(&seg, 1, false, (uint32_t)p.k, st, s_hist, s_w, 0);
        }
        // winners -> my slot (the list of the next round) and the next union list; losers leave the map
        const int nur = (nu + 31) / 32 * 32;
        for (int c = gtid; c < nur; c += gthreads) {
            const bool in = c < nu;
            const int idx = in ? __ldcg(candA + c) : 0;
            const float v = in ? __ldcg(p.g + idx) : 0.f;
            const bool win = in && fabsf(v) >= thr2 && v != 0.f;
            const int pos = warp_append(&wc[2 * round + 1], win);
            if (win && pos < p.L.gcap && pos < chalf) { gi[pos] = idx; gv[pos] = v; candB[pos] = idx; }
            else if (in) {
                p.g[idx] = 0.f;
                atomicAnd(p.bitmap + (idx >> 5), ~(1u << (idx & 31)));
            }
        }
        grid_sync(&st->bar);
        m = min(__ldcg(&wc[2 * round + 1]), min(p.L.gcap, chalf));
        int* t = candA; candA = candB; candB = t;
    }

    // ---------------------------------------------------------------- broadcast of the surviving list (rank 0's slot)
    if (rank == 0 && blockIdx.x == 0 && tid < P)
        st_release_sys_u64(tree_mbox(p.peers[tid], p.L, par, 0), make_mail(tree_tag(epoch, kBcastRound), (uint32_t)m));
    // wipe my merge scratch: the bucket becomes all-zero again, the bitmap empty
    if (scattered) {
        for (int c = gtid; c < m; c += gthreads) {
            const int idx = __ldcg(candA + c);
            p.g[idx] = 0.f;
            p.bitmap[idx >> 5] = 0u;
        }
    }
    grid_sync(&st->bar);
    if (tid == 0) s_cnt = (int)wait_mailbox(tree_mbox(me, p.L, par, 0), tree_tag(epoch, kBcastRound), sg);
    __syncthreads();
    const int mf = s_cnt;
    {
        const float fP = (float)P;
        ChunkSrc src{gat_idx(p.peers[0], p.L, par), gat_val(p.peers[0], p.L, par), mf};
        int* flist = candA;                                      // local copy of the final indices (bitmap clean-up)
        pull_chunks(&src, 1, p.pull_tma != 0, &s_pull, pipe_it, [&](int, int idx, float val) {
            const bool ok = (unsigned)idx < (unsigned)n;
            if (ok) {
                p.g[idx] = val / fP;
                atomicOr(p.bitmap + (idx >> 5), 1u << (idx & 31));
            }
            const int pos = warp_append_active(&wc[2 * kBcastRound], ok);
            if (ok && pos < chalf) flist[pos] = idx;
        });
    }
    grid_sync(&st->bar);
    // put-back: my original picks that are not in the final list return to my residual (it was zeroed at selection)
    for (int e = gtid; e < m0; e += gthreads) {
        const int idx = p.sel_idx[e];
        if ((__ldcg(p.bitmap + (idx >> 5)) & (1u << (idx & 31))) == 0u) p.res[idx] += p.sel_val[e];
    }
    grid_sync(&st->bar);
    {
        const int nf = min(__ldcg(&wc[2 * kBcastRound]), chalf);
        for (int c = gtid; c < nf; c += gthreads) p.bitmap[__ldcg(candA + c) >> 5] = 0u;
    }
    grid_sync(&st->bar);
    if (blockIdx.x == 0) {
        for (int q = tid; q < 2 * kBcastRound + 2; q += kThreads) wc[q] = 0;
        if (tid == 0) {
            st->epoch = epoch;
            st->local_thr = thr;
            st->local_thr_used = thr;
            st->stat_local_count = m0;
            st->stat_global_count = mf;
            st->stat_recv_total = recv_total;
            st->stat_gather_total = mf;
            st->gather_cursor = 0;
            st->clip_sumsq = 0.0;
            const unsigned long long og = *reinterpret_cast<volatile unsigned long long*>(&st->cum_overflow_gather);
            st->stat_overflow_gather = (int)min(og - st->snap_overflow_gather, 0x7fffffffULL);
            st->snap_overflow_gather = og;
            st->stat_overflow_send = 0;
        }
    }
}

int gtopk_max_coop_grid(int device) {
    int sms = 0, per = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, gtopk_kernel, kThreads, 0);
    if (per < 1) per = 1;
    if (per > 2) per = 2;
    return sms * per;
}

cudaError_t launch_gtopk(const TreeParams& p, int grid, cudaStream_t stream) {
    void* args[] = {(void*)&p};
    return cudaLaunchCooperativeKernel((void*)gtopk_kernel, dim3(grid), dim3(kThreads), args, 0, stream);
}

}  // namespace okt
