// Shared declarations of the fused sparse-allreduce kernels: device-resident per-bucket state,
// launch parameters, symmetric-block layout.  Included by the .cu files (nvcc) and bindings.cpp (g++).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

#ifndef OKT_MAXP
#define OKT_MAXP 16
#endif

namespace okt {

constexpr int kThreads = 512;             // threads per CTA of the persistent kernels
constexpr int kWarps = kThreads / 32;
constexpr int kChunk = 1024;              // (idx,val) entries per pulled chunk (4 KB + 4 KB)
constexpr int kHistBins = 2048;           // 11-bit radix digit
constexpr int kMaxWarpsTotal = 16384;     // per-warp counters for the quantile cuts
constexpr int kGuardMax = 64;            // rungs of the over-selection ladder (fine guard rungs + coarse cap rungs)
constexpr int kGuardFineMax = 15;         // most fine (reference guard) rungs
constexpr int kCtasPerSm = 1;           // persistent kernels: one 512-thread CTA per SM (<= 128 registers/thread)
constexpr int kPackTile = 2;            // 128-bit vectors per thread per tile of the streaming pass
constexpr int kPackStages = 4;          // TMA ring depth of the streaming pass
constexpr int kPackSmemBytes = kPackStages * 2 * kPackTile * kThreads * 16;   // (grad + residual) tiles: 128 KB
constexpr int kScanStages = 2 * kPackStages;   // the region scan reuses the whole ring as 8 single-array stages
constexpr int kStrideGridMax = 132 * 8;  // grid-stride elementwise kernels: 8 CTAs of 256 threads on each of H100's 132 SMs

// one record per call, written by block 0 at the end of the fused kernel (observability: --trace, PROFILING)
constexpr int kTraceLen = 256;
struct TraceRec {
    uint32_t epoch;
    int local_count, global_count, recv_total, gather_total, overflow_send, overflow_gather, redo;
    float local_thr, global_thr;
    // phase durations in microseconds (globaltimer, block 0): exact-threshold/re-partition work, pack pass, wait for
    // the peers' reduce-scatter flags (= how far the slowest peer is behind), reduce, global selection, wait for the
    // allgather flags, final phase
    float us_local, us_pack, us_wait_rs, us_reduce, us_gselect, us_wait_ag, us_final;
    unsigned long long t_begin;                                   // globaltimer at kernel entry
};

// ---- device-resident, zero-initialised, one per bucket ---------------------------------------
struct OktState {
    unsigned long long bar;               // grid-barrier ticket counter
    unsigned int tick[4];                 // last-CTA-done tickets (pack / gselect / final / spare), self-resetting
    float local_thr;                      // threshold carried into the next call (after adaptation)
    float local_thr_used;                 // threshold actually applied in the last call (after guard)
    float global_thr;
    uint32_t epoch;                       // completed calls; the running call uses epoch + 1
    int edges[OKT_MAXP + 1];              // region edges, edges[0] = 0, edges[P] = n
    int send_cursor[OKT_MAXP];            // per-destination slot cursors (reset in-kernel)
    int gather_cursor;
    int cand_cursor;                      // first-touch candidate list of the reduce phase (reset in-kernel)
    int guard_counts[kGuardMax];          // selected elements whose HIGHEST passed ladder rung is j (suffix sums = #(|acc| > T_j))
    uint32_t sel_prefix;                  // radix-select running prefix / remaining rank
    uint32_t sel_krem;
    int tie_cursor;                       // TopkDSA: elements at |x| == threshold seen by the pack pass (reset by its publisher)
    int cuts[OKT_MAXP];
    // statistics of the last call (read lazily by the host; never on the hot path)
    int stat_local_count;
    int stat_global_count;
    int stat_recv_total;                  // entries pulled in the reduce phase
    int stat_gather_total;                // entries pulled in the final phase
    int stat_overflow_send;               // entries dropped in the LAST call because a send slot was full
    int stat_overflow_gather;             // same for the allgather slot
    int stat_redo;                        // pack passes repeated in the last call (overflow policy: raise threshold + redo)
    int stat_dense_fallback;              // 1 if the last call took TopkDSA's dense allgather path
    int stat_mode;
    int fault;                            // FaultCode of the first bounded wait that timed out (0 = healthy)
    float pack_thr;                       // threshold the pack pass finally selected with (after overflow redos)
    unsigned long long cum_overflow_send;     // cumulative (64-bit: a diverging run must not wrap the counter)
    unsigned long long cum_overflow_gather;
    unsigned long long cum_redo;
    unsigned long long snap_overflow_send;    // cumulative values at the end of the previous call
    unsigned long long snap_overflow_gather;
    unsigned long long snap_redo;
    unsigned long long t_phase[8];        // globaltimer stamps (block 0): 0 after local phase, 1 pack done, 2 reduce done,
                                          // 3 gselect done, 4 end, 5 kernel entry, 6 rs flags in, 7 ag flags in
    double gs_sum, gs_sumsq;              // Gaussiank moments
    double clip_sumsq;                    // norm_clip: sum of squares of the incoming gradient (reset at the end of the call)
    uint32_t hist[kHistBins];
    int wcounts[kMaxWarpsTotal];
    TraceRec trace[kTraceLen];            // per-call history ring (index = epoch % kTraceLen), see read_trace
};

// ---- byte offsets inside every rank's symmetric block (identical on all ranks) -----------------
//
// Send slots.  LOSSLESS layout (cap == 0, the default): ONE buffer of ~n entries in which destination d's slot
// starts at  slot_off(d) = align4(edges[d]) + 4 d  -- its capacity is at least the length of region d, i.e. at
// least the number of elements that can possibly be selected for d, so the exchange can never overflow, whatever
// the threshold (the reference gets the same guarantee from host-side Alltoall count handshakes,
// VGG/allreducer.py:708-726).  Sender and receiver derive the offsets from the region edges both already hold.
// BOUNDED layout (cap > 0): P slots of `cap` entries; overflow is handled by the in-kernel policy (raise the
// threshold and redo the pack pass; classic-residual schemes keep the unsent entries in the residual).
// The send slots are single-buffered: a peer has finished pulling call e's slots before it publishes its
// allgather flag of call e, which every rank waits for before it leaves call e.  The gather slots are
// double-buffered by call parity (the gather-type kernels have no second handshake).
struct SymmLayout {
    size_t rs_mbox;      // uint64 [2][MAXP]       reduce-scatter mailbox: (epoch<<32 | count) from src
    size_t rs_thr;       // float  [2][MAXP]       src's final local threshold (receiver-side filter)
    size_t ag_mbox;      // uint64 [2][MAXP]       allgather mailbox
    size_t cut_mbox;     // uint64 [2][MAXP]
    size_t cut_data;     // int32  [2][MAXP][MAXP]
    size_t done_mbox;    // uint64 [2][MAXP]       "finished reading your memory" flags (dense fallback, tree schemes)
    size_t tree_mbox;    // uint64 [2][MAXP]       gTopk: per-round list-ready flags (((epoch<<5)|round) << 32 | count)
    size_t scale_mbox;   // uint64 [2][MAXP]       loss scaling: src's non-finite flag of the bucket (epoch<<32 | flag)
    size_t send_idx;    // int32  [scap]          my selections, bucketed by destination region
    size_t send_val;     // float  [scap]
    size_t gat_idx;      // int32  [2][gcap]       my region's globally selected entries
    size_t gat_val;      // float  [2][gcap]
    size_t total;
    int cap;             // bounded per-destination capacity; 0 = lossless layout
    int scap;            // entries in the send buffer
    int gcap;
};

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

inline SymmLayout make_layout(int P, int n, int cap, int gcap) {
    SymmLayout L;
    size_t o = 0;
    L.rs_mbox = o;  o += sizeof(uint64_t) * 2 * OKT_MAXP;
    L.rs_thr = o;   o += sizeof(float) * 2 * OKT_MAXP;
    L.ag_mbox = o;  o += sizeof(uint64_t) * 2 * OKT_MAXP;
    L.cut_mbox = o; o += sizeof(uint64_t) * 2 * OKT_MAXP;
    L.cut_data = o; o += sizeof(int) * 2 * OKT_MAXP * OKT_MAXP;
    L.done_mbox = o; o += sizeof(uint64_t) * 2 * OKT_MAXP;
    L.tree_mbox = o; o += sizeof(uint64_t) * 2 * OKT_MAXP;
    L.scale_mbox = o; o += sizeof(uint64_t) * 2 * OKT_MAXP;
    o = align_up(o, 1024);
    const size_t scap = cap > 0 ? (size_t)P * cap : align_up((size_t)n, 4) + 4 * (size_t)OKT_MAXP + 1024;
    L.send_idx = o; o += sizeof(int) * scap;   o = align_up(o, 1024);
    L.send_val = o; o += sizeof(float) * scap; o = align_up(o, 1024);
    L.gat_idx = o;  o += sizeof(int) * 2 * (size_t)gcap;      o = align_up(o, 1024);
    L.gat_val = o;  o += sizeof(float) * 2 * (size_t)gcap;    o = align_up(o, 1024);
    L.total = o;
    L.cap = cap;
    L.scap = (int)scap;
    L.gcap = gcap;
    return L;
}

enum Phase : int {
    PH_LOCAL = 0,      // two-pass iterations: acc -> residual, exact k-th |acc| or guard, re-partition
    PH_PACK = 1,       // (accumulate +) select + pack per destination region
    PH_PUBLISH_RS = 2, // finalise threshold, publish counts to the region owners
    PH_REDUCE = 3,     // pull every source's slot for my region, scatter-add
    PH_GSELECT = 4,    // global selection on my region, pack the allgather slot
    PH_PUBLISH_AG = 5,
    PH_FINAL = 6,      // pull all slots, (exact top-k,) scatter result, clear residual, adapt
    PH_END = 7
};

enum ResidualMode : int { RES_OKTOPK = 0, RES_LOCAL_GT = 1, RES_LOCAL_GE = 2 };
enum GlobalMode : int { GLB_THRESHOLD = 0, GLB_EXACT_TOPK = 1, GLB_ALL_NONZERO = 2 };

// Where the gradient that the call reduces comes from: an ordered table of (source, bucket element offset, length)
// segments.  Either ONE segment that is the bucket itself (the gradient was landed there; the pack pass then clears
// the bucket for the reduce / final phases), or the tensors autograd produced, read in place (the bucket must be
// all-zero on entry and is not cleared).  Bucket elements that no segment covers read as zero.  Offsets are multiples
// of 4 elements and sources 16-byte aligned; a length need not be.  Passed by value: a captured CUDA graph keeps the
// addresses of its capture.  Sized for the largest bucket of the bench workloads (BERT-base: 132 tensors) with the
// whole OktParams under the classic 4 KB kernel-parameter limit.
constexpr int kSrcSegMax = 160;
// Early pack (see oktopk_segment_kernel): a threshold-reuse call whose bucket was partly packed during backward by segment
// launches gets the vector ranges that are still to be packed; a segment launch gets its one range.
constexpr int kPackRangeMax = 32;
constexpr int kSegStages = 2;           // TMA ring depth of a segment launch (64 KB of shared memory)
constexpr int kSegTiles = 4;            // tiles per CTA of a segment launch: short-lived CTAs, no cooperative grid ...

struct OktParams {
    float* g;            // gradient bucket (result written in place)
    float* res;          // residual / accumulator
    OktState* st;
    int* cand;           // local scratch: region-local indices that received a contribution (capacity ccap)
    int ccap;
    int cand_mode;       // 1: first-touch candidate list (low density), 0: region scan (high density)
    float prefilter;     // exact iterations: radix-select only elements above prefilter * carried threshold (0 = all)
    char* peers[OKT_MAXP];   // every rank's symmetric block as mapped into this process
    float* peer_g[OKT_MAXP]; // every rank's gradient bucket (null when g is not the symmetric bucket): dense fallback
    SymmLayout L;
    int n, P, rank, k;
    int exact_local, repartition, uniform_regions;
    int residual_mode, global_mode;
    int deterministic, pull_tma;
    int phase_begin, phase_end;
    // Over-selection ladder T_0 = thr, T_j = T_{j-1} * (j <= guard_loops ? guard_factor : cap_factor).  The reference's
    // guard (VGG/compression.py:392-404) climbs the first guard_loops rungs while the count exceeds guard_limit; the cap
    // (cap_limit > 0, an extension of this library: the counts of ALL rungs come out of the same streaming pass for free) keeps
    // climbing the coarse rungs while the count exceeds cap_limit, so a stale threshold can never ship more than
    // cap_limit entries per rank.
    int guard_loops, guard_limit;
    float guard_factor;
    int cap_limit, cap_rungs;
    float cap_factor;
    double l_low_cnt, l_high_cnt;       // local adaptation bounds, already multiplied by k
    float l_factor;
    double g_low_cnt, g_high_cnt;
    float g_inc, g_dec;
    unsigned long long timeout_ns;      // bound of every cross-GPU wait (0 = unbounded)
    int max_redo;                       // bounded slots: how many times the pack pass may be repeated with a raised threshold
    float redo_factor;                  // first raise; squared after every further attempt
    int dense_nnz_limit;                // GLB_ALL_NONZERO (TopkDSA): total gathered nnz >= this => dense allgather path (0 = never)
    int* host_fault;                    // mapped pinned int: fault code mirrored to the host without a sync (may be null)
    const int* skip;                    // loss scaling: the bucket verdict of unscale_check (null = scaling off); set = return
    int trace;                          // 1: write a TraceRec per call
    int zero_g;                         // 1: the pack pass clears the bucket (the gradient was landed in it)
    int nsrc;                           // gradient-source segments (see kSrcSegMax)
    int src_off[kSrcSegMax];
    int src_len[kSrcSegMax];
    const float* src[kSrcSegMax];
    // 0: the pack pass covers the whole bucket.  1: it covers only the float4 ranges [pk_lo[r], pk_hi[r]), r < pk_nr
    // (pk_nr may be 0); the rest was packed by segment launches of this call.  Ignored by two-pass calls.
    int pk_mode, pk_nr;
    int pk_lo[kPackRangeMax];
    int pk_hi[kPackRangeMax];
};
static_assert(sizeof(OktParams) <= 4096, "OktParams must fit the 4 KB kernel-parameter limit");

// ---- gather-type schemes (TopkAopt / Gaussiank / TopkA): select -> own slot -> everyone adds all ---
enum GatherSelect : int { GS_THRESHOLD_REUSE = 0, GS_GAUSSIAN = 1, GS_EXACT_TOPK = 2 };

struct GatherParams {
    float* g;
    float* res;
    OktState* st;
    char* peers[OKT_MAXP];
    SymmLayout L;
    int n, P, rank, k;
    int select_mode;          // GatherSelect
    int exact_now;            // GS_THRESHOLD_REUSE: recompute the exact threshold in this call
    int gauss_mode;           // 0 vgg, 1 lstm, 2 bert
    int gauss_loops;
    float gauss_factor;
    float density;
    int pull_tma;
    unsigned long long timeout_ns;
    int reselect;             // TopkA2: global top-k re-selection of the gathered union + put-back of the losers
    float clip_max_norm;      // > 0: scale the incoming gradient so that its L2 norm is at most this (norm_clip)
    unsigned* bitmap;         // n/32 words, all-zero between calls (exact first-touch detection for the union list)
    int* cand;                // union candidate list (capacity ccap)
    int ccap;
    int* host_fault;
    const int* skip;          // loss scaling: bucket verdict (null = scaling off)
};

// ---- gTopk: log2(P) rounds of pairwise list merges toward rank 0, then a broadcast ------------------
struct TreeParams {
    float* g;
    float* res;
    OktState* st;
    char* peers[OKT_MAXP];
    SymmLayout L;
    int n, P, rank, k;
    int pull_tma;
    unsigned long long timeout_ns;
    float clip_max_norm;
    unsigned* bitmap;         // n/32 words, all-zero between calls
    int* cand;                // two union lists of ccap/2 entries each (ping-pong across rounds)
    int ccap;
    int* sel_idx;             // my original picks (for the put-back of the non-survivors), capacity selcap
    float* sel_val;
    int selcap;
    int* host_fault;
    const int* skip;          // loss scaling: bucket verdict (null = scaling off)
};

// ---- dense allreduce over peer memory -------------------------------------------------------------
struct DenseParams {
    float* bufs[OKT_MAXP];    // every rank's gradient bucket (symmetric allocation)
    uint64_t* flags[OKT_MAXP];  // every rank's flag block: uint64 [2][grid][MAXP]
    unsigned long long* epoch;  // local, one counter per CTA
    int n, P, rank;
    float scale;              // 1/P
    int* fault;               // bucket fault word (OktState::fault)
    unsigned long long timeout_ns;
    float* mc;                // multicast (NVLS) mapping of the bucket, or null: switch-side reduction with multimem.*
    int* host_fault;
    const int* skip;          // loss scaling: bucket verdict (null = scaling off)
};

// ---- host-callable launchers (implemented in the .cu files) ----------------------------------------
int okt_max_coop_grid(int device);
cudaError_t launch_oktopk(const OktParams& p, int grid, cudaStream_t stream);
// threshold-reuse pack of the ranges p.pk_lo[r] .. p.pk_hi[r], r < p.pk_nr, ahead of the call (no publish), on one
// CTA per kSegTiles tiles but at most max_ctas
cudaError_t launch_oktopk_segment(const OktParams& p, int max_ctas, cudaStream_t stream);
cudaError_t launch_gather_scheme(const GatherParams& p, int grid, cudaStream_t stream);
cudaError_t launch_gtopk(const TreeParams& p, int grid, cudaStream_t stream);
int gtopk_max_coop_grid(int device);
int gather_max_coop_grid(int device);
cudaError_t launch_dense_allreduce(const DenseParams& p, int grid, cudaStream_t stream);
cudaError_t launch_kth_abs(const float* x, int n, int k, OktState* st, float* out_thr, int grid, cudaStream_t stream);
// fused optimizer updates: scal -> the step's scalars in device memory ({lr} for SGD and BertAdam); skip -> the step
// verdict of loss scaling (null = off): when set, p / m / v are left alone and only the gradient is cleared
cudaError_t launch_fused_sgd(float* p, float* g, float* mom, int n, float momentum, float dampening, float weight_decay,
                             int nesterov, int first_step, int zero_grad, const float* scal, const int* fault,
                             const int* skip, cudaStream_t stream);
// Early SGD update (sgd_ahead_kernel / fused_sgd_tail_kernel in optim.cu).  SgdRanges: float4 vector ranges [lo, hi) of a
// (bucket, param group) slice, in slice order, at most kPackRangeMax of them; SgdHyper: torch.optim.SGD's group options.
struct SgdRanges {
    int nr;
    int lo[kPackRangeMax];
    int hi[kPackRangeMax];
};
struct SgdHyper {
    float momentum, dampening, wd;
    int nesterov, first;
};
// the zero-gradient update over `r` in place, old p / m to the stash sp / sm (sm: only with momentum), on at most
// max_ctas CTAs; never on a first step
cudaError_t launch_sgd_ahead(float* p, float* mom, float* sp, float* sm, const SgdRanges& r, const SgdHyper& h,
                             int max_ctas, const float* scal, cudaStream_t stream);
// the rest of a step whose `ahead` ranges had launch_sgd_ahead: there, every vector with a written gradient is
// recomputed from the stash (fault or skip: every vector is restored from it); `dense` and the scalar tail of the
// n-element slice take fused_sgd's update
cudaError_t launch_fused_sgd_tail(float* p, float* g, float* mom, const float* sp, const float* sm, int n,
                                  const SgdRanges& ahead, const SgdRanges& dense, const SgdHyper& h, int zero_grad,
                                  const float* scal, const int* fault, const int* skip, cudaStream_t stream);
cudaError_t launch_fused_bert_adam(float* p, float* g, float* m, float* v, int n, float b1, float b2, float eps,
                                   float weight_decay, int zero_grad, const float* scal, const int* fault,
                                   const int* skip, cudaStream_t stream);
// torch.optim.Adam / AdamW update; scal -> {1 - lr*wd, -lr / (1 - beta1^t), sqrt(1 - beta2^t)} of this step
cudaError_t launch_fused_adam(float* p, float* g, float* m, float* v, int n, double beta1, double beta2, float eps,
                              float weight_decay, int decoupled, int zero_grad, const float* scal, const int* fault,
                              const int* skip, cudaStream_t stream);

// ---- dynamic loss scaling (csrc/scale.cu) ------------------------------------------------------------
// One per optimizer, in device memory.  found_inf is the step verdict: the OR of the bucket verdicts of the step.
struct LossScaleDev {
    float scale;
    float inv_scale;                  // fp32 of 1 / (double)scale, as torch.amp.GradScaler computes it
    int growth_tracker;
    int found_inf;
    long long skipped;                // steps skipped so far
    long long adam_step;              // steps applied so far: the bias-correction step of the wrapped Adam
};
// One per bucket, device-local: the last-CTA ticket and epoch of unscale_check and the agreed bucket verdict.
struct ScaleSync {
    int flag;                         // OR of the CTAs' local non-finite flags (reset by the last CTA)
    unsigned int ticket;
    unsigned int epoch;               // completed checks; the mailbox words carry epoch + 1
    int verdict;                      // 1: some rank saw a non-finite value, every rank skips the bucket's reduction
};
constexpr int kScaleThreads = 256;
constexpr int kScalePerCta = 8192;    // floats per CTA
struct ScaleParams {
    LossScaleDev* ls;
    ScaleSync* sync;
    int* fault;                       // bucket fault word (OktState::fault)
    int* host_fault;
    char* peers[OKT_MAXP];            // every rank's symmetric comm block (the scale mailboxes are at L.scale_mbox)
    size_t mbox_off;
    int P, rank;
    unsigned long long timeout_ns;
    int nseg;                         // the source table of the direct Ok-Topk path, or one segment = the landed bucket
    int len[kSrcSegMax];
    int blk_begin[kSrcSegMax + 1];    // first CTA of segment t (CTAs dealt proportionally to length)
    float* src[kSrcSegMax];
};
static_assert(sizeof(ScaleParams) <= 4096, "ScaleParams must fit the 4 KB kernel-parameter limit");
cudaError_t launch_unscale_check(const ScaleParams& p, cudaStream_t stream);
// end of step: growth / backoff of torch._amp_update_scale_, new inv_scale, skipped-step and Adam step counts, verdict
// cleared.  adam_scalars (start of step): the wrapped Adam's per-group scalars for step adam_step + 1, in double, from
// hyper = {lr, weight_decay, beta1, beta2} per group into scal (3 floats per group).
cudaError_t launch_scale_update(LossScaleDev* ls, double growth_factor, double backoff_factor, int growth_interval,
                                cudaStream_t stream);
cudaError_t launch_adam_scalars(const LossScaleDev* ls, const double* hyper, float* scal, int groups, cudaStream_t stream);
// dense switch carry-over under loss scaling: g += res; res = 0 -- unless the bucket verdict is set
cudaError_t launch_carry_residual(float* g, float* res, int n, const int* skip, cudaStream_t stream);
// multi-tensor gradient landing: copy up to kLandMax autograd-produced gradient tensors into the flat bucket in ONE launch
constexpr int kLandMax = 96;
struct LandParams {
    const float* src[kLandMax];
    long long dst_off[kLandMax];      // element offset inside the bucket
    int numel[kLandMax];
    int blk_begin[kLandMax + 1];      // first CTA of tensor t (CTAs are dealt proportionally to size)
    int count;
};
cudaError_t launch_land(const LandParams& lp, float* bucket, cudaStream_t stream);
// The storage type of the fp32 / bf16 / fp16 kernels' tensors: the code ops/ext.DTYPE_CODE passes, made a type by
// csrc/elem.cuh's with_dtype.
enum class Dtype : int { kF32 = 0, kBF16 = 1, kF16 = 2 };
// fused (conv-bias +) BatchNorm + ReLU [+ 2x2 max-pool when W > 0], channels_last, training mode (csrc/bnrelu.cu):
// one cooperative kernel per pass.  `slot` names the call site's grid hand-off counters; max_ctas > 0 caps the grid.
// x, y, dy and dx are of type `dtype`; parameters, statistics, partials and dgamma / dbeta are fp32.  A non-null `res`
// (same type and [M, C] layout as x; W == 0 and relu only) makes it  y = relu(bn(x) + res)  and the backward writes the
// residual's gradient `dres`.
int bn_tile_rows(int M, int C);
bool bn_sliced(int M, int C, int W);      // the channel-sliced kernels run (given max_ctas <= 0): no `partial`, no hand-off
cudaError_t launch_bn_forward(const void* x, void* y, unsigned char* arg, float* partial, const float* gamma, const float* beta,
                              const float* cbias, float* save_mean, float* save_invstd, float* rmean, float* rvar, long long* nbt,
                              float momentum, float eps, int relu, int M, int C, int W, int slot, int max_ctas, Dtype dtype,
                              cudaStream_t stream, const void* res = nullptr);
cudaError_t launch_bn_backward(const void* x, const void* dy, const unsigned char* arg, void* dx, float* partial,
                               const float* gamma, const float* beta, const float* save_mean, const float* save_invstd,
                               float* dgamma, float* dbeta, int relu, int M, int C, int W, int slot, int max_ctas, Dtype dtype,
                               cudaStream_t stream, const void* res = nullptr, void* dres = nullptr);
cudaError_t launch_maxpool2_fwd(const float* x, float* y, unsigned char* arg, int N, int H, int W, int C, cudaStream_t stream);
cudaError_t launch_maxpool2_bwd(const float* dy, const unsigned char* arg, float* dx, int N, int H, int W, int C,
                                cudaStream_t stream);
// fused  y = LayerNorm(x + dropout(a))  over rows of H elements (csrc/layernorm.cu): x, y, dx, gamma, beta, dgamma,
// dbeta, mean and rstd are fp32; a and da are of type `a_dtype` (a Dtype).  keep_thr >= 2^32 turns the dropout
// off (seed may then be null).  The backward pass writes its [ln_bwd_grid(R), 2H] column partials to `partial`.
bool ln_supported_h(int H);
int ln_bwd_grid(int R);
cudaError_t launch_ln_forward(const float* x, const void* a, float* y, const float* gamma, const float* beta, float* mean,
                              float* rstd, const unsigned long long* seed, int R, int H, long long keep_thr, float scale,
                              float eps, Dtype a_dtype, cudaStream_t stream);
cudaError_t launch_ln_backward(const float* x, const void* a, const float* dy, const float* gamma, const float* mean,
                               const float* rstd, const unsigned long long* seed, float* dx, void* da, float* partial,
                               float* dgamma, float* dbeta, int R, int H, long long keep_thr, float scale, Dtype a_dtype,
                               cudaStream_t stream);
// dgamma | dbeta = the sum of the G rows of partial [G, 2H], in a fixed order (the last launch of launch_ln_backward)
cudaError_t launch_ln_dgb(const float* partial, int G, int H, float* dgamma, float* dbeta, cudaStream_t stream);
// fused embedding sum + LayerNorm + dropout of BERT's input block (csrc/embedding.cu): ids and tt [R] int64, token r at
// position r % S; word [nv, H], pos [np, H], typ [nt, H], gamma, beta, y, stats ([mean; rstd], 2R) and de [R, H] fp32;
// ovf one int64 that counts ids outside [0, nv) and types outside [0, nt) (or null).  Needs emb_supported(R, S, H, np).
// The backward pass takes partial of ln_bwd_grid(R) 2H floats and writes every element of dword, dpos and dtyp.  One
// launch forward, three backward.
bool emb_supported(int R, int S, int H, int np);
cudaError_t launch_emb_forward(const long long* ids, const long long* tt, const float* word, const float* pos,
                               const float* typ, const float* gamma, const float* beta, float* y, float* stats,
                               long long* ovf, const unsigned long long* seed, int R, int S, int H, int nv, int nt,
                               long long keep_thr, float scale, float eps, cudaStream_t stream);
cudaError_t launch_emb_backward(const long long* ids, const long long* tt, const float* word, const float* pos,
                                const float* typ, const float* gamma, const float* stats, const float* dy,
                                const unsigned long long* seed, float* de, float* partial, float* dgamma,
                                float* dbeta, float* dword, float* dpos, float* dtyp, int R, int S, int H, int nv, int np,
                                int nt, long long keep_thr, float scale, cudaStream_t stream);
// fused softmax cross-entropy, mean over the rows whose target is not ignore_index (csrc/xent.cu): x and dx [R, V] of
// type `dtype` (a Dtype), 16-byte aligned; t [R] int64; lse [R + 1] fp32 (per-row log-sum-exp, then n);
// rowloss [R] fp32 scratch; loss and g one fp32 each.  Two launches forward, one backward.
cudaError_t launch_xent_forward(const void* x, const long long* t, float* lse, float* rowloss, float* loss, int R,
                                long long V, long long ignore_index, Dtype dtype, cudaStream_t stream);
cudaError_t launch_xent_backward(const void* x, const long long* t, const float* lse, const float* g, void* dx, int R,
                                 long long V, long long ignore_index, Dtype dtype, cudaStream_t stream);
// fused softmax + CTC loss, blank 0, summed, zero_infinity (csrc/ctc.cu): x and dx [T, N, C] of type `dtype` (a Dtype);
// targets [nt] int64 (targets64 = 1) or int32; tn, ln [N] int32 input / target lengths; ws ctc_workspace_floats(T, N, nt)
// fp32, written by the forward pass and read by the backward pass; ab ctc_ab_floats(T, N, nt) fp32 scratch of the
// backward pass; loss and g one fp32 each.  Needs ctc_supported(T, N, C, nt).  Two launches forward, one backward.
bool ctc_supported(int T, int N, int C, long long nt);
long long ctc_workspace_floats(int T, int N, long long nt);
long long ctc_ab_floats(int T, int N, long long nt);
cudaError_t launch_ctc_forward(const void* x, const void* targets, int targets64, const int* tn, const int* ln, float* ws,
                               float* loss, int T, int N, int C, long long nt, Dtype dtype, cudaStream_t stream);
cudaError_t launch_ctc_backward(const void* x, const void* targets, int targets64, const int* tn, const int* ln,
                                const float* ws, float* ab, const float* g, void* dx, int T, int N, int C, long long nt,
                                Dtype dtype, cudaStream_t stream);
// batch-norm over the frames of the longest utterance, training mode (csrc/frame_bn.cu): conv = 1 takes x [N, C, F, Tb]
// and applies the masked Hardtanh(0, 20) of DeepSpeech's conv blocks; conv = 0 takes x [Tb, N, C] (F ignored).  x, y,
// dy and dx of type `dtype` (a Dtype); len [N] int32 on the device; gamma, beta, mean, rstd, rmean, rvar, dgamma and
// dbeta [C] fp32; nbt one int64 (num_batches_tracked) or null.  Needs frame_bn_supported.  One launch each.
bool frame_bn_supported(int conv, int N, int C, int F, int Tb);
cudaError_t launch_frame_bn_forward(int conv, const void* x, const int* len, const float* gamma, const float* beta,
                                    void* y, float* mean, float* rstd, float* rmean, float* rvar, long long* nbt,
                                    int N, int C, int F, int Tb, float eps, float momentum, Dtype dtype,
                                    cudaStream_t stream);
cudaError_t launch_frame_bn_backward(int conv, const void* x, const void* dy, const int* len, const float* gamma,
                                     const float* beta, const float* mean, const float* rstd, void* dx, float* dgamma,
                                     float* dbeta, int N, int C, int F, int Tb, Dtype dtype, cudaStream_t stream);
// fixed-capacity gather of the labelled masked-LM rows (csrc/mlm_gather.cu): labels and tgt int64, rows [M] and slot
// [R] int32, count one int64, overflow one int64 that accumulates max(count - M, 0) (or null); x [R, H] and out [M, H],
// dout [M, H] and dx [R, H] of type `dtype` (a Dtype).  One launch each.
cudaError_t launch_mlm_select(const long long* labels, int R, long long ignore_index, int M, int* rows, long long* tgt,
                              int* slot, long long* count, long long* overflow, cudaStream_t stream);
cudaError_t launch_mlm_gather(const void* x, const int* rows, void* out, int M, int H, Dtype dtype, cudaStream_t stream);
cudaError_t launch_mlm_scatter(const void* dout, const int* slot, void* dx, int R, int H, Dtype dtype,
                               cudaStream_t stream);
// persistent LSTM recurrence, time-major (csrc/lstm.cu): one cooperative launch per pass, ceil(H / u) CTAs of u hidden
// units each per direction, `rows` batch rows of the per-step operand staged in shared memory at a time.  gx [T, N, 4H]
// (the input projection with both biases), whh [H4, H] row-major, len [N] int32 in [1, T]; y, cs [T, N, H], gates and dg
// [T, N, 4H].  gx, whh, y, dy and dg are of type `dtype` (a Dtype); gates and cs are fp32.  `bar` is a zeroed
// 64-bit grid-barrier counter.  whh, y and dg aligned to four elements (16 bytes in fp32, 8 in bf16 / fp16), H % 4 == 0.
// whh_rev non-null runs a bidirectional layer, whh_rev being the reverse direction's W_hh: gx, y, cs, gates and dg are
// then [2, T, N, .] (forward direction first), dy stays [T, N, H] (the same for both), and bar holds two counters.
cudaError_t launch_lstm_forward(const void* gx, const void* whh, const void* whh_rev, const int* len, void* y,
                                float* gates, float* cs, unsigned long long* bar, int T, int N, int H, int u, int rows,
                                cudaStream_t stream, Dtype dtype);
cudaError_t launch_lstm_backward(const void* dy, const float* gates, const float* cs, const void* whh,
                                 const void* whh_rev, const int* len, void* dg, unsigned long long* bar, int T, int N,
                                 int H, int u, int rows, cudaStream_t stream, Dtype dtype);
// one layer of a stacked LSTM from an initial state, every row of length T, the step product on the tensor cores
// (csrc/lstm.cu).  gx, whh, y, dy, dg as above; h0 and dhn [N, H] of type `dtype`, c0, dcn and dc0 [N, H] fp32; dhn and
// dcn may be null (zero).  whh, h0, y and dg aligned to four elements, H % 4 == 0.  bf16 / fp16 stage `rows` batch rows
// at a time and keep all of the CTA's W_hh slice on chip (r_on and kc are ignored).  fp32 (N <= 64): the CTA keeps its
// first r_on weight rows on chip (forward: of its 4u gate rows, at most 128; backward: of its u columns) and streams
// the rest from L2 every step, staging all N rows kc columns at a time (kc % 8 == 0); `rows` is only checked; the
// backward pass's whh is W_hh^T [H, 4H].
cudaError_t launch_lstm_seq_forward(const void* gx, const void* whh, const void* h0, const float* c0, void* y,
                                    float* gates, float* cs, unsigned long long* bar, int T, int N, int H, int u,
                                    int rows, int r_on, int kc, cudaStream_t stream, Dtype dtype);
cudaError_t launch_lstm_seq_backward(const void* dy, const float* gates, const float* cs, const void* whh,
                                     const float* c0, const void* dhn, const float* dcn, void* dg, float* dc0,
                                     unsigned long long* bar, int T, int N, int H, int u, int rows, int r_on, int kc,
                                     cudaStream_t stream, Dtype dtype);
// fused self-attention, head dim 64 (csrc/attention.cu): qkv and dqkv [B, S, 3 H 64], out and dout [B, S, H 64], all of
// type `dtype` (a Dtype), 16-byte aligned; mask [B, S] fp32 additive key bias or null; lse and delta [B, H, S]
// fp32 (lse written by the forward pass, delta scratch of the backward pass).  keep_thr >= 2^32 turns the dropout off
// (seed may then be null); `scale` is the kept elements' 1 / (1 - p).  One launch forward, two backward.
bool attn_supported(int B, int S, int H);
cudaError_t launch_attn_forward(const void* qkv, const float* mask, const unsigned long long* seed, void* out, float* lse,
                                int B, int S, int H, long long keep_thr, float scale, Dtype dtype, cudaStream_t stream);
cudaError_t launch_attn_backward(const void* qkv, const void* out, const void* dout, const float* mask,
                                 const unsigned long long* seed, const float* lse, float* delta, void* dqkv, int B, int S,
                                 int H, long long keep_thr, float scale, Dtype dtype, cudaStream_t stream);
cudaError_t launch_momentum_correct(float* g, float* buf, int n, float momentum, cudaStream_t stream);
cudaError_t launch_l2norm_sq(const float* x, int n, float* out, cudaStream_t stream);
cudaError_t launch_scale(float* x, int n, const float* norm_sq, float max_norm, cudaStream_t stream);

}  // namespace okt
