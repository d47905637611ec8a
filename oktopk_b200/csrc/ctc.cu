// Fused softmax + CTC loss (blank 0, summed over the utterances, zero_infinity), forward and backward:
//
//   loss = sum over n of ctc_n,   ctc_n = -log p(l_n | x[:Tn, n])  under softmax(x[t, n, :]) over the C classes
//   dx[t, n, c] = (softmax(x)[t, n, c] - posterior_n(t, c)) . g   for t < Tn,   0 for t >= Tn
//
// with posterior_n(t, c) the probability that an alignment of l_n emits class c at frame t.  x is [T, N, C] (time-major,
// contiguous), targets are the labels of all utterances concatenated (int32 or int64), Tn and Ln int32 on the device.
// This is what DeepSpeech's stock loss computes as ctc_loss(log_softmax(x).float(), ...) plus both backward passes,
// without the [T, N, C] log-softmax tensor, the widening copy or the host copies of the lengths.
//
// Sizes: the launch geometry and the workspace depend on T, N, C and targets.numel() = nt only, never on a device value,
// so the op is safe inside a CUDA graph.  One CTA of kCtcThreads per utterance.  Each utterance's extended label
// sequence has S = 2 Ln + 1 states (blank, l1, blank, ..., lLn, blank); thread i holds states [i K, i K + K) in
// registers, K = kCtcK.  An utterance's offsets (Σ_{m<n} Ln into the targets, Σ_{m<n} S_m into the α workspace) are
// prefix sums of the lengths, taken by its CTA.  sum_n S_n = 2 nt + N, so the workspace is
//   nll [N] | lse [T, N] | α [T (2 nt + N)]   fp32,
// utterance n's α block being [T, S_n] at T Σ_{m<n} S_m.  nt <= kCtcMaxTargets keeps every S within the CTA's states.
//
// Forward (ctc_fwd_kernel + ctc_reduce_kernel).  First every warp takes frames t < Tn in turn and writes the frame's
// log-sum-exp over C to lse.  Then the α recursion runs serially over t.  An utterance whose S fits in one warp (S <= 32 K,
// so Ln <= 63) runs it on warp 0 alone with shuffles and no barrier; a longer one runs it on its first ceil(S / 32 K) warps
// with one named barrier per step, the two α values at each warp boundary passed through shared memory (double
// buffered).  Each step's emissions x[t, n, l_s] - lse[t] are loaded one step ahead.  α goes to the workspace, and the
// utterance's log-likelihood is log(α[Tn-1][S-1] + α[Tn-1][S-2]).  A one-warp kernel then adds the utterances' losses
// (an +inf one as 0) in a fixed order: lanes in utterance order, then a fixed shuffle tree.
//
// Backward (ctc_bwd_kernel).  The β recursion runs backwards over t with the same thread layout; at each t the CTA
// writes α[t][s] + β[t][s] (logs) to `ab`, laid out as α, so that the forward's workspace stays intact.  After a barrier every warp takes frames in turn: the blank class's
// log-sum over the even states is reduced across the warp in a fixed tree, each label class's over its odd states in
// ascending order along a per-class list built once per utterance, and the frame's C gradient entries are written.
// The posterior of class c at frame t is exp(A_c - lp_c - Z_t), A_c that log-sum, lp_c the log-softmax, and
// Z_t = log sum_c exp(A_c - lp_c) the frame's own total (which is log p(l | x) in exact arithmetic): the fp32 error
// that α and β carry in common over a long recursion cancels, where dividing by the forward's p(l | x) would keep it.
//
// Numerics: log-sum-exps, α, β and all sums are fp32 (expf / logf, no fast-math), x widened exactly; dx is computed in fp32
// and rounded once to x's type, to nearest even, an fp16 gradient past 65504 becoming inf.  g (the loss's incoming
// gradient, which carries a loss scale) is read from device memory.  No atomics: results are bitwise reproducible.
//
// Edge cases (per utterance, the others unaffected, except after a bad target length):
//   - Ln = 0: the all-blank alignment, ctc = -sum_t log softmax(x)[t, 0].
//   - Infeasible (Ln plus its repeated neighbours > Tn): ctc = +inf; zero_infinity makes its loss and gradient 0.
//   - Tn = 0: ctc = 0 if Ln = 0, else +inf (then 0), and no gradient, as torch.
//   - A label outside [0, C) or Tn outside [0, T]: ctc = NaN and a NaN gradient on frames t < Tn (every frame when Tn
//     itself is out of range).
//   - A negative Ln at utterance m, or one that takes sum_{n<=m} Ln past nt: the target offsets of m and of every later
//     utterance are undefined, so all of them are NaN as above; the utterances before m are unaffected.  Torch
//     device-asserts or raises on these and on the previous case instead.
//   - Frames t >= Tn are never read; their gradient is exactly 0 even if they hold inf or NaN (stock log_softmax's
//     backward makes it NaN there).
//   - A -inf logit within an utterance's frames: the frame's log-sum-exp skips it, so the loss stays finite, as torch's;
//     the gradient is NaN in every class of each frame holding one, as torch's is.  A NaN or +inf logit there makes
//     the loss and gradient NaN (not zeroed: only a +inf ctc is).
#include "common.cuh"
#include "elem.cuh"
#include "oktopk.cuh"

namespace okt {

constexpr int kCtcK = 4;                                     // α / β states per thread
constexpr int kCtcThreads = 1024;
constexpr int kCtcWarps = kCtcThreads / 32;
constexpr int kCtcMaxStates = kCtcThreads * kCtcK;           // 4096
constexpr long long kCtcMaxTargets = (kCtcMaxStates - 1) / 2; // 2047: S = 2 Ln + 1 <= 2 nt + 1 <= 4095
constexpr int kCtcMaxC = 128;

__device__ __forceinline__ long long ctc_label(const void* t, int t64, long long i) {
    return t64 ? __ldg(static_cast<const long long*>(t) + i) : (long long)__ldg(static_cast<const int*>(t) + i);
}

// log(e^a + e^b + e^c).  All -inf stays -inf; a NaN argument gives NaN (fmaxf alone would drop it).
__device__ __forceinline__ float ctc_lse3(float a, float b, float c) {
    const float m = fmaxf(fmaxf(a, b), c);
    if (m == -INFINITY) return a + b + c;
    return m + logf(expf(a - m) + expf(b - m) + expf(c - m));
}

// Online log-sum-exp pair (m, s): the running max and the sum of exp(v - m); -inf adds 0, a NaN reaches s.
__device__ __forceinline__ void ctc_acc(float& m, float& s, float v) {
    const float mn = fmaxf(m, v);
    s = s * (m == mn ? 1.f : expf(m - mn)) + (v == -INFINITY ? 0.f : expf(v - mn));
    m = mn;
}
__device__ __forceinline__ void ctc_combine(float& m, float& s, float m2, float s2) {
    const float mn = fmaxf(m, m2);
    s = s * (m == mn ? 1.f : expf(m - mn)) + s2 * (m2 == mn ? 1.f : expf(m2 - mn));
    m = mn;
}

__device__ __forceinline__ void ctc_bar(int nthreads) { asm volatile("bar.sync 1, %0;" ::"r"(nthreads) : "memory"); }

// The utterance's lengths, target offset and validity, read by warp 0 into shared memory.
struct CtcUtt {
    long long toff;
    int Tn, Ln, ok;
};

__device__ __forceinline__ void ctc_setup(const int* __restrict__ tn, const int* __restrict__ ln, int n, int T,
                                          long long nt, CtcUtt* u) {
    if (threadIdx.x >= 32) return;
    const int lane = lane_id();
    long long sum = 0;
    int neg = 0;
    for (int m = lane; m < n; m += 32) {
        const int l = __ldg(ln + m);
        sum += l;
        neg |= l < 0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    neg = __any_sync(0xffffffffu, neg);
    if (lane == 0) {
        const int Tn = __ldg(tn + n), Ln = __ldg(ln + n);
        u->toff = sum;
        u->Tn = Tn;
        u->Ln = Ln;
        u->ok = !neg && Tn >= 0 && Tn <= T && Ln >= 0 && sum + Ln <= nt;
    }
}

// This thread's K states: their class and whether the skip transition into them (α) is allowed.  Returns whether a
// label is outside [0, C).
__device__ __forceinline__ int ctc_states(const void* tg, int t64, long long toff, int S, int C, int (&lab)[kCtcK],
                                          bool (&skip)[kCtcK]) {
    int bad = 0;
#pragma unroll
    for (int k = 0; k < kCtcK; ++k) {
        const int s = threadIdx.x * kCtcK + k;
        lab[k] = 0;
        skip[k] = false;
        if (s < S && (s & 1)) {
            const long long l = ctc_label(tg, t64, toff + (s >> 1));
            if (l < 0 || l >= C) bad = 1;
            else lab[k] = (int)l;
            skip[k] = s >= 3 && l != ctc_label(tg, t64, toff + (s >> 1) - 1);
        }
    }
    return bad;
}

template <typename T>
__global__ void __launch_bounds__(kCtcThreads) ctc_fwd_kernel(const T* __restrict__ x, const void* __restrict__ tg,
                                                              int t64, const int* __restrict__ tn,
                                                              const int* __restrict__ ln, float* __restrict__ nll,
                                                              float* lse, float* alpha, int Tmax, int N, int C,
                                                              long long nt) {
    using A = Elem<T>;
    __shared__ CtcUtt s_u;
    __shared__ float s_bnd[2][kCtcWarps][2];
    const int n = blockIdx.x, tid = threadIdx.x, lane = lane_id(), warp = tid >> 5;
    ctc_setup(tn, ln, n, Tmax, nt, &s_u);
    __syncthreads();
    const long long toff = s_u.toff;
    const int Tn = s_u.Tn, Ln = s_u.Ln;
    const int S = s_u.ok ? 2 * Ln + 1 : 0;
    int lab[kCtcK];
    bool skip[kCtcK];
    const int bad = ctc_states(tg, t64, toff, S, C, lab, skip);
    const bool ok = s_u.ok && !__syncthreads_or(bad);
    if (!ok) {
        if (tid == 0) nll[n] = __int_as_float(0x7fffffff);
        return;
    }
    if (Tn == 0) {
        if (tid == 0) nll[n] = Ln == 0 ? 0.f : INFINITY;
        return;
    }
    // 1. the log-sum-exp of each frame
    const size_t rs = (size_t)N * C;                           // elements between frames
    for (int t = warp; t < Tn; t += kCtcWarps) {
        const T* row = x + (size_t)t * rs + (size_t)n * C;
        float m = -INFINITY, s = 0.f;
        for (int c = lane; c < C; c += 32) ctc_acc(m, s, A::ld(row + c));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ctc_combine(m, s, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, s, o));
        if (lane == 0) lse[(size_t)t * N + n] = m + logf(s);
    }
    __syncthreads();
    // 2. the α recursion on the first nw warps
    const int nw = (S + 32 * kCtcK - 1) / (32 * kCtcK);
    float* al = alpha + (size_t)Tmax * (size_t)(2 * toff + n);
    if (warp < nw) {
        const int s0 = tid * kCtcK;
        float a[kCtcK];                                        // α[t-1]; before t = 0, the start state 0
#pragma unroll
        for (int k = 0; k < kCtcK; ++k) a[k] = s0 + k == 0 ? 0.f : -INFINITY;
        if (nw > 1) {
            if (lane == 31) { s_bnd[1][warp][0] = a[kCtcK - 1]; s_bnd[1][warp][1] = a[kCtcK - 2]; }
            ctc_bar(nw * 32);
        }
        const T* xn = x + (size_t)n * C;
        float xv[kCtcK], lt = lse[n];
#pragma unroll
        for (int k = 0; k < kCtcK; ++k) xv[k] = A::ld(xn + lab[k]);
        for (int t = 0; t < Tn; ++t) {
            float e[kCtcK];
#pragma unroll
            for (int k = 0; k < kCtcK; ++k) e[k] = xv[k] - lt;
            if (t + 1 < Tn) {                                  // the next step's emissions, ahead
                const T* r = xn + (size_t)(t + 1) * rs;
#pragma unroll
                for (int k = 0; k < kCtcK; ++k) xv[k] = A::ld(r + lab[k]);
                lt = lse[(size_t)(t + 1) * N + n];
            }
            float p1 = __shfl_up_sync(0xffffffffu, a[kCtcK - 1], 1), p2 = __shfl_up_sync(0xffffffffu, a[kCtcK - 2], 1);
            if (lane == 0) {
                p1 = warp > 0 ? s_bnd[(t + 1) & 1][warp - 1][0] : -INFINITY;
                p2 = warp > 0 ? s_bnd[(t + 1) & 1][warp - 1][1] : -INFINITY;
            }
            float b[kCtcK];
#pragma unroll
            for (int k = 0; k < kCtcK; ++k) {
                const float q1 = k >= 1 ? a[k - 1] : p1;
                const float q2 = k >= 2 ? a[k - 2] : (k == 1 ? p1 : p2);
                b[k] = s0 + k < S ? ctc_lse3(a[k], q1, skip[k] ? q2 : -INFINITY) + e[k] : -INFINITY;
            }
            float* at = al + (size_t)t * S;
#pragma unroll
            for (int k = 0; k < kCtcK; ++k) {
                a[k] = b[k];
                if (s0 + k < S) at[s0 + k] = b[k];
            }
            if (nw > 1) {
                if (lane == 31) { s_bnd[t & 1][warp][0] = a[kCtcK - 1]; s_bnd[t & 1][warp][1] = a[kCtcK - 2]; }
                ctc_bar(nw * 32);
            }
        }
    }
    __syncthreads();
    if (tid == 0) {
        const float* at = al + (size_t)(Tn - 1) * S;
        const float v1 = at[S - 1], v2 = S >= 2 ? at[S - 2] : -INFINITY;
        nll[n] = -ctc_lse3(v1, v2, -INFINITY);
    }
}

// loss = sum of nll[n] (+inf as 0), lanes over n in order, then a fixed shuffle tree.
__global__ void __launch_bounds__(32) ctc_reduce_kernel(const float* __restrict__ nll, int N, float* __restrict__ loss) {
    float s = 0.f;
    for (int n = lane_id(); n < N; n += 32) {
        const float v = nll[n];
        s += v == INFINITY ? 0.f : v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane_id() == 0) *loss = s;
}

template <typename T>
__global__ void __launch_bounds__(kCtcThreads) ctc_bwd_kernel(const T* __restrict__ x, const void* __restrict__ tg,
                                                              int t64, const int* __restrict__ tn,
                                                              const int* __restrict__ ln, const float* __restrict__ nll,
                                                              const float* __restrict__ lse,
                                                              const float* __restrict__ alpha, float* ab,
                                                              const float* __restrict__ g, T* __restrict__ dx, int Tmax,
                                                              int N, int C, long long nt) {
    using A = Elem<T>;
    __shared__ CtcUtt s_u;
    __shared__ float s_bnd[2][kCtcWarps][2];
    __shared__ int s_head[kCtcMaxC];                           // per class: its first odd state's label index, or -1
    __shared__ int s_next[kCtcMaxTargets];                     // per label index: the next one of the same class
    __shared__ float s_v[kCtcWarps][kCtcMaxC], s_lp[kCtcWarps][kCtcMaxC];   // per warp: the frame's A_c - lp_c, lp_c
    const int n = blockIdx.x, tid = threadIdx.x, lane = lane_id(), warp = tid >> 5;
    ctc_setup(tn, ln, n, Tmax, nt, &s_u);
    __syncthreads();
    const long long toff = s_u.toff;
    const int Tn = s_u.Tn, Ln = s_u.Ln;
    const int S = s_u.ok ? 2 * Ln + 1 : 0;
    int lab[kCtcK];
    bool skip[kCtcK];
    const int bad = ctc_states(tg, t64, toff, S, C, lab, skip);
    const bool ok = s_u.ok && !__syncthreads_or(bad);
    const size_t rs = (size_t)N * C;
    const float nl = __ldg(nll + n);
    // what the frames t < Tv get: the gradient (mode 0), NaN (1) or 0 (2: zero_infinity, and Tn = 0)
    const int mode = !ok ? 1 : (nl == INFINITY || Tn == 0) ? 2 : 0;
    const int Tv = ok || (Tn >= 0 && Tn <= Tmax) ? Tn : Tmax;
    const size_t ao = (size_t)Tmax * (size_t)(ok ? 2 * toff + n : 0);
    const float* al = alpha + ao;
    float* abn = ab + ao;
    if (mode == 0) {
        if (tid == 0) {                                        // the per-class lists, in ascending state order
            for (int c = 0; c < C; ++c) s_head[c] = -1;
            for (int j = Ln - 1; j >= 0; --j) {
                const int c = (int)ctc_label(tg, t64, toff + j);
                s_next[j] = s_head[c];
                s_head[c] = j;
            }
        }
        // the β recursion on the first nw warps, writing α[t] + β[t]
        const int nw = (S + 32 * kCtcK - 1) / (32 * kCtcK);
        if (warp < nw) {
            const int s0 = tid * kCtcK;
            bool skb[kCtcK];                                   // β: may s skip to s + 2
#pragma unroll
            for (int k = 0; k < kCtcK; ++k) {
                const int s = s0 + k;
                skb[k] = (s & 1) && s + 2 < S &&
                         ctc_label(tg, t64, toff + (s >> 1)) != ctc_label(tg, t64, toff + (s >> 1) + 1);
            }
            float b[kCtcK];                                    // β[t+1]; after Tn - 1, the end state S - 1
#pragma unroll
            for (int k = 0; k < kCtcK; ++k) b[k] = s0 + k == S - 1 ? 0.f : -INFINITY;
            if (nw > 1) {
                if (lane == 0) { s_bnd[1][warp][0] = b[0]; s_bnd[1][warp][1] = b[1]; }
                ctc_bar(nw * 32);
            }
            const T* xn = x + (size_t)n * C;
            float xv[kCtcK], lt = __ldg(lse + (size_t)(Tn - 1) * N + n);
#pragma unroll
            for (int k = 0; k < kCtcK; ++k) xv[k] = A::ld(xn + (size_t)(Tn - 1) * rs + lab[k]);
            for (int i = 0; i < Tn; ++i) {
                const int t = Tn - 1 - i;
                float e[kCtcK];
#pragma unroll
                for (int k = 0; k < kCtcK; ++k) e[k] = xv[k] - lt;
                if (t > 0) {
                    const T* r = xn + (size_t)(t - 1) * rs;
#pragma unroll
                    for (int k = 0; k < kCtcK; ++k) xv[k] = A::ld(r + lab[k]);
                    lt = __ldg(lse + (size_t)(t - 1) * N + n);
                }
                float q1 = __shfl_down_sync(0xffffffffu, b[0], 1), q2 = __shfl_down_sync(0xffffffffu, b[1], 1);
                if (lane == 31) {
                    q1 = warp + 1 < nw ? s_bnd[(i + 1) & 1][warp + 1][0] : -INFINITY;
                    q2 = warp + 1 < nw ? s_bnd[(i + 1) & 1][warp + 1][1] : -INFINITY;
                }
                float c[kCtcK];
#pragma unroll
                for (int k = 0; k < kCtcK; ++k) {
                    const float r1 = k + 1 < kCtcK ? b[k + 1] : q1;
                    const float r2 = k + 2 < kCtcK ? b[k + 2] : (k + 2 == kCtcK ? q1 : q2);
                    c[k] = s0 + k < S ? ctc_lse3(b[k], r1, skb[k] ? r2 : -INFINITY) + e[k] : -INFINITY;
                }
                const float* at = al + (size_t)t * S;
                float* abt = abn + (size_t)t * S;
#pragma unroll
                for (int k = 0; k < kCtcK; ++k) {
                    b[k] = c[k];
                    if (s0 + k < S) abt[s0 + k] = __ldg(at + s0 + k) + c[k];
                }
                if (nw > 1) {
                    if (lane == 0) { s_bnd[i & 1][warp][0] = b[0]; s_bnd[i & 1][warp][1] = b[1]; }
                    ctc_bar(nw * 32);
                }
            }
        }
    }
    __syncthreads();
    // the frames: the gradient (or NaN) on t < Tv, 0 after
    const float gs = __ldg(g);
    for (int t = warp; t < Tmax; t += kCtcWarps) {
        const size_t ro = (size_t)t * rs + (size_t)n * C;
        if (t >= Tv || mode != 0) {
            const float v = t < Tv && mode == 1 ? __int_as_float(0x7fffffff) : 0.f;
            for (int c = lane; c < C; c += 32) dx[ro + c] = A::narrow1(v);
            continue;
        }
        const float* at = abn + (size_t)t * S;
        float m = -INFINITY, s = 0.f;                          // the blank class: the even states
        for (int j = lane; j <= Ln; j += 32) ctc_acc(m, s, at[2 * j]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ctc_combine(m, s, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, s, o));
        const float lt = __ldg(lse + (size_t)t * N + n);
        float mz = -INFINITY, sz = 0.f;                        // Z_t over the classes
        for (int c = lane; c < C; c += 32) {
            float mc = c == 0 ? m : -INFINITY, sc = c == 0 ? s : 0.f;
            for (int j = s_head[c]; j >= 0; j = s_next[j]) ctc_acc(mc, sc, at[2 * j + 1]);
            const float lp = A::ld(x + ro + c) - lt;
            const float v = mc + logf(sc) - lp;
            s_v[warp][c] = v;
            s_lp[warp][c] = lp;
            ctc_acc(mz, sz, v);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ctc_combine(mz, sz, __shfl_xor_sync(0xffffffffu, mz, o), __shfl_xor_sync(0xffffffffu, sz, o));
        const float z = mz + logf(sz);
        __syncwarp();
        for (int c = lane; c < C; c += 32)
            dx[ro + c] = A::narrow1((expf(s_lp[warp][c]) - expf(s_v[warp][c] - z)) * gs);
        __syncwarp();                                          // s_v / s_lp are reused by the warp's next frame
    }
}

template <typename T>
static cudaError_t ctc_forward_t(const void* x, const void* t, int t64, const int* tn, const int* ln, float* ws,
                                 float* loss, int T_, int N, int C, long long nt, cudaStream_t stream) {
    float* nll = ws;
    float* lse = ws + N;
    float* alpha = lse + (size_t)T_ * N;
    ctc_fwd_kernel<T><<<N, kCtcThreads, 0, stream>>>(static_cast<const T*>(x), t, t64, tn, ln, nll, lse, alpha, T_, N, C,
                                                     nt);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    ctc_reduce_kernel<<<1, 32, 0, stream>>>(nll, N, loss);
    return cudaGetLastError();
}

template <typename T>
static cudaError_t ctc_backward_t(const void* x, const void* t, int t64, const int* tn, const int* ln, const float* ws,
                                  float* ab, const float* g, void* dx, int T_, int N, int C, long long nt,
                                  cudaStream_t stream) {
    const float* nll = ws;
    const float* lse = ws + N;
    const float* alpha = ws + N + (size_t)T_ * N;
    ctc_bwd_kernel<T><<<N, kCtcThreads, 0, stream>>>(static_cast<const T*>(x), t, t64, tn, ln, nll, lse, alpha, ab, g,
                                                     static_cast<T*>(dx), T_, N, C, nt);
    return cudaGetLastError();
}

bool ctc_supported(int T, int N, int C, long long nt) {
    return T > 0 && N > 0 && C > 0 && C <= kCtcMaxC && nt >= 0 && nt <= kCtcMaxTargets;
}

long long ctc_workspace_floats(int T, int N, long long nt) { return (long long)N + (long long)T * (2 * nt + 2LL * N); }
long long ctc_ab_floats(int T, int N, long long nt) { return (long long)T * (2 * nt + N); }

cudaError_t launch_ctc_forward(const void* x, const void* targets, int targets64, const int* tn, const int* ln, float* ws,
                               float* loss, int T, int N, int C, long long nt, Dtype dtype, cudaStream_t stream) {
    if (!ctc_supported(T, N, C, nt)) return cudaErrorInvalidValue;
    return with_dtype(dtype, [&](auto e) {
        return ctc_forward_t<decltype(e)>(x, targets, targets64, tn, ln, ws, loss, T, N, C, nt, stream);
    });
}

cudaError_t launch_ctc_backward(const void* x, const void* targets, int targets64, const int* tn, const int* ln,
                                const float* ws, float* ab, const float* g, void* dx, int T, int N, int C, long long nt,
                                Dtype dtype, cudaStream_t stream) {
    if (!ctc_supported(T, N, C, nt)) return cudaErrorInvalidValue;
    return with_dtype(dtype, [&](auto e) {
        return ctc_backward_t<decltype(e)>(x, targets, targets64, tn, ln, ws, ab, g, dx, T, N, C, nt, stream);
    });
}

}  // namespace okt
