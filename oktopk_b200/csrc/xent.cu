// Fused softmax cross-entropy with ignore_index, mean reduction, forward and backward:
//
//   loss = mean over rows r with t[r] != ignore of (lse_r - x[r, t[r]]),   lse_r = log sum_j exp x[r, j]
//   dx[r, j] = (exp(x[r, j] - lse_r) - [j == t[r]]) . g / n      (0 on an ignored row),  n = #rows not ignored
//
// BERT's masked-LM loss runs over [B S, vocab] logits of which only the masked positions (~11 % of the rows) are
// labelled.  Stock cross_entropy widens every row to fp32, runs log_softmax over all of them and back-propagates a mostly
// zero gradient through two more full passes.  Here the forward pass reads only the labelled rows and keeps one fp32
// log-sum-exp per row; the backward pass reads the labelled rows once more and writes the gradient once.
//
// Forward (xent_fwd_kernel + xent_reduce_kernel): one CTA per row, rows dealt by a grid-stride loop.  A CTA whose row is
// ignored moves on without reading it.  Otherwise every thread keeps an online (max, rescaled sum of exp) pair in fp32
// over its share of the row, and the pairs are combined over the warp and then over the warps in a fixed order; thread
// 0 writes lse_r and the row loss lse_r - x[r, t[r]].  A second one-CTA kernel adds the labelled rows' losses in double
// in a fixed order, counts n and writes loss = sum / n and n: no atomics, no host synchronisation, bitwise reproducible.
//
// Backward (xent_bwd_kernel): one CTA per row, grid-stride.  g (the loss's incoming gradient, which carries a loss
// scale) and n are read from device memory, so a replayed CUDA graph sees their current values.  Ignored rows get
// 128-bit zero stores only; labelled rows compute the formula above in fp32 and round once to the logits' type.
//
// Rows: V is arbitrary (30522 in BERT), so a row starts at any 2- or 4-byte offset mod 16.  Each row is a scalar head
// up to the first 16-byte boundary, a body of 128-bit vectors and a scalar tail; x and dx start 16-byte aligned, so the
// two split alike.  Row offsets are 64-bit.
//
// Types: x and dx are fp32, bf16 or fp16; lse, the losses and all arithmetic are fp32.  Rounding is .to(dtype)'s: to
// nearest even, fp16 overflowing to inf (so a loss-scaled overflow reaches the scaler's device-side check).
//
// Edges: n == 0 gives loss 0/0 = NaN and an all-zero gradient, as torch.  A NaN or +inf in a labelled row makes that
// row's lse, loss and gradient NaN; -inf entries contribute exp = 0.  A target outside [0, V) that is not `ignore`
// counts in n and gives a NaN row loss and a NaN gradient row (torch's kernel device-asserts instead).  An ignored row is
// never read, so its gradient is 0 even if it holds inf or NaN (stock log_softmax backward makes it NaN).
#include "common.cuh"
#include "elem.cuh"
#include "oktopk.cuh"

namespace okt {

constexpr int kXeFwdThreads = 512;
constexpr int kXeBwdThreads = 256;
constexpr int kXeRedThreads = 256;
constexpr int kXeMaxBlocks = 8192;

// A row's scalar head (elements before its first 16-byte boundary) and its count of 16-byte vectors after it; the tail
// is what is left.  `row` is T-aligned.
template <typename T>
__device__ __forceinline__ void xe_split(const T* row, long long V, long long& head, long long& nvec) {
    head = (long long)(((16u - ((unsigned)(uintptr_t)row & 15u)) & 15u) / sizeof(T));
    if (head > V) head = V;
    nvec = (V - head) / Elem<T>::kVec;
}

// Online log-sum-exp state (m, s): the row's running max and sum of exp(x - m).  A pair whose max is unchanged keeps
// its sum (so an inf or -inf max does not make inf - inf); a -inf element adds 0; a NaN anywhere reaches s.
__device__ __forceinline__ float xe_rescale(float m, float mn) { return m == mn ? 1.f : expf(m - mn); }
__device__ __forceinline__ float xe_term(float x, float mn) { return x == -INFINITY ? 0.f : expf(x - mn); }

template <int K>
__device__ __forceinline__ void xe_update(float& m, float& s, const float (&f)[K]) {
    float mv = f[0];
#pragma unroll
    for (int i = 1; i < K; ++i) mv = fmaxf(mv, f[i]);
    const float mn = fmaxf(m, mv);
    float add = 0.f;
#pragma unroll
    for (int i = 0; i < K; ++i) add += xe_term(f[i], mn);
    s = fmaf(s, xe_rescale(m, mn), add);
    m = mn;
}

__device__ __forceinline__ void xe_combine(float& m, float& s, float m2, float s2) {
    const float mn = fmaxf(m, m2);
    s = s * xe_rescale(m, mn) + s2 * xe_rescale(m2, mn);
    m = mn;
}

template <typename T>
__global__ void __launch_bounds__(kXeFwdThreads) xent_fwd_kernel(const T* __restrict__ x, const long long* __restrict__ t,
                                                                 float* __restrict__ lse, float* __restrict__ rowloss,
                                                                 int R, long long V, long long ignore) {
    using A = Elem<T>;
    constexpr int kVec = A::kVec, kWarps = kXeFwdThreads / 32, kUnroll = 4;
    __shared__ float s_m[kWarps], s_s[kWarps];
    const int tid = threadIdx.x, lane = lane_id(), warp = tid >> 5;
    for (int r = blockIdx.x; r < R; r += gridDim.x) {
        const long long tr = __ldg(t + r);
        if (tr == ignore) continue;                              // uniform over the CTA: the row is never read
        const T* row = x + (size_t)r * (size_t)V;
        long long head, nvec;
        xe_split(row, V, head, nvec);
        float m = -INFINITY, s = 0.f;
        if (tid < head) { const float f[1] = {A::ld(row + tid)}; xe_update(m, s, f); }
        const uint4* body = reinterpret_cast<const uint4*>(row + head);
        long long k = tid;
        for (; k + (kUnroll - 1) * kXeFwdThreads < nvec; k += kUnroll * kXeFwdThreads) {
            uint4 u[kUnroll];
#pragma unroll
            for (int i = 0; i < kUnroll; ++i) u[i] = __ldg(body + k + i * kXeFwdThreads);
#pragma unroll
            for (int i = 0; i < kUnroll; ++i) { float f[kVec]; A::wide(u[i], f); xe_update(m, s, f); }
        }
        for (; k < nvec; k += kXeFwdThreads) { float f[kVec]; A::wide(__ldg(body + k), f); xe_update(m, s, f); }
        const long long tail = head + nvec * kVec + tid;
        if (tail < V) { const float f[1] = {A::ld(row + tail)}; xe_update(m, s, f); }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) xe_combine(m, s, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, s, o));
        if (lane == 0) { s_m[warp] = m; s_s[warp] = s; }
        __syncthreads();
        if (tid == 0) {
            m = s_m[0];
            s = s_s[0];
            for (int w = 1; w < kWarps; ++w) xe_combine(m, s, s_m[w], s_s[w]);
            const float l = m + logf(s);
            lse[r] = l;
            rowloss[r] = (tr >= 0 && tr < V) ? l - A::ld(row + tr) : __int_as_float(0x7fffffff);
        }
        __syncthreads();                                         // s_m / s_s are reused by the next row
    }
}

// loss = (sum of the labelled rows' losses, in row order per thread, then the threads in a fixed tree) / n; lse[R] = n.
__global__ void __launch_bounds__(kXeRedThreads) xent_reduce_kernel(const float* __restrict__ rowloss,
                                                                    const long long* __restrict__ t, int R,
                                                                    long long ignore, float* __restrict__ lse,
                                                                    float* __restrict__ loss) {
    __shared__ double s_sum[kXeRedThreads / 32];
    __shared__ int s_cnt[kXeRedThreads / 32];
    const int tid = threadIdx.x, lane = lane_id(), warp = tid >> 5;
    double sum = 0.0;
    int cnt = 0;
    for (int r = tid; r < R; r += kXeRedThreads)
        if (t[r] != ignore) { sum += (double)rowloss[r]; ++cnt; }
    sum = warp_sum_d(sum);
    cnt = warp_sum(cnt);
    if (lane == 0) { s_sum[warp] = sum; s_cnt[warp] = cnt; }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < kXeRedThreads / 32; ++w) { sum += s_sum[w]; cnt += s_cnt[w]; }
        lse[R] = (float)cnt;
        *loss = (float)(sum / (double)cnt);                      // n == 0: 0 / 0 = NaN
    }
}

template <typename T>
__global__ void __launch_bounds__(kXeBwdThreads) xent_bwd_kernel(const T* __restrict__ x, const long long* __restrict__ t,
                                                                 const float* __restrict__ lse, const float* __restrict__ g,
                                                                 T* __restrict__ dx, int R, long long V, long long ignore) {
    using A = Elem<T>;
    constexpr int kVec = A::kVec;
    const int tid = threadIdx.x;
    const float gn = __ldg(g) / __ldg(lse + R);
    for (int r = blockIdx.x; r < R; r += gridDim.x) {
        const long long tr = __ldg(t + r);
        const size_t base = (size_t)r * (size_t)V;
        T* drow = dx + base;
        long long head, nvec;
        xe_split(drow, V, head, nvec);
        uint4* dbody = reinterpret_cast<uint4*>(drow + head);
        const long long tail = head + nvec * kVec + tid;
        if (tr == ignore) {
            if (tid < head) drow[tid] = A::narrow1(0.f);
            for (long long k = tid; k < nvec; k += kXeBwdThreads) dbody[k] = make_uint4(0u, 0u, 0u, 0u);
            if (tail < V) drow[tail] = A::narrow1(0.f);
            continue;
        }
        const T* row = x + base;
        const float l = __ldg(lse + r);
        const float c = (tr >= 0 && tr < V) ? gn : __int_as_float(0x7fffffff);    // a bad target: a NaN row
        if (tid < head) drow[tid] = A::narrow1((expf(A::ld(row + tid) - l) - (tid == tr ? 1.f : 0.f)) * c);
        const uint4* body = reinterpret_cast<const uint4*>(row + head);
        for (long long k = tid; k < nvec; k += kXeBwdThreads) {
            float f[kVec];
            A::wide(__ldg(body + k), f);
            const long long j0 = head + k * kVec;
#pragma unroll
            for (int i = 0; i < kVec; ++i) f[i] = (expf(f[i] - l) - (j0 + i == tr ? 1.f : 0.f)) * c;
            dbody[k] = A::narrow(f);
        }
        if (tail < V) drow[tail] = A::narrow1((expf(A::ld(row + tail) - l) - (tail == tr ? 1.f : 0.f)) * c);
    }
}

static int xe_grid(int R) { return R < kXeMaxBlocks ? R : kXeMaxBlocks; }

template <typename T>
static cudaError_t xent_forward_t(const void* x, const long long* t, float* lse, float* rowloss, float* loss, int R,
                                  long long V, long long ignore, cudaStream_t stream) {
    xent_fwd_kernel<T><<<xe_grid(R), kXeFwdThreads, 0, stream>>>(static_cast<const T*>(x), t, lse, rowloss, R, V, ignore);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    xent_reduce_kernel<<<1, kXeRedThreads, 0, stream>>>(rowloss, t, R, ignore, lse, loss);
    return cudaGetLastError();
}

template <typename T>
static cudaError_t xent_backward_t(const void* x, const long long* t, const float* lse, const float* g, void* dx, int R,
                                   long long V, long long ignore, cudaStream_t stream) {
    xent_bwd_kernel<T><<<xe_grid(R), kXeBwdThreads, 0, stream>>>(static_cast<const T*>(x), t, lse, g, static_cast<T*>(dx),
                                                                 R, V, ignore);
    return cudaGetLastError();
}

cudaError_t launch_xent_forward(const void* x, const long long* t, float* lse, float* rowloss, float* loss, int R,
                                long long V, long long ignore_index, Dtype dtype, cudaStream_t stream) {
    if (R <= 0 || V <= 0) return cudaErrorInvalidValue;
    return with_dtype(dtype, [&](auto e) {
        return xent_forward_t<decltype(e)>(x, t, lse, rowloss, loss, R, V, ignore_index, stream);
    });
}

cudaError_t launch_xent_backward(const void* x, const long long* t, const float* lse, const float* g, void* dx, int R,
                                 long long V, long long ignore_index, Dtype dtype, cudaStream_t stream) {
    if (R <= 0 || V <= 0) return cudaErrorInvalidValue;
    return with_dtype(dtype, [&](auto e) { return xent_backward_t<decltype(e)>(x, t, lse, g, dx, R, V, ignore_index, stream); });
}

}  // namespace okt
