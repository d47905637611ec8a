// Persistent LSTM recurrence (time-major T x N, torch's gate order i, f, g, o, zero initial state):
//
//   a_t = gx_t + W_hh h_{t-1}                  gx = x W_ih^T + b_ih + b_hh for all t: one GEMM in torch beforehand
//   i, f, o = sigmoid(a_i, a_f, a_o), g = tanh(a_g),   c_t = f c_{t-1} + i g,   h_t = o tanh(c_t)
//
// Utterance b has length len_b: y_t = h_t for t < len_b and exactly 0 after (what pad_packed_sequence gives).
//
// cuDNN's fp32 RNN runs this as a small GEMM and an element-wise kernel per timestep and pass, each re-reading the
// 4H x H recurrent matrix from L2.  Here one cooperative kernel walks all timesteps of a pass, and the matrix stays in
// shared memory: CTA b owns the u hidden units [b u, b u + u) (u = ceil(H / #SMs): H = 800 on 132 SMs gives u = 7 on
// 115 CTAs, 89.6 KB of weights each).
//
// Forward (lstm_fwd_kernel): the CTA keeps the 4u rows of W_hh of its units' gates and their cell states c.  At step t
// it stages h_{t-1} = y_{t-1} (all N x H of it, `rows` batch rows at a time) from L2 into shared memory, forms its 4u x N
// gate sums, then its units' c_t and h_t; it writes y_t, the activated gates and c_t (for the backward pass) and crosses
// the grid barrier, after which every CTA can read all of y_t.
//
// Backward (lstm_bwd_kernel), t from Tm-1 down to 0 (Tm: below): the CTA keeps the 4H x u columns of W_hh of the same
// units, so that dh_rec[j] = sum_k W_hh[k, j] dgates_{t+1}[k] is local.  At step t it stages dgates_{t+1} (N x 4H)
// and forms its u x N dh_rec; with dy_t, the saved gates and c, and its carried dc it writes dgates_t for its units' 4
// gate rows and crosses the barrier.  For t >= len_b, dgates and the carried dc are exactly 0.  dx, dW_ih, dW_hh and the
// bias gradients are GEMMs and sums over dgates in torch.
//
// The barrier is common.cuh's ticket grid_sync on a counter the caller zeroes: one per step, the only cross-CTA
// dependency being the whole of y_t (dgates_t), which every CTA reads.  Operands written by other CTAs in this launch
// are read with ld.global.cg (L2), never through L1.
//
// Every sum has a fixed order: lane l of a warp adds the four-element columns l, l + 32, ... of a dot product in order,
// and the 32 lanes are combined by a fixed butterfly.  No atomics touch data, so results are bitwise reproducible.
//
// Storage type S (float, __nv_bfloat16 or __half) is that of the five tensors that are 16-bit under autocast: W_hh (in
// global and in shared memory), gx, y, dy and dgates, and so of the staged h_{t-1} and dgates_{t+1}.  The saved gates and
// c, the gate and dh sums, the cell state, the carried dc and every accumulator are fp32 whatever S is.  A 16-bit
// element is widened on load and enters the same fmaf chain in the same order, so a 16-bit launch is the fp32 kernel run
// on the widened operands, except where a y or dgates it stored (rounded to nearest even, not saturated: an fp16
// overflow is inf) is read back at the next step.
//
// Bound: both passes walk only the Tm = min(max_n len_n, T) steps some row still needs (lstm_steps).  Every CTA reads the
// same N lengths, so every CTA gets the same Tm and crosses the same number of barriers.  For t in [Tm, T) y (forward)
// and dgates (backward) are written as exact zeros before the walk: no other CTA reads them, so they need no barrier.
// The saved gates and c at those times are never read and stay unwritten.  So a launch over a T padded past the longest
// utterance costs the recurrence nothing, and gives y and dgates on [0, Tm) bit for bit what a launch at T = Tm gives.
//
// Directions: a bidirectional layer runs both of its directions in one launch of dirs * g CTAs (g = ceil(H / u)).  CTA
// b serves direction d = b / g with units [(b % g) u, ...) of that direction's own W_hh.  Every per-timestep tensor is
// direction-major, [dirs, T, N, .], so direction 0 sees exactly the one-direction layout; dy is shared, since the layer's
// output is y[0] + y[1].  The two recurrences are independent: each direction syncs only its own g CTAs, on its own
// counter bar[d].  At step s, row n of direction d works on time t = pi_d,n(s) (lstm_time): s forward; len_n - 1 - s
// for s < len_n and s after that in reverse.  pi is a permutation of [0, T), so the reverse direction starts from a zero
// state at len_n - 1 (packed-sequence semantics), writes every time once, and writes exact zeros at t >= len_n like the
// forward one.  What the forward direction indexes by t (gx, gates, c, y, dy, dgates; h_{t-1} = y at pi(s - 1),
// dgates_{t+1} at pi(s + 1), c_{t-1} at pi(s - 1)) the reverse one indexes by pi.
#include "common.cuh"
#include "elem.cuh"
#include "oktopk.cuh"

namespace okt {

constexpr int kLstmThreads = 512;                // ops/fused_lstm.py LSTM_THREADS
constexpr int kLstmWarps = kLstmThreads / 32;
constexpr int kLstmNB = 4;                       // batch rows of one warp task in lstm_dots
constexpr int kMaxLstmBatch = 64;                // ops/fused_lstm.py MAX_BATCH: the fp32 stacked-layer step's M tiles

// whh[1] is null for a one-direction layer; g = ceil(H / u) CTAs per direction.
template <typename S>
struct LstmFwdArgs {
    const S* gx;
    const S* whh[2];
    const int* len;
    S* y;
    float* gates;
    float* cs;
    unsigned long long* bar;
    int T, N, H, u, rows, g;
};

template <typename S>
struct LstmBwdArgs {
    const S* dy;
    const float* gates;
    const float* cs;
    const S* whh[2];
    const int* len;
    S* dg;
    unsigned long long* bar;
    int T, N, H, u, rows, g;
};

__device__ __forceinline__ float lstm_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

// The time that row n (length L) of a direction works on at step s (the file header's pi).
__device__ __forceinline__ int lstm_time(int s, int L, bool rev) { return rev && s < L ? L - 1 - s : s; }

// The header's Tm: the longest of the N lengths, at most T (and 0 if none is positive).
__device__ __forceinline__ int lstm_steps(const int* __restrict__ len, int N, int T) {
    int m = 0;
    for (int n = 0; n < N; ++n) m = max(m, __ldg(len + n));
    return min(m, T);
}

// Copy batch rows [n0, n0 + nrows) of the [T, N, K] tensor V (K % 4 == 0, Vec-aligned), which other CTAs wrote in this
// launch, to shared memory: row n from time lstm_time(s, len_n, rev).  Forward that is one contiguous block; in
// reverse each row has its own time.
template <typename S>
__device__ __forceinline__ void lstm_stage(S* __restrict__ sV, const S* V, int n0, int nrows, int K, int N, int s,
                                           const int* __restrict__ len, bool rev) {
    using Vec = typename Elem<S>::V;
    Vec* d = reinterpret_cast<Vec*>(sV);
    const int K4 = K >> 2, n4 = nrows * K4;
    if (!rev) {
        const Vec* src = reinterpret_cast<const Vec*>(V + (size_t)s * N * K + (size_t)n0 * K);
        for (int i = threadIdx.x; i < n4; i += kLstmThreads) d[i] = __ldcg(src + i);
        return;
    }
    for (int i = threadIdx.x; i < n4; i += kLstmThreads) {
        const int r = i / K4, k = i - r * K4, n = n0 + r;
        const size_t t = lstm_time(s, __ldg(len + n), true);
        d[i] = __ldcg(reinterpret_cast<const Vec*>(V + (t * N + n) * K) + k);
    }
}

// out[r N + n0 + j] = sum_k sW[r K + k] sV[j K + k] for r < R, j < nc.  A warp takes one (r, kLstmNB rows of sV) task at
// a time; the order of every sum is fixed (see the file header), whichever warp runs it.
template <typename S>
__device__ __forceinline__ void lstm_dots(const S* __restrict__ sW, const S* __restrict__ sV,
                                          float* __restrict__ out, int R, int K, int nc, int n0, int N) {
    using El = Elem<S>;
    using Vec = typename El::V;
    const int K4 = K >> 2, lane = lane_id(), warp = threadIdx.x >> 5;
    const int nb = (nc + kLstmNB - 1) / kLstmNB;
    const Vec* W4 = reinterpret_cast<const Vec*>(sW);
    const Vec* V4 = reinterpret_cast<const Vec*>(sV);
    for (int task = warp; task < R * nb; task += kLstmWarps) {
        const int r = task / nb, j0 = (task - r * nb) * kLstmNB;
        const Vec* w = W4 + (size_t)r * K4;
        float acc[kLstmNB];
#pragma unroll
        for (int j = 0; j < kLstmNB; ++j) acc[j] = 0.f;
#pragma unroll 2                 // two k steps of loads in flight for every S, not left to how costly widening S looks
        for (int k = lane; k < K4; k += 32) {
            const float4 a = El::wide(w[k]);
#pragma unroll
            for (int j = 0; j < kLstmNB; ++j) {
                if (j0 + j < nc) {
                    const float4 b = El::wide(V4[(size_t)(j0 + j) * K4 + k]);
                    acc[j] = fmaf(a.x, b.x, acc[j]);
                    acc[j] = fmaf(a.y, b.y, acc[j]);
                    acc[j] = fmaf(a.z, b.z, acc[j]);
                    acc[j] = fmaf(a.w, b.w, acc[j]);
                }
            }
        }
#pragma unroll
        for (int j = 0; j < kLstmNB; ++j) acc[j] = warp_sum_f(acc[j]);
        if (lane == 0) {
#pragma unroll
            for (int j = 0; j < kLstmNB; ++j)
                if (j0 + j < nc) out[r * N + n0 + j0 + j] = acc[j];
        }
    }
}

// out[r N + n] = sum_k sW[r K + k] V[t_n, n, k] over all N rows of V (global [T, N, K], written in this launch), `rows`
// at a time, t_n = lstm_time(s, len_n, rev).
template <typename S>
__device__ __forceinline__ void lstm_matvec(const S* __restrict__ sW, S* __restrict__ sV, const S* V,
                                            float* __restrict__ out, int R, int K, int N, int rows, int s,
                                            const int* __restrict__ len, bool rev) {
    for (int n0 = 0; n0 < N; n0 += rows) {
        const int nc = min(rows, N - n0);
        lstm_stage(sV, V, n0, nc, K, N, s, len, rev);
        __syncthreads();
        lstm_dots(sW, sV, out, R, K, nc, n0, N);
        __syncthreads();
    }
}

// Shared memory: W [4u][H] and h_{t-1} rows [rows][H] of S | gate sums [4u][N] | c [u][N] of float.  H % 4 == 0 makes
// the two S sections multiples of 8 bytes, so the float sections are aligned for either S.
template <typename S>
__global__ void __launch_bounds__(kLstmThreads, 1) lstm_fwd_kernel(const LstmFwdArgs<S> p) {
    using El = Elem<S>;
    using Vec = typename El::V;
    extern __shared__ float4 lstm_smem[];
    const int H = p.H, N = p.N, u = p.u, R = 4 * u, H4 = H >> 2;
    const int d = blockIdx.x / p.g;
    const bool rev = d != 0;
    const int u0 = (blockIdx.x - d * p.g) * u, nu = min(u, H - u0);
    const size_t dTNH = (size_t)d * p.T * N * H;                     // this direction's [T, N, .] blocks
    const S* whh = rev ? p.whh[1] : p.whh[0];
    const S* gx0 = p.gx + 4 * dTNH;
    S* y = p.y + dTNH;
    float* gates = p.gates + 4 * dTNH;
    float* cs = p.cs + dTNH;
    unsigned long long* bar = p.bar + d;
    S* sW = reinterpret_cast<S*>(lstm_smem);
    S* sV = sW + (size_t)R * H;
    float* sG = reinterpret_cast<float*>(sV + (size_t)p.rows * H);
    float* sC = sG + R * N;
    for (int i = threadIdx.x; i < R * H4; i += kLstmThreads) {      // local row q u + j = W_hh row q H + u0 + j
        const int lr = i / H4, k = i - lr * H4, q = lr / u, j = lr - q * u;
        Vec v = El::zero();
        if (j < nu) v = __ldg(reinterpret_cast<const Vec*>(whh + (size_t)(q * H + u0 + j) * H) + k);
        reinterpret_cast<Vec*>(sW)[i] = v;
    }
    for (int i = threadIdx.x; i < u * N; i += kLstmThreads) sC[i] = 0.f;
    const int Tm = lstm_steps(p.len, N, p.T);
    for (int i = threadIdx.x; i < (p.T - Tm) * nu * N; i += kLstmThreads) {       // y past every length: exact zeros
        const int j = i % nu, r = i / nu;
        y[((size_t)Tm * N + r) * H + u0 + j] = El::narrow1(0.f);
    }
    for (int s = 0; s < Tm; ++s) {
        if (s == 0) {
            for (int i = threadIdx.x; i < R * N; i += kLstmThreads) sG[i] = 0.f;
            __syncthreads();
        } else {
            lstm_matvec(sW, sV, y, sG, R, H, N, p.rows, s - 1, p.len, rev);         // h_{t-1}: y at pi(s - 1)
        }
        for (int i = threadIdx.x; i < nu * N; i += kLstmThreads) {
            const int j = i / N, n = i - j * N, unit = u0 + j;
            const int L = __ldg(p.len + n);
            const size_t row = (size_t)lstm_time(s, L, rev) * N + n;
            const S* gx = gx0 + row * 4 * H + unit;
            float* gs = gates + row * 4 * H + unit;
            const size_t o = row * H + unit;
            if (s < L) {
                const float gi = lstm_sigmoid(sG[(0 * u + j) * N + n] + El::ld(gx));
                const float gf = lstm_sigmoid(sG[(1 * u + j) * N + n] + El::ld(gx + H));
                const float gg = tanhf(sG[(2 * u + j) * N + n] + El::ld(gx + 2 * H));
                const float go = lstm_sigmoid(sG[(3 * u + j) * N + n] + El::ld(gx + 3 * H));
                const float c = gf * sC[j * N + n] + gi * gg;
                sC[j * N + n] = c;
                gs[0] = gi; gs[H] = gf; gs[2 * H] = gg; gs[3 * H] = go;
                cs[o] = c;
                y[o] = El::narrow1(go * tanhf(c));
            } else {
                gs[0] = 0.f; gs[H] = 0.f; gs[2 * H] = 0.f; gs[3 * H] = 0.f;
                cs[o] = 0.f;
                y[o] = El::narrow1(0.f);
            }
        }
        if (s + 1 < Tm) grid_sync(bar, p.g);
    }
}

// Shared memory: W^T [u][4H] and dgates_{t+1} rows [rows][4H] of S | dh_rec [u][N] | carried dc [u][N] of float.
template <typename S>
__global__ void __launch_bounds__(kLstmThreads, 1) lstm_bwd_kernel(const LstmBwdArgs<S> p) {
    using El = Elem<S>;
    extern __shared__ float4 lstm_smem[];
    const int H = p.H, N = p.N, u = p.u, G = 4 * H;
    const int d = blockIdx.x / p.g;
    const bool rev = d != 0;
    const int u0 = (blockIdx.x - d * p.g) * u, nu = min(u, H - u0);
    const size_t dTNH = (size_t)d * p.T * N * H;                     // this direction's [T, N, .] blocks; dy is shared
    const S* whh = rev ? p.whh[1] : p.whh[0];
    const float* gates = p.gates + 4 * dTNH;
    const float* cs = p.cs + dTNH;
    S* dg0 = p.dg + 4 * dTNH;
    unsigned long long* bar = p.bar + d;
    S* sW = reinterpret_cast<S*>(lstm_smem);
    S* sV = sW + (size_t)u * G;
    float* sD = reinterpret_cast<float*>(sV + (size_t)p.rows * G);
    float* sDC = sD + u * N;
    for (int i = threadIdx.x; i < u * G; i += kLstmThreads) {       // sW[j][k] = W_hh[k][u0 + j]
        const int k = i / u, j = i - k * u;
        sW[(size_t)j * G + k] = j < nu ? __ldg(whh + (size_t)k * H + u0 + j) : El::narrow1(0.f);
    }
    for (int i = threadIdx.x; i < u * N; i += kLstmThreads) sDC[i] = 0.f;
    const int Tm = lstm_steps(p.len, N, p.T);
    for (int i = threadIdx.x; i < (p.T - Tm) * nu * N; i += kLstmThreads) {       // dgates past every length: zeros
        const int j = i % nu, r = i / nu;
        S* dg = dg0 + ((size_t)Tm * N + r) * G + u0 + j;
        dg[0] = dg[H] = dg[2 * H] = dg[3 * H] = El::narrow1(0.f);
    }
    for (int s = Tm - 1; s >= 0; --s) {
        if (s == Tm - 1) {
            for (int i = threadIdx.x; i < u * N; i += kLstmThreads) sD[i] = 0.f;
            __syncthreads();
        } else {
            lstm_matvec(sW, sV, dg0, sD, u, G, N, p.rows, s + 1, p.len, rev);       // dgates at pi(s + 1)
        }
        for (int i = threadIdx.x; i < nu * N; i += kLstmThreads) {
            const int j = i / N, n = i - j * N, unit = u0 + j;
            const int L = __ldg(p.len + n);
            const size_t row = (size_t)lstm_time(s, L, rev) * N + n;
            const size_t o = row * H + unit;
            S* dg = dg0 + row * G + unit;
            if (s < L) {
                const float* gs = gates + row * G + unit;
                const float gi = __ldg(gs), gf = __ldg(gs + H), gg = __ldg(gs + 2 * H), go = __ldg(gs + 3 * H);
                const float tc = tanhf(__ldg(cs + o));
                const float cp = s > 0 ? __ldg(cs + ((size_t)lstm_time(s - 1, L, rev) * N + n) * H + unit) : 0.f;
                const float dh = El::ld(p.dy + o) + sD[j * N + n];
                const float dc = dh * go * (1.f - tc * tc) + sDC[j * N + n];
                dg[0] = El::narrow1(dc * gg * gi * (1.f - gi));
                dg[H] = El::narrow1(dc * cp * gf * (1.f - gf));
                dg[2 * H] = El::narrow1(dc * gi * (1.f - gg * gg));
                dg[3 * H] = El::narrow1(dh * tc * go * (1.f - go));
                sDC[j * N + n] = dc * gf;
            } else {
                dg[0] = dg[H] = dg[2 * H] = dg[3 * H] = El::narrow1(0.f);
                sDC[j * N + n] = 0.f;
            }
        }
        if (s > 0) grid_sync(bar, p.g);
    }
}

// What a launch needs to know about the device and the kernel, queried once per device (the SM count), per larger
// shared-memory size (the kernel's opt-in limit only ever grows) and per new size (the occupancy): the eager AN4 step
// launches these kernels ten times, and its host side is what limits it.
constexpr int kLstmMaxDevices = 64;
struct LstmLaunchCache {
    int sms = 0;
    size_t smem_set = 0;
    size_t occ_smem = 0;
    int occ_per = 0;
};

// Cooperative launch of `grid` CTAs with `smem` bytes each; an error if they cannot all be co-resident.
template <typename Args>
static cudaError_t lstm_launch(void (*kernel)(const Args), const Args& p, int grid, size_t smem, cudaStream_t stream) {
    static LstmLaunchCache cache[kLstmMaxDevices];             // one table per kernel: each has its own Args
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= kLstmMaxDevices) return cudaErrorInvalidDevice;
    LstmLaunchCache& c = cache[dev];
    if (c.sms == 0) e = cudaDeviceGetAttribute(&c.sms, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess && smem > c.smem_set) {
        e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) c.smem_set = smem;
    }
    if (e == cudaSuccess && smem != c.occ_smem) {
        int per = 0;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, kernel, kLstmThreads, smem);
        if (e == cudaSuccess) {
            c.occ_smem = smem;
            c.occ_per = per;
        }
    }
    if (e != cudaSuccess) {
        c.sms = 0;
        (void)cudaGetLastError();
        return e;
    }
    if (c.occ_per * c.sms < grid) return cudaErrorCooperativeLaunchTooLarge;
    void* args[] = {(void*)&p};
    e = cudaLaunchCooperativeKernel((void*)kernel, dim3(grid), dim3(kLstmThreads), args, smem, stream);
    (void)cudaGetLastError();       // a failed launch must not surface again at the next launcher's error check
    return e;
}

static bool lstm_shape_ok(int T, int N, int H, int u, int rows) {
    return T > 0 && N > 0 && H > 0 && H % 4 == 0 && u > 0 && u <= H && rows > 0 && rows <= N;
}

// whh_rev null: one direction, g = ceil(H / u) CTAs; else both, 2 g CTAs.
template <typename S>
static cudaError_t lstm_forward_t(const void* gx, const void* whh, const void* whh_rev, const int* len, void* y,
                                  float* gates, float* cs, unsigned long long* bar, int T, int N, int H, int u, int rows,
                                  cudaStream_t stream) {
    const int g = (H + u - 1) / u;
    const LstmFwdArgs<S> p{static_cast<const S*>(gx), {static_cast<const S*>(whh), static_cast<const S*>(whh_rev)}, len,
                           static_cast<S*>(y), gates, cs, bar, T, N, H, u, rows, g};
    const size_t smem = sizeof(S) * ((size_t)4 * u * H + (size_t)rows * H) + sizeof(float) * (size_t)5 * u * N;
    return lstm_launch(lstm_fwd_kernel<S>, p, whh_rev ? 2 * g : g, smem, stream);
}

template <typename S>
static cudaError_t lstm_backward_t(const void* dy, const float* gates, const float* cs, const void* whh,
                                   const void* whh_rev, const int* len, void* dg, unsigned long long* bar, int T, int N,
                                   int H, int u, int rows, cudaStream_t stream) {
    const int g = (H + u - 1) / u;
    const LstmBwdArgs<S> p{static_cast<const S*>(dy), gates, cs,
                           {static_cast<const S*>(whh), static_cast<const S*>(whh_rev)}, len, static_cast<S*>(dg), bar,
                           T, N, H, u, rows, g};
    const size_t smem = sizeof(S) * ((size_t)4 * u * H + (size_t)rows * 4 * H) + sizeof(float) * (size_t)2 * u * N;
    return lstm_launch(lstm_bwd_kernel<S>, p, whh_rev ? 2 * g : g, smem, stream);
}

cudaError_t launch_lstm_forward(const void* gx, const void* whh, const void* whh_rev, const int* len, void* y,
                                float* gates, float* cs, unsigned long long* bar, int T, int N, int H, int u, int rows,
                                cudaStream_t stream, Dtype dtype) {
    if (!lstm_shape_ok(T, N, H, u, rows)) return cudaErrorInvalidValue;
    return with_dtype(dtype, [&](auto e) {
        return lstm_forward_t<decltype(e)>(gx, whh, whh_rev, len, y, gates, cs, bar, T, N, H, u, rows, stream);
    });
}

cudaError_t launch_lstm_backward(const void* dy, const float* gates, const float* cs, const void* whh,
                                 const void* whh_rev, const int* len, void* dg, unsigned long long* bar, int T, int N,
                                 int H, int u, int rows, cudaStream_t stream, Dtype dtype) {
    if (!lstm_shape_ok(T, N, H, u, rows)) return cudaErrorInvalidValue;
    return with_dtype(dtype, [&](auto e) {
        return lstm_backward_t<decltype(e)>(dy, gates, cs, whh, whh_rev, len, dg, bar, T, N, H, u, rows, stream);
    });
}

// ---- One layer of a stacked language-model LSTM (PTB): carried state, step product on the tensor cores ----------------
//
// lstm_seq_fwd_kernel / lstm_seq_bwd_kernel run the recurrence above for a single uni-directional layer in which every
// row has length T, from an initial state (h0, c0), in bf16 or fp16 (below) and in fp32 (the fp32 section further down:
// same kernels, another prologue and step product).  The split into CTAs of u units, the grid
// barrier, the cell code and the stores are those of lstm_fwd_kernel / lstm_bwd_kernel; what differs:
//   - forward, step 0 stages h0 where the other steps stage y_{t-1}, and c starts from c0.  h_n = y[T-1] and
//     c_n = cs[T-1], so neither has a store of its own;
//   - backward, at t = T-1 the recurrent dh is dh_n and the carried dc is dc_n (either null: 0); c_{-1} is c0, and the
//     carried dc after t = 0 is written to dc0 (fp32).  dh0 = dgates_0 W_hh is a GEMM in torch;
//   - the step product runs on mma.sync m16n8k16 with fp32 accumulation (lstm_mma_dots): batch rows on the M side (a
//     missing row is a zero fragment), the CTA's weight rows on the n side (forward: its 4u gate rows of W_hh;
//     backward: its u columns), K = H (forward) or 4H (backward).  Rows of both operands lie lstm_seq_ld(K) elements
//     apart in shared memory, zero from K on: that pads K to a multiple of 16 and makes the row stride an odd multiple of
//     16 bytes, so the eight rows a fragment load touches fall in distinct banks.  Weight rows are not padded: a weight
//     row past the CTA's last is a zero fragment too.
//   - a warp task is one (16 batch rows, 8 weight rows, 1 / ksplit of the k steps); its k steps alternate between two
//     accumulators, added at the end.  With ksplit > 1 the partial sums are added in split order after a block barrier,
//     so, as everywhere in this file, every sum has a fixed order whichever warp runs it and no atomics touch data.
// lstm_seq_ksplit is mirrored by ops/fused_lstm.py, which sizes the shared memory from it.

template <typename S>
struct LstmSeqFwdArgs {
    const S* gx;
    const S* whh;
    const S* h0;
    const float* c0;
    S* y;
    float* gates;
    float* cs;
    unsigned long long* bar;
    int T, N, H, u, rows, ksplit;
    int r_on, kc;                   // fp32 only: weight rows in shared memory, staged chunk width (lstm_f32_product)
};

template <typename S>
struct LstmSeqBwdArgs {
    const S* dy;
    const float* gates;
    const float* cs;
    const S* whh;
    const float* c0;
    const S* dhn;                   // null: 0
    const float* dcn;               // null: 0
    S* dg;
    float* dc0;
    unsigned long long* bar;
    int T, N, H, u, rows, ksplit;
    int r_on, kc;                   // fp32 only, as LstmSeqFwdArgs
};

__host__ __device__ __forceinline__ int lstm_seq_ld(int K) { return ((K + 15) & ~15) + 8; }

// K splits of a step product over `rows` batch rows and R weight rows: enough to give every warp a task, at most one
// per k step.
__host__ __device__ __forceinline__ int lstm_seq_ksplit(int rows, int R, int K) {
    const int tiles = ((rows + 15) >> 4) * ((R + 7) >> 3);
    return max(1, min(kLstmWarps / tiles, (K + 15) >> 4));
}

__device__ __forceinline__ uint32_t lstm_u32(const void* p) { return *reinterpret_cast<const uint32_t*>(p); }

// sP[(ks nc + j) R + r] = the ks-th split of sum_k sV[j ld + k] sW[r ld + k], j < nc, r < R, over k < 16 KS (zero
// past K).  Fragment layout as the PTX ISA's m16n8k16 row.col: lane (g, t) = (lane / 4, lane % 4) loads A rows g and
// g + 8 and B row g, at k = 2t and 2t + 8.
template <typename S>
__device__ __forceinline__ void lstm_mma_dots(const S* __restrict__ sW, const S* __restrict__ sV,
                                              float* __restrict__ sP, int R, int ld, int KS, int nc, int ksplit) {
    const int lane = lane_id(), warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const int NT = (R + 7) >> 3, tasks = ((nc + 15) >> 4) * NT * ksplit;
    for (int task = warp; task < tasks; task += kLstmWarps) {
        const int ks = task % ksplit, tile = task / ksplit, mt = tile / NT, nt = tile - mt * NT;
        const int j0 = mt * 16 + g, j1 = j0 + 8, r = nt * 8 + g;
        const bool ok0 = j0 < nc, ok1 = j1 < nc, okw = r < R;
        const S* a0 = sV + (size_t)(ok0 ? j0 : 0) * ld + 2 * t;
        const S* a1 = sV + (size_t)(ok1 ? j1 : 0) * ld + 2 * t;
        const S* b = sW + (size_t)(okw ? r : 0) * ld + 2 * t;
        const int k_lo = ks * KS / ksplit, k_hi = (ks + 1) * KS / ksplit;
        float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
        auto step = [&](float (&d)[4], int kk) {
            const int k = kk * 16;
            const uint32_t fa[4] = {ok0 ? lstm_u32(a0 + k) : 0u, ok1 ? lstm_u32(a1 + k) : 0u,
                                    ok0 ? lstm_u32(a0 + k + 8) : 0u, ok1 ? lstm_u32(a1 + k + 8) : 0u};
            const uint32_t fb[2] = {okw ? lstm_u32(b + k) : 0u, okw ? lstm_u32(b + k + 8) : 0u};
            mma_m16n8k16<S>(d, fa, fb);
        };
        int kk = k_lo;
#pragma unroll 2
        for (; kk + 1 < k_hi; kk += 2) {
            step(acc[0], kk);
            step(acc[1], kk + 1);
        }
        if (kk < k_hi) step(acc[0], kk);
        float* P = sP + (size_t)ks * nc * R;
        const int rc = nt * 8 + 2 * t;                          // C fragment: rows g, g + 8; columns 2t, 2t + 1
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int j = h ? j1 : j0;
            if (!(h ? ok1 : ok0)) continue;
            if (rc < R) P[j * R + rc] = acc[0][2 * h] + acc[1][2 * h];
            if (rc + 1 < R) P[j * R + rc + 1] = acc[0][2 * h + 1] + acc[1][2 * h + 1];
        }
    }
}

// out[r N + n] = sum_k sW[r ld + k] V[n K + k] for r < R and all N rows of V (global [N, K], possibly written in this
// launch), `rows` at a time through sV (whose rows are zero from K to ld, as are sW's).
template <typename S>
__device__ __forceinline__ void lstm_seq_product(const S* __restrict__ sW, S* __restrict__ sV, float* __restrict__ sP,
                                                 float* __restrict__ out, const S* V, int R, int K, int N, int rows,
                                                 int ksplit) {
    using Vec = typename Elem<S>::V;
    const int ld = lstm_seq_ld(K), K4 = K >> 2, KS = (K + 15) >> 4;
    for (int n0 = 0; n0 < N; n0 += rows) {
        const int nc = min(rows, N - n0);
        const Vec* src = reinterpret_cast<const Vec*>(V + (size_t)n0 * K);
        for (int i = threadIdx.x; i < nc * K4; i += kLstmThreads) {
            const int j = i / K4, k = i - j * K4;
            reinterpret_cast<Vec*>(sV + (size_t)j * ld)[k] = __ldcg(src + i);
        }
        __syncthreads();
        lstm_mma_dots(sW, sV, sP, R, ld, KS, nc, ksplit);
        __syncthreads();
        for (int i = threadIdx.x; i < R * nc; i += kLstmThreads) {
            const int r = i / nc, j = i - r * nc;
            float a = sP[j * R + r];
            for (int ks = 1; ks < ksplit; ++ks) a += sP[((size_t)ks * nc + j) * R + r];
            out[r * N + n0 + j] = a;
        }
    }
    __syncthreads();
}

// Zero columns [K, ld) of `nrows` shared-memory rows.
template <typename S>
__device__ __forceinline__ void lstm_seq_zero_tail(S* s, int nrows, int K) {
    const int ld = lstm_seq_ld(K), w = ld - K;
    for (int i = threadIdx.x; i < nrows * w; i += kLstmThreads) {
        const int r = i / w;
        s[(size_t)r * ld + K + (i - r * w)] = Elem<S>::narrow1(0.f);
    }
}

// ---- fp32: W_hh split between shared memory and L2, 3xTF32 step product ---------------------------------------------
//
// The fp32 slice of W_hh at H = 1500 (288 KB per CTA at u = 12) does not fit in shared memory, but all of W_hh (36 MB)
// fits in L2.  So the CTA keeps its first r_on weight rows in shared memory, loaded once, and reads the others from
// global memory at every step with an L2 evict_last policy; nothing else runs during the launch to evict them.  The
// step operand (all N batch rows) is staged kc columns at a time, double-buffered with cp.async, which leaves most of
// shared memory to the weights.  The product runs in 3xTF32 on mma.sync m16n8k8 (elem.cuh), batch rows on the M side,
// weight rows on the n side.  Rows of W in shared memory lie lstm_f32_ld(K) floats apart and staged rows kc + 4 apart,
// both = 4 (mod 8): the eight rows a fragment load touches (g = 0..7, column t) then fall in distinct banks.
// Backward, the weight rows are the CTA's u columns of W_hh, which the fp32 launch reads as rows of W_hh^T [H][4H], so
// that a streamed row is contiguous.  lstm_f32_ld and lstm_f32_ksplit are mirrored by ops/fused_lstm.py.

__host__ __device__ __forceinline__ int lstm_f32_ld(int K) { return ((K + 7) & ~7) + 4; }

// One task per warp: 8 weight rows and 1 / ksplit of each chunk's k8 steps, for every batch row.
__host__ __device__ __forceinline__ int lstm_f32_ksplit(int R) { return max(1, kLstmWarps / ((R + 7) >> 3)); }

__device__ __forceinline__ void lstm_cp_async16(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src)
                 : "memory");
}
__device__ __forceinline__ void lstm_cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void lstm_cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

__device__ __forceinline__ uint64_t lstm_evict_last_policy() {
    uint64_t pol;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
// A weight, read-only for the whole launch: through the non-coherent path, kept in L2.
__device__ __forceinline__ float lstm_ldg_last(const float* p, uint64_t pol) {
    float v;
    asm("ld.global.nc.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(pol));
    return v;
}

// Zero columns [K, ld) of `nrows` fp32 shared-memory rows `ld` apart.
__device__ __forceinline__ void lstm_f32_zero_tail(float* s, int nrows, int K, int ld) {
    const int w = ld - K;
    for (int i = threadIdx.x; i < nrows * w; i += kLstmThreads) {
        const int r = i / w;
        s[(size_t)r * ld + K + (i - r * w)] = 0.f;
    }
}

// out[r N + n] = sum_k W_r[k] V[n K + k] for r < R and n < N; V is global [N, K], possibly written in this launch.
// W_r is row r of sW (lstm_f32_ld(K) apart, zero from K on) for r < r_on, else the global row grow(r) (null: a zero
// row).  V goes through sV [2][N][kc + 4] one kc-column chunk at a time, the next chunk's cp.async under this one's
// products; zero columns pad the last chunk to a whole k8 step.  Warp w < NT ksplit (NT = ceil(R / 8)) takes weight
// rows [8 nt, 8 nt + 8), nt = w / ksplit, and the (w % ksplit)-th part of every chunk's k8 steps, for all batch rows
// (16 per M tile, rows past N zero fragments): so each streamed weight element is loaded once per step.  Its sums stay
// in registers across the chunks, go to sP [ksplit][N][R] at the end, and are added in split order: fixed whichever warp
// runs what, and no atomics.
template <class RowPtr>
__device__ __forceinline__ void lstm_f32_product(const float* __restrict__ sW, float* __restrict__ sV,
                                                 float* __restrict__ sP, float* __restrict__ out, const float* V, int R,
                                                 int r_on, int K, int N, int kc, int ksplit, RowPtr grow,
                                                 uint64_t pol) {
    constexpr int kMT = (kMaxLstmBatch + 15) / 16, kPf = 8;        // M tiles at most; k8 steps of weights in flight
    const int lane = lane_id(), warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const int ldw = lstm_f32_ld(K), ldv = kc + 4, K4 = K >> 2, nch = (K + kc - 1) / kc, MT = (N + 15) >> 4;
    const int nt = warp / ksplit, ks = warp - nt * ksplit, r = nt * 8 + g;
    const bool active = r - g < R, on = r < r_on;
    const float* wg = active && !on && r < R ? grow(r) : nullptr;
    const float* ws = sW + (size_t)(on ? r : 0) * ldw;
    float acc[kMT][4];
#pragma unroll
    for (int m = 0; m < kMT; ++m) acc[m][0] = acc[m][1] = acc[m][2] = acc[m][3] = 0.f;
    auto stage = [&](int c) {
        float* d = sV + (size_t)(c & 1) * N * ldv;
        const int k0 = c * kc, w4 = min(kc >> 2, K4 - (k0 >> 2)), pad = ((4 * w4 + 7) & ~7) - 4 * w4;
        for (int i = threadIdx.x; i < N * w4; i += kLstmThreads) {
            const int n = i / w4, k = i - n * w4;
            lstm_cp_async16(d + (size_t)n * ldv + 4 * k, V + (size_t)n * K + k0 + 4 * k);
        }
        lstm_cp_async_commit();
        for (int i = threadIdx.x; i < N * pad; i += kLstmThreads) d[(size_t)(i / pad) * ldv + 4 * w4 + i % pad] = 0.f;
    };
    stage(0);
    for (int c = 0; c < nch; ++c) {
        lstm_cp_async_wait_all();
        __syncthreads();                // chunk c landed, and every warp is done with chunk c - 1's buffer
        if (c + 1 < nch) stage(c + 1);
        if (!active) continue;
        const float* v = sV + (size_t)(c & 1) * N * ldv;
        const int k0 = c * kc, S = (min(kc, K - k0) + 7) >> 3;
        const int s_hi = (ks + 1) * S / ksplit;
        for (int s0 = ks * S / ksplit; s0 < s_hi; s0 += kPf) {
            float b[kPf][2];
#pragma unroll
            for (int i = 0; i < kPf; ++i) {             // fragment b0 (k = t), b1 (k = t + 4) of weight row r
                const int k = k0 + 8 * (s0 + i) + t;
                const bool in = s0 + i < s_hi;
                if (on) {
                    b[i][0] = in ? ws[k] : 0.f;
                    b[i][1] = in ? ws[k + 4] : 0.f;
                } else {
                    b[i][0] = wg && in && k < K ? lstm_ldg_last(wg + k, pol) : 0.f;
                    b[i][1] = wg && in && k + 4 < K ? lstm_ldg_last(wg + k + 4, pol) : 0.f;
                }
            }
#pragma unroll
            for (int i = 0; i < kPf; ++i) {
                if (s0 + i >= s_hi) break;
                uint32_t bh[2], bl[2];
                tf32_split(b[i][0], bh[0], bl[0]);
                tf32_split(b[i][1], bh[1], bl[1]);
                const int kl = 8 * (s0 + i) + t;
#pragma unroll
                for (int m = 0; m < kMT; ++m) {
                    if (m >= MT) break;
                    const int j0 = 16 * m + g, j1 = j0 + 8;
                    const float* v0 = v + (size_t)(j0 < N ? j0 : 0) * ldv + kl;
                    const float* v1 = v + (size_t)(j1 < N ? j1 : 0) * ldv + kl;
                    const float a[4] = {j0 < N ? v0[0] : 0.f, j1 < N ? v1[0] : 0.f, j0 < N ? v0[4] : 0.f,
                                        j1 < N ? v1[4] : 0.f};
                    uint32_t ah[4], al[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) tf32_split(a[q], ah[q], al[q]);
                    mma_m16n8k8_3xtf32(acc[m], ah, al, bh, bl);
                }
            }
        }
    }
    if (active) {
        float* P = sP + (size_t)ks * N * R;
        const int rc = nt * 8 + 2 * t;                              // C fragment: rows g, g + 8; columns 2t, 2t + 1
#pragma unroll
        for (int m = 0; m < kMT; ++m) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int j = 16 * m + g + 8 * h;
                if (j >= N) continue;
                if (rc < R) P[j * R + rc] = acc[m][2 * h];
                if (rc + 1 < R) P[j * R + rc + 1] = acc[m][2 * h + 1];
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < R * N; i += kLstmThreads) {
        const int rr = i / N, n = i - rr * N;
        float a = sP[n * R + rr];
        for (int k = 1; k < ksplit; ++k) a += sP[((size_t)k * N + n) * R + rr];
        out[i] = a;
    }
    __syncthreads();
}

// Shared memory: W [4u][ld] and h_{t-1} rows [rows][ld] of S, ld = lstm_seq_ld(H) | partial sums [ksplit][rows][4u],
// gate sums [4u][N] and c [u][N] of float.  ld % 8 == 0 keeps every section 16-byte aligned.
// fp32: W [r_on][lstm_f32_ld(H)] | two h_{t-1} chunks [2][N][kc + 4] | partial sums [ksplit][N][4u] | gate sums, c.
template <typename S>
__global__ void __launch_bounds__(kLstmThreads, 1) lstm_seq_fwd_kernel(const LstmSeqFwdArgs<S> p) {
    using El = Elem<S>;
    using Vec = typename El::V;
    constexpr bool kF32 = std::is_same<S, float>::value;
    extern __shared__ float4 lstm_smem[];
    const int H = p.H, N = p.N, u = p.u, R = 4 * u, H4 = H >> 2;
    const int ld = kF32 ? lstm_f32_ld(H) : lstm_seq_ld(H), won = kF32 ? p.r_on : R;    // rows of W in shared memory
    const int u0 = blockIdx.x * u, nu = min(u, H - u0);
    S* sW = reinterpret_cast<S*>(lstm_smem);
    S* sV = sW + (size_t)won * ld;
    float* sP = reinterpret_cast<float*>(sV + (kF32 ? (size_t)2 * N * (p.kc + 4) : (size_t)p.rows * ld));
    float* sG = sP + (size_t)p.ksplit * (kF32 ? N : p.rows) * R;
    float* sC = sG + R * N;
    for (int i = threadIdx.x; i < won * H4; i += kLstmThreads) {    // local row q u + j = W_hh row q H + u0 + j
        const int lr = i / H4, k = i - lr * H4, q = lr / u, j = lr - q * u;
        Vec v = El::zero();
        if (j < nu) v = __ldg(reinterpret_cast<const Vec*>(p.whh + (size_t)(q * H + u0 + j) * H) + k);
        reinterpret_cast<Vec*>(sW + (size_t)lr * ld)[k] = v;
    }
    uint64_t pol = 0;
    if constexpr (kF32) {
        lstm_f32_zero_tail(sW, won, H, ld);
        pol = lstm_evict_last_policy();
    } else {
        lstm_seq_zero_tail(sW, R, H);
        lstm_seq_zero_tail(sV, p.rows, H);
    }
    auto grow = [&](int lr) -> const float* {                       // fp32: streamed local row lr, as above
        const int q = lr / u, j = lr - q * u;
        return j < nu ? reinterpret_cast<const float*>(p.whh) + (size_t)(q * H + u0 + j) * H : nullptr;
    };
    for (int i = threadIdx.x; i < u * N; i += kLstmThreads) {
        const int j = i / N, n = i - j * N;
        sC[i] = j < nu ? __ldg(p.c0 + (size_t)n * H + u0 + j) : 0.f;
    }
    for (int s = 0; s < p.T; ++s) {
        const S* hp = s == 0 ? p.h0 : p.y + (size_t)(s - 1) * N * H;
        if constexpr (kF32)
            lstm_f32_product(sW, sV, sP, sG, hp, R, won, H, N, p.kc, p.ksplit, grow, pol);
        else
            lstm_seq_product(sW, sV, sP, sG, hp, R, H, N, p.rows, p.ksplit);
        for (int i = threadIdx.x; i < nu * N; i += kLstmThreads) {
            const int j = i / N, n = i - j * N, unit = u0 + j;
            const size_t row = (size_t)s * N + n;
            const S* gx = p.gx + row * 4 * H + unit;
            float* gs = p.gates + row * 4 * H + unit;
            const size_t o = row * H + unit;
            const float gi = lstm_sigmoid(sG[(0 * u + j) * N + n] + El::ld(gx));
            const float gf = lstm_sigmoid(sG[(1 * u + j) * N + n] + El::ld(gx + H));
            const float gg = tanhf(sG[(2 * u + j) * N + n] + El::ld(gx + 2 * H));
            const float go = lstm_sigmoid(sG[(3 * u + j) * N + n] + El::ld(gx + 3 * H));
            const float c = gf * sC[j * N + n] + gi * gg;
            sC[j * N + n] = c;
            gs[0] = gi; gs[H] = gf; gs[2 * H] = gg; gs[3 * H] = go;
            p.cs[o] = c;
            p.y[o] = El::narrow1(go * tanhf(c));
        }
        if (s + 1 < p.T) grid_sync(p.bar);
    }
}

// Shared memory: W^T [u][ld] and dgates_{t+1} rows [rows][ld] of S, ld = lstm_seq_ld(4H) | partial sums
// [ksplit][rows][u], dh_rec [u][N] and carried dc [u][N] of float.
template <typename S>
__global__ void __launch_bounds__(kLstmThreads, 1) lstm_seq_bwd_kernel(const LstmSeqBwdArgs<S> p) {
    using El = Elem<S>;
    constexpr bool kF32 = std::is_same<S, float>::value;
    extern __shared__ float4 lstm_smem[];
    const int H = p.H, N = p.N, u = p.u, G = 4 * H;
    const int ld = kF32 ? lstm_f32_ld(G) : lstm_seq_ld(G), won = kF32 ? p.r_on : u;     // rows of W^T in shared memory
    const int u0 = blockIdx.x * u, nu = min(u, H - u0);
    S* sW = reinterpret_cast<S*>(lstm_smem);
    S* sV = sW + (size_t)won * ld;
    float* sP = reinterpret_cast<float*>(sV + (kF32 ? (size_t)2 * N * (p.kc + 4) : (size_t)p.rows * ld));
    float* sD = sP + (size_t)p.ksplit * (kF32 ? N : p.rows) * u;
    float* sDC = sD + u * N;
    uint64_t pol = 0;
    if constexpr (kF32) {                                           // whh is W_hh^T: sW[j][k] = W_hh^T[u0 + j][k]
        const int G4 = G >> 2;
        for (int i = threadIdx.x; i < won * G4; i += kLstmThreads) {
            const int j = i / G4, k = i - j * G4;
            reinterpret_cast<float4*>(sW + (size_t)j * ld)[k] =
                j < nu ? __ldg(reinterpret_cast<const float4*>(p.whh + (size_t)(u0 + j) * G) + k) : El::zero();
        }
        lstm_f32_zero_tail(sW, won, G, ld);
        pol = lstm_evict_last_policy();
    } else {
        for (int i = threadIdx.x; i < u * G; i += kLstmThreads) {   // sW[j][k] = W_hh[k][u0 + j]
            const int k = i / u, j = i - k * u;
            sW[(size_t)j * ld + k] = j < nu ? __ldg(p.whh + (size_t)k * H + u0 + j) : El::narrow1(0.f);
        }
        lstm_seq_zero_tail(sW, u, G);
        lstm_seq_zero_tail(sV, p.rows, G);
    }
    auto grow = [&](int j) -> const float* {                        // fp32: streamed row j of W_hh^T's slice
        return j < nu ? reinterpret_cast<const float*>(p.whh) + (size_t)(u0 + j) * G : nullptr;
    };
    for (int i = threadIdx.x; i < u * N; i += kLstmThreads) {
        const int j = i / N, n = i - j * N;
        const size_t o = (size_t)n * H + u0 + j;
        sD[i] = j < nu && p.dhn ? El::ld(p.dhn + o) : 0.f;
        sDC[i] = j < nu && p.dcn ? __ldg(p.dcn + o) : 0.f;
    }
    __syncthreads();
    for (int s = p.T - 1; s >= 0; --s) {
        if (s < p.T - 1) {
            const S* dgn = p.dg + (size_t)(s + 1) * N * G;
            if constexpr (kF32)
                lstm_f32_product(sW, sV, sP, sD, dgn, u, won, G, N, p.kc, p.ksplit, grow, pol);
            else
                lstm_seq_product(sW, sV, sP, sD, dgn, u, G, N, p.rows, p.ksplit);
        }
        for (int i = threadIdx.x; i < nu * N; i += kLstmThreads) {
            const int j = i / N, n = i - j * N, unit = u0 + j;
            const size_t row = (size_t)s * N + n;
            const size_t o = row * H + unit;
            S* dg = p.dg + row * G + unit;
            const float* gs = p.gates + row * G + unit;
            const float gi = __ldg(gs), gf = __ldg(gs + H), gg = __ldg(gs + 2 * H), go = __ldg(gs + 3 * H);
            const float tc = tanhf(__ldg(p.cs + o));
            const float cp = s > 0 ? __ldg(p.cs + o - (size_t)N * H) : __ldg(p.c0 + (size_t)n * H + unit);
            const float dh = El::ld(p.dy + o) + sD[j * N + n];
            const float dc = dh * go * (1.f - tc * tc) + sDC[j * N + n];
            dg[0] = El::narrow1(dc * gg * gi * (1.f - gi));
            dg[H] = El::narrow1(dc * cp * gf * (1.f - gf));
            dg[2 * H] = El::narrow1(dc * gi * (1.f - gg * gg));
            dg[3 * H] = El::narrow1(dh * tc * go * (1.f - go));
            sDC[j * N + n] = dc * gf;
            if (s == 0) p.dc0[(size_t)n * H + unit] = dc * gf;
        }
        if (s > 0) grid_sync(p.bar);
    }
}

static size_t lstm_seq_fwd_smem(int H, int N, int u, int rows, int elem) {
    const int R = 4 * u;
    return (size_t)elem * (R + rows) * lstm_seq_ld(H) +
           sizeof(float) * ((size_t)lstm_seq_ksplit(rows, R, H) * rows * R + (size_t)R * N + (size_t)u * N);
}

static size_t lstm_seq_bwd_smem(int H, int N, int u, int rows, int elem) {
    return (size_t)elem * (u + rows) * lstm_seq_ld(4 * H) +
           sizeof(float) * ((size_t)lstm_seq_ksplit(rows, u, 4 * H) * rows * u + (size_t)2 * u * N);
}

// fp32: r_on weight rows in shared memory, two staged chunks of kc columns of the N batch rows.
static size_t lstm_f32_fwd_smem(int H, int N, int u, int r_on, int kc) {
    const int R = 4 * u;
    return sizeof(float) * ((size_t)r_on * lstm_f32_ld(H) + (size_t)2 * N * (kc + 4) +
                            (size_t)lstm_f32_ksplit(R) * N * R + (size_t)R * N + (size_t)u * N);
}

static size_t lstm_f32_bwd_smem(int H, int N, int u, int r_on, int kc) {
    return sizeof(float) * ((size_t)r_on * lstm_f32_ld(4 * H) + (size_t)2 * N * (kc + 4) +
                            (size_t)lstm_f32_ksplit(u) * N * u + (size_t)2 * u * N);
}

// The fp32 split: R weight rows per CTA, at most 8 per warp; r_on of them on chip; chunks of whole k8 steps.
static bool lstm_f32_ok(int N, int R, int r_on, int kc) {
    return N <= kMaxLstmBatch && R <= 8 * kLstmWarps && r_on >= 0 && r_on <= R && kc > 0 && kc % 8 == 0;
}

cudaError_t launch_lstm_seq_forward(const void* gx, const void* whh, const void* h0, const float* c0, void* y,
                                    float* gates, float* cs, unsigned long long* bar, int T, int N, int H, int u,
                                    int rows, int r_on, int kc, cudaStream_t stream, Dtype dtype) {
    if (!lstm_shape_ok(T, N, H, u, rows)) return cudaErrorInvalidValue;
    if (dtype == Dtype::kF32 && !lstm_f32_ok(N, 4 * u, r_on, kc)) return cudaErrorInvalidValue;
    return with_dtype(dtype, [&](auto e) {
        using S = decltype(e);
        constexpr bool kF32 = std::is_same<S, float>::value;
        const LstmSeqFwdArgs<S> p{static_cast<const S*>(gx), static_cast<const S*>(whh), static_cast<const S*>(h0), c0,
                                  static_cast<S*>(y), gates, cs, bar, T, N, H, u, rows,
                                  kF32 ? lstm_f32_ksplit(4 * u) : lstm_seq_ksplit(rows, 4 * u, H), r_on, kc};
        const size_t smem = kF32 ? lstm_f32_fwd_smem(H, N, u, r_on, kc) : lstm_seq_fwd_smem(H, N, u, rows, sizeof(S));
        return lstm_launch(lstm_seq_fwd_kernel<S>, p, (H + u - 1) / u, smem, stream);
    });
}

cudaError_t launch_lstm_seq_backward(const void* dy, const float* gates, const float* cs, const void* whh,
                                     const float* c0, const void* dhn, const float* dcn, void* dg, float* dc0,
                                     unsigned long long* bar, int T, int N, int H, int u, int rows, int r_on, int kc,
                                     cudaStream_t stream, Dtype dtype) {
    if (!lstm_shape_ok(T, N, H, u, rows)) return cudaErrorInvalidValue;
    if (dtype == Dtype::kF32 && !lstm_f32_ok(N, u, r_on, kc)) return cudaErrorInvalidValue;
    return with_dtype(dtype, [&](auto e) {
        using S = decltype(e);
        constexpr bool kF32 = std::is_same<S, float>::value;
        const LstmSeqBwdArgs<S> p{static_cast<const S*>(dy), gates, cs, static_cast<const S*>(whh), c0,
                                  static_cast<const S*>(dhn), dcn, static_cast<S*>(dg), dc0, bar, T, N, H, u, rows,
                                  kF32 ? lstm_f32_ksplit(u) : lstm_seq_ksplit(rows, u, 4 * H), r_on, kc};
        const size_t smem = kF32 ? lstm_f32_bwd_smem(H, N, u, r_on, kc) : lstm_seq_bwd_smem(H, N, u, rows, sizeof(S));
        return lstm_launch(lstm_seq_bwd_kernel<S>, p, (H + u - 1) / u, smem, stream);
    });
}

}  // namespace okt
