// Fused batch-norm of the AN4 DeepSpeech model over the frames of the longest utterance, forward and backward, in
// training mode.  len [N] int32 are the utterances' frame lengths on the device; Tb is the tensor's frame width and
//
//   Tm = min(max(0, max_n len_n), Tb).
//
// Two layouts:
//   - conv block, x [N, C, F, Tb] (NCHW): the masked Conv -> BN -> Hardtanh(0, 20) of DeepSpeech's conv stack.  Frame
//     (n, t) is valid when t < len_n.  The statistics of channel c are over (n, f, t < Tm), an invalid frame read as 0;
//     the count is N F Tm.  y = valid ? clamp(a (x - mean) + beta, 0, 20) : +0, with a = gamma rstd.  Backward: dz = dy
//     where the frame is valid and 0 < z < 20 (torch's strict hardtanh backward), else 0; dbeta = sum dz,
//     dgamma = sum dz xhat over the counted frames, dx = valid ? a (dz - dbeta / n - xhat dgamma / n) : +0.
//   - sequence, x [Tb, N, C] (BatchNorm1d on T N rows): the statistics are over the row prefix [0, Tm N); y and dx
//     are +0 on the rows after it.
// mean and rstd = 1 / sqrt(var + eps) (biased var) are saved per channel for the backward pass.  The running statistics
// move as torch's: r = (1 - momentum) r + momentum s, with the unbiased variance var n / (n - 1); for a count of n <= 1
// the biased variance (0 at n = 1) is used instead, where torch raises, so running_var stays finite.  The first CTA
// adds 1 to num_batches_tracked (if given).
//
// Summation order: two passes (the sum, then the squared deviations from the mean), each thread adding its fixed
// share of the counted elements in order, then a fixed tree over the CTA.  The sums are accumulated in fp64 (the
// elements are widened exactly), so the statistics and dgamma / dbeta carry only their final rounding to fp32.  Conv block: one CTA of kFbnConvThreads
// per channel; warp w takes rows r = n F + f with r = w mod kFbnConvWarps, lane l the frames t = l mod 32 of each.
// Sequence: one CTA per kFbnSeqCols columns; thread (g, j) adds column j over the rows r = g mod kFbnSeqGroups, and
// the kFbnSeqGroups partial sums are added in a pairwise tree.  The order
// depends on (Tm, N, F, C) and the lengths only, never on Tb: a launch at a padded width equals, bit for bit, a launch
// on the tensor cropped to Tm frames.  No
// atomics, no grid-wide hand-off: every CTA owns its channels from the first load to the last store, and the elements
// are re-read (from L2) by each pass.
//
// Types: x, y, dy and dx are fp32, bf16 or fp16 (elem.cuh: widened exactly, fp32 arithmetic, y and dx rounded once);
// gamma, beta, the saved and running statistics and dgamma / dbeta are fp32.
#include "common.cuh"
#include "elem.cuh"
#include "oktopk.cuh"

namespace okt {

constexpr int kFbnConvThreads = 1024;
constexpr int kFbnConvWarps = kFbnConvThreads / 32;
constexpr int kFbnSeqCols = 16;
constexpr int kFbnSeqGroups = 32;
constexpr int kFbnSeqThreads = kFbnSeqCols * kFbnSeqGroups;
constexpr float kFbnClampMax = 20.f;

__device__ __forceinline__ int fbn_bound(const int* len, int N, int Tb) {
    int m = 0;
    for (int n = 0; n < N; ++n) m = max(m, __ldg(len + n));
    return min(m, Tb);
}

// The sum of v over the CTA of kFbnConvThreads, the same in every thread: a shuffle tree in each warp, then the same
// tree over the warps' sums.  Ends with a barrier, so `sh` (kFbnConvWarps floats) may be reused at once.
__device__ __forceinline__ double fbn_conv_sum(double v, double* sh) {
    v = warp_sum_d(v);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    v = warp_sum_d(sh[threadIdx.x & 31]);
    __syncthreads();
    return v;
}

// The sum over the kFbnSeqGroups row groups of this thread's column, a pairwise tree in group order, the same in
// every group.
__device__ __forceinline__ double fbn_seq_sum(double v, double (*sh)[kFbnSeqCols]) {
    const int j = threadIdx.x % kFbnSeqCols, g = threadIdx.x / kFbnSeqCols;
    sh[g][j] = v;
    __syncthreads();
#pragma unroll
    for (int s = kFbnSeqGroups / 2; s > 0; s >>= 1) {
        if (g < s) sh[g][j] += sh[g + s][j];
        __syncthreads();
    }
    const double r = sh[0][j];
    __syncthreads();
    return r;
}

// The channel's statistics and their running averages, by one thread.
__device__ __forceinline__ void fbn_store_stats(int c, float mean, float var, float rstd, long long cnt, float* mean_out,
                                                float* rstd_out, float* rmean, float* rvar, float momentum) {
    mean_out[c] = mean;
    rstd_out[c] = rstd;
    const float unbiased = cnt > 1 ? var * ((float)cnt / (float)(cnt - 1)) : var;
    rmean[c] = (1.f - momentum) * rmean[c] + momentum * mean;
    rvar[c] = (1.f - momentum) * rvar[c] + momentum * unbiased;
}

__device__ __forceinline__ float fbn_clamp(float z) { return z < 0.f ? 0.f : (z > kFbnClampMax ? kFbnClampMax : z); }

// ------------------------------------------------------------------------------------------------------ conv block
template <typename T>
__global__ void __launch_bounds__(kFbnConvThreads)
fbn_conv_fwd_kernel(const T* __restrict__ x, const int* __restrict__ len, const float* __restrict__ gamma,
                    const float* __restrict__ beta, T* __restrict__ y, float* __restrict__ mean_out,
                    float* __restrict__ rstd_out, float* rmean, float* rvar, long long* nbt, int N, int C, int F,
                    int Tb, float eps, float momentum) {
    __shared__ double sh[kFbnConvWarps];
    const int c = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int Tm = fbn_bound(len, N, Tb), R = N * F;
    const long long cnt = (long long)R * Tm;
    const double inv_cnt = 1.0 / (double)max(cnt, 1LL);

    double s = 0.0;
    for (int r = warp; r < R; r += kFbnConvWarps) {
        const int n = r / F;
        const int L = min(__ldg(len + n), Tm);
        const T* p = x + ((size_t)(n * C + c) * F + (r - n * F)) * Tb;
        for (int t = lane; t < L; t += 32) s += (double)Elem<T>::ld(p + t);
    }
    const double mean_d = fbn_conv_sum(s, sh) * inv_cnt;

    double q = 0.0;
    for (int r = warp; r < R; r += kFbnConvWarps) {
        const int n = r / F;
        const int L = min(__ldg(len + n), Tm);
        const T* p = x + ((size_t)(n * C + c) * F + (r - n * F)) * Tb;
        for (int t = lane; t < Tm; t += 32) {
            const double d = (t < L ? (double)Elem<T>::ld(p + t) : 0.0) - mean_d;
            q = fma(d, d, q);
        }
    }
    const double var_d = fbn_conv_sum(q, sh) * inv_cnt;
    const float mean = (float)mean_d, var = (float)var_d;
    const float rstd = (float)(1.0 / sqrt(var_d + (double)eps));
    const float a = gamma[c] * rstd, b = beta[c];

    for (int r = warp; r < R; r += kFbnConvWarps) {
        const int n = r / F;
        const int L = min(__ldg(len + n), Tm);
        const size_t off = ((size_t)(n * C + c) * F + (r - n * F)) * Tb;
        for (int t = lane; t < Tb; t += 32)
            y[off + t] = Elem<T>::narrow1(t < L ? fbn_clamp(fmaf(Elem<T>::ld(x + off + t) - mean, a, b)) : 0.f);
    }
    if (threadIdx.x == 0) {
        fbn_store_stats(c, mean, var, rstd, cnt, mean_out, rstd_out, rmean, rvar, momentum);
        if (c == 0 && nbt != nullptr) *nbt += 1;
    }
}

template <typename T>
__global__ void __launch_bounds__(kFbnConvThreads)
fbn_conv_bwd_kernel(const T* __restrict__ x, const T* __restrict__ dy, const int* __restrict__ len,
                    const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ mean_in,
                    const float* __restrict__ rstd_in, T* __restrict__ dx, float* __restrict__ dgamma,
                    float* __restrict__ dbeta, int N, int C, int F, int Tb) {
    __shared__ double sh[kFbnConvWarps];
    const int c = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int Tm = fbn_bound(len, N, Tb), R = N * F;
    const long long cnt = (long long)R * Tm;
    const double inv_cnt = 1.0 / (double)max(cnt, 1LL);
    const float mean = mean_in[c], rstd = rstd_in[c];
    const float a = gamma[c] * rstd, b = beta[c];

    // only valid frames can have dz != 0, and the counted frames past a length add 0 to both sums
    double sd = 0.0, sdx = 0.0;
    for (int r = warp; r < R; r += kFbnConvWarps) {
        const int n = r / F;
        const int L = min(__ldg(len + n), Tm);
        const size_t off = ((size_t)(n * C + c) * F + (r - n * F)) * Tb;
        for (int t = lane; t < L; t += 32) {
            const float d = Elem<T>::ld(x + off + t) - mean;
            const float z = fmaf(d, a, b);
            const float g = (z > 0.f && z < kFbnClampMax) ? Elem<T>::ld(dy + off + t) : 0.f;
            sd += (double)g;
            sdx = fma((double)g, (double)Elem<T>::ld(x + off + t) - (double)mean, sdx);
        }
    }
    const double db_d = fbn_conv_sum(sd, sh);
    const double dg_d = fbn_conv_sum(sdx, sh) * (double)rstd;
    const float db = (float)db_d, dg = (float)dg_d;
    const float k1 = (float)(db_d * inv_cnt), k2 = (float)(dg_d * inv_cnt * (double)rstd);

    for (int r = warp; r < R; r += kFbnConvWarps) {
        const int n = r / F;
        const int L = min(__ldg(len + n), Tm);
        const size_t off = ((size_t)(n * C + c) * F + (r - n * F)) * Tb;
        for (int t = lane; t < Tb; t += 32) {
            float v = 0.f;
            if (t < L) {
                const float d = Elem<T>::ld(x + off + t) - mean;
                const float z = fmaf(d, a, b);
                const float g = (z > 0.f && z < kFbnClampMax) ? Elem<T>::ld(dy + off + t) : 0.f;
                v = a * (g - k1 - d * k2);
            }
            dx[off + t] = Elem<T>::narrow1(v);
        }
    }
    if (threadIdx.x == 0) {
        dgamma[c] = dg;
        dbeta[c] = db;
    }
}

// -------------------------------------------------------------------------------------------------------- sequence
template <typename T>
__global__ void __launch_bounds__(kFbnSeqThreads)
fbn_seq_fwd_kernel(const T* __restrict__ x, const int* __restrict__ len, const float* __restrict__ gamma,
                   const float* __restrict__ beta, T* __restrict__ y, float* __restrict__ mean_out,
                   float* __restrict__ rstd_out, float* rmean, float* rvar, long long* nbt, int N, int H, int Tb,
                   float eps, float momentum) {
    __shared__ double sh[kFbnSeqGroups][kFbnSeqCols];
    const int j = threadIdx.x % kFbnSeqCols, g = threadIdx.x / kFbnSeqCols;
    const int c = blockIdx.x * kFbnSeqCols + j;
    const bool own = c < H;
    const int cc = own ? c : H - 1;                  // threads past H read a real column and store nothing
    const int Tm = fbn_bound(len, N, Tb);
    const long long R = (long long)Tm * N, Rb = (long long)Tb * N;
    const double inv_cnt = 1.0 / (double)max(R, 1LL);

    double s = 0.0;
    for (long long r = g; r < R; r += kFbnSeqGroups) s += (double)Elem<T>::ld(x + r * H + cc);
    const double mean_d = fbn_seq_sum(s, sh) * inv_cnt;

    double q = 0.0;
    for (long long r = g; r < R; r += kFbnSeqGroups) {
        const double d = (double)Elem<T>::ld(x + r * H + cc) - mean_d;
        q = fma(d, d, q);
    }
    const double var_d = fbn_seq_sum(q, sh) * inv_cnt;
    if (!own) return;
    const float mean = (float)mean_d, var = (float)var_d;
    const float rstd = (float)(1.0 / sqrt(var_d + (double)eps));
    const float a = gamma[c] * rstd, b = beta[c];

    for (long long r = g; r < Rb; r += kFbnSeqGroups)
        y[r * H + c] = Elem<T>::narrow1(r < R ? fmaf(Elem<T>::ld(x + r * H + c) - mean, a, b) : 0.f);
    if (g == 0) {
        fbn_store_stats(c, mean, var, rstd, R, mean_out, rstd_out, rmean, rvar, momentum);
        if (c == 0 && nbt != nullptr) *nbt += 1;
    }
}

template <typename T>
__global__ void __launch_bounds__(kFbnSeqThreads)
fbn_seq_bwd_kernel(const T* __restrict__ x, const T* __restrict__ dy, const int* __restrict__ len,
                   const float* __restrict__ gamma, const float* __restrict__ mean_in,
                   const float* __restrict__ rstd_in, T* __restrict__ dx, float* __restrict__ dgamma,
                   float* __restrict__ dbeta, int N, int H, int Tb) {
    __shared__ double sh[kFbnSeqGroups][kFbnSeqCols];
    const int j = threadIdx.x % kFbnSeqCols, g = threadIdx.x / kFbnSeqCols;
    const int c = blockIdx.x * kFbnSeqCols + j;
    const bool own = c < H;
    const int cc = own ? c : H - 1;
    const int Tm = fbn_bound(len, N, Tb);
    const int R = Tm * N, Rb = Tb * N;
    const double inv_cnt = 1.0 / (double)max(R, 1);
    const float mean = mean_in[cc], rstd = rstd_in[cc];

    double sd = 0.0, sdx = 0.0;
    for (int r = g; r < R; r += kFbnSeqGroups) {
        const double gy = (double)Elem<T>::ld(dy + (size_t)r * H + cc);
        sd += gy;
        sdx = fma(gy, (double)Elem<T>::ld(x + (size_t)r * H + cc) - (double)mean, sdx);
    }
    const double db_d = fbn_seq_sum(sd, sh);
    const double dg_d = fbn_seq_sum(sdx, sh) * (double)rstd;
    if (!own) return;
    const float db = (float)db_d, dg = (float)dg_d;
    const float a = gamma[c] * rstd, k1 = (float)(db_d * inv_cnt), k2 = (float)(dg_d * inv_cnt * (double)rstd);

    for (int r = g; r < Rb; r += kFbnSeqGroups) {
        float v = 0.f;
        if (r < R) v = a * (Elem<T>::ld(dy + (size_t)r * H + c) - k1 - (Elem<T>::ld(x + (size_t)r * H + c) - mean) * k2);
        dx[(size_t)r * H + c] = Elem<T>::narrow1(v);
    }
    if (g == 0) {
        dgamma[c] = dg;
        dbeta[c] = db;
    }
}

bool frame_bn_supported(int conv, int N, int C, int F, int Tb) {
    if (N <= 0 || C <= 0 || Tb <= 0 || (conv && F <= 0)) return false;
    const long long per_channel = (long long)N * (conv ? F : 1) * Tb;
    return per_channel < (1LL << 24) && per_channel * C < (1LL << 40);   // counts exact in fp32
}

cudaError_t launch_frame_bn_forward(int conv, const void* x, const int* len, const float* gamma, const float* beta,
                                    void* y, float* mean, float* rstd, float* rmean, float* rvar, long long* nbt,
                                    int N, int C, int F, int Tb, float eps, float momentum, Dtype dtype,
                                    cudaStream_t stream) {
    return with_dtype(dtype, [&](auto tag) {
        using T = decltype(tag);
        if (conv)
            fbn_conv_fwd_kernel<T><<<C, kFbnConvThreads, 0, stream>>>(
                static_cast<const T*>(x), len, gamma, beta, static_cast<T*>(y), mean, rstd, rmean, rvar, nbt, N, C, F,
                Tb, eps, momentum);
        else
            fbn_seq_fwd_kernel<T><<<(C + kFbnSeqCols - 1) / kFbnSeqCols, kFbnSeqThreads, 0, stream>>>(
                static_cast<const T*>(x), len, gamma, beta, static_cast<T*>(y), mean, rstd, rmean, rvar, nbt, N, C,
                Tb, eps, momentum);
        return cudaGetLastError();
    });
}

cudaError_t launch_frame_bn_backward(int conv, const void* x, const void* dy, const int* len, const float* gamma,
                                     const float* beta, const float* mean, const float* rstd, void* dx, float* dgamma,
                                     float* dbeta, int N, int C, int F, int Tb, Dtype dtype, cudaStream_t stream) {
    return with_dtype(dtype, [&](auto tag) {
        using T = decltype(tag);
        if (conv)
            fbn_conv_bwd_kernel<T><<<C, kFbnConvThreads, 0, stream>>>(
                static_cast<const T*>(x), static_cast<const T*>(dy), len, gamma, beta, mean, rstd, static_cast<T*>(dx),
                dgamma, dbeta, N, C, F, Tb);
        else
            fbn_seq_bwd_kernel<T><<<(C + kFbnSeqCols - 1) / kFbnSeqCols, kFbnSeqThreads, 0, stream>>>(
                static_cast<const T*>(x), static_cast<const T*>(dy), len, gamma, mean, rstd, static_cast<T*>(dx),
                dgamma, dbeta, N, C, Tb);
        return cudaGetLastError();
    });
}

}  // namespace okt
