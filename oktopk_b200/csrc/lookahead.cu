// Fused look-ahead convolution + Hardtanh(0, 20) of the AN4 DeepSpeech model, forward and backward.  x, y [Tb, N, H]
// (time-major, the LSTM stack's layout), W [H, K] with K = context + 1 taps, len [N] int32 the utterances' frame
// lengths on the device, and
//
//   Tm = min(max(0, max_n len_n), Tb),   L_n = min(len_n, Tm).
//
//   z[t, n, h] = sum_{k < K} W[h, k] x[t + k, n, h]     (x read as 0 where t + k >= L_n)
//   y[t, n, h] = t < L_n ? clamp(z, 0, 20) : +0
//
// Backward: dz = dy where the frame is valid and 0 < y < 20 (torch's strict Hardtanh backward, decided by the stored y
// alone), else 0; dx[t] = t < L_n ? sum_k W[h, k] dz[t - k] : +0; dW[h, k] = sum over t < Tm and n of x[t + k] dz[t].
// Frames past L_n are never read: the forward pass writes +0 there, and past Tm it reads no x at all.
//
// Geometry.  A CTA is kLaWarps warps over a slice of kLaCols channels, lane l owning channel h = slice + l, so every
// load and store of a warp is one coalesced row segment.
//   - Forward (one launch): CTA (slice, c) writes the kLaRows rows r = t N + n of chunk c, warp w the rows r = w
//     (mod kLaWarps); z sums its taps k = 0, 1, ... in fp32 fmaf.
//   - Backward (one launch): CTAs (slice, k) for k < K compute dW[., k]; CTAs (slice, K + c) write dx on the rows of
//     chunk c, summing the taps k = 0, 1, ... in fp32 fmaf, with dz recomputed from (y, dy) for each tap.
// Summation order of dW: warp w adds the rows r = w (mod kLaWarps) of [0, Tm N) in order, each product x dz exact in fp64
// and accumulated in fp64; the kLaWarps partial sums are added in a fixed pairwise tree and rounded once to fp32.  The
// order depends on (Tm, N, H, K) and the lengths only, never on Tb: a launch at a padded width equals, bit for bit, a
// launch on the tensor cropped to Tm frames, and runs repeat bit for bit.  No atomics.
//
// A product x dz is added for every valid frame t, with x = 0 past the length, so that a non-finite dz reaches dW as
// it does through the stock convolution's zero padding (0 * inf = NaN), and loss scaling's check sees it.
//
// Types: x, y, dy and dx are fp32, bf16 or fp16 (elem.cuh: widened exactly, fp32 arithmetic, y and dx rounded once);
// W and dW are fp32.
#include "common.cuh"
#include "elem.cuh"
#include "oktopk.cuh"

namespace okt {

constexpr int kLaMaxTaps = 32;
constexpr int kLaCols = 32;
constexpr int kLaWarps = 16;
constexpr int kLaThreads = kLaCols * kLaWarps;
constexpr int kLaRows = 16;
constexpr float kLaClampMax = 20.f;

__device__ __forceinline__ int la_bound(const int* len, int N, int Tb) {
    int m = 0;
    for (int n = 0; n < N; ++n) m = max(m, __ldg(len + n));
    return min(m, Tb);
}

// clamp(z, 0, 20) with -0 stored as +0; a NaN stays NaN, as torch's hardtanh.
__device__ __forceinline__ float la_clamp(float z) {
    if (z <= 0.f) return 0.f;
    return z >= kLaClampMax ? kLaClampMax : z;
}

// dz at element `off` of a valid frame: dy where 0 < y < 20, else 0 (both loads issued at once).
template <typename T>
__device__ __forceinline__ float la_dz(const T* __restrict__ y, const T* __restrict__ dy, size_t off) {
    const float v = Elem<T>::ld(y + off), g = Elem<T>::ld(dy + off);
    return (v > 0.f && v < kLaClampMax) ? g : 0.f;
}

template <typename T>
__global__ void __launch_bounds__(kLaThreads)
la_fwd_kernel(const T* __restrict__ x, const float* __restrict__ w, const int* __restrict__ len, T* __restrict__ y,
              int N, int H, int Tb, int K) {
    const int h = blockIdx.x * kLaCols + (threadIdx.x & 31), warp = threadIdx.x >> 5;
    if (h >= H) return;
    const int Tm = la_bound(len, N, Tb);
    const float* wh = w + (size_t)h * K;
    const size_t step = (size_t)N * H;
    const int rend = min(Tb * N, (int)(blockIdx.y + 1) * kLaRows);
    for (int r = blockIdx.y * kLaRows + warp; r < rend; r += kLaWarps) {
        const int t = r / N, n = r - t * N;
        const size_t off = (size_t)r * H + h;
        float v = 0.f;
        if (t < Tm) {
            const int L = min(__ldg(len + n), Tm);
            if (t < L) {
                const int kend = min(K, L - t);
                const T* p = x + off;
                float z = 0.f;
#pragma unroll 8
                for (int k = 0; k < kend; ++k, p += step) z = fmaf(__ldg(wh + k), Elem<T>::ld(p), z);
                v = la_clamp(z);
            }
        }
        y[off] = Elem<T>::narrow1(v);
    }
}

template <typename T>
__global__ void __launch_bounds__(kLaThreads)
la_bwd_kernel(const T* __restrict__ x, const T* __restrict__ y, const T* __restrict__ dy, const float* __restrict__ w,
              const int* __restrict__ len, T* __restrict__ dx, float* __restrict__ dw, int N, int H, int Tb, int K) {
    __shared__ double sh[kLaWarps][kLaCols];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int h = blockIdx.x * kLaCols + lane;
    const int Tm = la_bound(len, N, Tb);
    const size_t step = (size_t)N * H;

    if ((int)blockIdx.y < K) {                           // dW[., k]
        const int k = blockIdx.y;
        const int hc = min(h, H - 1);                    // lanes past H read a real channel and store nothing
        const int R = Tm * N;
        double s = 0.0;
#pragma unroll 2
        for (int r = warp; r < R; r += kLaWarps) {
            const int t = r / N, n = r - t * N;
            const int L = min(__ldg(len + n), Tm);
            if (t >= L) continue;
            const size_t off = (size_t)r * H + hc;
            const float g = la_dz(y, dy, off);
            const float xv = t + k < L ? Elem<T>::ld(x + off + k * step) : 0.f;
            s = fma((double)xv, (double)g, s);
        }
        sh[warp][lane] = s;
        __syncthreads();
#pragma unroll
        for (int st = kLaWarps / 2; st > 0; st >>= 1) {
            if (warp < st) sh[warp][lane] += sh[warp + st][lane];
            __syncthreads();
        }
        if (warp == 0 && h < H) dw[(size_t)h * K + k] = (float)sh[0][lane];
        return;
    }

    if (h >= H) return;                                  // dx on the rows of chunk blockIdx.y - K
    const float* wh = w + (size_t)h * K;
    const int c = blockIdx.y - K, rend = min(Tb * N, (c + 1) * kLaRows);
    for (int r = c * kLaRows + warp; r < rend; r += kLaWarps) {
        const int t = r / N, n = r - t * N;
        const size_t off = (size_t)r * H + h;
        float v = 0.f;
        if (t < Tm) {
            const int L = min(__ldg(len + n), Tm);
            if (t < L) {
                const int kend = min(K, t + 1);
#pragma unroll 8
                for (int k = 0; k < kend; ++k) v = fmaf(__ldg(wh + k), la_dz(y, dy, off - k * step), v);
            }
        }
        dx[off] = Elem<T>::narrow1(v);
    }
}

bool lookahead_supported(int N, int H, int Tb, int K) {
    if (N <= 0 || H <= 0 || Tb <= 0 || K <= 0 || K > kLaMaxTaps) return false;
    const long long rows = (long long)Tb * N;
    return rows * H < (1LL << 40) && (rows + kLaRows - 1) / kLaRows + K <= 65535;
}

int lookahead_max_taps() { return kLaMaxTaps; }

cudaError_t launch_lookahead_forward(const void* x, const float* w, const int* len, void* y, int N, int H, int Tb,
                                     int K, Dtype dtype, cudaStream_t stream) {
    const dim3 grid((H + kLaCols - 1) / kLaCols, (Tb * N + kLaRows - 1) / kLaRows);
    return with_dtype(dtype, [&](auto tag) {
        using T = decltype(tag);
        la_fwd_kernel<T><<<grid, kLaThreads, 0, stream>>>(static_cast<const T*>(x), w, len, static_cast<T*>(y), N, H,
                                                           Tb, K);
        return cudaGetLastError();
    });
}

cudaError_t launch_lookahead_backward(const void* x, const void* y, const void* dy, const float* w, const int* len,
                                      void* dx, float* dw, int N, int H, int Tb, int K, Dtype dtype,
                                      cudaStream_t stream) {
    const dim3 grid((H + kLaCols - 1) / kLaCols, K + (Tb * N + kLaRows - 1) / kLaRows);
    return with_dtype(dtype, [&](auto tag) {
        using T = decltype(tag);
        la_bwd_kernel<T><<<grid, kLaThreads, 0, stream>>>(static_cast<const T*>(x), static_cast<const T*>(y),
                                                           static_cast<const T*>(dy), w, len, static_cast<T*>(dx), dw,
                                                           N, H, Tb, K);
        return cudaGetLastError();
    });
}

}  // namespace okt
