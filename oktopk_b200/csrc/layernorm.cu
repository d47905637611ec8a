// Fused dropout + residual add + LayerNorm over rows of H elements, training mode, forward and backward:
//
//   z = x + keep . a . s            (s = 1/(1-p); keep from Philox4x32-10, regenerated in the backward pass)
//   y = (z - mean) . rstd . gamma + beta,   rstd = 1/sqrt(var + eps), var biased (as F.layer_norm)
//
// Every BertLayer ends its attention and its MLP block with  LayerNorm(x + dropout(a)),  a the output of a linear layer.
// Stock ops spend three kernels on it forward (dropout writing its output and a bool mask, add, layer_norm) and about
// three backward; here it is one kernel forward, and a row kernel plus a small column reduction backward.  The mask is
// never stored: the backward pass regenerates it from the same seed and recomputes z from x and a.
//
// Layout: x, a, y, dx, da are [R, H] row-major, H a multiple of 128 up to 1024 (templated on V = H/128).  One warp owns a
// row and holds it in registers: lane l keeps the float4 columns 4 (32 j + l) .. +3 for j < V, so every access of a warp
// is 512 contiguous bytes.  The row statistics are two passes over the registers (the mean, then the sum of squared
// deviations from it), each a warp butterfly: no shared memory, no atomics, no grid-wide hand-off.  Rows are dealt to
// warps by a grid-stride loop.
//
// Dropout: flat element i = row H + col is kept iff word i % 4 of Philox4x32-10(counter (i/4 low, i/4 high, 0, 0),
// key (seed low, seed high)) is below keep_thr = floor((1-p) 2^32).  H % 4 == 0, so a lane's float4 is exactly one
// Philox call.  The seed is read from device memory, so a captured launch draws a fresh mask at every replay when the
// seed is refreshed in front of it.  keep_thr >= 2^32 (p = 0) skips the generator: every element is kept with s = 1.
// A dropped element multiplies a by 0 (not a select), so an inf or NaN in a reaches z as it does through the stock
// dropout's  a * mask * s.
//
// Backward: dxhat = dy gamma,  dz = rstd (dxhat - mean(dxhat) - xhat mean(dxhat xhat)),  dx = dz,  da = dz keep s.
// Each lane accumulates its columns' dgamma = sum dy xhat and dbeta = sum dy over the rows of its warp; the warps of a
// CTA are added in warp order in shared memory and the CTA writes one [2H] row of `partial`; ln_dgb_kernel adds the
// rows of `partial` in a fixed order.  The grid depends on R alone, so the results are bitwise reproducible.
//
// Types: x, y, dx, gamma, beta, dgamma, dbeta and the saved statistics are fp32.  a and da are fp32, bf16 or fp16 (under
// autocast the residual stream and layer_norm stay fp32 while the linear layer hands over 16-bit output).  A 16-bit a is
// widened on load, exactly; da is rounded once (to nearest even) from the fp32 dz keep s.  The 16-bit kernels are
// therefore, bit for bit, the fp32 kernel run on a.float() with da rounded.
#include "common.cuh"
#include "devlib.cuh"
#include "elem.cuh"
#include "oktopk.cuh"

namespace okt {

constexpr int kLnWarps = 4;                    // rows in flight per CTA
constexpr int kLnThreads = 32 * kLnWarps;
constexpr int kLnFwdMaxBlocks = 8192;
constexpr int kLnBwdMaxBlocks = 256;           // rows of the backward pass's column partials

// z = x + a m for one lane's float4 column j of a row; the forward and backward passes share it, so z is bitwise the same
template <typename T>
__device__ __forceinline__ float4 ln_z(const float* x, const T* a, const float4& m, size_t off) {
    const float4 xv = *reinterpret_cast<const float4*>(x + off);
    const float4 av = Elem<T>::wide(*reinterpret_cast<const typename Elem<T>::V*>(a + off));
    return make_float4(fmaf(av.x, m.x, xv.x), fmaf(av.y, m.y, xv.y), fmaf(av.z, m.z, xv.z), fmaf(av.w, m.w, xv.w));
}

template <int V, typename T>
__global__ void __launch_bounds__(kLnThreads) ln_fwd_kernel(const float* __restrict__ x, const T* __restrict__ a,
                                                            float* __restrict__ y, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, float* __restrict__ mean,
                                                            float* __restrict__ rstd, const unsigned long long* seed,
                                                            int R, long long keep_thr, float scale, float eps) {
    constexpr int H = 128 * V;
    const int lane = lane_id();
    const LnDrop d = ln_drop(seed, keep_thr, scale);
    for (int row = blockIdx.x * kLnWarps + (threadIdx.x >> 5); row < R; row += gridDim.x * kLnWarps) {
        const size_t base = (size_t)row * H;
        float4 z[V];
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < V; ++j) {
            const size_t off = base + (j * 32 + lane) * 4;
            z[j] = ln_z(x, a, ln_mult(d, ln_keep(d, off)), off);
            sum += (z[j].x + z[j].y) + (z[j].z + z[j].w);
        }
        const float mu = warp_sum_f(sum) / (float)H;
        float sq = 0.f;
#pragma unroll
        for (int j = 0; j < V; ++j) {
            z[j] = make_float4(z[j].x - mu, z[j].y - mu, z[j].z - mu, z[j].w - mu);
            sq += (z[j].x * z[j].x + z[j].y * z[j].y) + (z[j].z * z[j].z + z[j].w * z[j].w);
        }
        const float rs = rsqrtf(warp_sum_f(sq) / (float)H + eps);
#pragma unroll
        for (int j = 0; j < V; ++j) {
            const int col = (j * 32 + lane) * 4;
            const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + col));
            const float4 b = __ldg(reinterpret_cast<const float4*>(beta + col));
            *reinterpret_cast<float4*>(y + base + col) =
                make_float4(fmaf(z[j].x * rs, g.x, b.x), fmaf(z[j].y * rs, g.y, b.y), fmaf(z[j].z * rs, g.z, b.z),
                            fmaf(z[j].w * rs, g.w, b.w));
        }
        if (lane == 0) { mean[row] = mu; rstd[row] = rs; }
    }
}

// (minimum 1 CTA per SM: with the default heuristic ptxas caps H = 384 at 96 registers and spills)
template <int V, typename T>
__global__ void __launch_bounds__(kLnThreads, 1) ln_bwd_kernel(const float* __restrict__ x, const T* __restrict__ a,
                                                            const float* __restrict__ dy, const float* __restrict__ gamma,
                                                            const float* __restrict__ mean, const float* __restrict__ rstd,
                                                            const unsigned long long* seed, float* __restrict__ dx,
                                                            T* __restrict__ da, float* __restrict__ partial, int R,
                                                            long long keep_thr, float scale) {
    constexpr int H = 128 * V;
    __shared__ float4 s_part[2 * H / 4];                  // [dgamma | dbeta] of this CTA's rows
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    const LnDrop d = ln_drop(seed, keep_thr, scale);
    float4 pg[V], pb[V];
#pragma unroll
    for (int j = 0; j < V; ++j) pg[j] = pb[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int row = blockIdx.x * kLnWarps + warp; row < R; row += gridDim.x * kLnWarps) {
        const size_t base = (size_t)row * H;
        const float mu = mean[row], rs = rstd[row];
        float4 xh[V], g[V];
        uint32_t keep = 0;                                // 4 bits per float4 column, V <= 8
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int j = 0; j < V; ++j) {
            const int col = (j * 32 + lane) * 4;
            const uint32_t k = ln_keep(d, base + col);
            keep |= k << (4 * j);
            const float4 z = ln_z(x, a, ln_mult(d, k), base + col);
            xh[j] = make_float4((z.x - mu) * rs, (z.y - mu) * rs, (z.z - mu) * rs, (z.w - mu) * rs);
            const float4 dyv = *reinterpret_cast<const float4*>(dy + base + col);
            const float4 gm = __ldg(reinterpret_cast<const float4*>(gamma + col));
            g[j] = make_float4(dyv.x * gm.x, dyv.y * gm.y, dyv.z * gm.z, dyv.w * gm.w);
            s1 += (g[j].x + g[j].y) + (g[j].z + g[j].w);
            s2 += (g[j].x * xh[j].x + g[j].y * xh[j].y) + (g[j].z * xh[j].z + g[j].w * xh[j].w);
            pg[j] = make_float4(fmaf(dyv.x, xh[j].x, pg[j].x), fmaf(dyv.y, xh[j].y, pg[j].y), fmaf(dyv.z, xh[j].z, pg[j].z),
                                fmaf(dyv.w, xh[j].w, pg[j].w));
            pb[j] = make_float4(pb[j].x + dyv.x, pb[j].y + dyv.y, pb[j].z + dyv.z, pb[j].w + dyv.w);
        }
        const float c1 = warp_sum_f(s1) / (float)H, c2 = warp_sum_f(s2) / (float)H;
#pragma unroll
        for (int j = 0; j < V; ++j) {
            const int col = (j * 32 + lane) * 4;
            const float4 dz = make_float4(rs * (g[j].x - c1 - xh[j].x * c2), rs * (g[j].y - c1 - xh[j].y * c2),
                                          rs * (g[j].z - c1 - xh[j].z * c2), rs * (g[j].w - c1 - xh[j].w * c2));
            const float4 m = ln_mult(d, keep >> (4 * j));
            *reinterpret_cast<float4*>(dx + base + col) = dz;
            *reinterpret_cast<typename Elem<T>::V*>(da + base + col) =
                Elem<T>::narrow(make_float4(dz.x * m.x, dz.y * m.y, dz.z * m.z, dz.w * m.w));
        }
    }
    // the CTA's column partials, warps added in warp order
    for (int w = 0; w < kLnWarps; ++w) {
        if (warp == w) {
#pragma unroll
            for (int j = 0; j < V; ++j) {
                const int c4 = j * 32 + lane;
                if (w == 0) {
                    s_part[c4] = pg[j];
                    s_part[H / 4 + c4] = pb[j];
                } else {
                    const float4 og = s_part[c4], ob = s_part[H / 4 + c4];
                    s_part[c4] = make_float4(og.x + pg[j].x, og.y + pg[j].y, og.z + pg[j].z, og.w + pg[j].w);
                    s_part[H / 4 + c4] = make_float4(ob.x + pb[j].x, ob.y + pb[j].y, ob.z + pb[j].z, ob.w + pb[j].w);
                }
            }
        }
        __syncthreads();
    }
    float4* out = reinterpret_cast<float4*>(partial) + (size_t)blockIdx.x * (2 * H / 4);
    for (int c4 = threadIdx.x; c4 < 2 * H / 4; c4 += kLnThreads) out[c4] = s_part[c4];
}

// dgamma | dbeta = the sum of the G rows of `partial` [G, 2H]: column c's rows g = w, w + 8, ... are added by warp w in
// order, then the 8 warp sums in warp order.
constexpr int kLnDgbWarps = 8;

__global__ void __launch_bounds__(32 * kLnDgbWarps) ln_dgb_kernel(const float* __restrict__ partial, int G, int H,
                                                                 float* __restrict__ dgamma, float* __restrict__ dbeta) {
    __shared__ float s[kLnDgbWarps][32];
    const int lane = lane_id(), w = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + lane;                 // 2H is a multiple of 32
    float acc = 0.f;
    for (int g = w; g < G; g += kLnDgbWarps) acc += partial[(size_t)g * 2 * H + c];
    s[w][lane] = acc;
    __syncthreads();
    if (w == 0) {
        float t = s[0][lane];
#pragma unroll
        for (int k = 1; k < kLnDgbWarps; ++k) t += s[k][lane];
        if (c < H) dgamma[c] = t; else dbeta[c - H] = t;
    }
}

bool ln_supported_h(int H) { return H >= 128 && H <= 1024 && H % 128 == 0; }

static int ln_rows_grid(int R, int cap) {
    const long long b = ((long long)R + kLnWarps - 1) / kLnWarps;
    return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

int ln_bwd_grid(int R) { return ln_rows_grid(R, kLnBwdMaxBlocks); }

cudaError_t launch_ln_dgb(const float* partial, int G, int H, float* dgamma, float* dbeta, cudaStream_t stream) {
    ln_dgb_kernel<<<2 * H / 32, 32 * kLnDgbWarps, 0, stream>>>(partial, G, H, dgamma, dbeta);
    return cudaGetLastError();
}

template <typename T>
static cudaError_t ln_forward_t(const float* x, const void* a, float* y, const float* gamma, const float* beta, float* mean,
                                float* rstd, const unsigned long long* seed, int R, int H, long long keep_thr, float scale,
                                float eps, cudaStream_t stream) {
    const int grid = ln_rows_grid(R, kLnFwdMaxBlocks);
    const T* at = static_cast<const T*>(a);
    switch (H / 128) {
#define OKT_LN_FWD(V) case V: ln_fwd_kernel<V, T><<<grid, kLnThreads, 0, stream>>>(x, at, y, gamma, beta, mean, rstd, seed, \
                                                                                   R, keep_thr, scale, eps); break;
        OKT_LN_FWD(1) OKT_LN_FWD(2) OKT_LN_FWD(3) OKT_LN_FWD(4) OKT_LN_FWD(5) OKT_LN_FWD(6) OKT_LN_FWD(7) OKT_LN_FWD(8)
#undef OKT_LN_FWD
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

template <typename T>
static cudaError_t ln_backward_t(const float* x, const void* a, const float* dy, const float* gamma, const float* mean,
                                 const float* rstd, const unsigned long long* seed, float* dx, void* da, float* partial,
                                 float* dgamma, float* dbeta, int R, int H, long long keep_thr, float scale,
                                 cudaStream_t stream) {
    const int grid = ln_bwd_grid(R);
    const T* at = static_cast<const T*>(a);
    T* dat = static_cast<T*>(da);
    switch (H / 128) {
#define OKT_LN_BWD(V) case V: ln_bwd_kernel<V, T><<<grid, kLnThreads, 0, stream>>>(x, at, dy, gamma, mean, rstd, seed, dx, \
                                                                                   dat, partial, R, keep_thr, scale); break;
        OKT_LN_BWD(1) OKT_LN_BWD(2) OKT_LN_BWD(3) OKT_LN_BWD(4) OKT_LN_BWD(5) OKT_LN_BWD(6) OKT_LN_BWD(7) OKT_LN_BWD(8)
#undef OKT_LN_BWD
        default: return cudaErrorInvalidValue;
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    return launch_ln_dgb(partial, grid, H, dgamma, dbeta, stream);
}

static bool ln_args_ok(int R, int H, long long keep_thr, const unsigned long long* seed) {
    return R > 0 && ln_supported_h(H) && keep_thr >= 0 && keep_thr <= kLnKeepAll && (keep_thr == kLnKeepAll || seed != nullptr);
}

cudaError_t launch_ln_forward(const float* x, const void* a, float* y, const float* gamma, const float* beta, float* mean,
                              float* rstd, const unsigned long long* seed, int R, int H, long long keep_thr, float scale,
                              float eps, Dtype a_dtype, cudaStream_t stream) {
    if (!ln_args_ok(R, H, keep_thr, seed)) return cudaErrorInvalidValue;
    return with_dtype(a_dtype, [&](auto e) {
        return ln_forward_t<decltype(e)>(x, a, y, gamma, beta, mean, rstd, seed, R, H, keep_thr, scale, eps, stream);
    });
}

cudaError_t launch_ln_backward(const float* x, const void* a, const float* dy, const float* gamma, const float* mean,
                               const float* rstd, const unsigned long long* seed, float* dx, void* da, float* partial,
                               float* dgamma, float* dbeta, int R, int H, long long keep_thr, float scale, Dtype a_dtype,
                               cudaStream_t stream) {
    if (!ln_args_ok(R, H, keep_thr, seed)) return cudaErrorInvalidValue;
    return with_dtype(a_dtype, [&](auto e) {
        return ln_backward_t<decltype(e)>(x, a, dy, gamma, mean, rstd, seed, dx, da, partial, dgamma, dbeta, R, H, keep_thr,
                                          scale, stream);
    });
}

}  // namespace okt
