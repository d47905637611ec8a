// Fused flat-buffer optimizer steps (K12): one streaming pass over (param, grad, state) instead
// of the reference's per-parameter Python loops (VGG/distributed_optimizer.py:107-145 SGD with
// weight decay / momentum / dampening / nesterov; BERT/bert/transformers/optimization.py:183-224
// BertAdam = Adam without bias correction + decoupled weight decay).  The gradient buffer is
// zeroed in the same pass so that the next backward accumulates into clean memory
// (zero_grad() becomes free).
#include "common.cuh"
#include "oktopk.cuh"

namespace okt {

constexpr int kOptThreads = 256;

// The pass all three update kernels share.  A bounded cross-GPU wait timed out inside the reduction of this bucket: the
// gradient is partial, do NOT apply it (the host sees the mirrored fault flag at its next step() and re-synchronises the
// replicas).  Otherwise the kScal per-step scalars are read from device memory (the launch is CUDA-graph replayable)
// and upd(s, p, g, m, v) updates every element; m and v are its first and, with kState == 2, second state element,
// loaded when `load` (else 0) and written back when `store`.  Only the non-zero gradient lines are zeroed: the
// reduced gradient is sparse, ~k/n of the lines are dirty.
template <int kScal, int kState, typename Upd>
__device__ __forceinline__ void update_pass(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m,
                                            float* __restrict__ v, int n, bool load, bool store, int zero_grad,
                                            const float* __restrict__ scal, const int* __restrict__ fault,
                                            const int* __restrict__ skip, Upd upd) {
    if (fault != nullptr && *reinterpret_cast<const volatile int*>(fault) != 0) return;
    const int n4 = n >> 2;
    float4* p4 = reinterpret_cast<float4*>(p);
    float4* g4 = reinterpret_cast<float4*>(g);
    float4* m4 = reinterpret_cast<float4*>(m);
    float4* v4 = reinterpret_cast<float4*>(v);
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    if (verdict_set(skip)) {              // loss scaling skips this step: parameters and state stay, the gradient is cleared
        if (!zero_grad) return;
        for (int i = blockIdx.x * kOptThreads + threadIdx.x; i < n4; i += gridDim.x * kOptThreads) {
            const float4 gw = ld_stream_f4(g4 + i);
            if (gw.x != 0.f || gw.y != 0.f || gw.z != 0.f || gw.w != 0.f) g4[i] = zero;
        }
        if (blockIdx.x == 0)
            for (int i = n4 * 4 + threadIdx.x; i < n; i += kOptThreads) g[i] = 0.f;
        return;
    }
    float s[kScal];
#pragma unroll
    for (int j = 0; j < kScal; ++j) s[j] = scal[j];
    for (int i = blockIdx.x * kOptThreads + threadIdx.x; i < n4; i += gridDim.x * kOptThreads) {
        float4 pw = p4[i], gw = ld_stream_f4(g4 + i), mw = zero, vw = zero;
        if (load) {
            mw = m4[i];
            if (kState == 2) vw = v4[i];
        }
        upd(s, pw.x, gw.x, mw.x, vw.x); upd(s, pw.y, gw.y, mw.y, vw.y);
        upd(s, pw.z, gw.z, mw.z, vw.z); upd(s, pw.w, gw.w, mw.w, vw.w);
        p4[i] = pw;
        if (store) {
            m4[i] = mw;
            if (kState == 2) v4[i] = vw;
        }
        if (zero_grad && (gw.x != 0.f || gw.y != 0.f || gw.z != 0.f || gw.w != 0.f)) g4[i] = zero;
    }
    if (blockIdx.x == 0)
        for (int i = n4 * 4 + threadIdx.x; i < n; i += kOptThreads) {
            float pw = p[i], gw = g[i], mw = 0.f, vw = 0.f;
            if (load) {
                mw = m[i];
                if (kState == 2) vw = v[i];
            }
            upd(s, pw, gw, mw, vw);
            p[i] = pw;
            if (store) {
                m[i] = mw;
                if (kState == 2) v[i] = vw;
            }
            if (zero_grad) g[i] = 0.f;
        }
}

// scal -> {lr}
__global__ void __launch_bounds__(kOptThreads) fused_sgd_kernel(float* __restrict__ p, float* __restrict__ g,
                                                                 float* __restrict__ mom, int n, float momentum,
                                                                 float dampening, float wd, int nesterov, int first,
                                                                 int zero_grad, const float* __restrict__ scal,
                                                                 const int* __restrict__ fault,
                                                                 const int* __restrict__ skip) {
    const float damp = first ? 0.f : dampening;       // torch: the first step copies d_p into the buffer
    // every rounding spelled out, so that where nvcc contracts into an fma cannot change the result
    update_pass<1, 1>(p, g, mom, nullptr, n, momentum != 0.f && !first, momentum != 0.f, zero_grad, scal, fault, skip,
                      [=](const float* s, float& pw, float gw, float& mw, float&) {
                          float d = __fmaf_rn(wd, pw, gw);
                          if (momentum != 0.f) {
                              mw = first ? d : __fmaf_rn(1.f - damp, d, __fmul_rn(momentum, mw));
                              d = nesterov ? __fmaf_rn(momentum, mw, d) : mw;
                          }
                          pw = __fmaf_rn(-s[0], d, pw);
                      });
}

// scal -> {scheduled lr}
__global__ void __launch_bounds__(kOptThreads) fused_bert_adam_kernel(float* __restrict__ p, float* __restrict__ g,
                                                                       float* __restrict__ m, float* __restrict__ v,
                                                                       int n, float b1, float b2, float eps, float wd,
                                                                       int zero_grad, const float* __restrict__ scal,
                                                                       const int* __restrict__ fault,
                                                                       const int* __restrict__ skip) {
    update_pass<1, 2>(p, g, m, v, n, true, true, zero_grad, scal, fault, skip,
                      [=](const float* s, float& pw, float gw, float& mw, float& vw) {
                          mw = b1 * mw + (1.f - b1) * gw;
                          vw = b2 * vw + (1.f - b2) * gw * gw;
                          float u = mw / (sqrtf(vw) + eps);
                          if (wd > 0.f) u += wd * pw;
                          pw -= s[0] * u;
                      });
}

// torch.optim.Adam / AdamW (foreach, non-capturable branch), one rounding per op.  The per-step scalars (decay = 1 - lr*wd,
// step_size = -lr / (1 - beta1^t), bc2_sqrt = sqrt(1 - beta2^t)) are computed on the host in double, so that a captured
// CUDA graph picks up the schedule and the bias correction of every replay.
// decoupled: AdamW (p *= 1 - lr*wd) instead of L2 (g += wd*p).  w = 1 - beta1 is the weight of torch's lerp, whose
// formula depends on whether the weight is below 0.5.  (48 registers, 5 CTAs per SM: capping at 32 for 8 CTAs spills
// around the IEEE division's slow path.)
__global__ void __launch_bounds__(kOptThreads) fused_adam_kernel(float* __restrict__ p, float* __restrict__ g,
                                                                  float* __restrict__ m, float* __restrict__ v, int n,
                                                                  float w, float b2, float omb2, float eps, float wd,
                                                                  int decoupled, int zero_grad,
                                                                  const float* __restrict__ scal,
                                                                  const int* __restrict__ fault,
                                                                  const int* __restrict__ skip) {
    const bool small_w = fabsf(w) < 0.5f;
    const float lw = small_w ? w : 1.f - w;
    update_pass<3, 2>(p, g, m, v, n, true, true, zero_grad, scal, fault, skip,
                      [=](const float* s, float& pw, float gw, float& mw, float& vw) {
                          const float decay = s[0], step_size = s[1], bc2_sqrt = s[2];
                          if (decoupled) pw = pw * decay;                  // decay == 1 exactly when wd == 0
                          else if (wd != 0.f) gw = gw + wd * pw;
                          mw = small_w ? mw + lw * (gw - mw) : gw - (gw - mw) * lw;
                          vw = vw * b2;
                          vw = vw + omb2 * gw * gw;
                          const float d = sqrtf(vw) / bc2_sqrt + eps;
                          pw = pw + (step_size * mw) / d;
                      });
}

// momentum correction (VGG/distributed_optimizer.py:81-88): buf = m*buf + g ; g = buf
__global__ void __launch_bounds__(kOptThreads) momentum_correct_kernel(float* __restrict__ g, float* __restrict__ buf,
                                                                        int n, float momentum) {
    for (int i = blockIdx.x * kOptThreads + threadIdx.x; i < n; i += gridDim.x * kOptThreads) {
        float b = momentum * buf[i] + g[i];
        buf[i] = b;
        g[i] = b;
    }
}

__global__ void __launch_bounds__(kOptThreads) l2norm_sq_kernel(const float* __restrict__ x, int n, float* out) {
    double acc = 0.0;
    for (int i = blockIdx.x * kOptThreads + threadIdx.x; i < n; i += gridDim.x * kOptThreads) {
        double v = (double)x[i];
        acc += v * v;
    }
    acc = warp_sum_d(acc);
    __shared__ double s[kOptThreads / 32];
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        double v = (threadIdx.x < kOptThreads / 32) ? s[threadIdx.x] : 0.0;
        v = warp_sum_d(v);
        if (threadIdx.x == 0) atomicAdd(out, (float)v);
    }
}

// x *= max_norm / norm  when norm > max_norm (norm^2 is on the device: no host sync)
__global__ void __launch_bounds__(kOptThreads) clip_scale_kernel(float* __restrict__ x, int n, const float* norm_sq,
                                                                  float max_norm) {
    const float nrm = sqrtf(*norm_sq);
    if (!(nrm > max_norm) || nrm == 0.f) return;
    const float s = max_norm / nrm;
    for (int i = blockIdx.x * kOptThreads + threadIdx.x; i < n; i += gridDim.x * kOptThreads) x[i] *= s;
}

static inline int opt_grid(int n) {
    int g = (n / 4 + kOptThreads - 1) / kOptThreads;
    if (g < 1) g = 1;
    if (g > kStrideGridMax) g = kStrideGridMax;
    return g;
}

cudaError_t launch_fused_sgd(float* p, float* g, float* mom, int n, float momentum, float dampening, float weight_decay,
                             int nesterov, int first_step, int zero_grad, const float* scal, const int* fault,
                             const int* skip, cudaStream_t stream) {
    fused_sgd_kernel<<<opt_grid(n), kOptThreads, 0, stream>>>(p, g, mom, n, momentum, dampening, weight_decay, nesterov,
                                                             first_step, zero_grad, scal, fault, skip);
    return cudaGetLastError();
}

cudaError_t launch_fused_bert_adam(float* p, float* g, float* m, float* v, int n, float b1, float b2, float eps,
                                   float weight_decay, int zero_grad, const float* scal, const int* fault,
                                   const int* skip, cudaStream_t stream) {
    fused_bert_adam_kernel<<<opt_grid(n), kOptThreads, 0, stream>>>(p, g, m, v, n, b1, b2, eps, weight_decay, zero_grad,
                                                                   scal, fault, skip);
    return cudaGetLastError();
}

cudaError_t launch_fused_adam(float* p, float* g, float* m, float* v, int n, double beta1, double beta2, float eps,
                              float weight_decay, int decoupled, int zero_grad, const float* scal, const int* fault,
                              const int* skip, cudaStream_t stream) {
    // 1 - beta in double, rounded once: torch passes these factors as Python floats
    fused_adam_kernel<<<opt_grid(n), kOptThreads, 0, stream>>>(p, g, m, v, n, (float)(1.0 - beta1), (float)beta2,
                                                              (float)(1.0 - beta2), eps, weight_decay, decoupled,
                                                              zero_grad, scal, fault, skip);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------------
// Multi-tensor gradient landing.  Autograd hands every parameter its gradient in a freshly allocated tensor; the
// bucket the communication kernels work on is one flat symmetric allocation.  Instead of letting autograd
// accumulate into pre-existing bucket views (one elementwise add kernel PER PARAMETER per step: 54 launches for
// VGG-16) the gradients of a whole bucket are copied in by ONE launch: the kernel receives the (pointer, offset,
// length) table by value, CTAs are dealt to tensors proportionally to their size.
// ------------------------------------------------------------------------------------------------------------
constexpr int kLandThreads = 256;
constexpr int kLandPerCta = 8192;     // floats per CTA

__global__ void __launch_bounds__(kLandThreads) land_kernel(const LandParams lp, float* __restrict__ bucket) {
    // which tensor does this CTA work on?  (binary search over the CTA prefix table)
    int lo = 0, hi = lp.count - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if ((int)blockIdx.x >= lp.blk_begin[mid]) lo = mid; else hi = mid - 1;
    }
    const int t = lo;
    const int part = blockIdx.x - lp.blk_begin[t];
    const float* __restrict__ src = lp.src[t];
    float* __restrict__ dst = bucket + lp.dst_off[t];
    const int numel = lp.numel[t];
    const int begin = part * kLandPerCta;
    const int end = min(numel, begin + kLandPerCta);
    if (src == nullptr) {                 // parameter without a gradient in this step: its slice of the bucket is zero
        for (int i = begin + threadIdx.x; i < end; i += kLandThreads) dst[i] = 0.f;
        return;
    }
    const bool aligned = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15u) == 0;
    if (aligned) {
        const int v0 = begin >> 2, v1 = end >> 2;
        const float4* s4 = reinterpret_cast<const float4*>(src);
        float4* d4 = reinterpret_cast<float4*>(dst);
        for (int v = v0 + threadIdx.x; v < v1; v += kLandThreads) st_stream_f4(d4 + v, ld_stream_f4(s4 + v));
        for (int i = (v1 << 2) + threadIdx.x; i < end; i += kLandThreads) dst[i] = src[i];
    } else {
        for (int i = begin + threadIdx.x; i < end; i += kLandThreads) dst[i] = src[i];
    }
}

cudaError_t launch_land(const LandParams& lp, float* bucket, cudaStream_t stream) {
    if (lp.count <= 0) return cudaSuccess;
    land_kernel<<<lp.blk_begin[lp.count], kLandThreads, 0, stream>>>(lp, bucket);
    return cudaGetLastError();
}

cudaError_t launch_momentum_correct(float* g, float* buf, int n, float momentum, cudaStream_t stream) {
    momentum_correct_kernel<<<opt_grid(n), kOptThreads, 0, stream>>>(g, buf, n, momentum);
    return cudaGetLastError();
}

cudaError_t launch_l2norm_sq(const float* x, int n, float* out, cudaStream_t stream) {
    cudaMemsetAsync(out, 0, sizeof(float), stream);
    l2norm_sq_kernel<<<opt_grid(n), kOptThreads, 0, stream>>>(x, n, out);
    return cudaGetLastError();
}

cudaError_t launch_scale(float* x, int n, const float* norm_sq, float max_norm, cudaStream_t stream) {
    clip_scale_kernel<<<opt_grid(n), kOptThreads, 0, stream>>>(x, n, norm_sq, max_norm);
    return cudaGetLastError();
}

}  // namespace okt
