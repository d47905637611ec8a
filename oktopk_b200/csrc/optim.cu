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

// The clip factor of an update, read where update_pass reads the gradient (see ClipRef in oktopk.cuh).  A thread's vector
// index only grows, so the per-segment lookup is a cursor that steps over the segment ends it passes: no search, no
// extra pass.
struct ClipCursor {
    const float* coef;
    const int* ends;
    int t;
    float f;
    __device__ __forceinline__ explicit ClipCursor(const ClipRef& c)
        : coef(c.coef), ends(c.ends), t(0), f(c.coef != nullptr ? c.coef[0] : 1.f) {}
    __device__ __forceinline__ float at(int vec) {
        if (ends != nullptr && vec >= __ldg(ends + t)) {
            do ++t; while (vec >= __ldg(ends + t));
            f = coef[t];
        }
        return f;
    }
};

__device__ __forceinline__ void scale4(float4& gw, float c) {
    gw.x = __fmul_rn(gw.x, c); gw.y = __fmul_rn(gw.y, c); gw.z = __fmul_rn(gw.z, c); gw.w = __fmul_rn(gw.w, c);
}

// The pass all three update kernels share.  A bounded cross-GPU wait timed out inside the reduction of this bucket: the
// gradient is partial, do NOT apply it (the host sees the mirrored fault flag at its next step() and re-synchronises the
// replicas).  Otherwise the kScal per-step scalars are read from device memory (the launch is CUDA-graph replayable)
// and upd(s, p, g, m, v) updates every element; m and v are its first and, with kState == 2, second state element,
// loaded when `load` (else 0) and written back when `store`.  Only the non-zero gradient lines are zeroed: the
// reduced gradient is sparse, ~k/n of the lines are dirty.  With a clip factor (clip.coef set) upd sees the gradient
// times the factor, one fp32 multiply as torch's _foreach_mul_ does it; the bucket keeps the unscaled value until it
// is zeroed.  A skipped step never reads the factor.
template <int kScal, int kState, typename Upd>
__device__ __forceinline__ void update_pass(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m,
                                            float* __restrict__ v, int n, bool load, bool store, int zero_grad,
                                            const float* __restrict__ scal, const int* __restrict__ fault,
                                            const int* __restrict__ skip, const ClipRef clip, Upd upd) {
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
    ClipCursor cc(clip);
    for (int i = blockIdx.x * kOptThreads + threadIdx.x; i < n4; i += gridDim.x * kOptThreads) {
        float4 pw = p4[i], gw = ld_stream_f4(g4 + i), mw = zero, vw = zero;
        const bool dirty = gw.x != 0.f || gw.y != 0.f || gw.z != 0.f || gw.w != 0.f;
        if (clip.coef != nullptr) scale4(gw, cc.at(i));
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
        if (zero_grad && dirty) g4[i] = zero;
    }
    if (blockIdx.x == 0)
        for (int i = n4 * 4 + threadIdx.x; i < n; i += kOptThreads) {
            float pw = p[i], gw = g[i], mw = 0.f, vw = 0.f;
            if (clip.coef != nullptr) gw = __fmul_rn(gw, cc.at(i >> 2));
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

// torch.optim.SGD on one element, the one definition fused_sgd_kernel, sgd_ahead_kernel and fused_sgd_tail_kernel share.
// Every rounding spelled out, so that where nvcc contracts into an fma cannot change the result.
__device__ __forceinline__ void sgd_update(const SgdHyper& h, float lr, float& pw, float gw, float& mw) {
    const float damp = h.first ? 0.f : h.dampening;    // torch: the first step copies d_p into the buffer
    float d = __fmaf_rn(h.wd, pw, gw);
    if (h.momentum != 0.f) {
        mw = h.first ? d : __fmaf_rn(1.f - damp, d, __fmul_rn(h.momentum, mw));
        d = h.nesterov ? __fmaf_rn(h.momentum, mw, d) : mw;
    }
    pw = __fmaf_rn(-lr, d, pw);
}

__device__ __forceinline__ void sgd_update4(const SgdHyper& h, float lr, float4& pw, const float4& gw, float4& mw) {
    sgd_update(h, lr, pw.x, gw.x, mw.x); sgd_update(h, lr, pw.y, gw.y, mw.y);
    sgd_update(h, lr, pw.z, gw.z, mw.z); sgd_update(h, lr, pw.w, gw.w, mw.w);
}

// scal -> {lr}; coef: the clip factor or null
__global__ void __launch_bounds__(kOptThreads) fused_sgd_kernel(float* __restrict__ p, float* __restrict__ g,
                                                                 float* __restrict__ mom, int n, const SgdHyper h,
                                                                 int zero_grad, const float* __restrict__ scal,
                                                                 const int* __restrict__ fault,
                                                                 const int* __restrict__ skip,
                                                                 const float* __restrict__ coef) {
    update_pass<1, 1>(p, g, mom, nullptr, n, h.momentum != 0.f && !h.first, h.momentum != 0.f, zero_grad, scal, fault,
                      skip, ClipRef{coef, nullptr},
                      [=](const float* s, float& pw, float gw, float& mw, float&) { sgd_update(h, s[0], pw, gw, mw); });
}

// ------------------------------------------------------------------------------------------------------------
// Early SGD update.  On a sparse step the reduced gradient is zero on all but ~k of the n elements, and there the update
// depends only on p, m and lr.  Once autograd has produced a parameter's gradient nothing in the step reads its weights
// again, so the zero-gradient update can run during backward, beside the bucket's early-pack segment: sgd_ahead_kernel
// stashes the old p and m and applies it in place.  After the Ok-Topk call fused_sgd_tail_kernel recomputes, from the
// stash, every vector of those ranges whose gradient the call wrote (any bit set: a -0 counts too), so that each element
// ends up with exactly fused_sgd_kernel's result, and runs fused_sgd_kernel's update over the ranges the ahead pass did
// not cover.
// ------------------------------------------------------------------------------------------------------------
constexpr int kAheadUnroll = 4;       // float4 vectors in flight per thread: the pass runs on a capped grid

__device__ __forceinline__ void st_evict_f4(float4* p, const float4& v) {
    asm volatile("st.global.cs.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// Loads and stores are evict-first: backward's activations keep L2.
__global__ void __launch_bounds__(kOptThreads) sgd_ahead_kernel(float* __restrict__ p, float* __restrict__ mom,
                                                                 float* __restrict__ sp, float* __restrict__ sm,
                                                                 const SgdRanges r, const SgdHyper h,
                                                                 const float* __restrict__ scal) {
    const float lr = scal[0];
    const bool use_m = h.momentum != 0.f;
    float4* p4 = reinterpret_cast<float4*>(p);
    float4* m4 = reinterpret_cast<float4*>(mom);
    float4* sp4 = reinterpret_cast<float4*>(sp);
    float4* sm4 = reinterpret_cast<float4*>(sm);
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    const int stride = gridDim.x * kOptThreads;
    for (int q = 0; q < r.nr; ++q) {
        const int hi = r.hi[q];
        for (int i0 = r.lo[q] + blockIdx.x * kOptThreads + threadIdx.x; i0 < hi; i0 += kAheadUnroll * stride) {
            float4 pw[kAheadUnroll], mw[kAheadUnroll];
#pragma unroll
            for (int u = 0; u < kAheadUnroll; ++u) {
                const int i = i0 + u * stride;
                pw[u] = mw[u] = zero;
                if (i < hi) {
                    pw[u] = ld_stream_f4(p4 + i);
                    if (use_m) mw[u] = ld_stream_f4(m4 + i);
                }
            }
#pragma unroll
            for (int u = 0; u < kAheadUnroll; ++u) {
                const int i = i0 + u * stride;
                if (i >= hi) continue;
                st_evict_f4(sp4 + i, pw[u]);
                if (use_m) st_evict_f4(sm4 + i, mw[u]);
                sgd_update4(h, lr, pw[u], zero, mw[u]);
                st_evict_f4(p4 + i, pw[u]);
                if (use_m) st_evict_f4(m4 + i, mw[u]);
            }
        }
    }
}

__device__ __forceinline__ bool any_bits(const float4& v) {
    return (__float_as_uint(v.x) | __float_as_uint(v.y) | __float_as_uint(v.z) | __float_as_uint(v.w)) != 0u;
}

// scal -> {lr}.  A vector is zeroed in g under fused_sgd_kernel's rule (a lane != 0), so the bucket ends up the same too.
// coef: the clip factor or null.  The ahead pass's zero-gradient update holds for any finite factor (0 * c == 0); a NaN
// factor reaches every element under torch's multiply, so then every vector of the ahead ranges is recomputed.
__global__ void __launch_bounds__(kOptThreads) fused_sgd_tail_kernel(float* __restrict__ p, float* __restrict__ g,
                                                                      float* __restrict__ mom,
                                                                      const float* __restrict__ sp,
                                                                      const float* __restrict__ sm, int n,
                                                                      const SgdRanges ahead, const SgdRanges dense,
                                                                      const SgdHyper h, int zero_grad,
                                                                      const float* __restrict__ scal,
                                                                      const int* __restrict__ fault,
                                                                      const int* __restrict__ skip,
                                                                      const float* __restrict__ coef) {
    const bool use_m = h.momentum != 0.f;
    float4* p4 = reinterpret_cast<float4*>(p);
    float4* g4 = reinterpret_cast<float4*>(g);
    float4* m4 = reinterpret_cast<float4*>(mom);
    const float4* sp4 = reinterpret_cast<const float4*>(sp);
    const float4* sm4 = reinterpret_cast<const float4*>(sm);
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    const int first = blockIdx.x * kOptThreads + threadIdx.x, stride = gridDim.x * kOptThreads;
    const bool faulted = fault != nullptr && *reinterpret_cast<const volatile int*>(fault) != 0;
    if (faulted || verdict_set(skip)) {
        // the step is not applied: p and m get their old values back; after a fault the gradient is left as it is
        // (fused_sgd_kernel returns at once), after a skip it is cleared as fused_sgd_kernel clears it
        for (int q = 0; q < ahead.nr; ++q)
            for (int i = ahead.lo[q] + first; i < ahead.hi[q]; i += stride) {
                p4[i] = sp4[i];
                if (use_m) m4[i] = sm4[i];
            }
        if (faulted) return;
        update_pass<1, 1>(p, g, mom, nullptr, n, false, false, zero_grad, scal, nullptr, skip, ClipRef{nullptr, nullptr},
                          [](const float*, float&, float, float&, float&) {});
        return;
    }
    const float lr = scal[0];
    const float c = coef != nullptr ? *coef : 1.f;
    const bool every = c != c;                          // NaN factor
    for (int q = 0; q < ahead.nr; ++q)
        for (int i = ahead.lo[q] + first; i < ahead.hi[q]; i += stride) {
            float4 gw = ld_stream_f4(g4 + i);
            if (!any_bits(gw) && !every) continue;      // the ahead pass's result stands
            const bool dirty = gw.x != 0.f || gw.y != 0.f || gw.z != 0.f || gw.w != 0.f;
            if (coef != nullptr) scale4(gw, c);
            float4 pw = sp4[i], mw = zero;
            if (use_m) mw = sm4[i];
            sgd_update4(h, lr, pw, gw, mw);
            p4[i] = pw;
            if (use_m) m4[i] = mw;
            if (zero_grad && dirty) g4[i] = zero;
        }
    for (int q = 0; q < dense.nr; ++q)
        for (int i = dense.lo[q] + first; i < dense.hi[q]; i += stride) {
            float4 pw = p4[i], gw = ld_stream_f4(g4 + i), mw = zero;
            const bool dirty = gw.x != 0.f || gw.y != 0.f || gw.z != 0.f || gw.w != 0.f;
            if (coef != nullptr) scale4(gw, c);
            if (use_m && !h.first) mw = m4[i];
            sgd_update4(h, lr, pw, gw, mw);
            p4[i] = pw;
            if (use_m) m4[i] = mw;
            if (zero_grad && dirty) g4[i] = zero;
        }
    if (blockIdx.x == 0)
        for (int i = (n >> 2) * 4 + threadIdx.x; i < n; i += kOptThreads) {
            float pw = p[i], gw = g[i], mw = 0.f;
            if (coef != nullptr) gw = __fmul_rn(gw, c);
            if (use_m && !h.first) mw = mom[i];
            sgd_update(h, lr, pw, gw, mw);
            p[i] = pw;
            if (use_m) mom[i] = mw;
            if (zero_grad) g[i] = 0.f;
        }
}

// scal -> {scheduled lr, max_grad_norm}; clip: none, or one factor per parameter (clip_reduced)
__global__ void __launch_bounds__(kOptThreads) fused_bert_adam_kernel(float* __restrict__ p, float* __restrict__ g,
                                                                       float* __restrict__ m, float* __restrict__ v,
                                                                       int n, float b1, float b2, float eps, float wd,
                                                                       int zero_grad, const float* __restrict__ scal,
                                                                       const int* __restrict__ fault,
                                                                       const int* __restrict__ skip, const ClipRef clip) {
    update_pass<1, 2>(p, g, m, v, n, true, true, zero_grad, scal, fault, skip, clip,
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
// formula depends on whether the weight is below 0.5.  (44 registers, 5 CTAs per SM: capping at 32 for 8 CTAs spills
// around the IEEE division's slow path.)
__global__ void __launch_bounds__(kOptThreads) fused_adam_kernel(float* __restrict__ p, float* __restrict__ g,
                                                                  float* __restrict__ m, float* __restrict__ v, int n,
                                                                  float w, float b2, float omb2, float eps, float wd,
                                                                  int decoupled, int zero_grad,
                                                                  const float* __restrict__ scal,
                                                                  const int* __restrict__ fault,
                                                                  const int* __restrict__ skip,
                                                                  const float* __restrict__ coef) {
    const bool small_w = fabsf(w) < 0.5f;
    const float lw = small_w ? w : 1.f - w;
    update_pass<3, 2>(p, g, m, v, n, true, true, zero_grad, scal, fault, skip, ClipRef{coef, nullptr},
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

// ------------------------------------------------------------------------------------------------------------
// Gradient clipping on the device.  grad_sumsq_kernel: one CTA per kSumsqChunk elements of a segment (a fixed function
// of the segment lengths, not of the device), each writing its sum of squares in fp64 to its own partial: no atomics.
// Within a CTA thread j sums the float4 vectors j, j + 256, ... and the scalar tail in order, then the warps and the
// eight warp sums are combined in a fixed tree.  clip_coef_kernel (one CTA) combines the partials in a fixed order too,
// so the norm and the factor are a function of the gradient's bits alone: bitwise equal buckets give bitwise equal
// factors on every rank.
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double block_sum_d(double v) {
    __shared__ double ws[kOptThreads / 32];
    v = warp_sum_d(v);
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < kOptThreads / 32; ++w) t += ws[w];
    __syncthreads();
    return t;                                           // thread 0's value
}

__global__ void __launch_bounds__(kOptThreads) grad_sumsq_kernel(const float* __restrict__ g, const SumsqSegs t,
                                                                  double* __restrict__ partial) {
    int lo = 0, hi = t.nseg - 1;                        // this CTA's segment (binary search over the CTA prefix table)
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if ((int)blockIdx.x >= t.blk_begin[mid]) lo = mid; else hi = mid - 1;
    }
    const int begin = (blockIdx.x - t.blk_begin[lo]) * kSumsqChunk;
    const int len = min(t.len[lo] - begin, kSumsqChunk);
    const float* x = g + t.off[lo] + begin;             // 16-byte aligned: offsets and kSumsqChunk are multiples of 4
    const float4* x4 = reinterpret_cast<const float4*>(x);
    double acc = 0.0;
    for (int i = threadIdx.x; i < (len >> 2); i += kOptThreads) {
        const float4 w = ld_stream_f4(x4 + i);
        acc += (double)w.x * w.x;
        acc += (double)w.y * w.y;
        acc += (double)w.z * w.z;
        acc += (double)w.w * w.w;
    }
    const int i = (len & ~3) + threadIdx.x;
    if (i < len) acc += (double)x[i] * x[i];
    acc = block_sum_d(acc);
    if (threadIdx.x == 0) partial[blockIdx.x] = acc;
}

// seg_blk null: one norm over the np partials, torch.nn.utils.clip_grad_norm_'s factor min(max_norm / (norm + 1e-6), 1)
// with its fp32 operations (reciprocal, then multiply: torch's scalar / tensor), NaN propagated by the clamp as
// torch.clamp does.  Else nseg segments, segment s over partials [seg_blk[s], seg_blk[s + 1]) with the bound
// scal[seg_scal[s]]: BertAdam's rule, max / (norm + 1e-6) only where norm > max > 0, in double as the host computed it.
__global__ void __launch_bounds__(kOptThreads) clip_coef_kernel(const double* __restrict__ partial, int np,
                                                                 const int* __restrict__ seg_blk,
                                                                 const int* __restrict__ seg_scal, int nseg,
                                                                 const float* __restrict__ scal, float max_norm,
                                                                 float* __restrict__ norm, float* __restrict__ coef) {
    if (seg_blk == nullptr) {
        double acc = 0.0;
        for (int i = threadIdx.x; i < np; i += kOptThreads) acc += partial[i];
        acc = block_sum_d(acc);
        if (threadIdx.x == 0) {
            const float nrm = (float)sqrt(acc);
            const float c = __fmul_rn(__frcp_rn(__fadd_rn(nrm, 1e-6f)), max_norm);
            *norm = nrm;
            *coef = c > 1.f ? 1.f : c;
        }
        return;
    }
    const int lane = threadIdx.x & 31;
    for (int s = threadIdx.x >> 5; s < nseg; s += kOptThreads / 32) {
        double acc = 0.0;
        for (int i = seg_blk[s] + lane; i < seg_blk[s + 1]; i += 32) acc += partial[i];
        acc = warp_sum_d(acc);
        if (lane == 0) {
            const float nrm = (float)sqrt(acc);
            const float mx = scal[seg_scal[s]];
            norm[s] = nrm;
            coef[s] = (mx > 0.f && nrm > mx) ? (float)((double)mx / ((double)nrm + 1e-6)) : 1.f;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------
// LAMB, as apex's FusedLAMB computes it by default (adam_w_mode, grad_averaging, no nvlamb).  Per parameter tensor w:
// u = m_hat / (sqrt(v_hat) + eps) + wd*w and w -= lr * r * u with the trust ratio r = ||w|| / ||u|| (1 where wd == 0
// or either norm is 0).  r needs the whole tensor's ||u|| before any element of w may change, so a (bucket, param
// group) slice takes three streaming passes:
//   lamb_moments_kernel  p, g, m, v in; m, v out; one CTA per kSumsqChunk elements of a segment (a parameter), as
//                        grad_sumsq_kernel lays them out, each writing its fp64 sums of w^2 and u^2 to its own
//                        partials; the dirty gradient lines cleared as update_pass clears them.  p is not written.
//   lamb_ratio_kernel    one CTA: each segment's partials summed in a fixed order into ||w||, ||u|| and r
//   lamb_apply_kernel    p, m, v in; u recomputed by lamb_u, the function pass 1 used, so bit for bit the same;
//                        p -= lr*r*u, r found per float4 vector by ClipCursor over the segment ends
// Storing u instead of recomputing it moves as many bytes (it has to be written and read back) and would need a
// scratch buffer, or the gradient bucket, which would then have to be cleared densely.  The partials depend on the
// segment lengths alone and nothing orders them but the code, so the step is a function of its inputs' bits.
// scal -> {lr, weight_decay, 1 - beta1^t, 1 - beta2^t} of the group: the step's scalars (1, 1 without bias correction).
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float lamb_u(const float* s, float pw, float mw, float vw, float eps) {
    const float mh = __fdiv_rn(mw, s[2]), vh = __fdiv_rn(vw, s[3]);
    return __fmaf_rn(s[1], pw, __fdiv_rn(mh, __fadd_rn(__fsqrt_rn(vh), eps)));
}

// new m and v of one element, its w^2 and u^2 added to the CTA's sums
__device__ __forceinline__ void lamb_moments(const LambHyper& h, const float* s, float pw, float gw, float& mw,
                                             float& vw, double& aw, double& au) {
    mw = __fmaf_rn(h.omb1, gw, __fmul_rn(h.b1, mw));
    vw = __fmaf_rn(h.omb2, __fmul_rn(gw, gw), __fmul_rn(h.b2, vw));
    const float u = lamb_u(s, pw, mw, vw, h.eps);
    aw += (double)pw * pw;
    au += (double)u * u;
}

__device__ __forceinline__ bool stopped(const int* fault) {
    return fault != nullptr && *reinterpret_cast<const volatile int*>(fault) != 0;
}

// coef: the global clip factor or null
__global__ void __launch_bounds__(kOptThreads) lamb_moments_kernel(const float* __restrict__ p, float* __restrict__ g,
                                                                    float* __restrict__ m, float* __restrict__ v,
                                                                    const LambSegs t, const LambHyper h, int zero_grad,
                                                                    const float* __restrict__ scal,
                                                                    const int* __restrict__ fault,
                                                                    const int* __restrict__ skip,
                                                                    const float* __restrict__ coef,
                                                                    double* __restrict__ part_w,
                                                                    double* __restrict__ part_u) {
    if (stopped(fault)) return;
    const int q = __ldg(t.blk) + blockIdx.x;            // this CTA's partial; its segment by binary search
    int lo = 0, hi = t.nseg - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (q >= __ldg(t.blk + mid)) lo = mid; else hi = mid - 1;
    }
    const int begin = (q - __ldg(t.blk + lo)) * kSumsqChunk;
    const int len = min(__ldg(t.len + lo) - begin, kSumsqChunk);
    const int base = __ldg(t.off + lo) + begin;          // a multiple of 4
    const float4* p4 = reinterpret_cast<const float4*>(p + base);
    float4* g4 = reinterpret_cast<float4*>(g + base);
    float4* m4 = reinterpret_cast<float4*>(m + base);
    float4* v4 = reinterpret_cast<float4*>(v + base);
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    const int n4 = len >> 2, tail = (len & ~3) + threadIdx.x;
    if (verdict_set(skip)) {              // loss scaling skips this step: parameters and state stay, the gradient is cleared
        if (!zero_grad) return;
        for (int i = threadIdx.x; i < n4; i += kOptThreads) {
            const float4 gw = ld_stream_f4(g4 + i);
            if (gw.x != 0.f || gw.y != 0.f || gw.z != 0.f || gw.w != 0.f) g4[i] = zero;
        }
        if (tail < len) g[base + tail] = 0.f;
        return;
    }
    float s[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) s[j] = scal[j];
    const float c = coef != nullptr ? *coef : 1.f;
    double aw = 0.0, au = 0.0;
    for (int i = threadIdx.x; i < n4; i += kOptThreads) {
        const float4 pw = p4[i];
        float4 gw = ld_stream_f4(g4 + i), mw = m4[i], vw = v4[i];
        const bool dirty = gw.x != 0.f || gw.y != 0.f || gw.z != 0.f || gw.w != 0.f;
        if (coef != nullptr) scale4(gw, c);
        lamb_moments(h, s, pw.x, gw.x, mw.x, vw.x, aw, au); lamb_moments(h, s, pw.y, gw.y, mw.y, vw.y, aw, au);
        lamb_moments(h, s, pw.z, gw.z, mw.z, vw.z, aw, au); lamb_moments(h, s, pw.w, gw.w, mw.w, vw.w, aw, au);
        m4[i] = mw;
        v4[i] = vw;
        if (zero_grad && dirty) g4[i] = zero;
    }
    if (tail < len) {                     // the segment's last len % 4 elements, one per thread
        const int i = base + tail;
        float gw = g[i], mw = m[i], vw = v[i];
        if (coef != nullptr) gw = __fmul_rn(gw, c);
        lamb_moments(h, s, p[i], gw, mw, vw, aw, au);
        m[i] = mw;
        v[i] = vw;
        if (zero_grad) g[i] = 0.f;
    }
    aw = block_sum_d(aw);
    au = block_sum_d(au);
    if (threadIdx.x == 0) {
        part_w[q] = aw;
        part_u[q] = au;
    }
}

// One CTA, a warp per segment as in clip_coef_kernel.  r in double from the fp64 norms, rounded once.
__global__ void __launch_bounds__(kOptThreads) lamb_ratio_kernel(const LambSegs t, const double* __restrict__ part_w,
                                                                  const double* __restrict__ part_u,
                                                                  const float* __restrict__ scal,
                                                                  const int* __restrict__ fault,
                                                                  const int* __restrict__ skip,
                                                                  float* __restrict__ norm_w,
                                                                  float* __restrict__ norm_u, float* __restrict__ ratio) {
    if (stopped(fault) || verdict_set(skip)) return;
    const bool decay = scal[1] != 0.f;
    const int lane = threadIdx.x & 31;
    for (int j = threadIdx.x >> 5; j < t.nseg; j += kOptThreads / 32) {
        double aw = 0.0, au = 0.0;
        for (int i = t.blk[j] + lane; i < t.blk[j + 1]; i += 32) {
            aw += part_w[i];
            au += part_u[i];
        }
        aw = warp_sum_d(aw);
        au = warp_sum_d(au);
        if (lane == 0) {
            const double wn = sqrt(aw), un = sqrt(au);
            norm_w[j] = (float)wn;
            norm_u[j] = (float)un;
            ratio[j] = (decay && wn > 0.0 && un > 0.0) ? (float)(wn / un) : 1.f;
        }
    }
}

// r: the trust ratios of the slice's segments and their ends (float4 vectors)
__global__ void __launch_bounds__(kOptThreads) lamb_apply_kernel(float* __restrict__ p, const float* __restrict__ m,
                                                                  const float* __restrict__ v, int n, float eps,
                                                                  const float* __restrict__ scal,
                                                                  const int* __restrict__ fault,
                                                                  const int* __restrict__ skip, const ClipRef r) {
    if (stopped(fault) || verdict_set(skip)) return;
    float s[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) s[j] = scal[j];
    ClipCursor rc(r);
    const int n4 = n >> 2;
    float4* p4 = reinterpret_cast<float4*>(p);
    const float4* m4 = reinterpret_cast<const float4*>(m);
    const float4* v4 = reinterpret_cast<const float4*>(v);
    for (int i = blockIdx.x * kOptThreads + threadIdx.x; i < n4; i += gridDim.x * kOptThreads) {
        float4 pw = p4[i];
        const float4 mw = ld_stream_f4(m4 + i), vw = ld_stream_f4(v4 + i);
        const float step = __fmul_rn(s[0], rc.at(i));
        pw.x = __fmaf_rn(-step, lamb_u(s, pw.x, mw.x, vw.x, eps), pw.x);
        pw.y = __fmaf_rn(-step, lamb_u(s, pw.y, mw.y, vw.y, eps), pw.y);
        pw.z = __fmaf_rn(-step, lamb_u(s, pw.z, mw.z, vw.z, eps), pw.z);
        pw.w = __fmaf_rn(-step, lamb_u(s, pw.w, mw.w, vw.w, eps), pw.w);
        p4[i] = pw;
    }
    if (blockIdx.x == 0)
        for (int i = n4 * 4 + threadIdx.x; i < n; i += kOptThreads) {
            const float step = __fmul_rn(s[0], rc.at(i >> 2));
            p[i] = __fmaf_rn(-step, lamb_u(s, p[i], m[i], v[i], eps), p[i]);
        }
}

static inline int opt_grid(int n) {
    int g = (n / 4 + kOptThreads - 1) / kOptThreads;
    if (g < 1) g = 1;
    if (g > kStrideGridMax) g = kStrideGridMax;
    return g;
}

cudaError_t launch_fused_sgd(float* p, float* g, float* mom, int n, float momentum, float dampening, float weight_decay,
                             int nesterov, int first_step, int zero_grad, const float* scal, const int* fault,
                             const int* skip, const float* coef, cudaStream_t stream) {
    const SgdHyper h{momentum, dampening, weight_decay, nesterov, first_step};
    fused_sgd_kernel<<<opt_grid(n), kOptThreads, 0, stream>>>(p, g, mom, n, h, zero_grad, scal, fault, skip, coef);
    return cudaGetLastError();
}

cudaError_t launch_sgd_ahead(float* p, float* mom, float* sp, float* sm, const SgdRanges& r, const SgdHyper& h,
                             int max_ctas, const float* scal, cudaStream_t stream) {
    if (h.first) return cudaErrorInvalidValue;
    long long vecs = 0;
    for (int q = 0; q < r.nr; ++q) vecs += r.hi[q] - r.lo[q];
    if (vecs <= 0) return cudaSuccess;
    long long grid = (vecs + kOptThreads * kAheadUnroll - 1) / (kOptThreads * kAheadUnroll);
    grid = std::min<long long>(grid, std::max(max_ctas, 1));
    sgd_ahead_kernel<<<(int)grid, kOptThreads, 0, stream>>>(p, mom, sp, sm, r, h, scal);
    return cudaGetLastError();
}

cudaError_t launch_fused_sgd_tail(float* p, float* g, float* mom, const float* sp, const float* sm, int n,
                                  const SgdRanges& ahead, const SgdRanges& dense, const SgdHyper& h, int zero_grad,
                                  const float* scal, const int* fault, const int* skip, const float* coef,
                                  cudaStream_t stream) {
    fused_sgd_tail_kernel<<<opt_grid(n), kOptThreads, 0, stream>>>(p, g, mom, sp, sm, n, ahead, dense, h, zero_grad,
                                                                  scal, fault, skip, coef);
    return cudaGetLastError();
}

cudaError_t launch_fused_bert_adam(float* p, float* g, float* m, float* v, int n, float b1, float b2, float eps,
                                   float weight_decay, int zero_grad, const float* scal, const int* fault,
                                   const int* skip, const ClipRef& clip, cudaStream_t stream) {
    fused_bert_adam_kernel<<<opt_grid(n), kOptThreads, 0, stream>>>(p, g, m, v, n, b1, b2, eps, weight_decay, zero_grad,
                                                                   scal, fault, skip, clip);
    return cudaGetLastError();
}

cudaError_t launch_fused_adam(float* p, float* g, float* m, float* v, int n, double beta1, double beta2, float eps,
                              float weight_decay, int decoupled, int zero_grad, const float* scal, const int* fault,
                              const int* skip, const float* coef, cudaStream_t stream) {
    // 1 - beta in double, rounded once: torch passes these factors as Python floats
    fused_adam_kernel<<<opt_grid(n), kOptThreads, 0, stream>>>(p, g, m, v, n, (float)(1.0 - beta1), (float)beta2,
                                                              (float)(1.0 - beta2), eps, weight_decay, decoupled,
                                                              zero_grad, scal, fault, skip, coef);
    return cudaGetLastError();
}

cudaError_t launch_fused_lamb(float* p, float* g, float* m, float* v, int n, double beta1, double beta2, float eps,
                              const LambSegs& t, int nblk, double* part_w, double* part_u, float* norm_w,
                              float* norm_u, float* ratio, int zero_grad, const float* scal, const int* fault,
                              const int* skip, const float* coef, cudaStream_t stream) {
    // 1 - beta in double, rounded once, as for Adam
    const LambHyper h{(float)beta1, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), eps};
    lamb_moments_kernel<<<nblk, kOptThreads, 0, stream>>>(p, g, m, v, t, h, zero_grad, scal, fault, skip, coef, part_w,
                                                          part_u);
    lamb_ratio_kernel<<<1, kOptThreads, 0, stream>>>(t, part_w, part_u, scal, fault, skip, norm_w, norm_u, ratio);
    lamb_apply_kernel<<<opt_grid(n), kOptThreads, 0, stream>>>(p, m, v, n, eps, scal, fault, skip,
                                                               ClipRef{ratio, t.ends});
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

cudaError_t launch_grad_sumsq(const float* g, const SumsqSegs& t, double* partial, cudaStream_t stream) {
    if (t.nseg <= 0) return cudaSuccess;
    grad_sumsq_kernel<<<t.blk_begin[t.nseg], kOptThreads, 0, stream>>>(g, t, partial);
    return cudaGetLastError();
}

cudaError_t launch_clip_coef(const double* partial, int np, const int* seg_blk, const int* seg_scal, int nseg,
                             const float* scal, float max_norm, float* norm, float* coef, cudaStream_t stream) {
    clip_coef_kernel<<<1, kOptThreads, 0, stream>>>(partial, np, seg_blk, seg_scal, nseg, scal, max_norm, norm, coef);
    return cudaGetLastError();
}

}  // namespace okt
