// Dynamic loss scaling on the device.
//
// unscale_check runs per bucket on the communication stream right before the bucket's reduction: it multiplies the
// gradient by inv_scale in place (the autograd tensors of the direct Ok-Topk path, or the landed bucket) and ORs a
// non-finite flag.  The last CTA then agrees on the flag with every peer through the bucket's symmetric block, writes
// the bucket verdict (which the reduction kernels read at entry: skip = return before any write) and ORs it into the
// optimizer's step verdict (which the update kernels read).  Nothing is decided on the host, so the step stays CUDA-graph
// replayable and adds no synchronisation.
#include "common.cuh"
#include "oktopk.cuh"

namespace okt {

__device__ __forceinline__ bool nonfinite(float x) { return (__float_as_uint(x) & 0x7f800000u) == 0x7f800000u; }

__global__ void __launch_bounds__(kScaleThreads) unscale_check_kernel(const ScaleParams p) {
    int lo = 0, hi = p.nseg - 1;             // which segment does this CTA work on?
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if ((int)blockIdx.x >= p.blk_begin[mid]) lo = mid; else hi = mid - 1;
    }
    const int t = lo;
    float* __restrict__ x = p.src[t];
    const long long begin = (long long)(blockIdx.x - p.blk_begin[t]) * kScalePerCta;   // 64-bit: no overflow near 2^31
    const long long end = min((long long)p.len[t], begin + kScalePerCta);
    const float inv = p.ls->inv_scale;
    bool bad = false;
    // torch's rule: the flag looks at the incoming value, the output is value * inv_scale (one fp32 rounding)
    const long long v0 = begin >> 2, v1 = end >> 2;      // begin is a multiple of 4; sources are 16-byte aligned
    float4* x4 = reinterpret_cast<float4*>(x);
    for (long long v = v0 + threadIdx.x; v < v1; v += kScaleThreads) {
        float4 w = ld_stream_f4(x4 + v);
        bad |= nonfinite(w.x) | nonfinite(w.y) | nonfinite(w.z) | nonfinite(w.w);
        w.x = __fmul_rn(w.x, inv); w.y = __fmul_rn(w.y, inv); w.z = __fmul_rn(w.z, inv); w.w = __fmul_rn(w.w, inv);
        st_stream_f4(x4 + v, w);
    }
    for (long long i = (v1 << 2) + threadIdx.x; i < end; i += kScaleThreads) {
        const float w = x[i];
        bad |= nonfinite(w);
        x[i] = __fmul_rn(w, inv);
    }
    if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(&p.sync->flag, 1);
    if (!last_cta_ticket(&p.sync->ticket) || threadIdx.x != 0) return;
    int flag = atomicExch(&p.sync->flag, 0);
    // a fault left by an earlier call of this bucket makes this rank skip: publish that, so every rank skips with it
    if (*reinterpret_cast<volatile int*>(p.fault) != FAULT_NONE) flag = 1;
    const uint32_t epoch = p.sync->epoch + 1u;
    p.sync->epoch = epoch;
    if (p.P > 1) {
        const int par = epoch & 1u;
        const uint64_t mail = make_mail(epoch, (uint32_t)flag);
        for (int d = 0; d < p.P; ++d)
            if (d != p.rank)
                st_release_sys_u64(reinterpret_cast<uint64_t*>(p.peers[d] + p.mbox_off) + par * OKT_MAXP + p.rank, mail);
        const SpinGuard sg{p.fault, p.timeout_ns, FAULT_SCALE_TIMEOUT, p.host_fault};
        const uint64_t* box = reinterpret_cast<const uint64_t*>(p.peers[p.rank] + p.mbox_off) + par * OKT_MAXP;
        for (int s = 0; s < p.P; ++s)
            if (s != p.rank) flag |= (int)wait_mailbox(box + s, epoch, sg);
        // a peer timed out in this exchange: the bucket is not reduced here (the update kernels also skip on the fault
        // word); the peer that did not show up is wedged or gone, and the host's fault handling resynchronises the replicas
        if (*reinterpret_cast<volatile int*>(p.fault) != FAULT_NONE) flag = 1;
    }
    flag = flag ? 1 : 0;
    p.sync->verdict = flag;
    if (flag) atomicOr(&p.ls->found_inf, 1);
}

__global__ void scale_update_kernel(LossScaleDev* ls, double growth_factor, double backoff_factor, int growth_interval) {
    // torch._amp_update_scale_ (aten/src/ATen/native/cuda/AmpKernels.cu), then GradScaler's inv_scale
    const int found = ls->found_inf;
    if (found) {
        ls->scale = (float)((double)ls->scale * backoff_factor);
        ls->growth_tracker = 0;
    } else {
        const int successful = ls->growth_tracker + 1;
        if (successful == growth_interval) {
            const float grown = (float)((double)ls->scale * growth_factor);
            if (isfinite(grown)) ls->scale = grown;
            ls->growth_tracker = 0;
        } else {
            ls->growth_tracker = successful;
        }
    }
    ls->inv_scale = (float)(1.0 / (double)ls->scale);
    ls->skipped += found;
    ls->adam_step += 1 - found;
    ls->found_inf = 0;
}

__global__ void adam_scalars_kernel(const LossScaleDev* ls, const double* hyper, float* scal, int groups, int lamb) {
    // torch's non-capturable Adam, in double: t = the step about to run (skipped steps do not count)
    const double t = (double)(ls->adam_step + 1);
    for (int gi = threadIdx.x; gi < groups; gi += blockDim.x) {
        const double lr = hyper[4 * gi], wd = hyper[4 * gi + 1], b1 = hyper[4 * gi + 2], b2 = hyper[4 * gi + 3];
        if (lamb) {                                     // _LambUpdate.scalars, in the same double arithmetic
            scal[4 * gi] = (float)lr;
            scal[4 * gi + 1] = (float)wd;
            scal[4 * gi + 2] = (float)(1.0 - pow(b1, t));
            scal[4 * gi + 3] = (float)(1.0 - pow(b2, t));
            continue;
        }
        scal[3 * gi] = (float)(1.0 - lr * wd);
        scal[3 * gi + 1] = (float)((lr / (1.0 - pow(b1, t))) * -1.0);
        scal[3 * gi + 2] = (float)sqrt(1.0 - pow(b2, t));
    }
}

__global__ void __launch_bounds__(kScaleThreads) carry_residual_kernel(float* __restrict__ g, float* __restrict__ res,
                                                                        int n, const int* __restrict__ skip) {
    if (*reinterpret_cast<const volatile int*>(skip) != 0) return;
    for (int i = blockIdx.x * kScaleThreads + threadIdx.x; i < n; i += gridDim.x * kScaleThreads) {
        g[i] = __fadd_rn(g[i], res[i]);
        res[i] = 0.f;
    }
}

cudaError_t launch_unscale_check(const ScaleParams& p, cudaStream_t stream) {
    if (p.nseg <= 0) return cudaErrorInvalidValue;
    unscale_check_kernel<<<p.blk_begin[p.nseg], kScaleThreads, 0, stream>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_scale_update(LossScaleDev* ls, double growth_factor, double backoff_factor, int growth_interval,
                                cudaStream_t stream) {
    scale_update_kernel<<<1, 1, 0, stream>>>(ls, growth_factor, backoff_factor, growth_interval);
    return cudaGetLastError();
}

cudaError_t launch_adam_scalars(const LossScaleDev* ls, const double* hyper, float* scal, int groups, int lamb,
                                cudaStream_t stream) {
    adam_scalars_kernel<<<1, 32, 0, stream>>>(ls, hyper, scal, groups, lamb);
    return cudaGetLastError();
}

cudaError_t launch_carry_residual(float* g, float* res, int n, const int* skip, cudaStream_t stream) {
    int grid = (n + kScaleThreads - 1) / kScaleThreads;
    if (grid < 1) grid = 1;
    if (grid > kStrideGridMax) grid = kStrideGridMax;
    carry_residual_kernel<<<grid, kScaleThreads, 0, stream>>>(g, res, n, skip);
    return cudaGetLastError();
}

}  // namespace okt
