// Dense allreduce over NVLink peer memory (two-shot, in place, one kernel): every gradient
// bucket lives in a symmetric IPC allocation, rank r owns the r-th shard, reads that shard from
// all P buckets with 128-bit peer loads, averages, and stores the result straight into all P
// buckets.  Cross-GPU synchronisation is per-CTA (CTA i of every rank handles slice i of every
// shard): a start barrier (everyone's backward has produced the bucket) and an end barrier
// (everyone's stores have landed) built from st.release.sys / ld.acquire.sys flags.
//
// Two data paths behind the same barriers:
//   * NVLS (p.mc != null): the bucket is also mapped through an NVSwitch MULTICAST object; `multimem.ld_reduce`
//     lets the switch add the P copies of a vector on the fly (one load returns the sum) and `multimem.st`
//     broadcasts the averaged vector to all P buckets with one store -- each GPU moves n/P in and n/P out over its
//     links instead of (P-1)/P*n each way;
//   * peer loads/stores (no multicast mapping): the owner reads the P copies with 128-bit peer loads.
// The launch is cooperative: the per-CTA cross-GPU barriers need CTA i of every rank to be resident, which a plain
// launch does not guarantee while backward kernels still hold SMs.
//
// Serves the dense baseline (`compressor none`), the dense warm-up iterations of every sparse
// scheme and TopkDSA's dense fallback -- reference: dense_allreduce / _dense_allreduce,
// VGG/allreducer.py:175-180,532-547 (host MPI.Allreduce on NumPy buffers).
#include "common.cuh"
#include "oktopk.cuh"

namespace okt {

constexpr int kDenseThreads = 512;
constexpr int kDenseTile = 2;
constexpr int kSrcGroup = 8;

__device__ __forceinline__ void cta_peer_barrier(const DenseParams& p, int phase, uint64_t ticket) {
    // flag block layout per rank: uint64 [2 phases][gridDim.x][OKT_MAXP]
    __syncthreads();
    const int tid = threadIdx.x;
    if (tid < p.P) {
        const size_t slot = ((size_t)phase * gridDim.x + blockIdx.x) * OKT_MAXP;
        fence_acq_rel_sys();
        st_release_sys_u64(p.flags[tid] + slot + p.rank, ticket);        // tell peer `tid` I am here
        const uint64_t* mine = p.flags[p.rank] + slot + tid;             // wait for peer `tid`
        const unsigned long long t0 = globaltimer_ns();
        uint32_t spins = 0;
        while (ld_acquire_sys_u64(mine) < ticket) {
            __nanosleep(20);
            if ((++spins & 1023u) == 0 && p.fault != nullptr) {
                if (*reinterpret_cast<volatile int*>(p.fault) != FAULT_NONE) break;
                if (p.timeout_ns != 0ULL && globaltimer_ns() - t0 > p.timeout_ns) {
                    raise_fault(SpinGuard{p.fault, p.timeout_ns, FAULT_DENSE_TIMEOUT, p.host_fault});
                    break;
                }
            }
        }
    }
    __syncthreads();
}

__global__ void __launch_bounds__(kDenseThreads, 1) dense_allreduce_kernel(const DenseParams p) {
    if (verdict_set(p.skip)) return;
    const int P = p.P, rank = p.rank;
    // one monotonically increasing ticket per CTA, device resident (CUDA-graph friendly)
    __shared__ unsigned long long s_ticket;
    if (threadIdx.x == 0) s_ticket = p.epoch[blockIdx.x] + 1ULL;
    __syncthreads();
    const uint64_t ticket = s_ticket;

    cta_peer_barrier(p, 0, ticket);

    const int n4 = p.n >> 2;                      // bucket sizes are padded to a multiple of 4
    const int shard4 = (n4 + P - 1) / P;
    const int lo = rank * shard4;
    const int hi = min(n4, lo + shard4);
    const float scale = p.scale;
    if (p.mc != nullptr) {
        // ---- NVLS: reduce in the switch, broadcast through the switch ---------------------------------------------
        float4* mc4 = reinterpret_cast<float4*>(p.mc);
        constexpr int kU = 4;                            // independent multimem loads in flight per thread
        const int trip = gridDim.x * kDenseThreads * kU;
        for (int base = lo + blockIdx.x * kDenseThreads * kU; base < hi; base += trip) {
            float4 acc[kU];
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const int v = base + u * kDenseThreads + threadIdx.x;
                if (v < hi)
                    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                                 : "=f"(acc[u].x), "=f"(acc[u].y), "=f"(acc[u].z), "=f"(acc[u].w) : "l"(mc4 + v) : "memory");
            }
#pragma unroll
            for (int u = 0; u < kU; ++u) {
                const int v = base + u * kDenseThreads + threadIdx.x;
                if (v < hi)
                    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
                                 ::"l"(mc4 + v), "f"(acc[u].x * scale), "f"(acc[u].y * scale), "f"(acc[u].z * scale),
                                   "f"(acc[u].w * scale) : "memory");
            }
        }
    } else {
    // kDenseTile vectors per thread per trip and all P peer loads of a vector issued back to back: NVLink
    // round trips are ~2-3 us, so bandwidth is bought with bytes in flight (512 thr x 2 x P x 16 B per SM).
    const int trip = gridDim.x * kDenseThreads * kDenseTile;
    for (int base = lo + blockIdx.x * kDenseThreads * kDenseTile; base < hi; base += trip) {
        float4 accs[kDenseTile];
#pragma unroll
        for (int u = 0; u < kDenseTile; ++u) accs[u] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
        for (int s0 = 0; s0 < P; s0 += kSrcGroup) {      // sources in groups of 8 (register budget), fixed order
            int4 raw[kDenseTile][kSrcGroup];
#pragma unroll
            for (int u = 0; u < kDenseTile; ++u) {
                const int v = base + u * kDenseThreads + threadIdx.x;
                if (v < hi) {
#pragma unroll
                    for (int s = 0; s < kSrcGroup; ++s)
                        if (s0 + s < P) raw[u][s] = ld_peer_i4(reinterpret_cast<const int4*>(p.bufs[s0 + s]) + v);
                }
            }
#pragma unroll
            for (int u = 0; u < kDenseTile; ++u) {
#pragma unroll
                for (int s = 0; s < kSrcGroup; ++s)      // every rank computes bitwise the same sum
                    if (s0 + s < P) {
                        accs[u].x += __int_as_float(raw[u][s].x); accs[u].y += __int_as_float(raw[u][s].y);
                        accs[u].z += __int_as_float(raw[u][s].z); accs[u].w += __int_as_float(raw[u][s].w);
                    }
            }
        }
#pragma unroll
        for (int u = 0; u < kDenseTile; ++u) {
            const int v = base + u * kDenseThreads + threadIdx.x;
            if (v < hi) {
                float4 acc = accs[u];
                acc.x *= scale; acc.y *= scale; acc.z *= scale; acc.w *= scale;
#pragma unroll 1
                for (int t = 0; t < P; ++t) {
                    const int s = (rank + t) % P;
                    st_stream_f4(reinterpret_cast<float4*>(p.bufs[s]) + v, acc);
                }
            }
        }
    }
    }
    // scalar tail (n % 4) is reduced by rank 0's CTA 0
    if (rank == 0 && blockIdx.x == 0) {
        for (int i = n4 * 4 + threadIdx.x; i < p.n; i += kDenseThreads) {
            float a = 0.f;
            for (int s = 0; s < P; ++s) a += ld_peer_f32(p.bufs[s] + i);
            a *= scale;
            for (int s = 0; s < P; ++s) p.bufs[s][i] = a;
        }
    }
    __threadfence_system();
    cta_peer_barrier(p, 1, ticket);
    if (threadIdx.x == 0) p.epoch[blockIdx.x] = ticket;
}

cudaError_t launch_dense_allreduce(const DenseParams& p, int grid, cudaStream_t stream) {
    void* args[] = {(void*)&p};
    return cudaLaunchCooperativeKernel((void*)dense_allreduce_kernel, dim3(grid), dim3(kDenseThreads), args, 0, stream);
}

}  // namespace okt
