// Device-side building blocks shared by every kernel of oktopk_b200 (sm_90a only).
//
//  * system-scope release/acquire flags for the cross-GPU handshakes (peer-visible mailboxes
//    in IPC-mapped memory reached through NVLink 4 / NVSwitch),
//  * a monotonic-ticket grid barrier for the persistent cooperative kernels,
//  * TMA 1-D bulk copies (cp.async.bulk global->shared, mbarrier completion) used to pull
//    remote (idx,val) chunks,
//  * 128-bit streaming loads/stores and warp-aggregated slot allocation.
//
// Replaces the reference's host-staged mpi4py calls (SURVEY 2.4 table B); nothing here is
// derived from reference code (it has no device code at all).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#ifndef OKT_MAXP
#define OKT_MAXP 16            // max ranks per node-level peer group
#endif

namespace okt {

// ----------------------------------------------------------------------------------------
// timers
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// ----------------------------------------------------------------------------------------
// memory-model primitives
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ void st_release_sys_u64(uint64_t* p, uint64_t v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t ld_acquire_sys_u64(const uint64_t* p) {
    uint64_t v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint64_t ld_relaxed_sys_u64(const uint64_t* p) {
    uint64_t v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_sys_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys_u64(uint64_t* p, uint64_t v) {
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_relaxed_sys_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_acquire_gpu_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t ld_acquire_gpu_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_gpu_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t atom_add_acq_rel_gpu_u32(uint32_t* p, uint32_t v) {
    uint32_t old;
    asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
    return old;
}
__device__ __forceinline__ void fence_acq_rel_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }
__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }


// Failure detection on the device: every cross-GPU spin is bounded.  When a peer does not show up within
// `timeout_ns` the waiter records a fault code in *fault (device memory, read lazily by the host) and gives up,
// so a dead or wedged peer turns into a reported error instead of a hung GPU.  Once a fault is recorded every
// later wait of the same bucket returns immediately.
enum FaultCode : int { FAULT_NONE = 0, FAULT_RS_TIMEOUT = 1, FAULT_AG_TIMEOUT = 2, FAULT_CUT_TIMEOUT = 3, FAULT_DENSE_TIMEOUT = 4,
                       FAULT_TREE_TIMEOUT = 5, FAULT_DONE_TIMEOUT = 6, FAULT_SCALE_TIMEOUT = 7 };

struct SpinGuard {
    int* fault;
    unsigned long long timeout_ns;
    int code;
    int* host_fault = nullptr;    // mapped pinned mirror of *fault: the host polls it at every step without a sync
};

// Record a fault once (first writer wins), mirror it to the host.  The fused optimizer kernels read *fault and skip
// the parameter update, so a partial (timed-out) reduction is never applied.
__device__ __forceinline__ void raise_fault(const SpinGuard& sg) {
    if (atomicCAS(sg.fault, FAULT_NONE, sg.code) == FAULT_NONE && sg.host_fault != nullptr) {
        *reinterpret_cast<volatile int*>(sg.host_fault) = sg.code;
        __threadfence_system();
    }
}

// Loss scaling: the bucket's (or step's) verdict, written by an earlier kernel of the stream; null when scaling is off.
// A reduction kernel returns at entry when it is set -- every rank holds the same verdict, so no peer waits for it.
__device__ __forceinline__ bool verdict_set(const int* skip) {
    return skip != nullptr && *reinterpret_cast<const volatile int*>(skip) != 0;
}

// Spin until the mailbox word carries `epoch` in its high half; returns the low half (payload), 0 on fault.
__device__ __forceinline__ uint32_t wait_mailbox(const uint64_t* box, uint32_t epoch, const SpinGuard& sg) {
    uint64_t v = ld_acquire_sys_u64(box);
    if ((uint32_t)(v >> 32) == epoch) return (uint32_t)v;
    const unsigned long long t0 = globaltimer_ns();
    uint32_t spins = 0;
    while ((uint32_t)(v >> 32) != epoch) {
        __nanosleep(20);
        if ((++spins & 1023u) == 0 && sg.fault != nullptr) {
            if (*reinterpret_cast<volatile int*>(sg.fault) != FAULT_NONE) return 0u;
            if (sg.timeout_ns != 0ULL && globaltimer_ns() - t0 > sg.timeout_ns) {
                raise_fault(sg);
                return 0u;
            }
        }
        v = ld_acquire_sys_u64(box);
    }
    return (uint32_t)v;
}
__device__ __forceinline__ uint64_t make_mail(uint32_t epoch, uint32_t payload) {
    return ((uint64_t)epoch << 32) | (uint64_t)payload;
}

// ----------------------------------------------------------------------------------------
// grid barrier (all CTAs co-resident: cooperative launch). 64-bit ticket counter: each barrier
// consumes exactly G tickets, so the target is derived from one's own ticket and the counter
// never has to be reset.  G is the number of CTAs that sync on `bar`: the whole grid, or a
// group of CTAs that shares nothing with the rest of the grid between barriers and has a
// counter of its own.
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ void grid_sync(unsigned long long* bar, unsigned long long G) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        unsigned long long old = atomicAdd(bar, 1ULL);
        unsigned long long target = (old / G + 1ULL) * G;
        while (ld_acquire_gpu_u64(bar) < target) { }
        __threadfence();
    }
    __syncthreads();
}
__device__ __forceinline__ void grid_sync(unsigned long long* bar) { grid_sync(bar, gridDim.x); }

// "Last CTA done" ticket: every CTA calls it once when it has finished a phase; exactly one call -- the last one of
// the grid -- returns true, with all other CTAs' prior global writes visible to it (and, through a subsequent
// system-scope release, to peers).  Replaces a grid barrier wherever only ONE thread has to act on "everybody is done"
// (publishing a count to the peers): nobody waits, the counter resets itself.
__device__ __forceinline__ bool last_cta_ticket(unsigned int* ticket) {
    __shared__ int s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned int old = atomicAdd(ticket, 1u);
        const int last = (old == gridDim.x - 1u) ? 1 : 0;
        if (last) { __threadfence(); *reinterpret_cast<volatile unsigned int*>(ticket) = 0u; }
        s_last = last;
    }
    __syncthreads();
    return s_last != 0;
}

// ----------------------------------------------------------------------------------------
// streaming 128-bit accesses
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ float4 ld_stream_f4(const float4* p) {
    float4 r;
    asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void st_stream_f4(float4* p, const float4& v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};"
                 ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// coherent-at-L2 scalar load (data that other CTAs updated with atomics / plain stores)
__device__ __forceinline__ float ld_cg_f32(const float* p) { return __ldcg(p); }
__device__ __forceinline__ int   ld_cg_s32(const int* p)   { return __ldcg(p); }
// peer loads after an acquire: volatile so neither the compiler nor a stale L1 line serves them
__device__ __forceinline__ float ld_peer_f32(const float* p) {
    float v; asm volatile("ld.relaxed.sys.global.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ int ld_peer_s32(const int* p) {
    int v; asm volatile("ld.relaxed.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ int4 ld_peer_i4(const int4* p) {
    int4 r;
    asm volatile("ld.relaxed.sys.global.v4.s32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p) : "memory");
    return r;
}
__device__ __forceinline__ void red_add_f32(float* p, float v) {
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

// ----------------------------------------------------------------------------------------
// mbarrier + TMA 1-D bulk copy (global -> shared::cta)
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// Intra-SM wait (TMA completion / ring-stage hand-over).  These can only stall on a programming error, so the spin is
// bounded: after ~4 s the kernel traps (a reported launch failure) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const unsigned long long t0 = globaltimer_ns();
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 4095u) == 0 && globaltimer_ns() - t0 > 4000000000ULL) __trap();
    }
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// bytes: multiple of 16; src/dst 16-byte aligned. src may be a peer GPU's memory.
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// order ALL prior generic-proxy accesses (global data other CTAs produced before the grid barrier, and this CTA's
// shared-memory reads of a ring stage) before subsequent async-proxy (TMA) operations
__device__ __forceinline__ void fence_proxy_async_all() {
    asm volatile("fence.proxy.async;" ::: "memory");
}
// make generic-proxy smem reads that preceded this point ordered before later async-proxy writes
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ----------------------------------------------------------------------------------------
// warp helpers
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Warp-aggregated append: every lane with `pred` gets a unique position from *cursor; one atomic
// per warp per call. All 32 lanes must call (converged).
__device__ __forceinline__ int warp_append(int* cursor, bool pred) {
    unsigned m = __ballot_sync(0xffffffffu, pred);
    if (m == 0) return -1;
    int leader = __ffs(m) - 1;
    int base = 0;
    if (lane_id() == leader) base = atomicAdd(cursor, __popc(m));
    base = __shfl_sync(0xffffffffu, base, leader);
    return pred ? base + __popc(m & ((1u << lane_id()) - 1u)) : -1;
}

// Same for a possibly partially-active warp (tail of a strided loop): aggregates over the active lanes only.
__device__ __forceinline__ int warp_append_active(int* cursor, bool pred) {
    const unsigned act = __activemask();
    const unsigned m = __ballot_sync(act, pred);
    if (m == 0) return -1;
    const int leader = __ffs(m) - 1;
    int base = 0;
    if (lane_id() == leader) base = atomicAdd(cursor, __popc(m));
    base = __shfl_sync(act, base, leader);
    return pred ? base + __popc(m & ((1u << lane_id()) - 1u)) : -1;
}

__device__ __forceinline__ uint32_t abs_bits(float x) { return __float_as_uint(x) & 0x7fffffffu; }

}  // namespace okt
