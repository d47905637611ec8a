// Python bindings (pybind11, no torch C++ dependency: tensors cross the boundary as raw device
// pointers + CUDA stream handles) and the symmetric peer-memory allocator.
//
// The allocator is the native replacement of the reference's mpi4py communicator bootstrap
// (VGG/allreducer.py:219-220): every rank cudaMalloc's a block, exports a CUDA IPC handle, and
// maps every peer's block into its own address space, after which kernels address peer memory
// with plain ld/st/red/cp.async.bulk over NVLink 4 / NVSwitch.
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>
#include <cuda.h>            // driver-API TYPES only: the entry points are resolved at run time (cudaGetDriverEntryPoint),
#include <cuda_runtime.h>    // so the module imports on a box without libcuda (the CPU build check)

#include <unistd.h>

#include <algorithm>
#include <cstring>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

#include "oktopk.cuh"

namespace py = pybind11;
using namespace okt;

static void ck(cudaError_t e, const char* what) {
    if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}
template <class T> static T* P_(uint64_t p) { return reinterpret_cast<T*>(p); }
static cudaStream_t S_(uint64_t s) { return reinterpret_cast<cudaStream_t>(s); }

// ------------------------------------------------------------------------------------------- symmetric memory
static py::tuple symm_alloc(size_t nbytes) {
    void* p = nullptr;
    ck(cudaMalloc(&p, nbytes), "cudaMalloc(symm)");
    ck(cudaMemset(p, 0, nbytes), "cudaMemset(symm)");
    cudaIpcMemHandle_t h;
    ck(cudaIpcGetMemHandle(&h, p), "cudaIpcGetMemHandle");
    return py::make_tuple((uint64_t)p, py::bytes(reinterpret_cast<const char*>(&h), sizeof(h)));
}
static uint64_t symm_open(const std::string& handle) {
    if (handle.size() != sizeof(cudaIpcMemHandle_t)) throw std::runtime_error("bad IPC handle size");
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handle.data(), sizeof(h));
    void* p = nullptr;
    ck(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle");
    return (uint64_t)p;
}
static void symm_close(uint64_t p) { ck(cudaIpcCloseMemHandle(P_<void>(p)), "cudaIpcCloseMemHandle"); }
static void symm_free(uint64_t p) { ck(cudaFree(P_<void>(p)), "cudaFree(symm)"); }
static uint64_t dev_alloc_zero(size_t nbytes) {
    void* p = nullptr;
    ck(cudaMalloc(&p, nbytes), "cudaMalloc");
    ck(cudaMemset(p, 0, nbytes), "cudaMemset");
    return (uint64_t)p;
}
static void dev_free(uint64_t p) {
    if (p) ck(cudaFree(P_<void>(p)), "cudaFree");
}
static void memset_async(uint64_t p, int value, size_t nbytes, uint64_t stream) {
    ck(cudaMemsetAsync(P_<void>(p), value, nbytes, S_(stream)), "cudaMemsetAsync");
}
static int can_access_peer(int dev, int peer) {
    int ok = 0;
    ck(cudaDeviceCanAccessPeer(&ok, dev, peer), "cudaDeviceCanAccessPeer");
    return ok;
}


// ------------------------------------------------------------------------------------------- VMM + NVSwitch multicast
// The NVLS dense path needs the bucket mapped through a MULTICAST object (multimem.ld_reduce / multimem.st address
// all P copies at once), which CUDA IPC handles cannot provide: the block is then allocated with the virtual-memory
// API (cuMemCreate, exported as a POSIX file descriptor that Python passes to the peers over a unix socket),
// mapped by every peer (unicast, as before) and bound to a multicast object created by rank 0.
// Driver entry points are looked up at run time so that this module has no link-time dependency on libcuda.
namespace drv {
template <class F> static F sym(const char* name) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &q);
    if (e != cudaSuccess || fn == nullptr || q != cudaDriverEntryPointSuccess)
        throw std::runtime_error(std::string("driver entry point not available: ") + name);
    return reinterpret_cast<F>(fn);
}
static void ckd(CUresult r, const char* what) {
    if (r != CUDA_SUCCESS) throw std::runtime_error(std::string(what) + ": CUresult " + std::to_string((int)r));
}
}  // namespace drv

static CUmemAllocationProp vmm_prop(int dev) {
    CUmemAllocationProp prop;
    std::memset(&prop, 0, sizeof(prop));
    prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    prop.location.id = dev;
    prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    return prop;
}

// {vmm: 0/1, posix_fd: 0/1, multicast: 0/1, granularity, mc_granularity}
static py::dict vmm_probe(int dev, int ndev) {
    py::dict d;
    d["vmm"] = 0; d["posix_fd"] = 0; d["multicast"] = 0; d["granularity"] = 0; d["mc_granularity"] = 0;
    try {
        auto getattr_ = drv::sym<CUresult (*)(int*, CUdevice_attribute, CUdevice)>("cuDeviceGetAttribute");
        int v = 0;
        if (getattr_(&v, CU_DEVICE_ATTRIBUTE_VIRTUAL_MEMORY_MANAGEMENT_SUPPORTED, dev) == CUDA_SUCCESS) d["vmm"] = v;
        if (getattr_(&v, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED, dev) == CUDA_SUCCESS) d["posix_fd"] = v;
        if (getattr_(&v, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev) == CUDA_SUCCESS) d["multicast"] = v;
        auto gran = drv::sym<CUresult (*)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags)>("cuMemGetAllocationGranularity");
        CUmemAllocationProp prop = vmm_prop(dev);
        size_t g = 0;
        if (gran(&g, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS) d["granularity"] = g;
        if (d["multicast"].cast<int>() && ndev > 1) {
            auto mgran = drv::sym<CUresult (*)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags)>("cuMulticastGetGranularity");
            CUmulticastObjectProp mp;
            std::memset(&mp, 0, sizeof(mp));
            mp.numDevices = ndev; mp.size = 1 << 21; mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
            size_t mg = 0;
            if (mgran(&mg, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS) d["mc_granularity"] = mg;
        }
    } catch (const std::exception& e) {
        d["error"] = std::string(e.what());
    }
    return d;
}

// physical allocation on `dev`, exported as a POSIX fd: (handle, fd)
static py::tuple vmm_create(size_t nbytes, int dev) {
    auto create = drv::sym<CUresult (*)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long)>("cuMemCreate");
    auto exp = drv::sym<CUresult (*)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long)>("cuMemExportToShareableHandle");
    CUmemAllocationProp prop = vmm_prop(dev);
    CUmemGenericAllocationHandle h = 0;
    drv::ckd(create(&h, nbytes, &prop, 0), "cuMemCreate");
    int fd = -1;
    drv::ckd(exp(&fd, h, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0), "cuMemExportToShareableHandle");
    return py::make_tuple((uint64_t)h, fd);
}
static uint64_t vmm_import(int fd) {
    auto imp = drv::sym<CUresult (*)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType)>("cuMemImportFromShareableHandle");
    CUmemGenericAllocationHandle h = 0;
    drv::ckd(imp(&h, reinterpret_cast<void*>(static_cast<uintptr_t>(fd)), CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR), "cuMemImportFromShareableHandle");
    return (uint64_t)h;
}
// map a (memory or multicast) handle into this process with read/write access for `dev`
static uint64_t vmm_map(uint64_t handle, size_t nbytes, int dev, size_t align) {
    auto reserve = drv::sym<CUresult (*)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long)>("cuMemAddressReserve");
    auto map = drv::sym<CUresult (*)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long)>("cuMemMap");
    auto access = drv::sym<CUresult (*)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t)>("cuMemSetAccess");
    CUdeviceptr va = 0;
    drv::ckd(reserve(&va, nbytes, align, 0, 0), "cuMemAddressReserve");
    drv::ckd(map(va, nbytes, 0, (CUmemGenericAllocationHandle)handle, 0), "cuMemMap");
    CUmemAccessDesc ad;
    std::memset(&ad, 0, sizeof(ad));
    ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    ad.location.id = dev;
    ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    drv::ckd(access(va, nbytes, &ad, 1), "cuMemSetAccess");
    return (uint64_t)va;
}
static void vmm_unmap(uint64_t va, size_t nbytes) {
    auto unmap = drv::sym<CUresult (*)(CUdeviceptr, size_t)>("cuMemUnmap");
    auto afree = drv::sym<CUresult (*)(CUdeviceptr, size_t)>("cuMemAddressFree");
    unmap((CUdeviceptr)va, nbytes);
    afree((CUdeviceptr)va, nbytes);
}
static void vmm_release(uint64_t handle) {
    auto rel = drv::sym<CUresult (*)(CUmemGenericAllocationHandle)>("cuMemRelease");
    rel((CUmemGenericAllocationHandle)handle);
}
// multicast object over `ndev` devices: (handle, fd).  Created by one rank, imported (vmm_import) by the others.
static py::tuple mc_create(size_t nbytes, int ndev) {
    auto create = drv::sym<CUresult (*)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*)>("cuMulticastCreate");
    auto exp = drv::sym<CUresult (*)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long)>("cuMemExportToShareableHandle");
    CUmulticastObjectProp mp;
    std::memset(&mp, 0, sizeof(mp));
    mp.numDevices = ndev; mp.size = nbytes; mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    CUmemGenericAllocationHandle h = 0;
    drv::ckd(create(&h, &mp), "cuMulticastCreate");
    int fd = -1;
    drv::ckd(exp(&fd, h, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0), "cuMemExportToShareableHandle(mc)");
    return py::make_tuple((uint64_t)h, fd);
}
static void mc_add_device(uint64_t mc, int dev) {
    auto add = drv::sym<CUresult (*)(CUmemGenericAllocationHandle, CUdevice)>("cuMulticastAddDevice");
    drv::ckd(add((CUmemGenericAllocationHandle)mc, dev), "cuMulticastAddDevice");
}
static void mc_bind(uint64_t mc, uint64_t mem, size_t nbytes) {
    auto bind = drv::sym<CUresult (*)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t, unsigned long long)>("cuMulticastBindMem");
    drv::ckd(bind((CUmemGenericAllocationHandle)mc, 0, (CUmemGenericAllocationHandle)mem, 0, nbytes, 0), "cuMulticastBindMem");
}

// ------------------------------------------------------------------------------------------- state access
static size_t state_bytes() { return sizeof(OktState); }

static py::dict layout_info(int P, int n, int cap, int gcap) {
    SymmLayout L = make_layout(P, n, cap, gcap);
    py::dict d;
    d["total"] = L.total; d["rs_mbox"] = L.rs_mbox; d["rs_thr"] = L.rs_thr; d["ag_mbox"] = L.ag_mbox;
    d["cut_mbox"] = L.cut_mbox; d["cut_data"] = L.cut_data; d["send_idx"] = L.send_idx; d["send_val"] = L.send_val;
    d["gat_idx"] = L.gat_idx; d["gat_val"] = L.gat_val; d["cap"] = L.cap; d["gcap"] = L.gcap; d["scap"] = L.scap;
    d["done_mbox"] = L.done_mbox; d["tree_mbox"] = L.tree_mbox; d["scale_mbox"] = L.scale_mbox;
    d["chunk"] = kChunk; d["maxp"] = OKT_MAXP; d["threads"] = kThreads;
    return d;
}

// Synchronous (stream-ordered copy + sync): observability only, never on the hot path.
static py::dict read_state(uint64_t st, int P, uint64_t stream) {
    static thread_local std::vector<char> host(offsetof(OktState, hist));
    ck(cudaMemcpyAsync(host.data(), P_<void>(st), host.size(), cudaMemcpyDeviceToHost, S_(stream)), "read_state");
    ck(cudaStreamSynchronize(S_(stream)), "read_state sync");
    const OktState* s = reinterpret_cast<const OktState*>(host.data());
    py::dict d;
    d["local_thr"] = s->local_thr; d["local_thr_used"] = s->local_thr_used; d["global_thr"] = s->global_thr;
    d["epoch"] = s->epoch;
    std::vector<int> e(s->edges, s->edges + P + 1);
    d["edges"] = e;
    d["local_count"] = s->stat_local_count; d["global_count"] = s->stat_global_count;
    d["recv_total"] = s->stat_recv_total; d["gather_total"] = s->stat_gather_total;
    d["overflow_send"] = s->stat_overflow_send; d["overflow_gather"] = s->stat_overflow_gather;
    d["redo"] = s->stat_redo; d["dense_fallback"] = s->stat_dense_fallback; d["pack_thr"] = s->pack_thr;
    d["cum_overflow_send"] = s->cum_overflow_send; d["cum_overflow_gather"] = s->cum_overflow_gather;
    d["cum_redo"] = s->cum_redo;
    d["fault"] = s->fault;
    // phase durations of the last fused call in microseconds: pack, reduce-scatter, global select, allgather+finalise
    auto us = [&](int a, int b) { return s->t_phase[b] >= s->t_phase[a] ? (double)(s->t_phase[b] - s->t_phase[a]) * 1e-3 : 0.0; };
    py::dict ph;
    ph["local"] = us(5, 0); ph["pack"] = us(0, 1); ph["wait_rs"] = us(1, 6); ph["reduce"] = us(6, 2); ph["gselect"] = us(2, 3);
    ph["wait_ag"] = us(3, 7); ph["final"] = us(7, 4); ph["total"] = us(5, 4);
    d["phase_us"] = ph;
    return d;
}

// The per-call history ring (one TraceRec per fused call, newest kTraceLen calls): --trace / settings.PROFILING.
static py::list read_trace(uint64_t st, uint64_t stream) {
    std::vector<TraceRec> host(kTraceLen);
    ck(cudaMemcpyAsync(host.data(), reinterpret_cast<char*>(P_<OktState>(st)) + offsetof(OktState, trace),
                       sizeof(TraceRec) * kTraceLen, cudaMemcpyDeviceToHost, S_(stream)), "read_trace");
    ck(cudaStreamSynchronize(S_(stream)), "read_trace sync");
    py::list out;
    for (const TraceRec& t : host) {
        if (t.epoch == 0) continue;
        py::dict d;
        d["epoch"] = t.epoch; d["local_count"] = t.local_count; d["global_count"] = t.global_count;
        d["recv_total"] = t.recv_total; d["gather_total"] = t.gather_total; d["overflow_send"] = t.overflow_send;
        d["overflow_gather"] = t.overflow_gather; d["redo"] = t.redo; d["local_thr"] = t.local_thr;
        d["global_thr"] = t.global_thr; d["us_local"] = t.us_local; d["us_pack"] = t.us_pack;
        d["us_wait_rs"] = t.us_wait_rs; d["us_reduce"] = t.us_reduce; d["us_gselect"] = t.us_gselect;
        d["us_wait_ag"] = t.us_wait_ag; d["us_final"] = t.us_final; d["t_begin"] = t.t_begin;
        out.append(d);
    }
    return out;
}

// A host-mapped pinned int: kernels mirror their fault code into it, the host polls it at every step for free.
static py::tuple host_flag_alloc() {
    int* h = nullptr;
    ck(cudaHostAlloc(reinterpret_cast<void**>(&h), sizeof(int) * 16, cudaHostAllocMapped), "cudaHostAlloc(flag)");
    for (int i = 0; i < 16; ++i) h[i] = 0;
    void* d = nullptr;
    ck(cudaHostGetDevicePointer(&d, h, 0), "cudaHostGetDevicePointer");
    return py::make_tuple((uint64_t)h, (uint64_t)d);
}
static void host_flag_free(uint64_t h) { if (h) cudaFreeHost(P_<void>(h)); }
static int host_flag_read(uint64_t h) { return h ? *reinterpret_cast<volatile int*>(h) : 0; }
static void host_flag_clear(uint64_t h) { if (h) *reinterpret_cast<volatile int*>(h) = 0; }

static void write_state(uint64_t st, float local_thr, float global_thr, const std::vector<int>& edges, uint64_t stream) {
    std::vector<char> host(offsetof(OktState, hist));
    ck(cudaMemcpyAsync(host.data(), P_<void>(st), host.size(), cudaMemcpyDeviceToHost, S_(stream)), "write_state rd");
    ck(cudaStreamSynchronize(S_(stream)), "write_state sync");
    OktState* s = reinterpret_cast<OktState*>(host.data());
    s->local_thr = local_thr;
    s->global_thr = global_thr;
    if (!edges.empty()) {
        if (edges.size() > OKT_MAXP + 1) throw std::runtime_error("too many region edges");
        for (size_t i = 0; i < edges.size(); ++i) s->edges[i] = edges[i];
    }
    // only the plain-data head is written back (bar / epoch / cursors are kernel-owned and unchanged here)
    ck(cudaMemcpyAsync(P_<void>(st), host.data(), host.size(), cudaMemcpyHostToDevice, S_(stream)), "write_state wr");
    ck(cudaStreamSynchronize(S_(stream)), "write_state sync2");
}

// ------------------------------------------------------------------------------------------- launchers
static void fill_peers(char** dst, const std::vector<uint64_t>& peers) {
    if (peers.size() > OKT_MAXP) throw std::runtime_error("world larger than OKT_MAXP");
    for (int i = 0; i < OKT_MAXP; ++i) dst[i] = nullptr;
    for (size_t i = 0; i < peers.size(); ++i) dst[i] = P_<char>(peers[i]);
}

static void oktopk_run(uint64_t g, uint64_t res, uint64_t st, const std::vector<uint64_t>& peers, int n, int rank,
                       int k, int cap, int gcap, py::dict o, int grid, uint64_t stream) {
    OktParams p;
    std::memset(&p, 0, sizeof(p));
    p.g = P_<float>(g); p.res = P_<float>(res); p.st = P_<OktState>(st);
    if (!o.contains("cand") || !o.contains("ccap")) throw std::runtime_error("oktopk_run: candidate scratch missing");
    p.cand = P_<int>(o["cand"].cast<uint64_t>()); p.ccap = o["ccap"].cast<int>();
    p.cand_mode = o.contains("cand_mode") ? o["cand_mode"].cast<int>() : 1;
    fill_peers(p.peers, peers);
    p.P = (int)peers.size(); p.rank = rank; p.n = n; p.k = k;
    p.L = make_layout(p.P, n, cap, gcap);
    auto geti = [&](const char* key, int dflt) { return o.contains(key) ? o[key].cast<int>() : dflt; };
    auto getf = [&](const char* key, double dflt) { return o.contains(key) ? o[key].cast<double>() : dflt; };
    for (int i = 0; i < OKT_MAXP; ++i) p.peer_g[i] = nullptr;
    if (o.contains("peer_g")) {
        auto pg = o["peer_g"].cast<std::vector<uint64_t>>();
        for (size_t i = 0; i < pg.size() && i < OKT_MAXP; ++i) p.peer_g[i] = P_<float>(pg[i]);
    }
    p.max_redo = geti("max_redo", 12);
    p.redo_factor = (float)getf("redo_factor", 1.5);
    p.dense_nnz_limit = geti("dense_nnz_limit", 0);
    p.host_fault = o.contains("host_fault") ? P_<int>(o["host_fault"].cast<uint64_t>()) : nullptr;
    p.skip = o.contains("skip") ? P_<const int>(o["skip"].cast<uint64_t>()) : nullptr;
    p.trace = geti("trace", 0);
    p.exact_local = geti("exact_local", 0);
    p.repartition = geti("repartition", 0);
    p.uniform_regions = geti("uniform_regions", 0);
    p.residual_mode = geti("residual_mode", RES_OKTOPK);
    p.global_mode = geti("global_mode", GLB_THRESHOLD);
    p.deterministic = geti("deterministic", 0);
    p.pull_tma = geti("pull_tma", 1);
    p.phase_begin = geti("phase_begin", 0);
    p.phase_end = geti("phase_end", PH_END);
    p.guard_loops = geti("guard_loops", 0);
    if (p.guard_loops > kGuardFineMax) p.guard_loops = kGuardFineMax;
    p.cap_limit = geti("cap_limit", 0);
    p.cap_rungs = geti("cap_rungs", 40);
    p.cap_factor = (float)getf("cap_factor", 1.19);
    p.guard_limit = geti("guard_limit", 0);
    p.guard_factor = (float)getf("guard_factor", 1.03);
    p.l_low_cnt = getf("l_low_cnt", 0.0); p.l_high_cnt = getf("l_high_cnt", 1e30);
    p.l_factor = (float)getf("l_factor", 1.012);
    p.g_low_cnt = getf("g_low_cnt", 0.0); p.g_high_cnt = getf("g_high_cnt", 1e30);
    p.g_inc = (float)getf("g_inc", 1.008); p.g_dec = (float)getf("g_dec", 1.008);
    p.prefilter = (float)getf("prefilter", 0.8);
    p.timeout_ns = (unsigned long long)(getf("timeout_s", 0.0) * 1e9);
    if (o.contains("srcs")) {
        // the gradient is read from these (pointer, bucket offset, length) segments; the bucket is all-zero on entry
        auto t = o["srcs"].cast<std::tuple<std::vector<uint64_t>, std::vector<long long>, std::vector<long long>>>();
        const auto& ptr = std::get<0>(t);
        const auto& off = std::get<1>(t);
        const auto& len = std::get<2>(t);
        if (off.size() != ptr.size() || len.size() != ptr.size()) throw std::runtime_error("oktopk_run: srcs table size mismatch");
        if (ptr.size() > (size_t)kSrcSegMax) throw std::runtime_error("oktopk_run: more gradient sources than kSrcSegMax");
        long long end = 0;
        for (size_t i = 0; i < ptr.size(); ++i) {
            if (off[i] < end || (off[i] & 3) || len[i] <= 0 || off[i] + len[i] > n || (ptr[i] & 15))
                throw std::runtime_error("oktopk_run: gradient sources must be 16-byte aligned, in bucket order, "
                                         "non-overlapping, at offsets that are multiples of 4 elements");
            p.src[i] = P_<const float>(ptr[i]);
            p.src_off[i] = (int)off[i];
            p.src_len[i] = (int)len[i];
            end = off[i] + len[i];
        }
        p.nsrc = (int)ptr.size();
        p.zero_g = 0;
    } else {
        // the gradient was landed in the bucket: one segment, cleared by the pack pass for the reduce / final phases
        if (g & 15) throw std::runtime_error("oktopk_run: the bucket must be 16-byte aligned");
        p.src[0] = P_<const float>(g);
        p.src_off[0] = 0;
        p.src_len[0] = n;
        p.nsrc = 1;
        p.zero_g = 1;
    }
    if (o.contains("pack_ranges")) {
        // early pack: element ranges [lo, hi) at multiples of 4 inside the bucket's whole float4 vectors.  A segment launch
        // (segment=1) packs its ranges; the call packs only its ranges, the rest having been packed by segments.
        auto rs = o["pack_ranges"].cast<std::vector<std::pair<long long, long long>>>();
        if (rs.size() > (size_t)kPackRangeMax) throw std::runtime_error("oktopk_run: more pack ranges than kPackRangeMax");
        long long end = 0;
        for (size_t i = 0; i < rs.size(); ++i) {
            const long long lo = rs[i].first, hi = rs[i].second;
            if (lo < end || hi < lo || (lo & 3) || (hi & 3) || hi > ((long long)n & ~3LL))
                throw std::runtime_error("oktopk_run: pack ranges must be ordered, disjoint, at multiples of 4 elements, "
                                         "inside the bucket's whole vectors");
            p.pk_lo[i] = (int)(lo >> 2);
            p.pk_hi[i] = (int)(hi >> 2);
            end = hi;
        }
        p.pk_mode = 1;
        p.pk_nr = (int)rs.size();
        if (geti("segment", 0)) {
            if (rs.empty() || p.zero_g || p.L.cap > 0 || p.residual_mode != RES_OKTOPK)
                throw std::runtime_error("oktopk_run: a segment launch takes ranges of an Ok-Topk bucket read from its "
                                         "sources in the lossless layout");
            ck(launch_oktopk_segment(p, geti("seg_ctas", 32), S_(stream)), "oktopk segment launch");
            return;
        }
    }
    if (geti("split_phases", 0)) {
        // ablation / debugging: one launch per phase instead of the single persistent kernel
        for (int ph = p.phase_begin; ph < p.phase_end; ++ph) {
            OktParams q = p;
            q.phase_begin = ph; q.phase_end = ph + 1;
            ck(launch_oktopk(q, grid, S_(stream)), "oktopk phase launch");
        }
    } else {
        ck(launch_oktopk(p, grid, S_(stream)), "oktopk fused launch");
    }
}

static void gather_run(uint64_t g, uint64_t res, uint64_t st, const std::vector<uint64_t>& peers, int n, int rank,
                       int k, int cap, int gcap, py::dict o, int grid, uint64_t stream) {
    GatherParams p;
    std::memset(&p, 0, sizeof(p));
    p.g = P_<float>(g); p.res = P_<float>(res); p.st = P_<OktState>(st);
    fill_peers(p.peers, peers);
    p.P = (int)peers.size(); p.rank = rank; p.n = n; p.k = k;
    p.L = make_layout(p.P, n, cap, gcap);
    p.reselect = o.contains("reselect") ? o["reselect"].cast<int>() : 0;
    p.clip_max_norm = o.contains("clip_max_norm") ? (float)o["clip_max_norm"].cast<double>() : 0.f;
    p.bitmap = o.contains("bitmap") ? P_<unsigned>(o["bitmap"].cast<uint64_t>()) : nullptr;
    p.cand = o.contains("cand") ? P_<int>(o["cand"].cast<uint64_t>()) : nullptr;
    p.ccap = o.contains("ccap") ? o["ccap"].cast<int>() : 0;
    p.host_fault = o.contains("host_fault") ? P_<int>(o["host_fault"].cast<uint64_t>()) : nullptr;
    p.skip = o.contains("skip") ? P_<const int>(o["skip"].cast<uint64_t>()) : nullptr;
    if (p.reselect && (p.bitmap == nullptr || p.cand == nullptr || p.ccap <= 0))
        throw std::runtime_error("gather_run: TopkA2 needs the bitmap and candidate scratch");
    p.select_mode = o["select_mode"].cast<int>();
    p.exact_now = o.contains("exact_now") ? o["exact_now"].cast<int>() : 0;
    p.gauss_mode = o.contains("gauss_mode") ? o["gauss_mode"].cast<int>() : 0;
    p.gauss_loops = o.contains("gauss_loops") ? o["gauss_loops"].cast<int>() : 20;
    p.gauss_factor = o.contains("gauss_factor") ? (float)o["gauss_factor"].cast<double>() : 1.02f;
    p.density = (float)o["density"].cast<double>();
    p.pull_tma = o.contains("pull_tma") ? o["pull_tma"].cast<int>() : 1;
    p.timeout_ns = o.contains("timeout_s") ? (unsigned long long)(o["timeout_s"].cast<double>() * 1e9) : 0ULL;
    ck(launch_gather_scheme(p, grid, S_(stream)), "gather scheme launch");
}

static void gtopk_run(uint64_t g, uint64_t res, uint64_t st, const std::vector<uint64_t>& peers, int n, int rank,
                      int k, int cap, int gcap, py::dict o, int grid, uint64_t stream) {
    TreeParams p;
    std::memset(&p, 0, sizeof(p));
    p.g = P_<float>(g); p.res = P_<float>(res); p.st = P_<OktState>(st);
    fill_peers(p.peers, peers);
    p.P = (int)peers.size(); p.rank = rank; p.n = n; p.k = k;
    if (p.P & (p.P - 1)) throw std::runtime_error("gTopk needs a power-of-two world size (VGG/allreducer.py:113)");
    p.L = make_layout(p.P, n, cap, gcap);
    p.pull_tma = o.contains("pull_tma") ? o["pull_tma"].cast<int>() : 1;
    p.timeout_ns = o.contains("timeout_s") ? (unsigned long long)(o["timeout_s"].cast<double>() * 1e9) : 0ULL;
    p.clip_max_norm = o.contains("clip_max_norm") ? (float)o["clip_max_norm"].cast<double>() : 0.f;
    p.bitmap = P_<unsigned>(o["bitmap"].cast<uint64_t>());
    p.cand = P_<int>(o["cand"].cast<uint64_t>());
    p.ccap = o["ccap"].cast<int>();
    p.sel_idx = P_<int>(o["sel_idx"].cast<uint64_t>());
    p.sel_val = P_<float>(o["sel_val"].cast<uint64_t>());
    p.selcap = o["selcap"].cast<int>();
    p.host_fault = o.contains("host_fault") ? P_<int>(o["host_fault"].cast<uint64_t>()) : nullptr;
    p.skip = o.contains("skip") ? P_<const int>(o["skip"].cast<uint64_t>()) : nullptr;
    ck(launch_gtopk(p, grid, S_(stream)), "gtopk launch");
}

static void land_grads(const std::vector<uint64_t>& srcs, const std::vector<long long>& offs, const std::vector<int>& numels,
                       uint64_t bucket, uint64_t stream) {
    const size_t T = srcs.size();
    if (offs.size() != T || numels.size() != T) throw std::runtime_error("land_grads: table size mismatch");
    constexpr int per = 8192;                           // kLandPerCta
    for (size_t b = 0; b < T; b += kLandMax) {
        LandParams lp;
        std::memset(&lp, 0, sizeof(lp));
        const int cnt = (int)std::min<size_t>(kLandMax, T - b);
        int blk = 0;
        for (int i = 0; i < cnt; ++i) {
            lp.src[i] = P_<const float>(srcs[b + i]);
            lp.dst_off[i] = offs[b + i];
            lp.numel[i] = numels[b + i];
            lp.blk_begin[i] = blk;
            blk += std::max(1, (numels[b + i] + per - 1) / per);
        }
        lp.blk_begin[cnt] = blk;
        lp.count = cnt;
        ck(launch_land(lp, P_<float>(bucket), S_(stream)), "land_grads");
    }
}

static void dense_run(const std::vector<uint64_t>& bufs, const std::vector<uint64_t>& flags, uint64_t epoch, int n,
                      int rank, int grid, uint64_t stream, uint64_t st, double timeout_s, uint64_t mc,
                      uint64_t host_fault, uint64_t skip) {
    DenseParams p;
    std::memset(&p, 0, sizeof(p));
    if (bufs.size() > OKT_MAXP || bufs.size() != flags.size()) throw std::runtime_error("bad peer tables");
    for (size_t i = 0; i < bufs.size(); ++i) { p.bufs[i] = P_<float>(bufs[i]); p.flags[i] = P_<uint64_t>(flags[i]); }
    p.epoch = P_<unsigned long long>(epoch);
    p.n = n; p.P = (int)bufs.size(); p.rank = rank; p.scale = 1.0f / (float)p.P;
    p.fault = st ? &P_<OktState>(st)->fault : nullptr;
    p.timeout_ns = (unsigned long long)(timeout_s * 1e9);
    p.mc = P_<float>(mc);
    p.host_fault = P_<int>(host_fault);
    p.skip = P_<const int>(skip);
    ck(launch_dense_allreduce(p, grid, S_(stream)), "dense allreduce launch");
}

static void kth_abs(uint64_t x, int n, int k, uint64_t st, uint64_t out, int grid, uint64_t stream) {
    ck(launch_kth_abs(P_<float>(x), n, k, P_<OktState>(st), P_<float>(out), grid, S_(stream)), "kth_abs launch");
}

static void fused_sgd(uint64_t p, uint64_t g, uint64_t mom, int n, double momentum, double dampening, double wd,
                      int nesterov, int first, int zero_grad, uint64_t stream, uint64_t scal_ptr, uint64_t fault_ptr,
                      uint64_t skip_ptr, uint64_t coef_ptr) {
    if (scal_ptr == 0) throw std::runtime_error("fused_sgd: scal_ptr must point at the group's device scalars");
    ck(launch_fused_sgd(P_<float>(p), P_<float>(g), P_<float>(mom), n, (float)momentum, (float)dampening, (float)wd,
                        nesterov, first, zero_grad, P_<float>(scal_ptr), P_<int>(fault_ptr), P_<int>(skip_ptr),
                        P_<const float>(coef_ptr), S_(stream)),
       "fused_sgd");
}
// [(lo, hi), ...] element ranges of an n-element (bucket, param group) slice, at multiples of 4 and inside its whole
// float4 vectors -> a table of vector ranges
static SgdRanges sgd_ranges(const std::vector<std::pair<long long, long long>>& rs, int n, const char* what) {
    if ((int)rs.size() > kPackRangeMax)
        throw std::runtime_error(std::string(what) + ": more than " + std::to_string(kPackRangeMax) + " ranges");
    SgdRanges r;
    std::memset(&r, 0, sizeof(r));
    r.nr = (int)rs.size();
    for (int q = 0; q < r.nr; ++q) {
        const long long lo = rs[q].first, hi = rs[q].second;
        if (lo < 0 || hi < lo || lo % 4 || hi % 4 || hi > 4LL * (n / 4))
            throw std::runtime_error(std::string(what) + ": ranges must lie at multiples of 4 inside the slice's whole "
                                     "float4 vectors");
        r.lo[q] = (int)(lo / 4);
        r.hi[q] = (int)(hi / 4);
    }
    return r;
}
static void sgd_ahead(uint64_t p, uint64_t mom, uint64_t sp, uint64_t sm, int n,
                      const std::vector<std::pair<long long, long long>>& ranges, double momentum, double dampening,
                      double wd, int nesterov, int max_ctas, uint64_t stream, uint64_t scal_ptr) {
    if (scal_ptr == 0) throw std::runtime_error("sgd_ahead: scal_ptr must point at the group's device scalars");
    if (momentum != 0.0 && (mom == 0 || sm == 0)) throw std::runtime_error("sgd_ahead: momentum needs mom and sm");
    const SgdHyper h{(float)momentum, (float)dampening, (float)wd, nesterov, 0};
    ck(launch_sgd_ahead(P_<float>(p), P_<float>(mom), P_<float>(sp), P_<float>(sm), sgd_ranges(ranges, n, "sgd_ahead"),
                        h, max_ctas, P_<float>(scal_ptr), S_(stream)),
       "sgd_ahead");
}
static void fused_sgd_tail(uint64_t p, uint64_t g, uint64_t mom, uint64_t sp, uint64_t sm, int n,
                           const std::vector<std::pair<long long, long long>>& ahead,
                           const std::vector<std::pair<long long, long long>>& dense, double momentum, double dampening,
                           double wd, int nesterov, int first, int zero_grad, uint64_t stream, uint64_t scal_ptr,
                           uint64_t fault_ptr, uint64_t skip_ptr, uint64_t coef_ptr) {
    if (scal_ptr == 0) throw std::runtime_error("fused_sgd_tail: scal_ptr must point at the group's device scalars");
    if (momentum != 0.0 && (mom == 0 || sm == 0)) throw std::runtime_error("fused_sgd_tail: momentum needs mom and sm");
    const SgdHyper h{(float)momentum, (float)dampening, (float)wd, nesterov, first};
    ck(launch_fused_sgd_tail(P_<float>(p), P_<float>(g), P_<float>(mom), P_<const float>(sp), P_<const float>(sm), n,
                             sgd_ranges(ahead, n, "fused_sgd_tail"), sgd_ranges(dense, n, "fused_sgd_tail"), h,
                             zero_grad, P_<float>(scal_ptr), P_<int>(fault_ptr), P_<int>(skip_ptr),
                             P_<const float>(coef_ptr), S_(stream)),
       "fused_sgd_tail");
}
static void fused_bert_adam(uint64_t p, uint64_t g, uint64_t m, uint64_t v, int n, double b1, double b2, double eps,
                            double wd, int zero_grad, uint64_t stream, uint64_t scal_ptr, uint64_t fault_ptr,
                            uint64_t skip_ptr, uint64_t coef_ptr, uint64_t ends_ptr) {
    if (scal_ptr == 0) throw std::runtime_error("fused_bert_adam: scal_ptr must point at the group's device scalars");
    if (ends_ptr != 0 && coef_ptr == 0) throw std::runtime_error("fused_bert_adam: segment ends need the factors");
    const ClipRef clip{P_<const float>(coef_ptr), P_<const int>(ends_ptr)};
    ck(launch_fused_bert_adam(P_<float>(p), P_<float>(g), P_<float>(m), P_<float>(v), n, (float)b1, (float)b2,
                              (float)eps, (float)wd, zero_grad, P_<float>(scal_ptr), P_<int>(fault_ptr), P_<int>(skip_ptr),
                              clip, S_(stream)),
       "fused_bert_adam");
}
static void fused_adam(uint64_t p, uint64_t g, uint64_t m, uint64_t v, int n, double beta1, double beta2, double eps,
                       double wd, int decoupled, int zero_grad, uint64_t stream, uint64_t scal_ptr, uint64_t fault_ptr,
                       uint64_t skip_ptr, uint64_t coef_ptr) {
    if (scal_ptr == 0) throw std::runtime_error("fused_adam: scal_ptr must point at the group's device scalars");
    ck(launch_fused_adam(P_<float>(p), P_<float>(g), P_<float>(m), P_<float>(v), n, beta1, beta2, (float)eps, (float)wd,
                         decoupled, zero_grad, P_<float>(scal_ptr), P_<int>(fault_ptr), P_<int>(skip_ptr),
                         P_<const float>(coef_ptr), S_(stream)),
       "fused_adam");
}
// LAMB on one (bucket, param group) slice, three launches (launch_fused_lamb).  off / len / blk / ends: device int32
// tables of the slice's nseg segments (blk: nseg + 1 entries); nblk = blk[nseg] - blk[0], which the host knows from the
// same table.
static void fused_lamb(uint64_t p, uint64_t g, uint64_t m, uint64_t v, int n, double beta1, double beta2, double eps,
                       int nseg, uint64_t off, uint64_t len, uint64_t blk, uint64_t ends, int nblk, uint64_t part_w,
                       uint64_t part_u, uint64_t norm_w, uint64_t norm_u, uint64_t ratio, int zero_grad,
                       uint64_t stream, uint64_t scal_ptr, uint64_t fault_ptr, uint64_t skip_ptr, uint64_t coef_ptr) {
    if (scal_ptr == 0) throw std::runtime_error("fused_lamb: scal_ptr must point at the group's device scalars");
    if (nseg <= 0 || nblk < nseg || n < 0 || !off || !len || !blk || !ends || !part_w || !part_u || !norm_w || !norm_u ||
        !ratio)
        throw std::runtime_error("fused_lamb: bad segment table or buffers");
    if ((p | g | m | v) % 16 || (part_w | part_u) % 8)
        throw std::runtime_error("fused_lamb: p, g, m and v must be 16-byte aligned");
    const LambSegs t{P_<const int>(off), P_<const int>(len), P_<const int>(blk), P_<const int>(ends), nseg};
    ck(launch_fused_lamb(P_<float>(p), P_<float>(g), P_<float>(m), P_<float>(v), n, beta1, beta2, (float)eps, t, nblk,
                         P_<double>(part_w), P_<double>(part_u), P_<float>(norm_w), P_<float>(norm_u), P_<float>(ratio),
                         zero_grad, P_<float>(scal_ptr), P_<int>(fault_ptr), P_<int>(skip_ptr),
                         P_<const float>(coef_ptr), S_(stream)),
       "fused_lamb");
}
// dtype of x, y, dy, dx: 0 = fp32, 1 = bf16, 2 = fp16 (parameters, statistics and dgamma / dbeta are fp32 in every case).
// res (forward and backward) and dres (backward), 0 = absent: y = relu(bn(x) + res) and dres = the residual's gradient,
// [M, C] in x's dtype, with relu = 1 and W = 0.
static Dtype dtype_arg(int dtype, const char* what) {
    if (dtype < 0 || dtype > 2) throw std::runtime_error(std::string(what) + ": dtype must be 0 (fp32), 1 (bf16) or 2 (fp16)");
    return static_cast<Dtype>(dtype);
}
static void bn_forward(uint64_t x, uint64_t y, uint64_t arg, uint64_t partial, uint64_t gamma, uint64_t beta, uint64_t cbias,
                       uint64_t save_mean, uint64_t save_invstd, uint64_t rmean, uint64_t rvar, uint64_t nbt, double momentum,
                       double eps, int relu, int M, int C, int W, int slot, int max_ctas, uint64_t stream, int dtype,
                       uint64_t res) {
    if (C % 4 != 0) throw std::runtime_error("bn_forward: channel count must be a multiple of 4");
    if (slot < 0) throw std::runtime_error("bn_forward: negative slot");
    if (res != 0 && (W != 0 || !relu)) throw std::runtime_error("bn_forward: a residual needs relu = 1 and no pool");
    ck(launch_bn_forward(P_<const void>(x), P_<void>(y), P_<unsigned char>(arg), P_<float>(partial), P_<const float>(gamma),
                         P_<const float>(beta), P_<const float>(cbias), P_<float>(save_mean), P_<float>(save_invstd),
                         P_<float>(rmean), P_<float>(rvar), P_<long long>(nbt), (float)momentum, (float)eps, relu, M, C, W, slot,
                         max_ctas, dtype_arg(dtype, "bn_forward"), S_(stream), P_<const void>(res)), "bn_forward");
}
static void bn_backward(uint64_t x, uint64_t dy, uint64_t arg, uint64_t dx, uint64_t partial, uint64_t gamma, uint64_t beta,
                        uint64_t save_mean, uint64_t save_invstd, uint64_t dgamma, uint64_t dbeta, int relu, int M, int C, int W,
                        int slot, int max_ctas, uint64_t stream, int dtype, uint64_t res, uint64_t dres) {
    if (slot < 0) throw std::runtime_error("bn_backward: negative slot");
    if ((res == 0) != (dres == 0)) throw std::runtime_error("bn_backward: res and dres go together");
    if (res != 0 && (W != 0 || !relu)) throw std::runtime_error("bn_backward: a residual needs relu = 1 and no pool");
    ck(launch_bn_backward(P_<const void>(x), P_<const void>(dy), P_<const unsigned char>(arg), P_<void>(dx), P_<float>(partial),
                          P_<const float>(gamma), P_<const float>(beta), P_<const float>(save_mean), P_<const float>(save_invstd),
                          P_<float>(dgamma), P_<float>(dbeta), relu, M, C, W, slot, max_ctas, dtype_arg(dtype, "bn_backward"),
                          S_(stream), P_<const void>(res), P_<void>(dres)), "bn_backward");
}
// y = LayerNorm(x + dropout(a)) over R rows of H: x, y, gamma, beta, mean, rstd (and in the backward dy, dx, dgamma,
// dbeta) fp32; a and da of type a_dtype (codes as dtype_arg).  seed: one int64 in device memory, read by the kernels;
// p_keep_thr = floor((1-p) 2^32), or 2^32 for no dropout (seed may then be 0).  partial: ln_bwd_grid(R) * 2H floats.
static void ln_check(const char* what, int R, int H, long long p_keep_thr, uint64_t seed, uint64_t mean, uint64_t rstd,
                     std::initializer_list<uint64_t> vec_ptrs) {
    if (R <= 0 || !ln_supported_h(H)) throw std::runtime_error(std::string(what) + ": needs R > 0 and H in 128, 256, ..., 1024");
    if (p_keep_thr < 0 || p_keep_thr > (1LL << 32)) throw std::runtime_error(std::string(what) + ": p_keep_thr out of range");
    if (p_keep_thr < (1LL << 32) && seed == 0) throw std::runtime_error(std::string(what) + ": dropout needs the seed");
    if (mean == 0 || rstd == 0) throw std::runtime_error(std::string(what) + ": mean and rstd are needed");
    for (uint64_t p : vec_ptrs)            // accessed as 128-bit (8-byte for a 16-bit a) vectors
        if (p == 0 || (p & 15)) throw std::runtime_error(std::string(what) + ": tensors must be non-null and 16-byte aligned");
}
static void ln_forward(uint64_t x, uint64_t a, uint64_t y, uint64_t gamma, uint64_t beta, uint64_t mean, uint64_t rstd,
                       uint64_t seed, int R, int H, long long p_keep_thr, double scale, double eps, int a_dtype,
                       uint64_t stream) {
    ln_check("ln_forward", R, H, p_keep_thr, seed, mean, rstd, {x, a, y, gamma, beta});
    ck(launch_ln_forward(P_<const float>(x), P_<const void>(a), P_<float>(y), P_<const float>(gamma), P_<const float>(beta),
                         P_<float>(mean), P_<float>(rstd), P_<const unsigned long long>(seed), R, H, p_keep_thr, (float)scale,
                         (float)eps, dtype_arg(a_dtype, "ln_forward"), S_(stream)), "ln_forward");
}
static void ln_backward(uint64_t x, uint64_t a, uint64_t dy, uint64_t gamma, uint64_t mean, uint64_t rstd, uint64_t seed,
                        uint64_t dx, uint64_t da, uint64_t partial, uint64_t dgamma, uint64_t dbeta, int R, int H,
                        long long p_keep_thr, double scale, int a_dtype, uint64_t stream) {
    ln_check("ln_backward", R, H, p_keep_thr, seed, mean, rstd, {x, a, dy, gamma, dx, da, partial, dgamma, dbeta});
    ck(launch_ln_backward(P_<const float>(x), P_<const void>(a), P_<const float>(dy), P_<const float>(gamma),
                          P_<const float>(mean), P_<const float>(rstd), P_<const unsigned long long>(seed), P_<float>(dx),
                          P_<void>(da), P_<float>(partial), P_<float>(dgamma), P_<float>(dbeta), R, H, p_keep_thr,
                          (float)scale, dtype_arg(a_dtype, "ln_backward"), S_(stream)), "ln_backward");
}
// y = dropout(LayerNorm(word[ids] + pos[r % S] + typ[tt])) over R = B S tokens (csrc/embedding.cu): ids, tt int64 [R];
// tables, gamma, beta, y, dy, de and the table gradients fp32; stats 2R floats ([mean; rstd]); ovf one int64 or 0;
// partial ln_bwd_grid(R) * 2H floats.  p_keep_thr and seed as for ln_forward.
static void emb_check(const char* what, int R, int S, int H, int np, int nv, int nt, long long p_keep_thr, uint64_t seed,
                      std::initializer_list<uint64_t> vec_ptrs, std::initializer_list<uint64_t> ptrs) {
    if (!emb_supported(R, S, H, np) || nv <= 0 || nt <= 0)
        throw std::runtime_error(std::string(what) + ": needs 0 < R = B S <= 4096, S <= the position rows, nonempty "
                                                     "tables and H in 128, 256, ..., 1024");
    if (p_keep_thr < 0 || p_keep_thr > (1LL << 32)) throw std::runtime_error(std::string(what) + ": p_keep_thr out of range");
    if (p_keep_thr < (1LL << 32) && seed == 0) throw std::runtime_error(std::string(what) + ": dropout needs the seed");
    for (uint64_t p : vec_ptrs)
        if (p == 0 || (p & 15)) throw std::runtime_error(std::string(what) + ": tensors must be non-null and 16-byte aligned");
    for (uint64_t p : ptrs)
        if (p == 0 || (p & 7)) throw std::runtime_error(std::string(what) + ": ids and statistics must be non-null and aligned");
}
static void emb_forward(uint64_t ids, uint64_t tt, uint64_t word, uint64_t pos, uint64_t typ, uint64_t gamma, uint64_t beta,
                        uint64_t y, uint64_t stats, uint64_t ovf, uint64_t seed, int R, int S, int H, int nv, int np, int nt,
                        long long p_keep_thr, double scale, double eps, uint64_t stream) {
    emb_check("emb_forward", R, S, H, np, nv, nt, p_keep_thr, seed, {word, pos, typ, gamma, beta, y}, {ids, tt, stats});
    if (ovf & 7) throw std::runtime_error("emb_forward: misaligned counter");
    ck(launch_emb_forward(P_<const long long>(ids), P_<const long long>(tt), P_<const float>(word), P_<const float>(pos),
                          P_<const float>(typ), P_<const float>(gamma), P_<const float>(beta), P_<float>(y),
                          P_<float>(stats), P_<long long>(ovf), P_<const unsigned long long>(seed), R, S, H, nv, nt,
                          p_keep_thr, (float)scale, (float)eps, S_(stream)), "emb_forward");
}
static void emb_backward(uint64_t ids, uint64_t tt, uint64_t word, uint64_t pos, uint64_t typ, uint64_t gamma,
                         uint64_t stats, uint64_t dy, uint64_t seed, uint64_t de, uint64_t partial,
                         uint64_t dgamma, uint64_t dbeta, uint64_t dword, uint64_t dpos, uint64_t dtyp, int R, int S, int H,
                         int nv, int np, int nt, long long p_keep_thr, double scale, uint64_t stream) {
    emb_check("emb_backward", R, S, H, np, nv, nt, p_keep_thr, seed,
              {word, pos, typ, gamma, dy, de, partial, dgamma, dbeta, dword, dpos, dtyp}, {ids, tt, stats});
    ck(launch_emb_backward(P_<const long long>(ids), P_<const long long>(tt), P_<const float>(word), P_<const float>(pos),
                           P_<const float>(typ), P_<const float>(gamma), P_<const float>(stats), P_<const float>(dy),
                           P_<const unsigned long long>(seed), P_<float>(de), P_<float>(partial),
                           P_<float>(dgamma), P_<float>(dbeta), P_<float>(dword), P_<float>(dpos), P_<float>(dtyp), R, S, H,
                           nv, np, nt, p_keep_thr, (float)scale, S_(stream)), "emb_backward");
}
// Fused self-attention, head dim 64 (csrc/attention.cu): qkv / dqkv [B, S, 3 H 64] and out / dout [B, S, H 64] of type
// dtype (codes as dtype_arg), 16-byte aligned; mask [B, S] fp32 or 0; lse [B, H, S, 2] and delta [B, H, S] fp32, 8-byte
// aligned.  p_keep_thr and seed as for ln_forward; scale = 1 / (1 - p).
static void attn_check(const char* what, int B, int S, int H, long long p_keep_thr, uint64_t seed,
                       std::initializer_list<uint64_t> vec_ptrs, std::initializer_list<uint64_t> f32_ptrs) {
    if (!attn_supported(B, S, H)) throw std::runtime_error(std::string(what) + ": needs B, H >= 1 and 1 <= S <= 512");
    if (p_keep_thr < 0 || p_keep_thr > (1LL << 32)) throw std::runtime_error(std::string(what) + ": p_keep_thr out of range");
    if (p_keep_thr < (1LL << 32) && seed == 0) throw std::runtime_error(std::string(what) + ": dropout needs the seed");
    for (uint64_t p : vec_ptrs)
        if (p == 0 || (p & 15)) throw std::runtime_error(std::string(what) + ": tensors must be non-null and 16-byte aligned");
    for (uint64_t p : f32_ptrs)
        if (p == 0 || (p & 7)) throw std::runtime_error(std::string(what) + ": lse / delta must be non-null, 8-byte aligned");
}
static void attn_forward(uint64_t qkv, uint64_t mask, uint64_t seed, uint64_t out, uint64_t lse, int B, int S, int H,
                         long long p_keep_thr, double scale, int dtype, uint64_t stream) {
    attn_check("attn_forward", B, S, H, p_keep_thr, seed, {qkv, out}, {lse});
    if (mask & 3) throw std::runtime_error("attn_forward: the mask must be fp32");
    ck(launch_attn_forward(P_<const void>(qkv), P_<const float>(mask), P_<const unsigned long long>(seed), P_<void>(out),
                           P_<float>(lse), B, S, H, p_keep_thr, (float)scale, dtype_arg(dtype, "attn_forward"), S_(stream)),
       "attn_forward");
}
static void attn_backward(uint64_t qkv, uint64_t out, uint64_t dout, uint64_t mask, uint64_t seed, uint64_t lse,
                          uint64_t delta, uint64_t dqkv, int B, int S, int H, long long p_keep_thr, double scale, int dtype,
                          uint64_t stream) {
    attn_check("attn_backward", B, S, H, p_keep_thr, seed, {qkv, out, dout, dqkv}, {lse, delta});
    if (mask & 3) throw std::runtime_error("attn_backward: the mask must be fp32");
    ck(launch_attn_backward(P_<const void>(qkv), P_<const void>(out), P_<const void>(dout), P_<const float>(mask),
                            P_<const unsigned long long>(seed), P_<const float>(lse), P_<float>(delta), P_<void>(dqkv), B, S,
                            H, p_keep_thr, (float)scale, dtype_arg(dtype, "attn_backward"), S_(stream)),
       "attn_backward");
}
// Softmax cross-entropy over R rows of V logits (x, dx of type dtype, codes as dtype_arg), targets t int64, mean over the
// rows whose target is not ignore_index.  lse: R + 1 floats (the rows' log-sum-exp, then n); rowloss: R floats; loss and
// g: one float each, in device memory.
static void xent_check(const char* what, int R, long long V, std::initializer_list<uint64_t> ptrs, uint64_t x, uint64_t t) {
    if (R <= 0 || V <= 0) throw std::runtime_error(std::string(what) + ": needs R > 0 and V > 0");
    for (uint64_t p : ptrs)
        if (p == 0) throw std::runtime_error(std::string(what) + ": null pointer");
    if ((x & 15) || (t & 7)) throw std::runtime_error(std::string(what) + ": logits must be 16-byte aligned, targets 8-byte");
}
static void xent_forward(uint64_t x, uint64_t t, uint64_t lse, uint64_t rowloss, uint64_t loss, int R, long long V,
                         long long ignore_index, int dtype, uint64_t stream) {
    xent_check("xent_forward", R, V, {x, t, lse, rowloss, loss}, x, t);
    ck(launch_xent_forward(P_<const void>(x), P_<const long long>(t), P_<float>(lse), P_<float>(rowloss), P_<float>(loss),
                           R, V, ignore_index, dtype_arg(dtype, "xent_forward"), S_(stream)), "xent_forward");
}
static void xent_backward(uint64_t x, uint64_t t, uint64_t lse, uint64_t g, uint64_t dx, int R, long long V,
                          long long ignore_index, int dtype, uint64_t stream) {
    xent_check("xent_backward", R, V, {x, t, lse, g, dx}, x, t);
    if (dx & 15) throw std::runtime_error("xent_backward: the gradient must be 16-byte aligned");
    ck(launch_xent_backward(P_<const void>(x), P_<const long long>(t), P_<const float>(lse), P_<const float>(g), P_<void>(dx),
                            R, V, ignore_index, dtype_arg(dtype, "xent_backward"), S_(stream)), "xent_backward");
}
// Softmax + CTC loss (csrc/ctc.cu) over x [T, N, C] (dtype codes as dtype_arg); targets [nt] int64 (targets64 = 1) or
// int32, 0 when nt = 0; tn / ln [N] int32; ws ctc_workspace_floats(T, N, nt) floats, ab ctc_ab_floats(T, N, nt); loss
// and g one float each.
static void ctc_check(const char* what, int T, int N, int C, long long nt, uint64_t x, uint64_t t, int t64, int dtype,
                      std::initializer_list<uint64_t> ptrs) {
    if (!ctc_supported(T, N, C, nt))
        throw std::runtime_error(std::string(what) + ": needs T, N > 0, 0 < C <= 128 and at most 2047 targets");
    for (uint64_t p : ptrs)
        if (p == 0) throw std::runtime_error(std::string(what) + ": null pointer");
    if (nt > 0 && t == 0) throw std::runtime_error(std::string(what) + ": null targets");
    if (t & (t64 ? 7 : 3)) throw std::runtime_error(std::string(what) + ": misaligned targets");
    if (x & (dtype == 0 ? 3 : 1)) throw std::runtime_error(std::string(what) + ": misaligned logits");
}
static void ctc_forward(uint64_t x, uint64_t t, int t64, uint64_t tn, uint64_t ln, uint64_t ws, uint64_t loss, int T, int N,
                        int C, long long nt, int dtype, uint64_t stream) {
    ctc_check("ctc_forward", T, N, C, nt, x, t, t64, dtype, {x, tn, ln, ws, loss});
    ck(launch_ctc_forward(P_<const void>(x), P_<const void>(t), t64, P_<const int>(tn), P_<const int>(ln), P_<float>(ws),
                          P_<float>(loss), T, N, C, nt, dtype_arg(dtype, "ctc_forward"), S_(stream)), "ctc_forward");
}
static void ctc_backward(uint64_t x, uint64_t t, int t64, uint64_t tn, uint64_t ln, uint64_t ws, uint64_t ab, uint64_t g,
                         uint64_t dx, int T, int N, int C, long long nt, int dtype, uint64_t stream) {
    ctc_check("ctc_backward", T, N, C, nt, x, t, t64, dtype, {x, tn, ln, ws, ab, g, dx});
    if (dx & (dtype == 0 ? 3 : 1)) throw std::runtime_error("ctc_backward: misaligned gradient");
    ck(launch_ctc_backward(P_<const void>(x), P_<const void>(t), t64, P_<const int>(tn), P_<const int>(ln),
                           P_<const float>(ws), P_<float>(ab), P_<const float>(g), P_<void>(dx), T, N, C, nt, dtype_arg(dtype, "ctc_backward"), S_(stream)),
       "ctc_backward");
}
// Batch-norm over the frames of the longest utterance (csrc/frame_bn.cu): conv = 1, x [N, C, F, Tb] with the conv
// blocks' masked Hardtanh; conv = 0, x [Tb, N, C].  x / y / dy / dx of type dtype (codes as dtype_arg); len [N] int32;
// gamma ... dbeta [C] fp32; nbt one int64 or 0.
static void frame_bn_check(const char* what, int conv, int N, int C, int F, int Tb, int dtype,
                           std::initializer_list<uint64_t> elems, std::initializer_list<uint64_t> ptrs) {
    if (!frame_bn_supported(conv, N, C, F, Tb))
        throw std::runtime_error(std::string(what) + ": needs N, C, F, Tb > 0 and fewer than 2^24 elements per channel");
    for (uint64_t p : ptrs)
        if (p == 0 || (p & 3)) throw std::runtime_error(std::string(what) + ": null or misaligned pointer");
    for (uint64_t p : elems)
        if (p == 0 || (p & (dtype == 0 ? 3 : 1))) throw std::runtime_error(std::string(what) + ": null or misaligned tensor");
}
static void frame_bn_forward(int conv, uint64_t x, uint64_t len, uint64_t gamma, uint64_t beta, uint64_t y, uint64_t mean,
                             uint64_t rstd, uint64_t rmean, uint64_t rvar, uint64_t nbt, int N, int C, int F, int Tb,
                             double eps, double momentum, int dtype, uint64_t stream) {
    frame_bn_check("frame_bn_forward", conv, N, C, F, Tb, dtype, {x, y}, {len, gamma, beta, mean, rstd, rmean, rvar});
    if (nbt & 7) throw std::runtime_error("frame_bn_forward: misaligned num_batches_tracked");
    ck(launch_frame_bn_forward(conv, P_<const void>(x), P_<const int>(len), P_<const float>(gamma), P_<const float>(beta),
                               P_<void>(y), P_<float>(mean), P_<float>(rstd), P_<float>(rmean), P_<float>(rvar),
                               P_<long long>(nbt), N, C, F, Tb, (float)eps, (float)momentum,
                               dtype_arg(dtype, "frame_bn_forward"), S_(stream)), "frame_bn_forward");
}
static void frame_bn_backward(int conv, uint64_t x, uint64_t dy, uint64_t len, uint64_t gamma, uint64_t beta, uint64_t mean,
                              uint64_t rstd, uint64_t dx, uint64_t dgamma, uint64_t dbeta, int N, int C, int F, int Tb,
                              int dtype, uint64_t stream) {
    frame_bn_check("frame_bn_backward", conv, N, C, F, Tb, dtype, {x, dy, dx}, {len, gamma, beta, mean, rstd, dgamma, dbeta});
    ck(launch_frame_bn_backward(conv, P_<const void>(x), P_<const void>(dy), P_<const int>(len), P_<const float>(gamma),
                                P_<const float>(beta), P_<const float>(mean), P_<const float>(rstd), P_<void>(dx),
                                P_<float>(dgamma), P_<float>(dbeta), N, C, F, Tb, dtype_arg(dtype, "frame_bn_backward"),
                                S_(stream)), "frame_bn_backward");
}
// Look-ahead convolution + Hardtanh (csrc/lookahead.cu): x / y / dy / dx [Tb, N, H] of type dtype (codes as
// dtype_arg); w / dw [H, K] fp32; len [N] int32.
static void lookahead_check(const char* what, int N, int H, int Tb, int K, int dtype,
                            std::initializer_list<uint64_t> elems, std::initializer_list<uint64_t> ptrs) {
    if (!lookahead_supported(N, H, Tb, K))
        throw std::runtime_error(std::string(what) + ": needs N, H, Tb > 0 and 1 <= K <= " +
                                 std::to_string(lookahead_max_taps()) + " taps");
    for (uint64_t p : ptrs)
        if (p == 0 || (p & 3)) throw std::runtime_error(std::string(what) + ": null or misaligned pointer");
    for (uint64_t p : elems)
        if (p == 0 || (p & (dtype == 0 ? 3 : 1))) throw std::runtime_error(std::string(what) + ": null or misaligned tensor");
}
static void lookahead_forward(uint64_t x, uint64_t w, uint64_t len, uint64_t y, int N, int H, int Tb, int K, int dtype,
                              uint64_t stream) {
    lookahead_check("lookahead_forward", N, H, Tb, K, dtype, {x, y}, {w, len});
    ck(launch_lookahead_forward(P_<const void>(x), P_<const float>(w), P_<const int>(len), P_<void>(y), N, H, Tb, K,
                                dtype_arg(dtype, "lookahead_forward"), S_(stream)), "lookahead_forward");
}
static void lookahead_backward(uint64_t x, uint64_t y, uint64_t dy, uint64_t w, uint64_t len, uint64_t dx, uint64_t dw,
                               int N, int H, int Tb, int K, int dtype, uint64_t stream) {
    lookahead_check("lookahead_backward", N, H, Tb, K, dtype, {x, y, dy, dx}, {w, len, dw});
    ck(launch_lookahead_backward(P_<const void>(x), P_<const void>(y), P_<const void>(dy), P_<const float>(w),
                                 P_<const int>(len), P_<void>(dx), P_<float>(dw), N, H, Tb, K,
                                 dtype_arg(dtype, "lookahead_backward"), S_(stream)), "lookahead_backward");
}
// Fixed-capacity gather of the labelled masked-LM rows (csrc/mlm_gather.cu): labels [R] int64, rows [M] int32, tgt [M]
// int64, slot [R] int32, count one int64, overflow one int64 or 0; x / dx [R, H] and out / dout [M, H] of type dtype.
static void mlm_select(uint64_t labels, uint64_t rows, uint64_t tgt, uint64_t slot, uint64_t count, uint64_t overflow,
                       int R, int M, long long ignore_index, uint64_t stream) {
    if (R <= 0 || M <= 0) throw std::runtime_error("mlm_select: needs R > 0 and M > 0");
    if (!labels || !rows || !tgt || !slot || !count) throw std::runtime_error("mlm_select: null pointer");
    if ((labels & 7) || (tgt & 7) || (count & 7) || (overflow & 7) || (rows & 3) || (slot & 3))
        throw std::runtime_error("mlm_select: misaligned pointer");
    ck(launch_mlm_select(P_<const long long>(labels), R, ignore_index, M, P_<int>(rows), P_<long long>(tgt),
                         P_<int>(slot), P_<long long>(count), P_<long long>(overflow), S_(stream)), "mlm_select");
}
static void mlm_copy_check(const char* what, int nrows, int H, uint64_t src, uint64_t idx, uint64_t dst, Dtype dt) {
    if (nrows <= 0 || H <= 0) throw std::runtime_error(std::string(what) + ": needs rows > 0 and H > 0");
    if (!src || !idx || !dst) throw std::runtime_error(std::string(what) + ": null pointer");
    const uint64_t mask = dt == Dtype::kF32 ? 3 : 1;
    if ((src & mask) || (dst & mask) || (idx & 3)) throw std::runtime_error(std::string(what) + ": misaligned pointer");
}
static void mlm_gather(uint64_t x, uint64_t rows, uint64_t out, int M, int H, int dtype, uint64_t stream) {
    const Dtype dt = dtype_arg(dtype, "mlm_gather");
    mlm_copy_check("mlm_gather", M, H, x, rows, out, dt);
    ck(launch_mlm_gather(P_<const void>(x), P_<const int>(rows), P_<void>(out), M, H, dt, S_(stream)), "mlm_gather");
}
static void mlm_scatter(uint64_t dout, uint64_t slot, uint64_t dx, int R, int H, int dtype, uint64_t stream) {
    const Dtype dt = dtype_arg(dtype, "mlm_scatter");
    mlm_copy_check("mlm_scatter", R, H, dout, slot, dx, dt);
    ck(launch_mlm_scatter(P_<const void>(dout), P_<const int>(slot), P_<void>(dx), R, H, dt, S_(stream)), "mlm_scatter");
}
// Persistent LSTM recurrence (csrc/lstm.cu), time-major: gx [T, N, 4H], whh [4H, H], len [N] int32 in [1, T],
// y / cs [T, N, H], gates / dy / dg as named; bar: one zeroed int64.  u hidden units per CTA, `rows` batch rows staged at
// a time (ops/fused_lstm.lstm_geometry).  gx, whh, y, dy and dg are of type dtype (codes as dtype_arg), gates and cs fp32.
// whh_rev != 0 (the reverse direction's W_hh) runs both directions of a bidirectional layer in the one launch: gx, y,
// cs, gates and dg are then [2, T, N, .], forward direction first, dy is the same [T, N, H] for both, and bar is two
// zeroed int64, one per direction.
static void lstm_check(const char* what, int T, int N, int H, int u, int rows, Dtype dtype,
                       std::initializer_list<uint64_t> ptrs, std::initializer_list<uint64_t> vec_ptrs, uint64_t bar) {
    if (T <= 0 || N <= 0 || H <= 0 || H % 4 || u <= 0 || rows <= 0 || rows > N)
        throw std::runtime_error(std::string(what) + ": needs T, N > 0, H > 0 a multiple of 4, u > 0 and 0 < rows <= N");
    for (uint64_t p : ptrs)
        if (p == 0) throw std::runtime_error(std::string(what) + ": null pointer");
    const uint64_t mask = dtype == Dtype::kF32 ? 15 : 7;            // read four elements at a time
    for (uint64_t p : vec_ptrs)
        if (p & mask)
            throw std::runtime_error(std::string(what) + ": W_hh (both directions') and the staged operand must be " +
                                     std::to_string(mask + 1) + "-byte aligned");
    if (bar & 7) throw std::runtime_error(std::string(what) + ": bar must be 8-byte aligned (one int64 per direction)");
}
static void lstm_forward(uint64_t gx, uint64_t whh, uint64_t len, uint64_t y, uint64_t gates, uint64_t cs, uint64_t bar,
                         int T, int N, int H, int u, int rows, uint64_t stream, int dtype, uint64_t whh_rev) {
    const Dtype dt = dtype_arg(dtype, "lstm_forward");
    lstm_check("lstm_forward", T, N, H, u, rows, dt, {gx, whh, len, y, gates, cs, bar}, {whh, whh_rev, y}, bar);
    ck(launch_lstm_forward(P_<const void>(gx), P_<const void>(whh), P_<const void>(whh_rev), P_<const int>(len),
                           P_<void>(y), P_<float>(gates), P_<float>(cs), P_<unsigned long long>(bar), T, N, H, u, rows,
                           S_(stream), dt),
       "lstm_forward");
}
static void lstm_backward(uint64_t dy, uint64_t gates, uint64_t cs, uint64_t whh, uint64_t len, uint64_t dg, uint64_t bar,
                          int T, int N, int H, int u, int rows, uint64_t stream, int dtype, uint64_t whh_rev) {
    const Dtype dt = dtype_arg(dtype, "lstm_backward");
    lstm_check("lstm_backward", T, N, H, u, rows, dt, {dy, gates, cs, whh, len, dg, bar}, {dg}, bar);
    ck(launch_lstm_backward(P_<const void>(dy), P_<const float>(gates), P_<const float>(cs), P_<const void>(whh),
                            P_<const void>(whh_rev), P_<const int>(len), P_<void>(dg), P_<unsigned long long>(bar), T, N,
                            H, u, rows, S_(stream), dt),
       "lstm_backward");
}
// One layer of a stacked LSTM from an initial state (csrc/lstm.cu lstm_seq_*): gx [T, N, 4H], whh [4H, H], y [T, N, H],
// h0 [N, H] of type dtype; c0 [N, H], gates, cs fp32; bar one zeroed int64.  Backward: dy [T, N, H] and dhn [N, H] (or
// 0) of type dtype, dcn [N, H] fp32 (or 0); writes dg [T, N, 4H] (dtype) and dc0 [N, H] (fp32).  fp32 takes the split
// of ops/fused_lstm.lstm_seq_f32_geometry: r_on weight rows on chip, kc-column chunks; its backward whh is W_hh^T
// [H, 4H] and every operand read in vectors (whh, h0, y, dg) is 16-byte aligned.
static void lstm_seq_forward(uint64_t gx, uint64_t whh, uint64_t h0, uint64_t c0, uint64_t y, uint64_t gates,
                             uint64_t cs, uint64_t bar, int T, int N, int H, int u, int rows, uint64_t stream,
                             int dtype, int r_on, int kc) {
    const Dtype dt = dtype_arg(dtype, "lstm_seq_forward");
    lstm_check("lstm_seq_forward", T, N, H, u, rows, dt, {gx, whh, h0, c0, y, gates, cs, bar}, {whh, h0, y}, bar);
    ck(launch_lstm_seq_forward(P_<const void>(gx), P_<const void>(whh), P_<const void>(h0), P_<const float>(c0),
                               P_<void>(y), P_<float>(gates), P_<float>(cs), P_<unsigned long long>(bar), T, N, H, u,
                               rows, r_on, kc, S_(stream), dt),
       "lstm_seq_forward");
}
static void lstm_seq_backward(uint64_t dy, uint64_t gates, uint64_t cs, uint64_t whh, uint64_t c0, uint64_t dhn,
                              uint64_t dcn, uint64_t dg, uint64_t dc0, uint64_t bar, int T, int N, int H, int u, int rows,
                              uint64_t stream, int dtype, int r_on, int kc) {
    const Dtype dt = dtype_arg(dtype, "lstm_seq_backward");
    lstm_check("lstm_seq_backward", T, N, H, u, rows, dt, {dy, gates, cs, whh, c0, dg, dc0, bar},
               dt == Dtype::kF32 ? std::initializer_list<uint64_t>{whh, dg} : std::initializer_list<uint64_t>{dg}, bar);
    ck(launch_lstm_seq_backward(P_<const void>(dy), P_<const float>(gates), P_<const float>(cs), P_<const void>(whh),
                                P_<const float>(c0), P_<const void>(dhn), P_<const float>(dcn), P_<void>(dg),
                                P_<float>(dc0), P_<unsigned long long>(bar), T, N, H, u, rows, r_on, kc, S_(stream), dt),
       "lstm_seq_backward");
}
static void maxpool2_fwd(uint64_t x, uint64_t y, uint64_t arg, int N, int H, int W, int C, uint64_t stream) {
    if ((C % 4) || (H % 2) || (W % 2)) throw std::runtime_error("maxpool2_fwd: needs C % 4 == 0 and even H, W");
    ck(launch_maxpool2_fwd(P_<const float>(x), P_<float>(y), P_<unsigned char>(arg), N, H, W, C, S_(stream)), "maxpool2_fwd");
}
static void maxpool2_bwd(uint64_t dy, uint64_t arg, uint64_t dx, int N, int H, int W, int C, uint64_t stream) {
    ck(launch_maxpool2_bwd(P_<const float>(dy), P_<const unsigned char>(arg), P_<float>(dx), N, H, W, C, S_(stream)), "maxpool2_bwd");
}
static void momentum_correct(uint64_t g, uint64_t buf, int n, double momentum, uint64_t stream) {
    ck(launch_momentum_correct(P_<float>(g), P_<float>(buf), n, (float)momentum, S_(stream)), "momentum_correct");
}
// Sum of squares of the segments (offsets, lengths) of the flat fp32 bucket g into partial[0, P), P = the sum over
// segments of max(1, ceil(len / SUMSQ_CHUNK)), in segment order.  More than kSrcSegMax segments take one launch per
// kSrcSegMax of them, each writing the next partials.
static void grad_sumsq(uint64_t g, const std::vector<long long>& offs, const std::vector<long long>& lens,
                       uint64_t partial, uint64_t stream) {
    const size_t T = offs.size();
    if (lens.size() != T || T == 0) throw std::runtime_error("grad_sumsq: bad segment table");
    if (g % 16 || partial % 8) throw std::runtime_error("grad_sumsq: misaligned bucket or partials");
    double* out = P_<double>(partial);
    for (size_t b = 0; b < T; b += kSrcSegMax) {
        SumsqSegs t;
        std::memset(&t, 0, sizeof(t));
        t.nseg = (int)std::min<size_t>(kSrcSegMax, T - b);
        long long blk = 0;
        for (int i = 0; i < t.nseg; ++i) {
            const long long o = offs[b + i], l = lens[b + i];
            if (o < 0 || o % 4 || l < 0 || o + l > (1LL << 31) - 1)
                throw std::runtime_error("grad_sumsq: segments must lie at multiples of 4 inside an int32 range");
            t.off[i] = (int)o;
            t.len[i] = (int)l;
            t.blk_begin[i] = (int)blk;
            blk += std::max(1LL, (l + kSumsqChunk - 1) / kSumsqChunk);
        }
        t.blk_begin[t.nseg] = (int)blk;
        ck(launch_grad_sumsq(P_<const float>(g), t, out, S_(stream)), "grad_sumsq");
        out += blk;
    }
}
static void clip_coef(uint64_t partial, int np, uint64_t seg_blk, uint64_t seg_scal, int nseg, uint64_t scal,
                      double max_norm, uint64_t norm, uint64_t coef, uint64_t stream) {
    if (seg_blk != 0 && (seg_scal == 0 || scal == 0 || nseg <= 0))
        throw std::runtime_error("clip_coef: per-segment factors need seg_scal, scal and nseg");
    ck(launch_clip_coef(P_<const double>(partial), np, P_<const int>(seg_blk), P_<const int>(seg_scal), nseg,
                        P_<const float>(scal), (float)max_norm, P_<float>(norm), P_<float>(coef), S_(stream)),
       "clip_coef");
}

// ------------------------------------------------------------------------------------------- loss scaling
// srcs = (pointers, lengths): the gradient tensors of the direct Ok-Topk path, or the landed bucket as one segment.
static void unscale_check(const std::vector<uint64_t>& srcs, const std::vector<long long>& lens, uint64_t ls, uint64_t sync,
                          uint64_t st, uint64_t host_fault, const std::vector<uint64_t>& peers, size_t mbox_off, int rank,
                          double timeout_s, uint64_t stream) {
    ScaleParams p;
    std::memset(&p, 0, sizeof(p));
    if (srcs.empty() || srcs.size() != lens.size()) throw std::runtime_error("unscale_check: bad source table");
    if (srcs.size() > (size_t)kSrcSegMax) throw std::runtime_error("unscale_check: more gradient sources than kSrcSegMax");
    if (peers.size() > OKT_MAXP) throw std::runtime_error("world larger than OKT_MAXP");
    int blk = 0;
    for (size_t i = 0; i < srcs.size(); ++i) {
        if ((srcs[i] & 15) || lens[i] <= 0 || lens[i] > (1LL << 31) - 1)
            throw std::runtime_error("unscale_check: sources must be 16-byte aligned and non-empty");
        p.src[i] = P_<float>(srcs[i]);
        p.len[i] = (int)lens[i];
        p.blk_begin[i] = blk;
        blk += (int)((lens[i] + kScalePerCta - 1) / kScalePerCta);
    }
    p.blk_begin[srcs.size()] = blk;
    p.nseg = (int)srcs.size();
    p.ls = P_<LossScaleDev>(ls);
    p.sync = P_<ScaleSync>(sync);
    p.fault = &P_<OktState>(st)->fault;
    p.host_fault = P_<int>(host_fault);
    for (size_t i = 0; i < peers.size(); ++i) p.peers[i] = P_<char>(peers[i]);
    p.mbox_off = mbox_off;
    p.P = (int)peers.size(); p.rank = rank;
    p.timeout_ns = (unsigned long long)(timeout_s * 1e9);
    ck(launch_unscale_check(p, S_(stream)), "unscale_check");
}

PYBIND11_MODULE(_C, m) {
    m.doc() = "oktopk_b200 native extension (sm_90a kernels + symmetric peer memory)";
    m.def("symm_alloc", &symm_alloc);
    m.def("symm_open", &symm_open);
    m.def("symm_close", &symm_close);
    m.def("symm_free", &symm_free);
    m.def("dev_alloc_zero", &dev_alloc_zero);
    m.def("dev_free", &dev_free);
    m.def("memset_async", &memset_async);
    m.def("can_access_peer", &can_access_peer);
    m.def("state_bytes", &state_bytes);
    m.def("layout_info", &layout_info);
    m.def("read_state", &read_state);
    m.def("write_state", &write_state);
    m.def("max_coop_grid", &okt_max_coop_grid);
    m.def("oktopk_run", &oktopk_run);
    m.def("gather_run", &gather_run);
    m.def("dense_run", &dense_run, py::arg("bufs"), py::arg("flags"), py::arg("epoch"), py::arg("n"), py::arg("rank"),
          py::arg("grid"), py::arg("stream"), py::arg("st") = 0, py::arg("timeout_s") = 0.0, py::arg("mc") = 0,
          py::arg("host_fault") = 0, py::arg("skip") = 0);
    m.def("gtopk_run", &gtopk_run);
    m.def("land_grads", &land_grads);
    m.def("read_trace", &read_trace);
    m.def("host_flag_alloc", &host_flag_alloc);
    m.def("host_flag_free", &host_flag_free);
    m.def("host_flag_read", &host_flag_read);
    m.def("host_flag_clear", &host_flag_clear);
    m.def("fault_ptr", [](uint64_t st) { return (uint64_t)&P_<OktState>(st)->fault; });
    m.def("gather_max_coop_grid", &gather_max_coop_grid);
    m.def("gtopk_max_coop_grid", &gtopk_max_coop_grid);
    m.def("vmm_probe", &vmm_probe);
    m.def("vmm_create", &vmm_create);
    m.def("vmm_import", &vmm_import);
    m.def("vmm_map", &vmm_map);
    m.def("vmm_unmap", &vmm_unmap);
    m.def("vmm_release", &vmm_release);
    m.def("mc_create", &mc_create);
    m.def("mc_add_device", &mc_add_device);
    m.def("mc_bind", &mc_bind);
    m.def("close_fd", [](int fd) { if (fd >= 0) ::close(fd); });
    m.def("clear_fault", [](uint64_t st, uint64_t stream) {
        ck(cudaMemsetAsync(&P_<OktState>(st)->fault, 0, sizeof(int), S_(stream)), "clear_fault");
    });
    m.def("kth_abs", &kth_abs);
    m.def("fused_sgd", &fused_sgd, py::arg("p"), py::arg("g"), py::arg("mom"), py::arg("n"), py::arg("momentum"),
          py::arg("dampening"), py::arg("wd"), py::arg("nesterov"), py::arg("first"), py::arg("zero_grad"),
          py::arg("stream"), py::arg("scal_ptr"), py::arg("fault_ptr") = 0, py::arg("skip_ptr") = 0,
          py::arg("coef_ptr") = 0);
    m.def("sgd_ahead", &sgd_ahead, py::arg("p"), py::arg("mom"), py::arg("sp"), py::arg("sm"), py::arg("n"),
          py::arg("ranges"), py::arg("momentum"), py::arg("dampening"), py::arg("wd"), py::arg("nesterov"),
          py::arg("max_ctas"), py::arg("stream"), py::arg("scal_ptr"));
    m.def("fused_sgd_tail", &fused_sgd_tail, py::arg("p"), py::arg("g"), py::arg("mom"), py::arg("sp"), py::arg("sm"),
          py::arg("n"), py::arg("ahead"), py::arg("dense"), py::arg("momentum"), py::arg("dampening"), py::arg("wd"),
          py::arg("nesterov"), py::arg("first"), py::arg("zero_grad"), py::arg("stream"), py::arg("scal_ptr"),
          py::arg("fault_ptr") = 0, py::arg("skip_ptr") = 0, py::arg("coef_ptr") = 0);
    m.def("fused_bert_adam", &fused_bert_adam, py::arg("p"), py::arg("g"), py::arg("m"), py::arg("v"), py::arg("n"),
          py::arg("b1"), py::arg("b2"), py::arg("eps"), py::arg("wd"), py::arg("zero_grad"), py::arg("stream"),
          py::arg("scal_ptr"), py::arg("fault_ptr") = 0, py::arg("skip_ptr") = 0, py::arg("coef_ptr") = 0,
          py::arg("ends_ptr") = 0);
    m.def("fused_adam", &fused_adam, py::arg("p"), py::arg("g"), py::arg("m"), py::arg("v"), py::arg("n"),
          py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("wd"), py::arg("decoupled"), py::arg("zero_grad"),
          py::arg("stream"), py::arg("scal_ptr"), py::arg("fault_ptr") = 0, py::arg("skip_ptr") = 0,
          py::arg("coef_ptr") = 0);
    m.def("fused_lamb", &fused_lamb, py::arg("p"), py::arg("g"), py::arg("m"), py::arg("v"), py::arg("n"),
          py::arg("beta1"), py::arg("beta2"), py::arg("eps"), py::arg("nseg"), py::arg("off"), py::arg("len"),
          py::arg("blk"), py::arg("ends"), py::arg("nblk"), py::arg("part_w"), py::arg("part_u"), py::arg("norm_w"),
          py::arg("norm_u"), py::arg("ratio"), py::arg("zero_grad"), py::arg("stream"), py::arg("scal_ptr"),
          py::arg("fault_ptr") = 0, py::arg("skip_ptr") = 0, py::arg("coef_ptr") = 0);
    m.def("momentum_correct", &momentum_correct);
    m.def("grad_sumsq", &grad_sumsq, py::arg("g"), py::arg("offs"), py::arg("lens"), py::arg("partial"),
          py::arg("stream"));
    m.def("clip_coef", &clip_coef, py::arg("partial"), py::arg("np"), py::arg("seg_blk"), py::arg("seg_scal"),
          py::arg("nseg"), py::arg("scal"), py::arg("max_norm"), py::arg("norm"), py::arg("coef"), py::arg("stream"));
    m.def("unscale_check", &unscale_check);
    m.def("scale_update", [](uint64_t ls, double growth, double backoff, int interval, uint64_t stream) {
        ck(launch_scale_update(P_<LossScaleDev>(ls), growth, backoff, interval, S_(stream)), "scale_update");
    });
    m.def("adam_scalars", [](uint64_t ls, uint64_t hyper, uint64_t scal, int groups, uint64_t stream, int lamb) {
        ck(launch_adam_scalars(P_<const LossScaleDev>(ls), P_<const double>(hyper), P_<float>(scal), groups, lamb,
                               S_(stream)),
           "adam_scalars");
    }, py::arg("ls"), py::arg("hyper"), py::arg("scal"), py::arg("groups"), py::arg("stream"), py::arg("lamb") = 0);
    m.def("carry_residual", [](uint64_t g, uint64_t res, int n, uint64_t skip, uint64_t stream) {
        ck(launch_carry_residual(P_<float>(g), P_<float>(res), n, P_<const int>(skip), S_(stream)), "carry_residual");
    });
    m.attr("LOSS_SCALE_BYTES") = sizeof(LossScaleDev);
    m.attr("SCALE_SYNC_BYTES") = sizeof(ScaleSync);
    m.attr("VERDICT_OFFSET") = offsetof(ScaleSync, verdict);
    m.def("maxpool2_fwd", &maxpool2_fwd);
    m.def("maxpool2_bwd", &maxpool2_bwd);
    m.def("bn_forward", &bn_forward, py::arg("x"), py::arg("y"), py::arg("arg"), py::arg("partial"), py::arg("gamma"),
          py::arg("beta"), py::arg("cbias"), py::arg("save_mean"), py::arg("save_invstd"), py::arg("rmean"), py::arg("rvar"),
          py::arg("nbt"), py::arg("momentum"), py::arg("eps"), py::arg("relu"), py::arg("M"), py::arg("C"), py::arg("W"),
          py::arg("slot"), py::arg("max_ctas"), py::arg("stream"), py::arg("dtype"), py::arg("res") = 0);
    m.def("bn_backward", &bn_backward, py::arg("x"), py::arg("dy"), py::arg("arg"), py::arg("dx"), py::arg("partial"),
          py::arg("gamma"), py::arg("beta"), py::arg("save_mean"), py::arg("save_invstd"), py::arg("dgamma"), py::arg("dbeta"),
          py::arg("relu"), py::arg("M"), py::arg("C"), py::arg("W"), py::arg("slot"), py::arg("max_ctas"), py::arg("stream"),
          py::arg("dtype"), py::arg("res") = 0, py::arg("dres") = 0);
    m.def("bn_tile_rows", &bn_tile_rows);
    m.def("bn_sliced", &bn_sliced, py::arg("M"), py::arg("C"), py::arg("W"));
    m.def("ln_forward", &ln_forward, py::arg("x"), py::arg("a"), py::arg("y"), py::arg("gamma"), py::arg("beta"),
          py::arg("mean"), py::arg("rstd"), py::arg("seed"), py::arg("R"), py::arg("H"), py::arg("p_keep_thr"),
          py::arg("scale"), py::arg("eps"), py::arg("a_dtype"), py::arg("stream"));
    m.def("ln_backward", &ln_backward, py::arg("x"), py::arg("a"), py::arg("dy"), py::arg("gamma"), py::arg("mean"),
          py::arg("rstd"), py::arg("seed"), py::arg("dx"), py::arg("da"), py::arg("partial"), py::arg("dgamma"),
          py::arg("dbeta"), py::arg("R"), py::arg("H"), py::arg("p_keep_thr"), py::arg("scale"), py::arg("a_dtype"),
          py::arg("stream"));
    m.def("ln_bwd_grid", &ln_bwd_grid);
    m.def("ln_supported_h", &ln_supported_h);
    m.def("emb_forward", &emb_forward, py::arg("ids"), py::arg("tt"), py::arg("word"), py::arg("pos"), py::arg("typ"),
          py::arg("gamma"), py::arg("beta"), py::arg("y"), py::arg("stats"), py::arg("ovf"), py::arg("seed"), py::arg("R"),
          py::arg("S"), py::arg("H"), py::arg("nv"), py::arg("np"), py::arg("nt"), py::arg("p_keep_thr"), py::arg("scale"),
          py::arg("eps"), py::arg("stream"));
    m.def("emb_backward", &emb_backward, py::arg("ids"), py::arg("tt"), py::arg("word"), py::arg("pos"), py::arg("typ"),
          py::arg("gamma"), py::arg("stats"), py::arg("dy"), py::arg("seed"), py::arg("de"), py::arg("partial"), py::arg("dgamma"), py::arg("dbeta"), py::arg("dword"), py::arg("dpos"), py::arg("dtyp"),
          py::arg("R"), py::arg("S"), py::arg("H"), py::arg("nv"), py::arg("np"), py::arg("nt"), py::arg("p_keep_thr"),
          py::arg("scale"), py::arg("stream"));
    m.def("emb_supported", &emb_supported);
    m.def("attn_forward", &attn_forward, py::arg("qkv"), py::arg("mask"), py::arg("seed"), py::arg("out"), py::arg("lse"),
          py::arg("B"), py::arg("S"), py::arg("H"), py::arg("p_keep_thr"), py::arg("scale"), py::arg("dtype"),
          py::arg("stream"));
    m.def("attn_backward", &attn_backward, py::arg("qkv"), py::arg("out"), py::arg("dout"), py::arg("mask"), py::arg("seed"),
          py::arg("lse"), py::arg("delta"), py::arg("dqkv"), py::arg("B"), py::arg("S"), py::arg("H"), py::arg("p_keep_thr"),
          py::arg("scale"), py::arg("dtype"), py::arg("stream"));
    m.def("attn_supported", &attn_supported);
    m.def("xent_forward", &xent_forward, py::arg("x"), py::arg("t"), py::arg("lse"), py::arg("rowloss"), py::arg("loss"),
          py::arg("R"), py::arg("V"), py::arg("ignore_index"), py::arg("dtype"), py::arg("stream"));
    m.def("xent_backward", &xent_backward, py::arg("x"), py::arg("t"), py::arg("lse"), py::arg("g"), py::arg("dx"),
          py::arg("R"), py::arg("V"), py::arg("ignore_index"), py::arg("dtype"), py::arg("stream"));
    m.def("ctc_forward", &ctc_forward, py::arg("x"), py::arg("t"), py::arg("t64"), py::arg("tn"), py::arg("ln"),
          py::arg("ws"), py::arg("loss"), py::arg("T"), py::arg("N"), py::arg("C"), py::arg("nt"), py::arg("dtype"),
          py::arg("stream"));
    m.def("ctc_backward", &ctc_backward, py::arg("x"), py::arg("t"), py::arg("t64"), py::arg("tn"), py::arg("ln"),
          py::arg("ws"), py::arg("ab"), py::arg("g"), py::arg("dx"), py::arg("T"), py::arg("N"), py::arg("C"), py::arg("nt"),
          py::arg("dtype"), py::arg("stream"));
    m.def("ctc_supported", &ctc_supported);
    m.def("frame_bn_forward", &frame_bn_forward, py::arg("conv"), py::arg("x"), py::arg("len"), py::arg("gamma"),
          py::arg("beta"), py::arg("y"), py::arg("mean"), py::arg("rstd"), py::arg("rmean"), py::arg("rvar"),
          py::arg("nbt"), py::arg("N"), py::arg("C"), py::arg("F"), py::arg("Tb"), py::arg("eps"), py::arg("momentum"),
          py::arg("dtype"), py::arg("stream"));
    m.def("frame_bn_backward", &frame_bn_backward, py::arg("conv"), py::arg("x"), py::arg("dy"), py::arg("len"),
          py::arg("gamma"), py::arg("beta"), py::arg("mean"), py::arg("rstd"), py::arg("dx"), py::arg("dgamma"),
          py::arg("dbeta"), py::arg("N"), py::arg("C"), py::arg("F"), py::arg("Tb"), py::arg("dtype"), py::arg("stream"));
    m.def("frame_bn_supported", &frame_bn_supported);
    m.def("lookahead_forward", &lookahead_forward, py::arg("x"), py::arg("w"), py::arg("len"), py::arg("y"), py::arg("N"),
          py::arg("H"), py::arg("Tb"), py::arg("K"), py::arg("dtype"), py::arg("stream"));
    m.def("lookahead_backward", &lookahead_backward, py::arg("x"), py::arg("y"), py::arg("dy"), py::arg("w"),
          py::arg("len"), py::arg("dx"), py::arg("dw"), py::arg("N"), py::arg("H"), py::arg("Tb"), py::arg("K"),
          py::arg("dtype"), py::arg("stream"));
    m.def("lookahead_supported", &lookahead_supported);
    m.def("lookahead_max_taps", &lookahead_max_taps);
    m.def("ctc_workspace_floats", &ctc_workspace_floats);
    m.def("ctc_ab_floats", &ctc_ab_floats);
    m.def("mlm_select", &mlm_select, py::arg("labels"), py::arg("rows"), py::arg("tgt"), py::arg("slot"), py::arg("count"),
          py::arg("overflow"), py::arg("R"), py::arg("M"), py::arg("ignore_index"), py::arg("stream"));
    m.def("mlm_gather", &mlm_gather, py::arg("x"), py::arg("rows"), py::arg("out"), py::arg("M"), py::arg("H"),
          py::arg("dtype"), py::arg("stream"));
    m.def("mlm_scatter", &mlm_scatter, py::arg("dout"), py::arg("slot"), py::arg("dx"), py::arg("R"), py::arg("H"),
          py::arg("dtype"), py::arg("stream"));
    m.def("lstm_forward", &lstm_forward, py::arg("gx"), py::arg("whh"), py::arg("len"), py::arg("y"), py::arg("gates"),
          py::arg("cs"), py::arg("bar"), py::arg("T"), py::arg("N"), py::arg("H"), py::arg("u"), py::arg("rows"),
          py::arg("stream"), py::arg("dtype") = 0, py::arg("whh_rev") = 0);
    m.def("lstm_backward", &lstm_backward, py::arg("dy"), py::arg("gates"), py::arg("cs"), py::arg("whh"), py::arg("len"),
          py::arg("dg"), py::arg("bar"), py::arg("T"), py::arg("N"), py::arg("H"), py::arg("u"), py::arg("rows"),
          py::arg("stream"), py::arg("dtype") = 0, py::arg("whh_rev") = 0);
    m.def("lstm_seq_forward", &lstm_seq_forward, py::arg("gx"), py::arg("whh"), py::arg("h0"), py::arg("c0"),
          py::arg("y"), py::arg("gates"), py::arg("cs"), py::arg("bar"), py::arg("T"), py::arg("N"), py::arg("H"),
          py::arg("u"), py::arg("rows"), py::arg("stream"), py::arg("dtype"), py::arg("r_on") = 0, py::arg("kc") = 0);
    m.def("lstm_seq_backward", &lstm_seq_backward, py::arg("dy"), py::arg("gates"), py::arg("cs"), py::arg("whh"),
          py::arg("c0"), py::arg("dhn"), py::arg("dcn"), py::arg("dg"), py::arg("dc0"), py::arg("bar"), py::arg("T"),
          py::arg("N"), py::arg("H"), py::arg("u"), py::arg("rows"), py::arg("stream"), py::arg("dtype"),
          py::arg("r_on") = 0, py::arg("kc") = 0);
    m.attr("MAXP") = OKT_MAXP;
    m.attr("TRACE_LEN") = kTraceLen;
    m.attr("LAND_MAX") = kLandMax;
    m.attr("SRC_SEG_MAX") = kSrcSegMax;
    m.attr("PACK_RANGE_MAX") = kPackRangeMax;
    m.attr("CHUNK") = kChunk;
    m.attr("SUMSQ_CHUNK") = kSumsqChunk;
}
