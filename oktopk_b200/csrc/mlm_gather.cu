// Fixed-capacity gather of BERT's labelled masked-LM rows, and its scatter back:
//
//   select:  slot[r] = #labelled rows before r    if label[r] != ignore and that number is < M, else -1
//            rows[s] = the row r with slot[r] == s, or -1;   tgt[s] = label[rows[s]], or ignore
//            count = #labelled rows (it may exceed M);        *overflow += max(count - M, 0)
//   gather:  out[s, :] = x[rows[s], :], or 0 where rows[s] == -1                                   out [M, H]
//   scatter: dx[r, :]  = dout[slot[r], :], or 0 where slot[r] == -1                                dx  [R, H]
//
// Only about 11 % of BERT's B S token rows carry a masked-LM label, and the head's transform and decoder GEMMs give the
// other rows logits the loss ignores and gradients that are exactly zero.  Gathering the labelled rows into a buffer of
// M rows, M fixed by the batch shape, cuts those GEMMs to M rows while every shape stays static, so a whole step can
// still be captured in a CUDA graph.
//
// Select (mlm_select_kernel): one CTA of 1024 threads walks the labels in tiles of 1024 rows.  In a tile every thread
// tests one row; a warp ballot and popcount give the row's rank in its warp, warp 0 scans the 32 warp counts, and the
// running total carries over to the next tile.  The order is the row order, with no atomics: the result does not depend
// on scheduling.  Labels are read once, coalesced.  After the last tile the unused slots are padded and thread 0 writes
// the count and adds the overflow.
//
// Gather / scatter (mlm_copy_kernel): a warp per destination row, grid-stride over rows, the lanes striding over the
// row in units of V: a 16-byte vector where the row length in bytes and both base pointers allow it (H = 768 and 1024
// in every type), else one element.  The copy is bitwise, so the kernels depend only on the element size.  The scatter
// writes every row of dx exactly once, zeros included: no separate fill, no atomics.
//
// No host synchronisation anywhere: every launch is graph-capturable.
#include "common.cuh"
#include "elem.cuh"
#include "oktopk.cuh"

namespace okt {

constexpr int kSelThreads = 1024;
constexpr int kCopyThreads = 256;
constexpr int kCopyRowsPerCta = kCopyThreads / 32;
constexpr int kCopyMaxBlocks = 8192;

__global__ void __launch_bounds__(kSelThreads) mlm_select_kernel(const long long* __restrict__ labels, int R,
                                                                 long long ignore, int M, int* __restrict__ rows,
                                                                 long long* __restrict__ tgt, int* __restrict__ slot,
                                                                 long long* __restrict__ count,
                                                                 long long* __restrict__ overflow) {
    __shared__ int s_off[kSelThreads / 32];
    __shared__ int s_tile;
    const int tid = threadIdx.x, lane = lane_id(), warp = tid >> 5;
    int base = 0;                                                 // labelled rows before the tile (the same in every thread)
    for (int r0 = 0; r0 < R; r0 += kSelThreads) {
        const int r = r0 + tid;
        const long long lab = r < R ? __ldg(labels + r) : ignore;
        const bool on = r < R && lab != ignore;
        const unsigned int bal = __ballot_sync(0xffffffffu, on);
        if (lane == 0) s_off[warp] = __popc(bal);
        __syncthreads();
        if (warp == 0) {                                          // exclusive scan of the 32 warp counts
            const int c = s_off[lane];
            int inc = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int v = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += v;
            }
            s_off[lane] = inc - c;
            if (lane == 31) s_tile = inc;
        }
        __syncthreads();
        const int pos = base + s_off[warp] + __popc(bal & ((1u << lane) - 1u));
        if (r < R) {
            const bool kept = on && pos < M;
            slot[r] = kept ? pos : -1;
            if (kept) {
                rows[pos] = r;
                tgt[pos] = lab;
            }
        }
        base += s_tile;
        __syncthreads();                                          // s_off / s_tile are rewritten by the next tile
    }
    for (int s = (base < M ? base : M) + tid; s < M; s += kSelThreads) {
        rows[s] = -1;
        tgt[s] = ignore;
    }
    if (tid == 0) {
        *count = base;
        if (overflow != nullptr && base > M) *overflow += (long long)(base - M);
    }
}

template <typename V> __device__ __forceinline__ V copy_zero() { return V(0); }
template <> __device__ __forceinline__ uint4 copy_zero<uint4>() { return make_uint4(0u, 0u, 0u, 0u); }

// dst[d, :] = src[idx[d], :] for idx[d] >= 0, else 0; rows of n units of V.
template <typename V>
__global__ void __launch_bounds__(kCopyThreads) mlm_copy_kernel(const V* __restrict__ src, const int* __restrict__ idx,
                                                                V* __restrict__ dst, int nrows, int n) {
    const int lane = lane_id();
    for (int d = blockIdx.x * kCopyRowsPerCta + (threadIdx.x >> 5); d < nrows; d += gridDim.x * kCopyRowsPerCta) {
        const int s = __ldg(idx + d);
        V* out = dst + (size_t)d * (size_t)n;
        if (s < 0) {
            for (int k = lane; k < n; k += 32) out[k] = copy_zero<V>();
        } else {
            const V* in = src + (size_t)s * (size_t)n;
            for (int k = lane; k < n; k += 32) out[k] = __ldg(in + k);
        }
    }
}

template <typename V>
static cudaError_t copy_rows_t(const void* src, const int* idx, void* dst, int nrows, int n, cudaStream_t stream) {
    int grid = (nrows + kCopyRowsPerCta - 1) / kCopyRowsPerCta;
    if (grid > kCopyMaxBlocks) grid = kCopyMaxBlocks;
    mlm_copy_kernel<V><<<grid, kCopyThreads, 0, stream>>>(static_cast<const V*>(src), idx, static_cast<V*>(dst), nrows, n);
    return cudaGetLastError();
}

// Rows of H elements of `esize` bytes: 16-byte vectors when the row length and both bases are multiples of 16 bytes.
static cudaError_t copy_rows(const void* src, const int* idx, void* dst, int nrows, int H, int esize, cudaStream_t stream) {
    const size_t row_bytes = (size_t)H * (size_t)esize;
    if (row_bytes % 16 == 0 && ((uintptr_t)src & 15) == 0 && ((uintptr_t)dst & 15) == 0)
        return copy_rows_t<uint4>(src, idx, dst, nrows, (int)(row_bytes / 16), stream);
    if (esize == 4) return copy_rows_t<unsigned int>(src, idx, dst, nrows, H, stream);
    return copy_rows_t<unsigned short>(src, idx, dst, nrows, H, stream);
}

cudaError_t launch_mlm_select(const long long* labels, int R, long long ignore_index, int M, int* rows, long long* tgt,
                              int* slot, long long* count, long long* overflow, cudaStream_t stream) {
    if (R <= 0 || M <= 0) return cudaErrorInvalidValue;
    mlm_select_kernel<<<1, kSelThreads, 0, stream>>>(labels, R, ignore_index, M, rows, tgt, slot, count, overflow);
    return cudaGetLastError();
}

cudaError_t launch_mlm_gather(const void* x, const int* rows, void* out, int M, int H, Dtype dtype, cudaStream_t stream) {
    if (M <= 0 || H <= 0) return cudaErrorInvalidValue;
    return with_dtype(dtype, [&](auto e) { return copy_rows(x, rows, out, M, H, sizeof(e), stream); });
}

cudaError_t launch_mlm_scatter(const void* dout, const int* slot, void* dx, int R, int H, Dtype dtype,
                               cudaStream_t stream) {
    if (R <= 0 || H <= 0) return cudaErrorInvalidValue;
    return with_dtype(dtype, [&](auto e) { return copy_rows(dout, slot, dx, R, H, sizeof(e), stream); });
}

}  // namespace okt
