// Fused (conv-bias +) BatchNorm [+ residual] + ReLU [+ 2x2 max-pool] for channels_last fp32, bf16 or fp16 activations, training mode,
// forward and backward: one kernel per pass -- cooperative with a grid-wide hand-off, or, on small layers, channel-sliced
// with none.
//
// The CNN zoo of the reference (VGG/models/vgg.py:28-36 and the ResNets) is stacks of  Conv2d -> BatchNorm2d -> ReLU
// [-> MaxPool2d].  Run through stock framework ops, a VGG-16 step at 16 images per GPU spends a quarter of its time in the
// glue around the convolutions: per layer a bias-add kernel, a batch-norm kernel, a clamp kernel and a counter increment
// in the forward pass; a threshold kernel, a batch-norm backward kernel and a bias-gradient reduction in the backward
// pass -- all of them latency-bound passes over tensors of 32 K .. 1 M elements.  Here the whole block is one kernel
// forward and one backward.  The activation [M, C] is cut into tiles of ~8 K elements (bn_geom); each CTA keeps its tile
// on chip (kBnHold float4 per thread and tensor, in registers) across one grid-wide hand-off:
//
//   forward : (1) per-tile partial sums of x and x^2 per channel, written to `partial`;
//             (2) the last CTA to arrive combines all partials once, in double (mean, 1/std), saves mean and 1/std,
//                 updates running_mean / running_var / num_batches_tracked and releases the other CTAs;
//             (3) every CTA writes  y = max(0, a_c x + b_c)  from its on-chip tile, or, when a 2x2 / stride-2 max-pool
//                 follows, only the pooled output and the one-byte arg-max: the pre-pool y is never written;
//   backward: (1) per-tile partials of  dbeta = sum(dy * [z>0])  and  dgamma = sum(dy * [z>0] * xhat), where with a pool
//                 dy is the pooled gradient expanded at the arg-max (zero elsewhere) in registers;
//             (2) the last CTA combines them and publishes dgamma, dbeta;
//             (3) dx = a_c (dy[z>0] - dbeta/M - xhat dgamma/M)  from the on-chip x and dy.
//
// The grid is min(tiles, co-resident CTAs) and the launch is cooperative, so every CTA is resident while the others wait
// for the combine.  A CTA's tiles after its first (only when tiles outnumber co-resident CTAs), and tiles larger than
// kBnHold float4 per thread, are read again from global memory in (3).  The tile partition, the per-thread summation
// order and the combine order do not depend on the grid, so neither do the results.
//
// Summation tree.  Every per-channel sum (x, x^2; dbeta, dgamma) is added in one fixed fp32 tree that depends on (M, C)
// alone, with bn_geom's tiles of rows_per_block rows and rpi row lanes:
//   1. per tile t and lane ty: the rows  t rows_per_block + ty + k rpi,  k ascending, one after the other (x^2 and dgamma
//      by fmaf into the running sum);
//   2. per tile: lanes ty = 0 .. rpi-1 in ascending order (bn_tile_partial);
//   3. across tiles (bn_combine_partials): the partial row is [sum | second sum], C/2 float4 columns, taken in chunks of
//      256 columns; in the chunk at c0,  w = min(256, C/2 - c0)  and  groups = 256 / w;  group j adds tiles j, j + groups,
//      ... in order, starting from 0.f, and the groups are then added in ascending order.
// Mean and 1/std come from the totals in double (bn_stats).
//
// Channel-sliced kernels (bn_fwd_sliced_kernel, bn_bwd_sliced_kernel; chosen by bn_geom's sc, see there).  Statistics are
// per channel, so a CTA that owns sc float4 columns and ALL rows needs nobody else: thread (column of the slice, tile,
// lane) does step 1 privately on rows it holds in registers, bn_slice_reduce does steps 2 and 3 in shared memory, and
// the CTA computes the statistics of its channels and writes y / dx from the held rows.  No partials, no g_bn_sync, no
// wait on another CTA, a plain launch.  Same tree and the same per-element device functions as the cooperative kernels,
// hence the same bits.  A grid cap (max_ctas > 0) always selects the cooperative kernels.  Layers with fewer than
// 2 kBnMinSlices float4 columns or more rows than a CTA's threads can hold stay cooperative.
//
// A bias added before a batch-norm cancels exactly: BN(x + b) = BN(x) with the batch mean shifted by b.  The forward pass
// therefore never adds it (only running_mean sees it), and its gradient -- identically zero, since the loss does not depend
// on it -- is not "computed" by a reduction over dy that can only return rounding noise.
//
// Residual (kRes, the end of a ResNet block: y = relu(bn(x) + r)): r is [M, C] in x's type and layout.  The statistics,
// running statistics and conv-bias rule are unchanged: the batch-norm only sees x.
//   forward : (3) writes  y = max(0, fma(x, a, b) + r)  (fp32 add of the widened r), reading r as y is stored;
//   backward: (1) recomputes the mask  [fma(x, a, b) + r > 0]  bit for bit, writes  dres = dy [mask]  (exact: dy or 0)
//                 and takes dbeta / dgamma over it; a held tile keeps the masked gradient on chip;
//             (3) dx by the same formula from the masked gradient: held, or the dres this CTA wrote in (1), read back.
// kRes and kPool never combine (no ResNet pools after the add); kRes = false compiles to the kernels without it.
//
// Layout: x is [M, C] row-major (NHWC with M = N*H*W), C a multiple of 4; each thread owns 4 consecutive channels
// (128-bit accesses) and strides over rows; tiles are contiguous row ranges.  With a pool, a tile is a whole number of
// image row pairs (rows_per_block % 2W == 0), so no 2x2 window straddles two tiles.
//
// Activation type: x, y, dy and dx are fp32 (one float4 per access), bf16 or fp16 (four 16-bit values in one 8-byte
// access), converted by elem.cuh's Elem.  A bf16 or fp16 load is widened to a float4, which is exact, and from there the
// arithmetic is the fp32 kernel's, operation for operation: same tiles, partials, combine, running-statistic fma, ReLU
// mask, pool arg-max and dx formula.  Only the stores of y and dx round to the 16-bit type, under elem.cuh's contract (to
// nearest even; an fp16 overflow is +-inf, which under loss scaling is how an fp16 step overflows and must reach the
// optimizer's non-finite check; fp16 subnormals are kept).  The bf16 and fp16 kernels are therefore, bit for bit, the
// fp32 kernel run on x.float() (and dy.float()) with y and dx rounded.  An inf or NaN in x or dy propagates as in that
// kernel, into the statistics and the running statistics too (as stock batch-norm does); there is no extra finite
// check.  gamma, beta, the conv bias, the running and saved statistics, the partials and dgamma / dbeta stay fp32 in
// every case, as in torch's batch-norm under autocast.
#include "common.cuh"
#include "elem.cuh"
#include "oktopk.cuh"

namespace okt {

constexpr int kBnThreads = 256;
constexpr int kBnMaxBlocks = 512;
constexpr int kBnHold = 8;             // float4 per thread and tensor held on chip: a whole ~8 K-element tile (bn_geom)
constexpr int kBnSyncSlots = 1024;
constexpr int kBnMinSlices = 32;       // channel-sliced kernels: at least this many CTAs, or the cooperative kernels run

// {arrival ticket, release generation} per call site (the caller picks the slot).  Zero at module load; every kernel
// leaves its ticket at zero and only advances the generation, so a CUDA graph replays the kernels without a reset node.
__device__ unsigned int g_bn_sync[kBnSyncSlots][2];

struct BnGeom {
    int M, C, cv;          // rows, channels, float4 columns (C/4)
    int tpr, rpi;          // threads per row, rows per block iteration
    int rows_per_block, nblk;
    int hold;              // a tile fits in kBnHold float4 per thread (one column tile)
    int W;                 // > 0: a 2x2 / stride-2 max-pool over images of width W follows
    int sc;                // > 0: the channel-sliced kernels can run, with sc float4 columns per CTA (2 .. 8)
};

__host__ __device__ inline BnGeom bn_geom(int M, int C) {
    BnGeom g;
    g.M = M; g.C = C; g.cv = C >> 2;
    g.tpr = g.cv < kBnThreads ? g.cv : kBnThreads;
    g.rpi = kBnThreads / g.tpr;
    if (g.rpi < 1) g.rpi = 1;
    // ~8 K elements per block: enough blocks to spread a 1 M-element tensor over the GPU, a few blocks for the tiny layers
    long long want = ((long long)M * C + 8191) / 8192;
    if (want < 1) want = 1;
    if (want > kBnMaxBlocks) want = kBnMaxBlocks;
    int rpb = (int)((M + want - 1) / want);
    rpb = (rpb + g.rpi - 1) / g.rpi * g.rpi;
    if (rpb < g.rpi) rpb = g.rpi;
    g.rows_per_block = rpb;
    g.nblk = (M + rpb - 1) / rpb;
    g.hold = g.cv <= kBnThreads && rpb / g.rpi <= kBnHold;
    g.W = 0;
    // Channel-sliced: one thread per (column of the slice, tile, row lane), so a CTA of sc columns has sc * nblk * rpi
    // threads.  The widest power-of-two slice that fits a CTA and still leaves kBnMinSlices CTAs; a one-column slice
    // (16 bytes per row, half a sector) does not qualify.
    g.sc = 0;
    if (g.hold) {
        int sc = 1;
        while (2 * sc * g.nblk * g.rpi <= kBnThreads && g.cv / (2 * sc) >= kBnMinSlices) sc *= 2;
        if (sc >= 2 && g.cv % sc == 0) g.sc = sc;
    }
    return g;
}

__device__ __forceinline__ float4 f4_fma(const float4& x, const float4& a, const float4& b) {
    return make_float4(fmaf(x.x, a.x, b.x), fmaf(x.y, a.y, b.y), fmaf(x.z, a.z, b.z), fmaf(x.w, a.w, b.w));
}

// one step of a 2x2 max-pool window: first maximum in row-major window order wins, NaN propagates (as at::max_pool2d)
__device__ __forceinline__ void pool_step(float4& m, uchar4& a, const float4& v, unsigned char k) {
    if (v.x > m.x || v.x != v.x) { m.x = v.x; a.x = k; }
    if (v.y > m.y || v.y != v.y) { m.y = v.y; a.y = k; }
    if (v.z > m.z || v.z != v.z) { m.z = v.z; a.z = k; }
    if (v.w > m.w || v.w != v.w) { m.w = v.w; a.w = k; }
}

// The 2x2 window of a pooled pixel whose first row is lr: at(lr, c), at(lr + 1, c), at(lr + W, c), at(lr + W + 1, c).
template <typename At>
__device__ __forceinline__ void pool_window(At at, int lr, int W, int c, float4& m, uchar4& a) {
    const float4 v1 = at(lr + 1, c), v2 = at(lr + W, c), v3 = at(lr + W + 1, c);
    m = at(lr, c);
    a = make_uchar4(0, 0, 0, 0);
    pool_step(m, a, v1, 1);
    pool_step(m, a, v2, 2);
    pool_step(m, a, v3, 3);
}

// One row's term of a thread's private sums of x and x^2.
__device__ __forceinline__ void bn_sum_sq(float4& s, float4& q, const float4& v) {
    s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    q.x = fmaf(v.x, v.x, q.x); q.y = fmaf(v.y, v.y, q.y); q.z = fmaf(v.z, v.z, q.z); q.w = fmaf(v.w, v.w, q.w);
}

// y = a x + b [ReLU], and with a residual y = max(0, (a x + b) + r)
__device__ __forceinline__ float4 bn_y(const float4& x, const float4& a, const float4& b, int relu) {
    float4 v = f4_fma(x, a, b);
    if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    return v;
}
__device__ __forceinline__ float4 bn_y_res(const float4& x, const float4& r, const float4& a, const float4& b) {
    float4 v = f4_fma(x, a, b);
    v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
    v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    return v;
}

// Combine the per-tile partials [nblk][2C] into s_tot[2C] with ALL threads of the block: a tile of up to 256 float4
// columns at a time, the threads that share a column stride over the tiles, then one shared-memory reduction.  The
// partials were written by other CTAs of the same kernel: L2-coherent loads.
__device__ __forceinline__ void bn_combine_partials(const float* __restrict__ partial, int nblk, int C, float* s_tot,
                                                    float4* s_scr) {
    const int cols = (2 * C) >> 2;                          // float4 columns of one partial row
    const float4* p4 = reinterpret_cast<const float4*>(partial);
    for (int c0 = 0; c0 < cols; c0 += kBnThreads) {
        const int w = min(kBnThreads, cols - c0);
        const int groups = kBnThreads / w;
        const int tx = threadIdx.x % w, ty = threadIdx.x / w;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        if (ty < groups)
            for (int b0 = ty; b0 < nblk; b0 += 8 * groups) {       // eight loads in flight, then the same in-order sum
                float4 v[8];
#pragma unroll
                for (int u = 0; u < 8; ++u)
                    if (b0 + u * groups < nblk) v[u] = __ldcg(p4 + (size_t)(b0 + u * groups) * cols + c0 + tx);
#pragma unroll
                for (int u = 0; u < 8; ++u)
                    if (b0 + u * groups < nblk) { acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w; }
            }
        s_scr[threadIdx.x] = acc;
        __syncthreads();
        if (ty == 0) {
            for (int j = 1; j < groups; ++j) {
                const float4 v = s_scr[j * w + tx];
                acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
            }
            reinterpret_cast<float4*>(s_tot)[c0 + tx] = acc;
        }
        __syncthreads();
    }
}

// Sum the per-thread column sums (s, q) of a tile over its rpi row groups, in a fixed order, into partial row `tile`.
__device__ __forceinline__ void bn_tile_partial(float4 s, float4 q, int tx, int ty, int col, const BnGeom& g, float4* s_red,
                                                float* __restrict__ partial, int tile) {
    if (ty < g.rpi) { s_red[ty * g.tpr + tx] = s; s_red[(g.rpi + ty) * g.tpr + tx] = q; }
    __syncthreads();
    if (ty == 0 && col < g.cv) {
        for (int j = 1; j < g.rpi; ++j) {
            const float4 a = s_red[j * g.tpr + tx], b = s_red[(g.rpi + j) * g.tpr + tx];
            s.x += a.x; s.y += a.y; s.z += a.z; s.w += a.w;
            q.x += b.x; q.y += b.y; q.z += b.z; q.w += b.w;
        }
        float4* p4 = reinterpret_cast<float4*>(partial + (size_t)tile * 2 * g.C);
        p4[col] = s;
        p4[g.cv + col] = q;
    }
    __syncthreads();
}

// Channel-sliced CTA: thread (tile t, lane ty, column cx of the slice) = threadIdx.x = (t * rpi + ty) * sc + cx holds its
// private sums (s, q).  Adds them in the order of the summation tree (file header), which is what bn_tile_partial and
// bn_combine_partials do across CTAs, and leaves the totals in s_tot: [sc] of s, then [sc] of q.
// s_scr: 2 * blockDim + 2 * nblk * sc float4 of scratch, free again on return.
__device__ __forceinline__ void bn_slice_reduce(const float4& s, const float4& q, const BnGeom& g, float4* s_scr,
                                                float4* s_tot) {
    const int sc = g.sc, lanes = g.nblk * g.rpi;
    float4* s_lane = s_scr;
    float4* s_tile = s_scr + 2 * blockDim.x;
    auto add = [](float4& a, const float4& b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; };
    s_lane[threadIdx.x] = s;
    s_lane[lanes * sc + threadIdx.x] = q;
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * g.nblk * sc; i += blockDim.x) {           // a tile's lanes, ascending
        const int which = i / (g.nblk * sc), t = i / sc % g.nblk, cx = i % sc;
        const float4* src = s_lane + (which * lanes + t * g.rpi) * sc + cx;
        float4 v = src[0];
        for (int j = 1; j < g.rpi; ++j) add(v, src[j * sc]);
        s_tile[i] = v;                                                          // [which][t][cx]
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * sc; i += blockDim.x) {                    // tiles j, j + groups, ...; then the groups
        const int which = i / sc, cx = i % sc;
        const int pcol = which * g.cv + blockIdx.x * sc + cx;                   // float4 column of a partial row [2C]
        const int groups = kBnThreads / min(kBnThreads, 2 * g.cv - pcol / kBnThreads * kBnThreads);
        float4 tot;
        for (int j = 0; j < groups; ++j) {
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int b = j; b < g.nblk; b += groups) add(acc, s_tile[(which * g.nblk + b) * sc + cx]);
            if (j == 0) tot = acc; else add(tot, acc);
        }
        s_tot[i] = tot;
    }
    __syncthreads();
}

// Grid-wide hand-off.  bn_arrive: once every CTA has written its partials, exactly one CTA (the last to arrive) gets
// true and does the combine.  bn_release: that CTA publishes its results; every other CTA waits there for them.  The
// generation is read before arriving, and the last CTA can only advance it after every arrival.
// Ordering is release/acquire by thread 0 on either side of a CTA barrier (cumulative over the CTA's writes); no
// sequentially consistent fence (__threadfence) sits on this latency-bound path.
__device__ __forceinline__ bool bn_arrive(unsigned int* sync, unsigned int& gen) {
    __shared__ unsigned int s_gen;
    __shared__ int s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
        s_gen = ld_acquire_gpu_u32(sync + 1);
        // release: this CTA's partials; acquire: those of every CTA that arrived before
        const unsigned int old = atom_add_acq_rel_gpu_u32(sync, 1u);
        s_last = old == gridDim.x - 1u;
        if (s_last) st_relaxed_gpu_u32(sync, 0u);       // every CTA has arrived: the next launch starts from zero
    }
    __syncthreads();
    gen = s_gen;
    return s_last != 0;
}

__device__ __forceinline__ void bn_release(unsigned int* sync, bool last, unsigned int gen) {
    __syncthreads();
    if (threadIdx.x == 0) {
        if (last) {
            st_release_gpu_u32(sync + 1, gen + 1u);
        } else {
            while (ld_acquire_gpu_u32(sync + 1) == gen) { }
        }
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------- forward
template <typename T>
struct BnFwdArgs {
    const T* x;
    T* y;                       // [M, C], or with a pool [M/4, C]
    unsigned char* arg;         // pool only: arg-max (0..3) per pooled element
    float* partial;             // [nblk][2][C]  (sum, sum of squares)
    const float* gamma; const float* beta; const float* cbias;
    float* save_mean; float* save_invstd; float* rmean; float* rvar; long long* nbt;
    float momentum, eps;
    int relu;
    unsigned int* sync;
    BnGeom g;
    const T* res;               // kRes only: the residual [M, C], added after the batch-norm, before the ReLU
};

// Channel c from its sums s of x and q of x^2 over the M rows: mean and 1/std in double, saved; running statistics with
// the unbiased variance and the conv-bias-shifted mean.
template <typename T>
__device__ __forceinline__ void bn_stats(const BnFwdArgs<T>& p, int c, float sf, float qf) {
    const BnGeom& g = p.g;
    const double s = (double)sf, q = (double)qf;
    const double mean = s / (double)g.M;
    double var = q / (double)g.M - mean * mean;
    if (var < 0.0) var = 0.0;
    const float invstd = (float)(1.0 / sqrt(var + (double)p.eps));
    p.save_mean[c] = (float)mean;
    p.save_invstd[c] = invstd;
    if (p.rmean != nullptr) {
        const float mb = (float)mean + (p.cbias != nullptr ? __ldg(p.cbias + c) : 0.f);
        const double unb = g.M > 1 ? var * (double)g.M / (double)(g.M - 1) : var;
        p.rmean[c] = fmaf(p.momentum, mb, __fmul_rn(1.f - p.momentum, p.rmean[c]));
        p.rvar[c] = fmaf(p.momentum, (float)unb, __fmul_rn(1.f - p.momentum, p.rvar[c]));
    }
}

// a = gamma / std, b = beta - mean a of channel c
template <typename T>
__device__ __forceinline__ void bn_scale_shift(const BnFwdArgs<T>& p, int c, float mean, float invstd, float& a, float& b) {
    a = __fmul_rn(__ldg(p.gamma + c), invstd);
    b = __fsub_rn(__ldg(p.beta + c), __fmul_rn(mean, a));      // no fma: backward recomputes it
}

template <bool kPool, bool kRes, typename T>
__global__ void __launch_bounds__(kBnThreads) bn_fwd_kernel(const BnFwdArgs<T> p) {
    static_assert(!(kPool && kRes), "no pool follows a residual add");
    using A = Elem<T>;
    using V = typename A::V;
    extern __shared__ float4 s_dyn[];         // [2][cv] combine totals, then a = gamma/std, b = beta - mean a | pool: held y
    __shared__ float4 s_red[2 * kBnThreads];
    const BnGeom& g = p.g;
    const int tx = threadIdx.x % g.tpr, ty = threadIdx.x / g.tpr;
    const V* x4 = reinterpret_cast<const V*>(p.x);
    auto ldx = [&](size_t o) { return A::wide(__ldg(x4 + o)); };
    const size_t st1 = (size_t)g.rpi * g.cv;
    V h[kBnHold];                             // the CTA's first tile (grid <= tiles: every CTA has one), as stored

    // (1) partial sums, four or more independent 128-bit loads in flight per thread
    for (int t = blockIdx.x; t < g.nblk; t += gridDim.x) {
        const bool held = g.hold && t == (int)blockIdx.x;
        const int row0 = t * g.rows_per_block, row1 = min(g.M, row0 + g.rows_per_block);
        for (int c0 = 0; c0 < g.cv; c0 += g.tpr) {
            const int col = c0 + tx;
            float4 s = make_float4(0.f, 0.f, 0.f, 0.f), q = s;
            if (ty < g.rpi && col < g.cv) {
                auto acc = [&](const float4& v) { bn_sum_sq(s, q, v); };
                int r = row0 + ty;
                if (held) {
#pragma unroll
                    for (int k = 0; k < kBnHold; ++k)
                        h[k] = r + k * g.rpi < row1 ? __ldg(x4 + (size_t)(r + k * g.rpi) * g.cv + col) : V{};
#pragma unroll
                    for (int k = 0; k < kBnHold; ++k)
                        if (r + k * g.rpi < row1) acc(A::wide(h[k]));
                } else {
                    for (; r + 3 * g.rpi < row1; r += 4 * g.rpi) {
                        const size_t o = (size_t)r * g.cv + col;
                        const float4 v0 = ldx(o), v1 = ldx(o + st1), v2 = ldx(o + 2 * st1), v3 = ldx(o + 3 * st1);
                        acc(v0); acc(v1); acc(v2); acc(v3);
                    }
                    for (; r < row1; r += g.rpi) acc(ldx((size_t)r * g.cv + col));
                }
            }
            bn_tile_partial(s, q, tx, ty, col, g, s_red, p.partial, t);
        }
    }

    // (2) one CTA combines; mean and 1/std in double; running statistics (unbiased variance), bias-shifted mean
    float* s_ab = reinterpret_cast<float*>(s_dyn);
    unsigned int gen;
    const bool last = bn_arrive(p.sync, gen);
    if (last) {
        float* s_tot = s_ab;                  // overwritten by a, b only after bn_release's barrier
        bn_combine_partials(p.partial, g.nblk, g.C, s_tot, s_red);
        for (int c = threadIdx.x; c < g.C; c += kBnThreads) bn_stats(p, c, s_tot[c], s_tot[g.C + c]);
        if (threadIdx.x == 0 && p.nbt != nullptr) *p.nbt += 1;
    }
    bn_release(p.sync, last, gen);
    for (int c = threadIdx.x; c < g.C; c += kBnThreads)
        bn_scale_shift(p, c, __ldcg(p.save_mean + c), __ldcg(p.save_invstd + c), s_ab[c], s_ab[g.C + c]);
    __syncthreads();

    // (3) y = max(0, a x + b), or its 2x2 max-pool, or with a residual r  y = max(0, (a x + b) + r)
    const float4* ab4 = s_dyn;                // [cv] a | [cv] b
    auto yval = [&](const float4& xin, int col) { return bn_y(xin, ab4[col], ab4[g.cv + col], p.relu); };
    const V* r4 = reinterpret_cast<const V*>(p.res);
    auto ldr = [&](size_t o) { return A::wide(__ldg(r4 + o)); };
    auto yres = [&](const float4& xin, const float4& rin, int col) {
        return bn_y_res(xin, rin, ab4[col], ab4[g.cv + col]);
    };
    V* y4 = reinterpret_cast<V*>(p.y);
    for (int t = blockIdx.x; t < g.nblk; t += gridDim.x) {
        const bool held = g.hold && t == (int)blockIdx.x;
        const int row0 = t * g.rows_per_block, row1 = min(g.M, row0 + g.rows_per_block);
        if (!kPool) {
            for (int c0 = 0; c0 < g.cv; c0 += g.tpr) {
                const int col = c0 + tx;
                if (ty >= g.rpi || col >= g.cv) continue;
                int r = row0 + ty;
                if (held) {
                    if constexpr (kRes) {
                        float4 q[kBnHold];
#pragma unroll
                        for (int k = 0; k < kBnHold; ++k)
                            if (r + k * g.rpi < row1) q[k] = ldr((size_t)(r + k * g.rpi) * g.cv + col);
#pragma unroll
                        for (int k = 0; k < kBnHold; ++k)
                            if (r + k * g.rpi < row1)
                                y4[(size_t)(r + k * g.rpi) * g.cv + col] = A::narrow(yres(A::wide(h[k]), q[k], col));
                    } else {
#pragma unroll
                        for (int k = 0; k < kBnHold; ++k)
                            if (r + k * g.rpi < row1) y4[(size_t)(r + k * g.rpi) * g.cv + col] = A::narrow(yval(A::wide(h[k]), col));
                    }
                    continue;
                }
                for (; r + 3 * g.rpi < row1; r += 4 * g.rpi) {
                    const size_t o = (size_t)r * g.cv + col;
                    const float4 v0 = ldx(o), v1 = ldx(o + st1), v2 = ldx(o + 2 * st1), v3 = ldx(o + 3 * st1);
                    if constexpr (kRes) {
                        const float4 q0 = ldr(o), q1 = ldr(o + st1), q2 = ldr(o + 2 * st1), q3 = ldr(o + 3 * st1);
                        y4[o] = A::narrow(yres(v0, q0, col)); y4[o + st1] = A::narrow(yres(v1, q1, col));
                        y4[o + 2 * st1] = A::narrow(yres(v2, q2, col)); y4[o + 3 * st1] = A::narrow(yres(v3, q3, col));
                    } else {
                        y4[o] = A::narrow(yval(v0, col)); y4[o + st1] = A::narrow(yval(v1, col));
                        y4[o + 2 * st1] = A::narrow(yval(v2, col)); y4[o + 3 * st1] = A::narrow(yval(v3, col));
                    }
                }
                for (; r < row1; r += g.rpi) {
                    const size_t o = (size_t)r * g.cv + col;
                    if constexpr (kRes) y4[o] = A::narrow(yres(ldx(o), ldr(o), col));
                    else y4[o] = A::narrow(yval(ldx(o), col));
                }
            }
        } else {
            // a held tile is staged in shared memory (its windows span threads); the window of pooled pixel pp is the
            // tile rows lr, lr+1, lr+W, lr+W+1; the tile's pooled pixels start at row0/4 (row0 is a multiple of 2W)
            float4* sy = s_dyn + g.C / 2;
            if (held) {
                if (ty < g.rpi) {
#pragma unroll
                    for (int k = 0; k < kBnHold; ++k)
                        if (row0 + ty + k * g.rpi < row1) sy[(ty + k * g.rpi) * g.cv + tx] = yval(A::wide(h[k]), tx);
                }
                __syncthreads();
            }
            auto at = [&](int lr, int c) { return held ? sy[lr * g.cv + c] : yval(ldx((size_t)(row0 + lr) * g.cv + c), c); };
            const int W = g.W, Wo = W >> 1, npool = (row1 - row0) / 4 * g.cv;
            uchar4* a4 = reinterpret_cast<uchar4*>(p.arg);
            for (int i = threadIdx.x; i < npool; i += kBnThreads) {
                const int c = i % g.cv, pp = i / g.cv;
                const int lr = (pp / Wo) * 2 * W + (pp % Wo) * 2;
                float4 m;
                uchar4 a;
                pool_window(at, lr, W, c, m, a);
                const size_t o = (size_t)(row0 / 4 + pp) * g.cv + c;
                y4[o] = A::narrow(m);
                a4[o] = a;
            }
        }
    }
}

// Channel-sliced forward (g.sc > 0): CTA b owns float4 columns [b sc, (b + 1) sc) and every row; blockDim = sc nblk rpi.
// No partials, no hand-off: the statistics of the owned channels never leave the CTA.
template <bool kPool, bool kRes, typename T>
__global__ void __launch_bounds__(kBnThreads) bn_fwd_sliced_kernel(const BnFwdArgs<T> p) {
    static_assert(!(kPool && kRes), "no pool follows a residual add");
    using A = Elem<T>;
    using V = typename A::V;
    extern __shared__ float4 s_dyn[];         // bn_slice_reduce's scratch, then with a pool the slice's y, [M][sc]
    __shared__ float4 s_tot[2 * 8], s_ab[2 * 8];   // the owned columns' totals [sc] | [sc]; a = gamma/std [sc] | b [sc]
    const BnGeom& g = p.g;
    const int sc = g.sc, cx = threadIdx.x % sc, ln = threadIdx.x / sc, col = blockIdx.x * sc + cx;
    const int row0 = ln / g.rpi * g.rows_per_block, row1 = min(g.M, row0 + g.rows_per_block), r = row0 + ln % g.rpi;
    const V* x4 = reinterpret_cast<const V*>(p.x);

    // (1) the thread's rows, held; their sums in row order
    V h[kBnHold];
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f), q = s;
#pragma unroll
    for (int k = 0; k < kBnHold; ++k) h[k] = r + k * g.rpi < row1 ? __ldg(x4 + (size_t)(r + k * g.rpi) * g.cv + col) : V{};
#pragma unroll
    for (int k = 0; k < kBnHold; ++k)
        if (r + k * g.rpi < row1) bn_sum_sq(s, q, A::wide(h[k]));

    // (2) totals of the owned channels, their statistics, a and b
    bn_slice_reduce(s, q, g, s_dyn, s_tot);
    const float* s_f = reinterpret_cast<const float*>(s_tot);
    float* s_abf = reinterpret_cast<float*>(s_ab);
    for (int i = threadIdx.x; i < 4 * sc; i += blockDim.x) {        // a CTA can have fewer threads than channels
        const int c = blockIdx.x * 4 * sc + i;
        bn_stats(p, c, s_f[i], s_f[4 * sc + i]);
        bn_scale_shift(p, c, p.save_mean[c], p.save_invstd[c], s_abf[i], s_abf[4 * sc + i]);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0 && p.nbt != nullptr) *p.nbt += 1;
    __syncthreads();

    // (3) y from the held rows
    const float4 a4 = s_ab[cx], b4 = s_ab[sc + cx];
    V* y4 = reinterpret_cast<V*>(p.y);
    if constexpr (kRes) {
        const V* r4 = reinterpret_cast<const V*>(p.res);
#pragma unroll
        for (int k0 = 0; k0 < kBnHold; k0 += 4) {               // four residual loads in flight beside the held rows
            float4 rr[4];
#pragma unroll
            for (int k = k0; k < k0 + 4; ++k)
                if (r + k * g.rpi < row1) rr[k - k0] = A::wide(__ldg(r4 + (size_t)(r + k * g.rpi) * g.cv + col));
#pragma unroll
            for (int k = k0; k < k0 + 4; ++k)
                if (r + k * g.rpi < row1)
                    y4[(size_t)(r + k * g.rpi) * g.cv + col] = A::narrow(bn_y_res(A::wide(h[k]), rr[k - k0], a4, b4));
        }
    } else if constexpr (!kPool) {
#pragma unroll
        for (int k = 0; k < kBnHold; ++k)
            if (r + k * g.rpi < row1) y4[(size_t)(r + k * g.rpi) * g.cv + col] = A::narrow(bn_y(A::wide(h[k]), a4, b4, p.relu));
    } else {
        // every 2x2 window of the owned columns lies in this CTA; rows and pooled pixels are global (the first row is 0)
#pragma unroll
        for (int k = 0; k < kBnHold; ++k)
            if (r + k * g.rpi < row1) s_dyn[(r + k * g.rpi) * sc + cx] = bn_y(A::wide(h[k]), a4, b4, p.relu);
        __syncthreads();
        auto at = [&](int lr, int c) { return s_dyn[lr * sc + c]; };
        const int W = g.W, Wo = W >> 1;
        uchar4* arg4 = reinterpret_cast<uchar4*>(p.arg);
        for (int i = threadIdx.x; i < g.M / 4 * sc; i += blockDim.x) {
            const int c = i % sc, pp = i / sc;
            float4 m;
            uchar4 am;
            pool_window(at, (pp / Wo) * 2 * W + (pp % Wo) * 2, W, c, m, am);
            const size_t o = (size_t)pp * g.cv + blockIdx.x * sc + c;
            y4[o] = A::narrow(m);
            arg4[o] = am;
        }
    }
}

// ---------------------------------------------------------------------------------------------- backward
template <typename T>
struct BnBwdArgs {
    const T* x;
    const T* dy;                // [M, C], or with a pool the pooled gradient [M/4, C]
    const unsigned char* arg;   // pool only: the forward's arg-max
    T* dx;
    float* partial;             // [nblk][2][C]  (dbeta, dgamma)
    const float* gamma; const float* beta; const float* save_mean; const float* save_invstd;
    float* dgamma; float* dbeta;
    int relu;
    unsigned int* sync;
    BnGeom g;
    const T* res;               // kRes only: the forward's residual [M, C]
    T* dres;                    // kRes only: its gradient dy * [z > 0], [M, C]
};

// Per-element arithmetic of the backward pass, shared by the cooperative and the channel-sliced kernels.
// Per-column constants; the forward output was max(0, fma(x, a, b)): same a, b, same fma => the same mask, bit for bit.
struct BnCol { float4 mean, istd, a, b; };

template <bool kPool, bool kRes, typename T>
struct BnBwdElem {
    using A = Elem<T>;
    using V = typename A::V;
    const BnBwdArgs<T>& p;

    // the gradient reaching the batch-norm output at row r: dy, or the pooled dy at the window's arg-max and 0 elsewhere
    // (row0: the first row of r's tile, a multiple of 2W; 0 takes r as a global row)
    __device__ __forceinline__ float4 grad(int row0, int r, int col) const {
        const BnGeom& g = p.g;
        const V* d4 = reinterpret_cast<const V*>(p.dy);
        if (!kPool) return A::wide(__ldg(d4 + (size_t)r * g.cv + col));
        const int lr = r - row0, hl = lr / g.W, w = lr - hl * g.W;
        const size_t o = (size_t)(row0 / 4 + (hl >> 1) * (g.W >> 1) + (w >> 1)) * g.cv + col;
        const int k = (hl & 1) * 2 + (w & 1);
        const float4 d = A::wide(__ldg(d4 + o));
        const uchar4 a = __ldg(reinterpret_cast<const uchar4*>(p.arg) + o);
        return make_float4(a.x == k ? d.x : 0.f, a.y == k ? d.y : 0.f, a.z == k ? d.z : 0.f, a.w == k ? d.w : 0.f);
    }
    __device__ __forceinline__ BnCol column(int col) const {
        BnCol k;
        k.mean = __ldg(reinterpret_cast<const float4*>(p.save_mean) + col);
        k.istd = __ldg(reinterpret_cast<const float4*>(p.save_invstd) + col);
        const float4 gm = __ldg(reinterpret_cast<const float4*>(p.gamma) + col);
        const float4 bt = __ldg(reinterpret_cast<const float4*>(p.beta) + col);
        k.a = make_float4(__fmul_rn(gm.x, k.istd.x), __fmul_rn(gm.y, k.istd.y), __fmul_rn(gm.z, k.istd.z), __fmul_rn(gm.w, k.istd.w));
        k.b = make_float4(__fsub_rn(bt.x, __fmul_rn(k.mean.x, k.a.x)), __fsub_rn(bt.y, __fmul_rn(k.mean.y, k.a.y)),
                          __fsub_rn(bt.z, __fmul_rn(k.mean.z, k.a.z)), __fsub_rn(bt.w, __fmul_rn(k.mean.w, k.a.w)));
        return k;
    }
    __device__ __forceinline__ void mask(const BnCol& k, const float4& v, float4& d) const {
        if (p.relu) {
            if (!(fmaf(v.x, k.a.x, k.b.x) > 0.f)) d.x = 0.f;
            if (!(fmaf(v.y, k.a.y, k.b.y) > 0.f)) d.y = 0.f;
            if (!(fmaf(v.z, k.a.z, k.b.z) > 0.f)) d.z = 0.f;
            if (!(fmaf(v.w, k.a.w, k.b.w) > 0.f)) d.w = 0.f;
        }
    }
    static __device__ __forceinline__ float4 xhat(const BnCol& k, const float4& v) {
        return make_float4((v.x - k.mean.x) * k.istd.x, (v.y - k.mean.y) * k.istd.y, (v.z - k.mean.z) * k.istd.z,
                           (v.w - k.mean.w) * k.istd.w);
    }
    // with a residual the forward output was max(0, fma(x, a, b) + r): the same mask, bit for bit, and the gradient of
    // both the batch-norm output and the residual is dy masked by it, which is written out as dres (exact)
    __device__ __forceinline__ void gate(const BnCol& k, const float4& v, const float4& q, size_t o, float4& d) const {
        if (!(fmaf(v.x, k.a.x, k.b.x) + q.x > 0.f)) d.x = 0.f;
        if (!(fmaf(v.y, k.a.y, k.b.y) + q.y > 0.f)) d.y = 0.f;
        if (!(fmaf(v.z, k.a.z, k.b.z) + q.z > 0.f)) d.z = 0.f;
        if (!(fmaf(v.w, k.a.w, k.b.w) + q.w > 0.f)) d.w = 0.f;
        reinterpret_cast<V*>(p.dres)[o] = A::narrow(d);
    }
    // one row's term of a thread's private sums of dbeta and dgamma (d with a residual: already gated)
    __device__ __forceinline__ void acc(const BnCol& k, const float4& v, float4 d, float4& sb, float4& sg) const {
        const float4 xh = xhat(k, v);
        if constexpr (!kRes) mask(k, v, d);
        sb.x += d.x; sb.y += d.y; sb.z += d.z; sb.w += d.w;
        sg.x = fmaf(d.x, xh.x, sg.x); sg.y = fmaf(d.y, xh.y, sg.y); sg.z = fmaf(d.z, xh.z, sg.z); sg.w = fmaf(d.w, xh.w, sg.w);
    }
    __device__ __forceinline__ float4 over_m(const float4& t) const {
        const double M = (double)p.g.M;
        return make_float4((float)(t.x / M), (float)(t.y / M), (float)(t.z / M), (float)(t.w / M));
    }
    // dx at offset off from x = v and the gradient d, with mb = dbeta / M and mg = dgamma / M
    __device__ __forceinline__ void dx(const BnCol& k, const float4& mb, const float4& mg, size_t off, const float4& v,
                                       float4 d) const {
        const float4 xh = xhat(k, v);
        if constexpr (!kRes) mask(k, v, d);
        reinterpret_cast<V*>(p.dx)[off] =
            A::narrow(make_float4(k.a.x * (d.x - mb.x - xh.x * mg.x), k.a.y * (d.y - mb.y - xh.y * mg.y),
                                  k.a.z * (d.z - mb.z - xh.z * mg.z), k.a.w * (d.w - mb.w - xh.w * mg.w)));
    }
};


template <bool kPool, bool kRes, typename T>
__global__ void __launch_bounds__(kBnThreads) bn_bwd_kernel(const BnBwdArgs<T> p) {
    static_assert(!(kPool && kRes), "no pool follows a residual add");
    using A = Elem<T>;
    using V = typename A::V;
    extern __shared__ float4 s_dyn[];         // [2][cv] combine totals
    __shared__ float4 s_red[2 * kBnThreads];
    const BnGeom& g = p.g;
    const int tx = threadIdx.x % g.tpr, ty = threadIdx.x / g.tpr;
    const BnBwdElem<kPool, kRes, T> el{p};
    const V* x4 = reinterpret_cast<const V*>(p.x);
    const V* r4 = reinterpret_cast<const V*>(p.res);
    V* dr4 = reinterpret_cast<V*>(p.dres);
    auto ldx = [&](size_t o) { return A::wide(__ldg(x4 + o)); };
    auto ldr = [&](size_t o) { return A::wide(__ldg(r4 + o)); };
    const size_t st1 = (size_t)g.rpi * g.cv;
    V hx[kBnHold];                            // the CTA's first tile: x as stored
    float4 hd[kBnHold];                       // and the incoming gradient (with a pool: expanded at the arg-max; with a
                                              // residual: already masked)

    // (1) partials, eight or more independent 128-bit loads in flight per thread
    for (int t = blockIdx.x; t < g.nblk; t += gridDim.x) {
        const bool held = g.hold && t == (int)blockIdx.x;
        const int row0 = t * g.rows_per_block, row1 = min(g.M, row0 + g.rows_per_block);
        for (int c0 = 0; c0 < g.cv; c0 += g.tpr) {
            const int col = c0 + tx;
            float4 sb = make_float4(0.f, 0.f, 0.f, 0.f), sg = sb;
            if (ty < g.rpi && col < g.cv) {
                const BnCol k = el.column(col);
                auto acc = [&](const float4& v, const float4& d) { el.acc(k, v, d, sb, sg); };
                int r = row0 + ty;
                if (held) {
#pragma unroll
                    for (int j = 0; j < kBnHold; ++j) {
                        const int rr = r + j * g.rpi;
                        hx[j] = rr < row1 ? __ldg(x4 + (size_t)rr * g.cv + col) : V{};
                        hd[j] = rr < row1 ? el.grad(row0, rr, col) : make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                    if constexpr (kRes) {
#pragma unroll
                        for (int j = 0; j < kBnHold; ++j)
                            if (r + j * g.rpi < row1) {
                                const size_t o = (size_t)(r + j * g.rpi) * g.cv + col;
                                el.gate(k, A::wide(hx[j]), ldr(o), o, hd[j]);
                            }
                    }
#pragma unroll
                    for (int j = 0; j < kBnHold; ++j)
                        if (r + j * g.rpi < row1) acc(A::wide(hx[j]), hd[j]);
                } else {
                    for (; r + 3 * g.rpi < row1; r += 4 * g.rpi) {
                        const size_t o = (size_t)r * g.cv + col;
                        const float4 v0 = ldx(o), v1 = ldx(o + st1), v2 = ldx(o + 2 * st1), v3 = ldx(o + 3 * st1);
                        float4 e0 = el.grad(row0, r, col), e1 = el.grad(row0, r + g.rpi, col), e2 = el.grad(row0, r + 2 * g.rpi, col),
                               e3 = el.grad(row0, r + 3 * g.rpi, col);
                        if constexpr (kRes) {
                            const float4 q0 = ldr(o), q1 = ldr(o + st1), q2 = ldr(o + 2 * st1), q3 = ldr(o + 3 * st1);
                            el.gate(k, v0, q0, o, e0); el.gate(k, v1, q1, o + st1, e1);
                            el.gate(k, v2, q2, o + 2 * st1, e2); el.gate(k, v3, q3, o + 3 * st1, e3);
                        }
                        acc(v0, e0); acc(v1, e1); acc(v2, e2); acc(v3, e3);
                    }
                    for (; r < row1; r += g.rpi) {
                        if constexpr (kRes) {
                            const size_t o = (size_t)r * g.cv + col;
                            const float4 v = ldx(o);
                            float4 e = el.grad(row0, r, col);
                            el.gate(k, v, ldr(o), o, e);
                            acc(v, e);
                        } else {
                            acc(ldx((size_t)r * g.cv + col), el.grad(row0, r, col));
                        }
                    }
                }
            }
            bn_tile_partial(sb, sg, tx, ty, col, g, s_red, p.partial, t);
        }
    }

    // (2) one CTA combines and publishes dbeta, dgamma
    unsigned int gen;
    const bool last = bn_arrive(p.sync, gen);
    if (last) {
        float* s_tot = reinterpret_cast<float*>(s_dyn);
        bn_combine_partials(p.partial, g.nblk, g.C, s_tot, s_red);
        for (int c = threadIdx.x; c < g.C; c += kBnThreads) { p.dbeta[c] = s_tot[c]; p.dgamma[c] = s_tot[g.C + c]; }
    }
    bn_release(p.sync, last, gen);

    // (3) input gradient
    for (int t = blockIdx.x; t < g.nblk; t += gridDim.x) {
        const bool held = g.hold && t == (int)blockIdx.x;
        const int row0 = t * g.rows_per_block, row1 = min(g.M, row0 + g.rows_per_block);
        for (int c0 = 0; c0 < g.cv; c0 += g.tpr) {
            const int col = c0 + tx;
            if (ty >= g.rpi || col >= g.cv) continue;
            const BnCol k = el.column(col);
            const float4 db = __ldcg(reinterpret_cast<const float4*>(p.dbeta) + col);
            const float4 dg = __ldcg(reinterpret_cast<const float4*>(p.dgamma) + col);
            const float4 mb = el.over_m(db), mg = el.over_m(dg);
            auto out = [&](size_t off, const float4& v, const float4& d) { el.dx(k, mb, mg, off, v, d); };
            int r = row0 + ty;
            if (held) {
#pragma unroll
                for (int j = 0; j < kBnHold; ++j)
                    if (r + j * g.rpi < row1) out((size_t)(r + j * g.rpi) * g.cv + col, A::wide(hx[j]), hd[j]);
                continue;
            }
            // with a residual, the masked gradient is the dres this thread wrote in (1): a coherent load, not __ldg
            auto grad3 = [&](int r3) -> float4 {
                if constexpr (kRes) return A::wide(__ldcg(dr4 + (size_t)r3 * g.cv + col));
                else return el.grad(row0, r3, col);
            };
            for (; r + 3 * g.rpi < row1; r += 4 * g.rpi) {
                const size_t o = (size_t)r * g.cv + col;
                const float4 v0 = ldx(o), v1 = ldx(o + st1), v2 = ldx(o + 2 * st1), v3 = ldx(o + 3 * st1);
                const float4 e0 = grad3(r), e1 = grad3(r + g.rpi), e2 = grad3(r + 2 * g.rpi), e3 = grad3(r + 3 * g.rpi);
                out(o, v0, e0); out(o + st1, v1, e1); out(o + 2 * st1, v2, e2); out(o + 3 * st1, v3, e3);
            }
            for (; r < row1; r += g.rpi) out((size_t)r * g.cv + col, ldx((size_t)r * g.cv + col), grad3(r));
        }
    }
}

// Channel-sliced backward (g.sc > 0): the thread layout of bn_fwd_sliced_kernel.
template <bool kPool, bool kRes, typename T>
__global__ void __launch_bounds__(kBnThreads) bn_bwd_sliced_kernel(const BnBwdArgs<T> p) {
    static_assert(!(kPool && kRes), "no pool follows a residual add");
    using A = Elem<T>;
    using V = typename A::V;
    extern __shared__ float4 s_dyn[];         // bn_slice_reduce's scratch
    __shared__ float4 s_tot[2 * 8];           // [sc] dbeta | [sc] dgamma of the owned columns
    const BnGeom& g = p.g;
    const int sc = g.sc, cx = threadIdx.x % sc, ln = threadIdx.x / sc, col = blockIdx.x * sc + cx;
    const int row0 = ln / g.rpi * g.rows_per_block, row1 = min(g.M, row0 + g.rows_per_block), r = row0 + ln % g.rpi;
    const BnBwdElem<kPool, kRes, T> el{p};
    const V* x4 = reinterpret_cast<const V*>(p.x);
    const BnCol k = el.column(col);

    // (1) the thread's rows of x and of the gradient (pooled: expanded; residual: gated, dres written), held; their sums
    V hx[kBnHold];
    float4 hd[kBnHold];
    float4 sb = make_float4(0.f, 0.f, 0.f, 0.f), sg = sb;
#pragma unroll
    for (int j = 0; j < kBnHold; ++j) {
        const int rr = r + j * g.rpi;
        hx[j] = rr < row1 ? __ldg(x4 + (size_t)rr * g.cv + col) : V{};
        hd[j] = rr < row1 ? el.grad(0, rr, col) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if constexpr (kRes) {
        const V* r4 = reinterpret_cast<const V*>(p.res);
#pragma unroll
        for (int j = 0; j < kBnHold; ++j)
            if (r + j * g.rpi < row1) {
                const size_t o = (size_t)(r + j * g.rpi) * g.cv + col;
                el.gate(k, A::wide(hx[j]), A::wide(__ldg(r4 + o)), o, hd[j]);
            }
    }
#pragma unroll
    for (int j = 0; j < kBnHold; ++j)
        if (r + j * g.rpi < row1) el.acc(k, A::wide(hx[j]), hd[j], sb, sg);

    // (2) dbeta, dgamma of the owned columns
    bn_slice_reduce(sb, sg, g, s_dyn, s_tot);
    if (threadIdx.x < sc) {
        reinterpret_cast<float4*>(p.dbeta)[blockIdx.x * sc + threadIdx.x] = s_tot[threadIdx.x];
        reinterpret_cast<float4*>(p.dgamma)[blockIdx.x * sc + threadIdx.x] = s_tot[sc + threadIdx.x];
    }

    // (3) input gradient
    const float4 mb = el.over_m(s_tot[cx]), mg = el.over_m(s_tot[sc + cx]);
#pragma unroll
    for (int j = 0; j < kBnHold; ++j)
        if (r + j * g.rpi < row1) el.dx(k, mb, mg, (size_t)(r + j * g.rpi) * g.cv + col, A::wide(hx[j]), hd[j]);
}

// ---------------------------------------------------------------------------------------------- launchers
int bn_tile_rows(int M, int C) { return bn_geom(M, C).rows_per_block; }

// Whether a call without a grid cap runs the channel-sliced kernels.  A pool of width W > 0 only has to be one the fused
// kernels take at all: a pooled slice's y, M * sc float4, never exceeds kBnHold * kBnThreads of them (32 KB).
bool bn_sliced(int M, int C, int W) { return bn_geom(M, C).sc > 0 && (W == 0 || (W % 2 == 0 && M % (2 * W) == 0)); }

static unsigned int* bn_sync_slot(int slot) {
    static unsigned int* base[64] = {nullptr};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return nullptr;
    if (base[dev] == nullptr) {
        void* a = nullptr;
        if (cudaGetSymbolAddress(&a, g_bn_sync) != cudaSuccess) return nullptr;
        base[dev] = static_cast<unsigned int*>(a);
    }
    return base[dev] + 2 * (size_t)(slot % kBnSyncSlots);
}

// Cooperative launch of min(tiles, co-resident CTAs [, max_ctas]) CTAs.
template <typename Args>
static cudaError_t bn_launch(void (*kernel)(const Args), Args p, size_t smem, int max_ctas, cudaStream_t stream) {
    int dev = 0, sms = 0, per = 0;
    cudaGetDevice(&dev);
    cudaError_t e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess && smem > 32 * 1024)
        e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, kernel, kBnThreads, smem);
    if (e != cudaSuccess) return e;
    if (per < 1) return cudaErrorInvalidConfiguration;
    int grid = p.g.nblk < per * sms ? p.g.nblk : per * sms;
    if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
    void* args[] = {(void*)&p};
    e = cudaLaunchCooperativeKernel((void*)kernel, dim3(grid), dim3(kBnThreads), args, smem, stream);
    (void)cudaGetLastError();       // a failed launch must not surface again at the next launcher's error check
    return e;
}

// Plain launch of a channel-sliced kernel: cv / sc CTAs of sc * nblk * rpi threads; `stage`: bytes of the pooled y.
template <typename Args>
static cudaError_t bn_launch_sliced(void (*kernel)(const Args), const Args& p, size_t stage, cudaStream_t stream) {
    const BnGeom& g = p.g;
    const int threads = g.sc * g.nblk * g.rpi;
    size_t smem = sizeof(float4) * (2 * threads + 2 * g.nblk * g.sc);           // bn_slice_reduce's scratch
    if (smem < stage) smem = stage;
    kernel<<<g.cv / g.sc, threads, smem, stream>>>(p);
    return cudaGetLastError();
}

static cudaError_t bn_prepare(BnGeom& g, unsigned int*& sync, int M, int C, int W, int slot) {
    g = bn_geom(M, C);
    g.W = W;
    if (W > 0 && (W % 2 != 0 || g.rows_per_block % (2 * W) != 0 || M % (2 * W) != 0)) return cudaErrorInvalidValue;
    sync = bn_sync_slot(slot);
    return sync == nullptr ? cudaErrorInvalidDevice : cudaSuccess;
}

template <typename T>
static cudaError_t bn_forward_t(const void* x, void* y, unsigned char* arg, float* partial, const float* gamma,
                                const float* beta, const float* cbias, float* save_mean, float* save_invstd, float* rmean,
                                float* rvar, long long* nbt, float momentum, float eps, int relu, int M, int C, int W, int slot,
                                int max_ctas, cudaStream_t stream, const void* res) {
    if (res != nullptr && (W > 0 || !relu)) return cudaErrorInvalidValue;      // a residual is always followed by the ReLU
    BnFwdArgs<T> p{static_cast<const T*>(x), static_cast<T*>(y), arg, partial, gamma, beta, cbias, save_mean, save_invstd,
                   rmean, rvar, nbt, momentum, eps, relu, nullptr, {}, static_cast<const T*>(res)};
    cudaError_t e = bn_prepare(p.g, p.sync, M, C, W, slot);
    if (e != cudaSuccess) return e;
    if (p.g.sc > 0 && max_ctas <= 0) {           // a grid cap asks for the cooperative kernels' loop over tiles
        if (W > 0) return bn_launch_sliced(bn_fwd_sliced_kernel<true, false, T>, p, sizeof(float4) * M * p.g.sc, stream);
        return res != nullptr ? bn_launch_sliced(bn_fwd_sliced_kernel<false, true, T>, p, 0, stream)
                              : bn_launch_sliced(bn_fwd_sliced_kernel<false, false, T>, p, 0, stream);
    }
    size_t smem = sizeof(float) * 2 * C;
    if (W > 0 && p.g.hold) smem += sizeof(float4) * p.g.rows_per_block * p.g.cv;
    if (W > 0) return bn_launch(bn_fwd_kernel<true, false, T>, p, smem, max_ctas, stream);
    return res != nullptr ? bn_launch(bn_fwd_kernel<false, true, T>, p, smem, max_ctas, stream)
                          : bn_launch(bn_fwd_kernel<false, false, T>, p, smem, max_ctas, stream);
}

template <typename T>
static cudaError_t bn_backward_t(const void* x, const void* dy, const unsigned char* arg, void* dx, float* partial,
                                 const float* gamma, const float* beta, const float* save_mean, const float* save_invstd,
                                 float* dgamma, float* dbeta, int relu, int M, int C, int W, int slot, int max_ctas,
                                 cudaStream_t stream, const void* res, void* dres) {
    if ((res == nullptr) != (dres == nullptr) || (res != nullptr && (W > 0 || !relu))) return cudaErrorInvalidValue;
    BnBwdArgs<T> p{static_cast<const T*>(x), static_cast<const T*>(dy), arg, static_cast<T*>(dx), partial, gamma, beta,
                   save_mean, save_invstd, dgamma, dbeta, relu, nullptr, {}, static_cast<const T*>(res),
                   static_cast<T*>(dres)};
    cudaError_t e = bn_prepare(p.g, p.sync, M, C, W, slot);
    if (e != cudaSuccess) return e;
    if (p.g.sc > 0 && max_ctas <= 0) {
        if (W > 0) return bn_launch_sliced(bn_bwd_sliced_kernel<true, false, T>, p, 0, stream);
        return res != nullptr ? bn_launch_sliced(bn_bwd_sliced_kernel<false, true, T>, p, 0, stream)
                              : bn_launch_sliced(bn_bwd_sliced_kernel<false, false, T>, p, 0, stream);
    }
    const size_t smem = sizeof(float) * 2 * C;
    if (W > 0) return bn_launch(bn_bwd_kernel<true, false, T>, p, smem, max_ctas, stream);
    return res != nullptr ? bn_launch(bn_bwd_kernel<false, true, T>, p, smem, max_ctas, stream)
                          : bn_launch(bn_bwd_kernel<false, false, T>, p, smem, max_ctas, stream);
}

cudaError_t launch_bn_forward(const void* x, void* y, unsigned char* arg, float* partial, const float* gamma, const float* beta,
                              const float* cbias, float* save_mean, float* save_invstd, float* rmean, float* rvar, long long* nbt,
                              float momentum, float eps, int relu, int M, int C, int W, int slot, int max_ctas, Dtype dtype,
                              cudaStream_t stream, const void* res) {
    return with_dtype(dtype, [&](auto e) {
        return bn_forward_t<decltype(e)>(x, y, arg, partial, gamma, beta, cbias, save_mean, save_invstd, rmean, rvar, nbt,
                                         momentum, eps, relu, M, C, W, slot, max_ctas, stream, res);
    });
}

cudaError_t launch_bn_backward(const void* x, const void* dy, const unsigned char* arg, void* dx, float* partial,
                               const float* gamma, const float* beta, const float* save_mean, const float* save_invstd,
                               float* dgamma, float* dbeta, int relu, int M, int C, int W, int slot, int max_ctas, Dtype dtype,
                               cudaStream_t stream, const void* res, void* dres) {
    return with_dtype(dtype, [&](auto e) {
        return bn_backward_t<decltype(e)>(x, dy, arg, dx, partial, gamma, beta, save_mean, save_invstd, dgamma, dbeta,
                                          relu, M, C, W, slot, max_ctas, stream, res, dres);
    });
}

}  // namespace okt

// ==============================================================================================================
// 2x2 / stride-2 max pooling, channels_last fp32, forward + backward.
// The stock NHWC pooling kernels take 11-13 us per call on the VGG activations (16x32x32x64 ... 16x2x2x512) plus a
// zero-fill of the input gradient; the windows of a stride-2 2x2 pool do not overlap, so the backward pass can WRITE all
// four positions of every window (gradient at the arg-max, zeros elsewhere) without atomics or a memset.  One thread =
// one output pixel x 4 channels (128-bit accesses); the arg-max (first maximum in row-major window order, like
// at::max_pool2d) is kept as one byte per output element.
// ==============================================================================================================
namespace okt {

constexpr int kPoolThreads = 256;

__global__ void __launch_bounds__(kPoolThreads) maxpool2_fwd_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                     unsigned char* __restrict__ arg, int N, int H, int W,
                                                                     int C) {
    const int cv = C >> 2, Ho = H >> 1, Wo = W >> 1;
    const long long total = (long long)N * Ho * Wo * cv;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    float4* y4 = reinterpret_cast<float4*>(y);
    uchar4* a4 = reinterpret_cast<uchar4*>(arg);
    for (long long t = (long long)blockIdx.x * kPoolThreads + threadIdx.x; t < total; t += (long long)gridDim.x * kPoolThreads) {
        const int c = (int)(t % cv);
        long long p = t / cv;
        const int wo = (int)(p % Wo); p /= Wo;
        const int ho = (int)(p % Ho);
        const int n = (int)(p / Ho);
        const size_t base = (((size_t)n * H + 2 * ho) * W + 2 * wo) * cv + c;
        const float4 v0 = __ldg(x4 + base), v1 = __ldg(x4 + base + cv);
        const float4 v2 = __ldg(x4 + base + (size_t)W * cv), v3 = __ldg(x4 + base + (size_t)W * cv + cv);
        float4 m = v0;
        uchar4 a = make_uchar4(0, 0, 0, 0);
        pool_step(m, a, v1, 1);
        pool_step(m, a, v2, 2);
        pool_step(m, a, v3, 3);
        y4[t] = m;
        a4[t] = a;
    }
}

__global__ void __launch_bounds__(kPoolThreads) maxpool2_bwd_kernel(const float* __restrict__ dy,
                                                                     const unsigned char* __restrict__ arg,
                                                                     float* __restrict__ dx, int N, int H, int W, int C) {
    const int cv = C >> 2, Ho = H >> 1, Wo = W >> 1;
    const long long total = (long long)N * Ho * Wo * cv;
    const float4* d4 = reinterpret_cast<const float4*>(dy);
    const uchar4* a4 = reinterpret_cast<const uchar4*>(arg);
    float4* o4 = reinterpret_cast<float4*>(dx);
    for (long long t = (long long)blockIdx.x * kPoolThreads + threadIdx.x; t < total; t += (long long)gridDim.x * kPoolThreads) {
        const int c = (int)(t % cv);
        long long p = t / cv;
        const int wo = (int)(p % Wo); p /= Wo;
        const int ho = (int)(p % Ho);
        const int n = (int)(p / Ho);
        const size_t base = (((size_t)n * H + 2 * ho) * W + 2 * wo) * cv + c;
        const float4 d = __ldg(d4 + t);
        const uchar4 a = a4[t];
        auto pick = [&](int k) {
            return make_float4(a.x == k ? d.x : 0.f, a.y == k ? d.y : 0.f, a.z == k ? d.z : 0.f, a.w == k ? d.w : 0.f);
        };
        o4[base] = pick(0);
        o4[base + cv] = pick(1);
        o4[base + (size_t)W * cv] = pick(2);
        o4[base + (size_t)W * cv + cv] = pick(3);
    }
}

static inline int pool_grid(long long total) {
    long long g = (total + kPoolThreads - 1) / kPoolThreads;
    if (g < 1) g = 1;
    if (g > kStrideGridMax) g = kStrideGridMax;
    return (int)g;
}

cudaError_t launch_maxpool2_fwd(const float* x, float* y, unsigned char* arg, int N, int H, int W, int C, cudaStream_t stream) {
    const long long total = (long long)N * (H / 2) * (W / 2) * (C / 4);
    maxpool2_fwd_kernel<<<pool_grid(total), kPoolThreads, 0, stream>>>(x, y, arg, N, H, W, C);
    return cudaGetLastError();
}
cudaError_t launch_maxpool2_bwd(const float* dy, const unsigned char* arg, float* dx, int N, int H, int W, int C,
                                cudaStream_t stream) {
    const long long total = (long long)N * (H / 2) * (W / 2) * (C / 4);
    maxpool2_bwd_kernel<<<pool_grid(total), kPoolThreads, 0, stream>>>(dy, arg, dx, N, H, W, C);
    return cudaGetLastError();
}

}  // namespace okt
