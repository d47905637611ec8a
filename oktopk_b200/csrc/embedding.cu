// Fused embedding sum + LayerNorm + dropout of BERT's input block, training mode, forward and backward:
//
//   e = (word[id] + pos[s]) + typ[tt]         (token r = b S + s; the stock order of the two adds)
//   y = keep . s . ((e - mean) . rstd . gamma + beta),   rstd = 1/sqrt(var + eps), var biased (as F.layer_norm)
//
// Stock ops spend three gathers, two adds, layer_norm and a dropout that stores its mask forward, and dropout,
// layer_norm backward and three embedding_dense_backward calls (each a sort, segment sums and a zero-filled dense table
// gradient) backward.  Here it is one kernel forward and three backward, and neither e nor the mask is stored: the
// backward pass regenerates the mask from the seed and recomputes e from the tables and the ids.
//
// Layout: ids and tt are [R] int64 (R = B S, the [B, S] id matrices flattened), word [nv, H], pos [np, H], typ [nt, H],
// y, dy and de [R, H], all fp32 and row-major, H a multiple of 128 up to 1024 (templated on V = H/128).  The row kernels
// deal one token row to one warp, lane l holding the float4 columns 4 (32 j + l) .. +3 for j < V, as in layernorm.cu,
// and take the row statistics the way ln_fwd_kernel does (the mean, then the mean squared deviation from it).
//
// Dropout: the scheme of layernorm.cu (devlib.cuh, ln_keep) over the element index r H + c of y.
//
// Ids out of range: an id outside [0, nv) or a type outside [0, nt) is never used as an address.  Its table row
// contributes 0 to e and receives no gradient, and the forward pass adds one per such index to *ovf (an integer
// atomic; the count, not the order, is all that is kept).
//
// Backward, in launch order:
//  1. emb_bwd_kernel: de = rstd (dxhat - mean(dxhat) - xhat mean(dxhat xhat)), dxhat = dy keep s gamma, and the
//     per-CTA dgamma / dbeta partials of ln_bwd_kernel;  2. ln_dgb_kernel (layernorm.cu) adds the partials in a fixed
//     order.
//  3. emb_tables_kernel writes every element of the three table gradients once.  Each CTA owns a range of rows of one
//     table and lists the tokens of each of its rows, in token order, by a stable counting sort of the R <= 4096 row
//     indices in shared memory (no global sort, no workspace).  A row's gradient is the sum of de over its list, added
//     in that order from +0, or exactly 0 for an empty list: the word rows of the ids present, the position rows s < S
//     (the tokens b S + s in b order), the token-type rows; every other row is 0.  There is no memset and no float
//     atomic, every sum runs in an order fixed by the ids alone, and the grids depend on R, S, H and the table sizes
//     only: the results are bitwise reproducible.  A row of one token is that token's de exactly.
#include "common.cuh"
#include "devlib.cuh"
#include "oktopk.cuh"

namespace okt {

constexpr int kEmbWarps = 4;                   // rows in flight per CTA of the row kernels
constexpr int kEmbThreads = 32 * kEmbWarps;
constexpr int kEmbFwdMaxBlocks = 8192;
constexpr int kEmbMaxTokens = 4096;            // R = B S, bounded by emb_tables_kernel's shared memory
constexpr int kEmbTgWarps = 8;
constexpr int kEmbTgThreads = 32 * kEmbTgWarps;
constexpr int kEmbTgRows = 64;                 // word / position rows per CTA of emb_tables_kernel
constexpr int kEmbBatch = 16;                  // de rows in flight per lane in the ordered sums

struct EmbRow {
    const float* w;                            // null: the id is out of range
    const float* p;
    const float* t;                            // null: the type is out of range
    int bad;                                   // how many of the two indices are out of range
};

__device__ __forceinline__ EmbRow emb_row(const long long* ids, const long long* tt, const float* word, const float* pos,
                                          const float* typ, int row, int S, int H, int nv, int nt) {
    const long long id = __ldg(ids + row), t = __ldg(tt + row);
    const bool iok = id >= 0 && id < nv, tok = t >= 0 && t < nt;
    EmbRow q;
    q.w = iok ? word + (size_t)id * H : nullptr;
    q.p = pos + (size_t)(row % S) * H;
    q.t = tok ? typ + (size_t)t * H : nullptr;
    q.bad = (int)!iok + (int)!tok;
    return q;
}

// e at one lane's float4 column; the forward and backward passes share it, so e is bitwise the same in both
__device__ __forceinline__ float4 emb_e(const EmbRow& q, int col) {
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 w = q.w ? __ldg(reinterpret_cast<const float4*>(q.w + col)) : z;
    const float4 p = __ldg(reinterpret_cast<const float4*>(q.p + col));
    const float4 t = q.t ? __ldg(reinterpret_cast<const float4*>(q.t + col)) : z;
    return make_float4((w.x + p.x) + t.x, (w.y + p.y) + t.y, (w.z + p.z) + t.z, (w.w + p.w) + t.w);
}

__device__ __forceinline__ float4 add4(float4 a, float4 b) {
    return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}

template <int V>
__global__ void __launch_bounds__(kEmbThreads) emb_fwd_kernel(const long long* __restrict__ ids,
                                                              const long long* __restrict__ tt,
                                                              const float* __restrict__ word, const float* __restrict__ pos,
                                                              const float* __restrict__ typ,
                                                              const float* __restrict__ gamma,
                                                              const float* __restrict__ beta, float* __restrict__ y,
                                                              float* __restrict__ stats, long long* ovf,
                                                              const unsigned long long* seed, int R, int S, int nv, int nt,
                                                              long long keep_thr, float scale, float eps) {
    constexpr int H = 128 * V;
    const int lane = lane_id();
    const LnDrop d = ln_drop(seed, keep_thr, scale);
    for (int row = blockIdx.x * kEmbWarps + (threadIdx.x >> 5); row < R; row += gridDim.x * kEmbWarps) {
        const EmbRow q = emb_row(ids, tt, word, pos, typ, row, S, H, nv, nt);
        const size_t base = (size_t)row * H;
        float4 z[V];
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < V; ++j) {
            z[j] = emb_e(q, (j * 32 + lane) * 4);
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
            const float4 m = ln_mult(d, ln_keep(d, base + col));
            *reinterpret_cast<float4*>(y + base + col) =
                make_float4(fmaf(z[j].x * rs, g.x, b.x) * m.x, fmaf(z[j].y * rs, g.y, b.y) * m.y,
                            fmaf(z[j].z * rs, g.z, b.z) * m.z, fmaf(z[j].w * rs, g.w, b.w) * m.w);
        }
        if (lane == 0) {
            stats[row] = mu;
            stats[R + row] = rs;
            if (q.bad && ovf) atomicAdd(reinterpret_cast<unsigned long long*>(ovf), (unsigned long long)q.bad);
        }
    }
}

// (minimum 1 CTA per SM, as ln_bwd_kernel)
template <int V>
__global__ void __launch_bounds__(kEmbThreads, 1) emb_bwd_kernel(const long long* __restrict__ ids,
                                                                 const long long* __restrict__ tt,
                                                                 const float* __restrict__ word,
                                                                 const float* __restrict__ pos,
                                                                 const float* __restrict__ typ,
                                                                 const float* __restrict__ gamma,
                                                                 const float* __restrict__ stats,
                                                                 const float* __restrict__ dy,
                                                                 const unsigned long long* seed, float* __restrict__ de,
                                                                 float* __restrict__ partial, int R, int S, int nv, int nt,
                                                                 long long keep_thr, float scale) {
    constexpr int H = 128 * V;
    __shared__ float4 s_part[2 * H / 4];                  // [dgamma | dbeta] of this CTA's rows
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    const LnDrop d = ln_drop(seed, keep_thr, scale);
    float4 pg[V], pb[V];
#pragma unroll
    for (int j = 0; j < V; ++j) pg[j] = pb[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int row = blockIdx.x * kEmbWarps + warp; row < R; row += gridDim.x * kEmbWarps) {
        const EmbRow q = emb_row(ids, tt, word, pos, typ, row, S, H, nv, nt);
        const size_t base = (size_t)row * H;
        const float mu = stats[row], rs = stats[R + row];
        float4 xh[V], g[V];
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int j = 0; j < V; ++j) {
            const int col = (j * 32 + lane) * 4;
            const float4 e = emb_e(q, col);
            xh[j] = make_float4((e.x - mu) * rs, (e.y - mu) * rs, (e.z - mu) * rs, (e.w - mu) * rs);
            const float4 m = ln_mult(d, ln_keep(d, base + col));
            const float4 dv = *reinterpret_cast<const float4*>(dy + base + col);
            const float4 dyv = make_float4(dv.x * m.x, dv.y * m.y, dv.z * m.z, dv.w * m.w);   // through the dropout
            const float4 gm = __ldg(reinterpret_cast<const float4*>(gamma + col));
            g[j] = make_float4(dyv.x * gm.x, dyv.y * gm.y, dyv.z * gm.z, dyv.w * gm.w);
            s1 += (g[j].x + g[j].y) + (g[j].z + g[j].w);
            s2 += (g[j].x * xh[j].x + g[j].y * xh[j].y) + (g[j].z * xh[j].z + g[j].w * xh[j].w);
            pg[j] = make_float4(fmaf(dyv.x, xh[j].x, pg[j].x), fmaf(dyv.y, xh[j].y, pg[j].y), fmaf(dyv.z, xh[j].z, pg[j].z),
                                fmaf(dyv.w, xh[j].w, pg[j].w));
            pb[j] = add4(pb[j], dyv);
        }
        const float c1 = warp_sum_f(s1) / (float)H, c2 = warp_sum_f(s2) / (float)H;
#pragma unroll
        for (int j = 0; j < V; ++j) {
            const int col = (j * 32 + lane) * 4;
            *reinterpret_cast<float4*>(de + base + col) =
                make_float4(rs * (g[j].x - c1 - xh[j].x * c2), rs * (g[j].y - c1 - xh[j].y * c2),
                            rs * (g[j].z - c1 - xh[j].z * c2), rs * (g[j].w - c1 - xh[j].w * c2));
        }
    }
    // the CTA's column partials, warps added in warp order
    for (int w = 0; w < kEmbWarps; ++w) {
        if (warp == w) {
#pragma unroll
            for (int j = 0; j < V; ++j) {
                const int c4 = j * 32 + lane;
                if (w == 0) {
                    s_part[c4] = pg[j];
                    s_part[H / 4 + c4] = pb[j];
                } else {
                    s_part[c4] = add4(s_part[c4], pg[j]);
                    s_part[H / 4 + c4] = add4(s_part[H / 4 + c4], pb[j]);
                }
            }
        }
        __syncthreads();
    }
    float4* out = reinterpret_cast<float4*>(partial) + (size_t)blockIdx.x * (2 * H / 4);
    for (int c4 = threadIdx.x; c4 < 2 * H / 4; c4 += kEmbThreads) out[c4] = s_part[c4];
}

// The sum of de's rows row_of(0), ..., row_of(n - 1) at float4 column col, added in that order from +0, kEmbBatch
// loads in flight.
template <class RowOf>
__device__ __forceinline__ float4 emb_sum_rows(const float* de, int H, int col, int n, RowOf row_of) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int k0 = 0; k0 < n; k0 += kEmbBatch) {
        float4 v[kEmbBatch];
#pragma unroll
        for (int k = 0; k < kEmbBatch; ++k)
            if (k0 + k < n) v[k] = __ldcg(reinterpret_cast<const float4*>(de + (size_t)row_of(k0 + k) * H + col));
#pragma unroll
        for (int k = 0; k < kEmbBatch; ++k)
            if (k0 + k < n) acc = add4(acc, v[k]);
    }
    return acc;
}

// CTA roles, in blockIdx order: nt V token-type CTAs (row b / V, float4 column chunk b % V: the longest sums start
// first and spread over SMs), then the position CTAs and the word CTAs, kEmbTgRows rows and all columns each.  Every
// CTA first lists the tokens of each of its rows in token order (a stable counting sort in shared memory: warp 0 walks
// the tokens 32 at a time and ranks equal rows with __match_any_sync), then its warps write the (row, column chunk)
// sums.
template <int V>
__global__ void __launch_bounds__(kEmbTgThreads) emb_tables_kernel(const float* __restrict__ de,
                                                                   const long long* __restrict__ ids,
                                                                   const long long* __restrict__ tt, int R, int S, int nv,
                                                                   int np, int nt, float* __restrict__ dword,
                                                                   float* __restrict__ dpos, float* __restrict__ dtyp) {
    constexpr int H = 128 * V;
    __shared__ int s_row[kEmbMaxTokens];                  // each token's row in this CTA's range, or -1
    __shared__ int s_tok[kEmbMaxTokens];                  // the tokens grouped by row, each group in token order
    __shared__ int s_start[kEmbTgRows + 1], s_cur[kEmbTgRows];
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    int b = blockIdx.x, table, r0, nrows, j0, nj;
    if (b < nt * V) {
        table = 2; r0 = b / V; nrows = 1; j0 = b % V; nj = 1;
    } else {
        b -= nt * V;
        const int npc = (np + kEmbTgRows - 1) / kEmbTgRows;
        table = b < npc ? 1 : 0;
        r0 = (b < npc ? b : b - npc) * kEmbTgRows;
        nrows = min(kEmbTgRows, (b < npc ? np : nv) - r0);
        j0 = 0; nj = V;
    }
    for (int r = threadIdx.x; r < R; r += kEmbTgThreads) {
        const long long x = table == 0 ? ids[r] : (table == 1 ? (long long)(r % S) : tt[r]);
        const long long i = x - r0;                       // x < 0 or past the table never lands in [0, nrows)
        s_row[r] = (i >= 0 && i < nrows) ? (int)i : -1;
    }
    if (threadIdx.x < kEmbTgRows) s_cur[threadIdx.x] = 0;
    __syncthreads();
    if (warp == 0) {
        const unsigned lt = (1u << lane) - 1u;
        for (int c0 = 0; c0 < R; c0 += 32) {              // rows' token counts
            const int i = c0 + lane < R ? s_row[c0 + lane] : -1;
            const unsigned m = __match_any_sync(0xffffffffu, i);
            if (i >= 0 && (m & lt) == 0) s_cur[i] += __popc(m);
            __syncwarp();
        }
        const int ca = s_cur[2 * lane], cb = s_cur[2 * lane + 1];
        int inc = ca + cb;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int x = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += x;
        }
        const int ex = inc - ca - cb;
        s_start[2 * lane] = s_cur[2 * lane] = ex;
        s_start[2 * lane + 1] = s_cur[2 * lane + 1] = ex + ca;
        if (lane == 31) s_start[kEmbTgRows] = inc;
        __syncwarp();
        for (int c0 = 0; c0 < R; c0 += 32) {              // stable placement
            const int r = c0 + lane;
            const int i = r < R ? s_row[r] : -1;
            const unsigned m = __match_any_sync(0xffffffffu, i);
            if (i >= 0) s_tok[s_cur[i] + __popc(m & lt)] = r;
            __syncwarp();
            if (i >= 0 && (m & lt) == 0) s_cur[i] += __popc(m);
            __syncwarp();
        }
    }
    __syncthreads();
    float* out = table == 0 ? dword : (table == 1 ? dpos : dtyp);
    for (int it = warp; it < nrows * nj; it += kEmbTgWarps) {
        const int i = it / nj, col = ((j0 + it % nj) * 32 + lane) * 4;
        const int st = s_start[i];
        const float4 acc = emb_sum_rows(de, H, col, s_start[i + 1] - st, [&](int k) { return s_tok[st + k]; });
        *reinterpret_cast<float4*>(out + (size_t)(r0 + i) * H + col) = acc;
    }
}

bool emb_supported(int R, int S, int H, int np) {
    return R > 0 && R <= kEmbMaxTokens && S > 0 && R % S == 0 && S <= np && ln_supported_h(H);
}

static bool emb_args_ok(int R, int S, int H, int np, int nv, int nt, long long keep_thr, const unsigned long long* seed) {
    return emb_supported(R, S, H, np) && nv > 0 && nt > 0 && keep_thr >= 0 && keep_thr <= kLnKeepAll &&
           (keep_thr == kLnKeepAll || seed != nullptr);
}

cudaError_t launch_emb_forward(const long long* ids, const long long* tt, const float* word, const float* pos,
                               const float* typ, const float* gamma, const float* beta, float* y, float* stats,
                               long long* ovf, const unsigned long long* seed, int R, int S, int H, int nv, int nt,
                               long long keep_thr, float scale, float eps, cudaStream_t stream) {
    if (!emb_args_ok(R, S, H, S, nv, nt, keep_thr, seed)) return cudaErrorInvalidValue;
    const long long nb = ((long long)R + kEmbWarps - 1) / kEmbWarps;
    const int grid = (int)(nb > kEmbFwdMaxBlocks ? kEmbFwdMaxBlocks : nb);
    switch (H / 128) {
#define OKT_EMB_FWD(V) case V: emb_fwd_kernel<V><<<grid, kEmbThreads, 0, stream>>>(ids, tt, word, pos, typ, gamma, beta, y, \
                                                                                   stats, ovf, seed, R, S, nv, nt, keep_thr,  \
                                                                                   scale, eps); break;
        OKT_EMB_FWD(1) OKT_EMB_FWD(2) OKT_EMB_FWD(3) OKT_EMB_FWD(4) OKT_EMB_FWD(5) OKT_EMB_FWD(6) OKT_EMB_FWD(7)
        OKT_EMB_FWD(8)
#undef OKT_EMB_FWD
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

cudaError_t launch_emb_backward(const long long* ids, const long long* tt, const float* word, const float* pos,
                                const float* typ, const float* gamma, const float* stats, const float* dy,
                                const unsigned long long* seed, float* de, float* partial, float* dgamma,
                                float* dbeta, float* dword, float* dpos, float* dtyp, int R, int S, int H, int nv, int np,
                                int nt, long long keep_thr, float scale, cudaStream_t stream) {
    if (!emb_args_ok(R, S, H, np, nv, nt, keep_thr, seed)) return cudaErrorInvalidValue;
    cudaError_t e;
    const int grid = ln_bwd_grid(R);
    const int tg_grid = nt * (H / 128) + (np + kEmbTgRows - 1) / kEmbTgRows + (nv + kEmbTgRows - 1) / kEmbTgRows;
    switch (H / 128) {
#define OKT_EMB_BWD(V) case V:                                                                                            \
        emb_bwd_kernel<V><<<grid, kEmbThreads, 0, stream>>>(ids, tt, word, pos, typ, gamma, stats, dy, seed, de, partial, \
                                                            R, S, nv, nt, keep_thr, scale);                              \
        if ((e = cudaGetLastError()) != cudaSuccess) return e;                                                            \
        if ((e = launch_ln_dgb(partial, grid, H, dgamma, dbeta, stream)) != cudaSuccess) return e;                       \
        emb_tables_kernel<V><<<tg_grid, kEmbTgThreads, 0, stream>>>(de, ids, tt, R, S, nv, np, nt, dword, dpos, dtyp);   \
        break;
        OKT_EMB_BWD(1) OKT_EMB_BWD(2) OKT_EMB_BWD(3) OKT_EMB_BWD(4) OKT_EMB_BWD(5) OKT_EMB_BWD(6) OKT_EMB_BWD(7)
        OKT_EMB_BWD(8)
#undef OKT_EMB_BWD
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

}  // namespace okt
