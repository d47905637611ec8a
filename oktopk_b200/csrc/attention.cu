// Fused self-attention for BERT's encoder layers, head dim D = 64, forward and backward, on the tensor cores:
//
//   s_ij = (q_i . k_j) / sqrt(D) + m_bj,   P_ij = softmax_j(s_ij),   O_i = sum_j keep(b,h,i,j) / (1-p) . P_ij . v_j
//
// what F.scaled_dot_product_attention(q, k, v, attn_mask=m, dropout_p=p) computes with a [B, 1, 1, S] additive key mask.
// Q, K and V are read straight out of the packed projection qkv [B, S, 3, H, D] (row stride 3 H D), the output goes
// straight to [B, S, H D] and the gradient straight to one [B, S, 3 H D] d(qkv): no permute copies.
//
// Tiling (FlashAttention-2): a CTA of 4 warps owns 64 rows of one (sequence, head); each warp owns 16 of them and every
// product is a warp-level mma.sync over 64-wide tiles staged in shared memory.  The forward pass (one CTA per query
// block) keeps a running row max, sum and fp32 accumulator over the key blocks and writes O and each row's final max m
// and log2 l of its sum (base 2: m + log2 l = log2 sum_j 2^(s_ij log2 e)); no S x S tensor is stored.  The two are kept
// apart because a row's max can be as large as the mask makes it, and m + log2 l in fp32 would then lose log2 l.  The
// backward pass recomputes P = 2^((s log2 e - m) - log2 l) in two kernels, each writing every element it owns exactly
// once, with no atomics:
//   attn_bwd_dq_kernel  (one CTA per query block): Delta_i = dO_i . O_i (written out), then over the key blocks
//                        dS = P o (dP o M - Delta) with dP = dO V^T, and dQ = sum dS K / sqrt(D);
//   attn_bwd_dkv_kernel (one CTA per key block, after it): over the query blocks, with S^T and dP^T,
//                        dV = sum (P o M)^T dO and dK = sum dS^T Q / sqrt(D).
// M = keep / (1-p) is the dropout multiplier; rowsum(dP o P) = Delta because O = (P o M) V.  Every sum runs in a fixed
// order set by the shapes alone, so the results are bitwise reproducible.
//
// Products: bf16 and fp16 use mma.sync m16n8k16 with fp32 accumulation; P and dS are rounded to the operand type before
// their products, as any 16-bit attention kernel does.  fp32 uses 3xTF32 (m16n8k8): each operand is split into a TF32
// high part and a TF32 remainder and a.b ~ ah.bh + ah.bl + al.bh, which keeps about fp32 accuracy (the dropped al.bl
// is below 2^-22 relative) at three tensor-core products instead of CUDA-core FMAs, the route torch's
// memory-efficient kernel takes for fp32.  The accumulator fragment of m16n8k8 and m16n8k16 is the same
// (c0, c1 at row g, columns 2t, 2t+1; c2, c3 at row g + 8), so one kernel body serves all three types; for TF32 the
// k slots t and t + 4 of a fragment are mapped onto columns 2t and 2t + 1 (a contraction does not care about k order),
// which lets P and dS go from an accumulator straight into the next product's A operand, as they do in 16 bits.
//
// Dropout (the fused LayerNorm's convention): element (b, h, i, j) has the flat index idx = ((b H + h) S + i) S + j over
// [B, H, S, S] and is kept iff word idx % 4 of Philox4x32-10(counter (idx/4 low, idx/4 high, 0, 0), key (seed low,
// seed high)) is below keep_thr = floor((1-p) 2^32).  The seed is one int64 read from device memory; keep_thr >= 2^32
// (p = 0) reads no seed and runs no generator.
//
// Ragged tiles: S need not be a multiple of 64.  Rows past S are staged as zeros; keys past S get the bias -inf, queries
// past S the row max +inf, so their P is exactly 0, and nothing past S is stored.  16-bit stores round to nearest
// even without saturating, so an overflow arrives as inf.
//
// Masks: a finite mask entry gives a finite bias.  Where m log2 e overflows fp32 (torch.finfo(torch.float32).min, or
// bf16's minimum widened) the bias saturates at -FLT_MAX, so a sequence masked at every key with such a minimum has
// every score at -FLT_MAX and averages V uniformly, as the float64 formula does.  A sequence whose mask is -inf at every
// key has m = -inf and l = 0 in every row: its O and d(qkv) are NaN, as softmax over an all -inf row is.
#include <cfloat>

#include "common.cuh"
#include "devlib.cuh"
#include "elem.cuh"
#include "oktopk.cuh"

namespace okt {

constexpr int kAttD = 64;                       // head dim
constexpr int kAttBlk = 64;                     // rows of a query or key tile
constexpr int kAttWarps = kAttBlk / 16;         // 16 rows per warp
constexpr int kAttThreads = 32 * kAttWarps;
constexpr int kAttLd = kAttD + 8;               // padded shared-memory row: fragment loads are bank-conflict free
constexpr int kAttNt = kAttBlk / 8;             // n-tiles of 8 columns across a 64-wide tile
constexpr int kAttMaxS = 512;
constexpr int kAttMaxDevices = 64;
constexpr long long kAttKeepAll = 1LL << 32;
constexpr float kAttLog2e = 1.4426950408889634f;
constexpr float kAttScale = 0.125f;             // 1 / sqrt(64)

// ---- the tensor-core product of one warp, per element type ------------------------------------------------------
// load_a:  A[16 x kK] rows row0.., columns k0.. of a row-major tile.
// load_bt: B[kK x 8] with B[k][n] = X[n0 + n][k0 + k]   (X row-major, k contiguous: QK^T-style)
// load_bn: B[kK x 8] with B[k][n] = X[k0 + k][n0 + n]   (PV-style)
// from_c:  the A operand of k chunk kc taken from a warp's 16 x 8N fp32 accumulator (P or dS)
template <typename T> struct AttnMma;

template <> struct AttnMma<float> {             // 3xTF32, m16n8k8 (elem.cuh)
    static constexpr int kK = 8;
    struct A { uint32_t h[4], l[4]; };
    struct B { uint32_t h[2], l[2]; };
    static __device__ __forceinline__ void split(float x, uint32_t& h, uint32_t& l) { tf32_split(x, h, l); }
    // slot order a0 (g, t) a1 (g+8, t) a2 (g, t+4) a3 (g+8, t+4); slot t is column 2t, slot t + 4 column 2t + 1
    static __device__ __forceinline__ A make_a(float g0, float g1, float g8a, float g8b) {
        A a;
        split(g0, a.h[0], a.l[0]);
        split(g8a, a.h[1], a.l[1]);
        split(g1, a.h[2], a.l[2]);
        split(g8b, a.h[3], a.l[3]);
        return a;
    }
    static __device__ __forceinline__ B make_b(float k0, float k1) {
        B b;
        split(k0, b.h[0], b.l[0]);
        split(k1, b.h[1], b.l[1]);
        return b;
    }
    static __device__ __forceinline__ A load_a(const float* s, int row0, int k0) {
        const int g = lane_id() >> 2, t = lane_id() & 3;
        const float2 r0 = *reinterpret_cast<const float2*>(s + (row0 + g) * kAttLd + k0 + 2 * t);
        const float2 r1 = *reinterpret_cast<const float2*>(s + (row0 + g + 8) * kAttLd + k0 + 2 * t);
        return make_a(r0.x, r0.y, r1.x, r1.y);
    }
    static __device__ __forceinline__ B load_bt(const float* s, int n0, int k0) {
        const int g = lane_id() >> 2, t = lane_id() & 3;
        const float2 r = *reinterpret_cast<const float2*>(s + (n0 + g) * kAttLd + k0 + 2 * t);
        return make_b(r.x, r.y);
    }
    static __device__ __forceinline__ B load_bn(const float* s, int k0, int n0) {
        const int g = lane_id() >> 2, t = lane_id() & 3;
        return make_b(s[(k0 + 2 * t) * kAttLd + n0 + g], s[(k0 + 2 * t + 1) * kAttLd + n0 + g]);
    }
    template <int N>
    static __device__ __forceinline__ A from_c(const float (&c)[N][4], int kc) {
        return make_a(c[kc][0], c[kc][1], c[kc][2], c[kc][3]);
    }
    // Chained through one accumulator, a 64-long sum's truncations bias it (24 of them, ~1e-5 relative at S = 512);
    // the elem.cuh product adds each k8 step to d with a rounded fp32 add instead.
    static __device__ __forceinline__ void mma(float (&d)[4], const A& a, const B& b) {
        mma_m16n8k8_3xtf32(d, a.h, a.l, b.h, b.l);
    }
};

template <typename T> struct AttnMma16 {        // bf16 / fp16, m16n8k16
    static constexpr int kK = 16;
    struct A { uint32_t r[4]; };
    struct B { uint32_t r[2]; };
    static __device__ __forceinline__ uint32_t u32(const T* p) { return *reinterpret_cast<const uint32_t*>(p); }
    static __device__ __forceinline__ uint32_t pack_raw(const T* lo, const T* hi) {
        return (uint32_t)*reinterpret_cast<const uint16_t*>(lo) | ((uint32_t)*reinterpret_cast<const uint16_t*>(hi) << 16);
    }
    static __device__ __forceinline__ uint32_t pack(float lo, float hi) { return Elem<T>::narrow2(lo, hi); }
    static __device__ __forceinline__ A load_a(const T* s, int row0, int k0) {
        const int g = lane_id() >> 2, t = lane_id() & 3;
        const T* p0 = s + (row0 + g) * kAttLd + k0 + 2 * t;
        const T* p1 = p0 + 8 * kAttLd;
        return A{{u32(p0), u32(p1), u32(p0 + 8), u32(p1 + 8)}};
    }
    static __device__ __forceinline__ B load_bt(const T* s, int n0, int k0) {
        const int g = lane_id() >> 2, t = lane_id() & 3;
        const T* p = s + (n0 + g) * kAttLd + k0 + 2 * t;
        return B{{u32(p), u32(p + 8)}};
    }
    static __device__ __forceinline__ B load_bn(const T* s, int k0, int n0) {
        const int g = lane_id() >> 2, t = lane_id() & 3;
        const T* p = s + (k0 + 2 * t) * kAttLd + n0 + g;
        return B{{pack_raw(p, p + kAttLd), pack_raw(p + 8 * kAttLd, p + 9 * kAttLd)}};
    }
    template <int N>
    static __device__ __forceinline__ A from_c(const float (&c)[N][4], int kc) {
        return A{{pack(c[2 * kc][0], c[2 * kc][1]), pack(c[2 * kc][2], c[2 * kc][3]), pack(c[2 * kc + 1][0], c[2 * kc + 1][1]),
                  pack(c[2 * kc + 1][2], c[2 * kc + 1][3])}};
    }
    static __device__ __forceinline__ void mma(float (&d)[4], const A& a, const B& b) { mma_m16n8k16<T>(d, a.r, b.r); }
};
template <> struct AttnMma<__nv_bfloat16> : AttnMma16<__nv_bfloat16> {};
template <> struct AttnMma<__half> : AttnMma16<__half> {};

// Stage rows [0, n) of a 64 x 64 block (global row stride `stride` elements, 16-byte aligned rows) into a padded
// shared tile; rows n..63 are zeros.
template <typename T>
__device__ __forceinline__ void att_stage(T* s, const T* g, long long stride, int n) {
    constexpr int kVec = 16 / sizeof(T), kPerRow = kAttD / kVec;
    for (int v = threadIdx.x; v < kAttBlk * kPerRow; v += kAttThreads) {
        const int r = v / kPerRow, c = (v % kPerRow) * kVec;
        const uint4 x = r < n ? __ldg(reinterpret_cast<const uint4*>(g + r * stride + c)) : make_uint4(0u, 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(s + r * kAttLd + c) = x;
    }
}

// acc += A B over k = 0..63: A the warp's 16 rows of tile `a`, B the 8N columns n0.. from tile `b` (load_bt when BT,
// else load_bn)
template <typename T, bool BT, int N>
__device__ __forceinline__ void att_product(float (&acc)[N][4], const T* a, int row0, const T* b, int n0 = 0) {
    using M = AttnMma<T>;
#pragma unroll
    for (int k0 = 0; k0 < kAttD; k0 += M::kK) {
        const typename M::A fa = M::load_a(a, row0, k0);
#pragma unroll
        for (int nt = 0; nt < N; ++nt)
            M::mma(acc[nt], fa, BT ? M::load_bt(b, n0 + nt * 8, k0) : M::load_bn(b, k0, n0 + nt * 8));
    }
}

// acc += C X: C the warp's 16 x 8N accumulator (P or dS), X the rows k0 .. k0 + 8N - 1 of a 64-wide tile indexed [k][n]
template <typename T, int N>
__device__ __forceinline__ void att_product_c(float (&acc)[kAttNt][4], const float (&c)[N][4], const T* x, int k0 = 0) {
    using M = AttnMma<T>;
#pragma unroll
    for (int kc = 0; kc < 8 * N / M::kK; ++kc) {
        const typename M::A fa = M::from_c(c, kc);
#pragma unroll
        for (int nt = 0; nt < kAttNt; ++nt) M::mma(acc[nt], fa, M::load_bn(x, k0 + kc * M::kK, nt * 8));
    }
}

template <int N>
__device__ __forceinline__ void att_zero(float (&c)[N][4]) {
#pragma unroll
    for (int nt = 0; nt < N; ++nt) c[nt][0] = c[nt][1] = c[nt][2] = c[nt][3] = 0.f;
}

struct AttDrop {
    bool on;
    uint32_t thr, k0, k1;
    float s;
};

__device__ __forceinline__ AttDrop att_drop(const unsigned long long* seed, long long keep_thr, float scale) {
    AttDrop d;
    d.on = keep_thr < kAttKeepAll;
    d.thr = (uint32_t)keep_thr;
    const unsigned long long k = d.on ? __ldg(seed) : 0ull;
    d.k0 = (uint32_t)k;
    d.k1 = (uint32_t)(k >> 32);
    d.s = scale;
    return d;
}

// the dropout multiplier of flat element idx: 1/(1-p) where kept, 0 where dropped, 1 without dropout
__device__ __forceinline__ float att_mult(const AttDrop& d, unsigned long long idx) {
    if (!d.on) return 1.f;
    const unsigned long long q = idx >> 2;
    const uint4 r = philox4x32_10(make_uint4((uint32_t)q, (uint32_t)(q >> 32), 0u, 0u), d.k0, d.k1);
    const uint32_t w = (idx & 2) ? ((idx & 1) ? r.w : r.z) : ((idx & 1) ? r.y : r.x);
    return w < d.thr ? d.s : 0.f;
}

// the key bias of key j in log2 units: the mask's entry (0 without one), -inf past S.  A finite entry saturates at
// +-FLT_MAX instead of overflowing to +-inf; +-inf and NaN entries pass through.
__device__ __forceinline__ float att_bias(const float* mask, int b, int S, int j) {
    if (j >= S) return -INFINITY;
    if (mask == nullptr) return 0.f;
    const float x = mask[(size_t)b * S + j];
    return isfinite(x) ? fminf(fmaxf(x * kAttLog2e, -FLT_MAX), FLT_MAX) : x;
}

template <typename T>
__global__ void __launch_bounds__(kAttThreads) attn_fwd_kernel(const T* __restrict__ qkv, const float* __restrict__ mask,
                                                               const unsigned long long* seed, T* __restrict__ out,
                                                               float2* __restrict__ lse, int S, int H, long long keep_thr,
                                                               float dscale) {
    extern __shared__ __align__(16) unsigned char att_smem[];
    T* sq = reinterpret_cast<T*>(att_smem);
    T* sk = sq + kAttBlk * kAttLd;
    T* sv = sk + kAttBlk * kAttLd;
    float* sbias = reinterpret_cast<float*>(sv + kAttBlk * kAttLd);
    const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * kAttBlk;
    const int lane = lane_id(), g = lane >> 2, t = lane & 3, row0 = (threadIdx.x >> 5) * 16;
    const int HD = H * kAttD;
    const long long ld3 = 3LL * HD, bh = (long long)b * H + h;
    const T* base = qkv + (long long)b * S * ld3 + h * kAttD;
    const AttDrop d = att_drop(seed, keep_thr, dscale);
    const float c = kAttScale * kAttLog2e;

    att_stage(sq, base + q0 * ld3, ld3, min(kAttBlk, S - q0));
    float o[kAttNt][4];
    att_zero(o);
    float mx[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    for (int k0 = 0; k0 < S; k0 += kAttBlk) {
        __syncthreads();                                        // the previous key block is consumed
        att_stage(sk, base + HD + k0 * ld3, ld3, min(kAttBlk, S - k0));
        att_stage(sv, base + 2 * HD + k0 * ld3, ld3, min(kAttBlk, S - k0));
        for (int j = threadIdx.x; j < kAttBlk; j += kAttThreads) sbias[j] = att_bias(mask, b, S, k0 + j);
        __syncthreads();
        float s[kAttNt][4];
        att_zero(s);
        att_product<T, true>(s, sq, row0, sk);
        float m[2] = {mx[0], mx[1]};
#pragma unroll
        for (int nt = 0; nt < kAttNt; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                s[nt][e] = fmaf(s[nt][e], c, sbias[nt * 8 + 2 * t + (e & 1)]);
                m[e >> 1] = fmaxf(m[e >> 1], s[nt][e]);
            }
        float ref[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 1));
            m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 2));
            ref[r] = m[r] == -INFINITY ? 0.f : m[r];            // a row with no finite score yet stays at 0
            const float alpha = exp2f(mx[r] - ref[r]);
            mx[r] = m[r];
            l[r] *= alpha;
#pragma unroll
            for (int nt = 0; nt < kAttNt; ++nt) {
                o[nt][2 * r] *= alpha;
                o[nt][2 * r + 1] *= alpha;
            }
        }
#pragma unroll
        for (int nt = 0; nt < kAttNt; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = e >> 1;
                const float p = exp2f(s[nt][e] - ref[r]);
                l[r] += p;
                const long long i = q0 + row0 + g + 8 * r, j = k0 + nt * 8 + 2 * t + (e & 1);
                s[nt][e] = p * att_mult(d, (unsigned long long)((bh * S + i) * S + j));
            }
        att_product_c<T>(o, s, sv);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
        const int i = q0 + row0 + g + 8 * r;
        if (i >= S) continue;
        const float inv = 1.f / l[r];
        T* orow = out + ((long long)b * S + i) * HD + h * kAttD + 2 * t;
#pragma unroll
        for (int nt = 0; nt < kAttNt; ++nt) Elem<T>::st2(orow + nt * 8, o[nt][2 * r] * inv, o[nt][2 * r + 1] * inv);
        if (t == 0) lse[bh * S + i] = make_float2(mx[r], log2f(l[r]));
    }
}

template <typename T>
__global__ void __launch_bounds__(kAttThreads) attn_bwd_dq_kernel(const T* __restrict__ qkv, const T* __restrict__ out,
                                                                  const T* __restrict__ dout, const float* __restrict__ mask,
                                                                  const unsigned long long* seed, const float2* __restrict__ lse,
                                                                  float* __restrict__ delta, T* __restrict__ dqkv, int S,
                                                                  int H, long long keep_thr, float dscale) {
    extern __shared__ __align__(16) unsigned char att_smem[];
    T* sq = reinterpret_cast<T*>(att_smem);
    T* sdo = sq + kAttBlk * kAttLd;
    T* sk = sdo + kAttBlk * kAttLd;
    T* sv = sk + kAttBlk * kAttLd;
    float* sbias = reinterpret_cast<float*>(sv + kAttBlk * kAttLd);
    const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * kAttBlk;
    const int lane = lane_id(), g = lane >> 2, t = lane & 3, row0 = (threadIdx.x >> 5) * 16;
    const int HD = H * kAttD;
    const long long ld3 = 3LL * HD, bh = (long long)b * H + h;
    const T* base = qkv + (long long)b * S * ld3 + h * kAttD;
    const AttDrop d = att_drop(seed, keep_thr, dscale);
    const float c = kAttScale * kAttLog2e;

    att_stage(sq, base + q0 * ld3, ld3, min(kAttBlk, S - q0));
    att_stage(sdo, dout + ((long long)b * S + q0) * HD + h * kAttD, HD, min(kAttBlk, S - q0));
    __syncthreads();
    // Delta of rows g, g + 8: lane t adds columns 16t .. 16t + 15, then the four lanes in lane order
    float dl[2];
    float2 ls[2];                                       // the row's max and log2 of its sum
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int i = q0 + row0 + g + 8 * r;
        float acc = 0.f;
        if (i < S) {
            const T* orow = out + ((long long)b * S + i) * HD + h * kAttD + 16 * t;
            const T* drow = sdo + (row0 + g + 8 * r) * kAttLd + 16 * t;
#pragma unroll
            for (int x = 0; x < 16; ++x) acc = fmaf(Elem<T>::f32(drow[x]), Elem<T>::f32(orow[x]), acc);
        }
        acc += __shfl_xor_sync(0xffffffffu, acc, 1);
        acc += __shfl_xor_sync(0xffffffffu, acc, 2);
        dl[r] = acc;
        ls[r] = i < S ? lse[bh * S + i] : make_float2(INFINITY, 0.f);
        if (t == 0 && i < S) delta[bh * S + i] = acc;
    }
    float dq[kAttNt][4];
    att_zero(dq);
    for (int k0 = 0; k0 < S; k0 += kAttBlk) {
        __syncthreads();
        att_stage(sk, base + HD + k0 * ld3, ld3, min(kAttBlk, S - k0));
        att_stage(sv, base + 2 * HD + k0 * ld3, ld3, min(kAttBlk, S - k0));
        for (int j = threadIdx.x; j < kAttBlk; j += kAttThreads) sbias[j] = att_bias(mask, b, S, k0 + j);
        __syncthreads();
        float s[kAttNt][4], dp[kAttNt][4];
        att_zero(s);
        att_zero(dp);
        att_product<T, true>(s, sq, row0, sk);
        att_product<T, true>(dp, sdo, row0, sv);
#pragma unroll
        for (int nt = 0; nt < kAttNt; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = e >> 1, col = nt * 8 + 2 * t + (e & 1);
                const float p = exp2f(fmaf(s[nt][e], c, sbias[col]) - ls[r].x - ls[r].y);
                const long long i = q0 + row0 + g + 8 * r, j = k0 + col;
                s[nt][e] = p * (dp[nt][e] * att_mult(d, (unsigned long long)((bh * S + i) * S + j)) - dl[r]);
            }
        att_product_c<T>(dq, s, sk);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int i = q0 + row0 + g + 8 * r;
        if (i >= S) continue;
        T* row = dqkv + ((long long)b * S + i) * ld3 + h * kAttD + 2 * t;
#pragma unroll
        for (int nt = 0; nt < kAttNt; ++nt) Elem<T>::st2(row + nt * 8, dq[nt][2 * r] * kAttScale, dq[nt][2 * r + 1] * kAttScale);
    }
}

template <typename T>
__global__ void __launch_bounds__(kAttThreads) attn_bwd_dkv_kernel(const T* __restrict__ qkv, const T* __restrict__ dout,
                                                                   const float* __restrict__ mask,
                                                                   const unsigned long long* seed,
                                                                   const float2* __restrict__ lse,
                                                                   const float* __restrict__ delta, T* __restrict__ dqkv,
                                                                   int S, int H, long long keep_thr, float dscale) {
    extern __shared__ __align__(16) unsigned char att_smem[];
    T* sk = reinterpret_cast<T*>(att_smem);
    T* sv = sk + kAttBlk * kAttLd;
    T* sq = sv + kAttBlk * kAttLd;
    T* sdo = sq + kAttBlk * kAttLd;
    float* smx = reinterpret_cast<float*>(sdo + kAttBlk * kAttLd);      // the query rows' max, log2 sum and Delta
    float* sll = smx + kAttBlk;
    float* sdl = sll + kAttBlk;
    const int b = blockIdx.z, h = blockIdx.y, j0 = blockIdx.x * kAttBlk;
    const int lane = lane_id(), g = lane >> 2, t = lane & 3, row0 = (threadIdx.x >> 5) * 16;
    const int HD = H * kAttD;
    const long long ld3 = 3LL * HD, bh = (long long)b * H + h;
    const T* base = qkv + (long long)b * S * ld3 + h * kAttD;
    const AttDrop d = att_drop(seed, keep_thr, dscale);
    const float c = kAttScale * kAttLog2e;

    att_stage(sk, base + HD + j0 * ld3, ld3, min(kAttBlk, S - j0));
    att_stage(sv, base + 2 * HD + j0 * ld3, ld3, min(kAttBlk, S - j0));
    const float kb[2] = {att_bias(mask, b, S, j0 + row0 + g), att_bias(mask, b, S, j0 + row0 + g + 8)};
    float dk[kAttNt][4], dv[kAttNt][4];
    att_zero(dk);
    att_zero(dv);
    for (int i0 = 0; i0 < S; i0 += kAttBlk) {
        __syncthreads();
        att_stage(sq, base + i0 * ld3, ld3, min(kAttBlk, S - i0));
        att_stage(sdo, dout + ((long long)b * S + i0) * HD + h * kAttD, HD, min(kAttBlk, S - i0));
        for (int i = threadIdx.x; i < kAttBlk; i += kAttThreads) {
            const bool in = i0 + i < S;
            const float2 st = in ? lse[bh * S + i0 + i] : make_float2(INFINITY, 0.f);
            smx[i] = st.x;
            sll[i] = st.y;
            sdl[i] = in ? delta[bh * S + i0 + i] : 0.f;
        }
        __syncthreads();
        // S^T and dP^T (rows keys, columns queries) over kCols query columns at a time: in fp32 the dK and dV
        // accumulators and the 3xTF32 operands leave no room for two full 16 x 64 tiles within 255 registers
        constexpr int kCols = sizeof(T) == 4 ? 32 : kAttBlk, kNc = kCols / 8;
#pragma unroll 1
        for (int c0 = 0; c0 < kAttBlk; c0 += kCols) {
            float s[kNc][4], dp[kNc][4];
            att_zero(s);
            att_zero(dp);
            att_product<T, true>(s, sk, row0, sq, c0);
            att_product<T, true>(dp, sv, row0, sdo, c0);
#pragma unroll
            for (int nt = 0; nt < kNc; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int r = e >> 1, col = c0 + nt * 8 + 2 * t + (e & 1);
                    const float p = exp2f(fmaf(s[nt][e], c, kb[r]) - smx[col] - sll[col]);
                    const long long i = i0 + col, j = j0 + row0 + g + 8 * r;
                    const float m = att_mult(d, (unsigned long long)((bh * S + i) * S + j));
                    s[nt][e] = p * m;
                    dp[nt][e] = p * (dp[nt][e] * m - sdl[col]);
                }
            att_product_c<T>(dk, dp, sq, c0);
            att_product_c<T>(dv, s, sdo, c0);
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int j = j0 + row0 + g + 8 * r;
        if (j >= S) continue;
        T* row = dqkv + ((long long)b * S + j) * ld3 + h * kAttD + 2 * t;
#pragma unroll
        for (int nt = 0; nt < kAttNt; ++nt) {
            Elem<T>::st2(row + HD + nt * 8, dk[nt][2 * r] * kAttScale, dk[nt][2 * r + 1] * kAttScale);
            Elem<T>::st2(row + 2 * HD + nt * 8, dv[nt][2 * r], dv[nt][2 * r + 1]);
        }
    }
}

bool attn_supported(int B, int S, int H) { return B >= 1 && B <= 65535 && H >= 1 && H <= 65535 && S >= 1 && S <= kAttMaxS; }

// Dynamic shared memory: 3 (forward) or 4 (backward) padded tiles and 64 or 192 floats.  fp32 needs more than the
// default 48 KB, so each kernel's limit is raised once per device and the launches after that query nothing.
template <typename T> constexpr size_t att_smem_fwd() { return 3 * kAttBlk * kAttLd * sizeof(T) + kAttBlk * sizeof(float); }
template <typename T> constexpr size_t att_smem_bwd() { return 4 * kAttBlk * kAttLd * sizeof(T) + 3 * kAttBlk * sizeof(float); }

template <typename T, int Kernel>
static cudaError_t att_prepare(const void* kernel, size_t smem) {
    static bool done[kAttMaxDevices];
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= kAttMaxDevices) return cudaErrorInvalidDevice;
    if (done[dev]) return cudaSuccess;
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        return e;
    }
    done[dev] = true;
    return cudaSuccess;
}

static dim3 att_grid(int B, int S, int H) { return dim3((S + kAttBlk - 1) / kAttBlk, H, B); }

template <typename T>
static cudaError_t attn_forward_t(const void* qkv, const float* mask, const unsigned long long* seed, void* out, float* lse,
                                  int B, int S, int H, long long keep_thr, float scale, cudaStream_t stream) {
    constexpr size_t smem = att_smem_fwd<T>();
    cudaError_t e = att_prepare<T, 0>((const void*)attn_fwd_kernel<T>, smem);
    if (e != cudaSuccess) return e;
    attn_fwd_kernel<T><<<att_grid(B, S, H), kAttThreads, smem, stream>>>(static_cast<const T*>(qkv), mask, seed,
                                                                        static_cast<T*>(out), reinterpret_cast<float2*>(lse),
                                                                        S, H, keep_thr, scale);
    return cudaGetLastError();
}

template <typename T>
static cudaError_t attn_backward_t(const void* qkv, const void* out, const void* dout, const float* mask,
                                   const unsigned long long* seed, const float* lse, float* delta, void* dqkv, int B, int S,
                                   int H, long long keep_thr, float scale, cudaStream_t stream) {
    constexpr size_t smem = att_smem_bwd<T>();
    cudaError_t e = att_prepare<T, 1>((const void*)attn_bwd_dq_kernel<T>, smem);
    if (e == cudaSuccess) e = att_prepare<T, 2>((const void*)attn_bwd_dkv_kernel<T>, smem);
    if (e != cudaSuccess) return e;
    const T* q = static_cast<const T*>(qkv);
    const T* dt = static_cast<const T*>(dout);
    T* dq = static_cast<T*>(dqkv);
    const float2* st = reinterpret_cast<const float2*>(lse);
    attn_bwd_dq_kernel<T><<<att_grid(B, S, H), kAttThreads, smem, stream>>>(q, static_cast<const T*>(out), dt, mask, seed,
                                                                           st, delta, dq, S, H, keep_thr, scale);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    attn_bwd_dkv_kernel<T><<<att_grid(B, S, H), kAttThreads, smem, stream>>>(q, dt, mask, seed, st, delta, dq, S, H,
                                                                            keep_thr, scale);
    return cudaGetLastError();
}

static bool attn_args_ok(int B, int S, int H, long long keep_thr, const unsigned long long* seed) {
    return attn_supported(B, S, H) && keep_thr >= 0 && keep_thr <= kAttKeepAll && (keep_thr == kAttKeepAll || seed != nullptr);
}

cudaError_t launch_attn_forward(const void* qkv, const float* mask, const unsigned long long* seed, void* out, float* lse,
                                int B, int S, int H, long long keep_thr, float scale, Dtype dtype, cudaStream_t stream) {
    if (!attn_args_ok(B, S, H, keep_thr, seed)) return cudaErrorInvalidValue;
    return with_dtype(dtype, [&](auto e) {
        return attn_forward_t<decltype(e)>(qkv, mask, seed, out, lse, B, S, H, keep_thr, scale, stream);
    });
}

cudaError_t launch_attn_backward(const void* qkv, const void* out, const void* dout, const float* mask,
                                 const unsigned long long* seed, const float* lse, float* delta, void* dqkv, int B, int S,
                                 int H, long long keep_thr, float scale, Dtype dtype, cudaStream_t stream) {
    if (!attn_args_ok(B, S, H, keep_thr, seed)) return cudaErrorInvalidValue;
    return with_dtype(dtype, [&](auto e) {
        return attn_backward_t<decltype(e)>(qkv, out, dout, mask, seed, lse, delta, dqkv, B, S, H, keep_thr, scale, stream);
    });
}

}  // namespace okt
