// Storage types of the kernels that run on fp32, bf16 or fp16 tensors (batch-norm, LayerNorm, cross-entropy, the
// LSTM and attention): Elem<T> widens a stored element to fp32 for the arithmetic and rounds an fp32 result back for a
// store, and with_dtype() turns a Dtype code into the storage type on the host.
//
// The numeric contract, the same in every kernel:
//   - widening is exact: a bf16 is the high half of its fp32, and every fp16, subnormals included, is an fp32;
//   - rounding is to nearest, ties to even, as torch's .to(dtype);
//   - nothing saturates: an fp16 result whose magnitude rounds past 65504 is stored as +-inf, so that an overflow under
//     loss scaling reaches the scaler's non-finite check; fp16 subnormals are kept, not flushed to zero (cvt.rn without
//     .ftz: the build passes neither -ftz nor --use_fast_math).
// fp32 storage is the identity.
//
// Elem<T>, at the width each kernel converts:
//   f32(x), ld(p)               one element widened; ld loads it through the read-only path
//   narrow1(v)                  one element rounded
//   wide2(w, lo, hi),           (16-bit types) the two elements of one 32-bit word, the low half first
//   narrow2(lo, hi)
//   st2(p, lo, hi)              two consecutive elements rounded and stored in one access
//   V, wide(v), narrow(f),      four consecutive elements in one access: float4, or a uint2 of two words
//   zero()
//   kVec, wide(u, f),           the kVec elements of one 16-byte vector (uint4)
//   narrow(f)
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "oktopk.cuh"

namespace okt {

// bf16 and fp16: everything is built from the four scalar and pair conversions specialised below.
template <typename T> struct Elem {
    static_assert(std::is_same<T, __nv_bfloat16>::value || std::is_same<T, __half>::value,
                  "Elem<T>: T is float, __nv_bfloat16 or __half");
    using V = uint2;                          // elements 0, 1 in x (low half first), 2, 3 in y
    static constexpr int kVec = 8;
    static __device__ __forceinline__ float f32(T x);
    static __device__ __forceinline__ T narrow1(float v);
    static __device__ __forceinline__ void wide2(unsigned int w, float& lo, float& hi);
    static __device__ __forceinline__ unsigned int narrow2(float lo, float hi);

    static __device__ __forceinline__ float ld(const T* p) { return f32(__ldg(p)); }
    static __device__ __forceinline__ void st2(T* p, float lo, float hi) {
        *reinterpret_cast<unsigned int*>(p) = narrow2(lo, hi);
    }
    static __device__ __forceinline__ uint2 zero() { return make_uint2(0u, 0u); }
    static __device__ __forceinline__ float4 wide(const uint2& v) {
        float4 f;
        wide2(v.x, f.x, f.y);
        wide2(v.y, f.z, f.w);
        return f;
    }
    static __device__ __forceinline__ uint2 narrow(const float4& f) { return make_uint2(narrow2(f.x, f.y), narrow2(f.z, f.w)); }
    static __device__ __forceinline__ void wide(const uint4& u, float (&f)[kVec]) {
        wide2(u.x, f[0], f[1]); wide2(u.y, f[2], f[3]); wide2(u.z, f[4], f[5]); wide2(u.w, f[6], f[7]);
    }
    static __device__ __forceinline__ uint4 narrow(const float (&f)[kVec]) {
        return make_uint4(narrow2(f[0], f[1]), narrow2(f[2], f[3]), narrow2(f[4], f[5]), narrow2(f[6], f[7]));
    }
};

template <> __device__ __forceinline__ float Elem<__nv_bfloat16>::f32(__nv_bfloat16 x) { return __bfloat162float(x); }
template <> __device__ __forceinline__ __nv_bfloat16 Elem<__nv_bfloat16>::narrow1(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ void Elem<__nv_bfloat16>::wide2(unsigned int w, float& lo, float& hi) {
    lo = __uint_as_float(w << 16);
    hi = __uint_as_float(w & 0xffff0000u);
}
template <> __device__ __forceinline__ unsigned int Elem<__nv_bfloat16>::narrow2(float lo, float hi) {
    const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<const unsigned int*>(&v);
}

template <> __device__ __forceinline__ float Elem<__half>::f32(__half x) { return __half2float(x); }
template <> __device__ __forceinline__ __half Elem<__half>::narrow1(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ void Elem<__half>::wide2(unsigned int w, float& lo, float& hi) {
    const float2 v = __half22float2(*reinterpret_cast<const __half2*>(&w));
    lo = v.x;
    hi = v.y;
}
template <> __device__ __forceinline__ unsigned int Elem<__half>::narrow2(float lo, float hi) {
    const __half2 v = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const unsigned int*>(&v);
}

template <> struct Elem<float> {
    using V = float4;
    static constexpr int kVec = 4;
    static __device__ __forceinline__ float f32(float x) { return x; }
    static __device__ __forceinline__ float narrow1(float v) { return v; }
    static __device__ __forceinline__ float ld(const float* p) { return __ldg(p); }
    static __device__ __forceinline__ void st2(float* p, float lo, float hi) {
        *reinterpret_cast<float2*>(p) = make_float2(lo, hi);
    }
    static __device__ __forceinline__ float4 zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
    static __device__ __forceinline__ float4 wide(const float4& v) { return v; }
    static __device__ __forceinline__ float4 narrow(const float4& v) { return v; }
    static __device__ __forceinline__ void wide(const uint4& u, float (&f)[kVec]) {
        f[0] = __uint_as_float(u.x); f[1] = __uint_as_float(u.y); f[2] = __uint_as_float(u.z); f[3] = __uint_as_float(u.w);
    }
    static __device__ __forceinline__ uint4 narrow(const float (&f)[kVec]) {
        return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
    }
};

// d += a b on the tensor cores, mma.sync m16n8k16 (row.col) with fp32 accumulation, for T = __nv_bfloat16 or __half:
// a holds the 16 x 16 A fragment and b the 16 x 8 B fragment in the PTX ISA's register layout.
template <typename T>
__device__ __forceinline__ void mma_m16n8k16(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]);
template <> __device__ __forceinline__ void mma_m16n8k16<__nv_bfloat16>(float (&d)[4], const uint32_t (&a)[4],
                                                                       const uint32_t (&b)[2]) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
template <> __device__ __forceinline__ void mma_m16n8k16<__half>(float (&d)[4], const uint32_t (&a)[4],
                                                                const uint32_t (&b)[2]) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// 3xTF32 for fp32 products on the tensor cores (attention, the stacked-layer LSTM): each operand is split into a TF32
// high part and a TF32 remainder, and a.b ~ ah.bh + ah.bl + al.bh, which keeps about fp32 accuracy (the dropped al.bl
// is below 2^-22 relative) at three tensor-core products.
//
// tf32(x): x rounded to nearest, the low 13 bits cleared, so that x - tf32(x) is the exact remainder.
__device__ __forceinline__ uint32_t tf32_hi(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r & 0xffffe000u;
}
__device__ __forceinline__ void tf32_split(float x, uint32_t& h, uint32_t& l) {
    h = tf32_hi(x);
    l = tf32_hi(x - __uint_as_float(h));
}

// d += a b, mma.sync m16n8k8 (row.col) in TF32 with fp32 accumulation; fragments in the PTX ISA's register layout:
// a0 (g, t), a1 (g + 8, t), a2 (g, t + 4), a3 (g + 8, t + 4); b0 (k = t, n = g), b1 (k = t + 4, n = g).
__device__ __forceinline__ void mma_m16n8k8_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// d += (ah + al)(bh + bl) in 3xTF32 over one k8 step.  The tensor cores truncate as they accumulate, so the three
// products go into a fresh zero accumulator, the small terms first, and that is added to d with a rounded fp32 add.
__device__ __forceinline__ void mma_m16n8k8_3xtf32(float (&d)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4],
                                                   const uint32_t (&bh)[2], const uint32_t (&bl)[2]) {
    float t[4] = {0.f, 0.f, 0.f, 0.f};
    mma_m16n8k8_tf32(t, al, bh);
    mma_m16n8k8_tf32(t, ah, bl);
    mma_m16n8k8_tf32(t, ah, bh);
#pragma unroll
    for (int i = 0; i < 4; ++i) d[i] += t[i];
}

// f(T{}) with T the storage type of `dtype`: a launcher calls its templated body through it once, whatever the type.
template <class F>
cudaError_t with_dtype(Dtype dtype, F&& f) {
    switch (dtype) {
        case Dtype::kF32: return f(float{});
        case Dtype::kBF16: return f(__nv_bfloat16{});
        case Dtype::kF16: return f(__half{});
    }
    return cudaErrorInvalidValue;
}

}  // namespace okt
