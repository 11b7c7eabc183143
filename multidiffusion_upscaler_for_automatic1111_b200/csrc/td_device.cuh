// Device-side helpers: element traits with explicit IEEE roundings, 128-bit
// read-only loads, unaligned-vector extraction by funnel shift, packed adds and
// exact divides, programmatic dependent launch and the cross-GPU flag wait.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace td {

// ---- element traits ------------------------------------------------------
// to_f32 is exact; from_f32 is round-to-nearest-even -- the same rounding
// torch applies when an fp32 intermediate is stored to a half/bf16 tensor.
template <typename T> struct Elem;
template <> struct Elem<__half> {
    static constexpr int kDtype = 0;
    __host__ __device__ static __forceinline__ float to_f32(__half v) { return __half2float(v); }
    __host__ __device__ static __forceinline__ __half from_f32(float f) { return __float2half_rn(f); }
    __device__ static __forceinline__ float bits_to_f32(uint16_t b) { return __half2float(__ushort_as_half(b)); }
    __device__ static __forceinline__ uint16_t f32_to_bits(float f) { return __half_as_ushort(__float2half_rn(f)); }
};
template <> struct Elem<__nv_bfloat16> {
    static constexpr int kDtype = 1;
    __host__ __device__ static __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
    __host__ __device__ static __forceinline__ __nv_bfloat16 from_f32(float f) { return __float2bfloat16_rn(f); }
    __device__ static __forceinline__ float bits_to_f32(uint16_t b) { return __uint_as_float(((uint32_t)b) << 16); }
    __device__ static __forceinline__ uint16_t f32_to_bits(float f) { return __bfloat16_as_ushort(__float2bfloat16_rn(f)); }
};
template <> struct Elem<float> {
    static constexpr int kDtype = 2;
    __host__ __device__ static __forceinline__ float to_f32(float v) { return v; }
    __host__ __device__ static __forceinline__ float from_f32(float f) { return f; }
};

// round an fp32 value through T (the "store to x_buffer, load it back" of the reference)
template <typename T> __device__ __forceinline__ float round_through(float f) { return Elem<T>::to_f32(Elem<T>::from_f32(f)); }
template <> __device__ __forceinline__ float round_through<float>(float f) { return f; }

// ---- 128-bit global access -------------------------------------------------
__device__ __forceinline__ uint4 ldg128(const void* p) {  // read-only path, keeps L1 (neighbour threads re-use the line)
    return __ldg(reinterpret_cast<const uint4*>(p));
}
__device__ __forceinline__ void stg128(void* p, const uint4& v) { *reinterpret_cast<uint4*>(p) = v; }
__device__ __forceinline__ void stg128_stream(void* p, const uint4& v) {  // write-once data: do not pollute L1
    asm volatile("st.global.L1::no_allocate.v4.b32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ---- unaligned 16-byte window out of two aligned 16-byte chunks -----------
// Given chunk A = elements [8k, 8k+8) and chunk B = [8k+8, 8k+16) of a row of
// 16-bit elements and a shift s in [0,8), returns elements [8k+s, 8k+s+8).
// `s` is uniform across the threads that handle the same tile column, so the
// switch does not diverge.
__device__ __forceinline__ uint4 window16(const uint4& A, const uint4& B, int s) {
    const uint32_t sh = (uint32_t)(s & 1) * 16u;
    uint4 o;
    switch (s >> 1) {
        case 0:
            o.x = __funnelshift_r(A.x, A.y, sh); o.y = __funnelshift_r(A.y, A.z, sh);
            o.z = __funnelshift_r(A.z, A.w, sh); o.w = __funnelshift_r(A.w, B.x, sh);
            break;
        case 1:
            o.x = __funnelshift_r(A.y, A.z, sh); o.y = __funnelshift_r(A.z, A.w, sh);
            o.z = __funnelshift_r(A.w, B.x, sh); o.w = __funnelshift_r(B.x, B.y, sh);
            break;
        case 2:
            o.x = __funnelshift_r(A.z, A.w, sh); o.y = __funnelshift_r(A.w, B.x, sh);
            o.z = __funnelshift_r(B.x, B.y, sh); o.w = __funnelshift_r(B.y, B.z, sh);
            break;
        default:
            o.x = __funnelshift_r(A.w, B.x, sh); o.y = __funnelshift_r(B.x, B.y, sh);
            o.z = __funnelshift_r(B.y, B.z, sh); o.w = __funnelshift_r(B.z, B.w, sh);
            break;
    }
    return o;
}
// Same for 32-bit elements: chunk = 4 elements, shift s in [0,4).
__device__ __forceinline__ uint4 window32(const uint4& A, const uint4& B, int s) {
    switch (s) {
        case 0: return A;
        case 1: return make_uint4(A.y, A.z, A.w, B.x);
        case 2: return make_uint4(A.z, A.w, B.x, B.y);
        default: return make_uint4(A.w, B.x, B.y, B.z);
    }
}

template <typename T> struct Vec {  // one 16-byte vector of T
    static constexpr int kElems = 16 / (int)sizeof(T);
    static constexpr int kLog2 = (sizeof(T) == 2) ? 3 : 2;
    __device__ static __forceinline__ uint4 window(const uint4& A, const uint4& B, int s) {
        if constexpr (sizeof(T) == 2) return window16(A, B, s);
        else return window32(A, B, s);
    }
    // element j of a packed vector as fp32
    __device__ static __forceinline__ float get(const uint4& v, int j) {
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        if constexpr (sizeof(T) == 2) {
            const uint32_t word = w[j >> 1];
            return Elem<T>::bits_to_f32((uint16_t)((j & 1) ? (word >> 16) : (word & 0xffffu)));
        } else {
            return __uint_as_float(w[j]);
        }
    }
};

// number of entries <= val in a non-decreasing int16 array (upper bound)
__device__ __forceinline__ int upper_bound16(const short* a, int n, int val) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if ((int)a[mid] <= val) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// largest i with a[i] <= val (or -1); `a` non-decreasing.  The estimate `inv_d` only affects speed, never the result.
__device__ __forceinline__ int last_le(const short* a, int n, int val, float inv_d) {
    int i = min(n - 1, max(0, (int)((float)val * inv_d)));
    while (i + 1 < n && (int)a[i + 1] <= val) ++i;
    while (i >= 0 && (int)a[i] > val) --i;
    return i;
}

// floor(n / d) for n, d < 2^16 with magic = ceil(2^32 / d) (magic_u16, td_launch.h); d == 1 is passed as magic 0.
__device__ __forceinline__ unsigned fastdiv(unsigned n, unsigned magic) { return magic ? __umulhi(n, magic) : n; }

// ---- packed 16-byte arithmetic -----------------------------------------------
// acc (+)= e on one 32-bit word of packed T, rounded through T: round_half(a + b) of the exact sum equals torch's
// half(float(a) + float(b)) (fp32 has >= 2p+2 bits: double rounding is innocuous)
template <typename T> __device__ __forceinline__ uint32_t packed_add(uint32_t a, uint32_t b);
template <> __device__ __forceinline__ uint32_t packed_add<__half>(uint32_t a, uint32_t b) {
    __half2 r = __hadd2(*reinterpret_cast<__half2*>(&a), *reinterpret_cast<__half2*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
}
template <> __device__ __forceinline__ uint32_t packed_add<__nv_bfloat16>(uint32_t a, uint32_t b) {
    __nv_bfloat162 r = __hadd2(*reinterpret_cast<__nv_bfloat162*>(&a), *reinterpret_cast<__nv_bfloat162*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
}
template <> __device__ __forceinline__ uint32_t packed_add<float>(uint32_t a, uint32_t b) {
    return __float_as_uint(__fadd_rn(__uint_as_float(a), __uint_as_float(b)));
}

// a / w correctly rounded, for w a positive integer <= 4096 with rcp = its correctly rounded reciprocal and a any 16-bit
// float value (checked exhaustively by td_debug_check_fast_div)
__device__ __forceinline__ float div_exact_small_int(float a, float w, float rcp) {
    const float q = __fmul_rn(a, rcp);
    const float r = __fmaf_rn(-q, w, a);
    const float q2 = __fmaf_rn(r, rcp, q);
    // w > 0: the quotient carries a's sign (this also keeps -0 / w = -0, which the fma chain turns into +0)
    return __uint_as_float((__float_as_uint(q2) & 0x7fffffffu) | (__float_as_uint(a) & 0x80000000u));
}

// ---- launch and cross-GPU ordering -------------------------------------------
// Programmatic dependent launch (sm_90+): a kernel launched with the stream-serialisation attribute (launch(), td_launch.h)
// may become resident while its predecessor in the stream drains.  pdl_wait() blocks until the predecessor has completed
// and its memory is visible -- it precedes every global read or write of the kernels, so stream order is kept; what
// overlaps is the launch itself, the parameter fetch and the index arithmetic.  Both are no-ops for an ordinary launch.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// Spin until *flag >= want (modulo 2^32), loading with acquire semantics at system scope: what the GPU that released the
// flag wrote before it is then visible to this thread (and, after a barrier, to its CTA).  Bounded: a peer that never
// signals (crashed / interrupted rank) becomes a launch error, not a hung GPU.
__device__ __forceinline__ void spin_until_ge(const uint32_t* flag, uint32_t want) {
    uint32_t v;
    unsigned long long spins = 0;
    do {
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
        if (++spins > (1ull << 31)) __trap();
    } while ((int32_t)(v - want) < 0);
}

}  // namespace td
