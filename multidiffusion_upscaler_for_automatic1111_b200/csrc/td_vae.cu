// Tiled-VAE hot path on sm_90a (scripts/tilevae.py of the reference):
//
//   td_gn_stats        <- get_var_mean            tilevae.py:207-215   one read of the activation
//   td_gn_apply        <- custom_group_norm       tilevae.py:218-245   } one read + one write
//                         + inplace_nonlinearity  tilevae.py:102-104   } (reference: 4 R+W passes)
//   td_copy_region     <- tile crop               tilevae.py:532-535   (reference: through HOST RAM)
//                         crop_valid_region+paste tilevae.py:248-259,632
//   td_resample_nearest, td_affine_clamp <- fast-mode estimator input  tilevae.py:545-559
//   td_vae_split_tiles <- split_tiles / get_best_tile_size             tilevae.py:390-462
//   td_vae_active_tiles   (new) the output rectangles an image-space inpaint mask reaches
//
// All HBM-bound streaming kernels: 128-bit vector access, fp32 statistics merged with
// warp shuffles (Chan's parallel update: no E[x^2]-E[x]^2 cancellation), grids sized to
// keep every SM busy.  No tensor cores on purpose (the convolutions are the dense part).
#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <vector>

#include "td_b200.h"
#include "td_device.cuh"
#include "td_internal.h"
#include "td_launch.h"

namespace {

using namespace td;

struct Moments {  // count, mean, sum of squared deviations, min, max
    float n, mean, m2, lo, hi;
};

__device__ __forceinline__ Moments merge(const Moments& a, const Moments& b) {
    if (b.n == 0.0f) return a;
    if (a.n == 0.0f) return b;
    Moments r;
    r.n = a.n + b.n;
    const float d = b.mean - a.mean;
    const float f = b.n / r.n;
    r.mean = a.mean + d * f;
    r.m2 = a.m2 + b.m2 + d * d * a.n * f;
    r.lo = fminf(a.lo, b.lo);
    r.hi = fmaxf(a.hi, b.hi);
    return r;
}

__device__ __forceinline__ Moments shfl_down(const Moments& m, int off) {
    Moments r;
    r.n = __shfl_down_sync(0xffffffffu, m.n, off);
    r.mean = __shfl_down_sync(0xffffffffu, m.mean, off);
    r.m2 = __shfl_down_sync(0xffffffffu, m.m2, off);
    r.lo = __shfl_down_sync(0xffffffffu, m.lo, off);
    r.hi = __shfl_down_sync(0xffffffffu, m.hi, off);
    return r;
}

__device__ __forceinline__ Moments block_merge(Moments m, Moments* s_part) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m = merge(m, shfl_down(m, off));
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_part[warp] = m;
    __syncthreads();
    if (warp == 0) {
        const int nw = blockDim.x >> 5;
        m = lane < nw ? s_part[lane] : Moments{0.f, 0.f, 0.f, FLT_MAX, -FLT_MAX};
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) m = merge(m, shfl_down(m, off));
    }
    return m;  // valid in thread 0
}

// per-thread accumulator on data shifted by the first value seen (keeps the sum of squares small:
// no E[x^2] - E[x]^2 cancellation).  3 fp32 ops per element; min / max only when asked for.
template <bool MINMAX>
struct Shifted {
    float k, s, ss, lo, hi;
    int n;
    __device__ __forceinline__ void init(float first) { k = first; s = 0.f; ss = 0.f; n = 0; lo = FLT_MAX; hi = -FLT_MAX; }
    __device__ __forceinline__ void add(float x) {
        const float d = x - k;
        s += d;
        ss = fmaf(d, d, ss);
        if constexpr (MINMAX) { lo = fminf(lo, x); hi = fmaxf(hi, x); }
    }
    __device__ __forceinline__ Moments moments() const {
        Moments m;
        m.n = (float)n;
        if (n == 0) { m.mean = 0.f; m.m2 = 0.f; m.lo = FLT_MAX; m.hi = -FLT_MAX; return m; }
        const float md = s / m.n;
        m.mean = k + md;
        m.m2 = fmaxf(ss - s * md, 0.f);
        m.lo = lo; m.hi = hi;
        return m;
    }
};

constexpr int kStatThreads = 256;

// One CTA reduces `chunk` elements of one contiguous segment (= one (batch, group)).
template <typename T, bool VECTOR, bool MINMAX>
__global__ void __launch_bounds__(kStatThreads)
gn_stats_partial_kernel(const T* __restrict__ x, long long seg_len, long long chunk, int chunks_per_seg, float* __restrict__ ws) {
    constexpr int VEC = Vec<T>::kElems;
    __shared__ Moments s_part[kStatThreads / 32];
    const int seg = blockIdx.y, ck = blockIdx.x;
    const T* base = x + (long long)seg * seg_len;
    const long long lo = (long long)ck * chunk, hi = min(lo + chunk, seg_len);
    Shifted<MINMAX> acc;
    acc.init(lo < hi ? Elem<T>::to_f32(base[lo]) : 0.f);   // block-uniform shift: the chunk's first element
    if constexpr (VECTOR) {
        const long long v_lo = lo / VEC, v_hi = hi / VEC;   // chunk and seg_len are multiples of VEC on this path
        for (long long v = v_lo + threadIdx.x; v < v_hi; v += 4 * kStatThreads) {
            uint4 q[4];
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (v + (long long)u * kStatThreads < v_hi) q[u] = ldg128(base + (v + (long long)u * kStatThreads) * VEC);
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (v + (long long)u * kStatThreads < v_hi) {
#pragma unroll
                    for (int j = 0; j < VEC; ++j) acc.add(Vec<T>::get(q[u], j));
                    acc.n += VEC;   // counted per vector, not per element
                }
        }
    } else {
        for (long long i = lo + threadIdx.x; i < hi; i += kStatThreads) { acc.add(Elem<T>::to_f32(base[i])); acc.n += 1; }
    }
    const Moments m = block_merge(acc.moments(), s_part);
    if (threadIdx.x == 0) {
        float* o = ws + ((long long)seg * chunks_per_seg + ck) * 5;
        o[0] = m.n; o[1] = m.mean; o[2] = m.m2; o[3] = m.lo; o[4] = m.hi;
    }
}

// One warp per segment merges the per-CTA partials.
__global__ void gn_stats_final_kernel(const float* __restrict__ ws, int chunks_per_seg, int nseg, float* __restrict__ mean,
                                      float* __restrict__ var, float* __restrict__ lo, float* __restrict__ hi, int unbiased) {
    const int seg = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (seg >= nseg) return;
    const int lane = threadIdx.x & 31;
    Moments m{0.f, 0.f, 0.f, FLT_MAX, -FLT_MAX};
    for (int k = lane; k < chunks_per_seg; k += 32) {
        const float* p = ws + ((long long)seg * chunks_per_seg + k) * 5;
        m = merge(m, Moments{p[0], p[1], p[2], p[3], p[4]});
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m = merge(m, shfl_down(m, off));
    if (lane == 0) {
        mean[seg] = m.mean;
        // an unbiased one-element segment gets 0 (torch: NaN); fast mode never asks for one
        var[seg] = m.m2 / (unbiased ? fmaxf(m.n - 1.f, 1.f) : m.n);
        if (lo) lo[seg] = m.lo;
        if (hi) hi[seg] = m.hi;
    }
}

// SiLU with the SFU approximations (ex2.approx + rcp.approx, ~1e-6 relative): two MUFU per element keep the
// kernel under its HBM time; the result is rounded to fp16 / bf16 (or compared at 3e-4 in fp32) anyway.
__device__ __forceinline__ float silu_f(float v) { return __fdividef(v, 1.0f + __expf(-v)); }

// y = act(((x - mean) * invstd) * gamma + beta): one CTA walks part of one (b, c) plane.
template <typename T, bool VECTOR>
__global__ void __launch_bounds__(256)
gn_apply_kernel(const T* __restrict__ x, T* __restrict__ y, int C, long long HW, int cpg, int groups,
                const float* __restrict__ mean, const float* __restrict__ var, const float* __restrict__ gamma,
                const float* __restrict__ beta, float eps, int act, int stats_per_batch) {
    constexpr int VEC = Vec<T>::kElems;
    const int plane = blockIdx.y;           // b * C + c
    const int b = plane / C, c = plane - b * C;
    const int sidx = (stats_per_batch ? b * groups : 0) + c / cpg;
    const float mu = mean[sidx];
    const float invstd = __fdiv_rn(1.0f, __fsqrt_rn(var[sidx] + eps));
    const float ga = gamma ? gamma[c] : 1.0f, be = beta ? beta[c] : 0.0f;
    const T* xp = x + (long long)plane * HW;
    T* yp = y + (long long)plane * HW;
    // ((v - mu) * invstd) * ga + be folded into one FMA per element (per-plane constants)
    const float A = invstd * ga, Bc = fmaf(-mu, A, be);
    auto f = [&](float v) {
        const float t = fmaf(v, A, Bc);
        return act ? silu_f(t) : t;
    };
    if constexpr (VECTOR) {
        const long long nv = HW / VEC;
        for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < nv; v += (long long)gridDim.x * blockDim.x) {
            const uint4 q = ldg128(xp + v * VEC);
            uint4 o;
            if constexpr (sizeof(T) == 2) {
                uint32_t w[4];
#pragma unroll
                for (int h = 0; h < 4; ++h)
                    w[h] = (uint32_t)Elem<T>::f32_to_bits(f(Vec<T>::get(q, 2 * h))) |
                           ((uint32_t)Elem<T>::f32_to_bits(f(Vec<T>::get(q, 2 * h + 1))) << 16);
                o = make_uint4(w[0], w[1], w[2], w[3]);
            } else {
                o = make_uint4(__float_as_uint(f(__uint_as_float(q.x))), __float_as_uint(f(__uint_as_float(q.y))),
                               __float_as_uint(f(__uint_as_float(q.z))), __float_as_uint(f(__uint_as_float(q.w))));
            }
            stg128(yp + v * VEC, o);
        }
    } else {
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (long long)gridDim.x * blockDim.x)
            yp[i] = Elem<T>::from_f32(f(Elem<T>::to_f32(xp[i])));
    }
}

// dst[p, r, c] = src[p, r, c] over a [planes, rows, cols] region of two strided tensors.
template <typename T, bool VECTOR>
__global__ void __launch_bounds__(256)
copy_region_kernel(const T* __restrict__ src, T* __restrict__ dst, int rows, int cols, long long src_plane, long long src_pitch,
                   long long dst_plane, long long dst_pitch) {
    constexpr int VEC = Vec<T>::kElems;
    const int p = blockIdx.z;
    const T* s = src + (long long)p * src_plane;
    T* d = dst + (long long)p * dst_plane;
    const int cv = VECTOR ? cols / VEC : cols;
    for (int r = blockIdx.y; r < rows; r += gridDim.y)
        for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < cv; c += gridDim.x * blockDim.x) {
            if constexpr (VECTOR) stg128(d + r * dst_pitch + (long long)c * VEC, ldg128(s + r * src_pitch + (long long)c * VEC));
            else d[r * dst_pitch + c] = s[r * src_pitch + c];
        }
}

// out[p, i, j] = in[p, sy[i], sx[j]]   (nearest-exact gather with host-computed index tables)
template <typename T>
__global__ void __launch_bounds__(256)
resample_kernel(const T* __restrict__ in, T* __restrict__ out, int H, int W, int oh, int ow, const int* __restrict__ sy,
                const int* __restrict__ sx) {
    const int p = blockIdx.z;
    for (int i = blockIdx.y; i < oh; i += gridDim.y)
        for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < ow; j += gridDim.x * blockDim.x)
            out[((long long)p * oh + i) * ow + j] = in[((long long)p * H + sy[i]) * W + sx[j]];
}

// x = clamp((x - mean_new[c]) / std_new[c] * std_old[c] + mean_old[c], lo, hi)   in place, per channel
template <typename T>
__global__ void __launch_bounds__(256)
affine_clamp_kernel(T* __restrict__ x, int C, long long HW, const float* __restrict__ mean_new, const float* __restrict__ std_new,
                    const float* __restrict__ mean_old, const float* __restrict__ std_old, const float* __restrict__ lo,
                    const float* __restrict__ hi) {
    const int plane = blockIdx.y, c = plane % C;
    const float mn = mean_new[c], sn = std_new[c], mo = mean_old[c], so = std_old[c];
    const float l = lo[0], h = hi[0];
    T* p = x + (long long)plane * HW;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (long long)gridDim.x * blockDim.x) {
        // torch evaluates each op in the tensor dtype: round through T after every step.  The _rn intrinsics keep
        // `* so + mo` from being contracted into one FMA where round_through is the identity (fp32).
        float v = Elem<T>::to_f32(p[i]);
        v = round_through<T>(__fsub_rn(v, mn));
        v = round_through<T>(__fdiv_rn(v, sn));
        v = round_through<T>(__fmul_rn(v, so));
        v = round_through<T>(__fadd_rn(v, mo));
        // torch.clamp's NaN rule: a NaN operand stays NaN, else a NaN bound is the result.  A constant channel makes
        // the estimator's (x - mean_new) / std_new 0 / 0; the NaN must reach the caller, which then disables fast mode.
        p[i] = Elem<T>::from_f32(isnan(v) ? v : isnan(l) ? l : isnan(h) ? h : fminf(fmaxf(v, l), h));
    }
}


struct StatPlan {
    long long seg_len, chunk;
    int nseg, chunks;
    bool vec;
};

StatPlan plan_stats(const void* x, long long nseg, long long seg_len, int dtype) {
    StatPlan p;
    const int es = td_dtype_size(dtype), vec = 16 / es;
    p.nseg = (int)nseg; p.seg_len = seg_len;
    p.vec = aligned16(x) && (seg_len % vec == 0);
    // ~64 KB per CTA, at least ~4 CTAs per SM overall, at most 1024 chunks per segment
    long long chunk = 65536 / es;
    long long chunks = (seg_len + chunk - 1) / chunk;
    const long long want = (148LL * 4 + nseg - 1) / nseg;
    if (chunks < want) chunks = std::min(want, std::max(1LL, seg_len / (kStatThreads * vec)));
    chunks = std::max(1LL, std::min(chunks, 1024LL));
    chunk = (seg_len + chunks - 1) / chunks;
    chunk = (chunk + vec - 1) / vec * vec;
    p.chunks = (int)((seg_len + chunk - 1) / chunk);
    p.chunk = chunk;
    return p;
}

}  // namespace

extern "C" int64_t td_gn_stats_workspace_bytes(int64_t nseg, int64_t seg_len, int dtype) {
    if (nseg <= 0 || seg_len <= 0 || td_dtype_size(dtype) == 0) return 0;
    return nseg * 1024 * 5 * (int64_t)sizeof(float);  // upper bound: 1024 chunks per segment
}

extern "C" int td_gn_stats(const void* x, int64_t nseg, int64_t seg_len, int dtype, int unbiased, void* workspace,
                           int64_t workspace_bytes, float* mean, float* var, float* seg_min, float* seg_max, void* stream) {
    if (x == nullptr || mean == nullptr || var == nullptr || workspace == nullptr || nseg <= 0 || seg_len <= 0) {
        td_set_error("td_gn_stats: bad arguments");
        return TD_ERR_INVALID_ARG;
    }
    if (td_dtype_size(dtype) == 0) { td_set_error("td_gn_stats: unknown dtype %d", dtype); return TD_ERR_INVALID_ARG; }
    if (nseg > 65535) { td_set_error("td_gn_stats: %lld segments exceed the grid limit", (long long)nseg); return TD_ERR_UNSUPPORTED; }
    const StatPlan p = plan_stats(x, nseg, seg_len, dtype);
    if ((int64_t)p.nseg * p.chunks * 5 * (int64_t)sizeof(float) > workspace_bytes) {
        td_set_error("td_gn_stats: workspace too small");
        return TD_ERR_CAPACITY;
    }
    cudaStream_t s = (cudaStream_t)stream;
    dim3 grid((unsigned)p.chunks, (unsigned)p.nseg);
    float* ws = (float*)workspace;
    const bool mm = seg_min != nullptr || seg_max != nullptr;
#define TD_LAUNCH(T) \
    if (p.vec && mm) gn_stats_partial_kernel<T, true, true><<<grid, kStatThreads, 0, s>>>((const T*)x, p.seg_len, p.chunk, p.chunks, ws); \
    else if (p.vec) gn_stats_partial_kernel<T, true, false><<<grid, kStatThreads, 0, s>>>((const T*)x, p.seg_len, p.chunk, p.chunks, ws); \
    else gn_stats_partial_kernel<T, false, true><<<grid, kStatThreads, 0, s>>>((const T*)x, p.seg_len, p.chunk, p.chunks, ws);
    if (dtype == TD_F16) { TD_LAUNCH(__half) } else if (dtype == TD_BF16) { TD_LAUNCH(__nv_bfloat16) } else { TD_LAUNCH(float) }
#undef TD_LAUNCH
    int st = launch_status("td_gn_stats (partial)");
    if (st != TD_OK) return st;
    gn_stats_final_kernel<<<(unsigned)((p.nseg + 7) / 8), 256, 0, s>>>(ws, p.chunks, p.nseg, mean, var, seg_min, seg_max, unbiased);
    return launch_status("td_gn_stats (final)");
}

extern "C" int td_gn_apply(const void* x, void* y, int B, int C, int64_t HW, int dtype, int groups, const float* mean,
                           const float* var, int stats_per_batch, const float* gamma, const float* beta, float eps, int act,
                           void* stream) {
    if (x == nullptr || y == nullptr || mean == nullptr || var == nullptr || B <= 0 || C <= 0 || HW <= 0 || groups <= 0) {
        td_set_error("td_gn_apply: bad arguments");
        return TD_ERR_INVALID_ARG;
    }
    if (C % groups != 0) { td_set_error("td_gn_apply: C=%d not divisible by %d groups", C, groups); return TD_ERR_INVALID_ARG; }
    const int es = td_dtype_size(dtype);
    if (es == 0) { td_set_error("td_gn_apply: unknown dtype %d", dtype); return TD_ERR_INVALID_ARG; }
    if ((long long)B * C > 65535) { td_set_error("td_gn_apply: B*C too large"); return TD_ERR_UNSUPPORTED; }
    const int vec = 16 / es;
    const bool v = aligned16(x) && aligned16(y) && HW % vec == 0;
    const long long per_thread = v ? HW / vec : HW;
    long long bx = (per_thread + 256 * 4 - 1) / (256 * 4);   // ~4 vectors per thread
    bx = std::max(1LL, std::min(bx, 4096LL));
    dim3 grid((unsigned)bx, (unsigned)(B * C));
    cudaStream_t s = (cudaStream_t)stream;
    const int cpg = C / groups;
#define TD_LAUNCH(T) \
    if (v) gn_apply_kernel<T, true><<<grid, 256, 0, s>>>((const T*)x, (T*)y, C, HW, cpg, groups, mean, var, gamma, beta, eps, act, stats_per_batch); \
    else gn_apply_kernel<T, false><<<grid, 256, 0, s>>>((const T*)x, (T*)y, C, HW, cpg, groups, mean, var, gamma, beta, eps, act, stats_per_batch);
    if (dtype == TD_F16) { TD_LAUNCH(__half) } else if (dtype == TD_BF16) { TD_LAUNCH(__nv_bfloat16) } else { TD_LAUNCH(float) }
#undef TD_LAUNCH
    return launch_status("td_gn_apply");
}

extern "C" int td_copy_region(const void* src, void* dst, int planes, int rows, int cols, int64_t src_plane_stride,
                              int64_t src_pitch, int64_t dst_plane_stride, int64_t dst_pitch, int dtype, void* stream) {
    if (src == nullptr || dst == nullptr || planes < 0 || rows < 0 || cols < 0) { td_set_error("td_copy_region: bad arguments"); return TD_ERR_INVALID_ARG; }
    const int es = td_dtype_size(dtype);
    if (es == 0) { td_set_error("td_copy_region: unknown dtype %d", dtype); return TD_ERR_INVALID_ARG; }
    if (planes == 0 || rows == 0 || cols == 0) return TD_OK;
    if (planes > 65535) { td_set_error("td_copy_region: too many planes"); return TD_ERR_UNSUPPORTED; }
    const int vec = 16 / es;
    const bool v = aligned16(src) && aligned16(dst) && cols % vec == 0 && src_pitch % vec == 0 && dst_pitch % vec == 0 &&
                   src_plane_stride % vec == 0 && dst_plane_stride % vec == 0;
    const int cv = v ? cols / vec : cols;
    dim3 grid((unsigned)std::max(1, std::min((cv + 255) / 256, 64)), (unsigned)std::min(rows, 65535), (unsigned)planes);
    cudaStream_t s = (cudaStream_t)stream;
    // 16-bit types are moved as opaque words
#define TD_LAUNCH(T) \
    if (v) copy_region_kernel<T, true><<<grid, 256, 0, s>>>((const T*)src, (T*)dst, rows, cols, src_plane_stride, src_pitch, dst_plane_stride, dst_pitch); \
    else copy_region_kernel<T, false><<<grid, 256, 0, s>>>((const T*)src, (T*)dst, rows, cols, src_plane_stride, src_pitch, dst_plane_stride, dst_pitch);
    if (es == 2) { TD_LAUNCH(__half) } else { TD_LAUNCH(float) }
#undef TD_LAUNCH
    return launch_status("td_copy_region");
}

extern "C" int td_resample_nearest(const void* in, void* out, int planes, int H, int W, int oh, int ow, const int32_t* src_y,
                                   const int32_t* src_x, int dtype, void* stream) {
    if (in == nullptr || out == nullptr || src_y == nullptr || src_x == nullptr || planes <= 0 || oh <= 0 || ow <= 0) {
        td_set_error("td_resample_nearest: bad arguments");
        return TD_ERR_INVALID_ARG;
    }
    const int es = td_dtype_size(dtype);
    if (es == 0) { td_set_error("td_resample_nearest: unknown dtype %d", dtype); return TD_ERR_INVALID_ARG; }
    if (planes > 65535) { td_set_error("td_resample_nearest: too many planes"); return TD_ERR_UNSUPPORTED; }
    dim3 grid((unsigned)std::max(1, std::min((ow + 255) / 256, 64)), (unsigned)std::min(oh, 65535), (unsigned)planes);
    cudaStream_t s = (cudaStream_t)stream;
    if (es == 2) resample_kernel<__half><<<grid, 256, 0, s>>>((const __half*)in, (__half*)out, H, W, oh, ow, src_y, src_x);
    else resample_kernel<float><<<grid, 256, 0, s>>>((const float*)in, (float*)out, H, W, oh, ow, src_y, src_x);
    return launch_status("td_resample_nearest");
}

extern "C" int td_affine_clamp(void* x, int B, int C, int64_t HW, int dtype, const float* mean_new, const float* std_new,
                               const float* mean_old, const float* std_old, const float* lo, const float* hi, void* stream) {
    if (x == nullptr || mean_new == nullptr || std_new == nullptr || mean_old == nullptr || std_old == nullptr || lo == nullptr ||
        hi == nullptr || B <= 0 || C <= 0 || HW <= 0) {
        td_set_error("td_affine_clamp: bad arguments");
        return TD_ERR_INVALID_ARG;
    }
    if ((long long)B * C > 65535) { td_set_error("td_affine_clamp: B*C too large"); return TD_ERR_UNSUPPORTED; }
    dim3 grid((unsigned)std::max(1LL, std::min((long long)(HW + 1023) / 1024, 1024LL)), (unsigned)(B * C));
    cudaStream_t s = (cudaStream_t)stream;
    if (dtype == TD_F16) affine_clamp_kernel<__half><<<grid, 256, 0, s>>>((__half*)x, C, HW, mean_new, std_new, mean_old, std_old, lo, hi);
    else if (dtype == TD_BF16) affine_clamp_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>((__nv_bfloat16*)x, C, HW, mean_new, std_new, mean_old, std_old, lo, hi);
    else if (dtype == TD_F32) affine_clamp_kernel<float><<<grid, 256, 0, s>>>((float*)x, C, HW, mean_new, std_new, mean_old, std_old, lo, hi);
    else { td_set_error("td_affine_clamp: unknown dtype %d", dtype); return TD_ERR_INVALID_ARG; }
    return launch_status("td_affine_clamp");
}

// ---- inpainting: the output rectangles an image-space mask reaches ---------------------------
namespace {

constexpr int kActiveThreads = 256;
constexpr int kActiveRows = 16;                 // mask rows (over all planes) per CTA: ~24 KB of a cfg4 fp16 rectangle
constexpr int kActiveRectsPerLaunch = 128;      // rectangles passed by value per launch (2 KB of parameters)

struct ActiveRects {
    int32_t r[kActiveRectsPerLaunch][4];        // [x1, x2, y1, y2]
};

// 1.0 in two packed 16-bit elements / one fp32: an element equals 1.0 exactly when its bits are these (1.0 has one encoding
// and a NaN never has it), so a 16-byte vector is tested with four integer compares
template <typename T> struct OneWord;
template <> struct OneWord<__half> { static constexpr uint32_t kBits = 0x3C003C00u; };
template <> struct OneWord<__nv_bfloat16> { static constexpr uint32_t kBits = 0x3F803F80u; };
template <> struct OneWord<float> { static constexpr uint32_t kBits = 0x3F800000u; };

// CTA (x, y): rows [x * kActiveRows, +kActiveRows) of rectangle y's planes * (y2 - y1) rows, one warp per row.  A row segment
// is read with 16-byte loads from its first 16-byte boundary on, its ragged ends element by element.  A CTA that finds an
// element != 1.0 stores 1; a CTA whose rectangle is already flagged reads nothing.
template <typename T>
__global__ void __launch_bounds__(kActiveThreads)
vae_active_tiles_kernel(const __grid_constant__ ActiveRects rects, const T* __restrict__ mask, int planes, int H, int W,
                        uint8_t* __restrict__ active) {
    constexpr int VEC = Vec<T>::kElems;
    constexpr uint32_t kOne = OneWord<T>::kBits;
    __shared__ int s_done;
    const int32_t* b = rects.r[blockIdx.y];
    const int x1 = b[0], n = b[1] - b[0], y1 = b[2], h = b[3] - b[2];
    const long long rows = (long long)planes * h;
    const long long j0 = (long long)blockIdx.x * kActiveRows, j1 = min(j0 + kActiveRows, rows);
    if (j0 >= rows) return;
    if (threadIdx.x == 0) s_done = *(volatile const uint8_t*)&active[blockIdx.y];
    __syncthreads();
    if (s_done) return;
    const int lane = threadIdx.x & 31;
    int found = 0;
    for (long long j = j0 + (threadIdx.x >> 5); j < j1; j += kActiveThreads / 32) {
        const long long pl = j / h, y = y1 + (j - pl * h);
        const T* row = mask + (pl * H + y) * W + x1;
        const int head = min(n, (int)(((16u - ((uintptr_t)row & 15u)) & 15u) / sizeof(T)));
        const int nv = (n - head) / VEC;
        const T* body = row + head;
        for (int v = lane; v < nv; v += 32) {
            const uint4 q = ldg128(body + (long long)v * VEC);
            found |= (q.x != kOne) | (q.y != kOne) | (q.z != kOne) | (q.w != kOne);
        }
        for (int i = lane; i < head; i += 32) found |= !(Elem<T>::to_f32(row[i]) == 1.0f);
        for (int i = head + nv * VEC + lane; i < n; i += 32) found |= !(Elem<T>::to_f32(row[i]) == 1.0f);
    }
    if (__syncthreads_or(found) && threadIdx.x == 0) active[blockIdx.y] = 1;
}

}  // namespace

extern "C" int td_vae_active_tiles(const void* mask, int planes, int H, int W, int dtype, const int32_t* rects_host, int n_rects,
                                   uint8_t* active_dev, void* stream) {
    const int es = td_dtype_size(dtype);
    if (es == 0) { td_set_error("td_vae_active_tiles: unknown dtype %d", dtype); return TD_ERR_INVALID_ARG; }
    if (mask == nullptr || active_dev == nullptr || rects_host == nullptr || ((uintptr_t)mask % (uintptr_t)es) != 0) {
        td_set_error("td_vae_active_tiles: null or misaligned mask / rectangles / output");
        return TD_ERR_INVALID_ARG;
    }
    if (planes <= 0 || H <= 0 || W <= 0 || n_rects <= 0) {
        td_set_error("td_vae_active_tiles: planes = %d, H = %d, W = %d, n_rects = %d must be positive", planes, H, W, n_rects);
        return TD_ERR_INVALID_ARG;
    }
    for (int t = 0; t < n_rects; ++t) {
        const int32_t* b = rects_host + 4LL * t;
        if (!(0 <= b[0] && b[0] < b[1] && b[1] <= W && 0 <= b[2] && b[2] < b[3] && b[3] <= H)) {
            td_set_error("td_vae_active_tiles: rectangle %d = [%d, %d) x [%d, %d) is empty or leaves the %d x %d mask", t, b[0], b[1],
                         b[2], b[3], W, H);
            return TD_ERR_INVALID_ARG;
        }
    }
    if ((long long)planes * H > INT32_MAX) {
        td_set_error("td_vae_active_tiles: %lld mask rows exceed the grid limit", (long long)planes * H);
        return TD_ERR_UNSUPPORTED;
    }
    cudaStream_t s = (cudaStream_t)stream;
    int st = launch_status("td_vae_active_tiles (zero)", cudaMemsetAsync(active_dev, 0, (size_t)n_rects, s));
    if (st != TD_OK) return st;
    for (int r0 = 0; r0 < n_rects; r0 += kActiveRectsPerLaunch) {
        const int k = std::min(kActiveRectsPerLaunch, n_rects - r0);
        ActiveRects p;
        long long rows = 0;
        for (int t = 0; t < k; ++t) {
            for (int e = 0; e < 4; ++e) p.r[t][e] = rects_host[4LL * (r0 + t) + e];
            rows = std::max(rows, (long long)planes * (p.r[t][3] - p.r[t][2]));
        }
        const dim3 grid((unsigned)((rows + kActiveRows - 1) / kActiveRows), (unsigned)k);
#define TD_LAUNCH(T) vae_active_tiles_kernel<T><<<grid, kActiveThreads, 0, s>>>(p, (const T*)mask, planes, H, W, active_dev + r0)
        if (dtype == TD_F16) TD_LAUNCH(__half);
        else if (dtype == TD_BF16) TD_LAUNCH(__nv_bfloat16);
        else TD_LAUNCH(float);
#undef TD_LAUNCH
        if ((st = launch_status("td_vae_active_tiles")) != TD_OK) return st;
    }
    return TD_OK;
}

// ---- host bookkeeping ----------------------------------------------------------------------
extern "C" int td_vae_best_tile_size(int lowerbound, int upperbound) {  // tilevae.py:390-403
    int divider = 32;
    while (divider >= 2) {
        const int rem = lowerbound % divider;
        if (rem == 0) return lowerbound;
        const int cand = lowerbound - rem + divider;
        if (cand <= upperbound) return cand;
        divider /= 2;
    }
    return lowerbound;
}

namespace {

// One axis of split_tiles (tilevae.py:405-462): tile k's input span [in0, in1) and output span [out0, out1), the output
// already scaled x8 (decoder) or //8 (encoder).  The bounded rule clips the input to [0, L) and snaps the outputs at
// the borders.  The periodic rule (seamless tiling) cuts L at b_k = m * floor(k * L / (n * m)), n = max(ceil(L / tile), 1),
// m = 8 for the encoder (whole latent pixels) and 1 for the decoder, b_n = L; the input span is [b_k - pad, b_{k+1} + pad)
// in UNwrapped coordinates (it may start below 0 or end past L: the tile load reads it modulo L), so every output span
// lies inside [0, L) and the output spans partition it.
struct VaeAxis {
    int n = 0;
    std::vector<int> in0, in1, out0, out1;
    void resize(int k) { n = k; in0.resize(k); in1.resize(k); out0.resize(k); out1.resize(k); }
};

int vae_axis(int L, int tile_size, int pad, int is_decoder, bool periodic, VaeAxis* a) {
    auto ceil_div = [](int x, int y) { return (int)std::ceil((double)x / (double)y); };
    auto scale = [&](int v) { return is_decoder ? v * 8 : (int)std::floor((double)v / 8.0); };
    if (!periodic) {
        const int n = std::max(ceil_div(L - 2 * pad, tile_size), 1);
        const int real = td_vae_best_tile_size(ceil_div(L - 2 * pad, n), tile_size);
        a->resize(n);
        for (int j = 0; j < n; ++j) {
            const int b0 = pad + j * real, b1 = std::min(pad + (j + 1) * real, L);
            a->out0[j] = scale(b0 > pad ? b0 : 0);
            a->out1[j] = scale(b1 < L - pad ? b1 : L);
            a->in0[j] = std::max(0, b0 - pad);
            a->in1[j] = std::min(L, b1 + pad);
        }
        return TD_OK;
    }
    const int m = is_decoder ? 1 : 8;
    const int n = std::max(ceil_div(L, tile_size), 1);
    a->resize(n);
    auto cut = [&](int k) { return k == n ? L : m * (int)(((long long)k * L) / ((long long)n * m)); };
    for (int k = 0; k < n; ++k) {
        const int b0 = cut(k), b1 = cut(k + 1);
        a->out0[k] = scale(b0);
        a->out1[k] = scale(b1);
        a->in0[k] = b0 - pad;
        a->in1[k] = b1 + pad;
    }
    return TD_OK;
}

}  // namespace

extern "C" int td_vae_split_tiles(int h, int w, int tile_size, int pad, int is_decoder, int wrap, int32_t* in_bboxes,
                                  int32_t* out_bboxes, int cap) {  // tilevae.py:405-462; bbox order [x1, x2, y1, y2]
    if (h <= 0 || w <= 0 || tile_size <= 0 || pad < 0 || (wrap & ~(int)(TD_WRAP_X | TD_WRAP_Y)) != 0) {
        td_set_error("td_vae_split_tiles: bad arguments");
        return TD_ERR_INVALID_ARG;
    }
    VaeAxis ax, ay;
    int st = vae_axis(w, tile_size, pad, is_decoder, (wrap & TD_WRAP_X) != 0, &ax);
    if (st != TD_OK) return st;
    st = vae_axis(h, tile_size, pad, is_decoder, (wrap & TD_WRAP_Y) != 0, &ay);
    if (st != TD_OK) return st;
    const long long T = (long long)ay.n * ax.n;
    if (in_bboxes == nullptr || out_bboxes == nullptr) return (int)T;
    if (T > cap) { td_set_error("td_vae_split_tiles: %lld tiles exceed capacity %d", T, cap); return TD_ERR_CAPACITY; }
    int32_t* ib = in_bboxes;
    int32_t* ob = out_bboxes;
    for (int i = 0; i < ay.n; ++i)
        for (int j = 0; j < ax.n; ++j) {
            *ob++ = ax.out0[j]; *ob++ = ax.out1[j]; *ob++ = ay.out0[i]; *ob++ = ay.out1[i];
            *ib++ = ax.in0[j]; *ib++ = ax.in1[j]; *ib++ = ay.in0[i]; *ib++ = ay.in1[i];
        }
    return (int)T;
}
