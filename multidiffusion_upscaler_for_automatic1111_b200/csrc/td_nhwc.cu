// Channels-last (NHWC) streaming kernels around the tensor-core convolutions of the tiled VAE (td_conv.cu):
//
//   td_nchw_to_nhwc        tile crop (tilevae.py:532-535) fused with the layout change and the channel zero-padding the
//                          implicit GEMM wants (z: 4 -> 64 channels)
//   td_nhwc_to_nchw_region crop_valid_region + paste (tilevae.py:248-259, :632) fused with the layout change back
//   td_upsample2x_nhwc     Upsample's F.interpolate(scale 2, nearest) in front of its conv (ldm Upsample; queue entry
//                          'upsample', tilevae.py:163)
//   td_gn_stats_nhwc       get_var_mean (tilevae.py:207-215) on channels-last data: ONE read
//   td_gn_apply_nhwc       custom_group_norm + SiLU (tilevae.py:218-245, :102-104): one read + one write
//                          (the *_batched entries: N images in one launch, each on the grid of its one-image call)
//   td_softmax_rows        softmax over the keys of the VAE attention (tile_utils/attn.py:58-60)
//
// All HBM-bound: 128-bit accesses along the channel dimension, per-thread constants hoisted out of the pixel loop,
// statistics merged with Chan's update (no E[x^2] - E[x]^2 cancellation).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>
#include <cstdint>

#include "td_b200.h"
#include "td_device.cuh"
#include "td_internal.h"
#include "td_launch.h"

namespace {

using namespace td;

constexpr int kNhwcThreads = 256;

int nhwc_sms() {   // grid sizing only: an H100's count when the query fails
    const DeviceProps d = device_props();
    return d.ok ? d.sms : 132;
}

template <typename T> __device__ __forceinline__ float vget(const uint4& v, int j) { return Vec<T>::get(v, j); }
template <typename T> __device__ __forceinline__ uint4 vpack(const float (&f)[8]) {
    uint32_t w[4];
#pragma unroll
    for (int h = 0; h < 4; ++h) w[h] = (uint32_t)Elem<T>::f32_to_bits(f[2 * h]) | ((uint32_t)Elem<T>::f32_to_bits(f[2 * h + 1]) << 16);
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// ---------------------------------------------------------------------------------------------------------------
// NCHW region -> NHWC (channel zero-padded): y[n, i, j, c] = c < C ? x[n, c, y0 + i, x0 + j] : 0
// one thread per (pixel, 8-channel vector); reads are coalesced along j for each channel plane.
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kNhwcThreads)
nchw_to_nhwc_kernel(const T* __restrict__ x, T* __restrict__ y, int C, long long x_plane, long long x_pitch, long long x_img,
                    int rows, int cols, int Cpad, long long total) {
    const int cv = Cpad / 8;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        // vector index slowest so that consecutive threads walk consecutive pixels of one channel group (coalesced reads)
        const long long pix_total = total / cv;
        const int v = (int)(i / pix_total);
        const long long pix = i - (long long)v * pix_total;
        const int j = (int)(pix % cols);
        const long long t = pix / cols;
        const int r = (int)(t % rows);
        const long long n = t / rows;
        float f[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int c = v * 8 + k;
            f[k] = c < C ? Elem<T>::to_f32(x[n * x_img + (long long)c * x_plane + (long long)r * x_pitch + j]) : 0.0f;
        }
        *reinterpret_cast<uint4*>(y + pix * Cpad + v * 8) = vpack<T>(f);
    }
}

// The same for a tile of a periodic canvas (seamless tiling): the tile's rows / columns start at (row0, col0) in
// unwrapped coordinates and are read modulo the canvas (H, W): y[n, i, j, c] = x[n, c, (row0 + i) mod H, (col0 + j) mod W].
template <typename T>
__global__ void __launch_bounds__(kNhwcThreads)
nchw_to_nhwc_wrap_kernel(const T* __restrict__ x, T* __restrict__ y, int C, long long x_plane, long long x_pitch, long long x_img,
                         int rows, int cols, int row0, int col0, int H, int W, int Cpad, long long total) {
    const int cv = Cpad / 8;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long pix_total = total / cv;
        const int v = (int)(i / pix_total);
        const long long pix = i - (long long)v * pix_total;
        const int j = (int)(pix % cols);
        const long long t = pix / cols;
        const int r = (int)(t % rows);
        const long long n = t / rows;
        int sy = (row0 + r) % H, sx = (col0 + j) % W;
        if (sy < 0) sy += H;
        if (sx < 0) sx += W;
        float f[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int c = v * 8 + k;
            f[k] = c < C ? Elem<T>::to_f32(x[n * x_img + (long long)c * x_plane + (long long)sy * x_pitch + sx]) : 0.0f;
        }
        *reinterpret_cast<uint4*>(y + pix * Cpad + v * 8) = vpack<T>(f);
    }
}

// NHWC -> NCHW region: y[n, c, i, j] = x[n, sy + i, sx + j, c] for c < C (crop + paste + layout in one pass)
template <typename T>
__global__ void __launch_bounds__(kNhwcThreads)
nhwc_to_nchw_region_kernel(const T* __restrict__ x, T* __restrict__ y, int C, long long x_pitch, int xW, long long x_img,
                           long long y_plane, long long y_pitch, long long y_img, int rows, int cols, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int j = (int)(i % cols);
        long long t = i / cols;
        const int r = (int)(t % rows);
        t /= rows;
        const int c = (int)(t % C);
        const long long n = t / C;
        y[n * y_img + (long long)c * y_plane + (long long)r * y_pitch + j] = x[n * x_img + ((long long)r * xW + j) * x_pitch + c];
    }
}

// nearest x2: y[n, 2i + a, 2j + b, :] = x[n, i, j, :]
template <typename T>
__global__ void __launch_bounds__(kNhwcThreads)
upsample2x_nhwc_kernel(const T* __restrict__ x, T* __restrict__ y, int H, int W, int cv, long long total) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int v = (int)(i % cv);
        long long t = i / cv;
        const int j = (int)(t % W);
        t /= W;
        const int r = (int)(t % H);
        const long long n = t / H;
        const uint4 q = ldg128(x + i * 8);
        T* o = y + (((n * 2 * H + 2 * r) * 2 * W) + 2 * j) * (long long)cv * 8 + v * 8;
        const long long row = (long long)2 * W * cv * 8;
        stg128_stream(o, q);
        stg128_stream(o + cv * 8, q);
        stg128_stream(o + row, q);
        stg128_stream(o + row + cv * 8, q);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// GroupNorm statistics, channels-last.  x: [P, C] per image, groups of cpg = C / groups adjacent channels.
// A thread owns one 8-channel vector position and walks pixels; its two 4-channel halves are accumulated on data
// shifted by the first value seen, turned into (n, mean, M2) and merged per group with Chan's update:
// thread -> CTA (shared memory) -> finaliser kernel.  blockIdx.y is the image: each image runs the grid, the partials
// and the merge order of its one-image launch, so its statistics are the same bits.
// ---------------------------------------------------------------------------------------------------------------
struct Mom { float n, mean, m2; };
__device__ __forceinline__ Mom mom_merge(const Mom& a, const Mom& b) {
    if (b.n == 0.0f) return a;
    if (a.n == 0.0f) return b;
    Mom r;
    r.n = a.n + b.n;
    const float d = b.mean - a.mean, f = b.n / r.n;
    r.mean = a.mean + d * f;
    r.m2 = a.m2 + b.m2 + d * d * a.n * f;
    return r;
}

template <typename T>
__global__ void __launch_bounds__(kNhwcThreads)
gn_stats_nhwc_partial_kernel(const T* __restrict__ x, long long P, int C, int groups, float* __restrict__ ws) {
    __shared__ Mom s_m[kNhwcThreads * 2];
    x += (long long)blockIdx.y * P * C;
    ws += (long long)blockIdx.y * gridDim.x * groups * 3;
    const int cv = C / 8, cpg = C / groups;
    const int ppi = kNhwcThreads / cv;                 // pixels per CTA iteration
    const int v = threadIdx.x % cv, pl = threadIdx.x / cv;
    float k0 = 0.f, k1 = 0.f, s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
    long long cnt = 0;
    if (pl < ppi) {
        bool first = true;
        for (long long p = (long long)blockIdx.x * ppi + pl; p < P; p += (long long)gridDim.x * ppi) {
            const uint4 u = ldg128(x + p * C + v * 8);
            if (first) { k0 = vget<T>(u, 0); k1 = vget<T>(u, 4); first = false; }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float d0 = vget<T>(u, j) - k0, d1 = vget<T>(u, 4 + j) - k1;
                s0 += d0; q0 = fmaf(d0, d0, q0);
                s1 += d1; q1 = fmaf(d1, d1, q1);
            }
            ++cnt;
        }
    }
    const float n = (float)(cnt * 4);
    Mom a{n, 0.f, 0.f}, b{n, 0.f, 0.f};
    if (cnt > 0) {
        const float m0 = s0 / n, m1 = s1 / n;
        a.mean = k0 + m0; a.m2 = fmaxf(q0 - s0 * m0, 0.f);
        b.mean = k1 + m1; b.m2 = fmaxf(q1 - s1 * m1, 0.f);
    }
    s_m[threadIdx.x * 2] = a;
    s_m[threadIdx.x * 2 + 1] = b;
    __syncthreads();
    if (threadIdx.x < groups) {
        const int g = threadIdx.x;
        Mom r{0.f, 0.f, 0.f};
        // halves of group g: channels [g*cpg, (g+1)*cpg) -> half index h = channel / 4 in [g*cpg/4, (g+1)*cpg/4)
        const int h_lo = g * cpg / 4, h_hi = (g + 1) * cpg / 4;
        for (int pl2 = 0; pl2 < ppi; ++pl2)
            for (int h = h_lo; h < h_hi; ++h) r = mom_merge(r, s_m[(pl2 * cv + (h >> 1)) * 2 + (h & 1)]);
        float* o = ws + ((long long)blockIdx.x * groups + g) * 3;
        o[0] = r.n; o[1] = r.mean; o[2] = r.m2;
    }
}

// One warp per (image, group): lanes stride over the per-CTA partials, then merge by shuffles (a single thread walking
// ~600 partials with a dependent divide each took 0.3 ms -- longer than the streaming pass it finishes).
__global__ void __launch_bounds__(256)
gn_stats_nhwc_final_kernel(const float* __restrict__ ws, int nblocks, int groups, int images, float* __restrict__ mean,
                           float* __restrict__ var) {
    const int gi = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (gi >= images * groups) return;
    const int img = gi / groups, g = gi - img * groups;
    ws += (long long)img * nblocks * groups * 3;
    Mom r{0.f, 0.f, 0.f};
    for (int b = lane; b < nblocks; b += 32) {
        const float* o = ws + ((long long)b * groups + g) * 3;
        r = mom_merge(r, Mom{o[0], o[1], o[2]});
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        Mom t;
        t.n = __shfl_xor_sync(0xffffffffu, r.n, off);
        t.mean = __shfl_xor_sync(0xffffffffu, r.mean, off);
        t.m2 = __shfl_xor_sync(0xffffffffu, r.m2, off);
        r = mom_merge(r, t);
    }
    if (lane == 0) {
        mean[gi] = r.mean;
        var[gi] = r.n > 0.f ? r.m2 / r.n : 0.f;    // biased (torch.var_mean(unbiased=False))
    }
}

// ---------------------------------------------------------------------------------------------------------------
// GroupNorm apply (+ SiLU), channels-last: y = act((x - mean[g]) * rsqrt(var[g] + eps) * gamma[c] + beta[c])
// blockIdx.y is the image; mean / var are [images, groups].
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kNhwcThreads)
gn_apply_nhwc_kernel(const T* __restrict__ x, T* __restrict__ y, long long P, int C, int groups, const float* __restrict__ mean,
                     const float* __restrict__ var, const float* __restrict__ gamma, const float* __restrict__ beta, float eps, int act) {
    x += (long long)blockIdx.y * P * C;
    y += (long long)blockIdx.y * P * C;
    mean += blockIdx.y * groups;
    var += blockIdx.y * groups;
    const int cv = C / 8, cpg = C / groups;
    const long long total = P * cv;
    const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int v = (int)(i0 % cv);                      // fixed per thread: the grid stride is a multiple of cv
    float sc[8], sh[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int c = v * 8 + k, g = c / cpg;
        const float rstd = 1.0f / sqrtf(var[g] + eps);
        const float ga = gamma != nullptr ? gamma[c] : 1.0f, be = beta != nullptr ? beta[c] : 0.0f;
        sc[k] = rstd * ga;
        sh[k] = fmaf(-mean[g], sc[k], be);
    }
    for (long long i = i0; i < total; i += (long long)gridDim.x * blockDim.x) {
        const uint4 u = ldg128(x + i * 8);
        float f[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            float t = fmaf(vget<T>(u, k), sc[k], sh[k]);
            if (act) t = __fdividef(t, 1.0f + __expf(-t));
            f[k] = t;
        }
        stg128_stream(y + i * 8, vpack<T>(f));
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Row softmax (attention weights): y[r, :cols] = softmax(x[r, :cols]), y[r, cols:pitch] = 0.  One CTA per row,
// two passes over the row (the second one hits L2): online (max, sum) then normalise.
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kNhwcThreads)
softmax_rows_kernel(const T* __restrict__ x, T* __restrict__ y, int cols, long long pitch) {
    __shared__ float s_m[kNhwcThreads / 32], s_s[kNhwcThreads / 32];
    const T* xr = x + (long long)blockIdx.x * pitch;
    T* yr = y + (long long)blockIdx.x * pitch;
    const int nv = (int)(pitch / 8);
    float m = -FLT_MAX, s = 0.f;
    for (int v = threadIdx.x; v < nv; v += kNhwcThreads) {
        const uint4 u = ldg128(xr + v * 8);
        float lm = -FLT_MAX;
#pragma unroll
        for (int k = 0; k < 8; ++k) if (v * 8 + k < cols) lm = fmaxf(lm, vget<T>(u, k));
        if (lm > m) { s *= __expf(m - lm); m = lm; }
#pragma unroll
        for (int k = 0; k < 8; ++k) if (v * 8 + k < cols) s += __expf(vget<T>(u, k) - m);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, m, off), os = __shfl_xor_sync(0xffffffffu, s, off);
        const float nm = fmaxf(m, om);
        s = s * __expf(m - nm) + os * __expf(om - nm);
        m = nm;
    }
    if ((threadIdx.x & 31) == 0) { s_m[threadIdx.x >> 5] = m; s_s[threadIdx.x >> 5] = s; }
    __syncthreads();
    float gm = -FLT_MAX, gs = 0.f;
#pragma unroll
    for (int w = 0; w < kNhwcThreads / 32; ++w) gm = fmaxf(gm, s_m[w]);
#pragma unroll
    for (int w = 0; w < kNhwcThreads / 32; ++w) gs += s_s[w] * __expf(s_m[w] - gm);
    const float inv = 1.0f / gs;
    for (int v = threadIdx.x; v < nv; v += kNhwcThreads) {
        const uint4 u = ldg128(xr + v * 8);
        float f[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) f[k] = (v * 8 + k < cols) ? __expf(vget<T>(u, k) - gm) * inv : 0.0f;
        stg128(yr + v * 8, vpack<T>(f));
    }
}

int grid_for(long long total, int per_block) {
    const long long want = (total + per_block - 1) / per_block;
    return (int)std::max(1LL, std::min(want, (long long)nhwc_sms() * 8));
}

bool half_like(int dtype) { return dtype == TD_F16 || dtype == TD_BF16; }

}  // namespace

extern "C" int td_nchw_to_nhwc(const void* x, void* y, int N, int C, int rows, int cols, int64_t x_img_stride, int64_t x_plane_stride,
                               int64_t x_pitch, int Cpad, int dtype, void* stream) {
    if (x == nullptr || y == nullptr || N <= 0 || C <= 0 || rows <= 0 || cols <= 0 || Cpad < C || Cpad % 8 != 0 || !half_like(dtype)) {
        td_set_error("td_nchw_to_nhwc: bad arguments (fp16 / bf16, Cpad >= C and a multiple of 8)");
        return TD_ERR_INVALID_ARG;
    }
    const long long total = (long long)N * rows * cols * (Cpad / 8);
    const int grid = grid_for(total, kNhwcThreads);
    if (dtype == TD_F16)
        nchw_to_nhwc_kernel<__half><<<grid, kNhwcThreads, 0, (cudaStream_t)stream>>>((const __half*)x, (__half*)y, C, x_plane_stride, x_pitch, x_img_stride, rows, cols, Cpad, total);
    else
        nchw_to_nhwc_kernel<__nv_bfloat16><<<grid, kNhwcThreads, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, C, x_plane_stride, x_pitch, x_img_stride, rows, cols, Cpad, total);
    return launch_status("td_nchw_to_nhwc");
}

extern "C" int td_nchw_to_nhwc_wrap(const void* x, void* y, int N, int C, int rows, int cols, int row0, int col0, int H, int W,
                                    int64_t x_img_stride, int64_t x_plane_stride, int64_t x_pitch, int Cpad, int dtype, void* stream) {
    if (x == nullptr || y == nullptr || N <= 0 || C <= 0 || rows <= 0 || cols <= 0 || H <= 0 || W <= 0 || Cpad < C || Cpad % 8 != 0 ||
        !half_like(dtype)) {
        td_set_error("td_nchw_to_nhwc_wrap: bad arguments (fp16 / bf16, Cpad >= C and a multiple of 8)");
        return TD_ERR_INVALID_ARG;
    }
    const long long total = (long long)N * rows * cols * (Cpad / 8);
    const int grid = grid_for(total, kNhwcThreads);
    if (dtype == TD_F16)
        nchw_to_nhwc_wrap_kernel<__half><<<grid, kNhwcThreads, 0, (cudaStream_t)stream>>>((const __half*)x, (__half*)y, C, x_plane_stride, x_pitch,
                                                                                        x_img_stride, rows, cols, row0, col0, H, W, Cpad, total);
    else
        nchw_to_nhwc_wrap_kernel<__nv_bfloat16><<<grid, kNhwcThreads, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, C,
                                                                                               x_plane_stride, x_pitch, x_img_stride, rows, cols,
                                                                                               row0, col0, H, W, Cpad, total);
    return launch_status("td_nchw_to_nhwc_wrap");
}

extern "C" int td_nhwc_to_nchw_region(const void* x, void* y, int N, int C, int rows, int cols, int64_t x_img_stride, int x_width,
                                      int64_t x_pitch, int64_t y_img_stride, int64_t y_plane_stride, int64_t y_pitch, int dtype, void* stream) {
    if (x == nullptr || y == nullptr || N <= 0 || C <= 0 || rows <= 0 || cols <= 0 || !half_like(dtype)) {
        td_set_error("td_nhwc_to_nchw_region: bad arguments");
        return TD_ERR_INVALID_ARG;
    }
    const long long total = (long long)N * C * rows * cols;
    const int grid = grid_for(total, kNhwcThreads);
    // fp16 and bf16 move as opaque 16-bit words
    nhwc_to_nchw_region_kernel<__half><<<grid, kNhwcThreads, 0, (cudaStream_t)stream>>>((const __half*)x, (__half*)y, C, x_pitch, x_width, x_img_stride,
                                                                                          y_plane_stride, y_pitch, y_img_stride, rows, cols, total);
    return launch_status("td_nhwc_to_nchw_region");
}

extern "C" int td_upsample2x_nhwc(const void* x, void* y, int N, int H, int W, int C, int dtype, void* stream) {
    if (x == nullptr || y == nullptr || N <= 0 || H <= 0 || W <= 0 || C <= 0 || C % 8 != 0 || !half_like(dtype)) {
        td_set_error("td_upsample2x_nhwc: bad arguments (C must be a multiple of 8)");
        return TD_ERR_INVALID_ARG;
    }
    const long long total = (long long)N * H * W * (C / 8);
    upsample2x_nhwc_kernel<__half><<<grid_for(total, kNhwcThreads), kNhwcThreads, 0, (cudaStream_t)stream>>>((const __half*)x, (__half*)y, H, W, C / 8, total);
    return launch_status("td_upsample2x_nhwc");
}

namespace {

// The one-image entries are the batched ones at N = 1: one plan, so a batched image gets its one-image bits.
int gn_stats_grid(int64_t pixels, int C) {
    const int ppi = kNhwcThreads / (C / 8);
    return (int)std::max<int64_t>(1, std::min<int64_t>((pixels + ppi - 1) / ppi, (int64_t)nhwc_sms() * 4));
}

int gn_stats_run(const char* what, const void* x, int N, int64_t pixels, int C, int groups, int dtype, void* workspace,
                 int64_t workspace_bytes, float* mean, float* var, void* stream) {
    if (x == nullptr || workspace == nullptr || mean == nullptr || var == nullptr || pixels <= 0 || N <= 0 || N > 65535 || !half_like(dtype)) {
        td_set_error("%s: bad arguments", what);
        return TD_ERR_INVALID_ARG;
    }
    if (groups <= 0 || groups > 64 || C <= 0 || C % groups != 0 || (C / groups) % 4 != 0 || C % 8 != 0 || kNhwcThreads % (C / 8) != 0) {
        td_set_error("%s: unsupported channel layout C=%d groups=%d (need C/groups %% 4 == 0 and C/8 dividing 256)", what, C, groups);
        return TD_ERR_UNSUPPORTED;
    }
    const int grid = gn_stats_grid(pixels, C);
    if ((int64_t)N * grid * groups * 3 * (int64_t)sizeof(float) > workspace_bytes) { td_set_error("%s: workspace too small", what); return TD_ERR_CAPACITY; }
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 g2(grid, N);
    if (dtype == TD_F16) gn_stats_nhwc_partial_kernel<__half><<<g2, kNhwcThreads, 0, st>>>((const __half*)x, pixels, C, groups, (float*)workspace);
    else gn_stats_nhwc_partial_kernel<__nv_bfloat16><<<g2, kNhwcThreads, 0, st>>>((const __nv_bfloat16*)x, pixels, C, groups, (float*)workspace);
    gn_stats_nhwc_final_kernel<<<(N * groups * 32 + 255) / 256, 256, 0, st>>>((const float*)workspace, grid, groups, N, mean, var);
    return launch_status(what);
}

int gn_apply_run(const char* what, const void* x, void* y, int N, int64_t pixels, int C, int groups, int dtype, const float* mean,
                 const float* var, const float* gamma, const float* beta, float eps, int act, void* stream) {
    if (x == nullptr || y == nullptr || mean == nullptr || var == nullptr || pixels <= 0 || N <= 0 || N > 65535 || !half_like(dtype)) {
        td_set_error("%s: bad arguments", what);
        return TD_ERR_INVALID_ARG;
    }
    if (groups <= 0 || C <= 0 || C % groups != 0 || C % 8 != 0 || kNhwcThreads % (C / 8) != 0) {
        td_set_error("%s: unsupported channel layout C=%d groups=%d", what, C, groups);
        return TD_ERR_UNSUPPORTED;
    }
    const long long total = (long long)pixels * (C / 8);
    const dim3 grid(grid_for(total, kNhwcThreads * 4), N);
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == TD_F16) gn_apply_nhwc_kernel<__half><<<grid, kNhwcThreads, 0, st>>>((const __half*)x, (__half*)y, pixels, C, groups, mean, var, gamma, beta, eps, act);
    else gn_apply_nhwc_kernel<__nv_bfloat16><<<grid, kNhwcThreads, 0, st>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, pixels, C, groups, mean, var, gamma, beta, eps, act);
    return launch_status(what);
}

}  // namespace

extern "C" int64_t td_gn_stats_nhwc_workspace_bytes(int64_t pixels, int C, int groups) {
    if (pixels <= 0 || C <= 0 || groups <= 0) return 0;
    return (int64_t)nhwc_sms() * 4 * groups * 3 * (int64_t)sizeof(float);
}

extern "C" int td_gn_stats_nhwc(const void* x, int64_t pixels, int C, int groups, int dtype, void* workspace, int64_t workspace_bytes,
                                float* mean, float* var, void* stream) {
    return gn_stats_run("td_gn_stats_nhwc", x, 1, pixels, C, groups, dtype, workspace, workspace_bytes, mean, var, stream);
}

extern "C" int td_gn_apply_nhwc(const void* x, void* y, int64_t pixels, int C, int groups, int dtype, const float* mean, const float* var,
                                const float* gamma, const float* beta, float eps, int act, void* stream) {
    return gn_apply_run("td_gn_apply_nhwc", x, y, 1, pixels, C, groups, dtype, mean, var, gamma, beta, eps, act, stream);
}

extern "C" int64_t td_gn_stats_nhwc_batched_workspace_bytes(int N, int64_t pixels, int C, int groups) {
    if (N <= 0 || pixels <= 0 || C <= 0 || groups <= 0) return 0;
    return (int64_t)N * td_gn_stats_nhwc_workspace_bytes(pixels, C, groups);
}

extern "C" int td_gn_stats_nhwc_batched(const void* x, int N, int64_t pixels, int C, int groups, int dtype, void* workspace,
                                        int64_t workspace_bytes, float* mean, float* var, void* stream) {
    if (x != nullptr && !aligned16(x)) { td_set_error("td_gn_stats_nhwc_batched: x must be 16-byte aligned"); return TD_ERR_INVALID_ARG; }
    return gn_stats_run("td_gn_stats_nhwc_batched", x, N, pixels, C, groups, dtype, workspace, workspace_bytes, mean, var, stream);
}

extern "C" int td_gn_apply_nhwc_batched(const void* x, void* y, int N, int64_t pixels, int C, int groups, int dtype, const float* mean,
                                        const float* var, const float* gamma, const float* beta, float eps, int act, void* stream) {
    if ((x != nullptr && !aligned16(x)) || (y != nullptr && !aligned16(y))) {
        td_set_error("td_gn_apply_nhwc_batched: x and y must be 16-byte aligned");
        return TD_ERR_INVALID_ARG;
    }
    return gn_apply_run("td_gn_apply_nhwc_batched", x, y, N, pixels, C, groups, dtype, mean, var, gamma, beta, eps, act, stream);
}

extern "C" int td_softmax_rows(const void* x, void* y, int rows, int cols, int64_t pitch, int dtype, void* stream) {
    if (x == nullptr || y == nullptr || rows <= 0 || cols <= 0 || pitch < cols || pitch % 8 != 0 || !half_like(dtype)) {
        td_set_error("td_softmax_rows: bad arguments (pitch >= cols and a multiple of 8)");
        return TD_ERR_INVALID_ARG;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == TD_F16) softmax_rows_kernel<__half><<<rows, kNhwcThreads, 0, st>>>((const __half*)x, (__half*)y, cols, pitch);
    else softmax_rows_kernel<__nv_bfloat16><<<rows, kNhwcThreads, 0, st>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, cols, pitch);
    return launch_status("td_softmax_rows");
}
