// DemoFusion extras on sm_90a (tile_methods/demofusion.py of the reference):
//
//   td_dilated_gather      <- x[:, :, by::s, bx::s] views + torch.cat               demofusion.py:283-308
//   td_demofusion_combine  <- strided `x_global[...] += view`, `/2` (mixture), `/weights`,
//                             and x_local*(1-c2) + x_global*c2                       demofusion.py:296-322
//   td_depthwise_conv2d    <- gaussian_filter (F.conv2d, groups=C)                   demofusion.py:173-178
//   td_depthwise_conv2d_wrap  the same stencil with circular indexing on the wrapped axes (seamless DemoFusion, new)
//
// The local windows reuse td_scatter_tiles / td_blend_multidiffusion (count-normalised blend) and the
// mean/std renormalisation reuses td_gn_stats + td_affine_clamp.  Small strided / stencil kernels:
// HBM- and latency-bound, no tensor cores.  Every arithmetic step is rounded through the latent dtype
// exactly where the reference's eager ops round.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "td_b200.h"
#include "td_device.cuh"
#include "td_internal.h"
#include "td_launch.h"

namespace {

using namespace td;

constexpr int kMaxViews = 64;     // views per launch (the caller batches 2 * s * s views, s <= 8)
constexpr int kMaxKernel = 15;

struct ViewTable {
    int n_views;                        // views in this launch
    int32_t bx[kMaxViews], by[kMaxViews];   // any offset the host check accepts (8 bits wrapped offsets >= 256)
    unsigned char second[kMaxViews];    // 1: read from the second (blurred) source
};

// out[(v*N + n), c, i, j] = src_v[n, c, by_v + i*s, bx_v + j*s]
template <typename T>
__global__ void __launch_bounds__(256)
dilated_gather_kernel(const T* __restrict__ x0, const T* __restrict__ x1, T* __restrict__ out, const __grid_constant__ ViewTable vt,
                      int NC, int H, int W, int s, int oh, int ow) {
    const int v = blockIdx.z;
    const T* src = vt.second[v] ? x1 : x0;
    const int bx = vt.bx[v], by = vt.by[v];
    const long long plane_elems = (long long)oh * ow;
    for (int p = blockIdx.y; p < NC; p += gridDim.y) {
        const T* sp = src + (long long)p * H * W;
        T* op = out + ((long long)v * NC + p) * plane_elems;
        for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < plane_elems; e += (long long)gridDim.x * blockDim.x) {
            const int i = (int)(e / ow), j = (int)(e - (long long)i * ow);
            op[e] = sp[(long long)(by + i * s) * W + (bx + j * s)];
        }
    }
}

struct CombineParams {
    int NC, H, W, s, oh, ow, end_y, end_x;
    int views_per_batch, n_views, mixture;
    float c2, one_minus_c2;
    const void* batch_ptrs[TD_MAX_BATCH_PTRS];
};

// out = T(T(x_local * (1-c2)) + T(x_global * c2)),  x_global = (mixture ? T(acc / 2) : acc),
// acc = sum in view order of the view outputs that land on this pixel (each add rounded through T).
template <typename T>
__global__ void __launch_bounds__(256)
demofusion_combine_kernel(const __grid_constant__ CombineParams p, const T* __restrict__ x_local, T* __restrict__ out) {
    const long long total = (long long)p.NC * p.H * p.W;
    const int half = p.mixture ? p.n_views / 2 : p.n_views;
    const long long view_plane = (long long)p.oh * p.ow;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(e % p.W);
        const long long r = e / p.W;
        const int y = (int)(r % p.H);
        const int plane = (int)(r / p.H);
        float acc = 0.0f;
        if (y < p.end_y && x < p.end_x) {
            const int by = y % p.s, bx = x % p.s, i = y / p.s, j = x / p.s;
            const int v0 = by * p.s + bx;   // views are listed row-major over (by, bx)
#pragma unroll 2
            for (int rep = 0; rep < 2; ++rep) {
                const int v = v0 + rep * half;
                if (rep == 1 && !p.mixture) break;
                const int b = v / p.views_per_batch, vi = v - b * p.views_per_batch;
                const T* vp = reinterpret_cast<const T*>(p.batch_ptrs[b]) + ((long long)vi * p.NC + plane) * view_plane + (long long)i * p.ow + j;
                acc = round_through<T>(__fadd_rn(acc, Elem<T>::to_f32(*vp)));
            }
        }
        float xg = acc;
        if (p.mixture) xg = round_through<T>(__fmul_rn(acc, 0.5f));           // x_global / 2
        const float a = round_through<T>(__fmul_rn(Elem<T>::to_f32(x_local[e]), p.one_minus_c2));
        const float b2 = round_through<T>(__fmul_rn(xg, p.c2));
        out[e] = Elem<T>::from_f32(__fadd_rn(a, b2));
    }
}

struct ConvKernel {
    int k;
    float w[kMaxKernel * kMaxKernel];   // already rounded through the latent dtype by the caller
};

// out[p, y, x] = T( sum_{dy,dx} x[p, y+dy-k/2, x+dx-k/2] * w[dy][dx] )  (fp32 accumulate, taps in (dy, dx) order)
// Zero padding on a bounded axis; on an axis whose WRAP bit is set the index is taken mod the axis length, with one
// conditional add or subtract because the host refuses k/2 > L there.  The body is __host__ __device__ so that the
// test-only harness tests/emul/demofusion_host_emul.cu can run it on a CPU (fmaf is one rounding on both sides).
template <typename T, int WRAP>
__host__ __device__ __forceinline__ T depthwise_conv_elem(const T* __restrict__ in, const ConvKernel& ck, int H, int W, long long e) {
    const int k = ck.k, pad = k / 2;
    const int x = (int)(e % W);
    const long long r = e / W;
    const int y = (int)(r % H);
    const T* ip = in + (r / H) * (long long)H * W;
    float acc = 0.0f;
    for (int dy = 0; dy < k; ++dy) {
        int yy = y + dy - pad;
        if constexpr ((WRAP & TD_WRAP_Y) != 0) {
            if (yy < 0) yy += H;
            else if (yy >= H) yy -= H;
        } else if ((unsigned)yy >= (unsigned)H) {
            continue;
        }
        for (int dx = 0; dx < k; ++dx) {
            int xx = x + dx - pad;
            if constexpr ((WRAP & TD_WRAP_X) != 0) {
                if (xx < 0) xx += W;
                else if (xx >= W) xx -= W;
            } else if ((unsigned)xx >= (unsigned)W) {
                continue;
            }
            acc = fmaf(Elem<T>::to_f32(ip[(long long)yy * W + xx]), ck.w[dy * k + dx], acc);
        }
    }
    return Elem<T>::from_f32(acc);
}

template <typename T, int WRAP>
__global__ void __launch_bounds__(256)
depthwise_conv_kernel(const T* __restrict__ in, T* __restrict__ out, const __grid_constant__ ConvKernel ck, int planes, int H, int W) {
    const long long total = (long long)planes * H * W;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x)
        out[e] = depthwise_conv_elem<T, WRAP>(in, ck, H, W, e);
}

// validation shared by td_depthwise_conv2d and td_depthwise_conv2d_wrap; fills `ck`
int conv_args(const char* who, const void* in, const void* out, int planes, int H, int W, const float* kernel_host, int k, int wrap,
              ConvKernel* ck) {
    if (in == nullptr || out == nullptr || kernel_host == nullptr || k <= 0 || k > kMaxKernel || (k & 1) == 0 || planes <= 0) {
        td_set_error("%s: bad arguments (odd k <= %d)", who, kMaxKernel);
        return TD_ERR_INVALID_ARG;
    }
    if ((wrap & ~(int)(TD_WRAP_X | TD_WRAP_Y)) != 0 || (wrap != 0 && (H <= 0 || W <= 0))) {
        td_set_error("%s: bad arguments (wrap=%d, %dx%d canvas)", who, wrap, H, W);
        return TD_ERR_INVALID_ARG;
    }
    if (((wrap & TD_WRAP_X) && k / 2 > W) || ((wrap & TD_WRAP_Y) && k / 2 > H)) {
        td_set_error("%s: kernel radius %d exceeds a wrapped axis of the %dx%d canvas", who, k / 2, H, W);
        return TD_ERR_INVALID_ARG;
    }
    ck->k = k;
    for (int i = 0; i < k * k; ++i) ck->w[i] = kernel_host[i];
    return TD_OK;
}

template <int WRAP>
void launch_conv(const void* in, void* out, const ConvKernel& ck, int planes, int H, int W, int dtype, cudaStream_t st) {
    const long long total = (long long)planes * H * W;
    const unsigned blocks = (unsigned)std::max(1LL, std::min((total + 255) / 256, 148LL * 32));
    if (dtype == TD_F16) depthwise_conv_kernel<__half, WRAP><<<blocks, 256, 0, st>>>((const __half*)in, (__half*)out, ck, planes, H, W);
    else if (dtype == TD_BF16) depthwise_conv_kernel<__nv_bfloat16, WRAP><<<blocks, 256, 0, st>>>((const __nv_bfloat16*)in, (__nv_bfloat16*)out, ck, planes, H, W);
    else depthwise_conv_kernel<float, WRAP><<<blocks, 256, 0, st>>>((const float*)in, (float*)out, ck, planes, H, W);
}


}  // namespace

extern "C" int td_dilated_gather(const void* x0, const void* x1, void* out, int N, int C, int H, int W, int s, int out_h, int out_w,
                                 const int32_t* view_bx, const int32_t* view_by, const int32_t* view_second, int n_views, int dtype,
                                 void* stream) {
    if (x0 == nullptr || out == nullptr || view_bx == nullptr || view_by == nullptr || n_views <= 0 || n_views > kMaxViews || s <= 0 ||
        N <= 0 || C <= 0 || out_h <= 0 || out_w <= 0) {
        td_set_error("td_dilated_gather: bad arguments");
        return TD_ERR_INVALID_ARG;
    }
    ViewTable vt;
    vt.n_views = n_views;
    for (int v = 0; v < n_views; ++v) {
        const int sec = view_second ? view_second[v] : 0;
        if (view_bx[v] < 0 || view_by[v] < 0 || view_bx[v] + (out_w - 1) * s >= W || view_by[v] + (out_h - 1) * s >= H || (sec && x1 == nullptr)) {
            td_set_error("td_dilated_gather: view %d out of range", v);
            return TD_ERR_INVALID_ARG;
        }
        vt.bx[v] = view_bx[v]; vt.by[v] = view_by[v]; vt.second[v] = (unsigned char)sec;
    }
    const int es = td_dtype_size(dtype);
    if (es == 0) { td_set_error("td_dilated_gather: unknown dtype"); return TD_ERR_INVALID_ARG; }
    const int NC = N * C;
    dim3 grid((unsigned)std::max(1, std::min((out_h * out_w + 255) / 256, 256)), (unsigned)std::min(NC, 65535), (unsigned)n_views);
    cudaStream_t st = (cudaStream_t)stream;
    if (es == 2) dilated_gather_kernel<__half><<<grid, 256, 0, st>>>((const __half*)x0, (const __half*)x1, (__half*)out, vt, NC, H, W, s, out_h, out_w);
    else dilated_gather_kernel<float><<<grid, 256, 0, st>>>((const float*)x0, (const float*)x1, (float*)out, vt, NC, H, W, s, out_h, out_w);
    return launch_status("td_dilated_gather");
}

extern "C" int td_demofusion_combine(const void* x_local, const void* const* view_batch_ptrs, int num_batches, int views_per_batch,
                                     int n_views, void* out, int N, int C, int H, int W, int s, int out_h, int out_w, int end_y,
                                     int end_x, int mixture, float c2, float one_minus_c2, int dtype, void* stream) {
    if (x_local == nullptr || out == nullptr || view_batch_ptrs == nullptr || num_batches <= 0 || num_batches > TD_MAX_BATCH_PTRS ||
        views_per_batch <= 0 || s <= 0 || n_views != (mixture ? 2 : 1) * s * s || (long long)num_batches * views_per_batch < n_views ||
        N <= 0 || C <= 0 || H <= 0 || W <= 0 || out_h <= 0 || out_w <= 0 || end_y > H || end_x > W) {
        td_set_error("td_demofusion_combine: bad arguments");
        return TD_ERR_INVALID_ARG;
    }
    // every pixel of [0, end) must map inside a view: i = y / s < out_h
    if ((end_y > 0 && (end_y - 1) / s >= out_h) || (end_x > 0 && (end_x - 1) / s >= out_w)) {
        td_set_error("td_demofusion_combine: views %dx%d do not cover [0, %d) x [0, %d) at scale %d", out_h, out_w, end_y, end_x, s);
        return TD_ERR_INVALID_ARG;
    }
    CombineParams p;
    p.NC = N * C; p.H = H; p.W = W; p.s = s; p.oh = out_h; p.ow = out_w; p.end_y = end_y; p.end_x = end_x;
    p.views_per_batch = views_per_batch; p.n_views = n_views; p.mixture = mixture; p.c2 = c2; p.one_minus_c2 = one_minus_c2;
    for (int b = 0; b < num_batches; ++b) {
        if (view_batch_ptrs[b] == nullptr) { td_set_error("td_demofusion_combine: null batch %d", b); return TD_ERR_INVALID_ARG; }
        p.batch_ptrs[b] = view_batch_ptrs[b];
    }
    const long long total = (long long)p.NC * H * W;
    const unsigned blocks = (unsigned)std::max(1LL, std::min((total + 255) / 256, 148LL * 32));
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == TD_F16) demofusion_combine_kernel<__half><<<blocks, 256, 0, st>>>(p, (const __half*)x_local, (__half*)out);
    else if (dtype == TD_BF16) demofusion_combine_kernel<__nv_bfloat16><<<blocks, 256, 0, st>>>(p, (const __nv_bfloat16*)x_local, (__nv_bfloat16*)out);
    else if (dtype == TD_F32) demofusion_combine_kernel<float><<<blocks, 256, 0, st>>>(p, (const float*)x_local, (float*)out);
    else { td_set_error("td_demofusion_combine: unknown dtype"); return TD_ERR_INVALID_ARG; }
    return launch_status("td_demofusion_combine");
}

extern "C" int td_depthwise_conv2d(const void* in, void* out, int planes, int H, int W, const float* kernel_host, int k, int dtype,
                                   void* stream) {
    ConvKernel ck;
    const int rc = conv_args("td_depthwise_conv2d", in, out, planes, H, W, kernel_host, k, 0, &ck);
    if (rc != TD_OK) return rc;
    if (dtype != TD_F16 && dtype != TD_BF16 && dtype != TD_F32) { td_set_error("td_depthwise_conv2d: unknown dtype"); return TD_ERR_INVALID_ARG; }
    launch_conv<0>(in, out, ck, planes, H, W, dtype, (cudaStream_t)stream);
    return launch_status("td_depthwise_conv2d");
}

extern "C" int td_depthwise_conv2d_wrap(const void* in, void* out, int planes, int H, int W, const float* kernel_host, int k, int wrap,
                                        int dtype, void* stream) {
    ConvKernel ck;
    const int rc = conv_args("td_depthwise_conv2d_wrap", in, out, planes, H, W, kernel_host, k, wrap, &ck);
    if (rc != TD_OK) return rc;
    if (dtype != TD_F16 && dtype != TD_BF16 && dtype != TD_F32) { td_set_error("td_depthwise_conv2d_wrap: unknown dtype"); return TD_ERR_INVALID_ARG; }
    cudaStream_t st = (cudaStream_t)stream;
    if (wrap == TD_WRAP_X) launch_conv<TD_WRAP_X>(in, out, ck, planes, H, W, dtype, st);
    else if (wrap == TD_WRAP_Y) launch_conv<TD_WRAP_Y>(in, out, ck, planes, H, W, dtype, st);
    else if (wrap == (TD_WRAP_X | TD_WRAP_Y)) launch_conv<TD_WRAP_X | TD_WRAP_Y>(in, out, ck, planes, H, W, dtype, st);
    else launch_conv<0>(in, out, ck, planes, H, W, dtype, st);
    return launch_status("td_depthwise_conv2d_wrap");
}

#ifdef TD_DEMOFUSION_HOST_EMULATION
// Test-only (tests/emul/demofusion_host_emul.cu includes this file with the macro set): the conv body on the host.
extern "C" int td_emul_depthwise_conv2d_wrap(const void* in, void* out, int planes, int H, int W, const float* kernel_host, int k, int wrap,
                                             int dtype) {
    ConvKernel ck;
    const int rc = conv_args("td_emul_depthwise_conv2d_wrap", in, out, planes, H, W, kernel_host, k, wrap, &ck);
    if (rc != TD_OK) return rc;
    const long long total = (long long)planes * H * W;
    for (long long e = 0; e < total; ++e) {
#define TD_CONV_EMUL(T)                                                                                                      \
    if (wrap == TD_WRAP_X) ((T*)out)[e] = depthwise_conv_elem<T, TD_WRAP_X>((const T*)in, ck, H, W, e);                      \
    else if (wrap == TD_WRAP_Y) ((T*)out)[e] = depthwise_conv_elem<T, TD_WRAP_Y>((const T*)in, ck, H, W, e);                 \
    else if (wrap == (TD_WRAP_X | TD_WRAP_Y)) ((T*)out)[e] = depthwise_conv_elem<T, TD_WRAP_X | TD_WRAP_Y>((const T*)in, ck, H, W, e); \
    else ((T*)out)[e] = depthwise_conv_elem<T, 0>((const T*)in, ck, H, W, e);
        if (dtype == TD_F16) { TD_CONV_EMUL(__half) }
        else if (dtype == TD_BF16) { TD_CONV_EMUL(__nv_bfloat16) }
        else { TD_CONV_EMUL(float) }
#undef TD_CONV_EMUL
    }
    return TD_OK;
}
#endif
