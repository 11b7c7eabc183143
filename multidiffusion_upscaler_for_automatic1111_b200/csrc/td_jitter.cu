// DemoFusion with random jitter (tile_methods/demofusion.py:101-139, :204, :254-264, :279-310 of the reference):
// every local window gets its own random offset on the zero-padded latent, so the window list is no longer
// the separable rows x cols grid the fused kernels of td_diffusion.cu are built around.  These are the
// list-driven forms -- plain one-element-per-thread kernels (a few hundred windows, HBM- and latency-bound):
//
//   td_scatter_bboxes              <- torch.cat([x_in[bbox.slicer] for bbox in bboxes])          demofusion.py:256
//   td_blend_bboxes                <- x_buffer[slicer] += tile; weights[slicer] += 1 (per window, in order),
//                                     weights==0 -> 1, x_local = x_buffer / weights               demofusion.py:259-264
//   td_demofusion_combine_offset   <- td_demofusion_combine with the dilated views starting at
//                                     jitter_range + (by, bx)                                      demofusion.py:279-322
//   td_scatter_bboxes_wrap,        <- the two list forms on a periodic canvas (seamless DemoFusion, new: the reference
//   td_blend_bboxes_wrap              has no wrap): modular on the wrapped axes, zero-fill / skip on the bounded ones
//
// Numerics as everywhere on this path: the canvas accumulates in the latent dtype with one rounding per
// window, windows in list order.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "td_b200.h"
#include "td_device.cuh"
#include "td_internal.h"
#include "td_launch.h"

namespace {

using namespace td;

// The per-element bodies are __host__ __device__ so that the index arithmetic and the rounding sequence of these
// kernels can also be executed on a CPU by the test-only harness tests/emul/jitter_host_emul.cu (the product
// library never runs them on the host: there is no CPU path).
template <typename T> struct JElem;
template <> struct JElem<__half> {
    static __host__ __device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
    static __host__ __device__ __forceinline__ __half from_f32(float f) { return __float2half_rn(f); }
};
template <> struct JElem<__nv_bfloat16> {
    static __host__ __device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
    static __host__ __device__ __forceinline__ __nv_bfloat16 from_f32(float f) { return __float2bfloat16_rn(f); }
};
template <> struct JElem<float> {
    static __host__ __device__ __forceinline__ float to_f32(float v) { return v; }
    static __host__ __device__ __forceinline__ float from_f32(float f) { return f; }
};
template <typename T> __host__ __device__ __forceinline__ float jround(float f) { return JElem<T>::to_f32(JElem<T>::from_f32(f)); }

// single IEEE roundings, never contracted into an FMA (the host build uses -ffp-contract=off)
__host__ __device__ __forceinline__ float jadd(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ __forceinline__ float jmul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ __forceinline__ float jdiv(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}
__host__ __device__ __forceinline__ int jload(const int32_t* p) {
#ifdef __CUDA_ARCH__
    return __ldg(p);
#else
    return *p;
#endif
}

// tiles[e] for the flat tile-batch index e = ((t*NC + plane)*th + v)*tw + u
template <typename T>
__host__ __device__ __forceinline__ T scatter_bboxes_elem(const T* __restrict__ x, const int32_t* __restrict__ origins, int NC, int H,
                                                          int W, int th, int tw, long long e) {
    const int u = (int)(e % tw);
    long long r = e / tw;
    const int v = (int)(r % th);
    r /= th;
    const int plane = (int)(r % NC);
    const int t = (int)(r / NC);
    const int ox = jload(origins + 2 * t), oy = jload(origins + 2 * t + 1);
    return x[((long long)plane * H + oy + v) * W + ox + u];
}

template <typename T>
__global__ void __launch_bounds__(256)
scatter_bboxes_kernel(const T* __restrict__ x, T* __restrict__ tiles, const int32_t* __restrict__ origins, int NC, int H, int W,
                      int th, int tw, long long total) {
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x)
        tiles[e] = scatter_bboxes_elem<T>(x, origins, NC, H, W, th, tw, e);
}

struct BlendListParams {
    int NC, H, W, th, tw, n_tiles, tile_bs;
    const void* batch_ptrs[TD_MAX_BATCH_PTRS];
};

// out[plane, y, x] = acc / max(count, 1); acc = windows covering (y, x) added in list order, each add rounded through T
template <typename T>
__host__ __device__ __forceinline__ float blend_bboxes_elem(const BlendListParams& p, const int32_t* __restrict__ origins, long long e) {
    const int x = (int)(e % p.W);
    const long long r = e / p.W;
    const int y = (int)(r % p.H);
    const int plane = (int)(r / p.H);
    float acc = 0.0f;
    int count = 0;
    for (int t = 0; t < p.n_tiles; ++t) {
        const int u = x - jload(origins + 2 * t), v = y - jload(origins + 2 * t + 1);
        if ((unsigned)u >= (unsigned)p.tw || (unsigned)v >= (unsigned)p.th) continue;
        const int b = t / p.tile_bs, ti = t - b * p.tile_bs;
        const T* tp = reinterpret_cast<const T*>(p.batch_ptrs[b]) + (((long long)ti * p.NC + plane) * p.th + v) * p.tw + u;
        acc = jround<T>(jadd(acc, JElem<T>::to_f32(*tp)));
        ++count;
    }
    return count > 1 ? jdiv(acc, (float)count) : acc;
}

template <typename T>
__global__ void __launch_bounds__(256)
blend_bboxes_kernel(const __grid_constant__ BlendListParams p, const int32_t* __restrict__ origins, float* __restrict__ out) {
    const long long total = (long long)p.NC * p.H * p.W;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x)
        out[e] = blend_bboxes_elem<T>(p, origins, e);
}

// ---- periodic canvas (seamless DemoFusion): the same list forms with a `wrap` mask (TD_WRAP_X | TD_WRAP_Y).  On a wrapped
// axis of length L a window covers (o + u) mod L, 0 <= o < L, tile <= L; on a bounded axis it may start before 0 or end
// past L (a jittered window with the latent not padded): the scatter reads zeros there and the blend drops those pixels.

// canvas index of o + u on one axis: one subtraction on a wrapped axis (o < L, u < tile <= L), -1 off a bounded one
__host__ __device__ __forceinline__ int wrap_axis_index(int o, int u, int L, bool wrapped) {
    const int i = o + u;
    if (wrapped) return i >= L ? i - L : i;
    return (unsigned)i < (unsigned)L ? i : -1;
}

// tile coordinate of canvas index i in the window starting at o: one addition on a wrapped axis (both in [0, L))
__host__ __device__ __forceinline__ int wrap_axis_offset(int i, int o, int L, bool wrapped) {
    const int u = i - o;
    return (wrapped && u < 0) ? u + L : u;
}

template <typename T>
__host__ __device__ __forceinline__ T scatter_bboxes_wrap_elem(const T* __restrict__ x, const int32_t* __restrict__ origins, int NC, int H,
                                                               int W, int th, int tw, int wrap, long long e) {
    const int u = (int)(e % tw);
    long long r = e / tw;
    const int v = (int)(r % th);
    r /= th;
    const int plane = (int)(r % NC);
    const int t = (int)(r / NC);
    const int xx = wrap_axis_index(jload(origins + 2 * t), u, W, (wrap & TD_WRAP_X) != 0);
    const int yy = wrap_axis_index(jload(origins + 2 * t + 1), v, H, (wrap & TD_WRAP_Y) != 0);
    if (xx < 0 || yy < 0) return T(0);
    return x[((long long)plane * H + yy) * W + xx];
}

template <typename T>
__global__ void __launch_bounds__(256)
scatter_bboxes_wrap_kernel(const T* __restrict__ x, T* __restrict__ tiles, const int32_t* __restrict__ origins, int NC, int H, int W,
                           int th, int tw, int wrap, long long total) {
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x)
        tiles[e] = scatter_bboxes_wrap_elem<T>(x, origins, NC, H, W, th, tw, wrap, e);
}

// blend_bboxes_elem with modular coverage on the wrapped axes
template <typename T>
__host__ __device__ __forceinline__ float blend_bboxes_wrap_elem(const BlendListParams& p, const int32_t* __restrict__ origins, int wrap,
                                                                 long long e) {
    const bool wx = (wrap & TD_WRAP_X) != 0, wy = (wrap & TD_WRAP_Y) != 0;
    const int x = (int)(e % p.W);
    const long long r = e / p.W;
    const int y = (int)(r % p.H);
    const int plane = (int)(r / p.H);
    float acc = 0.0f;
    int count = 0;
    for (int t = 0; t < p.n_tiles; ++t) {
        const int u = wrap_axis_offset(x, jload(origins + 2 * t), p.W, wx), v = wrap_axis_offset(y, jload(origins + 2 * t + 1), p.H, wy);
        if ((unsigned)u >= (unsigned)p.tw || (unsigned)v >= (unsigned)p.th) continue;
        const int b = t / p.tile_bs, ti = t - b * p.tile_bs;
        const T* tp = reinterpret_cast<const T*>(p.batch_ptrs[b]) + (((long long)ti * p.NC + plane) * p.th + v) * p.tw + u;
        acc = jround<T>(jadd(acc, JElem<T>::to_f32(*tp)));
        ++count;
    }
    return count > 1 ? jdiv(acc, (float)count) : acc;
}

template <typename T>
__global__ void __launch_bounds__(256)
blend_bboxes_wrap_kernel(const __grid_constant__ BlendListParams p, const int32_t* __restrict__ origins, int wrap, float* __restrict__ out) {
    const long long total = (long long)p.NC * p.H * p.W;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x)
        out[e] = blend_bboxes_wrap_elem<T>(p, origins, wrap, e);
}

struct CombineOffsetParams {
    int NC, H, W, s, oh, ow, end_y, end_x, off;
    int views_per_batch, n_views, mixture;
    float c2, one_minus_c2;
    const void* batch_ptrs[TD_MAX_BATCH_PTRS];
};

// out = T(T(x_local * (1-c2)) + T(x_global * c2)),  x_global = (mixture ? T(acc / 2) : acc), acc = the view outputs that
// land on this pixel added in view order (each add rounded through T); views start at off + (by, bx)
template <typename T>
__host__ __device__ __forceinline__ T combine_offset_elem(const CombineOffsetParams& p, const T* __restrict__ x_local, long long e) {
    const int half = p.mixture ? p.n_views / 2 : p.n_views;
    const long long view_plane = (long long)p.oh * p.ow;
    const int x = (int)(e % p.W);
    const long long r = e / p.W;
    const int y = (int)(r % p.H);
    const int plane = (int)(r / p.H);
    float acc = 0.0f;
    if (y >= p.off && x >= p.off && y < p.end_y && x < p.end_x) {
        const int yy = y - p.off, xx = x - p.off;
        const int by = yy % p.s, bx = xx % p.s, i = yy / p.s, j = xx / p.s;
        const int v0 = by * p.s + bx;   // views are listed row-major over (by, bx)
        for (int rep = 0; rep < (p.mixture ? 2 : 1); ++rep) {
            const int v = v0 + rep * half;
            const int b = v / p.views_per_batch, vi = v - b * p.views_per_batch;
            const T* vp = reinterpret_cast<const T*>(p.batch_ptrs[b]) + ((long long)vi * p.NC + plane) * view_plane + (long long)i * p.ow + j;
            acc = jround<T>(jadd(acc, JElem<T>::to_f32(*vp)));
        }
    }
    float xg = acc;
    if (p.mixture) xg = jround<T>(jmul(acc, 0.5f));                      // x_global / 2
    const float a = jround<T>(jmul(JElem<T>::to_f32(x_local[e]), p.one_minus_c2));
    const float b2 = jround<T>(jmul(xg, p.c2));
    return JElem<T>::from_f32(jadd(a, b2));
}

template <typename T>
__global__ void __launch_bounds__(256)
combine_offset_kernel(const __grid_constant__ CombineOffsetParams p, const T* __restrict__ x_local, T* __restrict__ out) {
    const long long total = (long long)p.NC * p.H * p.W;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x)
        out[e] = combine_offset_elem<T>(p, x_local, e);
}


unsigned blocks_for(long long total) { return (unsigned)std::max(1LL, std::min((total + 255) / 256, 148LL * 32)); }

int check_origins(const char* who, const int32_t* origins_host, int n_tiles, int H, int W, int th, int tw) {
    if (origins_host == nullptr) return TD_OK;
    for (int t = 0; t < n_tiles; ++t) {
        const int ox = origins_host[2 * t], oy = origins_host[2 * t + 1];
        if (ox < 0 || oy < 0 || ox + tw > W || oy + th > H) {
            td_set_error("%s: window %d at (%d, %d) size %dx%d leaves the %dx%d canvas", who, t, ox, oy, tw, th, W, H);
            return TD_ERR_INVALID_ARG;
        }
    }
    return TD_OK;
}

// the wrap forms' host checks: known wrap bits, host origins present, and per axis 0 <= o < L with tile <= L when wrapped,
// -(tile - 1) <= o <= L - 1 (at least one pixel on the canvas) when bounded
int check_origins_wrap(const char* who, const int32_t* origins_host, int n_tiles, int H, int W, int th, int tw, int wrap) {
    if ((wrap & ~(int)(TD_WRAP_X | TD_WRAP_Y)) != 0 || origins_host == nullptr) {
        td_set_error("%s: bad arguments (wrap=%d, host origins %s)", who, wrap, origins_host ? "given" : "missing");
        return TD_ERR_INVALID_ARG;
    }
    const bool wx = (wrap & TD_WRAP_X) != 0, wy = (wrap & TD_WRAP_Y) != 0;
    if ((wx && tw > W) || (wy && th > H)) {
        td_set_error("%s: window %dx%d exceeds a wrapped axis of the %dx%d canvas", who, tw, th, W, H);
        return TD_ERR_INVALID_ARG;
    }
    for (int t = 0; t < n_tiles; ++t) {
        const int ox = origins_host[2 * t], oy = origins_host[2 * t + 1];
        const bool okx = wx ? (ox >= 0 && ox < W) : (ox >= -(tw - 1) && ox <= W - 1);
        const bool oky = wy ? (oy >= 0 && oy < H) : (oy >= -(th - 1) && oy <= H - 1);
        if (!okx || !oky) {
            td_set_error("%s: window %d at (%d, %d) size %dx%d is out of range on the %dx%d canvas (wrap=%d)", who, t, ox, oy, tw, th, W, H,
                         wrap);
            return TD_ERR_INVALID_ARG;
        }
    }
    return TD_OK;
}

}  // namespace

extern "C" int td_scatter_bboxes(const void* x, void* tiles, const int32_t* origins_dev, const int32_t* origins_host, int n_tiles,
                                 int N, int C, int H, int W, int tile_h, int tile_w, int dtype, void* stream) {
    if (x == nullptr || tiles == nullptr || origins_dev == nullptr || n_tiles <= 0 || N <= 0 || C <= 0 || H <= 0 || W <= 0 ||
        tile_h <= 0 || tile_w <= 0 || tile_h > H || tile_w > W) {
        td_set_error("td_scatter_bboxes: bad arguments");
        return TD_ERR_INVALID_ARG;
    }
    int rc = check_origins("td_scatter_bboxes", origins_host, n_tiles, H, W, tile_h, tile_w);
    if (rc != TD_OK) return rc;
    const long long total = (long long)n_tiles * N * C * tile_h * tile_w;
    cudaStream_t st = (cudaStream_t)stream;
    const int es = td_dtype_size(dtype);
    if (es == 2) scatter_bboxes_kernel<uint16_t><<<blocks_for(total), 256, 0, st>>>((const uint16_t*)x, (uint16_t*)tiles, origins_dev, N * C, H, W, tile_h, tile_w, total);
    else if (es == 4) scatter_bboxes_kernel<uint32_t><<<blocks_for(total), 256, 0, st>>>((const uint32_t*)x, (uint32_t*)tiles, origins_dev, N * C, H, W, tile_h, tile_w, total);
    else { td_set_error("td_scatter_bboxes: unknown dtype"); return TD_ERR_INVALID_ARG; }
    return launch_status("td_scatter_bboxes");
}

extern "C" int td_blend_bboxes(const void* const* batch_ptrs, int num_batches, int tile_bs, const int32_t* origins_dev,
                               const int32_t* origins_host, int n_tiles, int N, int C, int H, int W, int tile_h, int tile_w,
                               int dtype, float* out, void* stream) {
    if (batch_ptrs == nullptr || origins_dev == nullptr || out == nullptr || num_batches <= 0 || num_batches > TD_MAX_BATCH_PTRS ||
        tile_bs <= 0 || n_tiles <= 0 || (long long)num_batches * tile_bs < n_tiles || (long long)(num_batches - 1) * tile_bs >= n_tiles ||
        N <= 0 || C <= 0 || H <= 0 || W <= 0 || tile_h <= 0 || tile_w <= 0 || tile_h > H || tile_w > W) {
        td_set_error("td_blend_bboxes: bad arguments");
        return TD_ERR_INVALID_ARG;
    }
    int rc = check_origins("td_blend_bboxes", origins_host, n_tiles, H, W, tile_h, tile_w);
    if (rc != TD_OK) return rc;
    BlendListParams p;
    p.NC = N * C; p.H = H; p.W = W; p.th = tile_h; p.tw = tile_w; p.n_tiles = n_tiles; p.tile_bs = tile_bs;
    for (int b = 0; b < num_batches; ++b) {
        if (batch_ptrs[b] == nullptr) { td_set_error("td_blend_bboxes: null batch %d", b); return TD_ERR_INVALID_ARG; }
        p.batch_ptrs[b] = batch_ptrs[b];
    }
    const long long total = (long long)p.NC * H * W;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == TD_F16) blend_bboxes_kernel<__half><<<blocks_for(total), 256, 0, st>>>(p, origins_dev, out);
    else if (dtype == TD_BF16) blend_bboxes_kernel<__nv_bfloat16><<<blocks_for(total), 256, 0, st>>>(p, origins_dev, out);
    else if (dtype == TD_F32) blend_bboxes_kernel<float><<<blocks_for(total), 256, 0, st>>>(p, origins_dev, out);
    else { td_set_error("td_blend_bboxes: unknown dtype"); return TD_ERR_INVALID_ARG; }
    return launch_status("td_blend_bboxes");
}

extern "C" int td_scatter_bboxes_wrap(const void* x, void* tiles, const int32_t* origins_dev, const int32_t* origins_host, int n_tiles,
                                      int N, int C, int H, int W, int tile_h, int tile_w, int wrap, int dtype, void* stream) {
    if (x == nullptr || tiles == nullptr || origins_dev == nullptr || n_tiles <= 0 || N <= 0 || C <= 0 || H <= 0 || W <= 0 ||
        tile_h <= 0 || tile_w <= 0) {
        td_set_error("td_scatter_bboxes_wrap: bad arguments");
        return TD_ERR_INVALID_ARG;
    }
    int rc = check_origins_wrap("td_scatter_bboxes_wrap", origins_host, n_tiles, H, W, tile_h, tile_w, wrap);
    if (rc != TD_OK) return rc;
    const long long total = (long long)n_tiles * N * C * tile_h * tile_w;
    cudaStream_t st = (cudaStream_t)stream;
    const int es = td_dtype_size(dtype);
    if (es == 2) scatter_bboxes_wrap_kernel<uint16_t><<<blocks_for(total), 256, 0, st>>>((const uint16_t*)x, (uint16_t*)tiles, origins_dev, N * C, H, W, tile_h, tile_w, wrap, total);
    else if (es == 4) scatter_bboxes_wrap_kernel<uint32_t><<<blocks_for(total), 256, 0, st>>>((const uint32_t*)x, (uint32_t*)tiles, origins_dev, N * C, H, W, tile_h, tile_w, wrap, total);
    else { td_set_error("td_scatter_bboxes_wrap: unknown dtype"); return TD_ERR_INVALID_ARG; }
    return launch_status("td_scatter_bboxes_wrap");
}

extern "C" int td_blend_bboxes_wrap(const void* const* batch_ptrs, int num_batches, int tile_bs, const int32_t* origins_dev,
                                    const int32_t* origins_host, int n_tiles, int N, int C, int H, int W, int tile_h, int tile_w, int wrap,
                                    int dtype, float* out, void* stream) {
    if (batch_ptrs == nullptr || origins_dev == nullptr || out == nullptr || num_batches <= 0 || num_batches > TD_MAX_BATCH_PTRS ||
        tile_bs <= 0 || n_tiles <= 0 || (long long)num_batches * tile_bs < n_tiles || (long long)(num_batches - 1) * tile_bs >= n_tiles ||
        N <= 0 || C <= 0 || H <= 0 || W <= 0 || tile_h <= 0 || tile_w <= 0) {
        td_set_error("td_blend_bboxes_wrap: bad arguments");
        return TD_ERR_INVALID_ARG;
    }
    int rc = check_origins_wrap("td_blend_bboxes_wrap", origins_host, n_tiles, H, W, tile_h, tile_w, wrap);
    if (rc != TD_OK) return rc;
    BlendListParams p;
    p.NC = N * C; p.H = H; p.W = W; p.th = tile_h; p.tw = tile_w; p.n_tiles = n_tiles; p.tile_bs = tile_bs;
    for (int b = 0; b < num_batches; ++b) {
        if (batch_ptrs[b] == nullptr) { td_set_error("td_blend_bboxes_wrap: null batch %d", b); return TD_ERR_INVALID_ARG; }
        p.batch_ptrs[b] = batch_ptrs[b];
    }
    const long long total = (long long)p.NC * H * W;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == TD_F16) blend_bboxes_wrap_kernel<__half><<<blocks_for(total), 256, 0, st>>>(p, origins_dev, wrap, out);
    else if (dtype == TD_BF16) blend_bboxes_wrap_kernel<__nv_bfloat16><<<blocks_for(total), 256, 0, st>>>(p, origins_dev, wrap, out);
    else if (dtype == TD_F32) blend_bboxes_wrap_kernel<float><<<blocks_for(total), 256, 0, st>>>(p, origins_dev, wrap, out);
    else { td_set_error("td_blend_bboxes_wrap: unknown dtype"); return TD_ERR_INVALID_ARG; }
    return launch_status("td_blend_bboxes_wrap");
}

extern "C" int td_demofusion_combine_offset(const void* x_local, const void* const* view_batch_ptrs, int num_batches,
                                            int views_per_batch, int n_views, void* out, int N, int C, int H, int W, int s,
                                            int out_h, int out_w, int offset, int end_y, int end_x, int mixture, float c2,
                                            float one_minus_c2, int dtype, void* stream) {
    if (x_local == nullptr || out == nullptr || view_batch_ptrs == nullptr || num_batches <= 0 || num_batches > TD_MAX_BATCH_PTRS ||
        views_per_batch <= 0 || s <= 0 || n_views != (mixture ? 2 : 1) * s * s || (long long)num_batches * views_per_batch < n_views ||
        offset < 0 || N <= 0 || C <= 0 || H <= 0 || W <= 0 || end_y > H || end_x > W || out_h <= 0 || out_w <= 0) {
        td_set_error("td_demofusion_combine_offset: bad arguments");
        return TD_ERR_INVALID_ARG;
    }
    // every pixel of [offset, end) must map inside a view: i = (y - offset) / s < out_h
    if ((end_y > offset && (end_y - 1 - offset) / s >= out_h) || (end_x > offset && (end_x - 1 - offset) / s >= out_w)) {
        td_set_error("td_demofusion_combine_offset: views %dx%d do not cover [%d, %d) x [%d, %d) at scale %d", out_h, out_w, offset, end_y,
                     offset, end_x, s);
        return TD_ERR_INVALID_ARG;
    }
    CombineOffsetParams p;
    p.NC = N * C; p.H = H; p.W = W; p.s = s; p.oh = out_h; p.ow = out_w; p.end_y = end_y; p.end_x = end_x; p.off = offset;
    p.views_per_batch = views_per_batch; p.n_views = n_views; p.mixture = mixture; p.c2 = c2; p.one_minus_c2 = one_minus_c2;
    for (int b = 0; b < num_batches; ++b) {
        if (view_batch_ptrs[b] == nullptr) { td_set_error("td_demofusion_combine_offset: null batch %d", b); return TD_ERR_INVALID_ARG; }
        p.batch_ptrs[b] = view_batch_ptrs[b];
    }
    const long long total = (long long)p.NC * H * W;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == TD_F16) combine_offset_kernel<__half><<<blocks_for(total), 256, 0, st>>>(p, (const __half*)x_local, (__half*)out);
    else if (dtype == TD_BF16) combine_offset_kernel<__nv_bfloat16><<<blocks_for(total), 256, 0, st>>>(p, (const __nv_bfloat16*)x_local, (__nv_bfloat16*)out);
    else if (dtype == TD_F32) combine_offset_kernel<float><<<blocks_for(total), 256, 0, st>>>(p, (const float*)x_local, (float*)out);
    else { td_set_error("td_demofusion_combine_offset: unknown dtype"); return TD_ERR_INVALID_ARG; }
    return launch_status("td_demofusion_combine_offset");
}

#ifdef TD_JITTER_HOST_EMULATION
// Test-only (tests/emul/jitter_host_emul.cu includes this file with the macro set): run the element bodies on the host.
extern "C" int td_emul_scatter_bboxes(const void* x, void* tiles, const int32_t* origins, int n_tiles, int N, int C, int H, int W,
                                      int tile_h, int tile_w, int elem_size) {
    const long long total = (long long)n_tiles * N * C * tile_h * tile_w;
    for (long long e = 0; e < total; ++e) {
        if (elem_size == 2) ((uint16_t*)tiles)[e] = scatter_bboxes_elem<uint16_t>((const uint16_t*)x, origins, N * C, H, W, tile_h, tile_w, e);
        else ((uint32_t*)tiles)[e] = scatter_bboxes_elem<uint32_t>((const uint32_t*)x, origins, N * C, H, W, tile_h, tile_w, e);
    }
    return TD_OK;
}

extern "C" int td_emul_blend_bboxes(const void* const* batch_ptrs, int num_batches, int tile_bs, const int32_t* origins, int n_tiles,
                                    int N, int C, int H, int W, int tile_h, int tile_w, int dtype, float* out) {
    BlendListParams p;
    p.NC = N * C; p.H = H; p.W = W; p.th = tile_h; p.tw = tile_w; p.n_tiles = n_tiles; p.tile_bs = tile_bs;
    for (int b = 0; b < num_batches; ++b) p.batch_ptrs[b] = batch_ptrs[b];
    const long long total = (long long)p.NC * H * W;
    for (long long e = 0; e < total; ++e) {
        if (dtype == TD_F16) out[e] = blend_bboxes_elem<__half>(p, origins, e);
        else if (dtype == TD_BF16) out[e] = blend_bboxes_elem<__nv_bfloat16>(p, origins, e);
        else out[e] = blend_bboxes_elem<float>(p, origins, e);
    }
    return TD_OK;
}

extern "C" int td_emul_scatter_bboxes_wrap(const void* x, void* tiles, const int32_t* origins, int n_tiles, int N, int C, int H, int W,
                                           int tile_h, int tile_w, int wrap, int elem_size) {
    const int rc = check_origins_wrap("td_emul_scatter_bboxes_wrap", origins, n_tiles, H, W, tile_h, tile_w, wrap);
    if (rc != TD_OK) return rc;
    const long long total = (long long)n_tiles * N * C * tile_h * tile_w;
    for (long long e = 0; e < total; ++e) {
        if (elem_size == 2) ((uint16_t*)tiles)[e] = scatter_bboxes_wrap_elem<uint16_t>((const uint16_t*)x, origins, N * C, H, W, tile_h, tile_w, wrap, e);
        else ((uint32_t*)tiles)[e] = scatter_bboxes_wrap_elem<uint32_t>((const uint32_t*)x, origins, N * C, H, W, tile_h, tile_w, wrap, e);
    }
    return TD_OK;
}

extern "C" int td_emul_blend_bboxes_wrap(const void* const* batch_ptrs, int num_batches, int tile_bs, const int32_t* origins, int n_tiles,
                                         int N, int C, int H, int W, int tile_h, int tile_w, int wrap, int dtype, float* out) {
    const int rc = check_origins_wrap("td_emul_blend_bboxes_wrap", origins, n_tiles, H, W, tile_h, tile_w, wrap);
    if (rc != TD_OK) return rc;
    BlendListParams p;
    p.NC = N * C; p.H = H; p.W = W; p.th = tile_h; p.tw = tile_w; p.n_tiles = n_tiles; p.tile_bs = tile_bs;
    for (int b = 0; b < num_batches; ++b) p.batch_ptrs[b] = batch_ptrs[b];
    const long long total = (long long)p.NC * H * W;
    for (long long e = 0; e < total; ++e) {
        if (dtype == TD_F16) out[e] = blend_bboxes_wrap_elem<__half>(p, origins, wrap, e);
        else if (dtype == TD_BF16) out[e] = blend_bboxes_wrap_elem<__nv_bfloat16>(p, origins, wrap, e);
        else out[e] = blend_bboxes_wrap_elem<float>(p, origins, wrap, e);
    }
    return TD_OK;
}

extern "C" int td_emul_combine_offset(const void* x_local, const void* const* view_batch_ptrs, int num_batches, int views_per_batch,
                                      int n_views, void* out, int N, int C, int H, int W, int s, int out_h, int out_w, int offset,
                                      int end_y, int end_x, int mixture, float c2, float one_minus_c2, int dtype) {
    CombineOffsetParams p;
    p.NC = N * C; p.H = H; p.W = W; p.s = s; p.oh = out_h; p.ow = out_w; p.end_y = end_y; p.end_x = end_x; p.off = offset;
    p.views_per_batch = views_per_batch; p.n_views = n_views; p.mixture = mixture; p.c2 = c2; p.one_minus_c2 = one_minus_c2;
    for (int b = 0; b < num_batches; ++b) p.batch_ptrs[b] = view_batch_ptrs[b];
    const long long total = (long long)p.NC * H * W;
    for (long long e = 0; e < total; ++e) {
        if (dtype == TD_F16) ((__half*)out)[e] = combine_offset_elem<__half>(p, (const __half*)x_local, e);
        else if (dtype == TD_BF16) ((__nv_bfloat16*)out)[e] = combine_offset_elem<__nv_bfloat16>(p, (const __nv_bfloat16*)x_local, e);
        else ((float*)out)[e] = combine_offset_elem<float>(p, (const float*)x_local, e);
    }
    return TD_OK;
}
#endif
