// Region prompt control: the custom-bbox composite of a tiled step as ONE kernel
//   MultiDiffusion       multidiffusion.py:187-216  (BACKGROUND adds into x_buffer, divide by weights, FOREGROUND feather)
//   Mixture of Diffusers mixtureofdiffusers.py:145-175 (BACKGROUND adds weighted by custom_weights, FOREGROUND feather)
// The reference issues 1-3 slice updates per region plus up to 8 whole-canvas element-wise ops; here every output
// element is produced once, gather form: start from the grid accumulator x_buffer, walk the regions covering the
// pixel IN LIST ORDER and reproduce the reference's roundings --
//   BACKGROUND   acc = round_T(float(acc) + float(r))                      (x_buffer[slicer] += x_tile_out)
//                acc = round_T(float(acc) + float(r) * w)                  (Mixture: x_tile_out * custom_weights, fp32 product)
//   normalise    o = weights > 1 ? float(acc) / weights : float(acc)       (MultiDiffusion only; IEEE divide)
//   FOREGROUND   fb = round_T(float(fb) + float(r)); fm += mask; fc += 1   (feather buffer in T, mask / count in fp32)
//   composite    if fc > 1: fbf = float(fb) / fc, fm = fm / fc;  if fc > 0: o = o * (1 - fm) + fbf * fm
//                (each product and the sum rounded separately: no FMA contraction)
// r is a region output read in ITS OWN dtype (td_region.dtype), which need not be T: the reference's `x_buffer[slicer] +=
// x_tile_out` with an fp32 UNet output on an fp16 canvas adds in fp32 and rounds once, so the output must not be rounded
// to T on its way in.  The dtype is uniform across a region, so the per-visit switch does not diverge.
// td_region_composite_rows runs the same kernel over a window of canvas rows (the row-strip shard composites only the
// rows a rank owns); td_region_composite is its [0, H) case.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "td_b200.h"
#include "td_device.cuh"
#include "td_internal.h"
#include "td_launch.h"

namespace {

using namespace td;

struct RegionParams {
    int n;
    int N, C, H, W;
    int row_begin, rows;              // canvas rows [row_begin, row_begin + rows) are produced; the rest of `out` is untouched
    int divide;                       // 1: MultiDiffusion normalisation by the weight canvas
    int x[TD_MAX_REGIONS], y[TD_MAX_REGIONS], w[TD_MAX_REGIONS], h[TD_MAX_REGIONS], mode[TD_MAX_REGIONS];
    int dtype[TD_MAX_REGIONS];            // td_dtype of out[r]
    const void* out[TD_MAX_REGIONS];      // region denoiser output [N, C, h, w] of dtype[r]
    const float* aux[TD_MAX_REGIONS];     // BACKGROUND: optional fp32 [h*w] multiplier; FOREGROUND: fp32 [h*w] feather mask
};

// Element i of a region output of td_dtype dt, exactly as fp32.
__device__ __forceinline__ float load_region_value(const void* p, long long i, int dt) {
    switch (dt) {
        case TD_F16: return Elem<__half>::to_f32(reinterpret_cast<const __half*>(p)[i]);
        case TD_BF16: return Elem<__nv_bfloat16>::to_f32(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
        default: return reinterpret_cast<const float*>(p)[i];
    }
}

template <typename T>
__global__ void __launch_bounds__(256)
region_composite_kernel(const __grid_constant__ RegionParams p, const T* __restrict__ x_buffer, const float* __restrict__ weights,
                        float* __restrict__ out) {
    const long long total = (long long)p.N * p.C * p.rows * p.W;
    for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (long long)gridDim.x * blockDim.x) {
        const int px = (int)(k % p.W);
        long long t = k / p.W;
        const int py = p.row_begin + (int)(t % p.rows);
        const long long plane = t / p.rows;            // n * C + c
        const long long i = (plane * p.H + py) * p.W + px;
        float acc = Elem<T>::to_f32(x_buffer[i]);
        float fb = 0.0f, fm = 0.0f, fc = 0.0f;
        for (int r = 0; r < p.n; ++r) {
            const int u = px - p.x[r], v = py - p.y[r];
            if ((unsigned)u >= (unsigned)p.w[r] || (unsigned)v >= (unsigned)p.h[r]) continue;
            const long long ro = (plane * p.h[r] + v) * (long long)p.w[r] + u;
            const float val = load_region_value(p.out[r], ro, p.dtype[r]);
            if (p.mode[r] == 0) {
                const float add = p.aux[r] != nullptr ? __fmul_rn(val, p.aux[r][(long long)v * p.w[r] + u]) : val;
                acc = round_through<T>(__fadd_rn(acc, add));
            } else {
                fb = round_through<T>(__fadd_rn(fb, val));
                fm = __fadd_rn(fm, p.aux[r][(long long)v * p.w[r] + u]);
                fc += 1.0f;
            }
        }
        float o = acc;
        if (p.divide) {
            const float w = weights[(long long)py * p.W + px];
            if (w > 1.0f) o = __fdiv_rn(acc, w);
        }
        if (fc > 0.0f) {
            float fbf = fb;
            if (fc > 1.0f) { fbf = __fdiv_rn(fb, fc); fm = __fdiv_rn(fm, fc); }
            o = __fadd_rn(__fmul_rn(o, __fsub_rn(1.0f, fm)), __fmul_rn(fbf, fm));
        }
        out[i] = o;
    }
}

// Both entry points: validation, parameter block and launch for canvas rows [row_begin, row_end).
int region_composite_launch(const char* fn, const void* x_buffer, const float* weights, const td_region* regions, int n_regions, int N,
                            int C, int H, int W, int dtype, float* out, int row_begin, int row_end, void* stream) {
    if (x_buffer == nullptr || out == nullptr || N <= 0 || C <= 0 || H <= 0 || W <= 0 || n_regions < 0 || (n_regions > 0 && regions == nullptr)) {
        td_set_error("%s: bad arguments", fn);
        return TD_ERR_INVALID_ARG;
    }
    if (dtype != TD_F16 && dtype != TD_BF16 && dtype != TD_F32) {
        td_set_error("%s: unknown dtype %d", fn, dtype);
        return TD_ERR_INVALID_ARG;
    }
    if (row_begin < 0 || row_begin > row_end || row_end > H) {
        td_set_error("%s: rows [%d,%d) outside [0,%d)", fn, row_begin, row_end, H);
        return TD_ERR_INVALID_ARG;
    }
    if (n_regions > TD_MAX_REGIONS) { td_set_error("%s: %d regions exceed TD_MAX_REGIONS=%d", fn, n_regions, TD_MAX_REGIONS); return TD_ERR_UNSUPPORTED; }
    RegionParams p;
    p.n = n_regions; p.N = N; p.C = C; p.H = H; p.W = W;
    p.row_begin = row_begin; p.rows = row_end - row_begin;
    p.divide = weights != nullptr ? 1 : 0;
    for (int r = 0; r < n_regions; ++r) {
        const td_region& g = regions[r];
        if (g.x < 0 || g.y < 0 || g.w <= 0 || g.h <= 0 || g.x + g.w > W || g.y + g.h > H || g.out == nullptr || (g.mode != 0 && g.mode != 1) ||
            (g.mode == 1 && g.aux == nullptr) || (g.dtype != TD_F16 && g.dtype != TD_BF16 && g.dtype != TD_F32)) {
            td_set_error("%s: region %d is invalid", fn, r);
            return TD_ERR_INVALID_ARG;
        }
        p.x[r] = g.x; p.y[r] = g.y; p.w[r] = g.w; p.h[r] = g.h; p.mode[r] = g.mode; p.dtype[r] = g.dtype; p.out[r] = g.out; p.aux[r] = g.aux;
    }
    if (p.rows == 0) return TD_OK;
    const long long total = (long long)N * C * p.rows * W;
    const int grid = (int)std::min<long long>((total + 255) / 256, 148LL * 16);
    cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case TD_F16: region_composite_kernel<__half><<<grid, 256, 0, st>>>(p, (const __half*)x_buffer, weights, out); break;
        case TD_BF16: region_composite_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(p, (const __nv_bfloat16*)x_buffer, weights, out); break;
        case TD_F32: region_composite_kernel<float><<<grid, 256, 0, st>>>(p, (const float*)x_buffer, weights, out); break;
    }
    return launch_status(fn);
}

}  // namespace

extern "C" int td_region_composite(const void* x_buffer, const float* weights, const td_region* regions, int n_regions, int N, int C,
                                   int H, int W, int dtype, float* out, void* stream) {
    return region_composite_launch("td_region_composite", x_buffer, weights, regions, n_regions, N, C, H, W, dtype, out, 0, H, stream);
}

extern "C" int td_region_composite_rows(const void* x_buffer, const float* weights, const td_region* regions, int n_regions, int N,
                                        int C, int H, int W, int dtype, float* out, int row_begin, int row_end, void* stream) {
    return region_composite_launch("td_region_composite_rows", x_buffer, weights, regions, n_regions, N, C, H, W, dtype, out, row_begin,
                                   row_end, stream);
}
