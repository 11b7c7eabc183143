// SpotDiffusion (new: the reference has no such method): the weight canvas of a tile plan written on the device.
//
//   td_grid_counts  <- td_grid_weights(g, NULL) + td_rescale_factor, without the host pass and the upload
//
// SpotDiffusion moves its windows on every denoiser call (td_grid_shift), so its MultiDiffusion blend needs a fresh count
// canvas per call.  The canvas of a separable plan is an outer product: weights[y][x] = rows covering y * columns covering x.
// Each CTA counts both axes into shared memory (two binary searches per position over the sorted origins, plus one across
// the seam on a wrapped axis), then streams the canvas -- and RN(1/count) -- out with 16-byte stores.  The product of two
// counts <= 256 is an integer below 2^24, exact in fp32, and so is every partial sum of td_grid_weights' `+= 1.0f`.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "td_b200.h"
#include "td_internal.h"
#include "td_launch.h"

namespace {

using namespace td;

constexpr int kCountThreads = 256;

struct CountParams {
    int W, H, tw, th, cols, rows, wrap;
    unsigned total;  // W * H < 2^30
    int32_t xs[TD_MAX_GRID_DIM], ys[TD_MAX_GRID_DIM];
};

// #{k : o[k] <= v} over non-decreasing o[0 .. n)
__device__ __forceinline__ int count_le(const int32_t* o, int n, int v) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int m = (lo + hi) >> 1;
        if (o[m] <= v) lo = m + 1; else hi = m;
    }
    return lo;
}

// Windows of length t at origins o covering position p: o in (p - t, p], and on a periodic axis also o in (p - t + L, L).
__device__ __forceinline__ int axis_count(const int32_t* o, int n, int L, int t, bool periodic, int p) {
    int c = count_le(o, n, p) - count_le(o, n, p - t);
    if (periodic && p < t) c += n - count_le(o, n, p - t + L);
    return c;
}

template <bool RCP>
__global__ void __launch_bounds__(kCountThreads)
grid_counts_kernel(const __grid_constant__ CountParams p, float* __restrict__ weights, float* __restrict__ rcp_weights) {
    extern __shared__ uint16_t cnt[];  // [W] column counts, then [H] row counts
    __shared__ int32_t org[2 * TD_MAX_GRID_DIM];
    for (int i = threadIdx.x; i < p.cols; i += blockDim.x) org[i] = p.xs[i];
    for (int i = threadIdx.x; i < p.rows; i += blockDim.x) org[TD_MAX_GRID_DIM + i] = p.ys[i];
    __syncthreads();
    for (int x = threadIdx.x; x < p.W; x += blockDim.x)
        cnt[x] = (uint16_t)axis_count(org, p.cols, p.W, p.tw, (p.wrap & TD_WRAP_X) != 0, x);
    for (int y = threadIdx.x; y < p.H; y += blockDim.x)
        cnt[p.W + y] = (uint16_t)axis_count(org + TD_MAX_GRID_DIM, p.rows, p.H, p.th, (p.wrap & TD_WRAP_Y) != 0, y);
    __syncthreads();
    const uint16_t* cy = cnt + p.W;
    const unsigned nvec = p.total >> 2;
    for (unsigned v = blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += gridDim.x * blockDim.x) {
        const unsigned i = v * 4u;
        unsigned y = i / (unsigned)p.W, x = i - y * (unsigned)p.W;
        float w[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            w[j] = (float)((int)cnt[x] * (int)cy[y]);
            if (++x == (unsigned)p.W) { x = 0; ++y; }
        }
        reinterpret_cast<float4*>(weights)[v] = make_float4(w[0], w[1], w[2], w[3]);
        if constexpr (RCP)
            reinterpret_cast<float4*>(rcp_weights)[v] =
                make_float4(__fdiv_rn(1.0f, w[0]), __fdiv_rn(1.0f, w[1]), __fdiv_rn(1.0f, w[2]), __fdiv_rn(1.0f, w[3]));
    }
    // the last W*H mod 4 elements
    const unsigned tail = nvec * 4u + threadIdx.x;
    if (blockIdx.x == 0 && tail < p.total) {
        const unsigned y = tail / (unsigned)p.W, x = tail - y * (unsigned)p.W;
        const float w = (float)((int)cnt[x] * (int)cy[y]);
        weights[tail] = w;
        if constexpr (RCP) rcp_weights[tail] = __fdiv_rn(1.0f, w);
    }
}

}  // namespace

extern "C" int td_grid_counts(const td_grid* g, float* weights, float* rcp_weights, void* stream) {
    if (g == nullptr || weights == nullptr) {
        td_set_error("grid_counts: null");
        return TD_ERR_INVALID_ARG;
    }
    if (g->rows <= 0 || g->cols <= 0 || g->rows > TD_MAX_GRID_DIM || g->cols > TD_MAX_GRID_DIM || g->W <= 0 || g->H <= 0 ||
        (g->wrap & ~(int)(TD_WRAP_X | TD_WRAP_Y)) != 0) {
        td_set_error("grid_counts: grid not initialised (rows=%d cols=%d W=%d H=%d wrap=%d)", g->rows, g->cols, g->W, g->H, g->wrap);
        return TD_ERR_INVALID_ARG;
    }
    if (g->H >= 32768 || g->W >= 32768) {
        td_set_error("grid_counts: canvas %dx%d too large", g->H, g->W);
        return TD_ERR_UNSUPPORTED;
    }
    const int W = g->W, H = g->H, tw = g->tile_w, th = g->tile_h;
    const bool px = (g->wrap & TD_WRAP_X) != 0, py = (g->wrap & TD_WRAP_Y) != 0;
    for (int c = 0; c < g->cols; ++c)
        if (g->xs[c] < 0 || g->xs[c] >= W || tw <= 0 || tw > W || (!px && g->xs[c] + tw > W)) {
            td_set_error("grid_counts: tile column %d (x=%d, w=%d) leaves the %d-wide canvas", c, g->xs[c], tw, W);
            return TD_ERR_INVALID_ARG;
        }
    for (int r = 0; r < g->rows; ++r)
        if (g->ys[r] < 0 || g->ys[r] >= H || th <= 0 || th > H || (!py && g->ys[r] + th > H)) {
            td_set_error("grid_counts: tile row %d (y=%d, h=%d) leaves the %d-high canvas", r, g->ys[r], th, H);
            return TD_ERR_INVALID_ARG;
        }
    for (int c = 1; c < g->cols; ++c)
        if (g->xs[c] < g->xs[c - 1]) {
            td_set_error("grid_counts: tile column origins out of order: xs[%d]=%d < xs[%d]=%d", c, g->xs[c], c - 1, g->xs[c - 1]);
            return TD_ERR_INVALID_ARG;
        }
    for (int r = 1; r < g->rows; ++r)
        if (g->ys[r] < g->ys[r - 1]) {
            td_set_error("grid_counts: tile row origins out of order: ys[%d]=%d < ys[%d]=%d", r, g->ys[r], r - 1, g->ys[r - 1]);
            return TD_ERR_INVALID_ARG;
        }
    if (!aligned16(weights) || (rcp_weights != nullptr && !aligned16(rcp_weights))) {
        td_set_error("grid_counts: weights and rcp_weights must be 16-byte aligned");
        return TD_ERR_INVALID_ARG;
    }
    CountParams p;
    p.W = W; p.H = H; p.tw = tw; p.th = th; p.cols = g->cols; p.rows = g->rows; p.wrap = g->wrap;
    p.total = (unsigned)W * (unsigned)H;
    std::copy(g->xs, g->xs + TD_MAX_GRID_DIM, p.xs);
    std::copy(g->ys, g->ys + TD_MAX_GRID_DIM, p.ys);
    const int smem = (int)(((size_t)(W + H) * sizeof(uint16_t) + 15) & ~(size_t)15);
    const DeviceProps dp = device_props();
    const unsigned nvec = p.total >> 2;
    const int want = (int)std::max(1u, (nvec + kCountThreads - 1) / kCountThreads);
    const int grid = std::min(want, dp.ok ? dp.sms * 4 : 528);
    cudaStream_t st = (cudaStream_t)stream;
    // no programmatic dependent launch: the canvas may still be read by the previous call's blend
    if (rcp_weights != nullptr) {
        int rc = smem_optin(grid_counts_kernel<true>, smem, "td_grid_counts");
        if (rc != TD_OK) return rc;
        return launch("td_grid_counts", grid_counts_kernel<true>, dim3(grid), dim3(kCountThreads), (size_t)smem, st, false, p, weights,
                      rcp_weights);
    }
    int rc = smem_optin(grid_counts_kernel<false>, smem, "td_grid_counts");
    if (rc != TD_OK) return rc;
    return launch("td_grid_counts", grid_counts_kernel<false>, dim3(grid), dim3(kCountThreads), (size_t)smem, st, false, p, weights,
                  rcp_weights);
}
