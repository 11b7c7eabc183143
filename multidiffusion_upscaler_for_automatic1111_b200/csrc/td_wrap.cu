// Seamless tiling on sm_90a: the scatter and both blends on a canvas that is periodic in x and / or y (td_grid.wrap).
//
// The arithmetic is that of td_diffusion.cu -- covering tiles visited in ascending tile index, one rounding through
// the canvas dtype per add, MultiDiffusion's `weights > 1 ? acc / weights : acc` in fp32, Mixture of Diffusers'
// separate fp32 products -- with modular coverage: canvas column x is covered by tile column c when
// (x - xs[c]) mod W < tile_w, and the tile element is read at that residue.  The extended (circularly padded)
// canvas is never materialised: every kernel computes the residues in its index arithmetic.
//
//   * scatter: one thread per 16-byte vector of the tile batch; the source window (xs + u) mod W is two aligned
//     canvas chunks funnel-shifted together, the second one being chunk 0 when the window crosses the seam (W is a
//     multiple of the vector, so the seam is a chunk boundary).
//   * blends: gather form, one thread per 16-byte vector of the canvas.  The covering tiles of an axis are two
//     ascending index ranges -- origins in (p - t, p] and, on a periodic axis, origins in (p - t + L, L) (tiles that
//     run past L and reach p after the seam) -- found by a search over the origins in shared memory.
//   * any width / alignment / mixed dtypes: one element per thread.
//   All launched with programmatic dependent launch, like the default kernels.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "td_b200.h"
#include "td_device.cuh"
#include "td_internal.h"
#include "td_launch.h"

namespace {

using namespace td;

struct WrapParams {
    int H, W, th, tw, rows, cols, N, C;
    int wrap_x, wrap_y;
    float inv_dx, inv_dy;  // origin-search estimates (any value is safe)
    int tile_bs;
    long long tile_stride;  // N*C*th*tw elements
    short ys[TD_MAX_GRID_DIM];
    short xs[TD_MAX_GRID_DIM];
    const void* batch_ptrs[TD_MAX_BATCH_PTRS];
};

enum { MODE_MD = 0, MODE_MOD = 1 };

// Tiles of one axis that cover at least one position of [lo, hi]: index range A = [a0, a1] (origins in (lo - t, hi])
// then, on a periodic axis, B = [b0, n) (origins in (lo - t + L, L)), ascending and disjoint.  `na` = |A|, `n` = |A|+|B|.
struct Cover {
    int a0, na, b0, n;
    __device__ __forceinline__ int at(int i) const { return i < na ? a0 + i : b0 + (i - na); }
};

__device__ __forceinline__ Cover cover(const short* o, int cnt, int lo, int hi, int t, int L, bool wrap, float inv) {
    Cover c;
    const int a1 = last_le(o, cnt, hi, inv);
    c.a0 = last_le(o, cnt, lo - t, inv) + 1;
    c.na = max(0, a1 - c.a0 + 1);
    c.b0 = wrap ? max(last_le(o, cnt, lo - t + L, inv) + 1, a1 + 1) : cnt;
    c.n = c.na + max(0, cnt - c.b0);
    return c;
}

__device__ __forceinline__ void load_origins(const WrapParams& p, short* s_ys, short* s_xs) {
    const int tid = threadIdx.y * blockDim.x + threadIdx.x, nt = blockDim.x * blockDim.y;
    for (int i = tid; i < p.rows; i += nt) s_ys[i] = p.ys[i];
    for (int i = tid; i < p.cols; i += nt) s_xs[i] = p.xs[i];
    __syncthreads();
}

// ---------------------------------------------------------------------------
// Scatter: tiles[(t - tile_begin)*N + n, c, v, u] = x[n, c, (ys + v) mod H, (xs + u) mod W]
// ---------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(128)
wrap_scatter_vec_kernel(const __grid_constant__ WrapParams p, const T* __restrict__ x, T* __restrict__ tiles, int tile_begin,
                        int rows_per_block) {
    constexpr int VEC = Vec<T>::kElems;
    constexpr int L2V = Vec<T>::kLog2;
    const int NC = p.N * p.C;
    const int tp = blockIdx.x;                      // (tile local, n, c) plane of the tile batch
    const int tl = tp / NC;
    const int plane = tp - tl * NC;
    const int t = tile_begin + tl;
    const int r = t / p.cols, c = t - r * p.cols;
    const int xs = p.xs[c], ys = p.ys[r];
    const int twv = p.tw >> L2V, wv = p.W >> L2V;
    const int v0 = blockIdx.y * rows_per_block;
    const int nvec = min(rows_per_block, p.th - v0) * twv;
    const T* src = x + (long long)plane * p.H * p.W;
    T* dst = tiles + ((long long)tp * p.th + v0) * p.tw;
    pdl_launch_dependents();
    pdl_wait();
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
        const int vi = i / twv, uv = i - vi * twv;
        int yy = ys + v0 + vi;
        if (yy >= p.H) yy -= p.H;                   // only on a periodic axis: bounded plans stay inside (validated)
        int xx = xs + uv * VEC;
        if (xx >= p.W) xx -= p.W;
        const int k0 = xx >> L2V, s = xx & (VEC - 1);
        const T* row = src + (long long)yy * p.W;
        const uint4 A = ldg128(row + (long long)k0 * VEC);
        uint4 B = make_uint4(0, 0, 0, 0);
        if (s != 0) B = ldg128(row + (long long)(k0 + 1 == wv ? 0 : k0 + 1) * VEC);   // across the seam: chunk 0
        stg128(dst + (long long)i * VEC, Vec<T>::window(A, B, s));
    }
}

template <typename T>
__global__ void __launch_bounds__(256)
wrap_scatter_generic_kernel(const __grid_constant__ WrapParams p, const T* __restrict__ x, T* __restrict__ tiles, int tile_begin,
                            long long total) {
    pdl_launch_dependents();
    pdl_wait();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    long long rem = idx;
    const int u = (int)(rem % p.tw); rem /= p.tw;
    const int v = (int)(rem % p.th); rem /= p.th;
    const int plane = (int)(rem % (p.N * p.C)); rem /= (p.N * p.C);
    const int t = tile_begin + (int)rem;
    const int r = t / p.cols, c = t - r * p.cols;
    int yy = p.ys[r] + v, xx = p.xs[c] + u;
    if (yy >= p.H) yy -= p.H;
    if (xx >= p.W) xx -= p.W;
    tiles[idx] = x[((long long)plane * p.H + yy) * p.W + xx];
}

// ---------------------------------------------------------------------------
// Blends, vector path: thread (threadIdx.x, threadIdx.y) owns the 16-byte vector blockIdx.x*32 + threadIdx.x of canvas
// row blockIdx.y*4 + threadIdx.y in plane blockIdx.z.
// ---------------------------------------------------------------------------
constexpr int kWrapBX = 32, kWrapBY = 4;

// Row-window form (td_blend_*_wrap_rows, row-strip shard): the grid covers the canvas rows [row_begin, row_end) only, with
// blockIdx.z = CTA row (slowest, walked from the window's end when `descending`) and blockIdx.y = plane.  A CTA any of whose
// rows is covered by a tile row outside the own bands [own_lo, own_hi) (every CTA when that range is empty) first waits
// until wait_flags[i] >= *wait_value for i < wait_count: its tile reads may come from a neighbour's halo push.
struct WindowParams {
    int row_begin, row_end, rb_count, descending;
    int wait_count, own_lo, own_hi;
    const uint32_t* wait_flags;
    const uint32_t* wait_value;
};

// a non-empty index range [s, s + n) of tile rows that is not inside the own bands
__device__ __forceinline__ bool leaves_own(const WindowParams& w, int s, int n) { return n > 0 && (s < w.own_lo || s + n > w.own_hi); }

template <typename T, int MODE>
struct VisitAcc {
    static constexpr int VEC = Vec<T>::kElems;
    static constexpr int L2V = Vec<T>::kLog2;
    // add the tile-row elements [b, b + VEC) that lie inside the tile (0 <= b + k < tw) into acc[k]
    __device__ static __forceinline__ void run(const T* __restrict__ trow, int b, int tw, const float* __restrict__ tw_row,
                                               const float* rsc, float* acc) {
        const int q = b >> L2V, s = b & (VEC - 1), twv = tw >> L2V;   // q = floor(b / VEC), also for b < 0
        const uint4 A = (q >= 0 && q < twv) ? ldg128(trow + (long long)q * VEC) : make_uint4(0, 0, 0, 0);
        const uint4 B = (s != 0 && q + 1 >= 0 && q + 1 < twv) ? ldg128(trow + (long long)(q + 1) * VEC) : make_uint4(0, 0, 0, 0);
        const uint4 w = Vec<T>::window(A, B, s);
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
            const int u = b + k;
            if (u >= 0 && u < tw) {
                float val = Vec<T>::get(w, k);
                if constexpr (MODE == MODE_MOD) val = __fmul_rn(val, __fmul_rn(tw_row[u], rsc[k]));
                acc[k] = round_through<T>(__fadd_rn(acc[k], val));
            }
        }
    }
};

template <typename T, int MODE, bool WRITE_BUF, bool WINDOW>
__global__ void __launch_bounds__(kWrapBX * kWrapBY)
wrap_blend_vec_kernel(const __grid_constant__ WrapParams p, const float* __restrict__ weights, const float* __restrict__ tile_weights,
                      const float* __restrict__ rescale, float* __restrict__ out_f32, T* __restrict__ out_buf,
                      const __grid_constant__ WindowParams w) {
    constexpr int VEC = Vec<T>::kElems;
    constexpr int L2V = Vec<T>::kLog2;
    __shared__ short s_ys[TD_MAX_GRID_DIM];
    __shared__ short s_xs[TD_MAX_GRID_DIM];
    load_origins(p, s_ys, s_xs);
    pdl_launch_dependents();
    const int xv = blockIdx.x * kWrapBX + threadIdx.x;
    const int y = WINDOW ? w.row_begin + (w.descending ? w.rb_count - 1 - (int)blockIdx.z : (int)blockIdx.z) * kWrapBY + (int)threadIdx.y
                         : (int)(blockIdx.y * kWrapBY + threadIdx.y);
    const int plane = WINDOW ? blockIdx.y : blockIdx.z;
    const int x = xv * VEC;
    const bool live = x < p.W && y < (WINDOW ? w.row_end : p.H);
    Cover cy{0, 0, 0, 0}, cx{0, 0, 0, 0};
    if (live) {
        cy = cover(s_ys, p.rows, y, y, p.th, p.H, p.wrap_y, p.inv_dy);
        cx = cover(s_xs, p.cols, x, x + VEC - 1, p.tw, p.W, p.wrap_x, p.inv_dx);
    }
    pdl_wait();
    if constexpr (WINDOW) {
        // both index ranges of the row cover: under wrap_y a row near the top is covered by band 0 AND by the last band(s)
        const bool foreign = live && (leaves_own(w, cy.a0, cy.na) || leaves_own(w, cy.b0, cy.n - cy.na));
        if (w.wait_count > 0 && __syncthreads_or(foreign)) {
            if (threadIdx.y == 0 && (int)threadIdx.x < w.wait_count) spin_until_ge(w.wait_flags + threadIdx.x, *w.wait_value);
            __syncthreads();   // publishes the acquire to the CTA before any tile read
        }
    }
    if (!live) return;
    const long long pix = (long long)y * p.W + x;
    float acc[VEC];
    float rsc[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) acc[k] = 0.0f;
    if constexpr (MODE == MODE_MOD) {
#pragma unroll
        for (int k = 0; k < VEC; k += 4) {
            const float4 r4 = __ldg(reinterpret_cast<const float4*>(rescale + pix + k));
            rsc[k] = r4.x; rsc[k + 1] = r4.y; rsc[k + 2] = r4.z; rsc[k + 3] = r4.w;
        }
    }
    for (int i = 0; i < cy.n; ++i) {
        const int r = cy.at(i);
        int v = y - (int)s_ys[r];
        if (v < 0) v += p.H;
        const float* tw_row = MODE == MODE_MOD ? tile_weights + (long long)v * p.tw : nullptr;
        for (int j = 0; j < cx.n; ++j) {
            const int c = cx.at(j);
            int b = x - (int)s_xs[c];                  // tile column of canvas element k is b + k
            if (j >= cx.na) b += p.W;                  // range B: the tile reaches x after the seam
            const int t = r * p.cols + c;
            const int bi = t / p.tile_bs;
            const T* trow = reinterpret_cast<const T*>(p.batch_ptrs[bi]) + (long long)(t - bi * p.tile_bs) * p.tile_stride +
                            ((long long)plane * p.th + v) * p.tw;
            VisitAcc<T, MODE>::run(trow, b, p.tw, tw_row, rsc, acc);
            // the vector straddles this tile's origin and the tile also reaches its left part after the seam
            // (a tile as wide as the canvas): those elements sit at b + W + k
            if (p.wrap_x && b < 0 && b + p.W < p.tw) VisitAcc<T, MODE>::run(trow, b + p.W, p.tw, tw_row, rsc, acc);
        }
    }
    if constexpr (MODE == MODE_MD) {
#pragma unroll
        for (int k = 0; k < VEC; k += 4) {
            const float4 w4 = __ldg(reinterpret_cast<const float4*>(weights + pix + k));
            const float w[4] = {w4.x, w4.y, w4.z, w4.w};
            float o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) o[e] = w[e] > 1.0f ? __fdiv_rn(acc[k + e], w[e]) : acc[k + e];
            *reinterpret_cast<float4*>(out_f32 + (long long)plane * p.H * p.W + pix + k) = make_float4(o[0], o[1], o[2], o[3]);
        }
    }
    if constexpr (WRITE_BUF) {
        union { uint4 u; T e[VEC]; } pk;
#pragma unroll
        for (int k = 0; k < VEC; ++k) pk.e[k] = Elem<T>::from_f32(acc[k]);
        stg128(out_buf + (long long)plane * p.H * p.W + pix, pk.u);
    }
    (void)L2V;
}

// Blends, generic path: one element per thread, any width / alignment, tile and canvas dtypes independent.
template <typename TIn, typename TAcc, int MODE>
__global__ void __launch_bounds__(256)
wrap_blend_generic_kernel(const __grid_constant__ WrapParams p, const float* __restrict__ weights, const float* __restrict__ tile_weights,
                          const float* __restrict__ rescale, float* __restrict__ out_f32, TAcc* __restrict__ out_buf, long long total) {
    __shared__ short s_ys[TD_MAX_GRID_DIM];
    __shared__ short s_xs[TD_MAX_GRID_DIM];
    load_origins(p, s_ys, s_xs);
    pdl_launch_dependents();
    pdl_wait();
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    long long rem = idx;
    const int x = (int)(rem % p.W); rem /= p.W;
    const int y = (int)(rem % p.H); rem /= p.H;
    const int plane = (int)rem;
    const Cover cy = cover(s_ys, p.rows, y, y, p.th, p.H, p.wrap_y, p.inv_dy);
    const Cover cx = cover(s_xs, p.cols, x, x, p.tw, p.W, p.wrap_x, p.inv_dx);
    float acc = 0.0f;
    float rsc = 0.0f;
    if constexpr (MODE == MODE_MOD) rsc = rescale[(long long)y * p.W + x];
    for (int i = 0; i < cy.n; ++i) {
        const int r = cy.at(i);
        int v = y - (int)s_ys[r];
        if (v < 0) v += p.H;
        for (int j = 0; j < cx.n; ++j) {
            const int c = cx.at(j);
            int u = x - (int)s_xs[c];
            if (u < 0) u += p.W;
            const int t = r * p.cols + c;
            const int b = t / p.tile_bs;
            const TIn* tp = reinterpret_cast<const TIn*>(p.batch_ptrs[b]) + (long long)(t - b * p.tile_bs) * p.tile_stride +
                            ((long long)plane * p.th + v) * p.tw + u;
            float val = Elem<TIn>::to_f32(*tp);
            if constexpr (MODE == MODE_MOD) val = __fmul_rn(val, __fmul_rn(tile_weights[(long long)v * p.tw + u], rsc));
            acc = round_through<TAcc>(__fadd_rn(acc, val));
        }
    }
    if constexpr (MODE == MODE_MD) {
        const float w = weights[(long long)y * p.W + x];
        out_f32[idx] = w > 1.0f ? __fdiv_rn(acc, w) : acc;
    }
    if (out_buf != nullptr) out_buf[idx] = Elem<TAcc>::from_f32(acc);
}

// ---------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------
void fill_params(const td_grid* g, int N, int C, WrapParams* p) {
    p->H = g->H; p->W = g->W; p->th = g->tile_h; p->tw = g->tile_w;
    p->rows = g->rows; p->cols = g->cols; p->N = N; p->C = C;
    p->wrap_x = (g->wrap & TD_WRAP_X) ? 1 : 0;
    p->wrap_y = (g->wrap & TD_WRAP_Y) ? 1 : 0;
    // periodic origins are floor(k * L / n): k ~ p * n / L; bounded ones follow split_bboxes' stride
    p->inv_dx = p->wrap_x ? (float)g->cols / (float)g->W
                          : (g->cols > 1 ? (float)(g->cols - 1) / (float)std::max(1, g->W - g->tile_w) : 0.0f);
    p->inv_dy = p->wrap_y ? (float)g->rows / (float)g->H
                          : (g->rows > 1 ? (float)(g->rows - 1) / (float)std::max(1, g->H - g->tile_h) : 0.0f);
    for (int i = 0; i < g->rows; ++i) p->ys[i] = (short)g->ys[i];
    for (int i = 0; i < g->cols; ++i) p->xs[i] = (short)g->xs[i];
    p->tile_bs = 1;
    p->tile_stride = (long long)N * C * g->tile_h * g->tile_w;
}

inline unsigned blocks_for(long long total, int threads) { return (unsigned)((total + threads - 1) / threads); }

template <typename T>
int scatter_impl(const WrapParams& p, const void* x, void* tiles, int tile_begin, int n_tiles, bool vec, bool pdl, cudaStream_t st) {
    const long long elems = (long long)n_tiles * p.N * p.C * p.th * p.tw;
    if (elems == 0) return TD_OK;
    if (vec) {
        const int twv = p.tw / Vec<T>::kElems;
        const int rows_per_block = std::max(1, std::min(p.th, (128 * 4 + twv - 1) / twv));   // ~4 vectors per thread
        dim3 grid((unsigned)(n_tiles * p.N * p.C), (unsigned)((p.th + rows_per_block - 1) / rows_per_block));
        return launch("td_scatter_tiles (wrap)", wrap_scatter_vec_kernel<T>, grid, dim3(128), 0, st, pdl, p, (const T*)x, (T*)tiles, tile_begin,
                      rows_per_block);
    }
    return launch("td_scatter_tiles (wrap)", wrap_scatter_generic_kernel<T>, dim3(blocks_for(elems, 256)), dim3(256), 0, st, pdl, p, (const T*)x,
                  (T*)tiles, tile_begin, elems);
}

// `win` null: the whole canvas; else its row window (rb_count > 0)
template <typename T, int MODE>
int blend_vec_impl(const WrapParams& p, const float* weights, const float* tile_weights, const float* rescale, float* out_f32,
                   void* out_buf, const WindowParams* win, bool pdl, cudaStream_t st) {
    const int wv = p.W / Vec<T>::kElems;
    const unsigned gx = (unsigned)((wv + kWrapBX - 1) / kWrapBX), planes = (unsigned)(p.N * p.C);
    const dim3 grid = win ? dim3(gx, planes, (unsigned)win->rb_count) : dim3(gx, (unsigned)((p.H + kWrapBY - 1) / kWrapBY), planes);
    if (grid.y > 65535u || grid.z > 65535u) { td_set_error("canvas too large for the wrap blend grid"); return TD_ERR_UNSUPPORTED; }
    const dim3 block(kWrapBX, kWrapBY);
    const bool buf = MODE == MODE_MOD || out_buf != nullptr;
    if (win) {
        auto kernel = buf ? wrap_blend_vec_kernel<T, MODE, true, true> : wrap_blend_vec_kernel<T, MODE, false, true>;
        return launch("td_blend (wrap, rows)", kernel, grid, block, 0, st, pdl, p, weights, tile_weights, rescale, out_f32, (T*)out_buf, *win);
    }
    const WindowParams whole = {};
    auto kernel = buf ? wrap_blend_vec_kernel<T, MODE, true, false> : wrap_blend_vec_kernel<T, MODE, false, false>;
    return launch("td_blend (wrap)", kernel, grid, block, 0, st, pdl, p, weights, tile_weights, rescale, out_f32, (T*)out_buf, whole);
}

// Does canvas row y lie in a tile row outside the own bands?  (host twin of the kernel's per-CTA wait test)
bool row_leaves_own(const WrapParams& p, int y, int own_lo, int own_hi) {
    for (int i = 0; i < p.rows; ++i) {
        if (i >= own_lo && i < own_hi) continue;
        int v = y - p.ys[i];
        if (v < 0 && p.wrap_y) v += p.H;
        if (v >= 0 && v < p.th) return true;
    }
    return false;
}

// Row-strip shard: the waiting CTAs run last.  The halo enters a strip from its top (a lower rank's bands, or across the
// seam the last bands of a wrapped canvas), so the window is normally walked from its end; the other way round when the
// waiting rows sit at its end.
int window_descending(const WrapParams& p, const WindowParams& w) {
    if (w.wait_count == 0 || w.own_hi <= w.own_lo) return 0;
    int first = -1, last = -1;
    for (int b = 0; b < w.rb_count; ++b) {
        const int y0 = w.row_begin + b * kWrapBY, y1 = std::min(y0 + kWrapBY, w.row_end);
        bool waits = false;
        for (int y = y0; y < y1 && !waits; ++y) waits = row_leaves_own(p, y, w.own_lo, w.own_hi);
        if (waits) { if (first < 0) first = b; last = b; }
    }
    return (first >= 0 && first + last <= w.rb_count - 1) ? 1 : 0;
}

template <int MODE>
int blend_generic_impl(int tile_dtype, int acc_dtype, const WrapParams& p, const float* w, const float* tw, const float* rs, float* out_f32,
                       void* out_buf, bool pdl, cudaStream_t st) {
    const long long total = (long long)p.N * p.C * p.H * p.W;
    const dim3 grid(blocks_for(total, 256));
#define TD_CASE(TI, TA, TIn, TAcc)                                                                                         \
    if (tile_dtype == TI && acc_dtype == TA)                                                                               \
        return launch("td_blend (wrap, generic)", wrap_blend_generic_kernel<TIn, TAcc, MODE>, grid, dim3(256), 0, st, pdl, p, w, tw, rs, \
                      out_f32, (TAcc*)out_buf, total);
    TD_CASE(TD_F16, TD_F16, __half, __half)
    TD_CASE(TD_F16, TD_BF16, __half, __nv_bfloat16)
    TD_CASE(TD_F16, TD_F32, __half, float)
    TD_CASE(TD_BF16, TD_F16, __nv_bfloat16, __half)
    TD_CASE(TD_BF16, TD_BF16, __nv_bfloat16, __nv_bfloat16)
    TD_CASE(TD_BF16, TD_F32, __nv_bfloat16, float)
    TD_CASE(TD_F32, TD_F16, float, __half)
    TD_CASE(TD_F32, TD_BF16, float, __nv_bfloat16)
    TD_CASE(TD_F32, TD_F32, float, float)
#undef TD_CASE
    td_set_error("unknown dtype pair (%d, %d)", tile_dtype, acc_dtype);
    return TD_ERR_INVALID_ARG;
}

int blend_vec_dispatch(const WrapParams& p, int tile_dtype, int mixture, const float* weights, const float* tile_weights, const float* rescale,
                       float* x_out, void* x_buffer, const WindowParams* win, bool pdl, cudaStream_t st) {
    if (mixture) {
        switch (tile_dtype) {
            case TD_F16: return blend_vec_impl<__half, MODE_MOD>(p, nullptr, tile_weights, rescale, nullptr, x_buffer, win, pdl, st);
            case TD_BF16: return blend_vec_impl<__nv_bfloat16, MODE_MOD>(p, nullptr, tile_weights, rescale, nullptr, x_buffer, win, pdl, st);
            default: return blend_vec_impl<float, MODE_MOD>(p, nullptr, tile_weights, rescale, nullptr, x_buffer, win, pdl, st);
        }
    }
    switch (tile_dtype) {
        case TD_F16: return blend_vec_impl<__half, MODE_MD>(p, weights, nullptr, nullptr, x_out, x_buffer, win, pdl, st);
        case TD_BF16: return blend_vec_impl<__nv_bfloat16, MODE_MD>(p, weights, nullptr, nullptr, x_out, x_buffer, win, pdl, st);
        default: return blend_vec_impl<float, MODE_MD>(p, weights, nullptr, nullptr, x_out, x_buffer, win, pdl, st);
    }
}

}  // namespace

int td_wrap_scatter(const td_grid* g, const void* x, void* tiles, int N, int C, int dtype, int tile_begin, int tile_end, bool vec, bool pdl,
                    void* stream) {
    WrapParams p;
    fill_params(g, N, C, &p);
    cudaStream_t st = (cudaStream_t)stream;
    if (td_dtype_size(dtype) == 2) return scatter_impl<__half>(p, x, tiles, tile_begin, tile_end - tile_begin, vec, pdl, st);   // 16-bit words, opaque
    return scatter_impl<float>(p, x, tiles, tile_begin, tile_end - tile_begin, vec, pdl, st);
}

int td_wrap_blend(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int tile_dtype, int acc_dtype,
                  int mixture, const float* weights, const float* tile_weights, const float* rescale, float* x_out, void* x_buffer,
                  bool vec, bool pdl, void* stream) {
    WrapParams p;
    fill_params(g, N, C, &p);
    p.tile_bs = tile_bs;
    for (int b = 0; b < num_batches; ++b) p.batch_ptrs[b] = batch_ptrs[b];
    cudaStream_t st = (cudaStream_t)stream;
    if (vec) return blend_vec_dispatch(p, tile_dtype, mixture, weights, tile_weights, rescale, x_out, x_buffer, nullptr, pdl, st);
    if (mixture) return blend_generic_impl<MODE_MOD>(tile_dtype, acc_dtype, p, nullptr, tile_weights, rescale, nullptr, x_buffer, pdl, st);
    return blend_generic_impl<MODE_MD>(tile_dtype, acc_dtype, p, weights, nullptr, nullptr, x_out, x_buffer, pdl, st);
}

int td_wrap_blend_rows(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int tile_dtype,
                       int mixture, const float* weights, const float* tile_weights, const float* rescale, float* x_out, void* x_buffer,
                       int row_begin, int row_end, const uint32_t* wait_flags, int wait_count, const uint32_t* wait_value,
                       int own_band_begin, int own_band_end, bool pdl, void* stream) {
    WrapParams p;
    fill_params(g, N, C, &p);
    p.tile_bs = tile_bs;
    for (int b = 0; b < num_batches; ++b) p.batch_ptrs[b] = batch_ptrs[b];
    WindowParams w;
    w.row_begin = row_begin;
    w.row_end = row_end;
    w.rb_count = (row_end - row_begin + kWrapBY - 1) / kWrapBY;
    w.wait_count = wait_flags != nullptr ? wait_count : 0;
    w.wait_flags = wait_flags;
    w.wait_value = wait_value;
    w.own_lo = w.wait_count > 0 ? own_band_begin : 0;   // no wait: the own-band test is never made
    w.own_hi = w.wait_count > 0 ? own_band_end : 0;
    w.descending = window_descending(p, w);
    return blend_vec_dispatch(p, tile_dtype, mixture, weights, tile_weights, rescale, x_out, x_buffer, &w, pdl, (cudaStream_t)stream);
}
