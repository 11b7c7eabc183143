// Per-sampler-step hot path of tiled diffusion on sm_90a:
//   scatter  (crop-with-overlap of the latent into the tile batch)      multidiffusion.py:155
//   blend    (ordered overlap accumulate + normalise, gather form)      multidiffusion.py:166-167,208
//            (gaussian-weighted, pre-normalised accumulate)             mixtureofdiffusers.py:122-126
//
// Design (H100-first, see DESIGN.md):
//   * ONE launch per step for all T tiles (the reference: T/TB cats + T..3T slice-adds).
//   * Gather form: each thread owns one 16-byte vector of the output canvas and
//     visits the tiles covering it in ascending tile index, rounding through the
//     canvas dtype after every add -> bit-identical to the reference's in-place
//     `x_buffer[slicer] += tile` sequence, with no atomics and no RMW traffic.
//   * Tile x-origins are arbitrary (46, 92, 231, ...), so tile rows and canvas rows
//     are mutually misaligned.  Every access is still a 128-bit aligned load: a
//     thread reads the two aligned 16-byte chunks that straddle its window and
//     extracts it with funnel shifts; the shift is uniform per tile column.
//   * Grid geometry (<= 256 row + 256 col origins) and the UNet's per-batch output
//     pointers travel in the kernel parameter block: no device tables, no H2D.
//   * All memory-bound: no tensor cores here on purpose.
//   * Defaults on H100 (DESIGN.md 4.4): the scatter is the row-block form of td_rows.cu
//     (scatter_vec_kernel where it does not apply, or with TD_FLAG_NO_TMA), both launched
//     with PDL; the MultiDiffusion blend is blend_md_async_kernel with one plane per CTA.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <mutex>
#include <vector>

#include "td_b200.h"
#include "td_device.cuh"
#include "td_internal.h"
#include "td_launch.h"
#include "td_tma.cuh"

namespace {

using namespace td;

struct GeomParams {
    int H, W, th, tw, rows, cols, N, C;
    float inv_dx, inv_dy;  // 1/stride estimates for the origin search (any value is safe)
    unsigned nc_magic, twv_magic;  // fast division by N*C and by tw/VEC (operands < 2^16)
    int dbg_no_tiles;              // TD_FLAG_DBG_NO_TILES: skip every tile visit (measures the launch + epilogue floor)
    short ys[TD_MAX_GRID_DIM];
    short xs[TD_MAX_GRID_DIM];
};

struct BlendParams {
    GeomParams g;
    int tile_bs, num_batches;
    unsigned bs_magic;  // fast division by tile_bs
    // cp.async kernel: tiles touching patch row / patch col i (first index, count), computed on the host
    unsigned char prow_lo[TD_MAX_GRID_DIM], prow_n[TD_MAX_GRID_DIM];
    unsigned char pcol_lo[TD_MAX_GRID_DIM], pcol_n[TD_MAX_GRID_DIM];
    const uint32_t* wait_flags;  // tile shard: spin until wait_flags[i] >= *wait_value for i < wait_world
    int wait_world;
    const uint32_t* wait_value;  // this rank's device-side step counter (bumped by td_peer_signal)
    int py0, py_count;      // cp.async kernels: first patch row and patch-row count of this launch (row-range blend; 0, 0 = all)
    int own_r_lo, own_r_hi; // row-strip shard: tile rows [lo, hi) are this rank's own outputs -- a CTA whose visits stay inside them
                            // skips the peer wait (lo == hi: every CTA waits)
    int sched;              // 0: blockIdx.y = patch row, .z = plane group; 1 / 2: blockIdx.z = patch row ascending / descending
                            // (slowest-varying), so that the CTAs that must wait for a neighbour's halo are scheduled last
    long long tile_stride;  // N*C*th*tw elements
    const void* batch_ptrs[TD_MAX_BATCH_PTRS];
};

enum { MODE_MD = 0, MODE_MOD = 1 };

__device__ __forceinline__ void load_origins(const GeomParams& g, short* s_ys, short* s_xs) {
    for (int i = threadIdx.x; i < g.rows; i += blockDim.x) s_ys[i] = g.ys[i];
    for (int i = threadIdx.x; i < g.cols; i += blockDim.x) s_xs[i] = g.xs[i];
    __syncthreads();
}

// ---------------------------------------------------------------------------
// Scatter, vector path (the default).  One block = `rows_per_block` rows of one (tile, n, c)
// plane; tile origin and the funnel shift are block-uniform.  Each thread moves
// 16-byte vectors: two aligned 128-bit loads of the (misaligned) canvas row,
// one aligned 128-bit store into the tile batch; 4 vectors in flight per thread.
// Launched with PDL.  A TMA-staged form (aligned-superset boxes through shared memory,
// re-aligned by the threads) measured slower (DESIGN.md 4.4).  A pure bulk copy -- a
// tensor-map box loaded at the tile's exact origin, stored back with cp.async.bulk -- does
// not apply at cfg2: its origins (0, 46, 92, ...) are not 16-byte aligned, and a box whose
// innermost start is not 16-byte aligned faults with an illegal instruction (td_tma.cuh).
// ---------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(128)
scatter_vec_kernel(const __grid_constant__ GeomParams g, const T* __restrict__ x, T* __restrict__ tiles,
                   int tile_begin, int rows_per_block) {
    constexpr int VEC = Vec<T>::kElems;
    constexpr int L2V = Vec<T>::kLog2;
    constexpr int UNROLL = 4;
    const unsigned tp = blockIdx.x;                       // (tile local, n, c) plane of the tile batch
    const unsigned tl = fastdiv(tp, g.nc_magic);
    const int plane = (int)(tp - tl * (unsigned)(g.N * g.C));
    const int t = tile_begin + (int)tl;
    const int r = t / g.cols, c = t - r * g.cols;
    const int xs = (int)g.xs[c], ys = (int)g.ys[r];
    const int twv = g.tw >> L2V;
    const int v0 = blockIdx.y * rows_per_block;
    const int nvec = min(rows_per_block, g.th - v0) * twv;
    const int s = xs & (VEC - 1), k0 = xs >> L2V;         // block-uniform shift
    const T* src = x + ((long long)plane * g.H + ys + v0) * g.W;
    T* dst = tiles + ((long long)tp * g.th + v0) * g.tw;
    pdl_launch_dependents();
    pdl_wait();   // x is read and tiles are written only after the previous kernel in the stream has completed
    for (int base = threadIdx.x; base < nvec; base += 128 * UNROLL) {
        uint4 A[UNROLL], B[UNROLL];
#pragma unroll
        for (int q = 0; q < UNROLL; ++q) {
            const int i = base + q * 128;
            A[q] = B[q] = make_uint4(0, 0, 0, 0);
            if (i < nvec) {
                const unsigned vi = fastdiv((unsigned)i, g.twv_magic);
                const int uv = i - (int)vi * twv;
                const T* row = src + (long long)vi * g.W + (long long)(k0 + uv) * VEC;
                A[q] = ldg128(row);
                if (s != 0) B[q] = ldg128(row + VEC);   // in-bounds: holds element xs+uv*VEC+VEC-1 < W, W % VEC == 0
            }
        }
#pragma unroll
        for (int q = 0; q < UNROLL; ++q) {
            const int i = base + q * 128;
            if (i < nvec) stg128(dst + (long long)i * VEC, Vec<T>::window(A[q], B[q], s));
        }
    }
}

// Scatter, generic path: any width / alignment, one element per thread.
template <typename T>
__global__ void __launch_bounds__(256)
scatter_generic_kernel(const __grid_constant__ GeomParams g, const T* __restrict__ x, T* __restrict__ tiles,
                       int tile_begin, long long total) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    long long rem = idx;
    const int u = (int)(rem % g.tw); rem /= g.tw;
    const int v = (int)(rem % g.th); rem /= g.th;
    const int plane = (int)(rem % (g.N * g.C)); rem /= (g.N * g.C);
    const int t = tile_begin + (int)rem;
    const int r = t / g.cols, c = t - r * g.cols;
    tiles[idx] = x[((long long)plane * g.H + (int)g.ys[r] + v) * g.W + (int)g.xs[c] + u];
}

// ---------------------------------------------------------------------------
// Blend, vector path.
//
// Work decomposition: a warp owns an 8-vector x 8-row patch of one canvas plane
// (lane = 8 vectors x 4 rows, 2 rows per thread); a block is 4 warps stacked in y.
// The covering tile rows / cols are computed once per warp (uniform loops); a lane
// takes part in a tile visit through predicated loads only.  Out-of-tile chunks are
// never loaded and read as -0.0, the exact additive identity (x + -0.0 == x for
// every x, signed zeros included), and because tw % VEC == 0 chunk validity IS
// element validity -- so the MultiDiffusion path needs no per-element masks and
// accumulates with packed HADD2: round_half(a + b) of the exact sum, which equals
// torch's half(float(a) + float(b)) (fp32 has >= 2p+2 bits: double rounding is innocuous).
// ---------------------------------------------------------------------------

constexpr int kBlendWarps = 2;       // warps per block, stacked in y
constexpr int kWarpVecs = 8;         // vectors per warp row (lane = 8 vectors x 4 rows)
constexpr int kGroup = 2;            // tile visits whose loads are in flight together

template <int MODE> struct BlendShape { static constexpr int kRPT = (MODE == 0) ? 4 : 2; };  // rows per thread

template <typename T, int MODE, bool WRITE_BUF>
__global__ void __launch_bounds__(kBlendWarps * 32)
blend_grid_vec_kernel(const __grid_constant__ BlendParams p, const float* __restrict__ weights,
                      const float* __restrict__ tile_weights, const float* __restrict__ rescale,
                      float* __restrict__ out_f32, T* __restrict__ out_buf) {
    constexpr int VEC = Vec<T>::kElems;
    constexpr int L2V = Vec<T>::kLog2;
    constexpr int RPT = BlendShape<MODE>::kRPT;
    constexpr int WROWS = 4 * RPT;                 // rows per warp patch
    constexpr uint32_t NEG0 = sizeof(T) == 2 ? 0x80008000u : 0x80000000u;
    __shared__ short s_ys[TD_MAX_GRID_DIM];
    __shared__ short s_xs[TD_MAX_GRID_DIM];
    const GeomParams& g = p.g;
    if (p.wait_flags != nullptr) {   // tile shard: peers' tile outputs must be complete before they are read
        if ((int)threadIdx.x < p.wait_world) spin_until_ge(p.wait_flags + threadIdx.x, *p.wait_value);
    }
    load_origins(g, s_ys, s_xs);   // (contains the __syncthreads that publishes the wait)

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int lx = lane & 7, ly = lane >> 3;
    const int plane = blockIdx.z;
    const int wv = g.W >> L2V;
    const int xv0 = blockIdx.x * kWarpVecs;                           // warp's first vector
    const int yw = (blockIdx.y * kBlendWarps + warp) * WROWS;         // warp's first row
    if (yw >= g.H) return;                                            // warp-uniform
    const int x_lo = xv0 * VEC, x_hi = min(x_lo + kWarpVecs * VEC, g.W) - 1;
    const int y_hi = min(yw + WROWS, g.H) - 1;

    // tiles touching this warp's patch (uniform across the warp)
    const int r_lo = last_le(s_ys, g.rows, yw - g.th, g.inv_dy) + 1;
    const int r_hi = last_le(s_ys, g.rows, y_hi, g.inv_dy);
    const int c_lo = last_le(s_xs, g.cols, x_lo - g.tw, g.inv_dx) + 1;
    const int c_hi = last_le(s_xs, g.cols, x_hi, g.inv_dx);
    const int nc = c_hi - c_lo + 1;
    const int nv = g.dbg_no_tiles ? 0 : (r_hi - r_lo + 1) * nc;       // visits, in ascending tile index

    const int xv = xv0 + lx;
    const bool x_ok = xv < wv;
    const int x0 = xv * VEC;
    int y[RPT];
    bool y_ok[RPT];
#pragma unroll
    for (int q = 0; q < RPT; ++q) { y[q] = yw + ly + 4 * q; y_ok[q] = x_ok && y[q] < g.H; }

    constexpr bool kPacked = (MODE == MODE_MD);   // accumulate directly in T (packed words)
    uint4 pacc[RPT];
    float facc[RPT][kPacked ? 1 : VEC];
    float rs[RPT][kPacked ? 1 : VEC];
#pragma unroll
    for (int q = 0; q < RPT; ++q) {
        pacc[q] = make_uint4(0, 0, 0, 0);
        if constexpr (!kPacked) {
#pragma unroll
            for (int j = 0; j < VEC; ++j) { facc[q][j] = 0.0f; rs[q][j] = 0.0f; }
            if (y_ok[q]) {
                const float4* rp = reinterpret_cast<const float4*>(rescale + (long long)y[q] * g.W + x0);
#pragma unroll
                for (int h = 0; h < VEC / 4; ++h) {
                    const float4 f = __ldg(rp + h);
                    rs[q][4 * h + 0] = f.x; rs[q][4 * h + 1] = f.y; rs[q][4 * h + 2] = f.z; rs[q][4 * h + 3] = f.w;
                }
            }
        }
    }

    const int twv = g.tw >> L2V;
    const int plane_off = plane * g.th * g.tw;     // < 2^31: checked on the host
    int r_cur = r_lo, c_cur = c_lo;
    for (int i0 = 0; i0 < nv; i0 += kGroup) {
        uint4 A[kGroup][RPT], B[kGroup][RPT];
        int sft[kGroup], u0s[kGroup], vrow[kGroup][RPT];
        bool live[kGroup][RPT];
        // ---- phase 1: issue every load of the group -----------------------------------------
#pragma unroll
        for (int gi = 0; gi < kGroup; ++gi) {
            const bool in = i0 + gi < nv;
            const int r = in ? r_cur : r_lo, c = in ? c_cur : c_lo;
            if (in) { if (++c_cur > c_hi) { c_cur = c_lo; ++r_cur; } }
            const unsigned t = (unsigned)(r * g.cols + c);
            const unsigned b = fastdiv(t, p.bs_magic);
            const T* tbase = reinterpret_cast<const T*>(p.batch_ptrs[b]) + (long long)(t - b * (unsigned)p.tile_bs) * p.tile_stride;
            const int ysr = (int)s_ys[r];
            const int u0 = x0 - (int)s_xs[c];      // tile-local column of element 0; u0 & (VEC-1) is warp-uniform
            const int k = u0 >> L2V, s = u0 & (VEC - 1);
            sft[gi] = s; u0s[gi] = u0;
            const bool okA = in && (unsigned)k < (unsigned)twv;
            const bool okB = in && s != 0 && (unsigned)(k + 1) < (unsigned)twv;
#pragma unroll
            for (int q = 0; q < RPT; ++q) {
                const int v = y[q] - ysr;
                const bool rok = y_ok[q] && (unsigned)v < (unsigned)g.th;
                vrow[gi][q] = v; live[gi][q] = rok && in;
                A[gi][q] = make_uint4(NEG0, NEG0, NEG0, NEG0);
                B[gi][q] = A[gi][q];
                const T* trow = tbase + (plane_off + v * g.tw + k * VEC);
                if (rok && okA) A[gi][q] = ldg128(trow);
                if (rok && okB) B[gi][q] = ldg128(trow + VEC);
            }
        }
        // ---- phase 2: consume in tile order ---------------------------------------------------
#pragma unroll
        for (int gi = 0; gi < kGroup; ++gi) {
#pragma unroll
            for (int q = 0; q < RPT; ++q) {
                const uint4 e = Vec<T>::window(A[gi][q], B[gi][q], sft[gi]);
                if constexpr (kPacked) {
                    pacc[q].x = packed_add<T>(pacc[q].x, e.x);
                    pacc[q].y = packed_add<T>(pacc[q].y, e.y);
                    pacc[q].z = packed_add<T>(pacc[q].z, e.z);
                    pacc[q].w = packed_add<T>(pacc[q].w, e.w);
                } else {
#pragma unroll
                    for (int j = 0; j < VEC; ++j) {
                        const int u = u0s[gi] + j;
                        const bool valid = live[gi][q] && (unsigned)u < (unsigned)g.tw;
                        // w = tile_weights * rescale_factor[slicer]; x_tile_out * w   (two fp32 roundings, no FMA)
                        const float tw_ = valid ? __ldg(tile_weights + vrow[gi][q] * g.tw + u) : 0.0f;
                        const float val = __fmul_rn(Vec<T>::get(e, j), __fmul_rn(tw_, rs[q][j]));
                        const float sum = round_through<T>(__fadd_rn(facc[q][j], val));
                        facc[q][j] = valid ? sum : facc[q][j];
                    }
                }
            }
        }
    }

#pragma unroll
    for (int q = 0; q < RPT; ++q) {
        if (!y_ok[q]) continue;
        const long long o = ((long long)plane * g.H + y[q]) * g.W + x0;
        float acc[VEC];
        if constexpr (kPacked) {
#pragma unroll
            for (int j = 0; j < VEC; ++j) acc[j] = Vec<T>::get(pacc[q], j);
        } else {
#pragma unroll
            for (int j = 0; j < VEC; ++j) acc[j] = facc[q][j];
        }
        if constexpr (MODE == MODE_MD) {
            // x_out = where(weights > 1, x_buffer / weights, x_buffer)  -- fp32, IEEE divide
            const float4* wp = reinterpret_cast<const float4*>(weights + (long long)y[q] * g.W + x0);
            float4* op = reinterpret_cast<float4*>(out_f32 + o);
#pragma unroll
            for (int h = 0; h < VEC / 4; ++h) {
                const float4 w = __ldg(wp + h);
                float4 f;
                f.x = w.x > 1.0f ? __fdiv_rn(acc[4 * h + 0], w.x) : acc[4 * h + 0];
                f.y = w.y > 1.0f ? __fdiv_rn(acc[4 * h + 1], w.y) : acc[4 * h + 1];
                f.z = w.z > 1.0f ? __fdiv_rn(acc[4 * h + 2], w.z) : acc[4 * h + 2];
                f.w = w.w > 1.0f ? __fdiv_rn(acc[4 * h + 3], w.w) : acc[4 * h + 3];
                op[h] = f;
            }
        }
        if constexpr (WRITE_BUF || MODE == MODE_MOD) {
            uint4 pk;
            if constexpr (kPacked) {
                pk = pacc[q];
            } else if constexpr (sizeof(T) == 2) {
                uint32_t w32[4];
#pragma unroll
                for (int h = 0; h < 4; ++h)
                    w32[h] = (uint32_t)Elem<T>::f32_to_bits(acc[2 * h]) | ((uint32_t)Elem<T>::f32_to_bits(acc[2 * h + 1]) << 16);
                pk = make_uint4(w32[0], w32[1], w32[2], w32[3]);
            } else {
                pk = make_uint4(__float_as_uint(acc[0]), __float_as_uint(acc[1]), __float_as_uint(acc[2]), __float_as_uint(acc[3]));
            }
            stg128(out_buf + o, pk);
        }
    }
}

// ---------------------------------------------------------------------------
// Blend + normalise, MultiDiffusion, cp.async path (the default when it applies).
//
// A CTA owns a 8-row x 8-vector (TD_AS_ROWS) patch of one canvas plane.  For every tile touching the
// patch (ascending tile index) the threads copy the aligned superset of the intersection
// (9 chunks x 8 rows) global -> shared with 16-byte cp.async; chunks outside the tile
// use src-size 0, i.e. the copy itself zero-fills them (exact: the accumulator starts at
// +0 and can never become -0).  Every copy of the CTA is in flight before the first wait:
// memory-level parallelism without staging registers and without the per-box cost of TMA.
// The consume loop is specialised on the per-tile shift s (uniform over the CTA): two
// LDS.128, at most four funnel shifts with an immediate, four packed adds.
// With integer weights (MultiDiffusion's always are) and their correctly rounded
// reciprocals supplied, the IEEE divide is q = a*rcp; r = fma(-q, w, a); q' = fma(r, rcp, q)
// -- correctly rounded for every 16-bit numerator and w <= 4096 (checked exhaustively by
// td_debug_check_fast_div / tests).
// ---------------------------------------------------------------------------
#ifndef TD_AS_X
#define TD_AS_X 8                                // tuning knob (-DTD_AS_X=): vectors per patch row
#endif
constexpr int kAsX = TD_AS_X;                    // vectors per patch row
#ifndef TD_AS_ROWS
#define TD_AS_ROWS 8                             // tuning knob (-DTD_AS_ROWS=): 8 / 16 / 32 measured 8.89 / 9.18 / 10.7 us (cfg2), 8 kept
#endif
constexpr int kAsY = TD_AS_ROWS;                 // patch rows
constexpr int kAsVecThreads = kAsX * kAsY;       // 64 threads own one output vector each
constexpr int kAsChunks = kAsX + 1;              // staged chunks per row (aligned superset)
constexpr int kAsSlots = kAsY * kAsChunks;       // 72 copy slots per tile visit: one per thread
constexpr int kAsThreads = (kAsSlots + 31) / 32 * 32;   // 96 = 3 warps: 72 copy threads
constexpr int kAsStage = kAsSlots * 16;          // 1152 bytes per tile visit

// 16-byte copy that writes zeros instead (no global access) when `neg_if_skip` is negative
__device__ __forceinline__ void cp_async16_zfill(uint32_t smem_dst, long long gmem_src, int neg_if_skip) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.lt.s32 p, %2, 0;\n\t"
        "cp.async.cg.shared.global [%0], [%1], 16, p;\n\t}"
        ::"r"(smem_dst), "l"(gmem_src), "r"(neg_if_skip)
        : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
    asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}

template <typename T, int S>
__device__ __forceinline__ void consume_shifted(uint4& acc, const unsigned char* p) {
    const uint4 A = lds128(p);
    uint4 e;
    if constexpr (S == 0) {
        e = A;
    } else {
        const uint4 B = lds128(p + 16);
        e = Vec<T>::window(A, B, S);    // S is a compile-time constant: register selection / immediate shifts only
    }
    acc.x = packed_add<T>(acc.x, e.x);
    acc.y = packed_add<T>(acc.y, e.y);
    acc.z = packed_add<T>(acc.z, e.z);
    acc.w = packed_add<T>(acc.w, e.w);
}

struct __align__(16) VisitEntry {   // per tile visit of a CTA, computed once by one thread
    long long origin;               // byte address of tile element (v0, k0*VEC) of this plane (may lie before the tile)
    int v0, k0;                     // tile row / tile chunk of the patch origin (may be negative)
};
constexpr int kAsMaxVisits = 64;

// Row-strip shard, cp.async blends: the peers' tile outputs must be complete before any copy of this CTA reads them.  Only
// CTAs whose visits leave the own bands [own_r_lo, own_r_hi) wait (all of them when the range is empty); the last warp spins
// and the CTA's next barrier publishes the wait to the other threads.
__device__ __forceinline__ void halo_wait(const BlendParams& p, int by, int r_lo, int tid) {
    const bool reads_halo = r_lo < p.own_r_lo || r_lo + (int)p.prow_n[by] > p.own_r_hi;   // always true when own_r_lo == own_r_hi
    if (p.wait_flags != nullptr && reads_halo && tid >= kAsThreads - 32 && tid - (kAsThreads - 32) < p.wait_world)
        spin_until_ge(p.wait_flags + (tid - (kAsThreads - 32)), *p.wait_value);
}

// Patch row and plane group of a cp.async blend CTA: sched 0 walks blockIdx.y = patch row, .z = plane group; sched 1 / 2 put
// the patch row on blockIdx.z (slowest-varying), ascending / descending from the window's start py0.
__device__ __forceinline__ int window_row_index(const BlendParams& p) {
    return p.sched == 0 ? (int)blockIdx.y : (p.sched == 2 ? p.py_count - 1 - (int)blockIdx.z : (int)blockIdx.z);
}
__device__ __forceinline__ int plane_group_index(const BlendParams& p) { return p.sched == 0 ? (int)blockIdx.z : (int)blockIdx.y; }

// Sparse blends (td_blend_*_sparse): the visit table of a cp.async CTA with the skipped tiles (slot[t] < 0) dropped and the others
// kept in tile order, compacted with one ballot per warp.  Tile t lives at position slot[t] of the compact batches.  Every thread of
// the CTA calls this (it contains the barrier that publishes the table); returns the number of visits kept.
template <typename T>
__device__ __forceinline__ int prepare_sparse_visits(const BlendParams& p, const int* __restrict__ slot, int nv, int r_lo, int c_lo,
                                                     int nc, int x_lo, int y_lo, long long plane_elems, VisitEntry* s_visit,
                                                     int* s_shift) {
    constexpr int L2V = Vec<T>::kLog2;
    constexpr int VEC = Vec<T>::kElems;
    __shared__ int s_kept[kAsThreads / 32];
    const GeomParams& g = p.g;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int r = 0, c = 0, sl = -1;
    if (tid < nv) {
        const int ri = tid / nc;
        r = r_lo + ri;
        c = c_lo + (tid - ri * nc);
        sl = __ldg(slot + r * g.cols + c);
    }
    const unsigned kept = __ballot_sync(0xffffffffu, sl >= 0);
    if (lane == 0) s_kept[warp] = __popc(kept);
    __syncthreads();
    int pos = __popc(kept & ((1u << lane) - 1u)), total = 0;
#pragma unroll
    for (int w = 0; w < kAsThreads / 32; ++w) {
        pos += w < warp ? s_kept[w] : 0;
        total += s_kept[w];
    }
    if (sl >= 0) {
        const unsigned b = fastdiv((unsigned)sl, p.bs_magic);
        const int u0 = x_lo - (int)g.xs[c];
        const int v0 = y_lo - (int)g.ys[r], k0 = u0 >> L2V;
        const long long elem = (long long)((unsigned)sl - b * (unsigned)p.tile_bs) * p.tile_stride + plane_elems +
                               (long long)v0 * g.tw + (long long)k0 * VEC;
        VisitEntry e;
        e.origin = (long long)reinterpret_cast<uintptr_t>(p.batch_ptrs[b]) + elem * (long long)sizeof(T);
        e.v0 = v0;
        e.k0 = k0;
        s_visit[pos] = e;
        s_shift[pos] = u0 & (VEC - 1);
    }
    __syncthreads();
    return total;
}

template <typename T, int S, int PPC>
__device__ __forceinline__ void consume_planes(uint4 (&acc)[PPC], const unsigned char* p) {
#pragma unroll
    for (int q = 0; q < PPC; ++q) consume_shifted<T, S>(acc[q], p + q * kAsStage);
}

// PPC = planes per CTA: the (n, c) planes of a patch share the visit table, the zero-fill predicate, the weights
// and the shift, so a CTA that blends PPC planes amortises its prologue and runs PPC independent add chains.
// SPARSE (td_blend_multidiffusion_sparse, PPC 1): `slot` maps tile t to its position in the compact batches, or -1 to drop its
// visits; without it the parameter is not read and the kernel's instruction stream is the dense one.
template <typename T, bool WRITE_BUF, bool FASTDIV, int PPC, bool SPARSE = false>
__global__ void __launch_bounds__(kAsThreads)
blend_md_async_kernel(const __grid_constant__ BlendParams p, const float* __restrict__ weights, const float* __restrict__ rcp_weights,
                      float* __restrict__ out_f32, T* __restrict__ out_buf, const int* __restrict__ slot) {
    constexpr int VEC = Vec<T>::kElems;
    constexpr int L2V = Vec<T>::kLog2;
    constexpr int BX = kAsX * VEC;
    extern __shared__ __align__(16) unsigned char td_smem[];
    __shared__ VisitEntry s_visit[kAsMaxVisits];
    __shared__ int s_shift[kAsMaxVisits];
    const GeomParams& g = p.g;
    const int tid = threadIdx.x;
    const int zy = window_row_index(p);
    const int plane = plane_group_index(p) * PPC;   // first plane of this CTA (PPC divides N*C)
    const int by = zy + p.py0;                // patch row (a row-range launch starts at py0)
    const int x_lo = blockIdx.x * BX, y_lo = by * kAsY;
    pdl_launch_dependents();

    // tiles touching this patch: host-computed per patch row / col (uniform constant-bank reads)
    const int r_lo = p.prow_lo[by], c_lo = p.pcol_lo[blockIdx.x];
    const int nc = p.pcol_n[blockIdx.x];
    int nv = g.dbg_no_tiles ? 0 : (int)p.prow_n[by] * nc;   // <= the host's stage count

    // this thread's output vector; its weights are fetched now so that their latency hides behind the tile copies
    const int tx = tid % kAsX, ty = tid / kAsX;
    const int x0 = x_lo + tx * VEC, y = y_lo + ty;
    const bool inside = tid < kAsVecThreads && x0 < g.W && y < g.H;
    const long long wo = (long long)y * g.W + x0;
    float4 wv[VEC / 4], rv[VEC / 4];
    pdl_wait();
#pragma unroll
    for (int h = 0; h < VEC / 4; ++h) {
        wv[h] = inside ? __ldg(reinterpret_cast<const float4*>(weights + wo) + h) : make_float4(1.f, 1.f, 1.f, 1.f);
        if constexpr (FASTDIV) rv[h] = inside ? __ldg(reinterpret_cast<const float4*>(rcp_weights + wo) + h) : make_float4(1.f, 1.f, 1.f, 1.f);
    }

    // halo_wait's test, written out here: calling halo_wait itself changes how the compiler schedules this kernel's prologue
    // (cfg2 blend measured about 0.5% slower on an H100 80GB HBM3 at 700 W).  The spin alone through spin_until_ge leaves the
    // instruction stream as it was with the loop written out (only register numbers differ).
    const bool reads_halo = r_lo < p.own_r_lo || r_lo + (int)p.prow_n[by] > p.own_r_hi;   // always true when own_r_lo == own_r_hi
    if (p.wait_flags != nullptr && reads_halo && tid >= kAsThreads - 32 && tid - (kAsThreads - 32) < p.wait_world)
        spin_until_ge(p.wait_flags + (tid - (kAsThreads - 32)), *p.wait_value);

    // ---- per-visit constants: thread i prepares visit i -------------------------------------------------
    const long long plane_bytes = (long long)g.th * g.tw * (long long)sizeof(T);
    if constexpr (SPARSE) {
        nv = prepare_sparse_visits<T>(p, slot, nv, r_lo, c_lo, nc, x_lo, y_lo, (long long)plane * g.th * g.tw, s_visit, s_shift);
    } else {
        if (tid < nv) {
            const int ri = tid / nc, ci = tid - ri * nc;
            const int r = r_lo + ri, c = c_lo + ci;
            const unsigned t = (unsigned)(r * g.cols + c);
            const unsigned b = fastdiv(t, p.bs_magic);
            const int u0 = x_lo - (int)g.xs[c];
            const int v0 = y_lo - (int)g.ys[r], k0 = u0 >> L2V;
            const long long elem = (long long)(t - b * (unsigned)p.tile_bs) * p.tile_stride + (long long)v0 * g.tw + (long long)k0 * VEC;
            VisitEntry e;
            e.origin = (long long)reinterpret_cast<uintptr_t>(p.batch_ptrs[b]) + elem * (long long)sizeof(T) + (long long)plane * plane_bytes;
            e.v0 = v0;
            e.k0 = k0;
            s_visit[tid] = e;
            s_shift[tid] = u0 & (VEC - 1);
        }
        __syncthreads();
    }

    // ---- issue every copy of this CTA: src = origin(visit) + offset(thread) + plane, zero-fill outside the tile -----
    if (tid < kAsSlots) {
        const int row = tid / kAsChunks, j = tid - row * kAsChunks;    // this thread's copy slot (same in every stage)
        const int th1 = g.th - 1 - row, tw1 = (g.tw >> L2V) - 1 - j;   // v0 <= th1 and k0 <= tw1 <=> inside the tile (upper bounds)
        const long long off = ((long long)row * g.tw + (long long)j * VEC) * (long long)sizeof(T);
        uint32_t dst = smem_u32(td_smem) + (uint32_t)tid * 16u;
#pragma unroll 4
        for (int i = 0; i < nv; ++i, dst += PPC * kAsStage) {
            const VisitEntry e = s_visit[i];
            // negative (= outside the tile) iff v < 0, v >= th, k < 0 or k >= twv, with v = v0 + row, k = k0 + j
            const int skip = (e.v0 + row) | (th1 - e.v0) | (e.k0 + j) | (tw1 - e.k0);
#pragma unroll
            for (int q = 0; q < PPC; ++q) cp_async16_zfill(dst + q * kAsStage, e.origin + off + q * plane_bytes, skip);
        }
    }
    cp_async_wait_all();
    __syncthreads();
    if (tid >= kAsVecThreads) return;

    // ---- consume in tile order ------------------------------------------------------------------------
    const unsigned char* mine = td_smem + (ty * kAsChunks + tx) * 16;
    uint4 acc[PPC];
#pragma unroll
    for (int q = 0; q < PPC; ++q) acc[q] = make_uint4(0, 0, 0, 0);
    {
        for (int i = 0; i < nv; ++i, mine += PPC * kAsStage) {
            const int s = s_shift[i];   // uniform over the CTA
            if constexpr (VEC == 8) {
                switch (s) {
                    case 0: consume_planes<T, 0, PPC>(acc, mine); break;
                    case 1: consume_planes<T, 1, PPC>(acc, mine); break;
                    case 2: consume_planes<T, 2, PPC>(acc, mine); break;
                    case 3: consume_planes<T, 3, PPC>(acc, mine); break;
                    case 4: consume_planes<T, 4, PPC>(acc, mine); break;
                    case 5: consume_planes<T, 5, PPC>(acc, mine); break;
                    case 6: consume_planes<T, 6, PPC>(acc, mine); break;
                    default: consume_planes<T, 7, PPC>(acc, mine); break;
                }
            } else {
                switch (s) {
                    case 0: consume_planes<T, 0, PPC>(acc, mine); break;
                    case 1: consume_planes<T, 1, PPC>(acc, mine); break;
                    case 2: consume_planes<T, 2, PPC>(acc, mine); break;
                    default: consume_planes<T, 3, PPC>(acc, mine); break;
                }
            }
        }
    }

    // ---- normalise + store --------------------------------------------------------------------------
    if (!inside) return;
#pragma unroll
    for (int q = 0; q < PPC; ++q) {
        const long long o = ((long long)(plane + q) * g.H + y) * g.W + x0;
        float4* op = reinterpret_cast<float4*>(out_f32 + o);
#pragma unroll
        for (int h = 0; h < VEC / 4; ++h) {
            const float4 w = wv[h];
            const float a0 = Vec<T>::get(acc[q], 4 * h + 0), a1 = Vec<T>::get(acc[q], 4 * h + 1);
            const float a2 = Vec<T>::get(acc[q], 4 * h + 2), a3 = Vec<T>::get(acc[q], 4 * h + 3);
            float4 f;   // x_out = where(weights > 1, x_buffer / weights, x_buffer)  -- fp32, correctly rounded divide
            if constexpr (FASTDIV) {
                const float4 rc = rv[h];
                f.x = w.x > 1.0f ? div_exact_small_int(a0, w.x, rc.x) : a0;
                f.y = w.y > 1.0f ? div_exact_small_int(a1, w.y, rc.y) : a1;
                f.z = w.z > 1.0f ? div_exact_small_int(a2, w.z, rc.z) : a2;
                f.w = w.w > 1.0f ? div_exact_small_int(a3, w.w, rc.w) : a3;
            } else {
                f.x = w.x > 1.0f ? __fdiv_rn(a0, w.x) : a0;
                f.y = w.y > 1.0f ? __fdiv_rn(a1, w.y) : a1;
                f.z = w.z > 1.0f ? __fdiv_rn(a2, w.z) : a2;
                f.w = w.w > 1.0f ? __fdiv_rn(a3, w.w) : a3;
            }
            op[h] = f;
        }
        if constexpr (WRITE_BUF) stg128(out_buf + o, acc[q]);
    }
}

// ---------------------------------------------------------------------------
// Blend, Mixture of Diffusers, cp.async path: same staging as blend_md_async_kernel; the consume
// step reproduces mixtureofdiffusers.py:125-126 per element --
//     w = tile_weights[v, u] * rescale[y, x]      (fp32 product, own rounding)
//     acc = round_T(float(acc) + float(tile) * w) (separate multiply and add, no FMA)
// The gaussian tile weights are read with three aligned 128-bit loads per vector (the 4-float shift
// is uniform over the CTA).  Elements outside the tile are skipped explicitly (see mod_accumulate).
// ---------------------------------------------------------------------------
// [jlo, jhi): the elements of this vector that lie inside the tile.  Elements outside must not be touched at all:
// with gaussian weights the accumulator CAN be -0.0 (a tiny negative sum rounds to -0 in fp16), and -0 + (+0) = +0.
template <typename T, int O>
__device__ __forceinline__ void mod_accumulate(float (&acc)[Vec<T>::kElems], const uint4& e, const float4& w0, const float4& w1,
                                               const float4& w2, const float (&rs)[Vec<T>::kElems], int jlo, int jhi) {
    constexpr int VEC = Vec<T>::kElems;
    const float wl[12] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w, w2.x, w2.y, w2.z, w2.w};
    if (jlo == 0 && jhi == VEC) {
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
            const float w = __fmul_rn(wl[O + j], rs[j]);
            const float val = __fmul_rn(Vec<T>::get(e, j), w);
            acc[j] = round_through<T>(__fadd_rn(acc[j], val));
        }
    } else {
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
            const float w = __fmul_rn(wl[O + j], rs[j]);
            const float val = __fmul_rn(Vec<T>::get(e, j), w);
            const float sum = round_through<T>(__fadd_rn(acc[j], val));
            acc[j] = (j >= jlo && j < jhi) ? sum : acc[j];
        }
    }
}

// WINDOW: a row-window launch (td_blend_mixture_rows: py0 / py_count, sched, halo wait); without it the grid is the whole
// canvas with blockIdx.y = patch row, and none of that code is compiled in (the whole-canvas blend keeps its instruction stream).
// SPARSE (td_blend_mixture_sparse, whole canvas only): visits through the slot table, as in blend_md_async_kernel.
template <typename T, bool WINDOW, bool SPARSE = false>
__global__ void __launch_bounds__(kAsThreads)
blend_mod_async_kernel(const __grid_constant__ BlendParams p, const float* __restrict__ tile_weights, const float* __restrict__ rescale,
                       T* __restrict__ out_buf, const int* __restrict__ slot) {
    constexpr int VEC = Vec<T>::kElems;
    constexpr int L2V = Vec<T>::kLog2;
    constexpr int BX = kAsX * VEC;
    extern __shared__ __align__(16) unsigned char td_smem[];
    __shared__ VisitEntry s_visit[kAsMaxVisits];
    __shared__ int s_shift[kAsMaxVisits];
    const GeomParams& g = p.g;
    const int tid = threadIdx.x;
    const int by = WINDOW ? window_row_index(p) + p.py0 : (int)blockIdx.y;
    const int plane = WINDOW ? plane_group_index(p) : (int)blockIdx.z;
    const int x_lo = blockIdx.x * BX, y_lo = by * kAsY;
    const int r_lo = p.prow_lo[by], c_lo = p.pcol_lo[blockIdx.x];
    const int nc = p.pcol_n[blockIdx.x];
    int nv = (int)p.prow_n[by] * nc;
    pdl_launch_dependents();

    const int tx = tid % kAsX, ty = tid / kAsX;
    const int x0 = x_lo + tx * VEC, y = y_lo + ty;
    const bool inside = tid < kAsVecThreads && x0 < g.W && y < g.H;
    float rs[VEC];
    pdl_wait();
#pragma unroll
    for (int h = 0; h < VEC / 4; ++h) {
        const float4 f = inside ? __ldg(reinterpret_cast<const float4*>(rescale + (long long)y * g.W + x0) + h) : make_float4(0.f, 0.f, 0.f, 0.f);
        rs[4 * h + 0] = f.x; rs[4 * h + 1] = f.y; rs[4 * h + 2] = f.z; rs[4 * h + 3] = f.w;
    }
#pragma unroll
    for (int j = 0; j < VEC; ++j)   // 1/0 = inf marks a pixel no tile covers: it receives only zero fill, keep 0 * w finite
        if (isinf(rs[j])) rs[j] = 0.0f;
    if constexpr (WINDOW) halo_wait(p, by, r_lo, tid);

    if constexpr (SPARSE) {
        nv = prepare_sparse_visits<T>(p, slot, nv, r_lo, c_lo, nc, x_lo, y_lo, (long long)plane * g.th * g.tw, s_visit, s_shift);
    } else {
        if (tid < nv) {
            const int ri = tid / nc, ci = tid - ri * nc;
            const int r = r_lo + ri, c = c_lo + ci;
            const unsigned t = (unsigned)(r * g.cols + c);
            const unsigned b = fastdiv(t, p.bs_magic);
            const int u0 = x_lo - (int)g.xs[c];
            const int v0 = y_lo - (int)g.ys[r], k0 = u0 >> L2V;
            const long long elem = (long long)(t - b * (unsigned)p.tile_bs) * p.tile_stride + (long long)plane * g.th * g.tw +
                                   (long long)v0 * g.tw + (long long)k0 * VEC;
            VisitEntry e;
            e.origin = (long long)reinterpret_cast<uintptr_t>(p.batch_ptrs[b]) + elem * (long long)sizeof(T);
            e.v0 = v0;
            e.k0 = k0;
            s_visit[tid] = e;
            s_shift[tid] = u0 & (VEC - 1);
        }
        __syncthreads();
    }
    if (tid < kAsSlots) {
        const int row = tid / kAsChunks, j = tid - row * kAsChunks;
        const int th1 = g.th - 1 - row, tw1 = (g.tw >> L2V) - 1 - j;
        const long long off = ((long long)row * g.tw + (long long)j * VEC) * (long long)sizeof(T);
        uint32_t dst = smem_u32(td_smem) + (uint32_t)tid * 16u;
#pragma unroll 4
        for (int i = 0; i < nv; ++i, dst += kAsStage) {
            const VisitEntry e = s_visit[i];
            const int skip = (e.v0 + row) | (th1 - e.v0) | (e.k0 + j) | (tw1 - e.k0);
            cp_async16_zfill(dst, e.origin + off, skip);
        }
    }
    cp_async_wait_all();
    __syncthreads();
    if (!inside) return;

    const unsigned char* mine = td_smem + (ty * kAsChunks + tx) * 16;
    const int tw4 = g.tw >> 2;   // tile-weight row in float4 chunks (tw % 8 == 0 on this path)
    float acc[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) acc[j] = 0.0f;
    for (int i = 0; i < nv; ++i, mine += kAsStage) {
        const VisitEntry e = s_visit[i];
        const int s = s_shift[i];
        const int v = e.v0 + ty;
        if ((unsigned)v >= (unsigned)g.th) continue;        // this row of the stage is all zero fill: nothing to add
        const uint4 A = lds128(mine);
        uint4 ev = A;
        if (s != 0) ev = Vec<T>::window(A, lds128(mine + 16), s);
        const int u = e.k0 * VEC + s + tx * VEC;            // tile column of element 0 (may be outside the tile)
        const int q0 = u >> 2, o = u & 3;                   // o == s & 3: uniform over the CTA
        const float4* wrow = reinterpret_cast<const float4*>(tile_weights + (long long)v * g.tw);
        const float4 w0 = __ldg(wrow + min(max(q0, 0), tw4 - 1));
        const float4 w1 = __ldg(wrow + min(max(q0 + 1, 0), tw4 - 1));
        const float4 w2 = __ldg(wrow + min(max(q0 + 2, 0), tw4 - 1));
        const int jlo = max(0, -u), jhi = min(VEC, g.tw - u);
        if (jhi <= jlo) continue;                           // vector entirely outside this tile
        switch (o) {
            case 0: mod_accumulate<T, 0>(acc, ev, w0, w1, w2, rs, jlo, jhi); break;
            case 1: mod_accumulate<T, 1>(acc, ev, w0, w1, w2, rs, jlo, jhi); break;
            case 2: mod_accumulate<T, 2>(acc, ev, w0, w1, w2, rs, jlo, jhi); break;
            default: mod_accumulate<T, 3>(acc, ev, w0, w1, w2, rs, jlo, jhi); break;
        }
    }

    const long long o_ = ((long long)plane * g.H + y) * g.W + x0;
    uint4 pk;
    if constexpr (sizeof(T) == 2) {
        uint32_t w32[4];
#pragma unroll
        for (int h = 0; h < 4; ++h)
            w32[h] = (uint32_t)Elem<T>::f32_to_bits(acc[2 * h]) | ((uint32_t)Elem<T>::f32_to_bits(acc[2 * h + 1]) << 16);
        pk = make_uint4(w32[0], w32[1], w32[2], w32[3]);
    } else {
        pk = make_uint4(__float_as_uint(acc[0]), __float_as_uint(acc[1]), __float_as_uint(acc[2]), __float_as_uint(acc[3]));
    }
    stg128(out_buf + o_, pk);
}

// ---------------------------------------------------------------------------
// Persistent, software-pipelined form of the cp.async blend (TD_FLAG_PIPELINE, opt-in): a CTA walks
// patches pi = blockIdx.x, += gridDim.x with two stage sets -- the copies of patch n+1
// are in flight while patch n is consumed, normalised and stored, so DRAM stays busy
// instead of all CTAs of a wave issuing, waiting and computing in lock step.  Fewer resident
// warps per SM and three barriers per patch can cost more than the overlap wins, so it is an
// opt-in, not the default.
// ---------------------------------------------------------------------------
template <typename T, bool WRITE_BUF, bool FASTDIV>
__global__ void __launch_bounds__(kAsThreads)
blend_md_pipe_kernel(const __grid_constant__ BlendParams p, const float* __restrict__ weights, const float* __restrict__ rcp_weights,
                     float* __restrict__ out_f32, T* __restrict__ out_buf, int nv_cap, int px_count, int py_count, int total_patches) {
    constexpr int VEC = Vec<T>::kElems;
    constexpr int L2V = Vec<T>::kLog2;
    constexpr int BX = kAsX * VEC;
    extern __shared__ __align__(16) unsigned char td_smem[];
    __shared__ VisitEntry s_visit[2][kAsMaxVisits];
    __shared__ int s_shift[2][kAsMaxVisits];
    const GeomParams& g = p.g;
    const int tid = threadIdx.x;
    const int set_bytes = nv_cap * kAsStage;

    // per-thread constants: copy slot (same in every stage) and output vector
    const int row = tid / kAsChunks, j = tid - row * kAsChunks;
    const int th1 = g.th - 1 - row, tw1 = (g.tw >> L2V) - 1 - j;
    const long long off = ((long long)row * g.tw + (long long)j * VEC) * (long long)sizeof(T);
    const uint32_t smem0 = smem_u32(td_smem);
    const int tx = tid % kAsX, ty = tid / kAsX;
    const bool vec_thread = tid < kAsVecThreads;

    struct Patch { int x_lo, y_lo, plane, nv; };
    auto decode = [&](int pi) {
        Patch q;
        const int px = pi % px_count, t = pi / px_count;
        const int py = t % py_count;
        q.plane = t / py_count;
        q.x_lo = px * BX; q.y_lo = py * kAsY;
        q.nv = g.dbg_no_tiles ? 0 : (int)p.prow_n[py] * (int)p.pcol_n[px];
        return q;
    };
    auto build_table = [&](const Patch& q, int set) {   // thread i prepares visit i
        if (tid < q.nv) {
            const int px = q.x_lo / BX, py = q.y_lo / kAsY;
            const int nc = p.pcol_n[px];
            const int ri = tid / nc, ci = tid - ri * nc;
            const int r = (int)p.prow_lo[py] + ri, c = (int)p.pcol_lo[px] + ci;
            const unsigned t = (unsigned)(r * g.cols + c);
            const unsigned b = fastdiv(t, p.bs_magic);
            const int u0 = q.x_lo - (int)g.xs[c];
            const int v0 = q.y_lo - (int)g.ys[r], k0 = u0 >> L2V;
            const long long elem = (long long)(t - b * (unsigned)p.tile_bs) * p.tile_stride + (long long)q.plane * g.th * g.tw +
                                   (long long)v0 * g.tw + (long long)k0 * VEC;
            VisitEntry e;
            e.origin = (long long)reinterpret_cast<uintptr_t>(p.batch_ptrs[b]) + elem * (long long)sizeof(T);
            e.v0 = v0;
            e.k0 = k0;
            s_visit[set][tid] = e;
            s_shift[set][tid] = u0 & (VEC - 1);
        }
    };
    auto issue = [&](const Patch& q, int set) {
        if (tid < kAsSlots) {
            uint32_t dst = smem0 + (uint32_t)(set * set_bytes) + (uint32_t)tid * 16u;
#pragma unroll 4
            for (int i = 0; i < q.nv; ++i, dst += kAsStage) {
                const VisitEntry e = s_visit[set][i];
                const int skip = (e.v0 + row) | (th1 - e.v0) | (e.k0 + j) | (tw1 - e.k0);
                cp_async16_zfill(dst, e.origin + off, skip);
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    float4 wv[VEC / 4], rv[VEC / 4], wn[VEC / 4], rn[VEC / 4];
    auto prefetch_weights = [&](const Patch& q) {
        const int x0 = q.x_lo + tx * VEC, y = q.y_lo + ty;
        const bool inside = vec_thread && x0 < g.W && y < g.H;
        const long long wo = (long long)y * g.W + x0;
#pragma unroll
        for (int h = 0; h < VEC / 4; ++h) {
            wn[h] = inside ? __ldg(reinterpret_cast<const float4*>(weights + wo) + h) : make_float4(1.f, 1.f, 1.f, 1.f);
            if constexpr (FASTDIV) rn[h] = inside ? __ldg(reinterpret_cast<const float4*>(rcp_weights + wo) + h) : make_float4(1.f, 1.f, 1.f, 1.f);
        }
    };

    int pi = blockIdx.x;
    if (pi >= total_patches) return;
    Patch nxt = decode(pi);
    build_table(nxt, 0);
    __syncthreads();
    issue(nxt, 0);
    prefetch_weights(nxt);
    int b = 0;
    while (true) {
        const Patch cur = nxt;
#pragma unroll
        for (int h = 0; h < VEC / 4; ++h) { wv[h] = wn[h]; if constexpr (FASTDIV) rv[h] = rn[h]; }
        const int next_pi = pi + gridDim.x;
        const bool has_next = next_pi < total_patches;
        __syncthreads();                       // everyone is done with set / table 1-b (consumed one iteration ago)
        if (has_next) { nxt = decode(next_pi); build_table(nxt, 1 - b); }
        __syncthreads();                       // table 1-b visible
        if (has_next) { issue(nxt, 1 - b); prefetch_weights(nxt); }
        else asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 1;" ::: "memory");
        __syncthreads();                       // set b has landed for every thread

        if (vec_thread) {
            const unsigned char* mine = td_smem + b * set_bytes + (ty * kAsChunks + tx) * 16;
            uint4 acc = make_uint4(0, 0, 0, 0);
            for (int i = 0; i < cur.nv; ++i, mine += kAsStage) {
                const int s = s_shift[b][i];   // uniform over the CTA
                if constexpr (VEC == 8) {
                    switch (s) {
                        case 0: consume_shifted<T, 0>(acc, mine); break;
                        case 1: consume_shifted<T, 1>(acc, mine); break;
                        case 2: consume_shifted<T, 2>(acc, mine); break;
                        case 3: consume_shifted<T, 3>(acc, mine); break;
                        case 4: consume_shifted<T, 4>(acc, mine); break;
                        case 5: consume_shifted<T, 5>(acc, mine); break;
                        case 6: consume_shifted<T, 6>(acc, mine); break;
                        default: consume_shifted<T, 7>(acc, mine); break;
                    }
                } else {
                    switch (s) {
                        case 0: consume_shifted<T, 0>(acc, mine); break;
                        case 1: consume_shifted<T, 1>(acc, mine); break;
                        case 2: consume_shifted<T, 2>(acc, mine); break;
                        default: consume_shifted<T, 3>(acc, mine); break;
                    }
                }
            }
            const int x0 = cur.x_lo + tx * VEC, y = cur.y_lo + ty;
            if (x0 < g.W && y < g.H) {
                const long long o = ((long long)cur.plane * g.H + y) * g.W + x0;
                float4* op = reinterpret_cast<float4*>(out_f32 + o);
#pragma unroll
                for (int h = 0; h < VEC / 4; ++h) {
                    const float4 w = wv[h];
                    const float a0 = Vec<T>::get(acc, 4 * h + 0), a1 = Vec<T>::get(acc, 4 * h + 1);
                    const float a2 = Vec<T>::get(acc, 4 * h + 2), a3 = Vec<T>::get(acc, 4 * h + 3);
                    float4 f;   // x_out = where(weights > 1, x_buffer / weights, x_buffer)  -- fp32, correctly rounded divide
                    if constexpr (FASTDIV) {
                        const float4 rc = rv[h];
                        f.x = w.x > 1.0f ? div_exact_small_int(a0, w.x, rc.x) : a0;
                        f.y = w.y > 1.0f ? div_exact_small_int(a1, w.y, rc.y) : a1;
                        f.z = w.z > 1.0f ? div_exact_small_int(a2, w.z, rc.z) : a2;
                        f.w = w.w > 1.0f ? div_exact_small_int(a3, w.w, rc.w) : a3;
                    } else {
                        f.x = w.x > 1.0f ? __fdiv_rn(a0, w.x) : a0;
                        f.y = w.y > 1.0f ? __fdiv_rn(a1, w.y) : a1;
                        f.z = w.z > 1.0f ? __fdiv_rn(a2, w.z) : a2;
                        f.w = w.w > 1.0f ? __fdiv_rn(a3, w.w) : a3;
                    }
                    op[h] = f;
                }
                if constexpr (WRITE_BUF) stg128(out_buf + o, acc);
            }
        }
        if (!has_next) break;
        pi = next_pi;
        b ^= 1;
    }
}

// exhaustive check of div_exact_small_int against the IEEE divide: every 16-bit pattern of T x w in [1, max_w]
template <typename T>
__global__ void check_fast_div_kernel(int max_w, unsigned long long* mismatches) {
    const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;   // 16-bit pattern
    if (idx >= 65536u) return;
    const float a = Elem<T>::bits_to_f32((uint16_t)idx);
    if (isnan(a) || isinf(a)) return;
    unsigned long long bad = 0;
    for (int wi = 1; wi <= max_w; ++wi) {
        const float w = (float)wi;
        const float rcp = __fdiv_rn(1.0f, w);
        const float q = div_exact_small_int(a, w, rcp);
        const float ref = __fdiv_rn(a, w);
        if (__float_as_uint(q) != __float_as_uint(ref)) ++bad;
    }
    if (bad) atomicAdd(mismatches, bad);
}

// ---------------------------------------------------------------------------
// Blend + normalise, MultiDiffusion, TMA path (TD_FLAG_TMA; kept as the measured alternative, see DESIGN.md).
//
// A CTA owns an 8-row x 16-vector patch of one canvas plane.  For every tile that
// touches the patch (ascending tile index) one thread issues ONE cp.async.bulk.tensor
// box load: the copy engine clips the box against the tile and zero-fills the rest.
// All boxes of a CTA are in flight at once (one mbarrier each, no staging registers);
// the threads then walk the stages in tile order.  TMA wants a 16-byte aligned inner
// start coordinate, so the box is the aligned superset of the patch (BX + VEC columns)
// and the per-tile shift s = (x_lo - xs) mod VEC -- uniform over the CTA -- is applied
// on the shared-memory read: two aligned LDS.128 + funnel shift, then a packed add.
// Zero fill is exact: the accumulator starts at +0 and can never become -0.
// ---------------------------------------------------------------------------
constexpr int kTmaBXV = 16;   // vectors per patch row
constexpr int kTmaBY = 8;     // patch rows
constexpr int kTmaThreads = kTmaBXV * kTmaBY;
constexpr int kTmaMaxVisits = 96;

template <int NB>
struct TmaBlendParams {
    GeomParams g;
    int tile_bs;
    unsigned bs_magic;
    int nv_cap;
    CUtensorMap maps[NB];
};

template <typename T, bool WRITE_BUF, int NB>
__global__ void __launch_bounds__(kTmaThreads)
blend_md_tma_kernel(const __grid_constant__ TmaBlendParams<NB> p, const float* __restrict__ weights,
                    float* __restrict__ out_f32, T* __restrict__ out_buf) {
    constexpr int VEC = Vec<T>::kElems;
    constexpr int L2V = Vec<T>::kLog2;
    constexpr int BX = kTmaBXV * VEC;
    constexpr int PITCH = (BX + VEC) * (int)sizeof(T);   // bytes per staged row (aligned superset)
    constexpr int STAGE = PITCH * kTmaBY;                // multiple of 128 B
    extern __shared__ __align__(128) unsigned char td_smem[];
    __shared__ short s_ys[TD_MAX_GRID_DIM];
    __shared__ short s_xs[TD_MAX_GRID_DIM];
    __shared__ signed char s_shift[kTmaMaxVisits];
    const GeomParams& g = p.g;
    uint64_t* bars = reinterpret_cast<uint64_t*>(td_smem + (size_t)p.nv_cap * STAGE);
    load_origins(g, s_ys, s_xs);

    const int plane = blockIdx.z;
    const int x_lo = blockIdx.x * BX, y_lo = blockIdx.y * kTmaBY;
    const int x_hi = min(x_lo + BX, g.W) - 1, y_hi = min(y_lo + kTmaBY, g.H) - 1;
    const int r_lo = last_le(s_ys, g.rows, y_lo - g.th, g.inv_dy) + 1;
    const int r_hi = last_le(s_ys, g.rows, y_hi, g.inv_dy);
    const int c_lo = last_le(s_xs, g.cols, x_lo - g.tw, g.inv_dx) + 1;
    const int c_hi = last_le(s_xs, g.cols, x_hi, g.inv_dx);
    const int nc = c_hi - c_lo + 1;
    const int nv = g.dbg_no_tiles ? 0 : (r_hi - r_lo + 1) * nc;   // <= nv_cap by construction on the host

    // visit i is owned by thread i: init its barrier, publish its shift, launch its box
    for (int i = threadIdx.x; i < nv; i += kTmaThreads) {
        const int ri = i / nc, ci = i - ri * nc;
        const int r = r_lo + ri, c = c_lo + ci;
        const unsigned t = (unsigned)(r * g.cols + c);
        const unsigned b = fastdiv(t, p.bs_magic);
        const int pz = (int)(t - b * (unsigned)p.tile_bs) * (g.N * g.C) + plane;   // plane inside batch tensor b
        const int u0 = x_lo - (int)s_xs[c];          // tile-local column of the patch's first pixel
        const int k = u0 >> L2V;                     // floor: aligned chunk holding it
        s_shift[i] = (signed char)(u0 & (VEC - 1));
        mbar_init(&bars[i], 1);
        fence_proxy_async();
        mbar_arrive_expect_tx(&bars[i], STAGE);
        tma_load_3d(td_smem + (size_t)i * STAGE, &p.maps[b], k * VEC, y_lo - (int)s_ys[r], pz, &bars[i]);
    }
    __syncthreads();

    const int tx = threadIdx.x % kTmaBXV, ty = threadIdx.x / kTmaBXV;
    const unsigned char* mine = td_smem + (size_t)ty * PITCH + (size_t)tx * 16;
    uint4 acc = make_uint4(0, 0, 0, 0);
    for (int i = 0; i < nv; ++i) {
        const int s = (int)s_shift[i];
        mbar_wait(&bars[i], 0);
        const uint4 A = lds128(mine + (size_t)i * STAGE);
        uint4 e = A;
        if (s != 0) {
            const uint4 B = lds128(mine + (size_t)i * STAGE + 16);
            e = Vec<T>::window(A, B, s);
        }
        acc.x = packed_add<T>(acc.x, e.x);
        acc.y = packed_add<T>(acc.y, e.y);
        acc.z = packed_add<T>(acc.z, e.z);
        acc.w = packed_add<T>(acc.w, e.w);
    }

    const int x0 = x_lo + tx * VEC, y = y_lo + ty;
    if (x0 >= g.W || y >= g.H) return;
    const long long o = ((long long)plane * g.H + y) * g.W + x0;
    const float4* wp = reinterpret_cast<const float4*>(weights + (long long)y * g.W + x0);
    float4* op = reinterpret_cast<float4*>(out_f32 + o);
#pragma unroll
    for (int h = 0; h < VEC / 4; ++h) {
        const float4 w = __ldg(wp + h);
        const float a0 = Vec<T>::get(acc, 4 * h + 0), a1 = Vec<T>::get(acc, 4 * h + 1);
        const float a2 = Vec<T>::get(acc, 4 * h + 2), a3 = Vec<T>::get(acc, 4 * h + 3);
        float4 f;   // x_out = where(weights > 1, x_buffer / weights, x_buffer)  -- fp32, IEEE divide
        f.x = w.x > 1.0f ? __fdiv_rn(a0, w.x) : a0;
        f.y = w.y > 1.0f ? __fdiv_rn(a1, w.y) : a1;
        f.z = w.z > 1.0f ? __fdiv_rn(a2, w.z) : a2;
        f.w = w.w > 1.0f ? __fdiv_rn(a3, w.w) : a3;
        op[h] = f;
    }
    if constexpr (WRITE_BUF) stg128(out_buf + o, acc);
}

// Blend, generic path: one element per thread, any width / alignment, tile
// dtype and canvas dtype independent.
// SPARSE: tile t is read at position slot[t] of the compact batches, and skipped when slot[t] < 0.
template <typename TIn, typename TAcc, int MODE, bool SPARSE = false>
__global__ void __launch_bounds__(256)
blend_grid_generic_kernel(const __grid_constant__ BlendParams p, const float* __restrict__ weights,
                          const float* __restrict__ tile_weights, const float* __restrict__ rescale,
                          float* __restrict__ out_f32, TAcc* __restrict__ out_buf, long long total, const int* __restrict__ slot) {
    __shared__ short s_ys[TD_MAX_GRID_DIM];
    __shared__ short s_xs[TD_MAX_GRID_DIM];
    const GeomParams& g = p.g;
    load_origins(g, s_ys, s_xs);
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    long long rem = idx;
    const int x = (int)(rem % g.W); rem /= g.W;
    const int y = (int)(rem % g.H); rem /= g.H;
    const int plane = (int)rem;
    const int r_lo = last_le(s_ys, g.rows, y - g.th, g.inv_dy) + 1;
    const int r_hi = last_le(s_ys, g.rows, y, g.inv_dy);
    const int c_lo = last_le(s_xs, g.cols, x - g.tw, g.inv_dx) + 1;
    const int c_hi = last_le(s_xs, g.cols, x, g.inv_dx);
    float acc = 0.0f;
    float rsc = 0.0f;
    if constexpr (MODE == MODE_MOD) rsc = rescale[(long long)y * g.W + x];
    for (int r = r_lo; r <= r_hi; ++r) {
        const int v = y - (int)s_ys[r];
        for (int c = c_lo; c <= c_hi; ++c) {
            int t = r * g.cols + c;
            if constexpr (SPARSE) {
                t = slot[t];
                if (t < 0) continue;
            }
            const int b = t / p.tile_bs;
            const int u = x - (int)s_xs[c];
            const TIn* tp = reinterpret_cast<const TIn*>(p.batch_ptrs[b]) + (long long)(t - b * p.tile_bs) * p.tile_stride +
                            ((long long)plane * g.th + v) * g.tw + u;
            float val = Elem<TIn>::to_f32(*tp);
            if constexpr (MODE == MODE_MOD) val = __fmul_rn(val, __fmul_rn(tile_weights[(long long)v * g.tw + u], rsc));
            acc = round_through<TAcc>(__fadd_rn(acc, val));
        }
    }
    if constexpr (MODE == MODE_MD) {
        const float w = weights[(long long)y * g.W + x];
        out_f32[idx] = w > 1.0f ? __fdiv_rn(acc, w) : acc;
    }
    if (out_buf != nullptr) out_buf[idx] = Elem<TAcc>::from_f32(acc);
}

// ---------------------------------------------------------------------------
// Host-side dispatch
// ---------------------------------------------------------------------------
constexpr uint32_t kOptInForms = TD_FLAG_ROWS | TD_FLAG_STRIP | TD_FLAG_TMA | TD_FLAG_PIPELINE;

// On an axis whose g->wrap bit is clear every tile must lie inside the canvas (the kernels of this file index the canvas
// without bounds checks); on a periodic axis an origin lies in [0, extent).
int fill_geom(const td_grid* g, int N, int C, GeomParams* o) {
    if (g == nullptr) { td_set_error("null grid"); return TD_ERR_INVALID_ARG; }
    if (N <= 0 || C <= 0) { td_set_error("N and C must be positive (N=%d C=%d)", N, C); return TD_ERR_INVALID_ARG; }
    if (g->rows <= 0 || g->cols <= 0 || g->rows > TD_MAX_GRID_DIM || g->cols > TD_MAX_GRID_DIM ||
        g->num_tiles != g->rows * g->cols || (g->wrap & ~(int)(TD_WRAP_X | TD_WRAP_Y)) != 0) {
        td_set_error("grid not initialised (rows=%d cols=%d wrap=%d)", g->rows, g->cols, g->wrap);
        return TD_ERR_INVALID_ARG;
    }
    if (g->H >= 32768 || g->W >= 32768) { td_set_error("canvas %dx%d too large", g->H, g->W); return TD_ERR_UNSUPPORTED; }
    if (g->tile_w <= 0 || g->tile_h <= 0 || g->tile_w > g->W || g->tile_h > g->H) {
        td_set_error("tile %dx%d does not fit the %dx%d canvas", g->tile_w, g->tile_h, g->W, g->H);
        return TD_ERR_INVALID_ARG;
    }
    for (int c = 0; c < g->cols; ++c)
        if (g->xs[c] < 0 || g->xs[c] >= g->W || (!(g->wrap & TD_WRAP_X) && g->xs[c] + g->tile_w > g->W)) {
            td_set_error("tile column %d (x=%d, w=%d) leaves the %d-wide canvas", c, g->xs[c], g->tile_w, g->W);
            return TD_ERR_INVALID_ARG;
        }
    for (int r = 0; r < g->rows; ++r)
        if (g->ys[r] < 0 || g->ys[r] >= g->H || (!(g->wrap & TD_WRAP_Y) && g->ys[r] + g->tile_h > g->H)) {
            td_set_error("tile row %d (y=%d, h=%d) leaves the %d-high canvas", r, g->ys[r], g->tile_h, g->H);
            return TD_ERR_INVALID_ARG;
        }
    // every origin search (last_le, the wrap blends' cover ranges, the row bands of td_rows.cu / td_strip.cu) assumes
    // non-decreasing origins: out of order, it finds tiles that do not cover the pixel and reads outside them
    for (int c = 1; c < g->cols; ++c)
        if (g->xs[c] < g->xs[c - 1]) {
            td_set_error("tile column origins out of order: xs[%d]=%d < xs[%d]=%d", c, g->xs[c], c - 1, g->xs[c - 1]);
            return TD_ERR_INVALID_ARG;
        }
    for (int r = 1; r < g->rows; ++r)
        if (g->ys[r] < g->ys[r - 1]) {
            td_set_error("tile row origins out of order: ys[%d]=%d < ys[%d]=%d", r, g->ys[r], r - 1, g->ys[r - 1]);
            return TD_ERR_INVALID_ARG;
        }
    o->H = g->H; o->W = g->W; o->th = g->tile_h; o->tw = g->tile_w;
    o->rows = g->rows; o->cols = g->cols; o->N = N; o->C = C;
    for (int i = 0; i < g->rows; ++i) o->ys[i] = (short)g->ys[i];
    for (int i = 0; i < g->cols; ++i) o->xs[i] = (short)g->xs[i];
    const unsigned nc = (unsigned)(N * C);
    if (nc >= 65536u) { td_set_error("N*C = %u too large", nc); return TD_ERR_UNSUPPORTED; }
    o->nc_magic = magic_u16(nc);
    o->twv_magic = 0;  // set by the vector launchers (depends on the element size)
    o->dbg_no_tiles = 0;
    o->inv_dx = g->cols > 1 ? (float)(g->cols - 1) / (float)std::max(1, g->W - g->tile_w) : 0.0f;
    o->inv_dy = g->rows > 1 ? (float)(g->rows - 1) / (float)std::max(1, g->H - g->tile_h) : 0.0f;
    return TD_OK;
}

inline unsigned blocks_for(long long total, int threads) { return (unsigned)((total + threads - 1) / threads); }

template <typename T>
int launch_scatter(GeomParams gp, const void* x, void* tiles, int tile_begin, int n_tiles, bool vec, bool pdl, cudaStream_t st) {
    const long long elems = (long long)n_tiles * gp.N * gp.C * gp.th * gp.tw;
    if (elems == 0) return TD_OK;
    if (vec) {
        const int twv = gp.tw / Vec<T>::kElems;
        gp.twv_magic = magic_u16((unsigned)twv);
        const int rows_per_block = std::max(1, std::min(gp.th, (128 * 4 + twv - 1) / twv));  // ~4 vectors per thread
        if ((long long)rows_per_block * twv >= 65536) { td_set_error("tile row too wide for the vector scatter"); return TD_ERR_UNSUPPORTED; }
        dim3 grid((unsigned)(n_tiles * gp.N * gp.C), (unsigned)((gp.th + rows_per_block - 1) / rows_per_block));
        return launch("td_scatter_tiles", scatter_vec_kernel<T>, grid, dim3(128), 0, st, pdl, gp, (const T*)x, (T*)tiles, tile_begin,
                      rows_per_block);
    }
    scatter_generic_kernel<T><<<blocks_for(elems, 256), 256, 0, st>>>(gp, (const T*)x, (T*)tiles, tile_begin, elems);
    return launch_status("td_scatter_tiles");
}

template <typename T, int MODE>
int launch_blend_vec(const BlendParams& bp, const float* weights, const float* tile_weights, const float* rescale,
                     float* out_f32, void* out_buf, cudaStream_t st) {
    const GeomParams& g = bp.g;
    const int wv = g.W / Vec<T>::kElems;
    const int rows_per_block = kBlendWarps * 4 * BlendShape<MODE>::kRPT;
    dim3 grid((unsigned)((wv + kWarpVecs - 1) / kWarpVecs), (unsigned)((g.H + rows_per_block - 1) / rows_per_block),
              (unsigned)(g.N * g.C));
    if (grid.y > 65535u || grid.z > 65535u) { td_set_error("canvas too large for the vector blend grid"); return TD_ERR_UNSUPPORTED; }
    if (MODE == MODE_MD && out_buf != nullptr)
        blend_grid_vec_kernel<T, MODE, true><<<grid, kBlendWarps * 32, 0, st>>>(bp, weights, tile_weights, rescale, out_f32, (T*)out_buf);
    else
        blend_grid_vec_kernel<T, MODE, false><<<grid, kBlendWarps * 32, 0, st>>>(bp, weights, tile_weights, rescale, out_f32, (T*)out_buf);
    return launch_status("td_blend (vec)");
}

// max number of tile rows (cols) touching any BY-row (BX-px) patch: bounds the TMA stage count
int max_union(const int32_t* org, int n, int extent, int size, int patch) {
    int best = 0;
    for (int lo = 0; lo < size; lo += patch) {
        const int hi = std::min(lo + patch, size) - 1;
        int cnt = 0;
        for (int i = 0; i < n; ++i)
            if (org[i] <= hi && org[i] + extent > lo) ++cnt;
        best = std::max(best, cnt);
    }
    return best;
}

template <typename T, bool WRITE_BUF, int NB>
int launch_blend_tma_nb(const td_grid* g, const BlendParams& bp, int tile_dtype, const float* weights, float* out_f32, void* out_buf,
                        int nv_cap, cudaStream_t st) {
    constexpr int VEC = Vec<T>::kElems;
    constexpr int BX = kTmaBXV * VEC;
    constexpr int STAGE = (BX + VEC) * (int)sizeof(T) * kTmaBY;
    static TmaBlendParams<NB> tp;   // filled per launch under a lock (the params are copied at launch)
    static std::mutex mu;
    std::lock_guard<std::mutex> lk(mu);
    tp.g = bp.g; tp.tile_bs = bp.tile_bs; tp.bs_magic = bp.bs_magic; tp.nv_cap = nv_cap;
    const int NC = bp.g.N * bp.g.C;
    for (int b = 0; b < bp.num_batches; ++b) {
        const int nt = std::min(bp.tile_bs, g->num_tiles - b * bp.tile_bs);
        int rc = td_encode_tensor_map_3d(&tp.maps[b], bp.batch_ptrs[b], tile_dtype, (uint64_t)nt * NC, (uint64_t)bp.g.th,
                                         (uint64_t)bp.g.tw, kTmaBY, BX + VEC);
        if (rc != TD_OK) return rc;
    }
    const int smem = nv_cap * (STAGE + 8);
    int rc = smem_optin(blend_md_tma_kernel<T, WRITE_BUF, NB>, smem, "td_blend_multidiffusion (tma)");
    if (rc != TD_OK) return rc;
    dim3 grid((unsigned)((bp.g.W + BX - 1) / BX), (unsigned)((bp.g.H + kTmaBY - 1) / kTmaBY), (unsigned)NC);
    blend_md_tma_kernel<T, WRITE_BUF, NB><<<grid, kTmaThreads, smem, st>>>(tp, weights, out_f32, (T*)out_buf);
    return launch_status("td_blend_multidiffusion (tma)");
}

// returns TD_OK if launched, 1 if the TMA path does not apply (caller falls back), <0 on error
template <typename T>
int try_launch_blend_tma(const td_grid* g, const BlendParams& bp, int tile_dtype, const float* weights, float* out_f32,
                         void* out_buf, cudaStream_t st) {
    constexpr int VEC = Vec<T>::kElems;
    constexpr int BX = kTmaBXV * VEC;
    constexpr int STAGE = (BX + VEC) * (int)sizeof(T) * kTmaBY;
    if (bp.g.N * bp.g.C > 65535 || (bp.g.H + kTmaBY - 1) / kTmaBY > 65535) return 1;
    const int nv_cap = max_union(g->ys, g->rows, g->tile_h, g->H, kTmaBY) * max_union(g->xs, g->cols, g->tile_w, g->W, BX);
    if (nv_cap <= 0 || nv_cap > kTmaMaxVisits || nv_cap * (STAGE + 8) > 200 * 1024) return 1;
    const bool wb = out_buf != nullptr;
    if (bp.num_batches <= 32)
        return wb ? launch_blend_tma_nb<T, true, 32>(g, bp, tile_dtype, weights, out_f32, out_buf, nv_cap, st)
                  : launch_blend_tma_nb<T, false, 32>(g, bp, tile_dtype, weights, out_f32, out_buf, nv_cap, st);
    return wb ? launch_blend_tma_nb<T, true, TD_MAX_BATCH_PTRS>(g, bp, tile_dtype, weights, out_f32, out_buf, nv_cap, st)
              : launch_blend_tma_nb<T, false, TD_MAX_BATCH_PTRS>(g, bp, tile_dtype, weights, out_f32, out_buf, nv_cap, st);
}

// tiles touching each patch along one axis: first index and count (both fit a byte: <= 256 tiles per axis)
void fill_patch_table(const int32_t* org, int n, int extent, int size, int patch, unsigned char* lo_out, unsigned char* n_out) {
    int idx = 0;
    for (int lo = 0; lo < size; lo += patch, ++idx) {
        const int hi = std::min(lo + patch, size) - 1;
        int first = -1, cnt = 0;
        for (int i = 0; i < n; ++i)
            if (org[i] <= hi && org[i] + extent > lo) { if (first < 0) first = i; ++cnt; }
        lo_out[idx] = (unsigned char)std::max(first, 0);
        n_out[idx] = (unsigned char)std::min(cnt, 255);
    }
}

template <typename T, bool WRITE_BUF, bool FASTDIV, int PPC, bool SPARSE = false>
int launch_blend_async_ppc(const BlendParams& bp, const float* weights, const float* rcp_weights, float* out_f32, void* out_buf,
                           int nv_cap, bool pdl, cudaStream_t st, const int* slot = nullptr) {
    constexpr int VEC = Vec<T>::kElems;
    constexpr int BX = kAsX * VEC;
    const int px = (bp.g.W + BX - 1) / BX, py = (bp.g.H + kAsY - 1) / kAsY, planes = bp.g.N * bp.g.C;
    const int smem = nv_cap * PPC * kAsStage;
    const char* what = "td_blend_multidiffusion (cp.async)";
    int rc = smem_optin(blend_md_async_kernel<T, WRITE_BUF, FASTDIV, PPC, SPARSE>, smem, what);
    if (rc != TD_OK) return rc;
    const unsigned gy = (unsigned)(bp.py_count > 0 ? bp.py_count : py), gz = (unsigned)(planes / PPC);
    dim3 grid((unsigned)px, bp.sched ? gz : gy, bp.sched ? gy : gz);
    return launch(what, blend_md_async_kernel<T, WRITE_BUF, FASTDIV, PPC, SPARSE>, grid, dim3(kAsThreads), (size_t)smem, st, pdl, bp,
                  weights, rcp_weights, out_f32, (T*)out_buf, slot);
}

// planes per CTA: at most TD_AS_PPC, 1 under TD_FLAG_ONE_PLANE (ppc_max)
#ifndef TD_AS_PPC
#define TD_AS_PPC 1   // tuning knob (-DTD_AS_PPC=): 1 / 2 / 4; cfg2 blend 12.5 us at 1 vs 13.35 us at 2 (H100 80GB HBM3, 700 W)
#endif
int ppc_max(uint32_t flags) { return (flags & TD_FLAG_ONE_PLANE) ? 1 : TD_AS_PPC; }

// SPARSE: one plane per CTA, never pipelined (the sparse entries take neither form)
template <typename T, bool WRITE_BUF, bool FASTDIV, bool SPARSE = false>
int launch_blend_async_impl(const BlendParams& bp, const float* weights, const float* rcp_weights, float* out_f32, void* out_buf,
                            int nv_cap, bool pipelined, bool pdl, int max_ppc, cudaStream_t st, const int* slot = nullptr) {
    constexpr int VEC = Vec<T>::kElems;
    constexpr int BX = kAsX * VEC;
    if constexpr (SPARSE)
        return launch_blend_async_ppc<T, WRITE_BUF, FASTDIV, 1, true>(bp, weights, rcp_weights, out_f32, out_buf, nv_cap, pdl, st, slot);
    const int px = (bp.g.W + BX - 1) / BX, py = (bp.g.H + kAsY - 1) / kAsY, planes = bp.g.N * bp.g.C;
    if (pipelined) {
        const int smem = 2 * nv_cap * kAsStage;
        const char* what = "td_blend_multidiffusion (cp.async)";
        int rc = smem_optin(blend_md_pipe_kernel<T, WRITE_BUF, FASTDIV>, smem, what);
        if (rc != TD_OK) return rc;
        const long long total = (long long)px * py * planes;
        const int per_sm = std::max(1, std::min(8, (220 * 1024) / (smem + 3 * 1024)));   // CTAs that fit one SM's shared memory
        const DeviceProps dev = device_props();
        const int sms = dev.ok ? dev.sms : 132;                                            // an H100's count when the query fails
        const int grid = (int)std::min<long long>(total, (long long)sms * per_sm);
        blend_md_pipe_kernel<T, WRITE_BUF, FASTDIV><<<grid, kAsThreads, smem, st>>>(bp, weights, rcp_weights, out_f32, (T*)out_buf, nv_cap,
                                                                                   px, py, (int)total);
        return launch_status(what);
    }
    if (max_ppc >= 4 && planes % 4 == 0 && 4 * nv_cap * kAsStage <= 64 * 1024)
        return launch_blend_async_ppc<T, WRITE_BUF, FASTDIV, 4>(bp, weights, rcp_weights, out_f32, out_buf, nv_cap, pdl, st);
    if (max_ppc >= 2 && planes % 2 == 0 && 2 * nv_cap * kAsStage <= 64 * 1024)
        return launch_blend_async_ppc<T, WRITE_BUF, FASTDIV, 2>(bp, weights, rcp_weights, out_f32, out_buf, nv_cap, pdl, st);
    return launch_blend_async_ppc<T, WRITE_BUF, FASTDIV, 1>(bp, weights, rcp_weights, out_f32, out_buf, nv_cap, pdl, st);
}

// Row-strip shard (patch tables filled): only the CTAs that read a neighbour's band wait; they sit at the end of the row range
// the halo enters from and are scheduled last (patch row = slowest grid dimension, walked away from that end).
void schedule_halo_waits_last(BlendParams& bp) {
    if (bp.wait_flags == nullptr || bp.own_r_hi <= bp.own_r_lo || bp.py_count <= 0) return;
    int first_wait = -1, last_wait = -1;
    for (int by = bp.py0; by < bp.py0 + bp.py_count; ++by) {
        const int lo = bp.prow_lo[by], n = bp.prow_n[by];
        if (n > 0 && (lo < bp.own_r_lo || lo + n > bp.own_r_hi)) { if (first_wait < 0) first_wait = by; last_wait = by; }
    }
    const int mid2 = 2 * bp.py0 + bp.py_count - 1;      // 2 x centre of the range
    bp.sched = (first_wait >= 0 && first_wait + last_wait <= mid2) ? 2 : 1;
}

template <typename T, bool WRITE_BUF, bool SPARSE>
int launch_blend_async(const td_grid* g, const BlendParams& bp_in, const float* weights, const float* rcp_weights, float* out_f32,
                       void* out_buf, int nv_cap, bool pipelined, bool pdl, int max_ppc, cudaStream_t st, const int* slot) {
    constexpr int VEC = Vec<T>::kElems;
    constexpr int BX = kAsX * VEC;
    BlendParams bp = bp_in;
    fill_patch_table(g->ys, g->rows, g->tile_h, g->H, kAsY, bp.prow_lo, bp.prow_n);
    fill_patch_table(g->xs, g->cols, g->tile_w, g->W, BX, bp.pcol_lo, bp.pcol_n);
    if (!pipelined) schedule_halo_waits_last(bp);
    if (rcp_weights != nullptr && sizeof(T) == 2)
        return launch_blend_async_impl<T, WRITE_BUF, true, SPARSE>(bp, weights, rcp_weights, out_f32, out_buf, nv_cap, pipelined, pdl,
                                                                   max_ppc, st, slot);
    return launch_blend_async_impl<T, WRITE_BUF, false, SPARSE>(bp, weights, nullptr, out_f32, out_buf, nv_cap, pipelined, pdl, max_ppc, st,
                                                                slot);
}

template <typename T, bool WINDOW, bool SPARSE = false>
int launch_blend_mod_async(const BlendParams& bp, int smem, const float* tile_weights, const float* rescale, void* out_buf, bool pdl,
                           cudaStream_t st, const int* slot = nullptr) {
    constexpr int BX = kAsX * Vec<T>::kElems;
    const char* what = "td_blend_mixture (cp.async)";
    int rc = smem_optin(blend_mod_async_kernel<T, WINDOW, SPARSE>, smem, what);
    if (rc != TD_OK) return rc;
    const unsigned gy = (unsigned)(WINDOW ? bp.py_count : (bp.g.H + kAsY - 1) / kAsY), gz = (unsigned)(bp.g.N * bp.g.C);
    dim3 grid((unsigned)((bp.g.W + BX - 1) / BX), bp.sched ? gz : gy, bp.sched ? gy : gz);
    return launch(what, blend_mod_async_kernel<T, WINDOW, SPARSE>, grid, dim3(kAsThreads), (size_t)smem, st, pdl, bp, tile_weights, rescale,
                  (T*)out_buf, slot);
}

// Mixture of Diffusers on the cp.async kernel; 0 launched, 1 not applicable, <0 error
template <typename T, bool SPARSE = false>
int try_launch_blend_mod_async(const td_grid* g, const BlendParams& bp_in, const float* tile_weights, const float* rescale, void* out_buf,
                               bool pdl, cudaStream_t st, const int* slot = nullptr) {
    constexpr int VEC = Vec<T>::kElems;
    constexpr int BX = kAsX * VEC;
    if (bp_in.g.N * bp_in.g.C > 65535 || (bp_in.g.H + kAsY - 1) / kAsY > 65535 || bp_in.tile_stride >= (1ll << 31)) return 1;
    if ((bp_in.g.H + kAsY - 1) / kAsY > TD_MAX_GRID_DIM || (bp_in.g.W + BX - 1) / BX > TD_MAX_GRID_DIM) return 1;
    if (!aligned16(tile_weights) || (bp_in.g.tw & 7) != 0) return 1;
    const int nv_cap = max_union(g->ys, g->rows, g->tile_h, g->H, kAsY) * max_union(g->xs, g->cols, g->tile_w, g->W, BX);
    if (nv_cap <= 0 || nv_cap > kAsMaxVisits || nv_cap > kAsThreads || nv_cap * kAsStage > 200 * 1024) return 1;
    BlendParams bp = bp_in;
    fill_patch_table(g->ys, g->rows, g->tile_h, g->H, kAsY, bp.prow_lo, bp.prow_n);
    fill_patch_table(g->xs, g->cols, g->tile_w, g->W, BX, bp.pcol_lo, bp.pcol_n);
    schedule_halo_waits_last(bp);
    if constexpr (SPARSE) return launch_blend_mod_async<T, false, true>(bp, nv_cap * kAsStage, tile_weights, rescale, out_buf, pdl, st, slot);
    return bp.py_count > 0 ? launch_blend_mod_async<T, true>(bp, nv_cap * kAsStage, tile_weights, rescale, out_buf, pdl, st)
                           : launch_blend_mod_async<T, false>(bp, nv_cap * kAsStage, tile_weights, rescale, out_buf, pdl, st);
}

// returns TD_OK if launched, 1 if the path does not apply (caller falls back), <0 on error
template <typename T, bool SPARSE = false>
int try_launch_blend_async(const td_grid* g, const BlendParams& bp, const float* weights, const float* rcp_weights, float* out_f32,
                           void* out_buf, bool pipelined, bool pdl, int max_ppc, cudaStream_t st, const int* slot = nullptr) {
    constexpr int VEC = Vec<T>::kElems;
    constexpr int BX = kAsX * VEC;
    if (bp.g.N * bp.g.C > 65535 || (bp.g.H + kAsY - 1) / kAsY > 65535) return 1;
    if (bp.tile_stride >= (1ll << 31)) return 1;
    const int nv_cap = max_union(g->ys, g->rows, g->tile_h, g->H, kAsY) * max_union(g->xs, g->cols, g->tile_w, g->W, BX);
    if (nv_cap <= 0 || nv_cap > kAsMaxVisits || nv_cap > kAsThreads || nv_cap * kAsStage > 200 * 1024) return 1;
    if ((bp.g.H + kAsY - 1) / kAsY > TD_MAX_GRID_DIM || (bp.g.W + BX - 1) / BX > TD_MAX_GRID_DIM) return 1;   // patch tables
    if (pipelined && 2 * nv_cap * kAsStage > 200 * 1024) pipelined = false;
    return out_buf != nullptr
               ? launch_blend_async<T, true, SPARSE>(g, bp, weights, rcp_weights, out_f32, out_buf, nv_cap, pipelined, pdl, max_ppc, st, slot)
               : launch_blend_async<T, false, SPARSE>(g, bp, weights, rcp_weights, out_f32, out_buf, nv_cap, pipelined, pdl, max_ppc, st, slot);
}

template <typename TIn, typename TAcc, int MODE, bool SPARSE>
int launch_blend_generic(const BlendParams& bp, const float* weights, const float* tile_weights, const float* rescale,
                         float* out_f32, void* out_buf, cudaStream_t st, const int* slot) {
    const GeomParams& g = bp.g;
    const long long total = (long long)g.N * g.C * g.H * g.W;
    blend_grid_generic_kernel<TIn, TAcc, MODE, SPARSE><<<blocks_for(total, 256), 256, 0, st>>>(bp, weights, tile_weights, rescale,
                                                                                               out_f32, (TAcc*)out_buf, total, slot);
    return launch_status("td_blend (generic)");
}

template <int MODE, bool SPARSE = false>
int dispatch_generic(int tile_dtype, int acc_dtype, const BlendParams& bp, const float* w, const float* tw, const float* rs,
                     float* out_f32, void* out_buf, cudaStream_t st, const int* slot = nullptr) {
#define TD_CASE(TI, TA, TIn, TAcc) \
    if (tile_dtype == TI && acc_dtype == TA) return launch_blend_generic<TIn, TAcc, MODE, SPARSE>(bp, w, tw, rs, out_f32, out_buf, st, slot);
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

// n_tiles: the tiles the batch table holds, the whole plan's by default (the sparse entries: the active tiles, possibly none -- then
// num_batches is 0 and batch_ptrs may be null)
int fill_blend(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int tile_dtype,
               int acc_dtype, BlendParams* bp, int n_tiles = -1) {
    int st = fill_geom(g, N, C, &bp->g);
    if (st != TD_OK) return st;
    if (n_tiles < 0) n_tiles = g->num_tiles;
    if (td_dtype_size(tile_dtype) == 0 || td_dtype_size(acc_dtype) == 0) { td_set_error("unknown dtype"); return TD_ERR_INVALID_ARG; }
    if (n_tiles == 0 ? (num_batches != 0 || tile_bs <= 0) : (batch_ptrs == nullptr || num_batches <= 0 || tile_bs <= 0)) {
        td_set_error("bad batch pointer table");
        return TD_ERR_INVALID_ARG;
    }
    if (num_batches > TD_MAX_BATCH_PTRS) {
        td_set_error("%d batch tensors exceed TD_MAX_BATCH_PTRS=%d (concatenate them first)", num_batches, TD_MAX_BATCH_PTRS);
        return TD_ERR_UNSUPPORTED;
    }
    if ((long long)num_batches * tile_bs < n_tiles || (num_batches > 0 && (long long)(num_batches - 1) * tile_bs >= n_tiles)) {
        td_set_error("batch table (%d x %d) does not cover %d tiles exactly", num_batches, tile_bs, n_tiles);
        return TD_ERR_INVALID_ARG;
    }
    for (int b = 0; b < num_batches; ++b) {
        if (batch_ptrs[b] == nullptr) { td_set_error("batch_ptrs[%d] is null", b); return TD_ERR_INVALID_ARG; }
        bp->batch_ptrs[b] = batch_ptrs[b];
    }
    bp->tile_bs = tile_bs;
    bp->wait_flags = nullptr; bp->wait_world = 0; bp->wait_value = nullptr;
    bp->py0 = 0; bp->py_count = 0;
    bp->own_r_lo = 0; bp->own_r_hi = 0; bp->sched = 0;
    bp->bs_magic = magic_u16((unsigned)tile_bs);
    bp->num_batches = num_batches;
    bp->tile_stride = (long long)N * C * g->tile_h * g->tile_w;
    return TD_OK;
}

// A periodic plan runs on td_wrap.cu, which has one form per operation: the opt-in forms of this file (ROWS / STRIP /
// TMA / PIPELINE), the peer blend and the row-strip blend do not take one.
int refuse_wrapped(const td_grid* g, const char* what) {
    if (g->wrap != 0) {
        td_set_error("%s: no form for a periodic plan (wrap=%d)", what, g->wrap);
        return TD_ERR_UNSUPPORTED;
    }
    return TD_OK;
}

bool blend_vec_ok(const BlendParams& bp, int tile_dtype, int acc_dtype, std::initializer_list<const void*> ptrs) {
    if (tile_dtype != acc_dtype) return false;
    if (bp.tile_stride >= (1ll << 31)) return false;  // the vector kernel uses 32-bit offsets inside a tile
    const int vec = 16 / td_dtype_size(tile_dtype);
    if (bp.g.W % vec != 0 || bp.g.tw % vec != 0) return false;
    for (int b = 0; b < bp.num_batches; ++b)
        if (!aligned16(bp.batch_ptrs[b])) return false;
    for (const void* p : ptrs)
        if (p != nullptr && !aligned16(p)) return false;
    return true;
}

}  // namespace

__global__ void empty_kernel() {}

extern "C" int td_debug_launch_empty(int blocks, int threads, void* stream) {
    if (blocks <= 0 || threads <= 0 || threads > 1024) { td_set_error("td_debug_launch_empty: bad launch shape"); return TD_ERR_INVALID_ARG; }
    empty_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>();
    return launch_status("td_debug_launch_empty");
}

extern "C" int td_scatter_tiles(const td_grid* g, const void* x, void* tiles, int N, int C, int dtype, int tile_begin,
                                int tile_end, uint32_t flags, void* stream) {
    GeomParams gp;
    int st = fill_geom(g, N, C, &gp);
    if (st != TD_OK) return st;
    if ((flags & kOptInForms) && (st = refuse_wrapped(g, "td_scatter_tiles")) != TD_OK) return st;
    if (tile_begin < 0 || tile_end < tile_begin || tile_end > g->num_tiles) {
        td_set_error("td_scatter_tiles: tile range [%d,%d) outside [0,%d)", tile_begin, tile_end, g->num_tiles);
        return TD_ERR_INVALID_ARG;
    }
    const int es = td_dtype_size(dtype);
    if (es == 0) { td_set_error("td_scatter_tiles: unknown dtype %d", dtype); return TD_ERR_INVALID_ARG; }
    if (tile_begin == tile_end) return TD_OK;   // an empty range (a shard without tiles) launches nothing: its output may be empty
    if (x == nullptr || tiles == nullptr) { td_set_error("td_scatter_tiles: null tensor"); return TD_ERR_INVALID_ARG; }
    const int vec = 16 / es;
    const bool pdl = !(flags & TD_FLAG_NO_PDL);
    const bool vec_ok = !(flags & TD_FLAG_FORCE_GENERIC) && gp.W % vec == 0 && gp.tw % vec == 0 && aligned16(x) && aligned16(tiles);
    if (g->wrap) return td_wrap_scatter(g, x, tiles, N, C, dtype, tile_begin, tile_end, vec_ok, pdl, stream);
    cudaStream_t s = (cudaStream_t)stream;
    if (vec_ok && !(flags & TD_FLAG_NO_TMA)) {   // default: row-block form (td_rows.cu); falls through when not applicable
        const int rc = td_rows_try_launch_scatter(g, x, tiles, N, C, dtype, tile_begin, tile_end, (flags & TD_FLAG_NO_PDL) ? 0 : 1, stream);
        if (rc <= 0) return rc;
    }
    // fp16 and bf16 are both moved as opaque 16-bit words
    if (es == 2) return launch_scatter<__half>(gp, x, tiles, tile_begin, tile_end - tile_begin, vec_ok, pdl, s);
    return launch_scatter<float>(gp, x, tiles, tile_begin, tile_end - tile_begin, vec_ok, pdl, s);
}

extern "C" int td_blend_multidiffusion(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N,
                                       int C, int tile_dtype, int acc_dtype, const float* weights, const float* rcp_weights,
                                       float* x_out, void* x_buffer, uint32_t flags, void* stream) {
    BlendParams bp;
    const bool pdl = !(flags & TD_FLAG_NO_PDL);
    int st = fill_blend(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, acc_dtype, &bp);
    if (st != TD_OK) return st;
    if (weights == nullptr || x_out == nullptr) { td_set_error("td_blend_multidiffusion: null weights / x_out"); return TD_ERR_INVALID_ARG; }
    if ((flags & kOptInForms) && (st = refuse_wrapped(g, "td_blend_multidiffusion")) != TD_OK) return st;
    const bool vec_ok = !(flags & TD_FLAG_FORCE_GENERIC) && blend_vec_ok(bp, tile_dtype, acc_dtype, {weights, rcp_weights, x_out, x_buffer});
    if (g->wrap)
        return td_wrap_blend(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, acc_dtype, 0, weights, nullptr, nullptr, x_out, x_buffer,
                             vec_ok, pdl, stream);
    bp.g.dbg_no_tiles = (flags & TD_FLAG_DBG_NO_TILES) ? 1 : 0;
    cudaStream_t s = (cudaStream_t)stream;
    if (vec_ok) {
        int rc = 1;
        if (flags & TD_FLAG_ROWS) {
            // opt-in: row-block form (td_rows.cu); falls through to the default kernels when not applicable
            rc = td_rows_try_launch_md(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, weights, rcp_weights, x_out, x_buffer,
                                       (flags & TD_FLAG_NO_PDL) ? 0 : 1, (flags & TD_FLAG_DBG_NO_TILES) ? 1 : 0, stream);
            if (rc <= 0) return rc;
        }
        if (flags & TD_FLAG_STRIP) {   // opt-in: strip form (td_strip.cu); falls through to the default when not applicable
            rc = td_strip_try_launch(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, weights, rcp_weights, x_out, x_buffer,
                                     (flags & TD_FLAG_NO_PDL) ? 0 : 1, (flags & TD_FLAG_ONE_PLANE) ? 1 : 2, stream);
            if (rc <= 0) return rc;
        }
        if (flags & TD_FLAG_TMA) {
            switch (tile_dtype) {
                case TD_F16: rc = try_launch_blend_tma<__half>(g, bp, tile_dtype, weights, x_out, x_buffer, s); break;
                case TD_BF16: rc = try_launch_blend_tma<__nv_bfloat16>(g, bp, tile_dtype, weights, x_out, x_buffer, s); break;
                default: rc = try_launch_blend_tma<float>(g, bp, tile_dtype, weights, x_out, x_buffer, s); break;
            }
        } else if (!(flags & TD_FLAG_NO_TMA)) {
            const bool pipe = (flags & TD_FLAG_PIPELINE) != 0;   // opt-in (see the comment above the kernel)
            switch (tile_dtype) {
                case TD_F16: rc = try_launch_blend_async<__half>(g, bp, weights, rcp_weights, x_out, x_buffer, pipe, pdl, ppc_max(flags), s); break;
                case TD_BF16: rc = try_launch_blend_async<__nv_bfloat16>(g, bp, weights, rcp_weights, x_out, x_buffer, pipe, pdl, ppc_max(flags), s); break;
                default: rc = try_launch_blend_async<float>(g, bp, weights, nullptr, x_out, x_buffer, pipe, pdl, ppc_max(flags), s); break;
            }
        }
        if (rc <= 0) return rc;   // launched or hard error; 1 = not applicable -> register-staged kernel
        switch (tile_dtype) {
            case TD_F16: return launch_blend_vec<__half, MODE_MD>(bp, weights, nullptr, nullptr, x_out, x_buffer, s);
            case TD_BF16: return launch_blend_vec<__nv_bfloat16, MODE_MD>(bp, weights, nullptr, nullptr, x_out, x_buffer, s);
            default: return launch_blend_vec<float, MODE_MD>(bp, weights, nullptr, nullptr, x_out, x_buffer, s);
        }
    }
    return dispatch_generic<MODE_MD>(tile_dtype, acc_dtype, bp, weights, nullptr, nullptr, x_out, x_buffer, s);
}

// The row window and the halo wait of a rows blend (td_blend_multidiffusion_rows / td_blend_mixture_rows), checked and set in
// bp.  `ptrs`: the buffers the vector path needs 16-byte aligned.  Returns TD_OK to launch, 1 for an empty window (nothing to
// launch), or a td_status.
static int setup_rows_window(const td_grid* g, BlendParams* bp, const char* what, int tile_dtype, int acc_dtype,
                             std::initializer_list<const void*> ptrs, int row_begin, int row_end, const uint32_t* wait_flags,
                             int wait_count, const uint32_t* wait_value, int own_band_begin, int own_band_end, int patch_rows = kAsY) {
    if (row_begin < 0 || row_end > g->H || row_begin > row_end || row_begin % 8 != 0 || (row_end % 8 != 0 && row_end != g->H)) {
        td_set_error("%s: rows [%d,%d) must lie in [0,%d) on multiples of 8", what, row_begin, row_end, g->H);
        return TD_ERR_INVALID_ARG;
    }
    if (wait_count < 0 || wait_count > TD_MAX_PEERS || (wait_count > 0 && (wait_flags == nullptr || wait_value == nullptr))) {
        td_set_error("%s: bad wait table", what);
        return TD_ERR_INVALID_ARG;
    }
    if (row_begin == row_end) return 1;
    if (!blend_vec_ok(*bp, tile_dtype, acc_dtype, ptrs)) {
        td_set_error("%s: needs the vector path (same tile / canvas dtype, W and tile_w multiples of the vector, 16-byte aligned buffers)", what);
        return TD_ERR_UNSUPPORTED;
    }
    // the window is cut into whole patch rows of the kernel (cp.async: kAsY rows, a build-time knob; 8 by default)
    if (row_begin % patch_rows != 0 || (row_end % patch_rows != 0 && row_end != g->H)) {
        td_set_error("%s: rows [%d,%d) are not aligned to the %d-row patches of this build", what, row_begin, row_end, patch_rows);
        return TD_ERR_UNSUPPORTED;
    }
    bp->py0 = row_begin / kAsY;
    bp->py_count = (row_end - row_begin + kAsY - 1) / kAsY;
    if (wait_count > 0) { bp->wait_flags = wait_flags; bp->wait_world = wait_count; bp->wait_value = wait_value; }
    if (own_band_begin < 0 || own_band_end > g->rows || own_band_begin > own_band_end) {
        td_set_error("%s: own bands [%d,%d) outside the %d tile rows", what, own_band_begin, own_band_end, g->rows);
        return TD_ERR_INVALID_ARG;
    }
    if (wait_count > 0 && own_band_end > own_band_begin) { bp->own_r_lo = own_band_begin; bp->own_r_hi = own_band_end; }   // -> schedule_halo_waits_last
    return TD_OK;
}

extern "C" int td_blend_multidiffusion_rows(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N,
                                            int C, int tile_dtype, int acc_dtype, const float* weights, const float* rcp_weights,
                                            float* x_out, void* x_buffer, int row_begin, int row_end, const uint32_t* wait_flags,
                                            int wait_count, const uint32_t* wait_value, int own_band_begin, int own_band_end,
                                            uint32_t flags, void* stream) {
    BlendParams bp;
    const bool pdl = !(flags & TD_FLAG_NO_PDL);
    int st = fill_blend(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, acc_dtype, &bp);
    if (st != TD_OK) return st;
    if ((st = refuse_wrapped(g, "td_blend_multidiffusion_rows")) != TD_OK) return st;
    if (weights == nullptr || x_out == nullptr) { td_set_error("td_blend_multidiffusion_rows: null weights / x_out"); return TD_ERR_INVALID_ARG; }
    st = setup_rows_window(g, &bp, "td_blend_multidiffusion_rows", tile_dtype, acc_dtype, {weights, rcp_weights, x_out, x_buffer}, row_begin,
                           row_end, wait_flags, wait_count, wait_value, own_band_begin, own_band_end);
    if (st != TD_OK) return st == 1 ? TD_OK : st;
    cudaStream_t s = (cudaStream_t)stream;
    int rc;
    switch (tile_dtype) {
        case TD_F16: rc = try_launch_blend_async<__half>(g, bp, weights, rcp_weights, x_out, x_buffer, false, pdl, ppc_max(flags), s); break;
        case TD_BF16: rc = try_launch_blend_async<__nv_bfloat16>(g, bp, weights, rcp_weights, x_out, x_buffer, false, pdl, ppc_max(flags), s); break;
        default: rc = try_launch_blend_async<float>(g, bp, weights, nullptr, x_out, x_buffer, false, pdl, ppc_max(flags), s); break;
    }
    if (rc == 1) { td_set_error("td_blend_multidiffusion_rows: geometry outside the cp.async kernel's limits"); return TD_ERR_UNSUPPORTED; }
    return rc;
}

extern "C" int td_debug_check_fast_div(int dtype, int max_w, unsigned long long* mismatches_dev, void* stream) {
    if (mismatches_dev == nullptr || max_w < 1 || (dtype != TD_F16 && dtype != TD_BF16)) {
        td_set_error("td_debug_check_fast_div: bad arguments");
        return TD_ERR_INVALID_ARG;
    }
    if (dtype == TD_F16) check_fast_div_kernel<__half><<<256, 256, 0, (cudaStream_t)stream>>>(max_w, mismatches_dev);
    else check_fast_div_kernel<__nv_bfloat16><<<256, 256, 0, (cudaStream_t)stream>>>(max_w, mismatches_dev);
    return launch_status("td_debug_check_fast_div");
}

extern "C" int td_blend_multidiffusion_peer(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N,
                                            int C, int tile_dtype, int acc_dtype, const float* weights, float* x_out,
                                            void* x_buffer, const uint32_t* wait_flags, int world, const uint32_t* wait_value,
                                            uint32_t flags, void* stream) {
    BlendParams bp;
    const bool pdl = !(flags & TD_FLAG_NO_PDL);
    int st = fill_blend(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, acc_dtype, &bp);
    if (st != TD_OK) return st;
    if ((st = refuse_wrapped(g, "td_blend_multidiffusion_peer")) != TD_OK) return st;
    if (weights == nullptr || x_out == nullptr) { td_set_error("td_blend_multidiffusion_peer: null weights / x_out"); return TD_ERR_INVALID_ARG; }
    if (wait_flags == nullptr || wait_value == nullptr || world <= 0 || world > TD_MAX_PEERS) { td_set_error("td_blend_multidiffusion_peer: bad wait table"); return TD_ERR_INVALID_ARG; }
    if (!blend_vec_ok(bp, tile_dtype, acc_dtype, {weights, x_out, x_buffer})) {
        td_set_error("td_blend_multidiffusion_peer: needs the vector path (same tile / canvas dtype, W and tile_w multiples of the vector, 16-byte aligned buffers)");
        return TD_ERR_UNSUPPORTED;
    }
    bp.wait_flags = wait_flags; bp.wait_world = world; bp.wait_value = wait_value;
    cudaStream_t s = (cudaStream_t)stream;
    if (flags & TD_FLAG_PEER_ASYNC) {   // cp.async-staged kernel over peer pointers: measured slower over NVLink than direct loads (opt-in)
        int rc;
        switch (tile_dtype) {
            case TD_F16: rc = try_launch_blend_async<__half>(g, bp, weights, nullptr, x_out, x_buffer, false, pdl, ppc_max(flags), s); break;
            case TD_BF16: rc = try_launch_blend_async<__nv_bfloat16>(g, bp, weights, nullptr, x_out, x_buffer, false, pdl, ppc_max(flags), s); break;
            default: rc = try_launch_blend_async<float>(g, bp, weights, nullptr, x_out, x_buffer, false, pdl, ppc_max(flags), s); break;
        }
        if (rc <= 0) return rc;
    }
    switch (tile_dtype) {
        case TD_F16: return launch_blend_vec<__half, MODE_MD>(bp, weights, nullptr, nullptr, x_out, x_buffer, s);
        case TD_BF16: return launch_blend_vec<__nv_bfloat16, MODE_MD>(bp, weights, nullptr, nullptr, x_out, x_buffer, s);
        default: return launch_blend_vec<float, MODE_MD>(bp, weights, nullptr, nullptr, x_out, x_buffer, s);
    }
}

extern "C" int td_blend_mixture(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C,
                                int tile_dtype, int acc_dtype, const float* tile_weights, const float* rescale,
                                void* x_buffer, uint32_t flags, void* stream) {
    BlendParams bp;
    const bool pdl = !(flags & TD_FLAG_NO_PDL);
    int st = fill_blend(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, acc_dtype, &bp);
    if (st != TD_OK) return st;
    if (tile_weights == nullptr || rescale == nullptr || x_buffer == nullptr) {
        td_set_error("td_blend_mixture: null tile_weights / rescale / x_buffer");
        return TD_ERR_INVALID_ARG;
    }
    if ((flags & kOptInForms) && (st = refuse_wrapped(g, "td_blend_mixture")) != TD_OK) return st;
    const bool vec_ok = !(flags & TD_FLAG_FORCE_GENERIC) && blend_vec_ok(bp, tile_dtype, acc_dtype, {rescale, x_buffer});
    if (g->wrap)
        return td_wrap_blend(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, acc_dtype, 1, nullptr, tile_weights, rescale, nullptr,
                             x_buffer, vec_ok, pdl, stream);
    cudaStream_t s = (cudaStream_t)stream;
    if (vec_ok) {
        if (flags & TD_FLAG_ROWS) {   // opt-in: row-block form (td_rows.cu)
            const int rc = td_rows_try_launch_mod(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, tile_weights, rescale, x_buffer,
                                                  (flags & TD_FLAG_NO_PDL) ? 0 : 1, stream);
            if (rc <= 0) return rc;
        }
        if (flags & TD_FLAG_STRIP) {   // opt-in: strip form (td_strip.cu); falls through to the default when not applicable
            const int rc = td_strip_try_launch_mod(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, tile_weights, rescale, x_buffer,
                                                   (flags & TD_FLAG_NO_PDL) ? 0 : 1, stream);
            if (rc <= 0) return rc;
        }
        if (!(flags & TD_FLAG_NO_TMA)) {
            int rc;
            switch (tile_dtype) {
                case TD_F16: rc = try_launch_blend_mod_async<__half>(g, bp, tile_weights, rescale, x_buffer, pdl, s); break;
                case TD_BF16: rc = try_launch_blend_mod_async<__nv_bfloat16>(g, bp, tile_weights, rescale, x_buffer, pdl, s); break;
                default: rc = try_launch_blend_mod_async<float>(g, bp, tile_weights, rescale, x_buffer, pdl, s); break;
            }
            if (rc <= 0) return rc;   // launched or hard error; 1 = not applicable -> register-staged kernel
        }
        switch (tile_dtype) {
            case TD_F16: return launch_blend_vec<__half, MODE_MOD>(bp, nullptr, tile_weights, rescale, nullptr, x_buffer, s);
            case TD_BF16: return launch_blend_vec<__nv_bfloat16, MODE_MOD>(bp, nullptr, tile_weights, rescale, nullptr, x_buffer, s);
            default: return launch_blend_vec<float, MODE_MOD>(bp, nullptr, tile_weights, rescale, nullptr, x_buffer, s);
        }
    }
    return dispatch_generic<MODE_MOD>(tile_dtype, acc_dtype, bp, nullptr, tile_weights, rescale, nullptr, x_buffer, s);
}

extern "C" int td_blend_mixture_rows(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C,
                                     int tile_dtype, int acc_dtype, const float* tile_weights, const float* rescale, void* x_buffer,
                                     int row_begin, int row_end, const uint32_t* wait_flags, int wait_count, const uint32_t* wait_value,
                                     int own_band_begin, int own_band_end, uint32_t flags, void* stream) {
    BlendParams bp;
    const bool pdl = !(flags & TD_FLAG_NO_PDL);
    int st = fill_blend(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, acc_dtype, &bp);
    if (st != TD_OK) return st;
    if ((st = refuse_wrapped(g, "td_blend_mixture_rows")) != TD_OK) return st;
    if (tile_weights == nullptr || rescale == nullptr || x_buffer == nullptr) {
        td_set_error("td_blend_mixture_rows: null tile_weights / rescale / x_buffer");
        return TD_ERR_INVALID_ARG;
    }
    st = setup_rows_window(g, &bp, "td_blend_mixture_rows", tile_dtype, acc_dtype, {tile_weights, rescale, x_buffer}, row_begin, row_end,
                           wait_flags, wait_count, wait_value, own_band_begin, own_band_end);
    if (st != TD_OK) return st == 1 ? TD_OK : st;
    cudaStream_t s = (cudaStream_t)stream;
    int rc;
    switch (tile_dtype) {
        case TD_F16: rc = try_launch_blend_mod_async<__half>(g, bp, tile_weights, rescale, x_buffer, pdl, s); break;
        case TD_BF16: rc = try_launch_blend_mod_async<__nv_bfloat16>(g, bp, tile_weights, rescale, x_buffer, pdl, s); break;
        default: rc = try_launch_blend_mod_async<float>(g, bp, tile_weights, rescale, x_buffer, pdl, s); break;
    }
    if (rc == 1) { td_set_error("td_blend_mixture_rows: geometry outside the cp.async kernel's limits"); return TD_ERR_UNSUPPORTED; }
    return rc;
}

// Row-strip shard on a periodic canvas (td_wrap.cu): the windowed wrap blends, validated as the rows entries above.  A bounded
// plan keeps td_blend_*_rows.
static int wrap_rows_entry(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int tile_dtype,
                           int acc_dtype, int mixture, const float* weights, const float* tile_weights, const float* rescale, float* x_out,
                           void* x_buffer, int row_begin, int row_end, const uint32_t* wait_flags, int wait_count,
                           const uint32_t* wait_value, int own_band_begin, int own_band_end, uint32_t flags, void* stream, const char* what) {
    BlendParams bp;
    const bool pdl = !(flags & TD_FLAG_NO_PDL);
    int st = fill_blend(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, acc_dtype, &bp);
    if (st != TD_OK) return st;
    if (g->wrap == 0) {
        td_set_error("%s: a bounded plan (wrap=0) takes td_blend_%s_rows", what, mixture ? "mixture" : "multidiffusion");
        return TD_ERR_UNSUPPORTED;
    }
    if (mixture ? (tile_weights == nullptr || rescale == nullptr || x_buffer == nullptr) : (weights == nullptr || x_out == nullptr)) {
        td_set_error("%s: null %s", what, mixture ? "tile_weights / rescale / x_buffer" : "weights / x_out");
        return TD_ERR_INVALID_ARG;
    }
    // the wrap blend's CTAs cover 4 canvas rows: any window on multiples of 8 is whole CTA rows
    st = mixture ? setup_rows_window(g, &bp, what, tile_dtype, acc_dtype, {rescale, x_buffer}, row_begin, row_end, wait_flags, wait_count,
                                     wait_value, own_band_begin, own_band_end, 8)
                 : setup_rows_window(g, &bp, what, tile_dtype, acc_dtype, {weights, x_out, x_buffer}, row_begin, row_end, wait_flags,
                                     wait_count, wait_value, own_band_begin, own_band_end, 8);
    if (st != TD_OK) return st == 1 ? TD_OK : st;
    return td_wrap_blend_rows(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, mixture, weights, tile_weights, rescale, x_out, x_buffer,
                              row_begin, row_end, wait_count > 0 ? wait_flags : nullptr, wait_count, wait_value, own_band_begin,
                              own_band_end, pdl, stream);
}

extern "C" int td_blend_multidiffusion_wrap_rows(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C,
                                                 int tile_dtype, int acc_dtype, const float* weights, float* x_out, void* x_buffer,
                                                 int row_begin, int row_end, const uint32_t* wait_flags, int wait_count,
                                                 const uint32_t* wait_value, int own_band_begin, int own_band_end, uint32_t flags,
                                                 void* stream) {
    return wrap_rows_entry(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, acc_dtype, 0, weights, nullptr, nullptr, x_out, x_buffer,
                           row_begin, row_end, wait_flags, wait_count, wait_value, own_band_begin, own_band_end, flags, stream,
                           "td_blend_multidiffusion_wrap_rows");
}

extern "C" int td_blend_mixture_wrap_rows(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C,
                                          int tile_dtype, int acc_dtype, const float* tile_weights, const float* rescale, void* x_buffer,
                                          int row_begin, int row_end, const uint32_t* wait_flags, int wait_count, const uint32_t* wait_value,
                                          int own_band_begin, int own_band_end, uint32_t flags, void* stream) {
    return wrap_rows_entry(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, acc_dtype, 1, nullptr, tile_weights, rescale, nullptr,
                           x_buffer, row_begin, row_end, wait_flags, wait_count, wait_value, own_band_begin, own_band_end, flags, stream,
                           "td_blend_mixture_wrap_rows");
}

// ---------------------------------------------------------------------------
// Inpainting: the tiles an inpaint mask reaches, and the blends over the compact batches of those tiles only.
// ---------------------------------------------------------------------------
namespace {

// One CTA per tile: the tile is active when any element of its window, over all planes, is not exactly 1 (NaN included).
template <typename T>
__global__ void __launch_bounds__(256)
active_tiles_kernel(const __grid_constant__ GeomParams g, const T* __restrict__ mask, int planes, uint8_t* __restrict__ active) {
    const int t = blockIdx.x;
    const int r = t / g.cols, c = t - r * g.cols;
    const long long row0 = g.ys[r], col0 = g.xs[c];
    const long long n = (long long)planes * g.th * g.tw;
    int found = 0;
    for (long long i = threadIdx.x; i < n && !found; i += blockDim.x) {
        const long long pv = i / g.tw;                       // plane * th + v
        const long long pl = pv / g.th, v = pv - pl * g.th, u = i - pv * g.tw;
        found = !(Elem<T>::to_f32(mask[(pl * g.H + row0 + v) * g.W + col0 + u]) == 1.0f);
    }
    found = __syncthreads_or(found);
    if (threadIdx.x == 0) active[t] = found ? 1 : 0;
}

// The slot table of a sparse blend: n_slots == T, every entry -1 or a position in the compact batches, the positions 0 .. K-1
// each used exactly once (K = the tiles kept).  Checked on the host copy; the kernels read the device copy.
int check_slots(const td_grid* g, const int32_t* slot_dev, const int32_t* slot_host, int n_slots, const char* what, int* n_active) {
    if (g == nullptr) { td_set_error("%s: null grid", what); return TD_ERR_INVALID_ARG; }
    if (slot_dev == nullptr || slot_host == nullptr || ((uintptr_t)slot_dev & 3u) != 0) {
        td_set_error("%s: null or misaligned slot table", what);
        return TD_ERR_INVALID_ARG;
    }
    if (g->num_tiles <= 0 || n_slots != g->num_tiles) {
        td_set_error("%s: slot table of %d entries for a plan of %d tiles", what, n_slots, g->num_tiles);
        return TD_ERR_INVALID_ARG;
    }
    int k = 0;
    for (int t = 0; t < n_slots; ++t) k += slot_host[t] >= 0;
    std::vector<unsigned char> seen((size_t)k, 0);
    for (int t = 0; t < n_slots; ++t) {
        const int s = slot_host[t];
        if (s < -1 || s >= k || (s >= 0 && seen[(size_t)s])) {
            td_set_error("%s: slot[%d] = %d is not -1 or an unused position below %d", what, t, s, k);
            return TD_ERR_INVALID_ARG;
        }
        if (s >= 0) seen[(size_t)s] = 1;
    }
    *n_active = k;
    return TD_OK;
}

// the sparse entries have the default cp.async form and the generic one: other form flags are refused
constexpr uint32_t kSparseFlags = TD_FLAG_FORCE_GENERIC | TD_FLAG_NO_PDL | TD_FLAG_ONE_PLANE;

int sparse_common(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int tile_dtype,
                  int acc_dtype, const int32_t* slot_dev, const int32_t* slot_host, int n_slots, uint32_t flags, const char* what,
                  BlendParams* bp) {
    int k = 0;
    int st = check_slots(g, slot_dev, slot_host, n_slots, what, &k);
    if (st != TD_OK) return st;
    if ((st = fill_blend(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, acc_dtype, bp, k)) != TD_OK) return st;
    if (g->wrap != 0) { td_set_error("%s: no form for a periodic plan (wrap=%d)", what, g->wrap); return TD_ERR_UNSUPPORTED; }
    if (flags & ~kSparseFlags) { td_set_error("%s: flags %#x name a form this entry does not have", what, flags); return TD_ERR_INVALID_ARG; }
    return TD_OK;
}

}  // namespace

extern "C" int td_grid_active_tiles(const td_grid* g, const void* mask, int planes, int dtype, uint8_t* active_dev, void* stream) {
    GeomParams gp;
    int st = fill_geom(g, 1, 1, &gp);
    if (st != TD_OK) return st;
    if (g->wrap != 0) { td_set_error("td_grid_active_tiles: no form for a periodic plan (wrap=%d)", g->wrap); return TD_ERR_UNSUPPORTED; }
    const int es = td_dtype_size(dtype);
    if (es == 0) { td_set_error("td_grid_active_tiles: unknown dtype %d", dtype); return TD_ERR_INVALID_ARG; }
    if (planes <= 0) { td_set_error("td_grid_active_tiles: planes = %d must be positive", planes); return TD_ERR_INVALID_ARG; }
    if (mask == nullptr || active_dev == nullptr || ((uintptr_t)mask % (uintptr_t)es) != 0) {
        td_set_error("td_grid_active_tiles: null or misaligned mask / output");
        return TD_ERR_INVALID_ARG;
    }
    cudaStream_t s = (cudaStream_t)stream;
    switch (dtype) {
        case TD_F16: active_tiles_kernel<__half><<<g->num_tiles, 256, 0, s>>>(gp, (const __half*)mask, planes, active_dev); break;
        case TD_BF16: active_tiles_kernel<__nv_bfloat16><<<g->num_tiles, 256, 0, s>>>(gp, (const __nv_bfloat16*)mask, planes, active_dev); break;
        default: active_tiles_kernel<float><<<g->num_tiles, 256, 0, s>>>(gp, (const float*)mask, planes, active_dev); break;
    }
    return launch_status("td_grid_active_tiles");
}

extern "C" int td_blend_multidiffusion_sparse(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C,
                                              int tile_dtype, int acc_dtype, const float* weights, const float* rcp_weights, float* x_out,
                                              void* x_buffer, const int32_t* slot_dev, const int32_t* slot_host, int n_slots,
                                              uint32_t flags, void* stream) {
    const char* what = "td_blend_multidiffusion_sparse";
    BlendParams bp;
    int st = sparse_common(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, acc_dtype, slot_dev, slot_host, n_slots, flags, what, &bp);
    if (st != TD_OK) return st;
    if (weights == nullptr || x_out == nullptr) { td_set_error("%s: null weights / x_out", what); return TD_ERR_INVALID_ARG; }
    const bool pdl = !(flags & TD_FLAG_NO_PDL);
    cudaStream_t s = (cudaStream_t)stream;
    if (!(flags & TD_FLAG_FORCE_GENERIC) && blend_vec_ok(bp, tile_dtype, acc_dtype, {weights, rcp_weights, x_out, x_buffer})) {
        int rc;
        switch (tile_dtype) {
            case TD_F16: rc = try_launch_blend_async<__half, true>(g, bp, weights, rcp_weights, x_out, x_buffer, false, pdl, 1, s, slot_dev); break;
            case TD_BF16: rc = try_launch_blend_async<__nv_bfloat16, true>(g, bp, weights, rcp_weights, x_out, x_buffer, false, pdl, 1, s, slot_dev); break;
            default: rc = try_launch_blend_async<float, true>(g, bp, weights, nullptr, x_out, x_buffer, false, pdl, 1, s, slot_dev); break;
        }
        if (rc <= 0) return rc;   // launched or hard error; 1 = outside the cp.async kernel's limits -> generic kernel
    }
    return dispatch_generic<MODE_MD, true>(tile_dtype, acc_dtype, bp, weights, nullptr, nullptr, x_out, x_buffer, s, slot_dev);
}

extern "C" int td_blend_mixture_sparse(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C,
                                       int tile_dtype, int acc_dtype, const float* tile_weights, const float* rescale, void* x_buffer,
                                       const int32_t* slot_dev, const int32_t* slot_host, int n_slots, uint32_t flags, void* stream) {
    const char* what = "td_blend_mixture_sparse";
    BlendParams bp;
    int st = sparse_common(g, batch_ptrs, num_batches, tile_bs, N, C, tile_dtype, acc_dtype, slot_dev, slot_host, n_slots, flags, what, &bp);
    if (st != TD_OK) return st;
    if (tile_weights == nullptr || rescale == nullptr || x_buffer == nullptr) {
        td_set_error("%s: null tile_weights / rescale / x_buffer", what);
        return TD_ERR_INVALID_ARG;
    }
    const bool pdl = !(flags & TD_FLAG_NO_PDL);
    cudaStream_t s = (cudaStream_t)stream;
    if (!(flags & TD_FLAG_FORCE_GENERIC) && blend_vec_ok(bp, tile_dtype, acc_dtype, {rescale, x_buffer})) {
        int rc;
        switch (tile_dtype) {
            case TD_F16: rc = try_launch_blend_mod_async<__half, true>(g, bp, tile_weights, rescale, x_buffer, pdl, s, slot_dev); break;
            case TD_BF16: rc = try_launch_blend_mod_async<__nv_bfloat16, true>(g, bp, tile_weights, rescale, x_buffer, pdl, s, slot_dev); break;
            default: rc = try_launch_blend_mod_async<float, true>(g, bp, tile_weights, rescale, x_buffer, pdl, s, slot_dev); break;
        }
        if (rc <= 0) return rc;
    }
    return dispatch_generic<MODE_MOD, true>(tile_dtype, acc_dtype, bp, nullptr, tile_weights, rescale, nullptr, x_buffer, s, slot_dev);
}
