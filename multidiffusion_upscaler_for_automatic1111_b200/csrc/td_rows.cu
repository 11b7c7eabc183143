// Row-block form of the per-step hot path (TD_FLAG_ROWS, opt-in -- see the end of this comment):
//   scatter                       multidiffusion.py:155, mixtureofdiffusers.py:88,104
//   blend + normalise (MD)        multidiffusion.py:166-167, :208
//   blend (Mixture of Diffusers)  mixtureofdiffusers.py:122-126
// Same gather form and the same rounding sequence as the kernels in td_diffusion.cu (bit-identical results, same
// fixtures); what changes is how the bytes move.
//
// Why: the whole step moves ~20 MB, i.e. ~3 us of HBM time, so the kernels are latency- and launch-bound, not
// bandwidth-bound (round-1 ncu: 2 waves of 2048 small CTAs, every wave paying prologue -> DRAM latency -> consume ->
// store; 4.35 M warp instructions for 0.3 M essential ones).  Here
//   * ONE wave: one persistent CTA per SM; the canvas is cut into units (RC canvas rows of one (n, c) plane) and
//     every CTA owns a contiguous run of units;
//   * a tile plane [th, tw] is contiguous in the UNet's output, so the rows of a tile that overlap a unit are ONE
//     contiguous chunk: a unit's staging is ~20-30 `cp.async.bulk` copies (UBLKCP, 1-D TMA, no tensor map, no
//     zero fill, ~1.3 KB each) issued by one warp, completing on one mbarrier per unit.  All units of a CTA are in
//     flight before the first wait (4 x ~30 KB at BASELINE cfg2), so the HBM pipe is full ~1 us after launch;
//   * consume: one thread per 16-byte canvas vector -- the SAME (row slot, vector) in every unit, so the tile columns
//     touching it, their shifts and edge predicates are computed once per kernel -- walks the covering tiles in
//     ascending tile index: two aligned LDS.128 + funnel shift (tile columns are 2-byte-misaligned against the
//     canvas), packed add rounded through the canvas dtype; chunks outside the tile are register zeros (x + (+0) is
//     exact for MultiDiffusion; the Mixture-of-Diffusers form masks per element because its accumulator can be -0);
//     threads wait for a unit on the CTA barrier (one thread blocks on the mbarrier): no spinning issue slots;
//   * normalise in registers, 32 bytes stored per thread (fp32 output, as the reference).
// Scatter is the mirror image: one bulk copy brings a unit's canvas rows in, threads re-align and write 128-bit
// vectors into the tile batch.
//
// Bit-identical to the default kernels on every fixture, but a 200 KB one-CTA-per-SM kernel cannot become resident
// while its predecessor drains (no programmatic-dependent-launch overlap), pays the full launch -> barrier init -> copy
// latency -> consume -> store chain once per launch, and many small (1.3 KB, 16-byte-aligned) bulk copies per SM are a
// poor fit for the copy engine.  Kept as an opt-in for geometries with few, large tiles; the default is many small
// co-resident CTAs.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstring>

#include "td_b200.h"
#include "td_device.cuh"
#include "td_internal.h"
#include "td_launch.h"
#include "td_tma.cuh"

namespace {

using namespace td;

constexpr int kRowsThreads = 512;
constexpr int kRowsMaxSlots = 8;
constexpr int kRowsMaxSegs = 8;          // tile-row bands that can overlap one unit
constexpr int kRowsMaxVec = 512;         // canvas vectors per row (W / VEC)
constexpr int kRowsSmemBudget = 200 * 1024;

struct RowsParams {
    int H, W, th, tw, rows, cols, NC;
    int tile_bs, num_batches;
    int RC, nblocks, nunits;             // canvas rows per unit, row blocks per plane, units = nblocks * NC
    int slot_bytes, nslots;
    int wv, twv;                         // canvas / tile row length in vectors
    int tile_begin, tile_end;            // scatter: tile range of this call
    int dbg_no_tiles;
    int aux_bytes;                       // Mixture of Diffusers: bytes of the gaussian tile weights staged once per CTA
    long long tile_stride;               // elements of one tile: NC * th * tw
    short ys[TD_MAX_GRID_DIM], xs[TD_MAX_GRID_DIM];
    unsigned char vcol_lo[kRowsMaxVec], vcol_n[kRowsMaxVec];   // tile columns touching canvas vector i: first, count
    const void* batch_ptrs[TD_MAX_BATCH_PTRS];
};

struct SegTable {                        // geometry of the unit staged in one slot (written by the producer warp)
    int nseg, y0, nrows, plane;
    int band[kRowsMaxSegs], yy0[kRowsMaxSegs], nr[kRowsMaxSegs], off[kRowsMaxSegs];
};

// global -> shared bulk copy (1-D TMA): src, dst 16-byte aligned, bytes % 16 == 0; completes on `bar` (complete_tx)
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// 32 bytes per thread as two 128-bit accesses (sm_90 has no 256-bit load / store)
__device__ __forceinline__ void stg256(float* p, const float (&f)[8]) {
    asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(f[0]), "f"(f[1]), "f"(f[2]), "f"(f[3]) : "memory");
    asm volatile("st.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p + 4), "f"(f[4]), "f"(f[5]), "f"(f[6]), "f"(f[7]) : "memory");
}
__device__ __forceinline__ void ldg256(const float* p, float (&f)[8]) {
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(f[0]), "=f"(f[1]), "=f"(f[2]), "=f"(f[3]) : "l"(p));
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(f[4]), "=f"(f[5]), "=f"(f[6]), "=f"(f[7]) : "l"(p + 4));
}

// ---- producer: stage unit `u` into slot `slot` (called by all 32 lanes of warp 0) -----------------------------
// blend: the rows of every covering tile that overlap the unit; scatter (SCATTER): the unit's canvas rows.
template <typename T, bool SCATTER>
__device__ __forceinline__ void rows_issue(const RowsParams& p, int u, int slot, unsigned char* slots, SegTable* segs, uint64_t* full,
                                           const T* __restrict__ canvas) {
    const int lane = threadIdx.x & 31;
    const int b = u / p.NC, plane = u - b * p.NC;
    const int y0 = b * p.RC, y1 = min(p.H, y0 + p.RC);
    SegTable& sg = segs[slot];
    // bands (tile rows) overlapping [y0, y1): contiguous in i because ys is non-decreasing
    int lo = p.rows, cnt = 0;
    for (int base = 0; base < p.rows; base += 32) {
        const int i = base + lane;
        const bool hit = i < p.rows && (int)p.ys[i] < y1 && (int)p.ys[i] + p.th > y0;
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        if (m) {
            if (cnt == 0) lo = base + __ffs(m) - 1;
            cnt += __popc(m);
        }
    }
    if (p.dbg_no_tiles) cnt = 0;
    cnt = min(cnt, kRowsMaxSegs);
    const uint32_t row_bytes = (uint32_t)p.tw * (uint32_t)sizeof(T);
    uint32_t total = 0;
    if (lane == 0) {
        sg.nseg = cnt; sg.y0 = y0; sg.nrows = y1 - y0; sg.plane = plane;
        int off = 0;
        for (int k = 0; k < cnt; ++k) {
            const int i = lo + k;
            const int a = max(y0, (int)p.ys[i]), e = min(y1, (int)p.ys[i] + p.th);
            sg.band[k] = i; sg.yy0[k] = a; sg.nr[k] = e - a; sg.off[k] = off;
            off += (e - a) * p.cols * (int)row_bytes;
        }
        total = SCATTER ? (uint32_t)(y1 - y0) * (uint32_t)p.W * (uint32_t)sizeof(T) : (uint32_t)off;
        mbar_arrive_expect_tx(&full[slot], total);
    }
    __syncwarp();
    const uint32_t dst0 = smem_u32(slots) + (uint32_t)slot * (uint32_t)p.slot_bytes;
    if constexpr (SCATTER) {
        if (lane == 0) bulk_g2s(dst0, canvas + ((long long)plane * p.H + y0) * p.W, (uint32_t)(y1 - y0) * (uint32_t)p.W * (uint32_t)sizeof(T), &full[slot]);
    } else {
        const int ncopies = cnt * p.cols;
        for (int idx = lane; idx < ncopies; idx += 32) {
            const int k = idx / p.cols, j = idx - k * p.cols;
            const int i = sg.band[k], nr = sg.nr[k];
            const unsigned t = (unsigned)(i * p.cols + j);
            const unsigned bi = t / (unsigned)p.tile_bs;
            const long long elem = (long long)(t - bi * (unsigned)p.tile_bs) * p.tile_stride + ((long long)plane * p.th + (sg.yy0[k] - (int)p.ys[i])) * p.tw;
            const T* src = reinterpret_cast<const T*>(p.batch_ptrs[bi]) + elem;
            bulk_g2s(dst0 + (uint32_t)sg.off[k] + (uint32_t)(j * nr) * row_bytes, src, (uint32_t)nr * row_bytes, &full[slot]);
        }
    }
}

// ---- shared-memory access by 32-bit shared-window address (no generic -> shared conversion per access) ------------
__device__ __forceinline__ uint4 lds128_u32(uint32_t addr) {
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ float lds_f32_u32(uint32_t addr) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
    return v;
}

// Per-thread constants of one tile column touching the thread's canvas vector.  A thread owns the SAME (row slot, canvas
// vector) in every unit, so everything that depends on the column only is computed once per kernel:
//   elements [u0, u0 + VEC) of a tile row = aligned chunks A = [a, a + VEC), B = [a + VEC, a + 2 VEC), shift s = u0 - a;
//   a chunk outside [0, tw) is register zeros (x + (+0) is exact for MultiDiffusion; MoD masks per element).
struct ColRef {
    int j;        // tile column
    int aoff;     // byte offset of chunk A inside the tile row (may be -16)
    int s;        // shift in elements, [0, VEC)
    int va, vb;   // chunk A / B inside the tile
    int u0;       // tile column of element 0 (MoD)
};
constexpr int kRowsMaxCols = 4;   // tile columns touching one canvas vector on this path (rows_plan checks)

template <typename T>
__device__ __forceinline__ void rows_col_refs(const RowsParams& p, int xv, ColRef (&cr)[kRowsMaxCols], int& jn) {
    constexpr int VEC = Vec<T>::kElems;
    const int jlo = p.vcol_lo[xv];
    jn = p.vcol_n[xv];
#pragma unroll
    for (int c = 0; c < kRowsMaxCols; ++c) {
        const int j = min(jlo + c, p.cols - 1);
        const int u0 = xv * VEC - (int)p.xs[j];
        const int a = u0 & ~(VEC - 1);
        cr[c].j = j;
        cr[c].u0 = u0;
        cr[c].s = u0 - a;
        cr[c].aoff = a * (int)sizeof(T);
        cr[c].va = (a >= 0 && a < p.tw) ? 1 : 0;
        cr[c].vb = (cr[c].s != 0 && a + VEC < p.tw) ? 1 : 0;
    }
}

template <typename T>
__device__ __forceinline__ uint4 rows_visit(uint32_t row_addr, const ColRef& c) {
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
    const uint32_t addr = row_addr + (uint32_t)c.aoff;
    const uint4 A = c.va ? lds128_u32(addr) : z;
    if (c.s == 0) return A;
    const uint4 B = c.vb ? lds128_u32(addr + 16u) : z;
    return Vec<T>::window(A, B, c.s);
}

struct RowsCommon {
    int u_begin, u_end;
};

__device__ __forceinline__ RowsCommon rows_partition(const RowsParams& p) {
    RowsCommon c;
    c.u_begin = (int)((long long)p.nunits * blockIdx.x / gridDim.x);
    c.u_end = (int)((long long)p.nunits * (blockIdx.x + 1) / gridDim.x);
    return c;
}

// One thread blocks on the unit's mbarrier, the CTA barrier releases everyone else (warps parked on a hardware barrier
// issue nothing, a spinning try_wait loop does); every thread then takes its own (immediately successful) acquire.
__device__ __forceinline__ void rows_wait_unit(uint64_t* bar, uint32_t parity) {
    if (threadIdx.x == 0) mbar_wait(bar, parity);
    __syncthreads();
    while (!mbar_try_wait(bar, parity)) {}
}

// =================================================================================================================
// MultiDiffusion blend + normalise
// =================================================================================================================
template <typename T, bool WRITE_BUF, bool FASTDIV>
__global__ void __launch_bounds__(kRowsThreads, 1)
blend_rows_md_kernel(const __grid_constant__ RowsParams p, const float* __restrict__ weights, const float* __restrict__ rcp_weights,
                     float* __restrict__ out_f32, T* __restrict__ out_buf) {
    constexpr int VEC = Vec<T>::kElems;
    extern __shared__ __align__(128) unsigned char rows_smem[];
    __shared__ __align__(8) uint64_t full[kRowsMaxSlots];
    __shared__ SegTable segs[kRowsMaxSlots];
    const int tid = threadIdx.x;
    const RowsCommon c = rows_partition(p);
    const int n = c.u_end - c.u_begin;
    if (tid == 0) {
        for (int s = 0; s < p.nslots; ++s) mbar_init(&full[s], 1);
        fence_mbar_init();
        fence_proxy_async();
    }
    // this thread's (row slot, canvas vector) and the tile columns touching the vector: fixed for the whole kernel
    const int r = tid / p.wv, xv = tid - r * p.wv;
    const int x0 = xv * VEC;
    ColRef cr[kRowsMaxCols];
    int jn = 0;
    const bool worker = r < p.RC;
    if (worker) rows_col_refs<T>(p, xv, cr, jn);
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();
    if (tid < 32)
        for (int k = 0; k < min(n, p.nslots); ++k) rows_issue<T, false>(p, c.u_begin + k, k, rows_smem, segs, full, (const T*)nullptr);

    float wv[8], rv[8];     // weights of this thread's pixel vector, kept across the units of one row block
    int cached_b = -1;
    const uint32_t row_bytes = (uint32_t)p.tw * (uint32_t)sizeof(T);
    const uint32_t smem0 = smem_u32(rows_smem);
    for (int k = 0; k < n; ++k) {
        const int slot = k % p.nslots;
        const int u = c.u_begin + k;
        const int b = u / p.NC, plane = u - b * p.NC;
        const int y0 = b * p.RC, nrows = min(p.H, y0 + p.RC) - y0;
        const bool active = worker && r < nrows;
        if (active && b != cached_b) {      // fetched before blocking on the copies: the latency hides behind them
            const long long wo = (long long)(y0 + r) * p.W + x0;
            if constexpr (VEC == 8) {
                ldg256(weights + wo, wv);
                if constexpr (FASTDIV) ldg256(rcp_weights + wo, rv);
            } else {
                const float4 f = __ldg(reinterpret_cast<const float4*>(weights + wo));
                wv[0] = f.x; wv[1] = f.y; wv[2] = f.z; wv[3] = f.w;
            }
            cached_b = b;
        }
        rows_wait_unit(&full[slot], (uint32_t)((k / p.nslots) & 1));
        if (active) {
            const SegTable& sg = segs[slot];
            const uint32_t sbase = smem0 + (uint32_t)slot * (uint32_t)p.slot_bytes;
            const int y = y0 + r;
            uint4 acc = make_uint4(0u, 0u, 0u, 0u);
            const int nseg = sg.nseg;
            for (int q = 0; q < nseg; ++q) {
                const int rr = y - sg.yy0[q], nr = sg.nr[q];
                if ((unsigned)rr >= (unsigned)nr) continue;
                const uint32_t colstride = (uint32_t)nr * row_bytes;
                const uint32_t rowbase = sbase + (uint32_t)sg.off[q] + (uint32_t)rr * row_bytes;
#pragma unroll
                for (int cc = 0; cc < kRowsMaxCols; ++cc) {
                    if (cc < jn) {
                        const uint4 e = rows_visit<T>(rowbase + (uint32_t)cr[cc].j * colstride, cr[cc]);
                        acc.x = packed_add<T>(acc.x, e.x);
                        acc.y = packed_add<T>(acc.y, e.y);
                        acc.z = packed_add<T>(acc.z, e.z);
                        acc.w = packed_add<T>(acc.w, e.w);
                    }
                }
            }
            // x_out = where(weights > 1, x_buffer / weights, x_buffer): fp32, correctly rounded divide
            const long long o = ((long long)plane * p.H + y) * p.W + x0;
            float f[8];
#pragma unroll
            for (int j = 0; j < VEC; ++j) {
                const float a = Vec<T>::get(acc, j);
                if constexpr (FASTDIV) f[j] = wv[j] > 1.0f ? div_exact_small_int(a, wv[j], rv[j]) : a;
                else f[j] = wv[j] > 1.0f ? __fdiv_rn(a, wv[j]) : a;
            }
            if constexpr (VEC == 8) stg256(out_f32 + o, f);
            else *reinterpret_cast<float4*>(out_f32 + o) = make_float4(f[0], f[1], f[2], f[3]);
            if constexpr (WRITE_BUF) stg128(out_buf + o, acc);
        }
        if (k + p.nslots < n) {          // slot reuse: every thread is done reading it
            __syncthreads();
            if (tid < 32) rows_issue<T, false>(p, c.u_begin + k + p.nslots, slot, rows_smem, segs, full, (const T*)nullptr);
        }
    }
}

// =================================================================================================================
// Mixture of Diffusers blend: w = tile_w[v, u] * rescale[y, x]; acc = round_T(float(acc) + float(tile) * w)
// (separate fp32 multiply / multiply / add roundings, elements outside the tile untouched: the accumulator can be -0)
// =================================================================================================================
template <typename T>
__global__ void __launch_bounds__(kRowsThreads, 1)
blend_rows_mod_kernel(const __grid_constant__ RowsParams p, const float* __restrict__ tile_weights, const float* __restrict__ rescale,
                      T* __restrict__ out_buf) {
    constexpr int VEC = Vec<T>::kElems;
    extern __shared__ __align__(128) unsigned char rows_smem[];
    __shared__ __align__(8) uint64_t full[kRowsMaxSlots];
    __shared__ __align__(8) uint64_t aux_full;
    __shared__ SegTable segs[kRowsMaxSlots];
    __shared__ short s_ys[TD_MAX_GRID_DIM];
    const int tid = threadIdx.x;
    const RowsCommon c = rows_partition(p);
    const int n = c.u_end - c.u_begin;
    unsigned char* slots = rows_smem + p.aux_bytes;                         // [gaussian th x tw fp32][slots]
    if (tid == 0) {
        for (int s = 0; s < p.nslots; ++s) mbar_init(&full[s], 1);
        mbar_init(&aux_full, 1);
        fence_mbar_init();
        fence_proxy_async();
    }
    for (int i = tid; i < p.rows; i += kRowsThreads) s_ys[i] = p.ys[i];
    const int r = tid / p.wv, xv = tid - r * p.wv;
    const int x0 = xv * VEC;
    ColRef cr[kRowsMaxCols];
    int jn = 0;
    const bool worker = r < p.RC;
    if (worker) rows_col_refs<T>(p, xv, cr, jn);
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();
    if (tid < 32) {
        if (tid == 0) {
            mbar_arrive_expect_tx(&aux_full, (uint32_t)p.aux_bytes);
            bulk_g2s(smem_u32(rows_smem), tile_weights, (uint32_t)p.aux_bytes, &aux_full);
        }
        __syncwarp();
        for (int k = 0; k < min(n, p.nslots); ++k) rows_issue<T, false>(p, c.u_begin + k, k, slots, segs, full, (const T*)nullptr);
    }
    float rs[8];
    int cached_b = -1;
    const uint32_t row_bytes = (uint32_t)p.tw * (uint32_t)sizeof(T);
    const uint32_t smem_tw = smem_u32(rows_smem), smem_slots = smem_u32(slots);
    rows_wait_unit(&aux_full, 0);
    for (int k = 0; k < n; ++k) {
        const int slot = k % p.nslots;
        const int u = c.u_begin + k;
        const int b = u / p.NC, plane = u - b * p.NC;
        const int y0 = b * p.RC, nrows = min(p.H, y0 + p.RC) - y0;
        const bool active = worker && r < nrows;
        if (active && b != cached_b) {
            const long long wo = (long long)(y0 + r) * p.W + x0;
            if constexpr (VEC == 8) ldg256(rescale + wo, rs);
            else {
                const float4 f = __ldg(reinterpret_cast<const float4*>(rescale + wo));
                rs[0] = f.x; rs[1] = f.y; rs[2] = f.z; rs[3] = f.w;
            }
            cached_b = b;
        }
        rows_wait_unit(&full[slot], (uint32_t)((k / p.nslots) & 1));
        if (active) {
            const SegTable& sg = segs[slot];
            const uint32_t sbase = smem_slots + (uint32_t)slot * (uint32_t)p.slot_bytes;
            const int y = y0 + r;
            float acc[VEC];
#pragma unroll
            for (int j = 0; j < VEC; ++j) acc[j] = 0.0f;
            const int nseg = sg.nseg;
            for (int q = 0; q < nseg; ++q) {
                const int rr = y - sg.yy0[q], nr = sg.nr[q];
                if ((unsigned)rr >= (unsigned)nr) continue;
                const uint32_t colstride = (uint32_t)nr * row_bytes;
                const uint32_t rowbase = sbase + (uint32_t)sg.off[q] + (uint32_t)rr * row_bytes;
                const int v = y - (int)s_ys[sg.band[q]];                            // tile row
                const uint32_t wrow = smem_tw + (uint32_t)(v * p.tw) * 4u;          // gaussian row in shared memory
#pragma unroll
                for (int cc = 0; cc < kRowsMaxCols; ++cc) {
                    if (cc < jn) {
                        const uint4 e = rows_visit<T>(rowbase + (uint32_t)cr[cc].j * colstride, cr[cc]);
                        const int u0 = cr[cc].u0;
#pragma unroll
                        for (int m = 0; m < VEC; ++m) {
                            const int uu = u0 + m;
                            if ((unsigned)uu < (unsigned)p.tw) {           // elements outside the tile are not touched
                                const float w = __fmul_rn(lds_f32_u32(wrow + (uint32_t)uu * 4u), rs[m]);
                                const float val = __fmul_rn(Vec<T>::get(e, m), w);
                                acc[m] = round_through<T>(__fadd_rn(acc[m], val));
                            }
                        }
                    }
                }
            }
            const long long o = ((long long)plane * p.H + y) * p.W + x0;
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
            stg128(out_buf + o, pk);
        }
        if (k + p.nslots < n) {
            __syncthreads();
            if (tid < 32) rows_issue<T, false>(p, c.u_begin + k + p.nslots, slot, slots, segs, full, (const T*)nullptr);
        }
    }
}

// =================================================================================================================
// Scatter: tiles[(t - tile_begin) * NC + plane, v, u] = x[plane, ys + v, xs + u]
// A thread owns one vector column `uv` of the tile rows for the whole kernel and walks (tile column, row) pairs with a
// stride: no division in the loop (pair -> (j, rr) by a multiply-shift).
// =================================================================================================================
template <typename T>
__global__ void __launch_bounds__(kRowsThreads, 1)
scatter_rows_kernel(const __grid_constant__ RowsParams p, const T* __restrict__ x, T* __restrict__ tiles) {
    constexpr int VEC = Vec<T>::kElems;
    extern __shared__ __align__(128) unsigned char rows_smem[];
    __shared__ __align__(8) uint64_t full[kRowsMaxSlots];
    __shared__ SegTable segs[kRowsMaxSlots];
    __shared__ short s_xs[TD_MAX_GRID_DIM], s_ys[TD_MAX_GRID_DIM];
    const int tid = threadIdx.x;
    const RowsCommon c = rows_partition(p);
    const int n = c.u_end - c.u_begin;
    if (tid == 0) {
        for (int s = 0; s < p.nslots; ++s) mbar_init(&full[s], 1);
        fence_mbar_init();
        fence_proxy_async();
    }
    for (int i = tid; i < p.cols; i += kRowsThreads) s_xs[i] = p.xs[i];
    for (int i = tid; i < p.rows; i += kRowsThreads) s_ys[i] = p.ys[i];
    const int slot_rows = kRowsThreads / p.twv;              // (column, row) pairs handled per sweep
    const int ps = tid / p.twv, uv = tid - ps * p.twv;
    const bool worker = ps < slot_rows;
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();
    if (tid < 32)
        for (int k = 0; k < min(n, p.nslots); ++k) rows_issue<T, true>(p, c.u_begin + k, k, rows_smem, segs, full, x);
    const uint32_t crow_bytes = (uint32_t)p.W * (uint32_t)sizeof(T);
    const uint32_t smem0 = smem_u32(rows_smem);
    const long long plane_elems = (long long)p.th * p.tw;
    for (int k = 0; k < n; ++k) {
        const int slot = k % p.nslots;
        rows_wait_unit(&full[slot], (uint32_t)((k / p.nslots) & 1));
        if (worker) {
            const SegTable& sg = segs[slot];
            const uint32_t sbase = smem0 + (uint32_t)slot * (uint32_t)p.slot_bytes;
            const int plane = sg.plane, y0 = sg.y0, nseg = sg.nseg;
            for (int q = 0; q < nseg; ++q) {
                const int i = sg.band[q], nr = sg.nr[q], yy0 = sg.yy0[q];
                const unsigned magic = ((1u << 20) + (unsigned)nr - 1u) / (unsigned)nr;       // pair / nr for pair < 16384
                const int npairs = nr * p.cols;
                const int v0 = yy0 - (int)s_ys[i];
                for (int pr = ps; pr < npairs; pr += slot_rows) {
                    const int j = (int)(((unsigned)pr * magic) >> 20), rr = pr - j * nr;
                    const int t = i * p.cols + j;
                    if (t < p.tile_begin || t >= p.tile_end) continue;
                    const int xx = (int)s_xs[j] + uv * VEC;
                    const int a = xx & ~(VEC - 1), s = xx - a;
                    const uint32_t addr = sbase + (uint32_t)(yy0 + rr - y0) * crow_bytes + (uint32_t)a * (uint32_t)sizeof(T);
                    const uint4 A = lds128_u32(addr);
                    uint4 e = A;
                    if (s != 0) e = Vec<T>::window(A, lds128_u32(addr + 16u), s);     // xx + VEC <= W: the next chunk exists
                    T* dst = tiles + ((long long)(t - p.tile_begin) * p.NC + plane) * plane_elems + (long long)(v0 + rr) * p.tw + uv * VEC;
                    stg128_stream(dst, e);
                }
            }
        }
        if (k + p.nslots < n) {
            __syncthreads();
            if (tid < 32) rows_issue<T, true>(p, c.u_begin + k + p.nslots, slot, rows_smem, segs, full, x);
        }
    }
}

// ---- host ---------------------------------------------------------------------------------------------------------
// Fills geometry, picks RC (canvas rows per unit) and the slot layout.  Returns false when the row-block form does
// not apply (the caller falls back to the kernels in td_diffusion.cu).  scatter: slots hold canvas rows.
bool rows_plan(const td_grid* g, int N, int C, int es, int budget_bytes, bool scatter, int sms, RowsParams* p) {
    const int VEC = 16 / es;
    if (g->W % VEC != 0 || g->tile_w % VEC != 0) return false;
    if (g->W / VEC > kRowsMaxVec || g->rows > TD_MAX_GRID_DIM || g->cols > TD_MAX_GRID_DIM) return false;
    if (g->H > 32767 || g->W > 32767) return false;
    std::memset(p, 0, sizeof(*p));
    p->H = g->H; p->W = g->W; p->th = g->tile_h; p->tw = g->tile_w; p->rows = g->rows; p->cols = g->cols; p->NC = N * C;
    p->wv = g->W / VEC; p->twv = g->tile_w / VEC;
    p->tile_stride = (long long)N * C * g->tile_h * g->tile_w;
    for (int i = 0; i < g->rows; ++i) p->ys[i] = (short)g->ys[i];
    for (int j = 0; j < g->cols; ++j) p->xs[j] = (short)g->xs[j];
    for (int v = 0; v < p->wv; ++v) {
        int lo = -1, n = 0;
        for (int j = 0; j < g->cols; ++j)
            if (g->xs[j] < (v + 1) * VEC && g->xs[j] + g->tile_w > v * VEC) {
                if (lo < 0) lo = j;
                ++n;
            }
        if (n > kRowsMaxCols) return false;
        p->vcol_lo[v] = (unsigned char)std::max(lo, 0);
        p->vcol_n[v] = (unsigned char)n;
    }
    // candidate RC: most balanced contiguous-unit partition over `sms` CTAs, ties -> larger RC (bigger copies)
    double best_eff = -1.0;
    int best_rc = 0, best_slot = 0, best_nslots = 0;
    for (int rc = 2; rc <= 32; ++rc) {
        const int nblocks = (g->H + rc - 1) / rc;
        int slot = 0, max_segs = 0;
        for (int b = 0; b < nblocks; ++b) {
            const int y0 = b * rc, y1 = std::min(g->H, y0 + rc);
            int bytes = 0, segs = 0;
            for (int i = 0; i < g->rows; ++i) {
                const int a = std::max(y0, g->ys[i]), e = std::min(y1, g->ys[i] + g->tile_h);
                if (e > a) { bytes += (e - a) * g->cols * g->tile_w * es; ++segs; }
            }
            if (scatter) bytes = (y1 - y0) * g->W * es;
            slot = std::max(slot, bytes);
            max_segs = std::max(max_segs, segs);
        }
        if (max_segs > kRowsMaxSegs) continue;
        if (!scatter && rc * (g->W / VEC) > kRowsThreads) continue;      // blend: one (row, vector) task per thread
        if (scatter && (g->tile_w / VEC > kRowsThreads || rc * g->cols >= 16384)) continue;
        slot = (slot + 127) & ~127;
        if (slot <= 0) continue;
        const int nslots = std::min(kRowsMaxSlots, budget_bytes / slot);
        if (nslots < 2) continue;
        const long long nunits = (long long)nblocks * N * C;
        // work of the busiest CTA, in canvas rows
        long long max_rows = 0, total_rows = (long long)g->H * N * C;
        int max_units = 0;
        for (int cta = 0; cta < sms; ++cta) {
            const long long u0 = nunits * cta / sms, u1 = nunits * (cta + 1) / sms;
            long long rows = 0;
            for (long long u = u0; u < u1; ++u) {
                const int b = (int)(u / (N * C));
                rows += std::min(g->H, (b + 1) * rc) - b * rc;
            }
            max_rows = std::max(max_rows, rows);
            max_units = std::max(max_units, (int)(u1 - u0));
        }
        if (max_rows == 0) continue;
        double eff = (double)total_rows / ((double)max_rows * sms);
        if (max_units > nslots) eff *= 0.9;                          // not everything in flight at once
        if (eff > best_eff + 1e-9 || (eff > best_eff - 1e-9 && rc > best_rc)) {
            best_eff = eff; best_rc = rc; best_slot = slot; best_nslots = nslots;
        }
    }
    if (best_rc == 0) return false;
    p->RC = best_rc;
    p->nblocks = (g->H + best_rc - 1) / best_rc;
    p->nunits = p->nblocks * N * C;
    p->slot_bytes = best_slot;
    p->nslots = best_nslots;
    return true;
}

bool rows_aligned(const void* ptr, size_t a) { return (reinterpret_cast<uintptr_t>(ptr) & (a - 1)) == 0; }

bool rows_fill_batches(RowsParams* p, const void* const* batch_ptrs, int num_batches, int tile_bs, int es) {
    if (num_batches > TD_MAX_BATCH_PTRS) return false;
    for (int b = 0; b < num_batches; ++b) {
        if (!aligned16(batch_ptrs[b])) return false;
        p->batch_ptrs[b] = batch_ptrs[b];
    }
    p->num_batches = num_batches;
    p->tile_bs = tile_bs;
    // every bulk-copy source must be 16-byte aligned: plane and row strides are multiples of tw * es
    return ((long long)p->tw * es) % 16 == 0;
}

// The row-block form declines (returns 1, the caller falls back) when its shared-memory opt-in fails.
template <typename T>
int rows_launch_md(const RowsParams& p, int grid, const float* weights, const float* rcp, float* x_out, void* x_buffer, bool pdl, cudaStream_t st) {
    const size_t smem = (size_t)p.nslots * p.slot_bytes;
    const bool fd = rcp != nullptr && sizeof(T) == 2;
    auto kernel = x_buffer != nullptr ? (fd ? blend_rows_md_kernel<T, true, true> : blend_rows_md_kernel<T, true, false>)
                                      : (fd ? blend_rows_md_kernel<T, false, true> : blend_rows_md_kernel<T, false, false>);
    const char* what = "td_blend_multidiffusion (row-block form)";
    if (smem_optin(kernel, kRowsSmemBudget, what) != TD_OK) return 1;
    return launch(what, kernel, dim3((unsigned)grid), dim3(kRowsThreads), smem, st, pdl, p, weights, rcp, x_out, (T*)x_buffer);
}

template <typename T>
int rows_launch_mod(const RowsParams& p, int grid, const float* tile_weights, const float* rescale, void* x_buffer, bool pdl, cudaStream_t st) {
    const size_t smem = (size_t)p.aux_bytes + (size_t)p.nslots * p.slot_bytes;
    const char* what = "td_blend_mixture (row-block form)";
    if (smem_optin(blend_rows_mod_kernel<T>, kRowsSmemBudget, what) != TD_OK) return 1;
    return launch(what, blend_rows_mod_kernel<T>, dim3((unsigned)grid), dim3(kRowsThreads), smem, st, pdl, p, tile_weights, rescale,
                  (T*)x_buffer);
}

template <typename T>
int rows_launch_scatter(const RowsParams& p, int grid, const void* x, void* tiles, bool pdl, cudaStream_t st) {
    const size_t smem = (size_t)p.nslots * p.slot_bytes;
    const char* what = "td_scatter_tiles (row-block form)";
    if (smem_optin(scatter_rows_kernel<T>, kRowsSmemBudget, what) != TD_OK) return 1;
    return launch(what, scatter_rows_kernel<T>, dim3((unsigned)grid), dim3(kRowsThreads), smem, st, pdl, p, (const T*)x, (T*)tiles);
}

}  // namespace

// TD_OK launched, 1 not applicable (caller falls back), < 0 error.
int td_rows_try_launch_md(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int dtype,
                          const float* weights, const float* rcp_weights, float* x_out, void* x_buffer, int pdl, int dbg_no_tiles,
                          void* stream) {
    const DeviceProps d = device_props();
    if (!d.ok || d.smem_optin < kRowsSmemBudget) return 1;
    const int es = td_dtype_size(dtype);
    RowsParams p;
    if (!rows_plan(g, N, C, es, kRowsSmemBudget, false, d.sms, &p)) return 1;
    if (!rows_fill_batches(&p, batch_ptrs, num_batches, tile_bs, es)) return 1;
    if (!rows_aligned(weights, 32) || !rows_aligned(x_out, 32) || (rcp_weights && !rows_aligned(rcp_weights, 32)) ||
        (x_buffer && !aligned16(x_buffer)))
        return 1;
    p.dbg_no_tiles = dbg_no_tiles;
    const int grid = std::min(d.sms, p.nunits);
    cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case TD_F16: return rows_launch_md<__half>(p, grid, weights, rcp_weights, x_out, x_buffer, pdl != 0, st);
        case TD_BF16: return rows_launch_md<__nv_bfloat16>(p, grid, weights, rcp_weights, x_out, x_buffer, pdl != 0, st);
        default: return rows_launch_md<float>(p, grid, weights, nullptr, x_out, x_buffer, pdl != 0, st);
    }
}

int td_rows_try_launch_mod(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int dtype,
                           const float* tile_weights, const float* rescale, void* x_buffer, int pdl, void* stream) {
    const DeviceProps d = device_props();
    if (!d.ok || d.smem_optin < kRowsSmemBudget) return 1;
    const int es = td_dtype_size(dtype);
    const int aux = (g->tile_h * g->tile_w * 4 + 127) & ~127;
    if (aux > kRowsSmemBudget / 2 || (g->tile_h * g->tile_w * 4) % 16 != 0) return 1;
    RowsParams p;
    if (!rows_plan(g, N, C, es, kRowsSmemBudget - aux, false, d.sms, &p)) return 1;
    if (!rows_fill_batches(&p, batch_ptrs, num_batches, tile_bs, es)) return 1;
    if (!aligned16(tile_weights) || !rows_aligned(rescale, 32) || !aligned16(x_buffer)) return 1;
    p.aux_bytes = aux;
    const int grid = std::min(d.sms, p.nunits);
    cudaStream_t st = (cudaStream_t)stream;
    // the staged gaussian is copied as `aux` bytes: the source must hold that many (th * tw * 4 rounded up to 128)
    if (aux != g->tile_h * g->tile_w * 4) return 1;
    switch (dtype) {
        case TD_F16: return rows_launch_mod<__half>(p, grid, tile_weights, rescale, x_buffer, pdl != 0, st);
        case TD_BF16: return rows_launch_mod<__nv_bfloat16>(p, grid, tile_weights, rescale, x_buffer, pdl != 0, st);
        default: return rows_launch_mod<float>(p, grid, tile_weights, rescale, x_buffer, pdl != 0, st);
    }
}

int td_rows_try_launch_scatter(const td_grid* g, const void* x, void* tiles, int N, int C, int dtype, int tile_begin, int tile_end,
                               int pdl, void* stream) {
    const DeviceProps d = device_props();
    if (!d.ok || d.smem_optin < kRowsSmemBudget) return 1;
    const int es = td_dtype_size(dtype);
    RowsParams p;
    if (!rows_plan(g, N, C, es, kRowsSmemBudget, true, d.sms, &p)) return 1;
    if (!aligned16(x) || !aligned16(tiles) || ((long long)g->W * es) % 16 != 0) return 1;
    p.tile_begin = tile_begin;
    p.tile_end = tile_end;
    const int grid = std::min(d.sms, p.nunits);
    cudaStream_t st = (cudaStream_t)stream;
    // fp16 and bf16 are both moved as opaque 16-bit words
    if (es == 2) return rows_launch_scatter<__half>(p, grid, x, tiles, pdl != 0, st);
    return rows_launch_scatter<float>(p, grid, x, tiles, pdl != 0, st);
}
