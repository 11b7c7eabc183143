// Strip form of the MultiDiffusion blend (TD_FLAG_STRIP, opt-in): multidiffusion.py:166-167 + :208 of the reference,
// same gather-form, same rounding sequence as blend_md_async_kernel (td_diffusion.cu), different work decomposition.
//
// The default kernel gives a CTA an 8-row x 64-px patch and stages, for every tile touching the patch, the patch-sized
// aligned superset -- mostly zero fill at tile edges -- and reserves shared memory for the worst patch, which caps the
// residency at about half the grid (two waves, DESIGN.md section 4).  Here a CTA owns 8 canvas rows x the FULL canvas
// width of one plane.  A tile visit then stages exactly the tile's row segment (tw elements + one zero chunk each
// side), no column clipping: ~12 B of shared memory per output pixel instead of ~27, so the whole grid is resident
// in one wave (cfg2: 512 CTAs x 512 threads, 54 KB each, 4 per SM).  The tile-column loop is CTA-uniform and the
// funnel shift depends on the tile column only.
//
// Not measured on hardware yet (written after the round-1 GPU budget was spent).  The three phases are __host__
// __device__ functions, so a test-only harness (tests/emul/strip_host_emul.cu) runs whole CTAs on the host --
// thread by thread, phase by phase -- against the reference's fixtures; the device-only primitives they wrap
// (cp.async zero-fill copy, funnel-shift window, packed add) are the ones the default kernel already uses.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <mutex>

#include "td_b200.h"
#include "td_device.cuh"
#include "td_internal.h"
#include "td_launch.h"

namespace {

using namespace td;

#ifndef TD_STRIP_ROWS
#define TD_STRIP_ROWS 8              // tuning knob (-DTD_STRIP_ROWS=): canvas rows per CTA
#endif
constexpr int kStripRows = TD_STRIP_ROWS;   // canvas rows per CTA
constexpr int kStripMaxVisits = 64;  // tile rows touching a strip x tile columns

struct StripParams {
    int H, W, th, tw, rows, cols, NC;
    int tile_bs;
    int xv, twv, cpr, spv;           // vectors per canvas row; chunks per tile row; staged chunks per row (twv + 2); slots per visit
    unsigned bs_magic, cols_magic, spv_magic, cpr_magic, xv_magic;   // ceil(2^32 / d) for operands < 2^16 (0: d == 1)
    long long tile_stride;           // elements of one tile: NC * th * tw
    short ys[TD_MAX_GRID_DIM], xs[TD_MAX_GRID_DIM];
    unsigned char prow_lo[TD_MAX_GRID_DIM], prow_n[TD_MAX_GRID_DIM];   // tile rows touching strip i: first index, count
    const void* batch_ptrs[TD_MAX_BATCH_PTRS];
};

struct __align__(8) StripVisit {
    long long origin;   // byte address of tile element (v0, 0) of this CTA's plane (v0 may lie outside the tile)
    int v0;             // tile row of the strip's first canvas row
    int qx;             // xs >> log2(VEC): first canvas vector the tile touches
    int s;              // xs & (VEC - 1): misalignment of the tile against the canvas vector grid
    int pad_;
};

__host__ __device__ __forceinline__ unsigned sdiv(unsigned n, unsigned magic) {
#ifdef __CUDA_ARCH__
    return magic ? __umulhi(n, magic) : n;
#else
    return magic ? (unsigned)(((unsigned long long)n * magic) >> 32) : n;
#endif
}

template <typename T> struct SElem;
template <> struct SElem<__half> {
    static __host__ __device__ __forceinline__ float to_f32(uint16_t b) { __half_raw r; r.x = b; return __half2float(__half(r)); }
    static __host__ __device__ __forceinline__ uint16_t from_f32(float f) { return __half_raw(__float2half_rn(f)).x; }
};
template <> struct SElem<__nv_bfloat16> {
    static __host__ __device__ __forceinline__ float to_f32(uint16_t b) {
        uint32_t u = ((uint32_t)b) << 16;
        float f;
        memcpy(&f, &u, 4);
        return f;
    }
    static __host__ __device__ __forceinline__ uint16_t from_f32(float f) { return __nv_bfloat16_raw(__float2bfloat16_rn(f)).x; }
};

__host__ __device__ __forceinline__ float s_add(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}

__host__ __device__ __forceinline__ float s_mul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}

// fp32 value rounded through T (the store to x_buffer and the load back of the reference)
template <typename T> __host__ __device__ __forceinline__ float s_round(float f) {
    if constexpr (sizeof(T) == 4) return f;
    else return SElem<T>::to_f32(SElem<T>::from_f32(f));
}

// one 32-bit word of packed T: a (+) b with one rounding per element through T
template <typename T> __host__ __device__ __forceinline__ uint32_t s_packed_add(uint32_t a, uint32_t b) {
    if constexpr (sizeof(T) == 4) {
        float fa, fb;
        memcpy(&fa, &a, 4);
        memcpy(&fb, &b, 4);
        const float r = s_add(fa, fb);
        uint32_t o;
        memcpy(&o, &r, 4);
        return o;
    } else {
        const uint16_t lo = SElem<T>::from_f32(s_add(SElem<T>::to_f32((uint16_t)(a & 0xffffu)), SElem<T>::to_f32((uint16_t)(b & 0xffffu))));
        const uint16_t hi = SElem<T>::from_f32(s_add(SElem<T>::to_f32((uint16_t)(a >> 16)), SElem<T>::to_f32((uint16_t)(b >> 16))));
        return (uint32_t)lo | ((uint32_t)hi << 16);
    }
}

// elements [sh, sh + VEC) of the 2*VEC elements in (A, B)
template <typename T> __host__ __device__ __forceinline__ uint4 s_window(const uint4& A, const uint4& B, int sh) {
#ifdef __CUDA_ARCH__
    return Vec<T>::window(A, B, sh);
#else
    unsigned char buf[32];
    memcpy(buf, &A, 16);
    memcpy(buf + 16, &B, 16);
    uint4 o;
    memcpy(&o, buf + (size_t)sh * sizeof(T), 16);
    return o;
#endif
}

template <typename T> __host__ __device__ __forceinline__ float s_get(const uint4& v, int j) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    if constexpr (sizeof(T) == 4) {
        float f;
        memcpy(&f, &w[j], 4);
        return f;
    } else {
        const uint32_t word = w[j >> 1];
        return SElem<T>::to_f32((uint16_t)((j & 1) ? (word >> 16) : (word & 0xffffu)));
    }
}

// 16-byte copy global -> shared, or 16 zero bytes (no global access) when !valid
__host__ __device__ __forceinline__ void s_copy16(unsigned char* dst, long long src, bool valid) {
#ifdef __CUDA_ARCH__
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst);
    const int neg_if_skip = valid ? 0 : -1;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.lt.s32 p, %2, 0;\n\t"
        "cp.async.cg.shared.global [%0], [%1], 16, p;\n\t}"
        ::"r"(d), "l"(src), "r"(neg_if_skip)
        : "memory");
#else
    if (valid) memcpy(dst, reinterpret_cast<const void*>(src), 16);
    else memset(dst, 0, 16);
#endif
}

__host__ __device__ __forceinline__ float s_div_exact(float a, float w, float rcp) {
    // correctly rounded a / w for |a| a 16-bit float value and integer w <= 4096, rcp = RN(1 / w)  (td_diffusion.cu)
#ifdef __CUDA_ARCH__
    const float q = __fmul_rn(a, rcp);
    const float r = __fmaf_rn(-q, w, a);
    const float q2 = __fmaf_rn(r, rcp, q);
#else
    const float q = a * rcp;
    const float r = fmaf(-q, w, a);
    const float q2 = fmaf(r, rcp, q);
#endif
    uint32_t uq, ua;
    memcpy(&uq, &q2, 4);
    memcpy(&ua, &a, 4);
    const uint32_t o = (uq & 0x7fffffffu) | (ua & 0x80000000u);
    float f;
    memcpy(&f, &o, 4);
    return f;
}

__host__ __device__ __forceinline__ float s_div_ieee(float a, float w) {
#ifdef __CUDA_ARCH__
    return __fdiv_rn(a, w);
#else
    return a / w;
#endif
}

// 16-byte accesses at addresses that are 16-byte aligned by construction
__host__ __device__ __forceinline__ uint4 s_ld16(const void* p) { return *reinterpret_cast<const uint4*>(p); }
__host__ __device__ __forceinline__ void s_st16(void* p, const uint4& v) { *reinterpret_cast<uint4*>(p) = v; }
__host__ __device__ __forceinline__ float4 s_ldf4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__host__ __device__ __forceinline__ void s_stf4(float* p, const float4& v) { *reinterpret_cast<float4*>(p) = v; }

__host__ __device__ __forceinline__ StripVisit* strip_visits(unsigned char* smem) { return reinterpret_cast<StripVisit*>(smem); }
__host__ __device__ __forceinline__ unsigned char* strip_stage(unsigned char* smem) { return smem + kStripMaxVisits * sizeof(StripVisit); }

// ---- phase 1: thread i prepares visit i = (tile row ri, tile column c), ascending tile index --------------------------
template <typename T>
__host__ __device__ __forceinline__ void strip_phase_table(const StripParams& p, int strip, int plane, int tid, unsigned char* smem) {
    constexpr int VEC = 16 / (int)sizeof(T);
    constexpr int L2V = (sizeof(T) == 2) ? 3 : 2;
    const int nvis = (int)p.prow_n[strip] * p.cols;
    if (tid >= nvis) return;
    const int ri = (int)sdiv((unsigned)tid, p.cols_magic), c = tid - ri * p.cols;
    const int r = (int)p.prow_lo[strip] + ri;
    const unsigned t = (unsigned)(r * p.cols + c);
    const unsigned b = sdiv(t, p.bs_magic);
    const int v0 = strip * kStripRows - (int)p.ys[r];
    const long long elem = (long long)(t - b * (unsigned)p.tile_bs) * p.tile_stride + (long long)plane * p.th * p.tw + (long long)v0 * p.tw;
    StripVisit e;
    e.origin = (long long)reinterpret_cast<uintptr_t>(p.batch_ptrs[b]) + elem * (long long)sizeof(T);
    e.v0 = v0;
    e.qx = (int)p.xs[c] >> L2V;
    e.s = (int)p.xs[c] & (VEC - 1);
    e.pad_ = 0;
    strip_visits(smem)[tid] = e;
}

// ---- phase 2: stage every visit's row segments: slot = (visit, plane, strip row, chunk), chunk 0 and twv+1 are zero pads ---
// PPC = planes per CTA: the (n, c) planes of a strip share the visit table, the predicates and the shifts.
template <typename T, int PPC = 1>
__host__ __device__ __forceinline__ void strip_phase_copy(const StripParams& p, int strip, int tid, int nthreads, unsigned char* smem) {
    constexpr int VEC = 16 / (int)sizeof(T);
    const int nvis = (int)p.prow_n[strip] * p.cols;
    const StripVisit* vis = strip_visits(smem);
    unsigned char* stage = strip_stage(smem);
    const long long plane_bytes = (long long)p.th * p.tw * (long long)sizeof(T);
    if (p.spv <= nthreads) {
        // a thread keeps ONE slot (strip row, chunk) and walks the visits with a stride of G = nthreads / spv groups:
        // row / chunk arithmetic once, ~10 instructions per copy
        const int groups = (int)sdiv((unsigned)nthreads, p.spv_magic);
        const int grp = (int)sdiv((unsigned)tid, p.spv_magic), q = tid - grp * p.spv;
        if (grp >= groups) return;
        const int row = (int)sdiv((unsigned)q, p.cpr_magic), j = q - row * p.cpr;
        const bool col_ok = j >= 1 && j <= p.twv;
        const long long off = ((long long)row * p.tw + (long long)(j - 1) * VEC) * (long long)sizeof(T);
        for (int i = grp; i < nvis; i += groups) {
            const StripVisit e = vis[i];
            const bool valid = col_ok && (unsigned)(e.v0 + row) < (unsigned)p.th;
#pragma unroll
            for (int pl = 0; pl < PPC; ++pl)
                s_copy16(stage + (((size_t)i * PPC + pl) * p.spv + q) * 16, e.origin + off + pl * plane_bytes, valid);
        }
        return;
    }
    const int total = nvis * p.spv;    // a staged row wider than the CTA (single tile column): flat slot loop
    for (int s = tid; s < total; s += nthreads) {
        const int i = (int)sdiv((unsigned)s, p.spv_magic), q = s - i * p.spv;
        const int row = (int)sdiv((unsigned)q, p.cpr_magic), j = q - row * p.cpr;
        const StripVisit e = vis[i];
        const bool valid = (unsigned)(e.v0 + row) < (unsigned)p.th && j >= 1 && j <= p.twv;
        const long long src = e.origin + ((long long)row * p.tw + (long long)(j - 1) * VEC) * (long long)sizeof(T);
#pragma unroll
        for (int pl = 0; pl < PPC; ++pl)
            s_copy16(stage + (((size_t)i * PPC + pl) * p.spv + q) * 16, src + pl * plane_bytes, valid);
    }
}

// ---- phase 3: one thread per canvas vector (of PPC planes): add the covering tiles in tile order, normalise, store --------
template <typename T, bool WRITE_BUF, bool FASTDIV, int PPC = 1>
__host__ __device__ __forceinline__ void strip_phase_consume(const StripParams& p, int strip, int plane, int tid, unsigned char* smem,
                                                             const float* __restrict__ weights, const float* __restrict__ rcp_weights,
                                                             float* __restrict__ out_f32, T* __restrict__ out_buf) {
    constexpr int VEC = 16 / (int)sizeof(T);
    const int ty = (int)sdiv((unsigned)tid, p.xv_magic), tx = tid - ty * p.xv;
    const int y = strip * kStripRows + ty;
    if (ty >= kStripRows || y >= p.H) return;
    const int nvis = (int)p.prow_n[strip] * p.cols;
    const StripVisit* vis = strip_visits(smem);
    const unsigned char* row0 = strip_stage(smem) + (size_t)ty * p.cpr * 16;
    const size_t plane_stage = (size_t)p.spv * 16;
    uint4 acc[PPC];
#pragma unroll
    for (int pl = 0; pl < PPC; ++pl) acc[pl] = make_uint4(0, 0, 0, 0);
    for (int i = 0; i < nvis; ++i) {
        const StripVisit e = vis[i];
        if ((unsigned)(e.v0 + ty) >= (unsigned)p.th) continue;     // this canvas row lies above / below the tile (its stage rows are zero)
        const unsigned char* rowp = row0 + (size_t)i * PPC * plane_stage;
        if (e.s == 0) {
            const int idx = tx - e.qx + 1;                 // staged chunk of tile chunk (tx - qx)
            if ((unsigned)(idx - 1) >= (unsigned)p.twv) continue;
#pragma unroll
            for (int pl = 0; pl < PPC; ++pl) {
                const uint4 v = s_ld16(rowp + pl * plane_stage + (size_t)idx * 16);
                acc[pl].x = s_packed_add<T>(acc[pl].x, v.x); acc[pl].y = s_packed_add<T>(acc[pl].y, v.y);
                acc[pl].z = s_packed_add<T>(acc[pl].z, v.z); acc[pl].w = s_packed_add<T>(acc[pl].w, v.w);
            }
        } else {
            const int idx = tx - e.qx;                     // staged chunk of tile chunk (tx - qx - 1); -1 is the left pad
            if ((unsigned)idx > (unsigned)p.twv) continue;
#pragma unroll
            for (int pl = 0; pl < PPC; ++pl) {
                const uint4 A = s_ld16(rowp + pl * plane_stage + (size_t)idx * 16), B = s_ld16(rowp + pl * plane_stage + (size_t)(idx + 1) * 16);
                const uint4 v = s_window<T>(A, B, VEC - e.s);
                acc[pl].x = s_packed_add<T>(acc[pl].x, v.x); acc[pl].y = s_packed_add<T>(acc[pl].y, v.y);
                acc[pl].z = s_packed_add<T>(acc[pl].z, v.z); acc[pl].w = s_packed_add<T>(acc[pl].w, v.w);
            }
        }
    }
    // x_out = where(weights > 1, x_buffer / weights, x_buffer): fp32, correctly rounded divide (multidiffusion.py:208)
    const int x0 = tx * VEC;
    const long long wo = (long long)y * p.W + x0;
#pragma unroll
    for (int h = 0; h < VEC / 4; ++h) {
        const float4 w = s_ldf4(weights + wo + 4 * h);
        float4 rc = make_float4(1.f, 1.f, 1.f, 1.f);
        if constexpr (FASTDIV) rc = s_ldf4(rcp_weights + wo + 4 * h);
#pragma unroll
        for (int pl = 0; pl < PPC; ++pl) {
            const long long o = ((long long)(plane + pl) * p.H + y) * p.W + x0;
            const float a0 = s_get<T>(acc[pl], 4 * h + 0), a1 = s_get<T>(acc[pl], 4 * h + 1);
            const float a2 = s_get<T>(acc[pl], 4 * h + 2), a3 = s_get<T>(acc[pl], 4 * h + 3);
            float4 f;
            if constexpr (FASTDIV) {
                f.x = w.x > 1.0f ? s_div_exact(a0, w.x, rc.x) : a0;
                f.y = w.y > 1.0f ? s_div_exact(a1, w.y, rc.y) : a1;
                f.z = w.z > 1.0f ? s_div_exact(a2, w.z, rc.z) : a2;
                f.w = w.w > 1.0f ? s_div_exact(a3, w.w, rc.w) : a3;
            } else {
                f.x = w.x > 1.0f ? s_div_ieee(a0, w.x) : a0;
                f.y = w.y > 1.0f ? s_div_ieee(a1, w.y) : a1;
                f.z = w.z > 1.0f ? s_div_ieee(a2, w.z) : a2;
                f.w = w.w > 1.0f ? s_div_ieee(a3, w.w) : a3;
            }
            s_stf4(out_f32 + o + 4 * h, f);
        }
    }
    if constexpr (WRITE_BUF) {
#pragma unroll
        for (int pl = 0; pl < PPC; ++pl) s_st16(out_buf + ((long long)(plane + pl) * p.H + y) * p.W + x0, acc[pl]);
    }
}

template <typename T, bool WRITE_BUF, bool FASTDIV, int PPC>
__global__ void __launch_bounds__(1024)
strip_blend_kernel(const __grid_constant__ StripParams p, const float* __restrict__ weights, const float* __restrict__ rcp_weights,
                   float* __restrict__ out_f32, T* __restrict__ out_buf) {
    extern __shared__ __align__(16) unsigned char td_strip_smem[];
    const int strip = blockIdx.x, plane = blockIdx.y * PPC, tid = threadIdx.x;
    // programmatic dependent launch: the next grid may become resident while this one drains; every global access of THIS
    // grid waits for its predecessor below
    pdl_launch_dependents();
    strip_phase_table<T>(p, strip, plane, tid, td_strip_smem);     // kernel parameters only
    pdl_wait();
    __syncthreads();
    strip_phase_copy<T, PPC>(p, strip, tid, (int)blockDim.x, td_strip_smem);
    asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    strip_phase_consume<T, WRITE_BUF, FASTDIV, PPC>(p, strip, plane, tid, td_strip_smem, weights, rcp_weights, out_f32, out_buf);
}

// ---- phase 3, Mixture of Diffusers (mixtureofdiffusers.py:122-126): per element of every covering tile, in tile order,
//      w = tile_weights[v, u] * rescale[y, x]   (fp32 product, its own rounding)
//      acc = round_T(acc + tile * w)            (separate multiply and add, no FMA)
// Elements outside the tile are skipped, never added as zeros: with gaussian weights the accumulator can be -0.0 and
// -0 + (+0) would flip the sign bit the reference keeps.  Returns x_buffer in the latent dtype (no division).
template <typename T>
__host__ __device__ __forceinline__ void strip_phase_consume_mod(const StripParams& p, int strip, int plane, int tid, unsigned char* smem,
                                                                 const float* __restrict__ tile_weights, const float* __restrict__ rescale,
                                                                 T* __restrict__ out_buf) {
    constexpr int VEC = 16 / (int)sizeof(T);
    const int ty = (int)sdiv((unsigned)tid, p.xv_magic), tx = tid - ty * p.xv;
    const int y = strip * kStripRows + ty;
    if (ty >= kStripRows || y >= p.H) return;
    const int nvis = (int)p.prow_n[strip] * p.cols;
    const StripVisit* vis = strip_visits(smem);
    const unsigned char* row0 = strip_stage(smem) + (size_t)ty * p.cpr * 16;
    const int x0 = tx * VEC;
    const long long wo = (long long)y * p.W + x0;
    float rs[VEC], acc[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) { rs[j] = rescale[wo + j]; acc[j] = 0.0f; }
    for (int i = 0; i < nvis; ++i) {
        const StripVisit e = vis[i];
        const int v = e.v0 + ty;                           // tile row of this canvas row
        if ((unsigned)v >= (unsigned)p.th) continue;
        const int u0 = (tx - e.qx) * VEC - e.s;            // tile column of this vector's first element
        const int jlo = u0 < 0 ? -u0 : 0, jhi = (p.tw - u0) < VEC ? (p.tw - u0) : VEC;
        if (jlo >= jhi) continue;
        const unsigned char* rowp = row0 + (size_t)i * p.spv * 16;
        uint4 t;
        if (e.s == 0) {
            t = s_ld16(rowp + (size_t)(tx - e.qx + 1) * 16);
        } else {
            const int idx = tx - e.qx;
            t = s_window<T>(s_ld16(rowp + (size_t)idx * 16), s_ld16(rowp + (size_t)(idx + 1) * 16), VEC - e.s);
        }
        const float* wrow = tile_weights + (long long)v * p.tw + u0;
#pragma unroll
        for (int j = 0; j < VEC; ++j) {
            if (j < jlo || j >= jhi) continue;
            const float w = s_mul(wrow[j], rs[j]);
            acc[j] = s_round<T>(s_add(acc[j], s_mul(s_get<T>(t, j), w)));
        }
    }
    const long long o = ((long long)plane * p.H + y) * p.W + x0;
    uint4 pk;
    if constexpr (sizeof(T) == 4) {
        uint32_t w32[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) memcpy(&w32[j], &acc[j], 4);
        pk = make_uint4(w32[0], w32[1], w32[2], w32[3]);
    } else {
        uint32_t w32[4];
#pragma unroll
        for (int h = 0; h < 4; ++h) w32[h] = (uint32_t)SElem<T>::from_f32(acc[2 * h]) | ((uint32_t)SElem<T>::from_f32(acc[2 * h + 1]) << 16);
        pk = make_uint4(w32[0], w32[1], w32[2], w32[3]);
    }
    s_st16(out_buf + o, pk);
}

template <typename T>
__global__ void __launch_bounds__(1024)
strip_blend_mod_kernel(const __grid_constant__ StripParams p, const float* __restrict__ tile_weights, const float* __restrict__ rescale,
                       T* __restrict__ out_buf) {
    extern __shared__ __align__(16) unsigned char td_strip_smem[];
    const int strip = blockIdx.x, plane = blockIdx.y, tid = threadIdx.x;
    pdl_launch_dependents();
    strip_phase_table<T>(p, strip, plane, tid, td_strip_smem);
    pdl_wait();
    __syncthreads();
    strip_phase_copy<T>(p, strip, tid, (int)blockDim.x, td_strip_smem);
    asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    strip_phase_consume_mod<T>(p, strip, plane, tid, td_strip_smem, tile_weights, rescale, out_buf);
}

// fills p and the launch shape; 0 = applicable, 1 = not applicable
int strip_plan(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int elem_size, StripParams* p,
               int* nthreads, int* smem_bytes, int* strips) {
    const int VEC = 16 / elem_size;
    if (g->W % VEC != 0 || g->tile_w % VEC != 0 || g->H >= 32768 || g->W >= 32768) return 1;
    p->H = g->H; p->W = g->W; p->th = g->tile_h; p->tw = g->tile_w; p->rows = g->rows; p->cols = g->cols; p->NC = N * C;
    p->tile_bs = tile_bs;
    p->xv = g->W / VEC; p->twv = g->tile_w / VEC; p->cpr = p->twv + 2; p->spv = kStripRows * p->cpr;
    if (p->xv * kStripRows > 1024 || p->NC > 65535) return 1;
    *strips = (g->H + kStripRows - 1) / kStripRows;
    if (*strips > TD_MAX_GRID_DIM || g->rows > TD_MAX_GRID_DIM || g->cols > TD_MAX_GRID_DIM) return 1;
    int nr_cap = 0;
    for (int s = 0; s < *strips; ++s) {
        const int lo = s * kStripRows, hi = std::min(lo + kStripRows, g->H) - 1;
        int first = -1, cnt = 0;
        for (int r = 0; r < g->rows; ++r)
            if (g->ys[r] <= hi && g->ys[r] + g->tile_h > lo) { if (first < 0) first = r; ++cnt; }
        // the tile rows touching a strip are contiguous (origins are non-decreasing): [first, first + cnt)
        p->prow_lo[s] = (unsigned char)std::max(first, 0);
        p->prow_n[s] = (unsigned char)cnt;
        nr_cap = std::max(nr_cap, cnt);
    }
    const int nv_cap = nr_cap * g->cols;
    if (nv_cap <= 0 || nv_cap > kStripMaxVisits) return 1;
    if ((long long)nv_cap * p->spv >= 65536) return 1;        // sdiv operand range
    *smem_bytes = kStripMaxVisits * (int)sizeof(StripVisit) + nv_cap * p->spv * 16;
    if (*smem_bytes > 200 * 1024) return 1;
    *nthreads = std::max(32, (p->xv * kStripRows + 31) / 32 * 32);
    if (nv_cap > *nthreads) return 1;                          // phase 1: one thread per visit
    p->tile_stride = (long long)p->NC * g->tile_h * g->tile_w;
    if (p->tile_stride >= (1ll << 31)) return 1;
    p->bs_magic = magic_u16((unsigned)tile_bs); p->cols_magic = magic_u16((unsigned)g->cols); p->spv_magic = magic_u16((unsigned)p->spv);
    p->cpr_magic = magic_u16((unsigned)p->cpr); p->xv_magic = magic_u16((unsigned)p->xv);
    if (g->num_tiles >= 65536 || kStripRows * p->xv >= 65536) return 1;
    for (int i = 0; i < g->rows; ++i) p->ys[i] = (short)g->ys[i];
    for (int i = 0; i < g->cols; ++i) p->xs[i] = (short)g->xs[i];
    for (int b = 0; b < num_batches; ++b) p->batch_ptrs[b] = batch_ptrs[b];
    return 0;
}

template <typename T, bool WRITE_BUF, bool FASTDIV, int PPC>
int strip_launch(const StripParams& p, int strips, int nthreads, int smem, const float* weights, const float* rcp, float* out_f32,
                 void* out_buf, bool pdl, cudaStream_t st) {
    const char* what = "td_blend_multidiffusion (strip)";
    const int rc = smem_optin(strip_blend_kernel<T, WRITE_BUF, FASTDIV, PPC>, smem, what);
    if (rc != TD_OK) return rc;
    return launch(what, strip_blend_kernel<T, WRITE_BUF, FASTDIV, PPC>, dim3((unsigned)strips, (unsigned)(p.NC / PPC)), dim3((unsigned)nthreads),
                  (size_t)smem, st, pdl, p, weights, rcp, out_f32, (T*)out_buf);
}

template <typename T, int PPC>
int strip_dispatch(const StripParams& p, int strips, int nthreads, int smem, const float* weights, const float* rcp, float* out_f32,
                   void* out_buf, bool pdl, cudaStream_t st) {
    const bool fast = rcp != nullptr && sizeof(T) == 2;
    if (out_buf != nullptr)
        return fast ? strip_launch<T, true, true, PPC>(p, strips, nthreads, smem, weights, rcp, out_f32, out_buf, pdl, st)
                    : strip_launch<T, true, false, PPC>(p, strips, nthreads, smem, weights, nullptr, out_f32, out_buf, pdl, st);
    return fast ? strip_launch<T, false, true, PPC>(p, strips, nthreads, smem, weights, rcp, out_f32, out_buf, pdl, st)
                : strip_launch<T, false, false, PPC>(p, strips, nthreads, smem, weights, nullptr, out_f32, out_buf, pdl, st);
}

// planes per CTA and the shared memory that goes with it (smem1 = the one-plane size from strip_plan)
int strip_pick_ppc(const StripParams& p, int smem1, int max_ppc, int* smem) {
    const int table = kStripMaxVisits * (int)sizeof(StripVisit);
    const int smem2 = table + 2 * (smem1 - table);
    if (max_ppc >= 2 && p.NC % 2 == 0 && smem2 <= 200 * 1024) { *smem = smem2; return 2; }
    *smem = smem1;
    return 1;
}

template <typename T>
int strip_launch_mod(const StripParams& p, int strips, int nthreads, int smem, const float* tile_weights, const float* rescale, void* out_buf,
                     bool pdl, cudaStream_t st) {
    const char* what = "td_blend_mixture (strip)";
    const int rc = smem_optin(strip_blend_mod_kernel<T>, smem, what);
    if (rc != TD_OK) return rc;
    return launch(what, strip_blend_mod_kernel<T>, dim3((unsigned)strips, (unsigned)p.NC), dim3((unsigned)nthreads), (size_t)smem, st, pdl, p,
                  tile_weights, rescale, (T*)out_buf);
}

std::mutex g_strip_mu;
StripParams g_strip_params;        // 2.7 KB: filled per launch under the lock (the parameters are copied at launch)

}  // namespace

// Mixture of Diffusers on strips; same return convention as td_strip_try_launch
int td_strip_try_launch_mod(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int dtype,
                            const float* tile_weights, const float* rescale, void* x_buffer, int pdl, void* stream) {
    std::lock_guard<std::mutex> lk(g_strip_mu);
    StripParams& p = g_strip_params;
    int nthreads = 0, smem = 0, strips = 0;
    if (strip_plan(g, batch_ptrs, num_batches, tile_bs, N, C, td_dtype_size(dtype), &p, &nthreads, &smem, &strips) != 0) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case TD_F16: return strip_launch_mod<__half>(p, strips, nthreads, smem, tile_weights, rescale, x_buffer, pdl != 0, st);
        case TD_BF16: return strip_launch_mod<__nv_bfloat16>(p, strips, nthreads, smem, tile_weights, rescale, x_buffer, pdl != 0, st);
        case TD_F32: return strip_launch_mod<float>(p, strips, nthreads, smem, tile_weights, rescale, x_buffer, pdl != 0, st);
        default: return 1;
    }
}

// TD_OK launched, 1 not applicable (the caller continues with the default kernels), < 0 error
int td_strip_try_launch(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int dtype,
                        const float* weights, const float* rcp_weights, float* x_out, void* x_buffer, int pdl, int max_ppc, void* stream) {
    std::lock_guard<std::mutex> lk(g_strip_mu);
    StripParams& p = g_strip_params;
    int nthreads = 0, smem1 = 0, strips = 0, smem = 0;
    if (strip_plan(g, batch_ptrs, num_batches, tile_bs, N, C, td_dtype_size(dtype), &p, &nthreads, &smem1, &strips) != 0) return 1;
    const int ppc = strip_pick_ppc(p, smem1, max_ppc, &smem);
    cudaStream_t st = (cudaStream_t)stream;
#define TD_STRIP_CASE(TYPE, RCP) \
    return ppc == 2 ? strip_dispatch<TYPE, 2>(p, strips, nthreads, smem, weights, RCP, x_out, x_buffer, pdl != 0, st) \
                    : strip_dispatch<TYPE, 1>(p, strips, nthreads, smem, weights, RCP, x_out, x_buffer, pdl != 0, st)
    switch (dtype) {
        case TD_F16: TD_STRIP_CASE(__half, rcp_weights);
        case TD_BF16: TD_STRIP_CASE(__nv_bfloat16, rcp_weights);
        case TD_F32: TD_STRIP_CASE(float, nullptr);
        default: return 1;
    }
#undef TD_STRIP_CASE
}

#ifdef TD_STRIP_HOST_EMULATION
// Test-only (tests/emul/strip_host_emul.cu): run every CTA of the strip kernel on the host, thread by thread, phase by phase.
template <typename T, int PPC>
static void emul_run(const StripParams& p, int strips, int nthreads, int smem_bytes, const float* weights, const float* rcp, float* out_f32,
                     void* out_buf) {
    unsigned char* smem = new unsigned char[smem_bytes + 16];
    for (int plane = 0; plane < p.NC; plane += PPC)
        for (int strip = 0; strip < strips; ++strip) {
            memset(smem, 0xCD, smem_bytes);       // stale shared memory must not matter
            for (int tid = 0; tid < nthreads; ++tid) strip_phase_table<T>(p, strip, plane, tid, smem);
            for (int tid = 0; tid < nthreads; ++tid) strip_phase_copy<T, PPC>(p, strip, tid, nthreads, smem);
            for (int tid = 0; tid < nthreads; ++tid) {
                if (out_buf != nullptr) {
                    if (rcp != nullptr && sizeof(T) == 2) strip_phase_consume<T, true, true, PPC>(p, strip, plane, tid, smem, weights, rcp, out_f32, (T*)out_buf);
                    else strip_phase_consume<T, true, false, PPC>(p, strip, plane, tid, smem, weights, nullptr, out_f32, (T*)out_buf);
                } else {
                    if (rcp != nullptr && sizeof(T) == 2) strip_phase_consume<T, false, true, PPC>(p, strip, plane, tid, smem, weights, rcp, out_f32, (T*)nullptr);
                    else strip_phase_consume<T, false, false, PPC>(p, strip, plane, tid, smem, weights, nullptr, out_f32, (T*)nullptr);
                }
            }
        }
    delete[] smem;
}

template <typename T>
static void emul_run_mod(const StripParams& p, int strips, int nthreads, int smem_bytes, const float* tile_weights, const float* rescale,
                         void* out_buf) {
    unsigned char* smem = new unsigned char[smem_bytes + 16];
    for (int plane = 0; plane < p.NC; ++plane)
        for (int strip = 0; strip < strips; ++strip) {
            memset(smem, 0xCD, smem_bytes);
            for (int tid = 0; tid < nthreads; ++tid) strip_phase_table<T>(p, strip, plane, tid, smem);
            for (int tid = 0; tid < nthreads; ++tid) strip_phase_copy<T>(p, strip, tid, nthreads, smem);
            for (int tid = 0; tid < nthreads; ++tid) strip_phase_consume_mod<T>(p, strip, plane, tid, smem, tile_weights, rescale, (T*)out_buf);
        }
    delete[] smem;
}

extern "C" int td_emul_strip_blend_mod(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int dtype,
                                       const float* tile_weights, const float* rescale, void* x_buffer) {
    static StripParams p;
    int nthreads = 0, smem = 0, strips = 0;
    if (strip_plan(g, batch_ptrs, num_batches, tile_bs, N, C, td_dtype_size(dtype), &p, &nthreads, &smem, &strips) != 0) return 1;
    if (dtype == TD_F16) emul_run_mod<__half>(p, strips, nthreads, smem, tile_weights, rescale, x_buffer);
    else if (dtype == TD_BF16) emul_run_mod<__nv_bfloat16>(p, strips, nthreads, smem, tile_weights, rescale, x_buffer);
    else emul_run_mod<float>(p, strips, nthreads, smem, tile_weights, rescale, x_buffer);
    return TD_OK;
}

extern "C" int td_emul_strip_blend(const td_grid* g, const void* const* batch_ptrs, int num_batches, int tile_bs, int N, int C, int dtype,
                                   const float* weights, const float* rcp_weights, float* x_out, void* x_buffer, int max_ppc, int* out_info) {
    static StripParams p;
    int nthreads = 0, smem1 = 0, strips = 0, smem = 0;
    if (strip_plan(g, batch_ptrs, num_batches, tile_bs, N, C, td_dtype_size(dtype), &p, &nthreads, &smem1, &strips) != 0) return 1;
    const int ppc = strip_pick_ppc(p, smem1, max_ppc, &smem);
    if (out_info != nullptr) { out_info[0] = strips; out_info[1] = nthreads; out_info[2] = smem; out_info[3] = ppc; }
#define TD_EMUL_CASE(TYPE, RCP) \
    do { if (ppc == 2) emul_run<TYPE, 2>(p, strips, nthreads, smem, weights, RCP, x_out, x_buffer); \
         else emul_run<TYPE, 1>(p, strips, nthreads, smem, weights, RCP, x_out, x_buffer); } while (0)
    if (dtype == TD_F16) TD_EMUL_CASE(__half, rcp_weights);
    else if (dtype == TD_BF16) TD_EMUL_CASE(__nv_bfloat16, rcp_weights);
    else TD_EMUL_CASE(float, nullptr);
#undef TD_EMUL_CASE
    return TD_OK;
}
#endif
