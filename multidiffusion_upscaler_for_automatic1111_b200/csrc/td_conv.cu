// Tiled-VAE convolutions and attention GEMMs on the Hopper tensor cores (sm_90a, wgmma):
//   the conv / upsample / downsample / attention tasks the reference executes at scripts/tilevae.py:618 through
//   third-party ldm modules (3x3 s1 p1 convs, 1x1 nin_shortcut / q / k / v / proj_out, nearest x2 + conv,
//   pad(0,1,0,1) + 3x3 s2 conv; tile_utils/attn.py:49-72 QK^T and PV) as ONE implicit-GEMM kernel:
//
//       D[pixel, co] = alpha * sum_{tap, ci} A[pixel + offset(tap), ci] * W[tap][co][ci]  + bias  (+ residual)
//
// Design:
//   * activations NHWC fp16 / bf16 (channels innermost): a 3x3 tap is a shifted 4-D TMA box {64 ch, BW, BH, 1} of the
//     SAME tensor -- signed start coordinates, out-of-bounds rows / columns zero-filled by the TMA unit = the
//     convolution's zero padding, no im2col buffer, no halo handling in software.  BW x BH = 128 output pixels = the
//     tile's M dimension; a stride-2 convolution is the same box with element strides {1,2,2,1};
//   * the box lands in shared memory as 128 rows x 128 bytes, 128-byte swizzled = the K-major wgmma operand layout;
//     weights [tap][Cout][Cin] load the same way ({64, BN, 1} boxes);
//   * warp roles: warp 8 is the TMA producer (one elected thread), warps 0-3 and 4-7 are two consumer warpgroups that
//     each issue wgmma.m64nBNk16 for 64 of the 128 pixel rows (four per 64-channel stage) and keep the 64 x BN fp32
//     accumulator tile in registers (BN / 2 per thread, <= 128: 288 threads leave 224 registers each);
//   * epilogue straight from the accumulator registers: alpha / bias / residual (/ frozen GroupNorm + SiLU) in fp32,
//     one rounding to fp16 / bf16, stores clipped to the output tensor; it overlaps the producer's loads of the next
//     tile;
//   * persistent: one CTA per SM walks the (pixel tile, Cout block) list, up to 8-stage smem ring (mbarrier full / empty).
// A plain GEMM (attention: S = Q K^T, O = P V, V^T = Wv X^T) is the 1x1 "image" with H = 1, W = M.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "td_b200.h"
#include "td_internal.h"
#include "td_tma.cuh"
#include "td_wgmma.cuh"

namespace {

using namespace td;

constexpr int kConvThreads = 288;         // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int kConvBM = 128;              // output pixels per tile
constexpr int kConvBK = 64;               // channels per stage (128 bytes of fp16 = one swizzle row)
constexpr int kConvStageA = kConvBM * kConvBK * 2;   // 16 KB
constexpr int kConvMaxStages = 8;

struct ConvParams {
    int taps_x, taps_y;        // kw, kh
    int stride;                // 1 or 2
    int pad_left, pad_top;
    int OW, OH, NI;            // grid of output pixels the tiles walk, and its "image" count
    int Cin_chunks;            // ceil(Cin / 64)
    int Cout;                  // real output channels (bias / residual / store guard)
    int n_blocks;              // ceil(Cout / BN)
    int BW, BH;                // pixel patch of one tile: BW * BH == 128 (16 x 8 image rows, 8 x 16, or 128 x 1 for a GEMM)
    int tiles_x, tiles_y;
    int num_tiles;             // NI * tiles_y * tiles_x * n_blocks
    int stages;
    int is_bf16;
    int bias_per_row;          // bias indexed by output pixel (GEMM row) instead of channel
    int post_act;              // with post_scale / post_shift: 1 = SiLU after the per-channel affine
    float alpha;
    int up2;                   // 1: nearest-2x upsample folded into the 3x3 convolution -- four 2x2 convolutions of the LOW-resolution
                               // image, one per output parity (py, px) = "image" index (py * 2 + px); weights [16 taps, Cout, Cin];
                               // tile pixel (x, y) of parity (py, px) is output pixel (2 x + px, 2 y + py)
    long long y_pitch, y2_pitch, res_pitch;   // elements between pixels
};

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_3d_u32(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ uint32_t pack2(float a, float b, int is_bf16) {
    if (is_bf16) {
        __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&h);
    }
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float unpack_lo(uint32_t w, int is_bf16) {
    return is_bf16 ? __uint_as_float(w << 16) : __half2float(__ushort_as_half((unsigned short)(w & 0xffffu)));
}
__device__ __forceinline__ float unpack_hi(uint32_t w, int is_bf16) {
    return is_bf16 ? __uint_as_float(w & 0xffff0000u) : __half2float(__ushort_as_half((unsigned short)(w >> 16)));
}

struct TileCoord { int img, py, px, nb; };
// work list: Cout block fastest, then pixel tile (consecutive CTAs read the same activation box from L2)
__device__ __forceinline__ TileCoord decode_tile(const ConvParams& p, int g) {
    TileCoord c;
    c.nb = g % p.n_blocks;
    int m = g / p.n_blocks;
    c.px = m % p.tiles_x; m /= p.tiles_x;
    c.py = m % p.tiles_y;
    c.img = m / p.tiles_y;
    return c;
}

// one output element pair (channels co, co + 1) of pixel row `off` (elements): fp32 -> dtype, clipped at Cout
__device__ __forceinline__ void store_pair(uint16_t* base, long long off, int co, int cout, float a, float b, int is_bf16) {
    const uint32_t w = pack2(a, b, is_bf16);
    if (co + 1 < cout) *reinterpret_cast<uint32_t*>(base + off + co) = w;
    else base[off + co] = (uint16_t)(w & 0xffffu);
}

template <int BN, bool BF16>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b, const __grid_constant__ ConvParams p,
                 const float* __restrict__ bias, const uint16_t* __restrict__ residual, const float* __restrict__ post_scale,
                 const float* __restrict__ post_shift, uint16_t* __restrict__ y, uint16_t* __restrict__ y2) {
    extern __shared__ unsigned char conv_smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[kConvMaxStages], empty_bar[kConvMaxStages];
    const uint32_t smem0 = (smem_u32(conv_smem_raw) + 1023u) & ~1023u;      // SWIZZLE_128B needs 1024-byte alignment
    constexpr uint32_t stage_bytes = (uint32_t)(kConvStageA + BN * 128);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }   // one arrive per consumer warpgroup
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        fence_proxy_async();
    }
    __syncthreads();
    const int ksteps = p.taps_x * p.taps_y * p.Cin_chunks;

    if (warp == 8) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            tma_prefetch_desc(&map_a); tma_prefetch_desc(&map_b);
            int stage = 0; uint32_t phase = 0;
            for (int g = blockIdx.x; g < p.num_tiles; g += gridDim.x) {
                const TileCoord c = decode_tile(p, g);
                // up2: output parity (py, px) shifts the 2x2 window by one low-resolution pixel and selects its 4 folded taps
                const int par = p.up2 ? c.img : 0;
                const int img = p.up2 ? 0 : c.img;
                const int x0 = c.px * p.BW * p.stride - p.pad_left + (par & 1);
                const int y0 = c.py * p.BH * p.stride - p.pad_top + (par >> 1);
                int tap = par * 4;
                for (int ty = 0; ty < p.taps_y; ++ty)
                    for (int tx = 0; tx < p.taps_x; ++tx, ++tap)
                        for (int kc = 0; kc < p.Cin_chunks; ++kc) {
                            mbar_wait(&empty_bar[stage], phase ^ 1u);
                            const uint32_t sa = smem0 + (uint32_t)stage * stage_bytes;
                            mbar_arrive_expect_tx(&full_bar[stage], stage_bytes);
                            tma_load_4d(sa, &map_a, kc * kConvBK, x0 + tx, y0 + ty, img, &full_bar[stage]);
                            tma_load_3d_u32(sa + kConvStageA, &map_b, kc * kConvBK, c.nb * BN, tap, &full_bar[stage]);
                            if (++stage == p.stages) { stage = 0; phase ^= 1u; }
                        }
            }
        }
        return;
    }

    // ===================== consumers: wgmma into registers, then the epilogue =====================
    const int wg = warp >> 2;                 // rows [64 wg, 64 wg + 64) of the tile
    const bool signal = (threadIdx.x & 127) == 0;
    float acc[BN / 2];
    int stage = 0; uint32_t phase = 0;
    for (int g = blockIdx.x; g < p.num_tiles; g += gridDim.x) {
        const TileCoord c = decode_tile(p, g);
        int prev = -1;
        for (int ks = 0; ks < ksteps; ++ks) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t sa = smem0 + (uint32_t)stage * stage_bytes;
            const uint64_t da = wgmma_desc_sw128(sa + (uint32_t)(wg * 64 * 128));
            const uint64_t db = wgmma_desc_sw128(sa + kConvStageA);
            wgmma_fence_acc(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < kConvBK / 16; ++k) {    // +32 bytes along K inside the swizzle row = +2 in the address field
                Wgmma<BN, BF16>::mma(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (ks | k) != 0 ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<1>();                          // the previous k-step's MMAs have read their stage: hand it back
            wgmma_fence_acc(acc);
            if (prev >= 0 && signal) mbar_arrive(&empty_bar[prev]);
            prev = stage;
            if (++stage == p.stages) { stage = 0; phase ^= 1u; }
        }
        wgmma_wait<0>();
        wgmma_fence_acc(acc);
        if (signal) mbar_arrive(&empty_bar[prev]);

        // accumulator rows of this thread: r0 and r0 + 8; columns 8 j + 2 (lane % 4) + {0, 1}
        const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        const int cq = 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = r0 + 8 * h;
            const int ly = row / p.BW, lx = row - ly * p.BW;
            const int ox = c.px * p.BW + lx, oy = c.py * p.BH + ly;
            if (ox >= p.OW || oy >= p.OH || c.img >= p.NI) continue;
            const long long pix = ((long long)c.img * p.OH + oy) * p.OW + ox;
            // output pixel: the parity view of the 2x-upsampled image when up2 (one image, N = 1), else the tile pixel
            const long long opix = p.up2 ? (long long)(2 * oy + (c.img >> 1)) * (2 * p.OW) + 2 * ox + (c.img & 1) : pix;
            const float bb = (bias != nullptr && p.bias_per_row) ? __ldg(bias + pix) : 0.0f;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int co = c.nb * BN + 8 * j + cq;
                if (co >= p.Cout) continue;
                const bool two = co + 1 < p.Cout;
                float b0 = bb, b1 = bb;
                if (bias != nullptr && !p.bias_per_row) { b0 = __ldg(bias + co); b1 = two ? __ldg(bias + co + 1) : 0.0f; }
                float v0 = __fmaf_rn(acc[4 * j + 2 * h], p.alpha, b0);
                float v1 = __fmaf_rn(acc[4 * j + 2 * h + 1], p.alpha, b1);
                if (residual != nullptr) {
                    const uint16_t* rp = residual + pix * p.res_pitch + co;
                    const uint32_t rw = two ? __ldg(reinterpret_cast<const unsigned int*>(rp)) : (uint32_t)__ldg(reinterpret_cast<const unsigned short*>(rp));
                    v0 += unpack_lo(rw, p.is_bf16);
                    v1 += unpack_hi(rw, p.is_bf16);
                }
                if (y2 != nullptr) store_pair(y, opix * p.y_pitch, co, p.Cout, v0, v1, p.is_bf16);   // the unnormalised result
                if (post_scale != nullptr) {
                    // the GroupNorm (+ SiLU) that follows this convolution, statistics frozen (fast mode):
                    // y = act(v * scale[c] + shift[c]) on the fp32 accumulator, before the one rounding to fp16
                    v0 = __fmaf_rn(v0, __ldg(post_scale + co), __ldg(post_shift + co));
                    if (two) v1 = __fmaf_rn(v1, __ldg(post_scale + co + 1), __ldg(post_shift + co + 1));
                    if (p.post_act) {
                        v0 = __fdividef(v0, 1.0f + __expf(-v0));
                        v1 = __fdividef(v1, 1.0f + __expf(-v1));
                    }
                }
                if (y2 != nullptr) store_pair(y2, opix * p.y2_pitch, co, p.Cout, v0, v1, p.is_bf16);
                else store_pair(y, opix * p.y_pitch, co, p.Cout, v0, v1, p.is_bf16);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------- host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn conv_encode_fn() {
    static EncodeTiledFn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
            return (EncodeTiledFn) nullptr;
        return (EncodeTiledFn)p;
    }();
    return fn;
}

template <int BN> bool conv_smem_optin(int bytes) {
    return cudaFuncSetAttribute(conv_gemm_kernel<BN, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) == cudaSuccess &&
           cudaFuncSetAttribute(conv_gemm_kernel<BN, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) == cudaSuccess;
}

struct ConvDev { int sms; int smem_optin; bool ok; };
ConvDev conv_dev() {
    static std::mutex mu;
    static ConvDev cache[64];
    static bool have[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return {0, 0, false};
    std::lock_guard<std::mutex> lk(mu);
    if (!have[dev]) {
        ConvDev d{0, 0, false};
        d.ok = cudaDeviceGetAttribute(&d.sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess &&
               cudaDeviceGetAttribute(&d.smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) == cudaSuccess;
        if (d.ok) {   // the opt-in limit covers static + dynamic shared memory: leave room for the kernel's static part
            cudaFuncAttributes fa;
            if (cudaFuncGetAttributes(&fa, conv_gemm_kernel<256, false>) != cudaSuccess) { cudaGetLastError(); d.ok = false; }
            else {
                d.smem_optin -= (int)fa.sharedSizeBytes;
                if (!conv_smem_optin<16>(d.smem_optin) || !conv_smem_optin<32>(d.smem_optin) || !conv_smem_optin<64>(d.smem_optin) ||
                    !conv_smem_optin<128>(d.smem_optin) || !conv_smem_optin<256>(d.smem_optin)) {
                    cudaGetLastError();
                    d.ok = false;
                }
            }
        }
        cache[dev] = d;
        have[dev] = true;
    }
    return cache[dev];
}

}  // namespace

int td_encode_map(CUtensorMap* out, const void* base, int is_bf16, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box, const uint32_t* estr, bool swizzle128, const char* what) {
    EncodeTiledFn fn = conv_encode_fn();
    if (fn == nullptr) { td_set_error("cuTensorMapEncodeTiled is not available from this driver"); return TD_ERR_CUDA; }
    cuuint64_t d[5]; cuuint64_t s[4]; cuuint32_t b[5]; cuuint32_t e[5];
    for (int i = 0; i < rank; ++i) { d[i] = dims[i]; b[i] = box[i]; e[i] = estr[i]; }
    for (int i = 0; i + 1 < rank; ++i) s[i] = strides_bytes[i];
    const CUresult r = fn(out, is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank,
                          const_cast<void*>(base), d, s, b, e, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        td_set_error("cuTensorMapEncodeTiled failed (%d) for %s: dims [%llu,%llu,%llu,%llu] box [%u,%u,%u,%u]", (int)r, what,
                     (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)(rank > 2 ? dims[2] : 0),
                     (unsigned long long)(rank > 3 ? dims[3] : 0), box[0], box[1], rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
        return TD_ERR_CUDA;
    }
    return TD_OK;
}

namespace {
// up2 = 1: `d` describes nearest-2x upsample + 3x3 / pad 1 (OH = 2 H, OW = 2 W) of ONE image; `w` holds the 16 folded taps.
int conv_run(const td_conv_desc* d, const void* x, const void* w, const float* bias, const void* residual, void* y, void* stream, int up2,
             size_t y2_off = 0) {
    if (d == nullptr || x == nullptr || w == nullptr || y == nullptr) { td_set_error("td_conv2d_nhwc: null argument"); return TD_ERR_INVALID_ARG; }
    if (d->dtype != TD_F16 && d->dtype != TD_BF16) { td_set_error("td_conv2d_nhwc: dtype must be fp16 or bf16"); return TD_ERR_UNSUPPORTED; }
    if (d->N <= 0 || d->H <= 0 || d->W <= 0 || d->OH <= 0 || d->OW <= 0 || d->Cin <= 0 || d->Cout <= 0) { td_set_error("td_conv2d_nhwc: non-positive size"); return TD_ERR_INVALID_ARG; }
    if (d->Cin % 8 != 0) { td_set_error("td_conv2d_nhwc: Cin (%d) must be a multiple of 8", d->Cin); return TD_ERR_UNSUPPORTED; }
    if ((d->kh != 1 && d->kh != 3) || d->kh != d->kw || (d->stride != 1 && d->stride != 2)) { td_set_error("td_conv2d_nhwc: only 1x1 / 3x3, stride 1 / 2"); return TD_ERR_UNSUPPORTED; }
    if (up2 && (d->kh != 3 || d->stride != 1 || d->pad_top != 1 || d->pad_left != 1 || d->OH != 2 * d->H || d->OW != 2 * d->W || d->N != 1 ||
                residual != nullptr || d->bias_per_row)) {
        td_set_error("td_upconv2x_nhwc: describes upsample(2x nearest) + 3x3 / stride 1 / pad 1 (OH = 2H, OW = 2W), no residual, bias per channel");
        return TD_ERR_INVALID_ARG;
    }
    // grid of output pixels the tiles walk: the low-resolution image (once per output parity) when the upsample is folded
    const int gOW = up2 ? d->W : d->OW, gOH = up2 ? d->H : d->OH, gN = up2 ? 4 : d->N;
    if (d->x_pitch < d->Cin || d->x_pitch % 8 != 0 || d->y_pitch < d->Cout || d->y_pitch % 8 != 0 || d->w_pitch < d->Cin || d->w_pitch % 8 != 0 ||
        (residual != nullptr && (d->res_pitch < d->Cout || d->res_pitch % 8 != 0))) {
        td_set_error("td_conv2d_nhwc: pitches must cover the channels and be multiples of 8 elements (16 bytes)");
        return TD_ERR_INVALID_ARG;
    }
    for (const void* ptr : {x, w, (const void*)y, residual, (const void*)(d->bias_per_row ? nullptr : bias), (const void*)d->post_scale, (const void*)d->post_shift})
        if (ptr != nullptr && (reinterpret_cast<uintptr_t>(ptr) & 15u) != 0) { td_set_error("td_conv2d_nhwc: tensors (and per-channel vectors) must be 16-byte aligned"); return TD_ERR_INVALID_ARG; }
    if (d->y2 != nullptr && (d->post_scale == nullptr || d->post_shift == nullptr || d->y2_pitch < d->Cout || d->y2_pitch % 8 != 0 ||
                             (reinterpret_cast<uintptr_t>(d->y2) & 15u) != 0)) {
        td_set_error("td_conv2d_nhwc: y2 needs post_scale / post_shift, a 16-byte aligned pointer and a pitch >= Cout in multiples of 8");
        return TD_ERR_INVALID_ARG;
    }
    if ((d->post_scale == nullptr) != (d->post_shift == nullptr)) { td_set_error("td_conv2d_nhwc: post_scale and post_shift come together"); return TD_ERR_INVALID_ARG; }
    const ConvDev dev = conv_dev();
    if (!dev.ok) { td_set_error("td_conv2d_nhwc: device query / shared-memory opt-in failed"); return TD_ERR_CUDA; }

    ConvParams p;
    std::memset(&p, 0, sizeof(p));
    p.taps_x = up2 ? 2 : d->kw; p.taps_y = up2 ? 2 : d->kh; p.stride = d->stride; p.pad_left = d->pad_left; p.pad_top = d->pad_top;
    p.OW = gOW; p.OH = gOH; p.NI = gN; p.up2 = up2;
    p.Cin_chunks = (d->Cin + 63) / 64;   // a partial last chunk is zero-filled by the TMA unit on BOTH operands
    p.Cout = d->Cout;
    int bn = 256;
    if (d->Cout < 256) { bn = 16; while (bn < d->Cout) bn *= 2; }
    p.n_blocks = (d->Cout + bn - 1) / bn;
    // pixel tile (128 pixels): wide for a GEMM (H == 1), 16 x 8 for images, 8 x 16 for narrow ones
    if (gOH == 1) { p.BW = 128; p.BH = 1; }
    else if (gOW >= 16) { p.BW = 16; p.BH = 8; }
    else { p.BW = 8; p.BH = 16; }
    p.tiles_x = (gOW + p.BW - 1) / p.BW;
    p.tiles_y = (gOH + p.BH - 1) / p.BH;
    const long long mt = (long long)gN * p.tiles_x * p.tiles_y;
    if (mt * p.n_blocks > 0x3fffffffLL) { td_set_error("td_conv2d_nhwc: too many tiles"); return TD_ERR_UNSUPPORTED; }
    p.num_tiles = (int)(mt * p.n_blocks);
    p.is_bf16 = d->dtype == TD_BF16;
    p.bias_per_row = d->bias_per_row;
    p.post_act = d->post_act;
    p.alpha = d->alpha;
    p.y_pitch = d->y_pitch;
    p.y2_pitch = d->y2 != nullptr ? d->y2_pitch : 0;
    p.res_pitch = residual != nullptr ? d->res_pitch : 0;
    const int stage_bytes = kConvStageA + bn * 128;
    p.stages = std::min(kConvMaxStages, (dev.smem_optin - 1024) / stage_bytes);
    if (p.stages < 2) { td_set_error("td_conv2d_nhwc: not enough shared memory"); return TD_ERR_UNSUPPORTED; }
    const size_t smem = (size_t)p.stages * stage_bytes + 1024;

    alignas(64) CUtensorMap ma, mb;
    {
        const uint64_t dims[4] = {(uint64_t)d->Cin, (uint64_t)d->W, (uint64_t)d->H, (uint64_t)d->N};
        const uint64_t str[3] = {(uint64_t)d->x_pitch * 2, (uint64_t)d->W * d->x_pitch * 2, (uint64_t)d->H * d->W * d->x_pitch * 2};
        const uint32_t box[4] = {64, (uint32_t)(p.BW * d->stride), (uint32_t)(p.BH * d->stride), 1};
        const uint32_t es[4] = {1, (uint32_t)d->stride, (uint32_t)d->stride, 1};
        const int rc = td_encode_map(&ma, x, p.is_bf16, 4, dims, str, box, es, true, "activations");
        if (rc != TD_OK) return rc;
    }
    {
        const uint64_t dims[3] = {(uint64_t)d->Cin, (uint64_t)d->Cout, (uint64_t)(up2 ? 16 : d->kh * d->kw)};
        const uint64_t str[2] = {(uint64_t)d->w_pitch * 2, (uint64_t)d->Cout * d->w_pitch * 2};
        const uint32_t box[3] = {64, (uint32_t)bn, 1};
        const uint32_t es[3] = {1, 1, 1};
        const int rc = td_encode_map(&mb, w, p.is_bf16, 3, dims, str, box, es, true, "weights");
        if (rc != TD_OK) return rc;
    }
    uint16_t* yo = static_cast<uint16_t*>(y);
    uint16_t* y2o = d->y2 != nullptr ? static_cast<uint16_t*>(d->y2) + (up2 ? y2_off : 0) : nullptr;
    const int grid = std::min(p.num_tiles, dev.sms);
    const uint16_t* res = static_cast<const uint16_t*>(residual);
    cudaStream_t st = (cudaStream_t)stream;
#define TD_CONV_LAUNCH(BN)                                                                                                          \
    (p.is_bf16 ? conv_gemm_kernel<BN, true><<<grid, kConvThreads, smem, st>>>(ma, mb, p, bias, res, d->post_scale, d->post_shift, yo, y2o) \
               : conv_gemm_kernel<BN, false><<<grid, kConvThreads, smem, st>>>(ma, mb, p, bias, res, d->post_scale, d->post_shift, yo, y2o))
    switch (bn) {
        case 16: TD_CONV_LAUNCH(16); break;
        case 32: TD_CONV_LAUNCH(32); break;
        case 64: TD_CONV_LAUNCH(64); break;
        case 128: TD_CONV_LAUNCH(128); break;
        default: TD_CONV_LAUNCH(256); break;
    }
#undef TD_CONV_LAUNCH
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { td_set_error("td_conv2d_nhwc: launch failed: %s", cudaGetErrorString(e)); return TD_ERR_CUDA; }
    return TD_OK;
}
}  // namespace

extern "C" int td_conv2d_nhwc(const td_conv_desc* d, const void* x, const void* w, const float* bias, const void* residual,
                              void* y, void* stream) {
    return conv_run(d, x, w, bias, residual, y, stream, 0);
}

extern "C" int td_upconv2x_nhwc(const td_conv_desc* d, const void* x, const void* w16, const float* bias, void* y, void* stream) {
    if (d == nullptr || x == nullptr || y == nullptr) { td_set_error("td_upconv2x_nhwc: null argument"); return TD_ERR_INVALID_ARG; }
    td_conv_desc one = *d;
    one.N = 1;
    for (int n = 0; n < d->N; ++n) {
        const uint16_t* xn = static_cast<const uint16_t*>(x) + (size_t)n * d->H * d->W * d->x_pitch;
        uint16_t* yn = static_cast<uint16_t*>(y) + (size_t)n * d->OH * d->OW * d->y_pitch;
        const int rc = conv_run(&one, xn, w16, bias, nullptr, yn, stream, 1, (size_t)n * d->OH * d->OW * (size_t)d->y2_pitch);
        if (rc != TD_OK) return rc;
    }
    return TD_OK;
}
