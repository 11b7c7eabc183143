// Fused single-head attention of the tiled VAE's mid-block (tile_utils/attn.py:49-72) on the Hopper tensor cores
// (sm_90a, wgmma):
//
//       O[t, :] = softmax(alpha * Q[t, :] K^T) V,   Q, K, V, O token-major [T, C] fp16 / bf16, fp32 accumulation
//
// with an online (running max / running sum) softmax, so nothing of size T x T is ever written: the memory a call
// needs is its four [T, C] operands, whatever T is.
//
// Design (C = 64 .. 512 in steps of 64 channels, "chunks" of one 128-byte swizzle row; the kernel is instantiated for
// 2 NC chunks, NC = ceil(C / 128), and the chunk past an odd C / 64 reads zeros from the TMA unit and is not stored):
//   * one CTA per 64-query block; its Q block stays resident in shared memory (C / 64 boxes {64 ch, 64 rows});
//   * warp 8 is the TMA producer: K and V blocks of 64 keys stream through an mbarrier full / empty ring, one stage
//     per block (K_0, V_0, K_1, V_1, ...); keys past T are zero-filled by the TMA unit, the inputs are not padded;
//   * warps 0-3 and 4-7 are two consumer warpgroups that split C: warpgroup w owns chunks [w NC, w NC + NC).
//     A 64 x 512 fp32 O block is 256 registers per thread for one warpgroup; the kernel has 168 (288 threads), so
//     above C = 384 each CTA produces one 256-channel slice of O (blockIdx.y), 64 accumulators per thread, and S is
//     computed once per slice (1.5x the tensor-core work of the unsplit form);
//       - each computes its partial S_w = Q[:, chunks_w] K[:, chunks_w]^T (wgmma m64n64k16, both operands in shared
//         memory); the two 64 x 64 fp32 partials are exchanged through shared memory and summed (fp32 addition is
//         commutative, so both warpgroups hold bit-identical S and apply the same softmax);
//       - keys past T are masked with -inf, then the running max / sum update and the O rescale;
//       - P (rounded to fp16 / bf16) goes straight from the S registers into the A operand of
//         O[:, out_w] += P V[:, out_w] (wgmma with A in registers, V read MN-major from the same swizzled boxes);
//   * the epilogue divides by the row sum and stores O from the registers, rows past T clipped; offsets are 64-bit.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstring>

#include "td_b200.h"
#include "td_internal.h"
#include "td_tma.cuh"
#include "td_wgmma.cuh"

namespace {

using namespace td;

constexpr int kAttnThreads = 288;          // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int kAttnRows = 64;              // queries per CTA = keys per K / V block
constexpr int kAttnChunkBytes = 64 * 128;  // one {64 channels, 64 rows} box: 64 rows of 128 bytes
constexpr int kAttnMaxChunks = 8;          // C <= 512
constexpr int kAttnMaxStages = 8;
constexpr int kAttnXchgBytes = 2 * 32 * 128 * 4;   // each warpgroup's 64 x 64 fp32 partial S, 32 values per thread

struct AttnParams {
    int T, C;
    int stages;
    int key_blocks;       // ceil(T / 64)
    float scale_log2;     // alpha * log2(e): the softmax runs on exp2
    long long o_pitch;
};

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void attn_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// the 256 consumer threads only (the producer warp has returned)
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

template <bool BF16> __device__ __forceinline__ uint32_t pack_pair(float a, float b) {
    if constexpr (BF16) {
        __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&h);
    } else {
        __half2 h = __floats2half2_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&h);
    }
}

// NC: 64-channel chunks per warpgroup for S, C <= 128 NC; chunks past C read zeros (TMA fill) and are not stored.
// NO: O chunks per warpgroup; blockIdx.y picks the slice of 2 NO output chunks (NO < NC: S is recomputed per slice).
template <bool BF16, int NC, int NO>
__global__ void __launch_bounds__(kAttnThreads, 1)
attn_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
            const __grid_constant__ AttnParams p, uint16_t* __restrict__ o) {
    extern __shared__ unsigned char attn_smem_raw[];
    __shared__ __align__(8) uint64_t full_bar[kAttnMaxStages], empty_bar[kAttnMaxStages], q_bar;
    const uint32_t smem0 = (smem_u32(attn_smem_raw) + 1023u) & ~1023u;      // SWIZZLE_128B needs 1024-byte alignment
    constexpr uint32_t stage_bytes = (uint32_t)(2 * NC * kAttnChunkBytes);
    const uint32_t sq = smem0;                                               // the Q block: one stage's size
    const uint32_t ring = smem0 + stage_bytes;
    float* xchg = reinterpret_cast<float*>(attn_smem_raw + (ring + (uint32_t)p.stages * stage_bytes - smem_u32(attn_smem_raw)));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * kAttnRows;
    const int obeg = blockIdx.y * 2 * NO;      // first output chunk of this CTA

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }   // one arrive per consumer warpgroup
        mbar_init(&q_bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        fence_proxy_async();
    }
    __syncthreads();

    if (warp == 8) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_q)) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_k)) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_v)) : "memory");
            mbar_arrive_expect_tx(&q_bar, stage_bytes);
            for (int c = 0; c < 2 * NC; ++c) tma_load_2d(sq + (uint32_t)(c * kAttnChunkBytes), &map_q, c * 64, q0, &q_bar);
            int stage = 0; uint32_t phase = 0;
            for (int j = 0; j < p.key_blocks; ++j)
                for (int kv = 0; kv < 2; ++kv) {
                    mbar_wait(&empty_bar[stage], phase ^ 1u);
                    const uint32_t sa = ring + (uint32_t)stage * stage_bytes;
                    if (kv == 0) {
                        mbar_arrive_expect_tx(&full_bar[stage], stage_bytes);
                        for (int c = 0; c < 2 * NC; ++c) tma_load_2d(sa + (uint32_t)(c * kAttnChunkBytes), &map_k, c * 64, j * kAttnRows, &full_bar[stage]);
                    } else {                       // only this CTA's slice of V
                        mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)(2 * NO * kAttnChunkBytes));
                        for (int c = 0; c < 2 * NO; ++c)
                            tma_load_2d(sa + (uint32_t)(c * kAttnChunkBytes), &map_v, (obeg + c) * 64, j * kAttnRows, &full_bar[stage]);
                    }
                    if (++stage == p.stages) { stage = 0; phase ^= 1u; }
                }
        }
        return;
    }

    // ===================== consumers =====================
    const int wg = warp >> 2;
    const int t = threadIdx.x & 127;
    const bool signal = t == 0;
    const int cbeg = wg * NC;
    float* xmine = xchg + wg * (32 * 128);
    const float* xother = xchg + (1 - wg) * (32 * 128);
    // accumulator rows of this thread: r and r + 8 of the block; columns 8 j + 2 (lane % 4) + {0, 1}
    const int r = (warp & 3) * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);

    float acc[NO][32];
#pragma unroll
    for (int cc = 0; cc < NO; ++cc)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[cc][i] = 0.0f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.0f, l1 = 0.0f;   // running max (log2 domain) / partial sum, rows r, r + 8

    mbar_wait(&q_bar, 0);
    int stage = 0; uint32_t phase = 0;
    for (int j = 0; j < p.key_blocks; ++j) {
        // ---- partial S over this warpgroup's channels, in two 32-key halves straight to shared memory: 128 O
        //      registers leave no room for a 64 x 64 S block in registers next to P
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sk = ring + (uint32_t)stage * stage_bytes;
        uint32_t sq_j = sq;
        asm volatile("" : "+r"(sq_j));        // keeps the loop-invariant Q descriptors from being hoisted into registers
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float s[16];
            wgmma_fence_acc(s);
            wgmma_fence();
#pragma unroll
            for (int cc = 0; cc < NC; ++cc) {
                const uint32_t off = (uint32_t)((cbeg + cc) * kAttnChunkBytes);
                const uint64_t da = wgmma_desc_sw128(sq_j + off), db = wgmma_desc_sw128(sk + off + (uint32_t)(h * 32 * 128));
#pragma unroll
                for (int k = 0; k < 4; ++k)      // +32 bytes along K inside the swizzle row = +2 in the address field
                    Wgmma<32, BF16>::mma(s, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (cc | k) != 0 ? 1u : 0u);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_acc(s);
            // thread-major (conflict-free); index 16 h + i = the accumulator index of the full 64-key block
#pragma unroll
            for (int i = 0; i < 16; ++i) xmine[(16 * h + i) * 128 + t] = s[i];
        }
        if (signal) attn_arrive(&empty_bar[stage]);
        if (++stage == p.stages) { stage = 0; phase ^= 1u; }
        consumers_sync();

        // ---- S = S_0 + S_1, online softmax in the log2 domain, keys past T masked
        const int kb = j * kAttnRows;
        const bool tail = kb + kAttnRows > p.T;
        // S value i of this thread: key column 8 (i / 4) + cq + (i % 2), row r + 8 ((i / 2) % 2)
        auto logit = [&](int i) {
            const float v = (xmine[i * 128 + t] + xother[i * 128 + t]) * p.scale_log2;
            return (tail && kb + 8 * (i >> 2) + cq + (i & 1) >= p.T) ? -INFINITY : v;
        };
        float mx0 = m0, mx1 = m1;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            if (i & 2) mx1 = fmaxf(mx1, logit(i));
            else mx0 = fmaxf(mx0, logit(i));
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float corr0 = exp2f(m0 - mx0), corr1 = exp2f(m1 - mx1);   // 0 on the first block (m = -inf)
        m0 = mx0; m1 = mx1;
        // P as the A operand: keys 16 kk .. 16 kk + 15 are S values 8 kk .. 8 kk + 7, pairs (row r, r + 8, r, r + 8)
        uint32_t pa[4][4];
        float ls0 = 0.0f, ls1 = 0.0f;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int i = 8 * kk + 2 * e;
                const float mx = (e & 1) ? mx1 : mx0;
                const float a = exp2f(logit(i) - mx), b = exp2f(logit(i + 1) - mx);
                if (e & 1) ls1 += a + b;
                else ls0 += a + b;
                pa[kk][e] = pack_pair<BF16>(a, b);
            }
        consumers_sync();                      // both warpgroups have read this block's partials before the next are written
        l0 = l0 * corr0 + ls0;
        l1 = l1 * corr1 + ls1;
#pragma unroll
        for (int cc = 0; cc < NO; ++cc)
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                acc[cc][4 * jj] *= corr0; acc[cc][4 * jj + 1] *= corr0;
                acc[cc][4 * jj + 2] *= corr1; acc[cc][4 * jj + 3] *= corr1;
            }

        // ---- O[:, this warpgroup's channels] += P V
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sv = ring + (uint32_t)stage * stage_bytes;
#pragma unroll
        for (int cc = 0; cc < NO; ++cc) wgmma_fence_acc(acc[cc]);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)            // 16 keys = two 8-row groups = 2048 bytes
#pragma unroll
            for (int cc = 0; cc < NO; ++cc)
                WgmmaRsT64<BF16>::mma(acc[cc], pa[kk], wgmma_desc_sw128(sv + (uint32_t)((wg * NO + cc) * kAttnChunkBytes + kk * 2048)), 1u);
        wgmma_commit();
        wgmma_wait<0>();
#pragma unroll
        for (int cc = 0; cc < NO; ++cc) wgmma_fence_acc(acc[cc]);
        if (signal) attn_arrive(&empty_bar[stage]);
        if (++stage == p.stages) { stage = 0; phase ^= 1u; }
    }

    // ---- epilogue: O / rowsum, one rounding, rows past T clipped
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
    const long long row0 = (long long)q0 + r;
#pragma unroll
    for (int cc = 0; cc < NO; ++cc) {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
            const int col = (obeg + wg * NO + cc) * 64 + 8 * jj + cq;
            if (col >= p.C) continue;                 // C % 64 == 0: whole chunks only
            if (row0 < p.T)
                *reinterpret_cast<uint32_t*>(o + row0 * p.o_pitch + col) = pack_pair<BF16>(acc[cc][4 * jj] * inv0, acc[cc][4 * jj + 1] * inv0);
            if (row0 + 8 < p.T)
                *reinterpret_cast<uint32_t*>(o + (row0 + 8) * p.o_pitch + col) =
                    pack_pair<BF16>(acc[cc][4 * jj + 2] * inv1, acc[cc][4 * jj + 3] * inv1);
        }
    }
}

int encode_operand(CUtensorMap* m, const void* base, int is_bf16, int T, int C, int64_t pitch, const char* what) {
    const uint64_t dims[2] = {(uint64_t)C, (uint64_t)T};
    const uint64_t str[1] = {(uint64_t)pitch * 2};
    const uint32_t box[2] = {64, (uint32_t)kAttnRows};
    const uint32_t es[2] = {1, 1};
    return td_encode_map(m, base, is_bf16, 2, dims, str, box, es, true, what);
}

// one launch of the <BF16, NC> form: shared-memory opt-in (per call: the call is one per VAE tile) and the ring depth
template <bool BF16, int NC, int NO>
int attn_launch(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv, AttnParams p, uint16_t* o, cudaStream_t st) {
    int dev = 0, optin = 0;
    cudaFuncAttributes fa;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
        cudaFuncGetAttributes(&fa, attn_kernel<BF16, NC, NO>) != cudaSuccess) {
        cudaGetLastError();
        td_set_error("td_attention: device / kernel query failed");
        return TD_ERR_CUDA;
    }
    optin -= (int)fa.sharedSizeBytes;        // the opt-in limit covers static + dynamic shared memory
    constexpr int stage_bytes = 2 * NC * kAttnChunkBytes;
    p.stages = std::min(kAttnMaxStages, (optin - 1024 - stage_bytes - kAttnXchgBytes) / stage_bytes);
    if (p.stages < 2) { td_set_error("td_attention: not enough shared memory"); return TD_ERR_UNSUPPORTED; }
    const int smem = 1024 + (1 + p.stages) * stage_bytes + kAttnXchgBytes;
    if (cudaFuncSetAttribute(attn_kernel<BF16, NC, NO>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) {
        cudaGetLastError();
        td_set_error("td_attention: shared-memory opt-in (%d bytes) failed", smem);
        return TD_ERR_CUDA;
    }
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, attn_kernel<BF16, NC, NO>, kAttnThreads, smem) != cudaSuccess || per_sm < 1) {
        cudaGetLastError();
        td_set_error("td_attention: the kernel (%d registers, %d bytes of shared memory) does not fit on an SM", fa.numRegs, smem);
        return TD_ERR_UNSUPPORTED;
    }
    attn_kernel<BF16, NC, NO><<<dim3(p.key_blocks, NC / NO), kAttnThreads, smem, st>>>(mq, mk, mv, p, o);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { td_set_error("td_attention: launch failed: %s", cudaGetErrorString(e)); return TD_ERR_CUDA; }
    return TD_OK;
}

template <bool BF16>
int attn_dispatch(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv, const AttnParams& p, uint16_t* o, cudaStream_t st) {
    switch ((p.C + 127) / 128) {
        case 1: return attn_launch<BF16, 1, 1>(mq, mk, mv, p, o, st);
        case 2: return attn_launch<BF16, 2, 2>(mq, mk, mv, p, o, st);
        case 3: return attn_launch<BF16, 3, 3>(mq, mk, mv, p, o, st);
        // C > 384: O in two 256-channel slices (64 accumulators per thread, not 128: the kernel has 168 registers)
        default: return attn_launch<BF16, 4, 2>(mq, mk, mv, p, o, st);
    }
}

}  // namespace

extern "C" int td_attention(const void* q, const void* k, const void* v, void* o, int T, int C, int64_t q_pitch, int64_t k_pitch,
                            int64_t v_pitch, int64_t o_pitch, float alpha, int dtype, void* stream) {
    if (q == nullptr || k == nullptr || v == nullptr || o == nullptr) { td_set_error("td_attention: null argument"); return TD_ERR_INVALID_ARG; }
    if (dtype != TD_F16 && dtype != TD_BF16) { td_set_error("td_attention: dtype must be fp16 or bf16"); return TD_ERR_UNSUPPORTED; }
    if (T <= 0 || C <= 0) { td_set_error("td_attention: non-positive size"); return TD_ERR_INVALID_ARG; }
    if (C % 64 != 0 || C > 64 * kAttnMaxChunks) { td_set_error("td_attention: C (%d) must be a multiple of 64 and <= 512", C); return TD_ERR_UNSUPPORTED; }
    for (int64_t pitch : {q_pitch, k_pitch, v_pitch, o_pitch})
        if (pitch < C || pitch % 8 != 0) { td_set_error("td_attention: pitches must cover C and be multiples of 8 elements (16 bytes)"); return TD_ERR_INVALID_ARG; }
    for (const void* ptr : {q, k, v, (const void*)o})
        if ((reinterpret_cast<uintptr_t>(ptr) & 15u) != 0) { td_set_error("td_attention: tensors must be 16-byte aligned"); return TD_ERR_INVALID_ARG; }

    AttnParams p;
    std::memset(&p, 0, sizeof(p));
    p.T = T;
    p.C = C;
    p.key_blocks = (T + kAttnRows - 1) / kAttnRows;
    p.scale_log2 = alpha * 1.4426950408889634f;
    p.o_pitch = o_pitch;
    const bool bf16 = dtype == TD_BF16;
    alignas(64) CUtensorMap mq, mk, mv;
    int rc = encode_operand(&mq, q, bf16, T, C, q_pitch, "q");
    if (rc == TD_OK) rc = encode_operand(&mk, k, bf16, T, C, k_pitch, "k");
    if (rc == TD_OK) rc = encode_operand(&mv, v, bf16, T, C, v_pitch, "v");
    if (rc != TD_OK) return rc;
    uint16_t* out = static_cast<uint16_t*>(o);
    cudaStream_t st = (cudaStream_t)stream;
    return bf16 ? attn_dispatch<true>(mq, mk, mv, p, out, st) : attn_dispatch<false>(mq, mk, mv, p, out, st);
}
