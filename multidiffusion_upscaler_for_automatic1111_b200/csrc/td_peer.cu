// Multi-GPU plumbing for the tile-sharded sampler step (one process per GPU):
//   * exchange buffers that every rank maps from its peers through CUDA IPC (NVLink / NVSwitch P2P),
//   * a step-counter signal written straight into the peers' flag arrays,
// so that the blend kernel can wait for its peers and read their tile outputs over NVLink in the
// SAME kernel that blends them (td_blend_multidiffusion_peer in td_diffusion.cu): no NCCL call, no
// gathered copy.  The reference has no multi-GPU path at all (SURVEY.md section 5).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstring>

#include "td_b200.h"
#include "td_device.cuh"
#include "td_internal.h"
#include "td_launch.h"

namespace {

struct SignalTable {
    uint32_t* ptrs[TD_MAX_PEERS];
};

// One warp: bump this rank's device-side step counter, then publish the new value into slot `rank`
// of every rank's flag array (release, system scope).  Keeping the counter on the device makes the
// launch replayable inside a CUDA graph (no host-supplied step number in the parameters).
__global__ void peer_signal_kernel(const __grid_constant__ SignalTable tbl, int world, int rank, uint32_t* step_counter) {
    const int t = threadIdx.x;
    uint32_t v = 0;
    if (t == 0) {
        v = *step_counter + 1u;
        *step_counter = v;
    }
    v = __shfl_sync(0xffffffffu, v, 0);
    if (t >= world) return;
    __threadfence_system();  // everything this GPU wrote before the signal is visible system-wide first
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(tbl.ptrs[t] + rank), "r"(v) : "memory");
}

// One warp: lane i spins until flags[i] >= *value (acquire, system scope).  Stream-ordered work after this kernel sees
// everything the signalling ranks wrote before their td_peer_signal.  Bounded spin: a missing peer traps (launch error).
__global__ void peer_wait_kernel(const uint32_t* flags, int count, const uint32_t* value) {
    const int t = threadIdx.x;
    if (t >= count) return;
    td::spin_until_ge(flags + t, *value);
}


// Halo push of the row-strip shard in ONE launch of TD_PUSH_CTAS CTAs: up to TD_MAX_PUSH_REGIONS strided 2-D regions are
// copied with 128-bit plain stores into peer memory (NVLink); then EVERY CTA publishes its share on its own -- CTA
// barrier, one `red.release.sys.add 1` per target into slot `rank` of the target's flag array -- so the data and the
// signal cost ONE NVLink round trip (a ticket + a single final release store costs two: measured 12.5 us vs 9.3 us
// for the three-launch form).  A slot therefore advances by TD_PUSH_CTAS per step and so do the waiters' `expect`
// counters: "slot >= expect" means all of that sender's CTAs have landed.
//   expect_own : bumped by TD_PUSH_CTAS when the kernel starts (CTA 0); with wait_count > 0, CTA 0 then waits until
//                wait_flags[i] >= *expect_own for i < wait_count -- stream-ordered work behind the launch sees the peers' pushes
//   bump_next  : another expect counter bumped by TD_PUSH_CTAS when CTA 0 is done (the tile-halo set's, by the latent-halo
//                push that ends a step: the blend that waits on it runs on this stream, the tile-halo push may not)
struct PushTable {
    td_push_region r[TD_MAX_PUSH_REGIONS];
    long long vec_end[TD_MAX_PUSH_REGIONS];   // exclusive prefix ends, in 16-byte vectors
    int n;
    uint32_t* targets[TD_MAX_PEERS];          // &flags_of_target[rank]
    int n_targets;
    uint32_t* expect_own;
    const uint32_t* wait_flags;
    int wait_count;
    uint32_t* bump_next;
};

__global__ void __launch_bounds__(256)
push_regions_kernel(const __grid_constant__ PushTable t) {
    __shared__ uint32_t s_want;
    if (blockIdx.x == 0 && threadIdx.x == 0 && t.expect_own != nullptr) {
        const uint32_t w = *t.expect_own + (uint32_t)TD_PUSH_CTAS;
        *t.expect_own = w;
        s_want = w;
    }
    const long long total = t.n > 0 ? t.vec_end[t.n - 1] : 0;
    const long long stride = (long long)gridDim.x * blockDim.x;
    // four independent 128-bit copies in flight per thread: NVLink stores need the depth, not the CTA count
    for (long long base = (long long)blockIdx.x * blockDim.x + threadIdx.x; base < total; base += 4 * stride) {
        uint4 val[4];
        unsigned char* dstp[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const long long i = base + u * stride;
            dstp[u] = nullptr;
            if (i >= total) continue;
            int k = 0;
            while (i >= t.vec_end[k]) ++k;
            const td_push_region& r = t.r[k];
            const long long j = i - (k > 0 ? t.vec_end[k - 1] : 0);
            const long long vpr = r.row_bytes >> 4;
            const long long row = j / vpr, v = j - row * vpr;
            const long long pl = row / r.rows, rr = row - pl * r.rows;
            val[u] = *reinterpret_cast<const uint4*>(static_cast<const unsigned char*>(r.src) + pl * r.src_plane_bytes + rr * r.src_pitch_bytes + v * 16);
            dstp[u] = static_cast<unsigned char*>(r.dst) + pl * r.dst_plane_bytes + rr * r.dst_pitch_bytes + v * 16;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (dstp[u] != nullptr) *reinterpret_cast<uint4*>(dstp[u]) = val[u];
    }
    __syncthreads();    // every thread's peer stores are ordered before the releases below (cumulative)
    if ((int)threadIdx.x < t.n_targets)
        asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(t.targets[threadIdx.x]), "r"(1u) : "memory");
    if (blockIdx.x != 0 || threadIdx.x >= 32) return;
    if ((int)threadIdx.x < t.wait_count) td::spin_until_ge(t.wait_flags + threadIdx.x, s_want);
    __syncwarp();
    if (threadIdx.x == 0 && t.bump_next != nullptr) *t.bump_next += (uint32_t)TD_PUSH_CTAS;
}

int cuda_fail(const char* what, cudaError_t e) {
    td_set_error("%s: %s", what, cudaGetErrorString(e));
    return TD_ERR_CUDA;
}

}  // namespace

extern "C" int td_dev_alloc(int64_t bytes, void** out) {
    if (bytes <= 0 || out == nullptr) { td_set_error("td_dev_alloc: bad arguments"); return TD_ERR_INVALID_ARG; }
    cudaError_t e = cudaMalloc(out, (size_t)bytes);
    if (e != cudaSuccess) return cuda_fail("td_dev_alloc", e);
    e = cudaMemset(*out, 0, (size_t)bytes);
    if (e != cudaSuccess) return cuda_fail("td_dev_alloc (memset)", e);
    return TD_OK;
}

extern "C" int td_dev_free(void* ptr) {
    if (ptr == nullptr) return TD_OK;
    cudaError_t e = cudaFree(ptr);
    return e == cudaSuccess ? TD_OK : cuda_fail("td_dev_free", e);
}

extern "C" int td_ipc_get_handle(const void* dev_ptr, void* handle_out) {
    if (dev_ptr == nullptr || handle_out == nullptr) { td_set_error("td_ipc_get_handle: null"); return TD_ERR_INVALID_ARG; }
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, const_cast<void*>(dev_ptr));
    if (e != cudaSuccess) return cuda_fail("td_ipc_get_handle", e);
    static_assert(sizeof(h) == TD_IPC_HANDLE_BYTES, "cudaIpcMemHandle_t size");
    std::memcpy(handle_out, &h, sizeof(h));
    return TD_OK;
}

extern "C" int td_ipc_open(const void* handle, void** dev_ptr_out) {
    if (handle == nullptr || dev_ptr_out == nullptr) { td_set_error("td_ipc_open: null"); return TD_ERR_INVALID_ARG; }
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handle, sizeof(h));
    cudaError_t e = cudaIpcOpenMemHandle(dev_ptr_out, h, cudaIpcMemLazyEnablePeerAccess);
    return e == cudaSuccess ? TD_OK : cuda_fail("td_ipc_open", e);
}

extern "C" int td_ipc_close(void* dev_ptr) {
    if (dev_ptr == nullptr) return TD_OK;
    cudaError_t e = cudaIpcCloseMemHandle(dev_ptr);
    return e == cudaSuccess ? TD_OK : cuda_fail("td_ipc_close", e);
}

extern "C" int td_peer_signal(void* const* flag_ptrs, int world, int rank, uint32_t* step_counter, void* stream) {
    if (flag_ptrs == nullptr || step_counter == nullptr || world <= 0 || world > TD_MAX_PEERS || rank < 0 || rank >= world) {
        td_set_error("td_peer_signal: bad arguments (world=%d rank=%d)", world, rank);
        return TD_ERR_INVALID_ARG;
    }
    SignalTable tbl;
    for (int i = 0; i < world; ++i) {
        if (flag_ptrs[i] == nullptr) { td_set_error("td_peer_signal: flag_ptrs[%d] is null", i); return TD_ERR_INVALID_ARG; }
        tbl.ptrs[i] = (uint32_t*)flag_ptrs[i];
    }
    peer_signal_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(tbl, world, rank, step_counter);
    return td::launch_status("td_peer_signal");
}

extern "C" int td_peer_wait(const uint32_t* flags, int count, const uint32_t* value, void* stream) {
    if (count < 0 || count > TD_MAX_PEERS || (count > 0 && (flags == nullptr || value == nullptr))) {
        td_set_error("td_peer_wait: bad arguments");
        return TD_ERR_INVALID_ARG;
    }
    if (count == 0) return TD_OK;
    peer_wait_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(flags, count, value);
    return td::launch_status("td_peer_wait");
}

extern "C" int td_push_regions(const td_push_region* regions, int n_regions, void* const* target_slots, int n_targets,
                               uint32_t* expect_own, const uint32_t* wait_flags, int wait_count, uint32_t* bump_next, void* stream) {
    if (n_regions < 0 || n_regions > TD_MAX_PUSH_REGIONS || (n_regions > 0 && regions == nullptr) || n_targets < 0 ||
        n_targets > TD_MAX_PEERS || (n_targets > 0 && target_slots == nullptr) || wait_count < 0 || wait_count > TD_MAX_PEERS ||
        (wait_count > 0 && (wait_flags == nullptr || expect_own == nullptr))) {
        td_set_error("td_push_regions: bad arguments (n_regions=%d n_targets=%d wait_count=%d)", n_regions, n_targets, wait_count);
        return TD_ERR_INVALID_ARG;
    }
    PushTable t;
    std::memset(&t, 0, sizeof(t));
    long long total = 0;
    for (int k = 0; k < n_regions; ++k) {
        const td_push_region& r = regions[k];
        const uintptr_t bits = reinterpret_cast<uintptr_t>(r.src) | reinterpret_cast<uintptr_t>(r.dst) | (uintptr_t)r.row_bytes |
                               (uintptr_t)r.src_plane_bytes | (uintptr_t)r.src_pitch_bytes | (uintptr_t)r.dst_plane_bytes | (uintptr_t)r.dst_pitch_bytes;
        if (r.src == nullptr || r.dst == nullptr || r.planes <= 0 || r.rows <= 0 || r.row_bytes <= 0 || (bits & 15u) != 0) {
            td_set_error("td_push_regions: region %d must be non-empty with 16-byte aligned pointers, pitches and row length", k);
            return TD_ERR_INVALID_ARG;
        }
        t.r[k] = r;
        total += (long long)r.planes * r.rows * (r.row_bytes >> 4);
        t.vec_end[k] = total;
    }
    t.n = n_regions;
    for (int i = 0; i < n_targets; ++i) {
        if (target_slots[i] == nullptr) { td_set_error("td_push_regions: target_slots[%d] is null", i); return TD_ERR_INVALID_ARG; }
        t.targets[i] = (uint32_t*)target_slots[i];
    }
    t.n_targets = n_targets; t.expect_own = expect_own; t.wait_flags = wait_flags; t.wait_count = wait_count; t.bump_next = bump_next;
    push_regions_kernel<<<TD_PUSH_CTAS, 256, 0, (cudaStream_t)stream>>>(t);
    return td::launch_status("td_push_regions");
}
