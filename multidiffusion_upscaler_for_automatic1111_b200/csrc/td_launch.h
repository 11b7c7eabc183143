// Host-side launch plumbing shared by the translation units of libtd_b200.so: kernel launch and its status, the
// per-device properties the launchers size their grids and shared memory from, the dynamic shared-memory opt-in, and the
// driver's tensor-map encoder.  Everything here is inline so that the host-emulation builds of td_strip.cu and
// td_jitter.cu (tests/emul) link without the rest of the library.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <map>
#include <mutex>
#include <utility>

#include "td_b200.h"
#include "td_internal.h"

namespace td {

// TD_OK, or TD_ERR_CUDA with "<what>: CUDA launch failed: <error>".  Reads (and so clears) the runtime's last error;
// `launch_err` is the status a cudaLaunchKernelEx call returned, if any.  Call it right after a <<<>>> launch.
inline int launch_status(const char* what, cudaError_t launch_err = cudaSuccess) {
    const cudaError_t last = cudaGetLastError();
    const cudaError_t e = launch_err != cudaSuccess ? launch_err : last;
    if (e != cudaSuccess) {
        td_set_error("%s: CUDA launch failed: %s", what, cudaGetErrorString(e));
        return TD_ERR_CUDA;
    }
    return TD_OK;
}

// Launch, with the programmatic-stream-serialisation attribute when `pdl` is set: inside a stream or a captured graph the
// kernel may then start while its predecessor drains (the kernel's pdl_wait() keeps stream order, td_device.cuh).
template <typename... KArgs, typename... Args>
int launch(const char* what, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl,
           const Args&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr = {};
    attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr.val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = pdl ? 1 : 0;
    return launch_status(what, cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...));
}

// SM count and the opt-in shared-memory limit per block of the current device, queried once per device.  ok == false:
// a query failed (each caller keeps its own fallback).
struct DeviceProps {
    int sms, smem_optin;
    bool ok;
};
inline DeviceProps device_props() {
    static std::mutex mu;
    static std::map<int, DeviceProps> cache;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return {0, 0, false}; }
    std::lock_guard<std::mutex> lk(mu);
    auto it = cache.find(dev);
    if (it != cache.end()) return it->second;
    DeviceProps d{0, 0, false};
    d.ok = cudaDeviceGetAttribute(&d.sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess &&
           cudaDeviceGetAttribute(&d.smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) == cudaSuccess && d.sms > 0;
    if (!d.ok) cudaGetLastError();
    cache[dev] = d;
    return d;
}

// Dynamic shared memory a kernel may request without opting in (48 KB minus its static allocation, with margin).
constexpr int kNoOptInSmem = 40 * 1024;

// Raise the kernel's dynamic shared-memory limit to `bytes` on the current device.  The attribute is per kernel and per
// device, so the size set is remembered per (kernel address, device) -- several instantiations share one function-pointer
// type -- and never lowered.  A no-op at or below kNoOptInSmem.  TD_OK, or TD_ERR_CUDA with the reason in td_last_error().
inline int smem_optin_bytes(const void* kernel, int bytes, const char* what) {
    if (bytes <= kNoOptInSmem) return TD_OK;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) {
        cudaGetLastError();
        td_set_error("%s: cudaGetDevice failed", what);
        return TD_ERR_CUDA;
    }
    static std::mutex mu;
    static std::map<std::pair<const void*, int>, int> configured;
    std::lock_guard<std::mutex> lk(mu);
    int& have = configured[{kernel, dev}];
    if (bytes <= have) return TD_OK;
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        td_set_error("%s: shared-memory opt-in (%d bytes) failed: %s", what, bytes, cudaGetErrorString(e));
        return TD_ERR_CUDA;
    }
    have = bytes;
    return TD_OK;
}
template <typename... KArgs>
int smem_optin(void (*kernel)(KArgs...), int bytes, const char* what) {
    return smem_optin_bytes(reinterpret_cast<const void*>(kernel), bytes, what);
}

// magic = ceil(2^32 / d) for fastdiv() (td_device.cuh), exact for operands < 2^16; 0 encodes d == 1
inline unsigned magic_u16(unsigned d) { return d <= 1 ? 0u : (unsigned)(((1ull << 32) + d - 1) / d); }

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda), looked up once.
// Null, with the reason in td_last_error(), when the driver does not provide it.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeTiledFn tensor_map_encoder() {
    static const EncodeTiledFn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
            return (EncodeTiledFn) nullptr;
        return (EncodeTiledFn)p;
    }();
    if (fn == nullptr) td_set_error("cuTensorMapEncodeTiled is not available from this driver");
    return fn;
}

}  // namespace td
