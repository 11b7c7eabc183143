// Host side of the TMA path: tensor-map encoding through the driver entry point
// (no link-time dependency on libcuda) with a small cache keyed by the tensor.
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstring>
#include <mutex>

#include "td_b200.h"
#include "td_internal.h"
#include "td_launch.h"
#include "td_tma.cuh"

namespace {

struct Key {
    const void* base;
    int dtype;
    uint64_t planes, rows, cols;
    uint32_t box_rows, box_cols;
    bool operator==(const Key& o) const {
        return base == o.base && dtype == o.dtype && planes == o.planes && rows == o.rows && cols == o.cols &&
               box_rows == o.box_rows && box_cols == o.box_cols;
    }
};
constexpr int kCache = 512;
struct Entry {
    Key key;
    bool used;
    alignas(64) CUtensorMap map;
};
Entry g_cache[kCache];
int g_next = 0;
std::mutex g_mu;

}  // namespace

int td_encode_tensor_map_3d(CUtensorMap* out, const void* base, int dtype, uint64_t planes, uint64_t rows, uint64_t cols,
                            uint32_t box_rows, uint32_t box_cols) {
    const Key key{base, dtype, planes, rows, cols, box_rows, box_cols};
    {
        std::lock_guard<std::mutex> lk(g_mu);
        for (int i = 0; i < kCache; ++i)
            if (g_cache[i].used && g_cache[i].key == key) {
                std::memcpy(out, &g_cache[i].map, sizeof(CUtensorMap));
                return TD_OK;
            }
    }
    const td::EncodeTiledFn fn = td::tensor_map_encoder();
    if (fn == nullptr) return TD_ERR_CUDA;
    const int es = td_dtype_size(dtype);
    const CUtensorMapDataType dt = dtype == TD_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                 : dtype == TD_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    const cuuint64_t dims[3] = {cols, rows, planes};
    const cuuint64_t strides[2] = {cols * (uint64_t)es, rows * cols * (uint64_t)es};  // bytes, dims 1..2
    const cuuint32_t box[3] = {box_cols, box_rows, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    alignas(64) CUtensorMap m;
    CUresult r = fn(&m, dt, 3, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        td_set_error("tensor-map encoding failed (%d) for [%llu,%llu,%llu] box [%u,%u]", (int)r,
                     (unsigned long long)planes, (unsigned long long)rows, (unsigned long long)cols, box_rows, box_cols);
        return TD_ERR_CUDA;
    }
    std::memcpy(out, &m, sizeof(CUtensorMap));
    {
        std::lock_guard<std::mutex> lk(g_mu);
        Entry& e = g_cache[g_next];
        g_next = (g_next + 1) % kCache;
        e.key = key;
        e.used = true;
        std::memcpy(&e.map, &m, sizeof(CUtensorMap));
    }
    return TD_OK;
}
