// What the library's translation units share beyond the C ABI: the error path of the entry points, the context's power table
// and SM count (api.cu), the owner of a pattern's device arrays, and the launch shape of the grid-stride kernels.
#pragma once
#include "../../include/fastecc_b200.h"
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <vector>

namespace fecc {

// Records the message for fastecc_b200_last_error() (per thread) and returns `code`.
int fail(int code, const char* fmt, ...);
// g^e, e in [0, 2^20), and the SM count of the context's device; nullptr / 0 before fastecc_b200_init().
const uint4* context_power_table();
int          context_num_sms();

// Consumes the CUDA runtime's per-thread last error once the library has handled or reported a failed runtime call.  Left
// pending, it would come back from the cudaGetLastError() that checks every launch, and a later call on the same thread would
// report the old failure for a launch that did happen.
inline void clear_cuda_error() { (void)cudaGetLastError(); }

// The return code of a failed runtime call `what`: FASTECC_B200_ENOMEM for an allocation failure, FASTECC_B200_ECUDA otherwise.
inline int cuda_fail(cudaError_t e, const char* what)
{
    clear_cuda_error();
    return fail(e == cudaErrorMemoryAllocation ? FASTECC_B200_ENOMEM : FASTECC_B200_ECUDA, "%s: %s", what, cudaGetErrorString(e));
}

// Device arrays freed with their owner (a pattern, or the temporaries of one pattern build).  An array of n = 0 elements gets
// one, so that every pointer is valid; a failed allocation returns nullptr and sets `failed`.
struct DeviceArrays {
    std::vector<void*> p;
    bool failed = false;
    DeviceArrays() = default;
    DeviceArrays(const DeviceArrays&) = delete;
    DeviceArrays& operator=(const DeviceArrays&) = delete;
    ~DeviceArrays() { for (void* q : p) cudaFree(q); }
    template <class T> T* alloc(size_t n)
    {
        void* q = nullptr;
        if (cudaMalloc(&q, (n ? n : 1) * sizeof(T)) != cudaSuccess) { clear_cuda_error(); failed = true; return nullptr; }
        p.push_back(q);
        return (T*)q;
    }
};

// Blocks of 256 threads for a grid-stride loop over n items: one item per thread, at most `cap` blocks, at least one.
inline unsigned grid_size(size_t n, size_t cap)
{
    const size_t blocks = (n + 255) / 256;
    return (unsigned)(blocks < cap ? (blocks ? blocks : 1) : cap);
}

#if defined(__CUDACC__)
// Words [w, w + 4) of `row`, of which only those below `size` are written: 16-byte stores, scalar ones in a partial last group.
__device__ __forceinline__ void store_row(uint32_t* row, size_t w, const uint4& v, size_t size)
{
    if (w + 4 <= size) { *reinterpret_cast<uint4*>(row + w) = v; return; }
    if (w < size) row[w] = v.x;
    if (w + 1 < size) row[w + 1] = v.y;
    if (w + 2 < size) row[w + 2] = v.z;
}
#endif

} // namespace fecc

#define CUDA_TRY(expr) do { const cudaError_t e_ = (expr); if (e_ != cudaSuccess) return ::fecc::cuda_fail(e_, #expr); } while (0)
#define TRY_RC(expr) do { if (const int rc_ = (expr)) return rc_; } while (0)
// i = this thread's first item, then every gridDim.x * blockDim.x-th, while below n; T is the index type.
#define FOR_GRID(T, i, n) for (T i = blockIdx.x * (T)blockDim.x + threadIdx.x; i < (n); i += (T)gridDim.x * blockDim.x)
