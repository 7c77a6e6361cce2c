#pragma once
#include <cuda_runtime.h>
#include "ntt_tile.cuh"
namespace fecc {
size_t      pass_smem_bytes(const PassParams& P, uint32_t tile_bytes);
// fills P.tables / P.table_set_stride and launches the kernel that writes table_bytes(P) bytes at `out`
cudaError_t launch_build_tables(PassParams& P, uint4* out, cudaStream_t stream);
// kernel (optional): receives the name of the kernel instantiation the pass was dispatched to (static storage)
cudaError_t launch_pass(const PassParams& P, int num_sms, cudaStream_t stream, const char** kernel = nullptr);
}
