// Order-3 / order-9 step of the N = 3 * 2^k and 9 * 2^k transforms (see mixed_radix.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
namespace fecc {
// rows r*k2 + n1 of src (k2 < M, n1 < r)  ->  rows k2 + M*k1 of dst; s4 16-byte chunks per row, rows pitch4 chunks apart
cudaError_t launch_radix_pass(const uint32_t* src, uint32_t* dst, uint32_t pitch4, uint32_t s4, uint32_t r, uint32_t M, bool inverse, const uint4* tw, int num_sms, cudaStream_t st);
// step 2 of the Reed-Solomon encode of N = r * M blocks (M <= 2^19), in place on rows r*k2 + n1 of x (k2 < M, n1 < r)
cudaError_t launch_radix_encode(uint32_t* x, uint32_t pitch4, uint32_t s4, uint32_t r, uint32_t M, const uint4* tw, int num_sms, cudaStream_t st);
// step 2 of the encode of N = r * M blocks into N / (s * 2^log_d2) parity blocks (s | r, 2^log_d2 <= M), in place: folded by
// 2^log_fold (<= 2^log_d2), it leaves w_{s*u}[t] in row r*t + d_u for t < M / 2^log_fold, u < r / s
cudaError_t launch_radix_fold(uint32_t* x, uint32_t pitch4, uint32_t s4, uint32_t r, uint32_t M, uint32_t s, uint32_t log_d2, uint32_t log_fold,
                              const uint4* tw, int num_sms, cudaStream_t st);
}
