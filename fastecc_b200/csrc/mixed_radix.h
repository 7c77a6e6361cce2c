// Order-3 / order-9 step of the N = 3 * 2^k and 9 * 2^k transforms (see mixed_radix.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
namespace fecc {
// The orders of the library: n = r * 2^log2_m with r in {1, 3, 9}; r = 0 if n is of no such form.
struct Order { uint32_t r, log2_m; };
inline Order split_order(size_t n)
{
    uint32_t l = 0;
    while (n && !(n & 1)) { n >>= 1; ++l; }
    return {n == 1 || n == 3 || n == 9 ? (uint32_t)n : 0u, l};
}
// The CRT split of a root of order r * 2^log2_m (r odd): a = (2^log2_m)^-1 mod r, b = r^-1 mod 2^log2_m (Newton: r*b = 1 mod 2^k).
struct CrtSplit { uint32_t a, b; };
inline CrtSplit crt_split(uint32_t r, uint32_t log2_m)
{
    const uint64_t m = 1ull << log2_m;
    uint32_t a = 0;
    while (a < r && (uint64_t)a * (m % r) % r != 1 % r) ++a;
    uint64_t b = 1;
    for (uint32_t i = 0; i < log2_m; ++i) b = b * (2 - (r * b) % m + m) % m;
    return {a, (uint32_t)(b % m)};
}

// rows r*k2 + n1 of src (k2 < M, n1 < r)  ->  rows k2 + M*k1 of dst; s4 16-byte chunks per row, rows pitch4 chunks apart
cudaError_t launch_radix_pass(const uint32_t* src, uint32_t* dst, uint32_t pitch4, uint32_t s4, uint32_t r, uint32_t M, bool inverse, const uint4* tw, int num_sms, cudaStream_t st);
// step 2 of the Reed-Solomon encode of N = r * M blocks (M <= 2^19), in place on rows r*k2 + n1 of x (k2 < M, n1 < r)
cudaError_t launch_radix_encode(uint32_t* x, uint32_t pitch4, uint32_t s4, uint32_t r, uint32_t M, const uint4* tw, int num_sms, cudaStream_t st);
// step 2 of the encode of N = r * M blocks into N / (s * 2^log_d2) parity blocks (s | r, 2^log_d2 <= M), in place: folded by
// 2^log_fold (<= 2^log_d2), it leaves w_{s*u}[t] in row r*t + d_u for t < M / 2^log_fold, u < r / s
cudaError_t launch_radix_fold(uint32_t* x, uint32_t pitch4, uint32_t s4, uint32_t r, uint32_t M, uint32_t s, uint32_t log_d2, uint32_t log_fold,
                              const uint4* tw, int num_sms, cudaStream_t st);
}
