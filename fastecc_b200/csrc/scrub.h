// Scrub of a stored stripe (include/fastecc_b200.h: fastecc_b200_rs_scrub, DESIGN 3i): the fold of every row into two words, the
// element-wise kernels on single-column rows and Berlekamp-Massey; api.cu runs them around the encode and the transforms.
#pragma once
#include "context.h"
#include <vector>

namespace fecc {
// Workspace rows are 4 words (16 bytes): rows [0, N) the data side, rows [N, N + M) the parity side.
// fold: zeroes nothing; adds, for m < N + M and f in {0, 1}, sum_c r_f,c * row_m[c] (c < size, row m = data m or parity m - N)
// into the 64-bit word f of workspace row m (64-bit adds of canonical partial sums; the caller zeroes the rows first).
cudaError_t launch_scrub_fold(const uint32_t* data, size_t dpitch, size_t N, const uint32_t* parity, size_t ppitch, size_t M, size_t size,
                              uint64_t seed, uint32_t* ws, int num_sms, cudaStream_t st);
// degraded fold (fastecc_b200_rs_scrub_degraded, DESIGN 3j): the same, but the data rows with lost[m] != 0 and the parity rows
// with cs[j].x == 0 (a repair pattern's d_lost and d_cs) are never loaded and add nothing; lost = nullptr: the plain fold
cudaError_t launch_degraded_fold(const uint32_t* data, size_t dpitch, size_t N, const uint32_t* parity, size_t ppitch, size_t M, size_t size,
                                 uint64_t seed, const uint8_t* lost, const uint4* cs, uint32_t* ws, int num_sms, cudaStream_t st);
// degraded syndrome: j < M: u_j = (ws[N + j] - ws[j]) * cs[j] (words 0, 1) into rows N + j and j
cudaError_t launch_degraded_syndrome(uint32_t* ws, size_t N, size_t M, const uint4* cs, cudaStream_t st);
// degraded roots: launch_scrub_roots over the rows i < n with lost[i] == 0 and cs[i].x != 0 (a null mask skips nothing)
cudaError_t launch_degraded_roots(const uint32_t* ws, size_t n, const uint8_t* lost, const uint4* cs, uint32_t* list, uint32_t* count, size_t cap,
                                  cudaStream_t st);
// reduce: the two 64-bit sums of rows [0, n) -> words {a0 mod P, a1 mod P, 0, 0}
cudaError_t launch_scrub_reduce(uint32_t* ws, size_t n, cudaStream_t st);
// syndrome: j < M: s_j = ws[N + j] - ws[j] (words 0, 1) into rows N + j and j; *nonzero = 1 if any s_j != 0
cudaError_t launch_scrub_syndrome(uint32_t* ws, size_t N, size_t M, uint32_t* nonzero, cudaStream_t st);
// roots: the rows i < n whose word 0 is zero, appended to list[0, cap) by an atomic counter *count (which counts them all)
cudaError_t launch_scrub_roots(const uint32_t* ws, size_t n, uint32_t* list, uint32_t* count, size_t cap, cudaStream_t st);
// product: j < M: ws[j] words 0, 1 = ws[j].word0 * ws[N + j] words 0, 1
cudaError_t launch_scrub_product(uint32_t* ws, size_t N, size_t M, cudaStream_t st);
// check: *fail = 1 if words 0 or 1 of a row k in [L, M) are nonzero
cudaError_t launch_scrub_check(const uint32_t* ws, size_t L, size_t M, uint32_t* fail, cudaStream_t st);
// Berlekamp-Massey over GF(P): the shortest C (C[0] = 1) with sum_i C[i] s[k - i] = 0 for k in [L, s.size()); returns L, and C
// without trailing zero coefficients.
size_t berlekamp_massey(const std::vector<uint32_t>& s, std::vector<uint32_t>& C);
}
