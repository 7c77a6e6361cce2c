// Update of a stored stripe in place when some data blocks change (include/fastecc_b200.h: fastecc_b200_rs_update, DESIGN 3h):
// the table T of one N and the two kernels of the direct path; api.cu chooses the path and runs the re-encode.
#pragma once
#include "context.h"

namespace fecc {
// T[t] = -2 / (N (rho^(2t+1) - 1)), t < N, rho = GF_Root(2N), as Barrett triples {w, whi, wlo, 0}: parity j' of the stripe is
// sum_i data_i * T[(D j' - i) mod N], D = N / M.  `T` holds N uint4.
cudaError_t launch_update_table(uint4* T, size_t N, cudaStream_t st);
// Changed row r < k (data row idx[r]): delta[r] = new[r] - data[idx[r]] (canonical, rows of s4 = ceil(size / 4) uint4), then
// data[idx[r]] = new[r] mod P, words [0, size) only.  delta = nullptr: only the data rows are written.
cudaError_t launch_update_delta(uint32_t* data, size_t dpitch, const uint32_t* nw, size_t npitch, uint4* delta, const uint32_t* idx, size_t k,
                                size_t size, int num_sms, cudaStream_t st);
// parity[j'] += sum_{r < k} delta[r] * T[(D j' - idx[r]) mod N] for j' < M, canonical, words [0, size) only.
cudaError_t launch_update_parity(uint32_t* parity, size_t ppitch, size_t M, const uint4* delta, const uint32_t* idx, size_t k, const uint4* T, size_t N,
                                 size_t size, cudaStream_t st);
}
