// Degraded read of a stored stripe (include/fastecc_b200.h: fastecc_b200_rs_reconstruct, DESIGN 3k): the two kernels of one call;
// api.cu chooses the parity rows J, computes the combination B on the host and runs them per column chunk.
#pragma once
#include "context.h"

namespace fecc {
// ws[k * 4 s4 + w] += sum_{i < N, i not lost} T[(D pos[k] - i) mod N] * data_i[w] for k < K <= 32, w < 4 s4, s4 = ceil(size / 4),
// as canonical partial sums added into the 64-bit words of ws (zeroed by the caller).  T: update.h's table of order N; lost: the
// a <= 32 lost data rows, ascending, never loaded.  Pad words up to 4 s4 are read and summed like the others.
cudaError_t launch_reconstruct_sum(const uint32_t* data, size_t dpitch, size_t N, size_t D, const uint4* T, const uint32_t* pos, size_t K,
                                   const uint32_t* lost, size_t a, size_t size, unsigned long long* ws, int num_sms, cudaStream_t st);
// Output row q < n_out, words [0, size): [q >= n_data] * r_(a + q - n_data) + sum_{j < a} B[q a + j] * (parity[pos[j]] - r_j), canonical,
// r_k = ws row k mod P; B: Barrett triples {w, whi, wlo, 0}.  Reads the a parity rows pos[0 .. a) only.
cudaError_t launch_reconstruct_combine(const unsigned long long* ws, const uint32_t* parity, size_t ppitch, const uint32_t* pos, size_t a, const uint4* B,
                                       size_t n_out, size_t n_data, uint32_t* out, size_t opitch, size_t size, int num_sms, cudaStream_t st);
}
