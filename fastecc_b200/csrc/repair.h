// Repair of a stored stripe (N data rows + M parity rows of fastecc_b200_rs_encode_asym_mixed[_dev]): the pattern and the four
// element-wise kernels of repair.cu; the sequence that runs them around the encode and the transforms is in api.cu.
#pragma once
#include "context.h"

namespace fecc {
// Everything that depends only on which blocks are lost (DESIGN 3g), as finish_repair_kernel fills it.  Per-row constants are
// Barrett triples {w, whi, wlo, 0} (gf::make_tw) of canonical w.
struct RepairTables {
    size_t N = 0, M = 0, ned = 0, nep = 0;
    uint32_t* d_ed = nullptr;        // [ned] lost data rows, ascending
    uint32_t* d_ep = nullptr;        // [nep] lost parity rows, ascending
    uint8_t*  d_lost = nullptr;      // [N]   1 on the lost data rows
    uint4*    d_cs = nullptr;        // [M]   -l(y_j') / 2: the syndrome scale, 0 exactly on the lost parity rows
    uint4*    d_cr = nullptr;        // [M]   rho^-k / M
    uint4*    d_ck = nullptr;        // [M]   k
    uint4*    d_cd = nullptr;        // [ned] N / D[2e]
    uint4*    d_cp = nullptr;        // [nep] -2 / (M * D[2Dj' + 1])
};
}

struct fastecc_b200_repair : fecc::RepairTables {
    fecc::DeviceArrays mem;          // owns the arrays of the tables
};

namespace fecc {
// All four work on a column chunk of `cols` words starting at word c0 (a multiple of 4) of the caller's rows, against a workspace
// of pitch wpitch words (rows [0, N) data side, rows [N, N + M) the k * P_k rows).  The caller's rows are written at words
// [c0, min(c0 + cols, size)) only.
// load: ws[i] = data[i] mod P, or 0 on a lost data row (lost[i] != 0), i < N; lost = nullptr: no row is lost
cudaError_t launch_repair_load(size_t N, const uint8_t* lost, const uint32_t* data, size_t dpitch, size_t c0, uint32_t* ws, size_t wpitch,
                               size_t cols, int num_sms, cudaStream_t st);
// syndrome: j' < M surviving: ws[j'] = (parity[j'] - ws[j']) * cs[j'];  lost (cs[j'] = 0): parity[j'] = ws[j'] (= G_j'), ws[j'] = 0;
// cs = nullptr: parity[j'] = ws[j'] for every j' < M, the workspace untouched (the store of a re-encode)
cudaError_t launch_repair_syndrome(size_t M, const uint4* cs, uint32_t* parity, size_t ppitch, size_t c0, size_t size, uint32_t* ws, size_t wpitch,
                                   size_t cols, int num_sms, cudaStream_t st);
// split: k < M: ws[N + k] = k * ws[k] (if parity was lost), ws[k] *= cr[k];  ws[M .. N) = 0 (if data was lost)
cudaError_t launch_repair_split(const fastecc_b200_repair* R, uint32_t* ws, size_t wpitch, size_t cols, int num_sms, cudaStream_t st);
// scatter: data[ed[i]] = ws[ed[i]] * cd[i];  parity[ep[i]] += ws[N + ep[i]] * cp[i]
cudaError_t launch_repair_scatter(const fastecc_b200_repair* R, uint32_t* data, size_t dpitch, uint32_t* parity, size_t ppitch, size_t c0, size_t size,
                                  const uint32_t* ws, size_t wpitch, size_t cols, int num_sms, cudaStream_t st);
}
