// Repair of a stored stripe in place (include/fastecc_b200.h: fastecc_b200_rs_repair*, DESIGN 3g): the N data rows and the M
// parity rows that fastecc_b200_rs_encode_asym_mixed[_dev] produces, with any |E_d| + |E_p| <= M of them lost.
//
// rho = GF_Root(2N), D = N / M, parity j' = f(y_j'), y_j' = rho^(2Dj' + 1); l = the locator of E = {2e} u {2Dj' + 1} in the
// 2N-row numbering (locator.h).  With G = the encode of the data with the lost rows zeroed, p = (f - g) * (l_p / r) has degree
// < M and p(y_j') = (parity_j' - G_j') * (-l(y_j') / 2) on the parity coset.  One inverse order-M transform gives P_k = M p_k rho^k;
// lost data e = N / D[2e] * NTT_N(P_k rho^-k / M)[e], lost parity j' = G_j' - 2 NTT_M(k P_k)[j'] / (M D[2Dj' + 1]), with
// D[m] = rho^m l'(rho^m).  This file holds the pattern (everything that depends only on which blocks are lost) and the four
// element-wise kernels; api.cu runs them around the encode and the transforms on its workspace.
#include "mixed_radix.h"
#include "locator.h"
#include "repair.h"
#include <algorithm>
#include <new>
#include <vector>

namespace {

using namespace fecc;
constexpr uint32_t P = gf::P;

// ---- the four element-wise kernels: flat over (row, 16-byte chunk), per-row constants as Barrett triples --------------------
// lost == nullptr: no row is lost (the re-encode of fastecc_b200_rs_update)
__global__ void __launch_bounds__(256) repair_load_kernel(const uint32_t* __restrict__ data, size_t dpitch, size_t c0, uint4* __restrict__ ws, size_t wpitch4,
                                                          uint32_t s4, uint32_t n, const uint8_t* __restrict__ lost)
{
    FOR_GRID(uint32_t, i, n) {
        const uint32_t row = i / s4, c = i - row * s4;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (!lost || !lost[row]) v = gf::canon4(__ldg(reinterpret_cast<const uint4*>(data + row * dpitch + c0) + c));
        ws[row * wpitch4 + c] = v;
    }
}

// cs == nullptr: every parity row takes G and the workspace is left as it is (the re-encode of fastecc_b200_rs_update)
__global__ void __launch_bounds__(256) repair_syndrome_kernel(uint32_t* __restrict__ parity, size_t ppitch, size_t c0, size_t size, uint4* __restrict__ ws,
                                                              size_t wpitch4, uint32_t s4, uint32_t n, const uint4* __restrict__ cs)
{
    const uint32_t zero = gf::opaque_zero();
    FOR_GRID(uint32_t, i, n) {
        const uint32_t row = i / s4, c = i - row * s4;
        const uint4 k = cs ? __ldg(cs + row) : make_uint4(0, 0, 0, 0);
        uint4* g = ws + row * wpitch4 + c;
        uint32_t* prow = parity + row * ppitch;
        const uint4 G = *g;
        if (k.x == 0) {                                          // lost: the parity of the zeroed data goes in place, u = 0
            store_row(prow, c0 + 4 * (size_t)c, G, size);
            if (cs) *g = make_uint4(0, 0, 0, 0);
        } else {
            const uint4 v = gf::canon4(*reinterpret_cast<const uint4*>(prow + c0 + 4 * (size_t)c));
            *g = gf::canon4(gf::mul4(make_uint4(gf::sub(v.x, G.x), gf::sub(v.y, G.y), gf::sub(v.z, G.z), gf::sub(v.w, G.w)), k, zero));
        }
    }
}

__global__ void __launch_bounds__(256) repair_split_kernel(uint4* __restrict__ ws, size_t wpitch4, uint32_t s4, uint32_t n, size_t N, size_t M,
                                                           const uint4* __restrict__ cr, const uint4* __restrict__ ck, bool derivative)
{
    const uint32_t zero = gf::opaque_zero();
    FOR_GRID(uint32_t, i, n) {
        const uint32_t row = i / s4, c = i - row * s4;
        uint4* x = ws + row * wpitch4 + c;
        if (row >= M) { *x = make_uint4(0, 0, 0, 0); continue; }   // the zero padding of the order-N transform
        const uint4 v = *x;
        if (derivative) {
            const uint4 k = __ldg(ck + row);
            ws[(N + row) * wpitch4 + c] = gf::canon4(gf::mul4(v, k, zero));
        }
        const uint4 k = __ldg(cr + row);
        *x = gf::canon4(gf::mul4(v, k, zero));
    }
}

__global__ void __launch_bounds__(256) repair_scatter_kernel(uint32_t* __restrict__ data, size_t dpitch, uint32_t* __restrict__ parity, size_t ppitch,
                                                             size_t c0, size_t size, const uint4* __restrict__ ws, size_t wpitch4, uint32_t s4, uint32_t n,
                                                             size_t N, uint32_t ned, const uint32_t* __restrict__ ed, const uint32_t* __restrict__ ep,
                                                             const uint4* __restrict__ cd, const uint4* __restrict__ cp)
{
    const uint32_t zero = gf::opaque_zero();
    FOR_GRID(uint32_t, i, n) {
        const uint32_t r = i / s4, c = i - r * s4;
        const size_t w = c0 + 4 * (size_t)c;
        if (r < ned) {                                           // data row e = N / D[2e] * NTT_N(...)[e]
            const uint32_t e = __ldg(ed + r);
            const uint4 k = __ldg(cd + r), v = ws[e * wpitch4 + c];
            store_row(data + e * dpitch, w, gf::canon4(gf::mul4(v, k, zero)), size);
        } else {                                                 // parity row j' = G_j' + NTT_M(k P_k)[j'] * (-2 / (M D))
            const uint32_t j = __ldg(ep + (r - ned));
            const uint4 k = __ldg(cp + (r - ned)), v = ws[(N + j) * wpitch4 + c];
            uint32_t* prow = parity + j * ppitch;
            const uint4 G = *reinterpret_cast<const uint4*>(prow + w);
            auto lane = [&](uint32_t g, uint32_t x) { return gf::sub(gf::canon(g), gf::canon(P - gf::mulc(x, k, zero))); };     // g - (-x k)
            store_row(prow, w, make_uint4(lane(G.x, v.x), lane(G.y, v.y), lane(G.z, v.z), lane(G.w, v.w)), size);
        }
    }
}

// ---- the pattern ---------------------------------------------------------------------------------------------------------
__device__ uint4 triple(uint32_t w) { const gf::Tw t = gf::make_tw(w); return make_uint4(t.w, t.whi, t.wlo, 0u); }

// lv4 / dl4: l(rho^m) and D[m] as erasure_locator leaves them (4-word rows).  inv2 = 1/2, inv_m = 1/M.
__global__ void finish_repair_kernel(const uint32_t* __restrict__ lv4, const uint32_t* __restrict__ dl4, LeafRoots L, const uint4* __restrict__ tw,
                                     size_t N, size_t M, uint32_t inv2, uint32_t inv_m, RepairTables R)
{
    const size_t n2 = 2 * N, D = N / M;
    FOR_GRID(size_t, i, M) {
        const uint32_t l = lv4[(2 * D * i + 1) * 4];
        R.d_cs[i] = triple(gf::mulmod(l ? P - l : 0u, inv2));                                  // -l(y_i) / 2
        R.d_cr[i] = triple(gf::mulmod(rho_pow(L, tw, (uint32_t)((n2 - i) % n2)), inv_m));     // rho^-i / M
        R.d_ck[i] = triple((uint32_t)i);
        if (i < R.ned) {
            const uint32_t e = R.d_ed[i];
            R.d_lost[e] = 1;
            R.d_cd[i] = triple(gf::mulmod((uint32_t)N, gf::inv(dl4[(size_t)2 * e * 4])));       // N / D[2e]
        }
        if (i < R.nep) {
            const size_t m = 2 * D * R.d_ep[i] + 1;
            R.d_cp[i] = triple(gf::mulmod(P - 2, gf::inv(gf::mulmod((uint32_t)M, dl4[m * 4]))));   // -2 / (M * D[2Dj' + 1])
        }
    }
}

int build_repair(fastecc_b200_repair* R, const uint32_t* lost_data, const uint32_t* lost_parity, cudaStream_t st, const char* who)
{
    const size_t N = R->N, M = R->M, ned = R->ned, nep = R->nep, me = ned + nep, D = N / M;
    DeviceArrays& m = R->mem;
    R->d_ed = m.alloc<uint32_t>(ned); R->d_ep = m.alloc<uint32_t>(nep); R->d_lost = m.alloc<uint8_t>(N);
    R->d_cs = m.alloc<uint4>(M); R->d_cr = m.alloc<uint4>(M); R->d_ck = m.alloc<uint4>(M); R->d_cd = m.alloc<uint4>(ned); R->d_cp = m.alloc<uint4>(nep);
    DeviceArrays tmp;
    uint32_t* d_idx = tmp.alloc<uint32_t>(me);
    if (m.failed || !d_idx) return fail(FASTECC_B200_ENOMEM, "%s: out of device memory", who);
    std::vector<uint32_t> pos;                                   // E in the 2N-row numbering, ascending
    pos.reserve(me);
    for (size_t i = 0; i < ned; ++i) pos.push_back(2 * lost_data[i]);
    for (size_t i = 0; i < nep; ++i) pos.push_back((uint32_t)(2 * D * lost_parity[i] + 1));
    std::inplace_merge(pos.begin(), pos.begin() + ned, pos.end());
    if (ned) CUDA_TRY(cudaMemcpyAsync(R->d_ed, lost_data, ned * 4, cudaMemcpyHostToDevice, st));
    if (nep) CUDA_TRY(cudaMemcpyAsync(R->d_ep, lost_parity, nep * 4, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemsetAsync(R->d_lost, 0, N, st));
    CUDA_TRY(cudaMemcpyAsync(d_idx, pos.data(), me * 4, cudaMemcpyHostToDevice, st));
    uint32_t *lv4 = nullptr, *dl4 = nullptr;
    TRY_RC(erasure_locator(2 * N, d_idx, me, tmp, &lv4, &dl4, st, who));
    finish_repair_kernel<<<grid_size(M, 4096), 256, 0, st>>>(lv4, dl4, leaf_roots(2 * N), context_power_table(), N, M, gf::inv(2), gf::inv((uint32_t)M), *R);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(st));                         // the scratch buffers are freed on return
    return 0;
}

} // namespace

namespace fecc {

cudaError_t launch_repair_load(size_t N, const uint8_t* lost, const uint32_t* data, size_t dpitch, size_t c0, uint32_t* ws, size_t wpitch,
                               size_t cols, int num_sms, cudaStream_t st)
{
    const uint32_t s4 = (uint32_t)((cols + 3) / 4), n = (uint32_t)(N * s4);
    repair_load_kernel<<<grid_size(n, (size_t)num_sms * 16), 256, 0, st>>>(data, dpitch, c0, reinterpret_cast<uint4*>(ws), wpitch / 4, s4, n, lost);
    return cudaGetLastError();
}

cudaError_t launch_repair_syndrome(size_t M, const uint4* cs, uint32_t* parity, size_t ppitch, size_t c0, size_t size, uint32_t* ws, size_t wpitch,
                                   size_t cols, int num_sms, cudaStream_t st)
{
    const uint32_t s4 = (uint32_t)((cols + 3) / 4), n = (uint32_t)(M * s4);
    repair_syndrome_kernel<<<grid_size(n, (size_t)num_sms * 16), 256, 0, st>>>(parity, ppitch, c0, size, reinterpret_cast<uint4*>(ws), wpitch / 4, s4, n, cs);
    return cudaGetLastError();
}

cudaError_t launch_repair_split(const fastecc_b200_repair* R, uint32_t* ws, size_t wpitch, size_t cols, int num_sms, cudaStream_t st)
{
    const uint32_t s4 = (uint32_t)((cols + 3) / 4), n = (uint32_t)((R->ned ? R->N : R->M) * s4);
    repair_split_kernel<<<grid_size(n, (size_t)num_sms * 16), 256, 0, st>>>(reinterpret_cast<uint4*>(ws), wpitch / 4, s4, n, R->N, R->M, R->d_cr, R->d_ck, R->nep != 0);
    return cudaGetLastError();
}

cudaError_t launch_repair_scatter(const fastecc_b200_repair* R, uint32_t* data, size_t dpitch, uint32_t* parity, size_t ppitch, size_t c0, size_t size,
                                  const uint32_t* ws, size_t wpitch, size_t cols, int num_sms, cudaStream_t st)
{
    const uint32_t s4 = (uint32_t)((cols + 3) / 4), n = (uint32_t)((R->ned + R->nep) * s4);
    repair_scatter_kernel<<<grid_size(n, (size_t)num_sms * 16), 256, 0, st>>>(data, dpitch, parity, ppitch, c0, size, reinterpret_cast<const uint4*>(ws), wpitch / 4, s4, n,
                                                                  R->N, (uint32_t)R->ned, R->d_ed, R->d_ep, R->d_cd, R->d_cp);
    return cudaGetLastError();
}

} // namespace fecc

extern "C" {

int fastecc_b200_rs_repair_pattern(size_t N, size_t M, const uint32_t* lost_data, size_t n_lost_data, const uint32_t* lost_parity, size_t n_lost_parity,
                                   void* stream, fastecc_b200_repair** out)
{
    const char* who = "fastecc_b200_rs_repair_pattern";
    if (!out) return fail(FASTECC_B200_EINVAL, "%s: null output", who);
    *out = nullptr;
    if (!context_power_table()) return fail(FASTECC_B200_ENOINIT, "%s: call fastecc_b200_init() first", who);
    const Order o = split_order(N);
    if (!o.r || o.log2_m > FASTECC_B200_MAX_LOG_N_ENCODE)
        return fail(FASTECC_B200_EINVAL, "%s: N=%zu must be 2^k, 3 * 2^k or 9 * 2^k with 2^k <= 2^19", who, N);
    if (M == 0 || N % M) return fail(FASTECC_B200_EINVAL, "%s: M=%zu must divide N=%zu", who, M, N);
    if ((n_lost_data && !lost_data) || (n_lost_parity && !lost_parity)) return fail(FASTECC_B200_EINVAL, "%s: null list of lost blocks", who);
    if (n_lost_data + n_lost_parity > M)
        return fail(FASTECC_B200_EINVAL, "%s: %zu blocks lost; M = %zu parity blocks recover at most %zu", who, n_lost_data + n_lost_parity, M, M);
    if (!ascending_below(lost_data, n_lost_data, N)) return fail(FASTECC_B200_EINVAL, "%s: lost data blocks must be ascending, distinct and below N=%zu", who, N);
    if (!ascending_below(lost_parity, n_lost_parity, M)) return fail(FASTECC_B200_EINVAL, "%s: lost parity blocks must be ascending, distinct and below M=%zu", who, M);
    fastecc_b200_repair* R = new (std::nothrow) fastecc_b200_repair;
    if (!R) return fail(FASTECC_B200_ENOMEM, "%s: out of host memory", who);
    R->N = N; R->M = M; R->ned = n_lost_data; R->nep = n_lost_parity;
    if (n_lost_data + n_lost_parity) {
        const int rc = build_repair(R, lost_data, lost_parity, (cudaStream_t)stream, who);
        if (rc) { delete R; return rc; }
    }
    *out = R;
    return 0;
}

void fastecc_b200_rs_repair_free(fastecc_b200_repair* R) { delete R; }               // null-safe

} // extern "C"
