// Repair of a stored stripe in place (include/fastecc_b200.h: fastecc_b200_rs_repair*, DESIGN 3g): the N data rows and the M
// parity rows that fastecc_b200_rs_encode_asym_mixed[_dev] produces, with any |E_d| + |E_p| <= M of them lost.
//
// rho = GF_Root(2N), D = N / M, parity j' = f(y_j'), y_j' = rho^(2Dj' + 1); l = the locator of E = {2e} u {2Dj' + 1} in the
// 2N-row numbering (locator.h).  With G = the encode of the data with the lost rows zeroed, p = (f - g) * (l_p / r) has degree
// < M and p(y_j') = (parity_j' - G_j') * (-l(y_j') / 2) on the parity coset.  One inverse order-M transform gives P_k = M p_k rho^k;
// lost data e = N / D[2e] * NTT_N(P_k rho^-k / M)[e], lost parity j' = G_j' - 2 NTT_M(k P_k)[j'] / (M D[2Dj' + 1]), with
// D[m] = rho^m l'(rho^m).  This file holds the pattern (everything that depends only on which blocks are lost) and the four
// element-wise kernels; api.cu runs them around the encode and the transforms on its workspace.
#include "../../include/fastecc_b200.h"
#include "gf.cuh"
#include "mixed_radix.h"
#include "locator.h"
#include "repair.h"
#include <cuda_runtime.h>
#include <algorithm>
#include <new>
#include <vector>

namespace fecc {
const uint4* context_power_table();          // api.cu: g^e, e in [0, 2^20), or nullptr before fastecc_b200_init()
int          fail(int code, const char* fmt, ...);
}

namespace {

using namespace fecc;
constexpr uint32_t P = gf::P;

// ---- the four element-wise kernels: flat over (row, 16-byte chunk), per-row constants as Barrett triples --------------------
__device__ __forceinline__ uint32_t mulc(uint32_t b, const uint4& k, uint32_t zero) { return gf::canon(gf::mul(b, k.x, k.y, k.z, zero)); }
__device__ __forceinline__ uint32_t subc(uint32_t a, uint32_t b) { return a >= b ? a - b : a + (P - b); }          // canonical a, b
__device__ __forceinline__ uint32_t addc(uint32_t a, uint32_t b) { return subc(a, gf::canon(P - b)); }
__device__ __forceinline__ uint4 canon4(uint4 v) { return make_uint4(gf::canon(v.x), gf::canon(v.y), gf::canon(v.z), gf::canon(v.w)); }

// words [w, w + 4) of `row`, of which only those below `size` are written (the last chunk of a row may be partial)
__device__ __forceinline__ void store_row(uint32_t* row, size_t w, const uint4& v, size_t size)
{
    if (w + 4 <= size) { *reinterpret_cast<uint4*>(row + w) = v; return; }
    if (w < size) row[w] = v.x;
    if (w + 1 < size) row[w + 1] = v.y;
    if (w + 2 < size) row[w + 2] = v.z;
}

#define FOR_CHUNK(i, n) for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += gridDim.x * blockDim.x)

__global__ void __launch_bounds__(256) repair_load_kernel(const uint32_t* __restrict__ data, size_t dpitch, size_t c0, uint4* __restrict__ ws, size_t wpitch4,
                                                          uint32_t s4, uint32_t n, const uint8_t* __restrict__ lost)
{
    FOR_CHUNK(i, n) {
        const uint32_t row = i / s4, c = i - row * s4;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (!lost[row]) v = canon4(__ldg(reinterpret_cast<const uint4*>(data + row * dpitch + c0) + c));
        ws[row * wpitch4 + c] = v;
    }
}

__global__ void __launch_bounds__(256) repair_syndrome_kernel(uint32_t* __restrict__ parity, size_t ppitch, size_t c0, size_t size, uint4* __restrict__ ws,
                                                              size_t wpitch4, uint32_t s4, uint32_t n, const uint4* __restrict__ cs)
{
    const uint32_t zero = gf::opaque_zero();
    FOR_CHUNK(i, n) {
        const uint32_t row = i / s4, c = i - row * s4;
        const uint4 k = __ldg(cs + row);
        uint4* g = ws + row * wpitch4 + c;
        uint32_t* prow = parity + row * ppitch;
        const uint4 G = *g;
        if (k.x == 0) {                                          // lost: the parity of the zeroed data goes in place, u = 0
            store_row(prow, c0 + 4 * (size_t)c, G, size);
            *g = make_uint4(0, 0, 0, 0);
        } else {
            const uint4 v = *reinterpret_cast<const uint4*>(prow + c0 + 4 * (size_t)c);
            *g = make_uint4(mulc(subc(gf::canon(v.x), G.x), k, zero), mulc(subc(gf::canon(v.y), G.y), k, zero),
                            mulc(subc(gf::canon(v.z), G.z), k, zero), mulc(subc(gf::canon(v.w), G.w), k, zero));
        }
    }
}

__global__ void __launch_bounds__(256) repair_split_kernel(uint4* __restrict__ ws, size_t wpitch4, uint32_t s4, uint32_t n, size_t N, size_t M,
                                                           const uint4* __restrict__ cr, const uint4* __restrict__ ck, bool derivative)
{
    const uint32_t zero = gf::opaque_zero();
    FOR_CHUNK(i, n) {
        const uint32_t row = i / s4, c = i - row * s4;
        uint4* x = ws + row * wpitch4 + c;
        if (row >= M) { *x = make_uint4(0, 0, 0, 0); continue; }   // the zero padding of the order-N transform
        const uint4 v = *x;
        if (derivative) {
            const uint4 k = __ldg(ck + row);
            ws[(N + row) * wpitch4 + c] = make_uint4(mulc(v.x, k, zero), mulc(v.y, k, zero), mulc(v.z, k, zero), mulc(v.w, k, zero));
        }
        const uint4 k = __ldg(cr + row);
        *x = make_uint4(mulc(v.x, k, zero), mulc(v.y, k, zero), mulc(v.z, k, zero), mulc(v.w, k, zero));
    }
}

__global__ void __launch_bounds__(256) repair_scatter_kernel(uint32_t* __restrict__ data, size_t dpitch, uint32_t* __restrict__ parity, size_t ppitch,
                                                             size_t c0, size_t size, const uint4* __restrict__ ws, size_t wpitch4, uint32_t s4, uint32_t n,
                                                             size_t N, uint32_t ned, const uint32_t* __restrict__ ed, const uint32_t* __restrict__ ep,
                                                             const uint4* __restrict__ cd, const uint4* __restrict__ cp)
{
    const uint32_t zero = gf::opaque_zero();
    FOR_CHUNK(i, n) {
        const uint32_t r = i / s4, c = i - r * s4;
        const size_t w = c0 + 4 * (size_t)c;
        if (r < ned) {                                           // data row e = N / D[2e] * NTT_N(...)[e]
            const uint32_t e = __ldg(ed + r);
            const uint4 k = __ldg(cd + r), v = ws[e * wpitch4 + c];
            store_row(data + e * dpitch, w, make_uint4(mulc(v.x, k, zero), mulc(v.y, k, zero), mulc(v.z, k, zero), mulc(v.w, k, zero)), size);
        } else {                                                 // parity row j' = G_j' + NTT_M(k P_k)[j'] * (-2 / (M D))
            const uint32_t j = __ldg(ep + (r - ned));
            const uint4 k = __ldg(cp + (r - ned)), v = ws[(N + j) * wpitch4 + c];
            uint32_t* prow = parity + j * ppitch;
            const uint4 G = *reinterpret_cast<const uint4*>(prow + w);
            store_row(prow, w, make_uint4(addc(gf::canon(G.x), mulc(v.x, k, zero)), addc(gf::canon(G.y), mulc(v.y, k, zero)),
                                          addc(gf::canon(G.z), mulc(v.z, k, zero)), addc(gf::canon(G.w), mulc(v.w, k, zero))), size);
        }
    }
}

unsigned chunk_grid(uint32_t n, int num_sms)
{
    const size_t blocks = ((size_t)n + 255) / 256, cap = (size_t)num_sms * 16;
    return (unsigned)(blocks < cap ? (blocks ? blocks : 1) : cap);
}

// ---- the pattern ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t mulmod(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) % P); }
__device__ uint32_t invmod(uint32_t x)
{
    uint32_t r = 1;
    for (uint32_t e = P - 2; e; e >>= 1) { if (e & 1u) r = mulmod(r, x); x = mulmod(x, x); }
    return r;
}
__device__ uint4 triple(uint32_t w)                              // gf::make_tw of canonical w
{
    const uint64_t n1 = (uint64_t)w << 32;
    const uint64_t whi = n1 / P, rem = n1 % P;
    return make_uint4(w, (uint32_t)whi, (uint32_t)((rem << 32) / P), 0u);
}
__device__ uint32_t rho_pow(const LeafRoots& L, const uint4* tw, uint32_t e)       // rho^e, e < 2N (as leaves_kernel in decode.cu)
{
    uint32_t r = tw[(size_t)((L.b2 * e) & L.mask) << L.log_step].x;
    if (L.r > 1) r = mulmod(r, L.zeta[(L.a2 * (e % L.r)) % L.r]);
    return r;
}

// lv4 / dl4: l(rho^m) and D[m] as erasure_locator leaves them (4-word rows).  inv2 = 1/2, inv_m = 1/M.
__global__ void finish_repair_kernel(const uint32_t* __restrict__ lv4, const uint32_t* __restrict__ dl4, LeafRoots L, const uint4* __restrict__ tw,
                                     size_t N, size_t M, uint32_t inv2, uint32_t inv_m, fastecc_b200_repair R)
{
    const size_t n2 = 2 * N, D = N / M;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < M; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t l = lv4[(2 * D * i + 1) * 4];
        R.d_cs[i] = triple(mulmod(l ? P - l : 0u, inv2));                                  // -l(y_i) / 2
        R.d_cr[i] = triple(mulmod(rho_pow(L, tw, (uint32_t)((n2 - i) % n2)), inv_m));     // rho^-i / M
        R.d_ck[i] = triple((uint32_t)i);
        if (i < R.ned) {
            const uint32_t e = R.d_ed[i];
            R.d_lost[e] = 1;
            R.d_cd[i] = triple(mulmod((uint32_t)N, invmod(dl4[(size_t)2 * e * 4])));       // N / D[2e]
        }
        if (i < R.nep) {
            const size_t m = 2 * D * R.d_ep[i] + 1;
            R.d_cp[i] = triple(mulmod(P - 2, invmod(mulmod((uint32_t)M, dl4[m * 4]))));   // -2 / (M * D[2Dj' + 1])
        }
    }
}

#define TRY_CUDA(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) \
    return fail(e_ == cudaErrorMemoryAllocation ? FASTECC_B200_ENOMEM : FASTECC_B200_ECUDA, "%s: %s", #expr, cudaGetErrorString(e_)); } while (0)

int build_repair(fastecc_b200_repair* R, const uint32_t* lost_data, const uint32_t* lost_parity, cudaStream_t st, const char* who)
{
    const size_t N = R->N, M = R->M, ned = R->ned, nep = R->nep, me = ned + nep, D = N / M;
    TRY_CUDA(cudaMalloc((void**)&R->d_ed, (ned ? ned : 1) * 4));
    TRY_CUDA(cudaMalloc((void**)&R->d_ep, (nep ? nep : 1) * 4));
    TRY_CUDA(cudaMalloc((void**)&R->d_lost, N));
    TRY_CUDA(cudaMalloc((void**)&R->d_cs, M * 16));
    TRY_CUDA(cudaMalloc((void**)&R->d_cr, M * 16));
    TRY_CUDA(cudaMalloc((void**)&R->d_ck, M * 16));
    TRY_CUDA(cudaMalloc((void**)&R->d_cd, (ned ? ned : 1) * 16));
    TRY_CUDA(cudaMalloc((void**)&R->d_cp, (nep ? nep : 1) * 16));
    std::vector<uint32_t> pos;                                   // E in the 2N-row numbering, ascending
    pos.reserve(me);
    for (size_t i = 0; i < ned; ++i) pos.push_back(2 * lost_data[i]);
    for (size_t i = 0; i < nep; ++i) pos.push_back((uint32_t)(2 * D * lost_parity[i] + 1));
    std::inplace_merge(pos.begin(), pos.begin() + ned, pos.end());
    Scratch tmp;
    uint32_t* d_idx = tmp.words(me);
    if (!d_idx) return fail(FASTECC_B200_ENOMEM, "%s: out of device memory", who);
    if (ned) TRY_CUDA(cudaMemcpyAsync(R->d_ed, lost_data, ned * 4, cudaMemcpyHostToDevice, st));
    if (nep) TRY_CUDA(cudaMemcpyAsync(R->d_ep, lost_parity, nep * 4, cudaMemcpyHostToDevice, st));
    TRY_CUDA(cudaMemsetAsync(R->d_lost, 0, N, st));
    TRY_CUDA(cudaMemcpyAsync(d_idx, pos.data(), me * 4, cudaMemcpyHostToDevice, st));
    uint32_t *lv4 = nullptr, *dl4 = nullptr;
    if (int rc = erasure_locator(2 * N, d_idx, me, tmp, &lv4, &dl4, st, who)) return rc;
    const unsigned grid = (unsigned)((M + 255) / 256 < 4096 ? (M + 255) / 256 : 4096);
    finish_repair_kernel<<<grid, 256, 0, st>>>(lv4, dl4, leaf_roots(2 * N), context_power_table(), N, M, gf::inv(2), gf::inv((uint32_t)M), *R);
    TRY_CUDA(cudaGetLastError());
    TRY_CUDA(cudaStreamSynchronize(st));                         // the scratch buffers are freed on return
    return 0;
}

bool ascending_below(const uint32_t* a, size_t n, size_t bound)
{
    for (size_t i = 0; i < n; ++i)
        if (a[i] >= bound || (i && a[i] <= a[i - 1])) return false;
    return true;
}

} // namespace

namespace fecc {

cudaError_t launch_repair_load(const fastecc_b200_repair* R, const uint32_t* data, size_t dpitch, size_t c0, uint32_t* ws, size_t wpitch,
                               size_t cols, int num_sms, cudaStream_t st)
{
    const uint32_t s4 = (uint32_t)((cols + 3) / 4), n = (uint32_t)(R->N * s4);
    repair_load_kernel<<<chunk_grid(n, num_sms), 256, 0, st>>>(data, dpitch, c0, reinterpret_cast<uint4*>(ws), wpitch / 4, s4, n, R->d_lost);
    return cudaGetLastError();
}

cudaError_t launch_repair_syndrome(const fastecc_b200_repair* R, uint32_t* parity, size_t ppitch, size_t c0, size_t size, uint32_t* ws, size_t wpitch,
                                   size_t cols, int num_sms, cudaStream_t st)
{
    const uint32_t s4 = (uint32_t)((cols + 3) / 4), n = (uint32_t)(R->M * s4);
    repair_syndrome_kernel<<<chunk_grid(n, num_sms), 256, 0, st>>>(parity, ppitch, c0, size, reinterpret_cast<uint4*>(ws), wpitch / 4, s4, n, R->d_cs);
    return cudaGetLastError();
}

cudaError_t launch_repair_split(const fastecc_b200_repair* R, uint32_t* ws, size_t wpitch, size_t cols, int num_sms, cudaStream_t st)
{
    const uint32_t s4 = (uint32_t)((cols + 3) / 4), n = (uint32_t)((R->ned ? R->N : R->M) * s4);
    repair_split_kernel<<<chunk_grid(n, num_sms), 256, 0, st>>>(reinterpret_cast<uint4*>(ws), wpitch / 4, s4, n, R->N, R->M, R->d_cr, R->d_ck, R->nep != 0);
    return cudaGetLastError();
}

cudaError_t launch_repair_scatter(const fastecc_b200_repair* R, uint32_t* data, size_t dpitch, uint32_t* parity, size_t ppitch, size_t c0, size_t size,
                                  const uint32_t* ws, size_t wpitch, size_t cols, int num_sms, cudaStream_t st)
{
    const uint32_t s4 = (uint32_t)((cols + 3) / 4), n = (uint32_t)((R->ned + R->nep) * s4);
    repair_scatter_kernel<<<chunk_grid(n, num_sms), 256, 0, st>>>(data, dpitch, parity, ppitch, c0, size, reinterpret_cast<const uint4*>(ws), wpitch / 4, s4, n,
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
        if (rc) { fastecc_b200_rs_repair_free(R); return rc; }
    }
    *out = R;
    return 0;
}

void fastecc_b200_rs_repair_free(fastecc_b200_repair* R)
{
    if (!R) return;
    cudaFree(R->d_ed); cudaFree(R->d_ep); cudaFree(R->d_lost); cudaFree(R->d_cs); cudaFree(R->d_cr); cudaFree(R->d_ck); cudaFree(R->d_cd); cudaFree(R->d_cp);
    delete R;
}

} // extern "C"
