// Update of a stored stripe in place when k of its N data blocks change (include/fastecc_b200.h: fastecc_b200_rs_update, DESIGN 3h).
//
// rho = GF_Root(2N), D = N / M.  Parity j' = f(rho^(2Dj'+1)) of the data interpolant f is linear in the data, and on this code's
// points its coefficient depends only on (D j' - i) mod N:  parity_j' = sum_i data_i * T[(D j' - i) mod N],
// T[t] = -2 / (N (rho^(2t+1) - 1)).  A change of rows C adds sum_{i in C} (new_i - old_i) * T[(D j' - i) mod N] to parity j':
// one read of the changed rows and one read and write of the M parity rows, whatever N.  This file holds the table and the two
// kernels of that direct path; the re-encode path for large k is the sequence in api.cu.
#include "locator.h"
#include "update.h"

namespace {

using namespace fecc;
constexpr uint32_t P = gf::P;

__global__ void update_table_kernel(uint4* __restrict__ T, uint32_t N, LeafRoots L, const uint4* __restrict__ tw)
{
    FOR_GRID(uint32_t, t, N) {
        const uint32_t x = rho_pow(L, tw, 2 * t + 1);                 // odd exponent: x != 1
        const gf::Tw w = gf::make_tw(gf::mulmod(P - 2, gf::inv(gf::mulmod(N, x - 1))));
#if defined(FECC_UPDATE_MUL_H)                                      // experiment switch (DESIGN 13): {w, wp} for gf::mul_h
        uint32_t lo, hi;
        gf::wp_bits(w.whi, w.wlo, lo, hi);
        T[t] = make_uint4(w.w, lo, hi, 0u);
#else
        T[t] = make_uint4(w.w, w.whi, w.wlo, 0u);
#endif
    }
}

// Flat over (changed row, 16-byte chunk).  Each word is read and then written by the same thread, so no old word is overwritten
// before it is read; the changed rows are distinct, so no two threads write one row.
__global__ void __launch_bounds__(256) update_delta_kernel(uint32_t* __restrict__ data, size_t dpitch, const uint32_t* __restrict__ nw, size_t npitch,
                                                           uint4* __restrict__ delta, const uint32_t* __restrict__ idx, uint32_t s4, uint32_t n, size_t size)
{
    FOR_GRID(uint32_t, i, n) {
        const uint32_t r = i / s4, c = i - r * s4;
        uint32_t* drow = data + (size_t)__ldg(idx + r) * dpitch;
        const uint4 v = gf::canon4(__ldg(reinterpret_cast<const uint4*>(nw + r * npitch) + c));
        if (delta) {
            const uint4 o = gf::canon4(reinterpret_cast<const uint4*>(drow)[c]);
            delta[(size_t)r * s4 + c] = make_uint4(gf::sub(v.x, o.x), gf::sub(v.y, o.y), gf::sub(v.z, o.z), gf::sub(v.w, o.w));
        }
        store_row(drow, 4 * (size_t)c, v, size);
    }
}

// A CTA owns kRows parity rows x kCols 16-byte chunks; warp w holds rows w, w + 8, w + 16, w + 24 of the tile, lane l chunk l.  The
// delta chunks of the tile's columns are staged in shared memory kGroup changed rows at a time; every lane of a warp reads the
// same T entry (one broadcast load).  Sums stay lazy (gf::addl of gf::mul in [0, P]) and are reduced once at the end.
constexpr uint32_t kCols = 32, kRows = 32, kGroup = 32;

__global__ void __launch_bounds__(256) update_parity_kernel(uint32_t* __restrict__ parity, size_t ppitch, uint32_t M, const uint4* __restrict__ delta,
                                                            const uint32_t* __restrict__ idx, uint32_t k, const uint4* __restrict__ T, uint32_t N,
                                                            uint32_t D, uint32_t s4, uint32_t col_blocks, size_t size)
{
    __shared__ uint4 sd[kGroup][kCols];
    __shared__ uint32_t se[kGroup];
    const uint32_t lane = threadIdx.x % 32, warp = threadIdx.x / 32;
    const uint32_t cb = blockIdx.x % col_blocks, c = cb * kCols + lane, j0 = blockIdx.x / col_blocks * kRows + warp;
    const uint32_t zero = gf::opaque_zero();
    uint4 acc[4];
    uint32_t base[4];                                               // D j' + N
#pragma unroll
    for (uint32_t u = 0; u < 4; ++u) {
        const uint32_t j = j0 + 8 * u;
        acc[u] = j < M && c < s4 ? reinterpret_cast<const uint4*>(parity + j * ppitch)[c] : make_uint4(0, 0, 0, 0);
        base[u] = D * j + N;
    }
    for (uint32_t g0 = 0; g0 < k; g0 += kGroup) {
        const uint32_t gn = k - g0 < kGroup ? k - g0 : kGroup;
        __syncthreads();                                            // the previous group is consumed
        for (uint32_t q = threadIdx.x; q < gn * kCols; q += blockDim.x) {
            const uint32_t r = q / kCols, cc = cb * kCols + q % kCols;
            sd[r][q % kCols] = cc < s4 ? __ldg(delta + (size_t)(g0 + r) * s4 + cc) : make_uint4(0, 0, 0, 0);
        }
        if (threadIdx.x < gn) se[threadIdx.x] = __ldg(idx + g0 + threadIdx.x);
        __syncthreads();
        for (uint32_t r = 0; r < gn; ++r) {
            const uint4 d = sd[r][lane];
            const uint32_t e = se[r];
#pragma unroll
            for (uint32_t u = 0; u < 4; ++u) {
                if (j0 + 8 * u >= M) continue;                      // the same for the whole warp
                uint32_t t = base[u] - e;
                if (t >= N) t -= N;
                const uint4 w = __ldg(T + t);
#if defined(FECC_UPDATE_MUL_H)
                acc[u].x = gf::addl(acc[u].x, gf::mul_h(d.x, w.x, w.y, w.z));
                acc[u].y = gf::addl(acc[u].y, gf::mul_h(d.y, w.x, w.y, w.z));
                acc[u].z = gf::addl(acc[u].z, gf::mul_h(d.z, w.x, w.y, w.z));
                acc[u].w = gf::addl(acc[u].w, gf::mul_h(d.w, w.x, w.y, w.z));
#else
                acc[u].x = gf::addl(acc[u].x, gf::mul(d.x, w.x, w.y, w.z, zero));
                acc[u].y = gf::addl(acc[u].y, gf::mul(d.y, w.x, w.y, w.z, zero));
                acc[u].z = gf::addl(acc[u].z, gf::mul(d.z, w.x, w.y, w.z, zero));
                acc[u].w = gf::addl(acc[u].w, gf::mul(d.w, w.x, w.y, w.z, zero));
#endif
            }
        }
    }
#pragma unroll
    for (uint32_t u = 0; u < 4; ++u) {
        const uint32_t j = j0 + 8 * u;
        if (j < M && c < s4) store_row(parity + j * ppitch, 4 * (size_t)c, gf::canon4(acc[u]), size);
    }
}

} // namespace

namespace fecc {

cudaError_t launch_update_table(uint4* T, size_t N, cudaStream_t st)
{
    update_table_kernel<<<grid_size(N, 4096), 256, 0, st>>>(T, (uint32_t)N, leaf_roots(2 * N), context_power_table());
    return cudaGetLastError();
}

cudaError_t launch_update_delta(uint32_t* data, size_t dpitch, const uint32_t* nw, size_t npitch, uint4* delta, const uint32_t* idx, size_t k,
                                size_t size, int num_sms, cudaStream_t st)
{
    const uint32_t s4 = (uint32_t)((size + 3) / 4), n = (uint32_t)(k * s4);
    update_delta_kernel<<<grid_size(n, (size_t)num_sms * 16), 256, 0, st>>>(data, dpitch, nw, npitch, delta, idx, s4, n, size);
    return cudaGetLastError();
}

cudaError_t launch_update_parity(uint32_t* parity, size_t ppitch, size_t M, const uint4* delta, const uint32_t* idx, size_t k, const uint4* T, size_t N,
                                 size_t size, cudaStream_t st)
{
    const uint32_t s4 = (uint32_t)((size + 3) / 4), col_blocks = (s4 + kCols - 1) / kCols;
    const size_t blocks = (M + kRows - 1) / kRows * col_blocks;
    update_parity_kernel<<<(unsigned)blocks, 256, 0, st>>>(parity, ppitch, (uint32_t)M, delta, idx, (uint32_t)k, T, (uint32_t)N, (uint32_t)(N / M), s4,
                                                           col_blocks, size);
    return cudaGetLastError();
}

} // namespace fecc
