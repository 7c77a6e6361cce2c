// Scrub of a stored stripe (include/fastecc_b200.h: fastecc_b200_rs_scrub, DESIGN 3i): detect that the parity is not the encode
// of the data and locate up to M/2 corrupted blocks, data and parity alike, from the stripe alone.
//
// Every column is a code word, so is every linear combination of columns: fold f in {0, 1} maps row m to
// a_f,m = sum_c r_f,c * row_m[c] with the header's seeded weights.  The syndrome s_j = a_f(parity j) - G_j, G = the encode of the
// folded data, is zero in both folds iff the stripe is clean (up to P^-2).  With S^ = INTT_M(s) / M and L(z) = l(rho z) the
// locator of the corrupted points, L * S^ = Phi mod (z^M - 1), deg Phi < t: Berlekamp-Massey on S^_0 .. S^_(2 max_bad - 1) of
// fold 0 gives C = L / L_0, which is trusted only if M * (C * S^ mod z^M - 1) vanishes on [deg C, M) in both folds and C has
// deg C distinct roots among zeta^j (parity) and rho^-1 omega^i (data).  This file holds the fold, the element-wise kernels on
// the single-column workspace and Berlekamp-Massey; api.cu runs them around the encode and the transforms.
// The degraded scrub (fastecc_b200_rs_scrub_degraded, DESIGN 3j) is the same with f known lost blocks: their rows are never
// loaded, the syndrome is weighted by the erasure locator (u_j = s_j * cs_j, zero on the lost parity rows), the checks start at f
// and f + L, and the root search skips the lost points.
#include "scrub.h"
#include "gf.cuh"

namespace {

using namespace fecc;
constexpr uint32_t P = gf::P;

// r_f,c: the (2c + f + 1)-th output of splitmix64 started at `seed`, mod P (include/fastecc_b200.h states it)
__device__ __forceinline__ uint32_t fold_weight(uint64_t seed, uint32_t f, uint64_t c)
{
    uint64_t z = seed + (2 * c + f + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return gf::reduce64(z ^ (z >> 31));
}

// A work item is one tile of W 16-byte chunks (W = 32, or the next power of two >= ceil(SIZE / 4) for short rows) of every row
// of one slice of rows.  Lane l of a warp owns chunk l % W of the tile, on rows 32 / W apart: it derives the Barrett triples of its
// four columns for both folds once per item, then per row loads 16 bytes, takes 8 products with lazy sums, and the W lanes of a row
// add their sums by shuffles; one lane adds the canonical result to the row's two 64-bit workspace words.  Columns past SIZE have
// the weight 0, so a pad word never reaches a sum.  Four rows per lane are loaded before any is used.
// Experiment switch (DESIGN 13): -DFECC_SCRUB_MUL_H takes the products' quotient on the FP64 unit (gf::mul_h, DESIGN 4), the
// triples then holding {w, wp bits}; the shipped build uses gf::mul.
constexpr uint32_t kFoldUnroll = 4;
#if defined(FECC_SCRUB_MUL_H)
#define FOLD_MUL(b, t) gf::mul_h(b, (t)[0], (t)[1], (t)[2])
#else
#define FOLD_MUL(b, t) gf::mul(b, (t)[0], (t)[1], (t)[2], zero)
#endif

// The fold's body, shared by the plain and the degraded scrub: a row m with skip(m) is never loaded and folds to 0.
template <class Skip>
__device__ __forceinline__ void fold_rows(const uint32_t* __restrict__ data, size_t dpitch, uint32_t N, const uint32_t* __restrict__ parity, size_t ppitch,
                                          uint32_t rows, uint32_t size, uint32_t s4, uint32_t log_w, uint32_t tiles, uint32_t items, uint32_t slice_rows,
                                          uint64_t seed, unsigned long long* __restrict__ ws, Skip skip)
{
    const uint32_t lane = threadIdx.x % 32, W = 1u << log_w, sub = lane & (W - 1), rw = 32 >> log_w, rlane = lane >> log_w;
    const uint32_t nwarps = gridDim.x * (blockDim.x / 32);
    const uint32_t zero = gf::opaque_zero();
    for (uint32_t item = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32; item < items; item += nwarps) {
        const uint32_t tile = item % tiles, c = tile * W + sub;
        const bool live = c < s4;
        uint32_t tw[2][4][3];
#pragma unroll
        for (uint32_t f = 0; f < 2; ++f)
#pragma unroll
            for (uint32_t k = 0; k < 4; ++k) {
                const uint32_t col = 4 * c + k;
                const gf::Tw t = gf::make_tw(live && col < size ? fold_weight(seed, f, col) : 0u);
                tw[f][k][0] = t.w; tw[f][k][1] = t.whi; tw[f][k][2] = t.wlo;
#if defined(FECC_SCRUB_MUL_H)
                gf::wp_bits(t.whi, t.wlo, tw[f][k][1], tw[f][k][2]);
#endif
            }
        const uint32_t r0 = item / tiles * slice_rows, r1 = min(rows, r0 + slice_rows);
        for (uint32_t base = r0; base < r1; base += kFoldUnroll * rw) {        // the same trip count on every lane of the warp
            uint4 v[kFoldUnroll];
#pragma unroll
            for (uint32_t u = 0; u < kFoldUnroll; ++u) {
                const uint32_t m = base + u * rw + rlane;
                v[u] = make_uint4(0, 0, 0, 0);
                if (live && m < r1 && !skip(m)) {
                    const uint32_t* row = m < N ? data + (size_t)m * dpitch : parity + (size_t)(m - N) * ppitch;
                    v[u] = __ldg(reinterpret_cast<const uint4*>(row) + c);
                }
            }
#pragma unroll
            for (uint32_t u = 0; u < kFoldUnroll; ++u) {
                uint32_t a[2];
#pragma unroll
                for (uint32_t f = 0; f < 2; ++f) {
                    uint32_t s = FOLD_MUL(v[u].x, tw[f][0]);
                    s = gf::addl(s, FOLD_MUL(v[u].y, tw[f][1]));
                    s = gf::addl(s, FOLD_MUL(v[u].z, tw[f][2]));
                    a[f] = gf::addl(s, FOLD_MUL(v[u].w, tw[f][3]));
                }
                for (uint32_t o = W / 2; o; o /= 2) {
                    const uint32_t b0 = __shfl_xor_sync(0xFFFFFFFFu, a[0], o), b1 = __shfl_xor_sync(0xFFFFFFFFu, a[1], o);
                    a[0] = gf::addl(a[0], gf::canon(b0));
                    a[1] = gf::addl(a[1], gf::canon(b1));
                }
                const uint32_t m = base + u * rw + rlane;
                if (sub == 0 && m < r1) {
                    atomicAdd(ws + 2 * (size_t)m, (unsigned long long)gf::canon(a[0]));
                    atomicAdd(ws + 2 * (size_t)m + 1, (unsigned long long)gf::canon(a[1]));
                }
            }
        }
    }
}

__global__ void __launch_bounds__(256, 4) scrub_fold_kernel(const uint32_t* __restrict__ data, size_t dpitch, uint32_t N, const uint32_t* __restrict__ parity,
                                                            size_t ppitch, uint32_t rows, uint32_t size, uint32_t s4, uint32_t log_w, uint32_t tiles,
                                                            uint32_t items, uint32_t slice_rows, uint64_t seed, unsigned long long* __restrict__ ws)
{
    fold_rows(data, dpitch, N, parity, ppitch, rows, size, s4, log_w, tiles, items, slice_rows, seed, ws, [](uint32_t) { return false; });
}

// The fold of a degraded stripe: the lost data rows (lost[m] != 0) and the lost parity rows (cs[j].x == 0) are never loaded.
__global__ void __launch_bounds__(256, 4) degraded_fold_kernel(const uint32_t* __restrict__ data, size_t dpitch, uint32_t N, const uint32_t* __restrict__ parity,
                                                               size_t ppitch, uint32_t rows, uint32_t size, uint32_t s4, uint32_t log_w, uint32_t tiles,
                                                               uint32_t items, uint32_t slice_rows, uint64_t seed, unsigned long long* __restrict__ ws,
                                                               const uint8_t* __restrict__ lost, const uint4* __restrict__ cs)
{
    fold_rows(data, dpitch, N, parity, ppitch, rows, size, s4, log_w, tiles, items, slice_rows, seed, ws,
              [=](uint32_t m) { return m < N ? __ldg(lost + m) != 0 : __ldg(&cs[m - N].x) == 0u; });
}

__global__ void scrub_reduce_kernel(uint4* __restrict__ ws, size_t n)
{
    FOR_GRID(size_t, i, n) {
        const uint4 v = ws[i];
        ws[i] = make_uint4(gf::reduce64(((uint64_t)v.y << 32) | v.x), gf::reduce64(((uint64_t)v.w << 32) | v.z), 0u, 0u);
    }
}

__global__ void scrub_syndrome_kernel(uint4* __restrict__ ws, size_t N, size_t M, uint32_t* __restrict__ nonzero)
{
    FOR_GRID(size_t, j, M) {
        const uint4 p = ws[N + j], g = ws[j];
        const uint4 s = make_uint4(gf::sub(p.x, g.x), gf::sub(p.y, g.y), 0u, 0u);
        ws[N + j] = s;
        ws[j] = s;
        if (s.x | s.y) *nonzero = 1;
    }
}

// u_j = (ws[N + j] - ws[j]) * cs_j in both folds, into rows N + j and j; cs_j = 0 on a lost parity row, so u_j = 0 there
__global__ void degraded_syndrome_kernel(uint4* __restrict__ ws, size_t N, size_t M, const uint4* __restrict__ cs)
{
    const uint32_t zero = gf::opaque_zero();
    FOR_GRID(size_t, j, M) {
        const uint4 p = ws[N + j], g = ws[j], k = __ldg(cs + j);
        const uint4 u = make_uint4(gf::mulc(gf::sub(p.x, g.x), k, zero), gf::mulc(gf::sub(p.y, g.y), k, zero), 0u, 0u);
        ws[N + j] = u;
        ws[j] = u;
    }
}

// scrub_roots_kernel over the surviving points only: row i is skipped if lost[i] != 0 or cs[i].x == 0 (either may be null)
__global__ void degraded_roots_kernel(const uint4* __restrict__ ws, size_t n, const uint8_t* __restrict__ lost, const uint4* __restrict__ cs,
                                      uint32_t* __restrict__ list, uint32_t* __restrict__ count, size_t cap)
{
    FOR_GRID(size_t, i, n) {
        if (ws[i].x || (lost && lost[i]) || (cs && !cs[i].x)) continue;
        const uint32_t k = atomicAdd(count, 1u);
        if (k < cap) list[k] = (uint32_t)i;
    }
}

__global__ void scrub_roots_kernel(const uint4* __restrict__ ws, size_t n, uint32_t* __restrict__ list, uint32_t* __restrict__ count, size_t cap)
{
    FOR_GRID(size_t, i, n) {
        if (ws[i].x) continue;
        const uint32_t k = atomicAdd(count, 1u);
        if (k < cap) list[k] = (uint32_t)i;
    }
}

__global__ void scrub_product_kernel(uint4* __restrict__ ws, size_t N, size_t M)
{
    const uint32_t zero = gf::opaque_zero();
    FOR_GRID(size_t, j, M) {
        const gf::Tw t = gf::make_tw(ws[j].x);                    // C(zeta^j) as a Barrett triple
        const uint4 k = make_uint4(t.w, t.whi, t.wlo, 0u), s = ws[N + j];
        ws[j] = make_uint4(gf::mulc(s.x, k, zero), gf::mulc(s.y, k, zero), 0u, 0u);
    }
}

__global__ void scrub_check_kernel(const uint4* __restrict__ ws, size_t L, size_t M, uint32_t* __restrict__ fail)
{
    FOR_GRID(size_t, k, M - L) {
        const uint4 v = ws[L + k];
        if (v.x | v.y) *fail = 1;
    }
}

} // namespace

namespace fecc {

cudaError_t launch_scrub_fold(const uint32_t* data, size_t dpitch, size_t N, const uint32_t* parity, size_t ppitch, size_t M, size_t size,
                              uint64_t seed, uint32_t* ws, int num_sms, cudaStream_t st)
{
    return launch_degraded_fold(data, dpitch, N, parity, ppitch, M, size, seed, nullptr, nullptr, ws, num_sms, st);
}

cudaError_t launch_degraded_fold(const uint32_t* data, size_t dpitch, size_t N, const uint32_t* parity, size_t ppitch, size_t M, size_t size,
                                 uint64_t seed, const uint8_t* lost, const uint4* cs, uint32_t* ws, int num_sms, cudaStream_t st)
{
    const uint32_t s4 = (uint32_t)((size + 3) / 4), rows = (uint32_t)(N + M);
    uint32_t log_w = 0;
    while (log_w < 5 && (1u << log_w) < s4) ++log_w;
    const uint32_t W = 1u << log_w, rw = 32 / W, tiles = (s4 + W - 1) / W;
    const size_t max_blocks = (size_t)num_sms * 4, max_warps = max_blocks * 8;
    const size_t groups = (rows + rw - 1) / rw;                         // row steps of a warp
    size_t slices = max_warps / tiles;
    slices = slices < 1 ? 1 : slices > groups ? groups : slices;
    const uint32_t slice_rows = (uint32_t)((groups + slices - 1) / slices * rw);
    slices = (rows + slice_rows - 1) / slice_rows;
    const size_t items = tiles * slices, blocks = (items + 7) / 8 < max_blocks ? (items + 7) / 8 : max_blocks;
    unsigned long long* const sums = reinterpret_cast<unsigned long long*>(ws);
    if (lost)
        degraded_fold_kernel<<<(unsigned)blocks, 256, 0, st>>>(data, dpitch, (uint32_t)N, parity, ppitch, rows, (uint32_t)size, s4, log_w, tiles,
                                                               (uint32_t)items, slice_rows, seed, sums, lost, cs);
    else
        scrub_fold_kernel<<<(unsigned)blocks, 256, 0, st>>>(data, dpitch, (uint32_t)N, parity, ppitch, rows, (uint32_t)size, s4, log_w, tiles,
                                                            (uint32_t)items, slice_rows, seed, sums);
    return cudaGetLastError();
}

cudaError_t launch_degraded_syndrome(uint32_t* ws, size_t N, size_t M, const uint4* cs, cudaStream_t st)
{
    degraded_syndrome_kernel<<<grid_size(M, 4096), 256, 0, st>>>(reinterpret_cast<uint4*>(ws), N, M, cs);
    return cudaGetLastError();
}

cudaError_t launch_degraded_roots(const uint32_t* ws, size_t n, const uint8_t* lost, const uint4* cs, uint32_t* list, uint32_t* count, size_t cap,
                                  cudaStream_t st)
{
    degraded_roots_kernel<<<grid_size(n, 4096), 256, 0, st>>>(reinterpret_cast<const uint4*>(ws), n, lost, cs, list, count, cap);
    return cudaGetLastError();
}

cudaError_t launch_scrub_reduce(uint32_t* ws, size_t n, cudaStream_t st)
{
    scrub_reduce_kernel<<<grid_size(n, 4096), 256, 0, st>>>(reinterpret_cast<uint4*>(ws), n);
    return cudaGetLastError();
}

cudaError_t launch_scrub_syndrome(uint32_t* ws, size_t N, size_t M, uint32_t* nonzero, cudaStream_t st)
{
    scrub_syndrome_kernel<<<grid_size(M, 4096), 256, 0, st>>>(reinterpret_cast<uint4*>(ws), N, M, nonzero);
    return cudaGetLastError();
}

cudaError_t launch_scrub_roots(const uint32_t* ws, size_t n, uint32_t* list, uint32_t* count, size_t cap, cudaStream_t st)
{
    scrub_roots_kernel<<<grid_size(n, 4096), 256, 0, st>>>(reinterpret_cast<const uint4*>(ws), n, list, count, cap);
    return cudaGetLastError();
}

cudaError_t launch_scrub_product(uint32_t* ws, size_t N, size_t M, cudaStream_t st)
{
    scrub_product_kernel<<<grid_size(M, 4096), 256, 0, st>>>(reinterpret_cast<uint4*>(ws), N, M);
    return cudaGetLastError();
}

cudaError_t launch_scrub_check(const uint32_t* ws, size_t L, size_t M, uint32_t* fail, cudaStream_t st)
{
    scrub_check_kernel<<<grid_size(M - L, 4096), 256, 0, st>>>(reinterpret_cast<const uint4*>(ws), L, M, fail);
    return cudaGetLastError();
}

// The textbook recurrence (Massey 1969): C the current connection polynomial, B the one before the last length change, b its
// discrepancy, m the steps since.  O(len(s) * L) products.  The discrepancy is summed unreduced in 128 bits (at most 4097
// products below 2^64) and reduced once; the update multiplies by the Barrett triple of d / b; 1 / b is computed when b changes
// (at a length change, the only step that also copies C).
size_t berlekamp_massey(const std::vector<uint32_t>& s, std::vector<uint32_t>& C)
{
    C.assign(1, 1u);
    std::vector<uint32_t> B(1, 1u), T;
    size_t L = 0, m = 1;
    uint32_t b_inv = 1;
    for (size_t n = 0; n < s.size(); ++n) {
        unsigned __int128 acc = s[n];
        const size_t top = L < C.size() ? L : C.size() - 1;
        for (size_t i = 1; i <= top; ++i) acc += (uint64_t)C[i] * s[n - i];
        const uint32_t d = (uint32_t)(acc % P);
        if (!d) { ++m; continue; }
        const gf::Tw k = gf::make_tw(gf::mulmod(d, b_inv));
        const bool grow = 2 * L <= n;
        if (grow) T = C;
        if (C.size() < B.size() + m) C.resize(B.size() + m, 0u);
        for (size_t i = 0; i < B.size(); ++i) C[i + m] = gf::sub(C[i + m], gf::canon(gf::mul(B[i], k.w, k.whi, k.wlo)));
        if (grow) { L = n + 1 - L; B.swap(T); b_inv = gf::inv(d); m = 1; }
        else ++m;
    }
    while (C.size() > 1 && !C.back()) C.pop_back();
    return L;
}

} // namespace fecc
