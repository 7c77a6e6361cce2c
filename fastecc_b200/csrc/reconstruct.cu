// Degraded read of a stored stripe (include/fastecc_b200.h: fastecc_b200_rs_reconstruct, DESIGN 3k): a few lost blocks rebuilt out
// of place from N surviving rows in one pass.
//
// On this code's points parity j = sum_i data_i * T[(D j - i) mod N] (update.h).  With E the a lost data rows and J the a lowest
// surviving parity rows, r_j = sum_{i not in E} T[(D j - i) mod N] * data_i leaves parity_j - r_j = sum_{e in E} T[(D j - e) mod N] x_e,
// an a x a Cauchy system (up to diagonal scalings) in the lost data x.  api.cu solves it on the host into a matrix B, so that every
// wanted block is [parity] r_q + sum_{j in J} B[q][j] (parity_j - r_j).  This file holds the pass over the surviving data rows
// (the K = a + |wanted parity| sums r) and the flat kernel that applies B.
#include "reconstruct.h"
#include "gf.cuh"

namespace {

using namespace fecc;
constexpr uint32_t kTile = 32;                                     // rows per tile, and 16-byte chunks per CTA
constexpr uint32_t kMaxK = FASTECC_B200_RECONSTRUCT_MAX;

// A CTA owns one slice of data rows x 32 16-byte chunks.  Per 32-row tile, the 256 threads stage the tile's data (thread t: chunk
// t % 32 of rows t / 32 + 8 s) and the T entries of the tile's rows for the K outputs in shared memory; the next tile is loaded
// into registers while the current one is consumed.  Warp w owns outputs g + G v (v < U, g = w % G) on rows h, h + S, .. of the
// tile (h = w / G, S = 8 / G), lane l chunk l: per row one 16-byte shared load, per output one broadcast triple and four products
// with lazy sums.  A tile's lost rows (a mask from a cursor over the ascending list) and rows past the slice are never loaded and
// count as zero; a tile without either loads unpredicated.  At the end every lane adds its canonical sums into the 64-bit
// workspace words of its outputs: at most 8 * (number of slices) terms below P each.
template <uint32_t U>
__global__ void __launch_bounds__(256, 2) reconstruct_sum_kernel(const uint32_t* __restrict__ data, size_t dpitch, uint32_t N, uint32_t D,
                                                                 const uint4* __restrict__ T, const uint32_t* __restrict__ pos, uint32_t K, uint32_t G,
                                                                 const uint32_t* __restrict__ lost, uint32_t a, uint32_t s4, uint32_t col_blocks,
                                                                 uint32_t slice_rows, unsigned long long* __restrict__ ws)
{
    extern __shared__ uint4 smem[];
    uint4* const sd = smem;                                        // [row][chunk]
    uint4* const stab = smem + kTile * kTile;                      // [output][row]
    __shared__ uint32_t sbase[kMaxK], slost[kMaxK];
    const uint32_t tid = threadIdx.x, lane = tid % 32, warp = tid / 32, g = warp % G, h = warp / G, S = 8 / G;
    const uint32_t c = blockIdx.x % col_blocks * kTile + lane;
    const uint32_t r0 = blockIdx.x / col_blocks * slice_rows, r1 = min(N, r0 + slice_rows);
    const bool live = c < s4;
    const uint32_t zero = gf::opaque_zero();
    const uint4 z4 = make_uint4(0, 0, 0, 0);
    if (tid < K) sbase[tid] = D * __ldg(pos + tid) + N;             // D j + N
    if (tid < a) slost[tid] = __ldg(lost + tid);
    __syncthreads();
    uint32_t cursor = 0;                                           // the first lost row at or past the tile
    uint4 pd[4], pt[4];
    auto fetch = [&](uint32_t i0) {
        while (cursor < a && slost[cursor] < i0) ++cursor;
        uint32_t skip = i0 + kTile > r1 ? ~0u << (r1 - i0) : 0u;
        for (uint32_t q = cursor; q < a && slost[q] < i0 + kTile; ++q) skip |= 1u << (slost[q] - i0);
        const uint4* col = reinterpret_cast<const uint4*>(data + (size_t)(i0 + warp) * dpitch) + c;
        if (!skip) {
#pragma unroll
            for (uint32_t s = 0; s < 4; ++s) pd[s] = live ? __ldg(col + 8 * s * dpitch / 4) : z4;
        } else {
#pragma unroll
            for (uint32_t s = 0; s < 4; ++s) pd[s] = live && !(skip >> (warp + 8 * s) & 1) ? __ldg(col + 8 * s * dpitch / 4) : z4;
        }
#pragma unroll
        for (uint32_t s = 0; s < 4; ++s) {
            const uint32_t k = warp + 8 * s;                       // the same for the whole warp
            pt[s] = z4;
            if (k < K && i0 + lane < r1) {
                uint32_t t = sbase[k] - (i0 + lane);
                if (t >= N) t -= N;
                pt[s] = __ldg(T + t);
            }
        }
    };
    uint4 acc[U];
#pragma unroll
    for (uint32_t v = 0; v < U; ++v) acc[v] = z4;
    if (r0 < r1) fetch(r0);
    for (uint32_t i0 = r0; i0 < r1; i0 += kTile) {
        __syncthreads();                                           // the previous tile is consumed
#pragma unroll
        for (uint32_t s = 0; s < 4; ++s) {
            sd[(warp + 8 * s) * kTile + lane] = pd[s];
            if (warp + 8 * s < K) stab[(warp + 8 * s) * kTile + lane] = pt[s];
        }
        __syncthreads();
        if (i0 + kTile < r1) fetch(i0 + kTile);
        for (uint32_t u = h; u < kTile; u += S) {
            const uint4 d = sd[u * kTile + lane];
#pragma unroll
            for (uint32_t v = 0; v < U; ++v) {
                const uint32_t k = g + G * v;
                if (k >= K) continue;                              // the same for the whole warp
                const uint4 w = stab[k * kTile + u];
                acc[v].x = gf::addl(acc[v].x, gf::mul(d.x, w.x, w.y, w.z, zero));
                acc[v].y = gf::addl(acc[v].y, gf::mul(d.y, w.x, w.y, w.z, zero));
                acc[v].z = gf::addl(acc[v].z, gf::mul(d.z, w.x, w.y, w.z, zero));
                acc[v].w = gf::addl(acc[v].w, gf::mul(d.w, w.x, w.y, w.z, zero));
            }
        }
    }
    if (!live) return;
#pragma unroll
    for (uint32_t v = 0; v < U; ++v) {
        const uint32_t k = g + G * v;
        if (k >= K) continue;
        unsigned long long* o = ws + ((size_t)k * s4 + c) * 4;
        atomicAdd(o + 0, (unsigned long long)gf::canon(acc[v].x));
        atomicAdd(o + 1, (unsigned long long)gf::canon(acc[v].y));
        atomicAdd(o + 2, (unsigned long long)gf::canon(acc[v].z));
        atomicAdd(o + 3, (unsigned long long)gf::canon(acc[v].w));
    }
}

// The four sums of chunk c of workspace row k, mod P
__device__ __forceinline__ uint4 sums(const ulonglong2* __restrict__ ws, uint32_t s4, uint32_t k, uint32_t c)
{
    const ulonglong2 lo = ws[((size_t)k * s4 + c) * 2], hi = ws[((size_t)k * s4 + c) * 2 + 1];
    return make_uint4(gf::reduce64(lo.x), gf::reduce64(lo.y), gf::reduce64(hi.x), gf::reduce64(hi.y));
}

// Flat over (output row, 16-byte chunk): the sums mod P, the a parity rows pos[0 .. a) taken mod P, B's triples, one store.
__global__ void __launch_bounds__(256) reconstruct_combine_kernel(const ulonglong2* __restrict__ ws, const uint32_t* __restrict__ parity, size_t ppitch,
                                                                  const uint32_t* __restrict__ pos, uint32_t a, const uint4* __restrict__ B, uint32_t n_data,
                                                                  uint32_t* __restrict__ out, size_t opitch, uint32_t s4, uint32_t n, size_t size)
{
    const uint32_t zero = gf::opaque_zero();
    FOR_GRID(uint32_t, i, n) {
        const uint32_t q = i / s4, c = i - q * s4;
        uint4 acc = q >= n_data ? sums(ws, s4, a + q - n_data, c) : make_uint4(0, 0, 0, 0);
        for (uint32_t j = 0; j < a; ++j) {
            const uint4 r = sums(ws, s4, j, c), b = __ldg(B + (size_t)q * a + j);
            const uint4 p = gf::canon4(__ldg(reinterpret_cast<const uint4*>(parity + (size_t)__ldg(pos + j) * ppitch) + c));
            acc.x = gf::addl(acc.x, gf::mul(gf::sub(p.x, r.x), b.x, b.y, b.z, zero));
            acc.y = gf::addl(acc.y, gf::mul(gf::sub(p.y, r.y), b.x, b.y, b.z, zero));
            acc.z = gf::addl(acc.z, gf::mul(gf::sub(p.z, r.z), b.x, b.y, b.z, zero));
            acc.w = gf::addl(acc.w, gf::mul(gf::sub(p.w, r.w), b.x, b.y, b.z, zero));
        }
        store_row(out + (size_t)q * opitch, 4 * (size_t)c, gf::canon4(acc), size);
    }
}

} // namespace

namespace fecc {

cudaError_t launch_reconstruct_sum(const uint32_t* data, size_t dpitch, size_t N, size_t D, const uint4* T, const uint32_t* pos, size_t K,
                                   const uint32_t* lost, size_t a, size_t size, unsigned long long* ws, int num_sms, cudaStream_t st)
{
    const uint32_t s4 = (uint32_t)((size + 3) / 4), col_blocks = (s4 + kTile - 1) / kTile, G = K <= 8 ? 1 : K <= 16 ? 2 : 4;
    const size_t tiles = (N + kTile - 1) / kTile;
    size_t slices = (size_t)num_sms * 8 / col_blocks;              // about 8 CTAs per SM, in equal slices of whole tiles
    slices = slices < 1 ? 1 : slices > tiles ? tiles : slices;
    const uint32_t slice_rows = (uint32_t)((tiles + slices - 1) / slices * kTile);
    slices = (N + slice_rows - 1) / slice_rows;
    const unsigned blocks = (unsigned)(slices * col_blocks);
    const size_t smem = (kTile + K) * kTile * sizeof(uint4);
#define RECONSTRUCT_SUM(U)                                                                                                                     \
    reconstruct_sum_kernel<U><<<blocks, 256, smem, st>>>(data, dpitch, (uint32_t)N, (uint32_t)D, T, pos, (uint32_t)K, G, lost, (uint32_t)a, s4, \
                                                         col_blocks, slice_rows, ws)
    if (K <= 1) RECONSTRUCT_SUM(1);
    else if (K <= 2) RECONSTRUCT_SUM(2);
    else if (K <= 4) RECONSTRUCT_SUM(4);
    else RECONSTRUCT_SUM(8);
#undef RECONSTRUCT_SUM
    return cudaGetLastError();
}

cudaError_t launch_reconstruct_combine(const unsigned long long* ws, const uint32_t* parity, size_t ppitch, const uint32_t* pos, size_t a, const uint4* B,
                                       size_t n_out, size_t n_data, uint32_t* out, size_t opitch, size_t size, int num_sms, cudaStream_t st)
{
    const uint32_t s4 = (uint32_t)((size + 3) / 4), n = (uint32_t)(n_out * s4);
    reconstruct_combine_kernel<<<grid_size(n, (size_t)num_sms * 16), 256, 0, st>>>(reinterpret_cast<const ulonglong2*>(ws), parity, ppitch, pos, (uint32_t)a, B,
                                                                                  (uint32_t)n_data, out, opitch, s4, n, size);
    return cudaGetLastError();
}

} // namespace fecc
