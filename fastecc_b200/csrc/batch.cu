// Encode of a batch of small stripes in one launch (include/fastecc_b200.h: fastecc_b200_rs_encode_batch, DESIGN 3l).
//
// On this code's points parity j = sum_i data_i * T[(D j - i) mod N] (update.h, DESIGN 3h), so for N <= 64 the M parity rows of a
// stripe are M x N products per word straight from the data rows: no transform, no workspace, one pass over the data.  update's
// parity kernel adds a product of this form into the parity from a delta workspace indexed by a list of changed rows; this one
// sums every row of the caller's layout for many stripes at once, so the two stay apart.
#include "batch.h"
#include "gf.cuh"

namespace {

using namespace fecc;
constexpr uint32_t kMaxN = FASTECC_B200_BATCH_MAX_N;
constexpr uint32_t kTileChunks = 2048;                             // staged 16-byte chunks per CTA: 32 KiB
constexpr uint32_t kMaxLoads = 11;                                 // chunks a thread loads per tile: ceil(rows per tile / W) <= 64 / 6

// The work item is (stripe, 16-byte chunk), flat: item = b * s4 + c, 64-bit.  A CTA takes G groups of 32 consecutive items; W
// warps share a group's M outputs, U each (M = W U, W <= 8, G W <= 8).  Per tile of R = 64 / G rows the CTA stages the data
// chunks of its 32 G items in shared memory (thread t loads chunk t % 32 G of rows t / 32 G + W s, 16-byte loads, pad words past
// SIZE zeroed), then warp (g, h) reads row r's chunk of item 32 g + lane from shared memory (conflict-free) and, per output
// j = h + W v, the broadcast triple T[(D j - i) mod N] staged once per CTA: four Barrett products with lazy sums.  One canon and
// one store per output; nothing past SIZE is written.
template <uint32_t U>
__global__ void __launch_bounds__(256, 2) batch_encode_kernel(const uint32_t* __restrict__ data, size_t dpitch, size_t dstride, uint32_t N,
                                                              uint32_t* __restrict__ parity, size_t ppitch, size_t pstride, uint32_t D, uint32_t W,
                                                              uint32_t G, const uint4* __restrict__ T, uint32_t s4, double inv_s4, uint64_t n_items,
                                                              size_t size)
{
    extern __shared__ uint4 sd[];                                  // [row of the tile][item of the CTA]
    __shared__ uint4 stab[kMaxN];
    const uint32_t tid = threadIdx.x, lane = tid % 32, warp = tid / 32, items = 32 * G, rows = kTileChunks / items;
    const uint32_t zero = gf::opaque_zero();
    const uint4 z4 = make_uint4(0, 0, 0, 0);
    if (tid < N) stab[tid] = __ldg(T + tid);

    // item -> (stripe, chunk) without a 64-bit division: the quotient from the FP64 unit is off by at most one for items < 2^52
    auto split = [&](uint64_t it, uint64_t& b, uint32_t& c) {
        b = (uint64_t)((double)it * inv_s4);
        int64_t r = (int64_t)(it - b * s4);
        if (r < 0) { --b; r += s4; }
        if (r >= (int64_t)s4) { ++b; r -= s4; }
        c = (uint32_t)r;
    };

    const uint32_t li = tid % items, lr = tid / items;             // the load side: one item per thread, rows lr + W s
    const uint64_t lit = (uint64_t)blockIdx.x * items + li;
    const bool lload = lit < n_items;
    uint64_t lb = 0;
    uint32_t lc = 0;
    if (lload) split(lit, lb, lc);
    const uint4* src = reinterpret_cast<const uint4*>(data + lb * dstride + (size_t)dpitch * lr) + lc;
    const size_t lstep = dpitch / 4 * W;                           // W rows, in chunks
    const uint32_t keep = size - 4 * (size_t)lc < 4 ? (uint32_t)(size - 4 * (size_t)lc) : 4u;

    const uint32_t g = warp / W, h = warp - g * W;                 // the compute side: item 32 g + lane, outputs h + W v
    const uint64_t cit = (uint64_t)blockIdx.x * items + 32 * g + lane;
    uint32_t base[U];
    uint4 acc[U];
#pragma unroll
    for (uint32_t v = 0; v < U; ++v) { base[v] = D * (h + W * v) + N; acc[v] = z4; }

    for (uint32_t i0 = 0; i0 < N; i0 += rows) {
        const uint32_t nr = N - i0 < rows ? N - i0 : rows;
        if (i0) __syncthreads();                                   // the previous tile is consumed
        uint4 buf[kMaxLoads];
#pragma unroll
        for (uint32_t s = 0; s < kMaxLoads; ++s) {
            const uint32_t r = lr + W * s;
            buf[s] = lload && r < nr ? __ldg(src + i0 * (dpitch / 4) + lstep * s) : z4;
        }
        if (keep < 4) {
#pragma unroll
            for (uint32_t s = 0; s < kMaxLoads; ++s) {
                if (keep < 2) buf[s].y = 0;
                if (keep < 3) buf[s].z = 0;
                buf[s].w = 0;
            }
        }
#pragma unroll
        for (uint32_t s = 0; s < kMaxLoads; ++s) {
            const uint32_t r = lr + W * s;
            if (r < nr) sd[r * items + li] = buf[s];
        }
        __syncthreads();
        for (uint32_t r = 0; r < nr; ++r) {
            const uint4 d = sd[r * items + 32 * g + lane];
            const uint32_t i = i0 + r;
#pragma unroll
            for (uint32_t v = 0; v < U; ++v) {
                uint32_t t = base[v] - i;
                if (t >= N) t -= N;
                const uint4 w = stab[t];
                acc[v].x = gf::addl(acc[v].x, gf::mul(d.x, w.x, w.y, w.z, zero));
                acc[v].y = gf::addl(acc[v].y, gf::mul(d.y, w.x, w.y, w.z, zero));
                acc[v].z = gf::addl(acc[v].z, gf::mul(d.z, w.x, w.y, w.z, zero));
                acc[v].w = gf::addl(acc[v].w, gf::mul(d.w, w.x, w.y, w.z, zero));
            }
        }
    }
    if (cit >= n_items) return;
    uint64_t cb;
    uint32_t cc;
    split(cit, cb, cc);
    uint32_t* dst = parity + cb * pstride + (size_t)ppitch * h + 4 * (size_t)cc;
    if (4 * (size_t)cc + 4 <= size) {                              // whole chunks (all but a row's partial last): one 16-byte store each;
#pragma unroll                                                     // __stcg keeps the compiler from merging it with the scalar path below
        for (uint32_t v = 0; v < U; ++v) __stcg(reinterpret_cast<uint4*>(dst + (size_t)ppitch * W * v), gf::canon4(acc[v]));
    } else {
#pragma unroll
        for (uint32_t v = 0; v < U; ++v) store_row(dst + (size_t)ppitch * W * v, 0, gf::canon4(acc[v]), size - 4 * (size_t)cc);
    }
}

} // namespace

namespace fecc {

cudaError_t launch_batch_encode(const uint32_t* data, size_t dpitch, size_t dstride, size_t N, uint32_t* parity, size_t ppitch, size_t pstride,
                                size_t M, size_t B, size_t size, const uint4* T, cudaStream_t st)
{
    uint32_t U = 1;                                                // the fewest outputs per warp with at most 8 warps per group
    while (M % U || M / U > 8) ++U;
    const uint32_t W = (uint32_t)(M / U), G = 8 / W >= 8 ? 8 : 8 / W >= 4 ? 4 : 8 / W >= 2 ? 2 : 1;
    const uint32_t s4 = (uint32_t)((size + 3) / 4), items = 32 * G, rows = kTileChunks / items;
    const uint64_t n_items = (uint64_t)B * s4;
    const unsigned blocks = (unsigned)((n_items + items - 1) / items);
    const size_t smem = (size_t)(N < rows ? N : rows) * items * sizeof(uint4);
#define BATCH_ENCODE(UU)                                                                                                                            \
    batch_encode_kernel<UU><<<blocks, 32 * W * G, smem, st>>>(data, dpitch, dstride, (uint32_t)N, parity, ppitch, pstride, (uint32_t)(N / M), W, G, T, \
                                                              s4, 1.0 / s4, n_items, size)
    switch (U) {
    case 1: BATCH_ENCODE(1); break;
    case 2: BATCH_ENCODE(2); break;
    case 3: BATCH_ENCODE(3); break;
    case 4: BATCH_ENCODE(4); break;
    case 6: BATCH_ENCODE(6); break;
    case 8: BATCH_ENCODE(8); break;
    default: return cudaErrorInvalidValue;                         // M <= 64 divides N: U is one of the above
    }
#undef BATCH_ENCODE
    return cudaGetLastError();
}

} // namespace fecc
