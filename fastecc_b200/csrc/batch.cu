// Encode of a batch of small stripes in one launch (include/fastecc_b200.h: fastecc_b200_rs_encode_batch, DESIGN 3l).
//
// On this code's points parity j = sum_i data_i * T[(D j - i) mod N] (update.h, DESIGN 3h), so for N <= 64 the M parity rows of a
// stripe are M x N products per word straight from the data rows: no transform, no workspace, one pass over the data.  update's
// parity kernel adds a product of this form into the parity from a delta workspace indexed by a list of changed rows; this one
// sums every row of the caller's layout for many stripes at once, so the two stay apart.
//
// The degraded read of a batch with one loss pattern (fastecc_b200_rs_reconstruct_batch, DESIGN 3m) has the same shape: every
// wanted block is a fixed n_out x N combination C of the N rows it reads, which api.cu folds from the single-stripe read's algebra.
#include "batch.h"
#include "gf.cuh"
#include <algorithm>

namespace {

using namespace fecc;
constexpr uint32_t kMaxN = FASTECC_B200_BATCH_MAX_N;
constexpr uint32_t kTileChunks = 2048;                             // staged 16-byte chunks per CTA: 32 KiB
constexpr uint32_t kMaxLoads = 11;                                 // chunks a thread loads per tile: ceil(rows per tile / W) <= 64 / 6

// Item -> (stripe, chunk) without a 64-bit division: the quotient from the FP64 unit is off by at most one for items < 2^52.
__device__ __forceinline__ void split_item(uint64_t it, uint32_t s4, double inv_s4, uint64_t& b, uint32_t& c)
{
    b = (uint64_t)((double)it * inv_s4);
    int64_t r = (int64_t)(it - b * s4);
    if (r < 0) { --b; r += s4; }
    if (r >= (int64_t)s4) { ++b; r -= s4; }
    c = (uint32_t)r;
}

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
    auto split = [&](uint64_t it, uint64_t& b, uint32_t& c) { split_item(it, s4, inv_s4, b, c); };

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

// 16 bytes global -> shared without registers; of the 16 only `bytes` are read, the rest of the destination is zero-filled.
__device__ __forceinline__ void copy16_async(uint4* dst, const void* src, uint32_t bytes)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void commit_async() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
// Waits until at most n of this thread's committed groups are still in flight (n < 4).
__device__ __forceinline__ void wait_async(uint32_t n)
{
    switch (n) {
    case 0: asm volatile("cp.async.wait_group 0;\n" ::: "memory"); break;
    case 1: asm volatile("cp.async.wait_group 1;\n" ::: "memory"); break;
    case 2: asm volatile("cp.async.wait_group 2;\n" ::: "memory"); break;
    default: asm volatile("cp.async.wait_group 3;\n" ::: "memory"); break;
    }
}

// Degraded read of a batch with one loss pattern (fastecc_b200_rs_reconstruct_batch, DESIGN 3m): wanted block q of every stripe =
// sum_s C[q][s] * source row s, the sources being the nd surviving data rows (data side) and then the parity rows J (parity side).
// A CTA stages C (n_out x N triples) and the N source row pointers once, then runs tiles of items = 2^lg_items consecutive items
// (32 <= items, N items >= 2048: every tile loads 32 to 48 KiB) in a grid-stride loop, through a ring of `stages` tile buffers in
// shared memory: thread t copies the tile's flat chunks f = t + 256 s, s < N items / 256 (row f >> lg_items, item f & (items - 1)),
// with 16-byte cp.async, `stages` - 1 tiles ahead of the one consumed; the copy of a partial last chunk reads the words below SIZE
// and zero-fills the pad words.  A work unit is a group g of 32 items with the outputs h + W v (v < U, W = ceil(n_out / U) <= 8);
// the 8 warps take the tile's units = items / 32 * W units in turn.  With fewer than 8 units (then U = 1) each unit's rows are
// split over R = `slices` warps, whose canonical partial sums the first one adds.  Per row one conflict-free 16-byte shared load,
// per output a broadcast triple and four Barrett products with lazy sums; one canon and one store per output.  Nothing but words
// [0, SIZE) of the output rows is written.
template <uint32_t U>
__global__ void __launch_bounds__(256, 2) batch_reconstruct_kernel(const uint32_t* __restrict__ data, size_t dpitch, size_t dstride,
                                                                   const uint32_t* __restrict__ parity, size_t ppitch, size_t pstride, uint32_t N,
                                                                   uint32_t nd, const uint4* __restrict__ C, const uint32_t* __restrict__ src,
                                                                   uint32_t n_out, uint32_t W, uint32_t slices, uint32_t stages, uint32_t* __restrict__ out,
                                                                   size_t opitch, size_t ostride, uint32_t lg_items, uint32_t s4, double inv_s4,
                                                                   uint64_t n_items, uint64_t n_tiles, size_t size)
{
    extern __shared__ uint4 smem[];
    uint4* const sc = smem;                                        // [output][source row]
    uint4* const ring = smem + n_out * N;                          // [stage][source row][item of the tile]
    __shared__ const uint32_t* srow[kMaxN];
    __shared__ uint4 spart[7 * 32];                                // partial sums of slices 1 .. 7: [slice - 1][unit][lane]
    const uint32_t tid = threadIdx.x, lane = tid % 32, warp = tid / 32, items = 1u << lg_items, chunks = N << lg_items, loads = chunks / 256;
    const uint32_t units = items / 32 * W, zero = gf::opaque_zero();
    const uint4 z4 = make_uint4(0, 0, 0, 0);
    for (uint32_t i = tid; i < n_out * N; i += 256) sc[i] = __ldg(C + i);
    if (tid < N) {
        const size_t r = __ldg(src + tid);
        srow[tid] = tid < nd ? data + r * dpitch : parity + r * ppitch;
    }
    __syncthreads();

    uint64_t next = blockIdx.x;                                    // the next tile to copy, into ring slot `put`
    uint32_t put = 0;
    auto issue = [&]() {
        if (next < n_tiles) {
            uint4* const slot = ring + (size_t)put * chunks;
            const uint64_t tile = next;
            for (uint32_t s = 0; s < loads; ++s) {
                const uint32_t f = tid + 256 * s, r = f >> lg_items;
                const uint64_t it = (tile << lg_items) + (f & (items - 1));
                if (it < n_items) {
                    uint64_t b;
                    uint32_t c;
                    split_item(it, s4, inv_s4, b, c);
                    const size_t keep = size - 4 * (size_t)c;
                    copy16_async(slot + f, srow[r] + b * (r < nd ? dstride : pstride) + 4 * (size_t)c, keep < 4 ? 4 * (uint32_t)keep : 16u);
                } else {
                    slot[f] = z4;
                }
            }
        }
        commit_async();
        next += gridDim.x;
        put = put + 1 == stages ? 0 : put + 1;
    };
    for (uint32_t k = 0; k + 1 < stages; ++k) issue();
    for (uint64_t tile = blockIdx.x, get = 0; tile < n_tiles; tile += gridDim.x, get = get + 1 == stages ? 0 : get + 1) {
        issue();                                                   // stages - 1 tiles ahead, into the slot consumed in the previous round
        wait_async(stages - 1);
        __syncthreads();                                           // this tile is in slot `get`
        const uint4* const sd = ring + (size_t)get * chunks;
        const uint32_t jobs = slices > 1 ? units * slices : units;
        for (uint32_t u = warp; u < jobs; u += 8) {
            const uint32_t unit = slices > 1 ? u % units : u, slice = slices > 1 ? u / units : 0;
            const uint32_t g = unit / W, h = unit - g * W;
            uint4 acc[U];
#pragma unroll
            for (uint32_t v = 0; v < U; ++v) acc[v] = z4;
            const uint4* col = sd + 32 * g + lane;
            for (uint32_t r = slice; r < N; r += slices) {
                const uint4 d = col[r << lg_items];
#pragma unroll
                for (uint32_t v = 0; v < U; ++v) {
                    if (h + W * v >= n_out) continue;              // the same for the whole warp
                    const uint4 w = sc[(h + W * v) * N + r];
                    acc[v].x = gf::addl(acc[v].x, gf::mul(d.x, w.x, w.y, w.z, zero));
                    acc[v].y = gf::addl(acc[v].y, gf::mul(d.y, w.x, w.y, w.z, zero));
                    acc[v].z = gf::addl(acc[v].z, gf::mul(d.z, w.x, w.y, w.z, zero));
                    acc[v].w = gf::addl(acc[v].w, gf::mul(d.w, w.x, w.y, w.z, zero));
                }
            }
            if (slices > 1) {                                      // U = 1 and one job per warp (warps 0 .. jobs - 1): slices 1 .. R - 1
                if (slice) {                                       // hand their canonical partial sums to slice 0 through barrier 1
                    spart[((slice - 1) * units + unit) * 32 + lane] = gf::canon4(acc[0]);
                    asm volatile("bar.arrive 1, %0;\n" ::"r"(32 * jobs) : "memory");
                    continue;
                }
                asm volatile("bar.sync 1, %0;\n" ::"r"(32 * jobs) : "memory");
                for (uint32_t k2 = 1; k2 < slices; ++k2) {
                    const uint4 p = spart[((k2 - 1) * units + unit) * 32 + lane];
                    acc[0].x = gf::addl(acc[0].x, p.x);
                    acc[0].y = gf::addl(acc[0].y, p.y);
                    acc[0].z = gf::addl(acc[0].z, p.z);
                    acc[0].w = gf::addl(acc[0].w, p.w);
                }
            }
            const uint64_t it = (tile << lg_items) + 32 * g + lane;
            if (it >= n_items) continue;
            uint64_t b;
            uint32_t c;
            split_item(it, s4, inv_s4, b, c);
            uint32_t* dst = out + b * ostride + (size_t)opitch * h + 4 * (size_t)c;
            if (4 * (size_t)c + 4 <= size) {
#pragma unroll
                for (uint32_t v = 0; v < U; ++v)
                    if (h + W * v < n_out) __stcg(reinterpret_cast<uint4*>(dst + (size_t)opitch * W * v), gf::canon4(acc[v]));
            } else {
#pragma unroll
                for (uint32_t v = 0; v < U; ++v)
                    if (h + W * v < n_out) store_row(dst + (size_t)opitch * W * v, 0, gf::canon4(acc[v]), size - 4 * (size_t)c);
            }
        }
        __syncthreads();                                           // the slot (and spart) is consumed
    }
    wait_async(0);
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

cudaError_t launch_batch_reconstruct(const uint32_t* data, size_t dpitch, size_t dstride, const uint32_t* parity, size_t ppitch, size_t pstride,
                                     size_t N, size_t nd, const uint4* C, const uint32_t* src, size_t n_out, uint32_t* out, size_t opitch,
                                     size_t ostride, size_t B, size_t size, int num_sms, cudaStream_t st)
{
    const uint32_t U = n_out <= 8 ? 1 : n_out <= 16 ? 2 : n_out <= 24 ? 3 : n_out <= 32 ? 4 : n_out <= 48 ? 6 : 8;
    const uint32_t W = (uint32_t)((n_out + U - 1) / U);
    uint32_t lg_items = 5;                                         // the fewest items, a power of two, with a tile of >= 2048 chunks
    while ((N << lg_items) < kTileChunks) ++lg_items;
    const uint32_t units = (1u << lg_items) / 32 * W, slices = U == 1 && units < 8 ? 8 / units : 1;
    // Ring stages: as many tiles (up to 4) as fit beside C in the shared memory of one of two CTAs per SM, at least one
    const size_t tile = (N << lg_items) * sizeof(uint4), coef = n_out * N * sizeof(uint4), budget = (size_t)109 << 10;
    const uint32_t stages = coef + 2 * tile <= budget ? (uint32_t)std::min<size_t>(4, (budget - coef) / tile) : 1;
    const uint32_t s4 = (uint32_t)((size + 3) / 4);
    const uint64_t n_items = (uint64_t)B * s4, n_tiles = (n_items + (1u << lg_items) - 1) >> lg_items;
    const size_t smem = coef + stages * tile;
    int per_sm = 0;
#define BATCH_RECONSTRUCT(UU)                                                                                                                    \
    do {                                                                                                                                         \
        if (cudaError_t e = cudaFuncSetAttribute(batch_reconstruct_kernel<UU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) return e; \
        if (cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, batch_reconstruct_kernel<UU>, 256, smem)) return e;           \
        const uint64_t cap = (uint64_t)(per_sm > 1 ? per_sm : 1) * num_sms;                                                                     \
        batch_reconstruct_kernel<UU><<<(unsigned)(n_tiles < cap ? n_tiles : cap), 256, smem, st>>>(                                                \
            data, dpitch, dstride, parity, ppitch, pstride, (uint32_t)N, (uint32_t)nd, C, src, (uint32_t)n_out, W, slices, stages, out, opitch,   \
            ostride, lg_items, s4, 1.0 / s4, n_items, n_tiles, size);                                                                            \
    } while (0)
    switch (U) {
    case 1: BATCH_RECONSTRUCT(1); break;
    case 2: BATCH_RECONSTRUCT(2); break;
    case 3: BATCH_RECONSTRUCT(3); break;
    case 4: BATCH_RECONSTRUCT(4); break;
    case 6: BATCH_RECONSTRUCT(6); break;
    default: BATCH_RECONSTRUCT(8); break;
    }
#undef BATCH_RECONSTRUCT
    return cudaGetLastError();
}

} // namespace fecc

namespace {

// Dynamic shared memory of batch_update_kernel's ring: with its 4.8 KiB of static arrays and the 1 KiB the SM reserves per CTA,
// two CTAs fit in the 228 KiB of an SM
constexpr uint32_t kUpdateRingBudget = 108 << 10;

// Update of a batch in place with one changed list (fastecc_b200_rs_update_batch, DESIGN 3n): parity j of every stripe +=
// sum_q (new_q - old_{e_q}) * T[(D j - e_q) mod N], and data row e_q := canon(new_q).  The skeleton of batch_reconstruct_kernel:
// persistent CTAs walk tiles of items = 2^lg_items consecutive items through a ring of `stages` slots filled by 16-byte cp.async
// (pad words zero-filled).  A tile holds rows = 2k + M rows: the k old changed data rows, the k new rows, then the M parity rows.
// Once a tile has landed, thread t takes the flat (changed row, item) pairs t + 256 s: it stores the canonical new chunk into the
// data row and leaves delta = subl(new, canon(old)) in the old row's slot, so every old word is in shared memory before it is
// overwritten.  After a barrier the work units (group g of 32 items, outputs h + W v) start from the stored parity chunk, raw, add
// delta times the broadcast triple from the T staged once per CTA with Barrett products and lazy sums (k M products per word), and
// end with one canon and one store; with fewer than 8 units the k rows are split over `slices` warps as in the degraded read.  The
// stripes are read through cp.async only (L2, never the non-coherent path), and nothing but words [0, SIZE) of the changed data
// rows and the parity rows is written; the layout rule makes each written word one that only its own item reads.
struct ChangedRows { uint32_t e[kMaxN]; };

template <uint32_t U>
__global__ void __launch_bounds__(256, 2) batch_update_kernel(uint32_t* data, size_t dpitch, size_t dstride, uint32_t N, uint32_t* parity,
                                                              size_t ppitch, size_t pstride, uint32_t M, const uint32_t* nw, size_t npitch,
                                                              size_t nstride, const ChangedRows ch, uint32_t k, const uint4* __restrict__ T,
                                                              uint32_t W, uint32_t slices, uint32_t stages, uint32_t lg_items, uint32_t s4,
                                                              double inv_s4, uint64_t n_items, uint64_t n_tiles, size_t size)
{
    extern __shared__ uint4 ring[];                                // [stage][row of the tile][item of the tile]
    __shared__ uint4 stab[kMaxN];
    __shared__ uint32_t se[kMaxN];
    __shared__ uint4 spart[7 * 32];                                // partial sums of slices 1 .. 7: [slice - 1][unit][lane]
    const uint32_t tid = threadIdx.x, lane = tid % 32, warp = tid / 32, items = 1u << lg_items, rows = 2 * k + M, chunks = rows << lg_items;
    const uint32_t units = items / 32 * W, D = N / M, zero = gf::opaque_zero();
    const uint4 z4 = make_uint4(0, 0, 0, 0);
    if (tid < N) stab[tid] = __ldg(T + tid);
    if (tid < k) se[tid] = ch.e[tid];
    __syncthreads();

    uint64_t next = blockIdx.x;                                    // the next tile to copy, into ring slot `put`
    uint32_t put = 0;
    auto issue = [&]() {
        if (next < n_tiles) {
            uint4* const slot = ring + (size_t)put * chunks;
            const uint64_t tile = next;
            for (uint32_t f = tid; f < chunks; f += 256) {
                const uint32_t r = f >> lg_items;
                const uint64_t it = (tile << lg_items) + (f & (items - 1));
                if (it < n_items) {
                    uint64_t b;
                    uint32_t c;
                    split_item(it, s4, inv_s4, b, c);
                    const uint32_t* row = r < k ? data + b * dstride + se[r] * dpitch
                                        : r < 2 * k ? nw + b * nstride + (r - k) * npitch : parity + b * pstride + (r - 2 * k) * ppitch;
                    const size_t keep = size - 4 * (size_t)c;
                    copy16_async(slot + f, row + 4 * (size_t)c, keep < 4 ? 4 * (uint32_t)keep : 16u);
                } else {
                    slot[f] = z4;
                }
            }
        }
        commit_async();
        next += gridDim.x;
        put = put + 1 == stages ? 0 : put + 1;
    };
    for (uint32_t s = 0; s + 1 < stages; ++s) issue();
    for (uint64_t tile = blockIdx.x, get = 0; tile < n_tiles; tile += gridDim.x, get = get + 1 == stages ? 0 : get + 1) {
        issue();                                                   // stages - 1 tiles ahead, into the slot consumed in the previous round
        wait_async(stages - 1);
        __syncthreads();                                           // this tile is in slot `get`
        uint4* const sd = ring + (size_t)get * chunks;
        for (uint32_t f = tid; f < k << lg_items; f += 256) {      // the new rows into the data, the deltas into the old rows' slots
            const uint32_t q = f >> lg_items;
            const uint64_t it = (tile << lg_items) + (f & (items - 1));
            const uint4 o = gf::canon4(sd[f]), n = sd[f + (k << lg_items)];
            sd[f] = make_uint4(gf::subl(n.x, o.x), gf::subl(n.y, o.y), gf::subl(n.z, o.z), gf::subl(n.w, o.w));
            if (it >= n_items) continue;
            uint64_t b;
            uint32_t c;
            split_item(it, s4, inv_s4, b, c);
            uint32_t* dst = data + b * dstride + se[q] * dpitch + 4 * (size_t)c;
            if (4 * (size_t)c + 4 <= size) __stcg(reinterpret_cast<uint4*>(dst), gf::canon4(n));
            else store_row(dst, 0, gf::canon4(n), size - 4 * (size_t)c);
        }
        __syncthreads();                                           // every delta of the tile is in place
        const uint32_t jobs = slices > 1 ? units * slices : units;
        for (uint32_t u = warp; u < jobs; u += 8) {
            const uint32_t unit = slices > 1 ? u % units : u, slice = slices > 1 ? u / units : 0;
            const uint32_t g = unit / W, h = unit - g * W;
            const uint4* col = sd + 32 * g + lane;
            uint4 acc[U];
            uint32_t base[U];
#pragma unroll
            for (uint32_t v = 0; v < U; ++v) {
                const uint32_t j = h + W * v;
                acc[v] = slice == 0 && j < M ? col[(2 * k + j) << lg_items] : z4;
                base[v] = D * j + N;
            }
            for (uint32_t q = slice; q < k; q += slices) {
                const uint4 d = col[q << lg_items];
                const uint32_t e = se[q];
#pragma unroll
                for (uint32_t v = 0; v < U; ++v) {
                    if (h + W * v >= M) continue;                  // the same for the whole warp
                    uint32_t t = base[v] - e;
                    if (t >= N) t -= N;
                    const uint4 w = stab[t];
                    acc[v].x = gf::addl(acc[v].x, gf::mul(d.x, w.x, w.y, w.z, zero));
                    acc[v].y = gf::addl(acc[v].y, gf::mul(d.y, w.x, w.y, w.z, zero));
                    acc[v].z = gf::addl(acc[v].z, gf::mul(d.z, w.x, w.y, w.z, zero));
                    acc[v].w = gf::addl(acc[v].w, gf::mul(d.w, w.x, w.y, w.z, zero));
                }
            }
            if (slices > 1) {                                      // U = 1 and one job per warp: slices 1 .. R - 1 hand their sums to slice 0
                if (slice) {
                    spart[((slice - 1) * units + unit) * 32 + lane] = gf::canon4(acc[0]);
                    asm volatile("bar.arrive 1, %0;\n" ::"r"(32 * jobs) : "memory");
                    continue;
                }
                asm volatile("bar.sync 1, %0;\n" ::"r"(32 * jobs) : "memory");
                for (uint32_t s = 1; s < slices; ++s) {
                    const uint4 p = spart[((s - 1) * units + unit) * 32 + lane];
                    acc[0].x = gf::addl(acc[0].x, p.x);
                    acc[0].y = gf::addl(acc[0].y, p.y);
                    acc[0].z = gf::addl(acc[0].z, p.z);
                    acc[0].w = gf::addl(acc[0].w, p.w);
                }
            }
            const uint64_t it = (tile << lg_items) + 32 * g + lane;
            if (it >= n_items) continue;
            uint64_t b;
            uint32_t c;
            split_item(it, s4, inv_s4, b, c);
            uint32_t* dst = parity + b * pstride + (size_t)ppitch * h + 4 * (size_t)c;
            if (4 * (size_t)c + 4 <= size) {
#pragma unroll
                for (uint32_t v = 0; v < U; ++v)
                    if (h + W * v < M) __stcg(reinterpret_cast<uint4*>(dst + (size_t)ppitch * W * v), gf::canon4(acc[v]));
            } else {
#pragma unroll
                for (uint32_t v = 0; v < U; ++v)
                    if (h + W * v < M) store_row(dst + (size_t)ppitch * W * v, 0, gf::canon4(acc[v]), size - 4 * (size_t)c);
            }
        }
        __syncthreads();                                           // the slot (and spart) is consumed
    }
    wait_async(0);
}

} // namespace

namespace fecc {

cudaError_t launch_batch_update(uint32_t* data, size_t dpitch, size_t dstride, size_t N, uint32_t* parity, size_t ppitch, size_t pstride, size_t M,
                                const uint32_t* changed, size_t k, const uint32_t* nw, size_t npitch, size_t nstride, size_t B, size_t size,
                                const uint4* T, int num_sms, cudaStream_t st)
{
    const uint32_t U = M <= 8 ? 1 : M <= 16 ? 2 : M <= 24 ? 3 : M <= 32 ? 4 : M <= 48 ? 6 : 8;
    const uint32_t W = (uint32_t)((M + U - 1) / U), rows = (uint32_t)(2 * k + M);
    uint32_t lg_items = 5;                                         // the fewest items, a power of two, with a tile of >= 2048 chunks
    while ((rows << lg_items) < kTileChunks) ++lg_items;
    const uint32_t units = (1u << lg_items) / 32 * W, slices = U == 1 && units < 8 ? (uint32_t)std::min<size_t>(8 / units, k) : 1;
    // Ring stages: as many tiles (up to 4) as fit in the shared memory of one of two CTAs per SM beside the static arrays, at least one
    const size_t tile = ((size_t)rows << lg_items) * sizeof(uint4), budget = (size_t)kUpdateRingBudget;
    const uint32_t stages = 2 * tile <= budget ? (uint32_t)std::min<size_t>(4, budget / tile) : 1;
    const uint32_t s4 = (uint32_t)((size + 3) / 4);
    const uint64_t n_items = (uint64_t)B * s4, n_tiles = (n_items + (1u << lg_items) - 1) >> lg_items;
    const size_t smem = stages * tile;
    ChangedRows ch{};
    for (size_t q = 0; q < k; ++q) ch.e[q] = changed[q];
    int per_sm = 0;
#define BATCH_UPDATE(UU)                                                                                                                     \
    do {                                                                                                                                     \
        if (cudaError_t e = cudaFuncSetAttribute(batch_update_kernel<UU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) return e;  \
        if (cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, batch_update_kernel<UU>, 256, smem)) return e;            \
        const uint64_t cap = (uint64_t)(per_sm > 1 ? per_sm : 1) * num_sms;                                                                  \
        batch_update_kernel<UU><<<(unsigned)(n_tiles < cap ? n_tiles : cap), 256, smem, st>>>(                                                 \
            data, dpitch, dstride, (uint32_t)N, parity, ppitch, pstride, (uint32_t)M, nw, npitch, nstride, ch, (uint32_t)k, T, W, slices, stages, \
            lg_items, s4, 1.0 / s4, n_items, n_tiles, size);                                                                                 \
    } while (0)
    switch (U) {
    case 1: BATCH_UPDATE(1); break;
    case 2: BATCH_UPDATE(2); break;
    case 3: BATCH_UPDATE(3); break;
    case 4: BATCH_UPDATE(4); break;
    case 6: BATCH_UPDATE(6); break;
    default: BATCH_UPDATE(8); break;
    }
#undef BATCH_UPDATE
    return cudaGetLastError();
}

} // namespace fecc
