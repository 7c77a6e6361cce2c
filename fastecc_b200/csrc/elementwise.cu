// Element-wise GF(P) helpers used around the transforms (erasure decoding, SURVEY 8f rank 4): products of two arrays
// (GF_Mul, GF(p).cpp:110-127), inverses (GF_Inv, GF(p).cpp:293-297: x^(P-2)) and "multiply block i by a constant c[i]"
// (the shape of the reference's scaling loop, RS.cpp:51-59, with an arbitrary constant per block).  The first two work on
// short vectors (one value per block); row_scale streams the block array once: HBM-bound, 16-byte accesses.
#include "elementwise.h"
#include "context.h"
#include "gf.cuh"

namespace fecc {

__global__ void gf_mul_kernel(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, uint32_t* __restrict__ out, size_t n)
{
    FOR_GRID(size_t, i, n) out[i] = gf::mulmod(a[i], b[i]);
}
__global__ void gf_inv_kernel(const uint32_t* __restrict__ a, uint32_t* __restrict__ out, size_t n)
{
    FOR_GRID(size_t, i, n) {
        const uint32_t x = a[i] % gf::P;
        out[i] = x ? gf::inv(x) : 0u;
    }
}

// One CTA per row (grid-stride over rows): thread 0 turns the row's constant into its Barrett/Shoup triple
// (gf::make_tw: two 64-by-32 divisions), every thread then multiplies 16-byte chunks with gf::mul4.
__global__ void __launch_bounds__(256) row_scale_kernel(uint4* __restrict__ d, size_t n_rows, uint32_t s4, uint32_t pitch4, const uint32_t* __restrict__ consts)
{
    __shared__ uint32_t tw[3];
    const uint32_t zero = gf::opaque_zero();
    for (size_t row = blockIdx.x; row < n_rows; row += gridDim.x) {
        __syncthreads();
        if (threadIdx.x == 0) { const gf::Tw t = gf::make_tw(consts[row] % gf::P); tw[0] = t.w; tw[1] = t.whi; tw[2] = t.wlo; }
        __syncthreads();
        const uint4 t = make_uint4(tw[0], tw[1], tw[2], 0u);
        uint4* r = d + row * pitch4;
        for (uint32_t c = threadIdx.x; c < s4; c += blockDim.x) r[c] = gf::canon4(gf::mul4(r[c], t, zero));
    }
}

// Cross-GPU barrier on a stream (one process per GPU, buffers mapped with CUDA IPC): rank r owns an array of n_ranks 32-bit
// flags.  Lane p of one warp writes `epoch` into flag [rank] of peer p (over NVLink) and then waits until its own flag [p]
// has reached `epoch`.  The kernel runs behind the pass whose peer stores it has to publish: those are complete when it
// starts (stream order), the fence orders them before the flag.  A peer that never arrives would spin forever, so the wait
// gives up after about ten seconds and reports through *err (the next host-side check fails loudly instead of hanging).
struct BarrierArgs { uint32_t* peers[8]; };
__global__ void shard_barrier_kernel_args(BarrierArgs a, const uint32_t* own, uint32_t n_ranks, uint32_t rank, uint32_t epoch, uint32_t* err)
{
    const uint32_t p = threadIdx.x;
    if (p >= n_ranks) return;
    __threadfence_system();
    volatile uint32_t* remote = a.peers[p] + rank;
    *remote = epoch;
    __threadfence_system();
    const volatile uint32_t* mine = own + p;
    const long long t0 = clock64();
    while ((int32_t)(*mine - epoch) < 0) {
        if (clock64() - t0 > 20000000000ll) { atomicExch(err, 1u); break; }
        __nanosleep(100);
    }
    __threadfence_system();
}

cudaError_t launch_shard_barrier(uint32_t* const* host_peers, uint32_t n_ranks, uint32_t rank, uint32_t epoch, cudaStream_t st)
{
    if (n_ranks > 8 || rank >= n_ranks) return cudaErrorInvalidValue;
    BarrierArgs a;
    for (uint32_t r = 0; r < 8; ++r) a.peers[r] = host_peers[r < n_ranks ? r : 0];
    // flag layout of a rank: [0, 8) arrival flags, [8] error word
    shard_barrier_kernel_args<<<1, 32, 0, st>>>(a, host_peers[rank], n_ranks, rank, epoch, host_peers[rank] + 8);
    return cudaGetLastError();
}

cudaError_t launch_gf_mul(const uint32_t* a, const uint32_t* b, uint32_t* out, size_t n, cudaStream_t st)
{
    if (!n) return cudaSuccess;
    gf_mul_kernel<<<grid_size(n, 4096), 256, 0, st>>>(a, b, out, n);
    return cudaGetLastError();
}
cudaError_t launch_gf_inv(const uint32_t* a, uint32_t* out, size_t n, cudaStream_t st)
{
    if (!n) return cudaSuccess;
    gf_inv_kernel<<<grid_size(n, 4096), 256, 0, st>>>(a, out, n);
    return cudaGetLastError();
}
cudaError_t launch_row_scale(uint32_t* d, size_t n_rows, uint32_t s4, uint32_t pitch4, const uint32_t* consts, int num_sms, cudaStream_t st)
{
    if (!n_rows) return cudaSuccess;
    const size_t cap = (size_t)num_sms * 8;
    row_scale_kernel<<<(unsigned)(n_rows < cap ? n_rows : cap), 256, 0, st>>>(reinterpret_cast<uint4*>(d), n_rows, s4, pitch4, consts);
    return cudaGetLastError();
}

} // namespace fecc
