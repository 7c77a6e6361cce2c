// Degenerate orders N = 1, 2, 4, 8, 16 (below the 32-row register block of ntt_pass_kernel) and the two layout
// helpers.  One thread per 16-byte column chunk evaluates the transform by its definition (Slow_NTT,
// ntt.cpp:451-483) -- at most 16x16 products per word -- using the same power table and GF primitives as the main kernel.
#include "small_dft.h"
#include "context.h"
#include "gf.cuh"

namespace fecc {

__device__ __forceinline__ uint4 add4(uint4 a, uint4 v)
{
    a.x = gf::addl(a.x, v.x); a.y = gf::addl(a.y, v.y); a.z = gf::addl(a.z, v.z); a.w = gf::addl(a.w, v.w);
    return a;
}

// out[k] = sum_n in[n] * g^(z*n*k)          (n, k < N <= 16)
__device__ __forceinline__ void dft_small(const uint4* in, uint4* out, uint32_t N, uint32_t z, const uint4* tw, uint32_t zero)
{
    for (uint32_t k = 0; k < N; ++k) {
        uint4 acc = make_uint4(0, 0, 0, 0);
        for (uint32_t n = 0; n < N; ++n)
            acc = add4(acc, gf::mul4(in[n], tw[(z * n * k) & (gf::M - 1)], zero));
        out[k] = acc;
    }
}

__global__ void small_dft_kernel(uint32_t* data, uint32_t pitch4, uint32_t s4, uint32_t N, uint32_t z,
                                 int encode, uint32_t q, uint4 invN, const uint4* tw)
{
    const uint32_t col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= s4) return;
    const uint32_t zero = gf::opaque_zero();
    uint4* d4 = reinterpret_cast<uint4*>(data);
    uint4 x[16], y[16];
    for (uint32_t n = 0; n < N; ++n) x[n] = d4[(size_t)n * pitch4 + col];
    if (!encode) {
        dft_small(x, y, N, z, tw, zero);
    } else {                                         // RS.cpp:41-63 by definition
        dft_small(x, y, N, (gf::M - 2 * q) & (gf::M - 1), tw, zero);
        for (uint32_t m = 0; m < N; ++m) y[m] = gf::mul4(gf::mul4(y[m], tw[(q * m) & (gf::M - 1)], zero), invN, zero);
        for (uint32_t m = 0; m < N; ++m) x[m] = y[m];
        dft_small(x, y, N, 2 * q, tw, zero);
    }
    for (uint32_t n = 0; n < N; ++n) d4[(size_t)n * pitch4 + col] = gf::canon4(y[n]);
}

cudaError_t launch_small_dft(uint32_t* data, uint32_t pitch4, uint32_t s4, uint32_t N, uint32_t z, int encode,
                             uint32_t q, uint4 invN, const uint4* tw, cudaStream_t stream)
{
    const unsigned threads = 128, blocks = (s4 + threads - 1) / threads;
    small_dft_kernel<<<blocks, threads, 0, stream>>>(data, pitch4, s4, N, z, encode, q, invN, tw);
    return cudaGetLastError();
}

// [N][size] with arbitrary pitch/alignment  <->  [N][pitch4*4] 16-byte aligned, pad words zero (grid-stride; 8 CTAs per SM of an H100)
__global__ void repack_kernel(const uint32_t* src, size_t src_pitch, uint32_t* dst, size_t dst_pitch,
                              size_t n_rows, uint32_t size, uint32_t copy_cols, uint32_t zero_from)
{
    const size_t total = n_rows * (size_t)copy_cols;
    FOR_GRID(size_t, i, total) {
        const size_t r = i / copy_cols; const uint32_t c = (uint32_t)(i - r * copy_cols);
        dst[r * dst_pitch + c] = (c < zero_from && c < size) ? src[r * src_pitch + c] : 0u;
    }
}
cudaError_t launch_pack(const uint32_t* src, size_t src_pitch, uint32_t* dst, size_t dst_pitch, size_t n_rows,
                        uint32_t size, cudaStream_t stream)
{
    repack_kernel<<<1056, 256, 0, stream>>>(src, src_pitch, dst, dst_pitch, n_rows, size, (uint32_t)dst_pitch, size);
    return cudaGetLastError();
}
cudaError_t launch_unpack(const uint32_t* src, size_t src_pitch, uint32_t* dst, size_t dst_pitch, size_t n_rows,
                          uint32_t size, cudaStream_t stream)
{
    repack_kernel<<<1056, 256, 0, stream>>>(src, src_pitch, dst, dst_pitch, n_rows, size, size, size);
    return cudaGetLastError();
}

} // namespace fecc
