// Which pipe does each instruction of the butterfly use on sm_90a?  Throughput of single SASS instructions and of the lazy
// add's two forms (IADD3 + @P VIADD, IADD3 + @P IMAD), alone and in pairs: two instructions on different pipes overlap,
// on one pipe their costs add (numbers and the pipe map they give: DESIGN.md section 4).  Scratch tool, not product.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o scratch/pipebench tools/pipebench.cu
//
// Every kernel is launched with exactly as many 256-thread CTAs as fit on the GPU at once (occupancy query, at most 4 per SM),
// so all warps run side by side; each CTA times its loop with clock64 and the longest span counts.  The figure printed is SM
// clock cycles per op per warp per SM sub-partition (SMSP): 2.0 for an instruction on a pipe of 16 lanes per SMSP.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t lo32(double x) { return (uint32_t)__double2loint(x); }

// the ops; `one` is a kernel argument equal to 1, which the compiler cannot fold
#define OP_IADD3   asm volatile("add.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(a[(i + 1) % NB]))     // a register operand that changes: no folding
#define OP_IMAD    asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(b[i]), "r"(c[i]))
#define OP_MNMX    asm volatile("{\n\t.reg .u32 t;\n\tsub.u32 t, %0, 0xFFF00001;\n\tmin.u32 %0, %0, t;\n\t}" : "+r"(a[i]))
#define OP_ADDL_V  asm volatile("{\n\t.reg .pred q;\n\t.reg .u32 k;\n\tadd.cc.u32 %0, %0, %1;\n\taddc.u32 k, 0, 0;\n\tsetp.ne.u32 q, k, 0;\n\t@q add.u32 %0, %0, 0xFFFFF;\n\t}" : "+r"(a[i]) : "r"(b[i]))
#define OP_ADDL_M  asm volatile("{\n\t.reg .pred q;\n\t.reg .u32 k;\n\tadd.cc.u32 %0, %0, %1;\n\taddc.u32 k, 0, 0;\n\tsetp.ne.u32 q, k, 0;\n\t@q mad.lo.u32 %0, %0, %2, 0xFFFFF;\n\t}" : "+r"(a[i]) : "r"(b[i]), "r"(one))
#define OP_I2F     { double t; asm volatile("cvt.rn.f64.u32 %0, %1;" : "=d"(t) : "r"(a[i])); a[i] = lo32(t); }
#define OP_DFMA    asm volatile("fma.rm.f64 %0, %0, %1, %2;" : "+d"(x[i]) : "d"(y[i]), "d"(z[i]))

template <int OP>
__global__ void __launch_bounds__(256) op_kernel(uint32_t* out, int iters, uint32_t one, long long* cyc)
{
    const int NB = 8;
    uint32_t a[NB], b[NB], c[NB], d[NB]; double x[NB], y[NB], z[NB];
#pragma unroll
    for (int i = 0; i < NB; i++) {
        a[i] = out[threadIdx.x + i * 256]; b[i] = out[threadIdx.x + i * 256 + 1] | 1; c[i] = out[threadIdx.x + i * 256 + 2]; d[i] = a[i] ^ c[i];
        x[i] = 1.0 + 1e-9 * a[i]; y[i] = 1.0 - 1e-12 * b[i]; z[i] = 1e-7 * c[i];
    }
    const long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int i = 0; i < NB; i++) {
            if (OP == 0) OP_IADD3;
            if (OP == 1) OP_IMAD;
            if (OP == 2) OP_MNMX;
            if (OP == 3) OP_ADDL_V;
            if (OP == 4) OP_ADDL_M;
            if (OP == 5) OP_I2F;
            if (OP == 6) OP_DFMA;
            if (OP == 7) { OP_IADD3; asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(d[i]) : "r"(b[i]), "r"(c[i])); }
            if (OP == 8) { OP_ADDL_V; asm volatile("{\n\t.reg .u32 t;\n\tsub.u32 t, %0, 0xFFF00001;\n\tmin.u32 %0, %0, t;\n\t}" : "+r"(d[i])); }
            if (OP == 9) { OP_ADDL_M; asm volatile("{\n\t.reg .u32 t;\n\tsub.u32 t, %0, 0xFFF00001;\n\tmin.u32 %0, %0, t;\n\t}" : "+r"(d[i])); }
            if (OP == 10) { OP_MNMX; asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(d[i]) : "r"(b[i]), "r"(c[i])); }
            if (OP == 11) { OP_DFMA; asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(d[i]) : "r"(b[i]), "r"(c[i])); }
            if (OP == 12) { OP_DFMA; OP_I2F; }
            if (OP == 13) { OP_ADDL_V; asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(d[i]) : "r"(b[i]), "r"(c[i])); }
        }
    }
    const long long t1 = clock64();
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < NB; i++) acc ^= a[i] ^ d[i] ^ lo32(x[i]);
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

int main()
{
    cudaDeviceProp pr; cudaGetDeviceProperties(&pr, 0);
    const int sms = pr.multiProcessorCount, iters = 4096;
    printf("dev %s sms %d\n", pr.name, sms);
    uint32_t* out; cudaMalloc(&out, 4 << 20); cudaMemset(out, 0x5a, 4 << 20);
    long long* cyc; cudaMalloc(&cyc, 8 * 4 * sms);
    long long* hc = new long long[4 * sms];
#define RUN(OP, label) { int occ = 0; cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, op_kernel<OP>, 256, 0); if (occ > 4) occ = 4; \
        const int grid = sms * occ; op_kernel<OP><<<grid, 256>>>(out, iters, 1u, cyc); cudaDeviceSynchronize(); long long best = 1ll << 62; \
        for (int r = 0; r < 3; r++) { op_kernel<OP><<<grid, 256>>>(out, iters, 1u, cyc); cudaMemcpy(hc, cyc, 8 * grid, cudaMemcpyDeviceToHost); \
            long long span = 0; for (int k = 0; k < grid; k++) span = hc[k] > span ? hc[k] : span; best = span < best ? span : best; } \
        printf("pipe %-40s %5.2f cycles per op per warp per SMSP  (%d warps per SMSP)\n", label, best / ((double)iters * 8 * 2 * occ), 2 * occ); }
    RUN(0, "add.u32 reg (ptxas: IADD3 / IMAD.IADD mix)");
    RUN(1, "IMAD");
    RUN(2, "VIADDMNMX.U32 (min(v, v-P))");
    RUN(3, "addl: IADD3 + @P VIADD");
    RUN(4, "addl: IADD3 + @P IMAD");
    RUN(5, "I2F.F64.U32");
    RUN(6, "DFMA.RM");
    RUN(7, "add.u32 reg | IMAD");
    RUN(8, "IADD3 + @P VIADD | VIADDMNMX");
    RUN(9, "IADD3 + @P IMAD | VIADDMNMX");
    RUN(10, "VIADDMNMX | IMAD");
    RUN(11, "DFMA.RM | IMAD");
    RUN(12, "DFMA.RM | I2F.F64.U32");
    RUN(13, "IADD3 + @P VIADD | IMAD");
    printf("status %s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
