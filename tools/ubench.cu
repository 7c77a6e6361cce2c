// Micro-benchmarks + primitive self-tests for GF(0xFFF00001) on sm_90a.  Scratch tool (not product).
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cuda_runtime.h>
#define P 0xFFF00001u
#define CC 0x000FFFFFu

__device__ __forceinline__ uint32_t addfix(uint32_t a, uint32_t v){
    uint32_t s;
    asm("{\n\t.reg .pred q;\n\t.reg .u32 c;\n\tadd.cc.u32 %0, %1, %2;\n\taddc.u32 c, 0, 0;\n\tsetp.ne.u32 q, c, 0;\n\t@q add.u32 %0, %0, 0xFFFFF;\n\t}" : "=r"(s) : "r"(a), "r"(v));
    return s;
}
template<int SV> __device__ __forceinline__ uint32_t subfix(uint32_t a, uint32_t v){
    uint32_t s;
    if (SV==0) asm("{\n\t.reg .pred q;\n\t.reg .u32 c;\n\tsub.cc.u32 %0, %1, %2;\n\taddc.u32 c, 0, 0;\n\tsetp.ne.u32 q, c, 0;\n\t@q sub.u32 %0, %0, 0xFFFFF;\n\t}" : "=r"(s) : "r"(a), "r"(v));
    if (SV==1) asm("{\n\t.reg .pred q;\n\t.reg .u32 c;\n\tsub.cc.u32 %0, %1, %2;\n\taddc.u32 c, 0, 0;\n\tsetp.eq.u32 q, c, 0;\n\t@q sub.u32 %0, %0, 0xFFFFF;\n\t}" : "=r"(s) : "r"(a), "r"(v));
    if (SV==2) asm("{\n\t.reg .pred q;\n\t.reg .u32 c;\n\tsub.cc.u32 %0, %1, %2;\n\tsubc.u32 c, 0, 0;\n\tsetp.ne.u32 q, c, 0;\n\t@q sub.u32 %0, %0, 0xFFFFF;\n\t}" : "=r"(s) : "r"(a), "r"(v));
    if (SV==3) { s = a - v; if (a < v) s -= CC; }
    return s;
}
// exact Barrett: w=(w, Whi, Wlo, _) -> v in [0,P], v == b*w mod P
__device__ __forceinline__ uint32_t mul_barrett(uint32_t b, uint32_t w, uint32_t whi, uint32_t wlo, uint32_t z){
    uint32_t t = __umulhi(b, wlo);
    uint64_t c64 = ((uint64_t)z << 32) | t;
    uint64_t Q = (uint64_t)b * whi + c64;
    return (uint32_t)(Q>>32) * CC + b * w;
}
__device__ __forceinline__ uint32_t mul_barrett_c(uint32_t b, uint32_t w, uint32_t whi, uint32_t wlo){
    uint32_t t = __umulhi(b, wlo);
    uint64_t Q = (uint64_t)b * whi + t;
    return (uint32_t)(Q>>32) * CC + b * w;
}
// Montgomery': wm = w*2^32 mod P, wmp = wm * Pinv mod 2^32 (Pinv = 0x00100001) ; canonical
template<int SV> __device__ __forceinline__ uint32_t mul_mont(uint32_t b, uint32_t wm, uint32_t wmp){
    uint32_t m = b * wmp;
    uint64_t Z = (uint64_t)b * wm;
    uint32_t h = (uint32_t)(((uint64_t)m * CC + Z) >> 32);
    return subfix<SV>(h, m);
}

// ---------------- correctness of primitives -----------------
__global__ void selftest(const uint32_t* av, const uint32_t* bv, const uint32_t* wv, const uint32_t* whi, const uint32_t* wlo,
                         const uint32_t* wm, const uint32_t* wmp, int n, unsigned long long* err){
    int i = blockIdx.x*blockDim.x+threadIdx.x; if (i>=n) return;
    uint32_t z; asm volatile("mov.u32 %0, 0;" : "=r"(z));
    uint32_t a=av[i], b=bv[i], w=wv[i];
    uint32_t ref = (uint32_t)(((uint64_t)b * w) % P);
    uint32_t v0 = mul_barrett(b,w,whi[i],wlo[i],z);
    uint32_t v1 = mul_barrett_c(b,w,whi[i],wlo[i]);
    if (!(v0==ref || (ref==0 && v0==P))) atomicAdd(err+0,1ull);
    if (v1!=v0) atomicAdd(err+1,1ull);
    uint32_t m3 = mul_mont<3>(b,wm[i],wmp[i]);
    if (m3!=ref) atomicAdd(err+2,1ull);
    if (mul_mont<0>(b,wm[i],wmp[i])!=ref) atomicAdd(err+3,1ull);
    if (mul_mont<1>(b,wm[i],wmp[i])!=ref) atomicAdd(err+4,1ull);
    if (mul_mont<2>(b,wm[i],wmp[i])!=ref) atomicAdd(err+5,1ull);
    // lazy add/sub: a in [0,2^32), v in [0,P]
    uint32_t v = ref; if ((i&15)==0) v = P; if ((i&15)==1) v = 0;
    uint64_t st = (uint64_t)a + v;  uint32_t sref = (uint32_t)(st >> 32 ? st - P : st);   // stays < 2^32
    int64_t dt = (int64_t)a - v;    uint32_t dref = (uint32_t)(dt < 0 ? dt + P : dt);
    if (addfix(a,v)!=sref) atomicAdd(err+6,1ull);
    if (subfix<0>(a,v)!=dref) atomicAdd(err+7,1ull);
    if (subfix<1>(a,v)!=dref) atomicAdd(err+8,1ull);
    if (subfix<2>(a,v)!=dref) atomicAdd(err+9,1ull);
    if (subfix<3>(a,v)!=dref) atomicAdd(err+10,1ull);
}

// ---------------- butterfly throughput -----------------
template<int VAR>
__global__ void __launch_bounds__(256) bfly_kernel(uint32_t* out, const uint4* __restrict__ tw, int iters, long long* cyc){
    const int NB = 8;
    uint32_t a[NB], b[NB]; uint4 w[NB];
    uint32_t z; asm volatile("mov.u32 %0, 0;" : "=r"(z));
    #pragma unroll
    for (int i=0;i<NB;i++){ a[i]=out[threadIdx.x+i*256]; b[i]=out[threadIdx.x+i*256+2048]; w[i]=tw[(threadIdx.x>>2)+i*64]; }
    long long t0 = clock64();
    for (int it=0; it<iters; it++){
        #pragma unroll
        for (int i=0;i<NB;i++){
            uint32_t v, s, d;
            if (VAR==0){ v = mul_barrett_c(b[i], w[i].x, w[i].y, w[i].z); s=a[i]+v; if (s<a[i]) s+=CC; d=subfix<3>(a[i],v);}
            if (VAR==1){ v = mul_barrett(b[i], w[i].x, w[i].y, w[i].z, z); s=addfix(a[i],v); d=subfix<0>(a[i],v);}
            if (VAR==2){ v = mul_mont<0>(b[i], w[i].x, w[i].y); s=addfix(a[i],v); d=subfix<0>(a[i],v);}
            if (VAR==3){ v = mul_barrett(b[i], w[i].x, w[i].y, w[i].z, z); s=addfix(a[i],v); d=subfix<3>(a[i],v);}
            if (VAR==4){ v = mul_barrett(b[i], w[i].x, w[i].y, w[i].z, z); s=a[i]^v; d=a[i]+v;}   // mul only + 2 cheap ALU
            a[i]=s; b[i]=d;
        }
        uint32_t t=a[0];
        #pragma unroll
        for (int i=0;i<NB-1;i++) a[i]=a[i+1];
        a[NB-1]=t;
    }
    long long t1 = clock64();
    if (threadIdx.x==0 && blockIdx.x==0) *cyc = t1-t0;
    #pragma unroll
    for (int i=0;i<NB;i++){ out[threadIdx.x+i*256]=a[i]; out[threadIdx.x+i*256+2048]=b[i]; }
}
template<int OP>
__global__ void __launch_bounds__(256) op_kernel(uint32_t* out, int iters, long long* cyc){
    const int NB=8;
    uint32_t a[NB], b[NB], c[NB];
    #pragma unroll
    for (int i=0;i<NB;i++){ a[i]=out[threadIdx.x+i*256]; b[i]=out[threadIdx.x+i*256+1]|1; c[i]=out[threadIdx.x+i*256+2];}
    long long t0 = clock64();
    for (int it=0; it<iters; it++){
        #pragma unroll
        for (int i=0;i<NB;i++){
            if (OP==0) asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(b[i]), "r"(c[i]));
            if (OP==1) asm volatile("mad.hi.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(b[i]), "r"(c[i]));
            if (OP==2) { uint64_t t; asm volatile("mad.wide.u32 %0, %1, %2, %3;" : "=l"(t) : "r"(a[i]), "r"(b[i]), "l"(((uint64_t)c[i]<<32)|a[i])); a[i]=(uint32_t)t; c[i]=(uint32_t)(t>>32);}
            if (OP==3) asm volatile("add.u32 %0, %0, %1;\n\t xor.b32 %0, %0, %2;" : "+r"(a[i]) : "r"(b[i]), "r"(c[i]));
            if (OP==4) { asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(b[i]), "r"(c[i])); asm volatile("add.u32 %0, %0, %1;\n\t xor.b32 %0, %0, %2;" : "+r"(c[i]) : "r"(b[i]), "r"(a[i])); }
            if (OP==5) { asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(b[i]), "r"(c[i])); asm volatile("xor.b32 %0, %0, %1;" : "+r"(c[i]) : "r"(b[i])); }
            if (OP==6) { a[i] = addfix(a[i], b[i]); }
            if (OP==7) { asm volatile("mad.hi.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(b[i]), "r"(c[i])); asm volatile("xor.b32 %0, %0, %1;" : "+r"(c[i]) : "r"(b[i])); }
            if (OP==8) { uint64_t t; asm volatile("mad.wide.u32 %0, %1, %2, %3;" : "=l"(t) : "r"(a[i]), "r"(b[i]), "l"(((uint64_t)c[i]<<32)|a[i])); a[i]=(uint32_t)t; c[i]=(uint32_t)(t>>32); asm volatile("xor.b32 %0, %0, %1;" : "+r"(c[i]) : "r"(b[i]));}
        }
    }
    long long t1 = clock64();
    if (threadIdx.x==0 && blockIdx.x==0) *cyc = t1-t0;
    uint32_t acc=0;
    #pragma unroll
    for (int i=0;i<NB;i++) acc ^= a[i]^c[i];
    out[blockIdx.x*blockDim.x+threadIdx.x]=acc;
}
static uint64_t rng=88172645463325252ull; static uint32_t rnd(){ rng^=rng<<13; rng^=rng>>7; rng^=rng<<17; return (uint32_t)(rng>>16);}
int main(){
    cudaDeviceProp pr; cudaGetDeviceProperties(&pr,0);
    int sms=pr.multiProcessorCount;
    printf("dev %s sms %d\n", pr.name, sms);
    // ---- selftest
    { int n=1<<22; uint32_t *h[7]; for(int k=0;k<7;k++) h[k]=(uint32_t*)malloc(n*4);
      for(int i=0;i<n;i++){ uint32_t a=rnd(), b=rnd(), w=rnd()%P;
        if(i%7==0) b = P; if (i%11==0) b=0xFFFFFFFFu; if (i%13==0) b=0; if (i%17==0) w=P-1; if(i%19==0) w=0; if (i%23==0) w=1; if (i%29==0) a=0xFFFFFFFFu; if (i%31==0) a=0;
        if (i%37==0) b=P-1;
        unsigned __int128 W = (((unsigned __int128)w)<<64)/P;
        h[0][i]=a; h[1][i]=b; h[2][i]=w; h[3][i]=(uint32_t)(W>>32); h[4][i]=(uint32_t)W;
        uint32_t wm = (uint32_t)((((uint64_t)w)<<32)%P); h[5][i]=wm; h[6][i]=wm*0x00100001u; }
      uint32_t* d[7]; for(int k=0;k<7;k++){ cudaMalloc(&d[k],n*4); cudaMemcpy(d[k],h[k],n*4,cudaMemcpyHostToDevice);} 
      unsigned long long* derr; cudaMalloc(&derr, 16*8); cudaMemset(derr,0,16*8);
      selftest<<<n/256,256>>>(d[0],d[1],d[2],d[3],d[4],d[5],d[6],n,derr);
      unsigned long long herr[16]; cudaMemcpy(herr,derr,16*8,cudaMemcpyDeviceToHost);
      const char* names[]={"barrett(opaque0)","barrett_c==barrett","mont<sub3>","mont<sub0>","mont<sub1>","mont<sub2>","addfix","subfix0(sub.cc,addc,ne)","subfix1(sub.cc,addc,eq)","subfix2(sub.cc,subc,ne)","subfix3(C)"};
      for(int k=0;k<11;k++) printf("selftest %-28s errors %llu / %d\n", names[k], herr[k], n);
      printf("selftest status %s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    }
    uint32_t* out; cudaMalloc(&out, 1<<20); 
    { uint32_t* h=(uint32_t*)malloc(1<<20); for(int i=0;i<(1<<18);i++) h[i]=rnd(); cudaMemcpy(out,h,1<<20,cudaMemcpyHostToDevice);} 
    uint4* tw; cudaMalloc(&tw, 1<<20); cudaMemcpy(tw,out,1<<20,cudaMemcpyDeviceToDevice);
    long long* cyc; cudaMalloc(&cyc,8);
    const int iters=2048;
    cudaEvent_t e0,e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int bps : {1,2,4}) {
      int grid=sms*bps;
      #define TIME(launch, label, per_iter_units) { launch; cudaDeviceSynchronize(); float best=1e30f; for(int r=0;r<3;r++){cudaEventRecord(e0); launch; cudaEventRecord(e1); cudaEventSynchronize(e1); float ms; cudaEventElapsedTime(&ms,e0,e1); if(ms<best)best=ms;} long long hc; cudaMemcpy(&hc,cyc,8,cudaMemcpyDeviceToHost); \
          double units=(double)iters*8*per_iter_units; \
          printf("%-22s warps/SM %2d: %.3f ms, %lld cyc (=> %.0f MHz), %.2f units/clk/SM, %.2f cyc per warp-unit per SMSP\n", label, bps*8, best, hc, hc/best/1e3, units*256*bps/hc, (double)hc/(units*bps*2)); }
      TIME((bfly_kernel<0><<<grid,256>>>(out,tw,iters,cyc)), "bfly barrettC+C", 1);
      TIME((bfly_kernel<1><<<grid,256>>>(out,tw,iters,cyc)), "bfly barrett+asm(8)", 1);
      TIME((bfly_kernel<2><<<grid,256>>>(out,tw,iters,cyc)), "bfly mont'+asm(9)", 1);
      TIME((bfly_kernel<3><<<grid,256>>>(out,tw,iters,cyc)), "bfly barrett+asm+C", 1);
      TIME((bfly_kernel<4><<<grid,256>>>(out,tw,iters,cyc)), "bfly mulonly(4F+2A)", 1);
      TIME((op_kernel<0><<<grid,256>>>(out,iters,cyc)), "op imad.lo", 1);
      TIME((op_kernel<1><<<grid,256>>>(out,iters,cyc)), "op imad.hi", 1);
      TIME((op_kernel<2><<<grid,256>>>(out,iters,cyc)), "op imad.wide", 1);
      TIME((op_kernel<3><<<grid,256>>>(out,iters,cyc)), "op add+xor (2)", 2);
      TIME((op_kernel<4><<<grid,256>>>(out,iters,cyc)), "op imad+add+xor (3)", 3);
      TIME((op_kernel<5><<<grid,256>>>(out,iters,cyc)), "op imad+xor (2)", 2);
      TIME((op_kernel<6><<<grid,256>>>(out,iters,cyc)), "op addcc+@viadd (2)", 2);
      TIME((op_kernel<7><<<grid,256>>>(out,iters,cyc)), "op imad.hi+xor (2)", 2);
      TIME((op_kernel<8><<<grid,256>>>(out,iters,cyc)), "op imad.wide+xor (2)", 2);
    }
    printf("status %s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
