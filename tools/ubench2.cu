// Micro-benchmark: can the FP64 pipe of the GPU take the quotient of the GF(0xFFF00001) constant product off the integer
// multiplier?  (VERDICT r01 "Next" #2.)  Scratch tool, not product.
//
//   Barrett (production r01):  q = hi32(b*Whi + hi32(b*Wlo))                        2 x IMAD.HI (4.3 cyc each, fmaheavy)
//                              v = b*w + q*(2^32-P)                                 2 x IMAD
//   Hybrid:                    q = lo32( fma.rm( double(b), wp, 2^52 ) ),  wp = RD(w/P)     FP64 pipe
//                              v = b*w + q*(2^32-P)   in [0, P + 2^11]              2 x IMAD
//                              v = min(v, v - P)                                    2 x ALU
//   double(b) is H1: {b, 0x43300000} - 2^52 (MOV + DADD), H3: cvt.rn.f64.u32 (I2F on the XU pipe),
//   H4: no conversion at all: fma.rm({b,0x43300000}, wp, 2^52*(1-wp)) with wp a multiple of 2^-52 (needs 8 more table bytes).
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cmath>
#include <cuda_runtime.h>
#define P 0xFFF00001u
#define CC 0x000FFFFFu

__device__ __forceinline__ uint32_t addfix(uint32_t a, uint32_t v){
    uint32_t s;
    asm("{\n\t.reg .pred q;\n\t.reg .u32 c;\n\tadd.cc.u32 %0, %1, %2;\n\taddc.u32 c, 0, 0;\n\tsetp.ne.u32 q, c, 0;\n\t@q add.u32 %0, %0, 0xFFFFF;\n\t}" : "=r"(s) : "r"(a), "r"(v));
    return s;
}
__device__ __forceinline__ uint32_t subfix(uint32_t a, uint32_t v){
    uint32_t s;
    asm("{\n\t.reg .pred q;\n\t.reg .u32 c;\n\tsub.cc.u32 %0, %1, %2;\n\taddc.u32 c, 0, 0;\n\tsetp.eq.u32 q, c, 0;\n\t@q sub.u32 %0, %0, 0xFFFFF;\n\t}" : "=r"(s) : "r"(a), "r"(v));
    return s;
}
__device__ __forceinline__ uint32_t mul_barrett(uint32_t b, uint32_t w, uint32_t whi, uint32_t wlo, uint32_t z){
    uint32_t t = __umulhi(b, wlo);
    uint64_t c64 = ((uint64_t)z << 32) | t;
    uint64_t Q = (uint64_t)b * whi + c64;
    return (uint32_t)(Q>>32) * CC + b * w;
}
__device__ __forceinline__ uint32_t lo32(double x){ uint32_t lo, hi; asm("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "d"(x)); return lo; }
__device__ __forceinline__ uint32_t fix(uint32_t v){ uint32_t t = v - P; return min(v, t); }
// H1: magic-number conversion
__device__ __forceinline__ uint32_t mul_h1(uint32_t b, uint32_t w, double wp){
    double d, bd, qd;
    asm("mov.b64 %0, {%1, %2};" : "=d"(d) : "r"(b), "r"(0x43300000u));
    asm("sub.rn.f64 %0, %1, 0d4330000000000000;" : "=d"(bd) : "d"(d));
    asm("fma.rm.f64 %0, %1, %2, 0d4330000000000000;" : "=d"(qd) : "d"(bd), "d"(wp));
    return fix(lo32(qd) * CC + b * w);
}
// H3: I2F conversion
__device__ __forceinline__ uint32_t mul_h3(uint32_t b, uint32_t w, double wp){
    double bd, qd;
    asm("cvt.rn.f64.u32 %0, %1;" : "=d"(bd) : "r"(b));
    asm("fma.rm.f64 %0, %1, %2, 0d4330000000000000;" : "=d"(qd) : "d"(bd), "d"(wp));
    return fix(lo32(qd) * CC + b * w);
}
// H4: no conversion; wp4 = floor(w*2^52/P)/2^52, c4 = 2^52*(1 - wp4)
__device__ __forceinline__ uint32_t mul_h4(uint32_t b, uint32_t w, double wp4, double c4){
    double d, qd;
    asm("mov.b64 %0, {%1, %2};" : "=d"(d) : "r"(b), "r"(0x43300000u));
    asm("fma.rm.f64 %0, %1, %2, %3;" : "=d"(qd) : "d"(d), "d"(wp4), "d"(c4));
    return fix(lo32(qd) * CC + b * w);
}
// unfixed variants (v in [0, P+2^11]) to see what the fix costs
__device__ __forceinline__ uint32_t mul_h1_nofix(uint32_t b, uint32_t w, double wp){
    double d, bd, qd;
    asm("mov.b64 %0, {%1, %2};" : "=d"(d) : "r"(b), "r"(0x43300000u));
    asm("sub.rn.f64 %0, %1, 0d4330000000000000;" : "=d"(bd) : "d"(d));
    asm("fma.rm.f64 %0, %1, %2, 0d4330000000000000;" : "=d"(qd) : "d"(bd), "d"(wp));
    return lo32(qd) * CC + b * w;
}

__global__ void selftest(const uint32_t* bv, const uint32_t* wv, const uint32_t* whi, const uint32_t* wlo, const double* wp, const double* wp4, const double* c4,
                         int n, unsigned long long* err, unsigned long long* stat){
    int i = blockIdx.x*blockDim.x+threadIdx.x; if (i>=n) return;
    uint32_t z; asm volatile("mov.u32 %0, 0;" : "=r"(z));
    uint32_t b=bv[i], w=wv[i];
    uint32_t ref = (uint32_t)(((uint64_t)b * w) % P);
    uint32_t v0 = mul_barrett(b,w,whi[i],wlo[i],z);
    if (!(v0==ref || (ref==0 && v0==P))) atomicAdd(err+0,1ull);
    if (mul_h1(b,w,wp[i]) != ref) atomicAdd(err+1,1ull);
    if (mul_h3(b,w,wp[i]) != ref) atomicAdd(err+2,1ull);
    if (mul_h4(b,w,wp4[i],c4[i]) != ref) atomicAdd(err+3,1ull);
    uint32_t u = mul_h1_nofix(b,w,wp[i]);
    if (u >= P) { atomicAdd(stat+0,1ull); if (u - P > 2048u) atomicAdd(err+4,1ull); }     // the rare "one too low" quotient
    if (u != ref && u != ref + P) atomicAdd(err+5,1ull);
}

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
            const double wp = __hiloint2double(w[i].w, w[i].z);
            const double c4 = __hiloint2double(w[i].y, w[i].x);      // (junk operands: timing only)
            if (VAR==0){ v = mul_barrett(b[i], w[i].x, w[i].y, w[i].z, z); }
            if (VAR==1){ v = mul_h1(b[i], w[i].x, wp); }
            if (VAR==2){ v = mul_h3(b[i], w[i].x, wp); }
            if (VAR==3){ v = mul_h4(b[i], w[i].x, wp, c4); }
            if (VAR==4){ v = (i & 1) ? mul_h1(b[i], w[i].x, wp) : mul_barrett(b[i], w[i].x, w[i].y, w[i].z, z); }     // half / half
            if (VAR==5){ v = (i & 1) ? mul_h3(b[i], w[i].x, wp) : mul_barrett(b[i], w[i].x, w[i].y, w[i].z, z); }
            if (VAR==6){ v = (i & 3) ? mul_h1(b[i], w[i].x, wp) : mul_barrett(b[i], w[i].x, w[i].y, w[i].z, z); }     // 3/4 hybrid
            if (VAR==7){ v = (i & 1) ? mul_h3(b[i], w[i].x, wp) : mul_h1(b[i], w[i].x, wp); }                         // spread the conversions over XU and FP64
            if (VAR==8){ v = mul_h1_nofix(b[i], w[i].x, wp); }
            if (VAR==9){ v = (i & 3) == 0 ? mul_barrett(b[i], w[i].x, w[i].y, w[i].z, z) : (i & 1) ? mul_h3(b[i], w[i].x, wp) : mul_h1(b[i], w[i].x, wp); }
            s=addfix(a[i],v); d=subfix(a[i],v);
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
    double x[NB], y[NB], zz[NB]; uint32_t a[NB], b[NB], c[NB];
    #pragma unroll
    for (int i=0;i<NB;i++){ a[i]=out[threadIdx.x+i*256]; b[i]=out[threadIdx.x+i*256+1]|1; c[i]=out[threadIdx.x+i*256+2];
        x[i] = 1.0 + 1e-9 * a[i]; y[i] = 1.0 - 1e-12 * b[i]; zz[i] = 1e-7 * c[i]; }
    long long t0 = clock64();
    for (int it=0; it<iters; it++){
        #pragma unroll
        for (int i=0;i<NB;i++){
            if (OP==0) asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(x[i]) : "d"(y[i]), "d"(zz[i]));
            if (OP==1) asm volatile("add.rn.f64 %0, %0, %1;" : "+d"(x[i]) : "d"(zz[i]));
            if (OP==2) asm volatile("mul.rn.f64 %0, %0, %1;" : "+d"(x[i]) : "d"(y[i]));
            if (OP==3) { double t; asm volatile("cvt.rn.f64.u32 %0, %1;" : "=d"(t) : "r"(a[i])); a[i] ^= lo32(t); }                 // I2F + 1 ALU
            if (OP==4) { asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(x[i]) : "d"(y[i]), "d"(zz[i])); asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(b[i]), "r"(c[i])); }
            if (OP==5) { asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(x[i]) : "d"(y[i]), "d"(zz[i])); asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(b[i]), "r"(c[i])); asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(c[i]) : "r"(b[i]), "r"(a[i])); }
            if (OP==6) { asm volatile("fma.rm.f64 %0, %0, %1, %2;" : "+d"(x[i]) : "d"(y[i]), "d"(zz[i])); }
            if (OP==7) { asm volatile("fma.rn.f64 %0, %0, %1, %2;" : "+d"(x[i]) : "d"(y[i]), "d"(zz[i])); asm volatile("add.rn.f64 %0, %0, %1;" : "+d"(zz[i]) : "d"(y[i]));
                         asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(b[i]), "r"(c[i])); asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(c[i]) : "r"(b[i]), "r"(a[i])); }   // 2 FP64 + 2 IMAD
            if (OP==8) { asm volatile("mad.lo.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(b[i]), "r"(c[i])); }
            if (OP==9) { asm volatile("mad.hi.u32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(b[i]), "r"(c[i])); }
        }
    }
    long long t1 = clock64();
    if (threadIdx.x==0 && blockIdx.x==0) *cyc = t1-t0;
    uint32_t acc=0;
    #pragma unroll
    for (int i=0;i<NB;i++) acc ^= a[i]^c[i]^lo32(x[i])^lo32(zz[i]);
    out[blockIdx.x*blockDim.x+threadIdx.x]=acc;
}
static uint64_t rng=88172645463325252ull; static uint32_t rnd(){ rng^=rng<<13; rng^=rng>>7; rng^=rng<<17; return (uint32_t)(rng>>16);}
static uint32_t mulmod(uint32_t a, uint32_t b){ return (uint32_t)(((uint64_t)a*b)%P); }
static uint32_t powmod(uint32_t x, uint64_t n){ uint32_t r=1; for(;n;n>>=1){ if(n&1) r=mulmod(r,x); x=mulmod(x,x);} return r; }
int main(){
    cudaDeviceProp pr; cudaGetDeviceProperties(&pr,0);
    int sms=pr.multiProcessorCount;
    printf("dev %s sms %d\n", pr.name, sms);
    { int n=1<<22; uint32_t *h[4]; for(int k=0;k<4;k++) h[k]=(uint32_t*)malloc(n*4);
      double *hd[3]; for(int k=0;k<3;k++) hd[k]=(double*)malloc(n*8);
      for(int i=0;i<n;i++){ uint32_t b=rnd(), w=rnd()%P;
        if (i%17==0) w=P-1; if(i%19==0) w=0; if (i%23==0) w=1;
        if(i%7==0) b = P; if (i%11==0) b=0xFFFFFFFFu; if (i%13==0) b=0; if (i%37==0) b=P-1;
        if (i%3==0 && w) { uint32_t r = rnd() % 5000; b = mulmod(r, powmod(w, P-2)); if (i%6==0 && (uint64_t)b + P <= 0xFFFFFFFFull) b += P; }   // adversarial: b*w mod P tiny
        unsigned __int128 W128 = (((unsigned __int128)w)<<64)/P; uint64_t W=(uint64_t)W128;
        h[0][i]=b; h[1][i]=w; h[2][i]=(uint32_t)(W>>32); h[3][i]=(uint32_t)W;
        uint64_t Wt = W; if (Wt) { int lz=__builtin_clzll(Wt); int sh=11-lz; if (sh>0) Wt &= ~((1ull<<sh)-1); }
        hd[0][i] = ldexp((double)Wt, -64);
        uint64_t n52 = W >> 12; hd[1][i] = ldexp((double)n52, -52); hd[2][i] = (double)((1ull<<52) - n52); }
      uint32_t* d[4]; for(int k=0;k<4;k++){ cudaMalloc(&d[k],n*4); cudaMemcpy(d[k],h[k],n*4,cudaMemcpyHostToDevice);}
      double* dd[3]; for(int k=0;k<3;k++){ cudaMalloc(&dd[k],n*8); cudaMemcpy(dd[k],hd[k],n*8,cudaMemcpyHostToDevice);}
      unsigned long long* derr; cudaMalloc(&derr, 32*8); cudaMemset(derr,0,32*8);
      selftest<<<n/256,256>>>(d[0],d[1],d[2],d[3],dd[0],dd[1],dd[2],n,derr,derr+16);
      unsigned long long herr[32]; cudaMemcpy(herr,derr,32*8,cudaMemcpyDeviceToHost);
      const char* names[]={"barrett","h1 (mov+dadd+dfma.rm)","h3 (i2f+dfma.rm)","h4 (dfma.rm, c-table)","h1 nofix: excess > 2048","h1 nofix: not ref / ref+P"};
      for(int k=0;k<6;k++) printf("selftest %-28s errors %llu / %d\n", names[k], herr[k], n);
      printf("selftest quotient one too low (v >= P before the fix): %llu / %d\n", herr[16], n);
      printf("selftest status %s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    }
    uint32_t* out; cudaMalloc(&out, 1<<20);
    { uint32_t* h=(uint32_t*)malloc(1<<20); for(int i=0;i<(1<<18);i++) h[i]=rnd(); cudaMemcpy(out,h,1<<20,cudaMemcpyHostToDevice);}
    uint4* tw; cudaMalloc(&tw, 1<<20);
    { uint32_t* h=(uint32_t*)malloc(1<<20); for(int i=0;i<(1<<18);i+=4){ h[i]=rnd(); h[i+1]=rnd(); double wp = (rnd() % P) / (double)P; memcpy(&h[i+2], &wp, 8);} cudaMemcpy(tw,h,1<<20,cudaMemcpyHostToDevice);}
    long long* cyc; cudaMalloc(&cyc,8);
    const int iters=2048;
    cudaEvent_t e0,e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int bps : {2,4}) {
      int grid=sms*bps;
      #define TIME(launch, label, per_iter_units) { launch; cudaDeviceSynchronize(); float best=1e30f; for(int r=0;r<3;r++){cudaEventRecord(e0); launch; cudaEventRecord(e1); cudaEventSynchronize(e1); float ms; cudaEventElapsedTime(&ms,e0,e1); if(ms<best)best=ms;} \
          double units=(double)iters*8*per_iter_units; \
          printf("%-34s warps/SM %2d: %.3f ms => %.2f cyc per warp-unit per SMSP @1.965GHz\n", label, bps*8, best, best*1e-3*1.965e9/(units*bps*2)); }
      TIME((bfly_kernel<0><<<grid,256>>>(out,tw,iters,cyc)), "bfly barrett (r01)", 1);
      TIME((bfly_kernel<1><<<grid,256>>>(out,tw,iters,cyc)), "bfly h1 mov+dadd+dfma", 1);
      TIME((bfly_kernel<2><<<grid,256>>>(out,tw,iters,cyc)), "bfly h3 i2f+dfma", 1);
      TIME((bfly_kernel<3><<<grid,256>>>(out,tw,iters,cyc)), "bfly h4 dfma(c-table)", 1);
      TIME((bfly_kernel<4><<<grid,256>>>(out,tw,iters,cyc)), "bfly 1/2 barrett 1/2 h1", 1);
      TIME((bfly_kernel<5><<<grid,256>>>(out,tw,iters,cyc)), "bfly 1/2 barrett 1/2 h3", 1);
      TIME((bfly_kernel<6><<<grid,256>>>(out,tw,iters,cyc)), "bfly 1/4 barrett 3/4 h1", 1);
      TIME((bfly_kernel<7><<<grid,256>>>(out,tw,iters,cyc)), "bfly 1/2 h1 1/2 h3", 1);
      TIME((bfly_kernel<8><<<grid,256>>>(out,tw,iters,cyc)), "bfly h1 without fix (invalid)", 1);
      TIME((bfly_kernel<9><<<grid,256>>>(out,tw,iters,cyc)), "bfly 1/4 barrett 3/8 h1 3/8 h3", 1);
      TIME((op_kernel<0><<<grid,256>>>(out,iters,cyc)), "op dfma", 1);
      TIME((op_kernel<6><<<grid,256>>>(out,iters,cyc)), "op dfma.rm", 1);
      TIME((op_kernel<1><<<grid,256>>>(out,iters,cyc)), "op dadd", 1);
      TIME((op_kernel<2><<<grid,256>>>(out,iters,cyc)), "op dmul", 1);
      TIME((op_kernel<3><<<grid,256>>>(out,iters,cyc)), "op i2f.f64.u32 + xor", 1);
      TIME((op_kernel<8><<<grid,256>>>(out,iters,cyc)), "op imad.lo", 1);
      TIME((op_kernel<9><<<grid,256>>>(out,iters,cyc)), "op imad.hi", 1);
      TIME((op_kernel<4><<<grid,256>>>(out,iters,cyc)), "op dfma + imad (per pair)", 1);
      TIME((op_kernel<5><<<grid,256>>>(out,iters,cyc)), "op dfma + 2 imad (per triple)", 1);
      TIME((op_kernel<7><<<grid,256>>>(out,iters,cyc)), "op dfma+dadd+2 imad (per quad)", 1);
    }
    printf("status %s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
