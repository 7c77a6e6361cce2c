// GF(0xFFF00001) arithmetic for the sm_90a NTT kernels (and a bit-identical host restatement used by the
// CPU emulation of the kernels and by the twiddle-table generator).
//
// Replaces, on the device, GF_Add / GF_Sub / GF_Mul of the reference (GF(p).cpp:37-48, 110-127).  The reference's
// 32-bit Barrett (GF_Mul32) needs a 64-bit conditional subtract per product; here every twiddle w is a constant
// known on the host, so we use an exact Barrett/Shoup product with a precomputed 64-bit quotient
//      W = floor(w * 2^64 / P) = (Whi:Wlo)
//      q = floor(b * W / 2^64) = hi32( b*Whi + hi32(b*Wlo) )            (2 x IMAD.HI)
//      v = lo32(b*w) - lo32(q*P) = b*w + q*(2^32-P)   (mod 2^32)         (2 x IMAD)
// q equals floor(b*w/P) exactly unless b*w is a multiple of P, in which case it may be one less; so
//      v == b*w mod P   with v in [0, P]          for ANY 32-bit b  (b need not be reduced).
// No conditional subtract.  That form (mul) serves the element-wise kernels and the small-order DFT.  The pass kernels use
// mul_h, which takes the quotient from the FP64 unit instead of two IMAD.HI (see below and DESIGN.md section 4).
// Values between butterflies are kept "lazy" in [0, 2^32) (congruent mod P):
//      addl(a, v):  a in [0,2^32), v in [0,P]  ->  a+v mod P  in [0,2^32)     (add, then +(2^32-P) on carry)
//      subl(a, v):  a in [0,2^32), v in [0,P]  ->  a-v mod P  in [0,2^32)     (sub, then -(2^32-P) on borrow)
// which are closed (proof in DESIGN.md section 4); canon() maps a lazy value to the canonical residue [0,P).
// The carry idioms below compile to IADD3 Rd,Pc + @Pc VIADD (2 SASS instructions); tools/ubench.cu self-tests them
// against 64-bit arithmetic on the GPU ("selftest" lines).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define GF_HD __host__ __device__ __forceinline__
#else
#define GF_HD inline
#endif

namespace gf {

constexpr uint32_t P  = 0xFFF00001u;
constexpr uint32_t C  = 0x000FFFFFu;          // 2^32 - P
constexpr uint32_t GEN = 19;                  // generator used by GF_Root (GF(p).cpp:272)
constexpr uint32_t LOG_M = 20;                // largest power-of-two order: P-1 = 2^20 * 4095
constexpr uint32_t M = 1u << LOG_M;

struct Tw { uint32_t w, whi, wlo, pad; };     // one entry of the global power table: w and W = floor(w*2^64/P); 16 bytes

// `zero` must be a register holding 0 that the compiler cannot constant-fold (see opaque_zero()): it becomes the
// high half of the 64-bit addend of the second IMAD.HI, which saves ptxas from re-materialising a zero register
// next to `t` for every product (one extra FMA-pipe instruction per butterfly otherwise).
GF_HD uint32_t mul(uint32_t b, uint32_t w, uint32_t whi, uint32_t wlo, uint32_t zero = 0)
{
#if defined(__CUDA_ARCH__)
    uint32_t t = __umulhi(b, wlo);
    uint64_t addend = ((uint64_t)zero << 32) | t;
    uint32_t q = (uint32_t)(((uint64_t)b * whi + addend) >> 32);
#else
    (void)zero;
    uint32_t t = (uint32_t)(((uint64_t)b * wlo) >> 32);
    uint32_t q = (uint32_t)(((uint64_t)b * whi + t) >> 32);
#endif
    return q * C + b * w;
}

// ---- the product of the pass kernels: quotient on the FP64 unit ----------------------------------------------------
// IMAD.HI issues at a fraction of the IMAD rate (tools/ubench2.cu measures both), so the two IMAD.HI of mul() dominate
// its multiplier time.  mul_h gets the quotient from one DFMA instead:
//      wp = RD53(W * 2^-64) <= w/P                          (53-bit truncation of the same W; stage tables hold it)
//      q  = lo32( fma.rm( double(b), wp, 2^52 ) ) = floor(b * wp)         exactly: one rounding, towards -inf, at ulp 1
//      v  = b*w + q*(2^32-P)  (mod 2^32)                                   2 x IMAD
// 0 <= b*(w/P - wp) < 2^32 * (2^-53 + 2^-64), so q is floor(b*w/P) or, only when (b*w mod P) <= 2^11, one less:
// v = b*w - q*P lies in [0, P + 2^11] and fits 32 bits; one VIADDMNMX (min(v, v-P) unsigned) brings it into [0, P).
// double(b) is an exact I2F.F64.U32.  Valid for ANY 32-bit b, like mul().  tools/ubench2.cu checks it on the GPU against
// 64-bit arithmetic, adversarial operands with small b*w mod P included; the CPU restatement below is tested bit for bit.
//
// wp_bits: the IEEE-754 encoding {lo, hi} of wp, built with integer operations only so that host and device agree.
GF_HD uint32_t clz64(uint64_t x)
{
#if defined(__CUDA_ARCH__)
    return (uint32_t)__clzll((long long)x);
#else
    return (uint32_t)__builtin_clzll(x);
#endif
}
GF_HD void wp_bits(uint32_t whi, uint32_t wlo, uint32_t& lo, uint32_t& hi)
{
    const uint64_t W = ((uint64_t)whi << 32) | wlo;
    if (!W) { lo = 0; hi = 0; return; }
    const uint32_t lz = clz64(W);
    const uint64_t m = W << lz;                                   // bit 63 set:  W*2^-64 = (m / 2^63) * 2^(-1-lz)
    const uint64_t bits = ((uint64_t)(1022u - lz) << 52) | ((m >> 11) & ((1ull << 52) - 1));      // truncation = round down
    lo = (uint32_t)bits; hi = (uint32_t)(bits >> 32);
}
#if defined(FECC_CVT_MAGIC)
#define FECC_CVT_DEFAULT 1
#else
#define FECC_CVT_DEFAULT 0
#endif
template <int CVT = FECC_CVT_DEFAULT>     // 0: I2F.F64.U32 (XU pipe); 1 (experiment): {b, 0x43300000} - 2^52 on the FP64 unit
GF_HD uint32_t mul_h(uint32_t b, uint32_t w, uint32_t wplo, uint32_t wphi)
{
    uint32_t q;
#if defined(__CUDA_ARCH__)
    double bd, qd;
    const double wp = __hiloint2double((int)wphi, (int)wplo);
    if (CVT == 1) asm("{\n\t.reg .f64 t;\n\tmov.b64 t, {%1, %2};\n\tsub.rn.f64 %0, t, 0d4330000000000000;\n\t}" : "=d"(bd) : "r"(b), "r"(0x43300000u));
    else          asm("cvt.rn.f64.u32 %0, %1;" : "=d"(bd) : "r"(b));
    asm("fma.rm.f64 %0, %1, %2, 0d4330000000000000;" : "=d"(qd) : "d"(bd), "d"(wp));
    q = (uint32_t)__double2loint(qd);
#else
    q = 0;                                                        // floor(b * wp) in integers: wp = mant * 2^(e-52)
    const uint64_t bits = ((uint64_t)wphi << 32) | wplo;
    if (bits) {
        const uint64_t mant = (bits & ((1ull << 52) - 1)) | (1ull << 52);
        const int sh = 52 - ((int)(bits >> 52) - 1023);           // >= 53 because wp < 1
        if (sh < 128) q = (uint32_t)(((unsigned __int128)b * mant) >> sh);
    }
#endif
    const uint32_t v = q * C + b * w, t = v - P;
    return v < t ? v : t;
}

GF_HD uint32_t addl(uint32_t a, uint32_t v)
{
#if defined(__CUDA_ARCH__)
    uint32_t s;
    asm("{\n\t.reg .pred q;\n\t.reg .u32 c;\n\tadd.cc.u32 %0, %1, %2;\n\taddc.u32 c, 0, 0;\n\tsetp.ne.u32 q, c, 0;\n\t@q add.u32 %0, %0, 0xFFFFF;\n\t}"
        : "=r"(s) : "r"(a), "r"(v));
    return s;
#else
    uint32_t s = a + v; return s < a ? s + C : s;
#endif
}

GF_HD uint32_t subl(uint32_t a, uint32_t v)
{
#if defined(__CUDA_ARCH__)
    // sub.cc leaves CF = NOT borrow for a following addc (the "subfix1" line of the tools/ubench.cu self-test);
    // so "c == 0" means a borrow happened.
    uint32_t s;
    asm("{\n\t.reg .pred q;\n\t.reg .u32 c;\n\tsub.cc.u32 %0, %1, %2;\n\taddc.u32 c, 0, 0;\n\tsetp.eq.u32 q, c, 0;\n\t@q sub.u32 %0, %0, 0xFFFFF;\n\t}"
        : "=r"(s) : "r"(a), "r"(v));
    return s;
#else
    uint32_t s = a - v; return a < v ? s - C : s;
#endif
}

GF_HD uint32_t opaque_zero()
{
#if defined(__CUDA_ARCH__)
    uint32_t z; asm volatile("mov.u32 %0, 0;" : "=r"(z)); return z;
#else
    return 0;
#endif
}

GF_HD uint32_t canon(uint32_t x) { return x >= P ? x - P : x; }

// x mod P without a division: 2^32 = 2^20 - 1 mod P, so fold the high word down until none is left (the 64-bit sums of the
// scrub's fold and of the degraded read).
GF_HD uint32_t reduce64(uint64_t x)
{
    while (x >> 32) x = (x >> 32) * C + (x & 0xFFFFFFFFull);
    return canon((uint32_t)x);
}

// a + b and a - b of canonical residues
GF_HD uint32_t add(uint32_t a, uint32_t b) { const uint32_t s = a + b; return (s < a || s >= P) ? s - P : s; }
GF_HD uint32_t sub(uint32_t a, uint32_t b) { return a >= b ? a - b : a + (P - b); }

#if defined(__CUDACC__)
// The product by a triple t = {w, Whi, Wlo} (a power-table entry or a per-row constant as a uint4, whose .w is unused; a kernel
// constant as a uint32_t[3]), canonical; and the four-lane forms: mul4 leaves each lane in [0, P] like mul(), canon4 reduces.
GF_HD uint32_t mulc(uint32_t b, uint4 t, uint32_t zero = 0) { return canon(mul(b, t.x, t.y, t.z, zero)); }
GF_HD uint32_t mulc(uint32_t b, const uint32_t (&t)[3], uint32_t zero = 0) { return canon(mul(b, t[0], t[1], t[2], zero)); }
GF_HD uint4 mul4(uint4 v, uint4 t, uint32_t zero = 0)
{
    return make_uint4(mul(v.x, t.x, t.y, t.z, zero), mul(v.y, t.x, t.y, t.z, zero), mul(v.z, t.x, t.y, t.z, zero), mul(v.w, t.x, t.y, t.z, zero));
}
GF_HD uint4 canon4(uint4 v) { return make_uint4(canon(v.x), canon(v.y), canon(v.z), canon(v.w)); }
#endif

// ---- products by arbitrary operands (tables, plan constants, the pattern builds of the erasure code) ----------------
GF_HD uint32_t mulmod(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) % P); }
GF_HD uint32_t powmod(uint32_t x, uint64_t n) { uint32_t r = 1; for (; n; n >>= 1) { if (n & 1) r = mulmod(r, x); x = mulmod(x, x); } return r; }
inline uint32_t root(uint32_t n) { return powmod(GEN, (P - 1) / n); }        // GF_Root, GF(p).cpp:267-276
GF_HD uint32_t inv(uint32_t x)  { return powmod(x, P - 2); }                 // GF_Inv,  GF(p).cpp:293-297
GF_HD Tw make_tw(uint32_t w)             // {w, floor(w*2^64/P)} by two 64/32 long-division steps
{
    const uint64_t n1 = (uint64_t)w << 32;
    const uint64_t whi = n1 / P, rem = n1 % P;
    const uint64_t wlo = (rem << 32) / P;
    Tw t; t.w = w; t.whi = (uint32_t)whi; t.wlo = (uint32_t)wlo; t.pad = 0; return t;
}

} // namespace gf
