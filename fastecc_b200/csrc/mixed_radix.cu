// Orders N = 3 * 2^k and 9 * 2^k (P - 1 = 2^20 * 3^2 * 5 * 7 * 13), so that block counts need not be rounded up to a power of
// two (SURVEY 8f rank 4 tail; the reference has the order-3 / order-9 codelets NTT3, NTT9 -- ntt.cpp:26-46, 114-146 -- and their
// composition with the power-of-two transforms on its roadmap, README.md:176).  Cooley-Tukey with N = r * M, r in {3, 9}, M = 2^k,
// input index n = n1 + r*n2, output index k = k2 + M*k1:
//     X[k2 + M*k1] = sum_{n1 < r}  w_r^(n1*k1)  *  [ w_N^(n1*k2) * Y_n1[k2] ],      Y_n1 = M-point NTT of x[n1 + r*n2] over n2
// with w_N = GF_Root(N), w_N^r = GF_Root(M) (the root of the power-of-two kernels) and w_N^M = GF_Root(r).  Step 1 -- the r
// transforms Y_n1 -- is the hot-path NTT run on every r-th row (same buffer, row pitch r times larger: api.cu).  Step 2 is this
// kernel: for every k2, read the r ADJACENT rows r*k2 + n1, multiply by the twiddles, do the order-r transform and write the r
// results to rows k2 + M*k1 of the destination (natural order; out of place).  HBM-bound: one read and one write of the array.
// The twiddle w_N^e is split by the CRT into (a root of order r) * (a root of order M): e = n1*k2,
//     w_N^e = GF_Root(r)^(a*e mod r) * GF_Root(M)^(b*e mod M),     a = M^-1 mod r,  b = r^-1 mod M,
// so it comes from a 9-entry constant table and the 2^20-entry power table the other kernels use.
// radix_encode_kernel (below) is the middle step of the Reed-Solomon encode of N = r * M data blocks, in place (DESIGN 3e).
#include "mixed_radix.h"
#include "context.h"
#include "gf.cuh"

namespace fecc {

struct RadixConsts {
    uint32_t zeta[9][3];       // GF_Root(r)^j (direction applied): {w, Whi, Wlo}
    uint32_t c1[3], c2[3];     // order-3 codelet: (X + X^2)/2, (X - X^2)/2 with X = GF_Root(3) (direction applied)
};

// order-3 transform of canonical residues (the arithmetic of the reference's NTT3 codelet, ntt.cpp:26-46)
__device__ __forceinline__ void dft3(uint32_t& f0, uint32_t& f1, uint32_t& f2, const RadixConsts& C)
{
    const uint32_t s = gf::add(f1, f2), d = gf::sub(f1, f2);
    const uint32_t u = gf::add(f0, gf::mulc(s, C.c1)), v = gf::mulc(d, C.c2);
    f0 = gf::add(f0, s); f1 = gf::add(u, v); f2 = gf::sub(u, v);
}

// order-R transform of canonical residues in place, outputs in natural order: the order-3 codelet, or the 3 x 3 four-step of the
// reference's NTT9 (ntt.cpp:114-146) whose transposed output is renamed back (free: registers)
template <int R>
__device__ __forceinline__ void dft_r(uint32_t (&f)[R], const RadixConsts& C)
{
    if constexpr (R == 3) {
        dft3(f[0], f[1], f[2], C);
    } else {
        dft3(f[0], f[3], f[6], C); dft3(f[1], f[4], f[7], C); dft3(f[2], f[5], f[8], C);
        f[4] = gf::mulc(f[4], C.zeta[1]); f[5] = gf::mulc(f[5], C.zeta[2]); f[7] = gf::mulc(f[7], C.zeta[2]); f[8] = gf::mulc(f[8], C.zeta[4]);
        dft3(f[0], f[1], f[2], C); dft3(f[3], f[4], f[5], C); dft3(f[6], f[7], f[8], C);
        uint32_t g[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) g[k] = f[(k % 3) * 3 + k / 3];
#pragma unroll
        for (int k = 0; k < 9; ++k) f[k] = g[k];
    }
}

template <int R>
__global__ void __launch_bounds__(256) radix_pass_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, uint32_t pitch4, uint32_t s4, uint32_t M, uint32_t log_m,
                                                         uint32_t a_inv, uint32_t b_inv, int inverse, RadixConsts C, const uint4* __restrict__ tw)
{
    const size_t total = (size_t)M * s4;
    FOR_GRID(size_t, i, total) {
        const uint32_t k2 = (uint32_t)(i / s4), c = (uint32_t)(i - (size_t)k2 * s4);
        uint32_t f[4][R];
#pragma unroll
        for (int n1 = 0; n1 < R; ++n1) {
            const uint4 v = src[((size_t)R * k2 + n1) * pitch4 + c];
            f[0][n1] = v.x; f[1][n1] = v.y; f[2][n1] = v.z; f[3][n1] = v.w;
            const unsigned long long e = (unsigned long long)n1 * k2;
            const uint32_t er = (uint32_t)((a_inv * (e % R)) % R); uint32_t em = (uint32_t)(((unsigned long long)b_inv * (e & (M - 1))) & (M - 1));
            if (inverse) em = (M - em) & (M - 1);                               // the power table is forward; C.zeta already has the direction
            const uint4 t = tw[(size_t)em << (20 - log_m)];                    // GF_Root(M)^(+-em)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                uint32_t x = gf::mulc(f[j][n1], t);      // inputs are taken mod P
                f[j][n1] = er ? gf::mulc(x, C.zeta[er]) : x;
            }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) dft_r<R>(f[j], C);
#pragma unroll
        for (int k1 = 0; k1 < R; ++k1)
            dst[((size_t)k2 + (size_t)M * k1) * pitch4 + c] = make_uint4(f[0][k1], f[1][k1], f[2][k1], f[3][k1]);
    }
}

static void fill3(uint32_t (&t)[3], uint32_t w) { const gf::Tw x = gf::make_tw(w); t[0] = x.w; t[1] = x.whi; t[2] = x.wlo; }

static void fill_codelets(RadixConsts& C, uint32_t r, bool inverse)
{
    uint32_t zr = gf::powmod(gf::GEN, (gf::P - 1) / r);                        // GF_Root(r), GF(p).cpp:267-276
    uint32_t z3 = gf::powmod(gf::GEN, (gf::P - 1) / 3);
    if (inverse) { zr = gf::inv(zr); z3 = gf::inv(z3); }
    for (uint32_t j = 0; j < 9; ++j) fill3(C.zeta[j], gf::powmod(zr, j));
    const uint32_t inv2 = (gf::P + 1) / 2, x1 = z3, x2 = gf::mulmod(z3, z3);
    fill3(C.c1, gf::mulmod((uint32_t)(((uint64_t)x1 + x2) % gf::P), inv2));
    fill3(C.c2, gf::mulmod((uint32_t)(((uint64_t)x1 + gf::P - x2) % gf::P), inv2));
}

// The launchers take what api.cu has validated: r in {3, 9} (s | r for the fold), M a power of two.
cudaError_t launch_radix_pass(const uint32_t* src, uint32_t* dst, uint32_t pitch4, uint32_t s4, uint32_t r, uint32_t M, bool inverse, const uint4* tw, int num_sms, cudaStream_t st)
{
    auto kernel = r == 3 ? radix_pass_kernel<3> : r == 9 ? radix_pass_kernel<9> : nullptr;
    if (!kernel || !M || (M & (M - 1)) || M > gf::M) return cudaErrorInvalidValue;
    uint32_t log_m = 0; while ((1u << log_m) < M) ++log_m;
    RadixConsts C;
    fill_codelets(C, r, inverse);
    const CrtSplit ab = crt_split(r, log_m);                                   // a = M^-1 mod r, b = r^-1 mod M
    kernel<<<grid_size((size_t)M * s4, (size_t)num_sms * 16), 256, 0, st>>>(reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst), pitch4, s4, M, log_m, ab.a, ab.b,
                                                             inverse ? 1 : 0, C, tw);
    return cudaGetLastError();
}

// ---- step 2 of the Reed-Solomon encode of N = r * M data blocks (DESIGN 3e) --------------------------------------------------
// Parity j = f(rho^(2j+1)), rho = GF_Root(2N), f(w^i) = data block i, w = rho^2 (RS.cpp:41-63 with these roots).  Step 1 (api.cu):
// r unnormalised inverse M-point transforms over rows n1 + r*n2 leave Y_n1[k2] in row n1 + r*k2.  This kernel, for every k2, in
// place on the r ADJACENT rows r*k2 + n1:
//     u[n1] = Y_n1[k2] * rho^(k2*(1 - 2*n1)) / N              (w^(-n1*k2) of the inverse transform and rho^k2 / N of the scaling)
//     a     = inverse order-r transform of u,   a[k1] *= sigma^k1,   sigma = rho^M = GF_Root(2r)     (rho^(M*k1) of the scaling)
//     v     = forward order-r transform of a,   v[j1] *= rho^(2*k2*j1)                                 (w^(k2*j1) of the forward one)
// and v[j1] goes back to row r*k2 + j1.  Step 3: r forward M-point transforms over rows j1 + r*k2 put parity j1 + r*j2 in row
// j1 + r*j2.  rho^e is split by the CRT as GF_Root(r)^(a2*e mod r) * GF_Root(2M)^(b2*e mod 2M), a2 = (2M)^-1 mod r,
// b2 = r^-1 mod 2M (2M <= 2^20: a power-table entry).  Inputs are taken mod P (M = 1: the caller's raw words); outputs canonical.
struct EncodeConsts {
    RadixConsts inv, fwd;      // order-r codelets of both directions (fwd.zeta = GF_Root(r)^j)
    uint32_t zin[9][3];        // GF_Root(r)^j / N
    uint32_t sigma[9][3];      // GF_Root(2r)^k
};

template <int R>
__device__ __forceinline__ void encode_codelets(const uint4* row, uint32_t pitch4, uint32_t k2, uint32_t mask, uint32_t sh, uint32_t a2, uint32_t b2,
                                                const EncodeConsts& C, const uint4* __restrict__ tw, uint32_t (&f)[4][R])
{
    const uint32_t k2r = k2 % R;
#pragma unroll
    for (int n1 = 0; n1 < R; ++n1) {
        const uint4 v = row[(size_t)n1 * pitch4];
        const uint32_t cr = (uint32_t)(((1 - 2 * n1) % R + R) % R);
        const uint32_t er = (a2 * ((k2r * cr) % R)) % R, em = (b2 * (k2 * (uint32_t)(1 - 2 * n1))) & mask;
        const uint4 t = tw[(size_t)em << sh];
        f[0][n1] = gf::mulc(gf::mulc(v.x, t), C.zin[er]);
        f[1][n1] = gf::mulc(gf::mulc(v.y, t), C.zin[er]);
        f[2][n1] = gf::mulc(gf::mulc(v.z, t), C.zin[er]);
        f[3][n1] = gf::mulc(gf::mulc(v.w, t), C.zin[er]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        dft_r<R>(f[j], C.inv);
#pragma unroll
        for (int k1 = 1; k1 < R; ++k1) f[j][k1] = gf::mulc(f[j][k1], C.sigma[k1]);
        dft_r<R>(f[j], C.fwd);
    }
}

template <int R>
__global__ void __launch_bounds__(256) radix_encode_kernel(uint4* __restrict__ x, uint32_t pitch4, uint32_t s4, uint32_t M, uint32_t log_m,
                                                           uint32_t a2, uint32_t b2, EncodeConsts C, const uint4* __restrict__ tw)
{
    const size_t total = (size_t)M * s4;
    const uint32_t mask = 2 * M - 1, sh = 19 - log_m;                           // GF_Root(2M)^e = tw[e << (20 - log2(2M))]
    FOR_GRID(size_t, i, total) {
        const uint32_t k2 = (uint32_t)(i / s4), c = (uint32_t)(i - (size_t)k2 * s4), k2r = k2 % R;
        uint4* row = x + (size_t)R * k2 * pitch4 + c;
        uint32_t f[4][R];
        encode_codelets<R>(row, pitch4, k2, mask, sh, a2, b2, C, tw, f);
        row[0] = make_uint4(f[0][0], f[1][0], f[2][0], f[3][0]);                 // j1 = 0: twiddle 1
#pragma unroll
        for (int j1 = 1; j1 < R; ++j1) {
            const uint32_t er = (a2 * ((k2r * 2 * j1) % R)) % R, em = (b2 * (2 * k2 * (uint32_t)j1)) & mask;
            const uint4 t = tw[(size_t)em << sh];
            uint32_t o[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t y = gf::mulc(f[j][j1], t);
                o[j] = er ? gf::mulc(y, C.fwd.zeta[er]) : y;
            }
            row[(size_t)j1 * pitch4] = make_uint4(o[0], o[1], o[2], o[3]);
        }
    }
}

// The constants of both step-2 kernels of the encode of N = r * M blocks; returns {a2, b2} = {(2M)^-1 mod r, r^-1 mod 2M}.
static CrtSplit fill_encode(EncodeConsts& C, uint32_t r, uint32_t M, uint32_t log_m)
{
    fill_codelets(C.inv, r, true);
    fill_codelets(C.fwd, r, false);
    const uint32_t zr = gf::powmod(gf::GEN, (gf::P - 1) / r), sigma = gf::powmod(gf::GEN, (gf::P - 1) / (2 * r)), inv_n = gf::inv(r * M);
    for (uint32_t j = 0; j < 9; ++j) { fill3(C.zin[j], gf::mulmod(gf::powmod(zr, j), inv_n)); fill3(C.sigma[j], gf::powmod(sigma, j)); }
    return crt_split(r, log_m + 1);
}

cudaError_t launch_radix_encode(uint32_t* x, uint32_t pitch4, uint32_t s4, uint32_t r, uint32_t M, const uint4* tw, int num_sms, cudaStream_t st)
{
    auto kernel = r == 3 ? radix_encode_kernel<3> : r == 9 ? radix_encode_kernel<9> : nullptr;
    if (!kernel || !M || (M & (M - 1)) || M > gf::M / 2) return cudaErrorInvalidValue;
    uint32_t log_m = 0; while ((1u << log_m) < M) ++log_m;
    EncodeConsts C;
    const CrtSplit ab = fill_encode(C, r, M, log_m);
    kernel<<<grid_size((size_t)M * s4, (size_t)num_sms * 16), 256, 0, st>>>(reinterpret_cast<uint4*>(x), pitch4, s4, M, log_m, ab.a, ab.b, C, tw);
    return cudaGetLastError();
}

// ---- step 2 of the encode of N = r * M data blocks into N / D parity blocks, D = s * 2^i, s | r (DESIGN 3f) ----------------
// Only parity p = D*j' is wanted.  With p = j1 + r*j2 (step 3's numbering): p = 0 mod s <=> j1 = 0 mod s, so only the outputs
// j1 = s*u (u < r/s) of the forward codelet are needed; p = 0 mod 2^i <=> j2 = c_j1 := -j1 * r^-1 mod 2^i.  Multiplying v_j1[k2]
// by GF_Root(M)^(k2*c_j1) = rho^(2r*k2*c_j1) moves that coset of step 3's outputs to the multiples of 2^i, which the sums
//     w_j1[t] = sum_{q < 2^f} v'_j1[t + T*q],    T = M / 2^f,  f <= i,
// followed by a T-point forward transform, produce at every 2^(i-f)-th output.  The twist folds into the output twiddle:
// rho^(2*k2*J_u), J_u = j1 + r*c_j1 = D*d_u, split by the CRT as in radix_encode_kernel.  Thread (t, chunk) reads the rows
// r*k2 + n1 of every k2 = t + T*q and writes w_j1[t] to row r*t + d_u -- rows that only it reads, so the pass is in place.
// f < i leaves T*s4 threads instead of (M / 2^i)*s4 when few parity blocks are wanted (the caller picks f).
struct FoldConsts {
    EncodeConsts e;
    uint32_t tr[9], tm[9];     // 2*J_u*a2 mod r and 2*J_u*b2 mod 2M: rho^(2*k2*J_u) = zeta[tr*k2 mod r] * GF_Root(2M)^(tm*k2 mod 2M)
    uint32_t d[9];             // output row offset d_u = J_u / D
};

template <int R, int S>
__global__ void __launch_bounds__(256) radix_fold_kernel(uint4* __restrict__ x, uint32_t pitch4, uint32_t s4, uint32_t M, uint32_t log_m,
                                                         uint32_t log_t, uint32_t n_fold, uint32_t a2, uint32_t b2, FoldConsts C, const uint4* __restrict__ tw)
{
    constexpr int U = R / S;
    const size_t total = (size_t)s4 << log_t;
    const uint32_t mask = 2 * M - 1, sh = 19 - log_m;
    FOR_GRID(size_t, i, total) {
        const uint32_t t = (uint32_t)(i / s4), c = (uint32_t)(i - (size_t)t * s4);
        uint32_t acc[U][4];
#pragma unroll
        for (int u = 0; u < U; ++u) acc[u][0] = acc[u][1] = acc[u][2] = acc[u][3] = 0;
        for (uint32_t q = 0; q < n_fold; ++q) {
            const uint32_t k2 = t + (q << log_t), k2r = k2 % R;
            const uint4* row = x + (size_t)R * k2 * pitch4 + c;
            uint32_t f[4][R];
            encode_codelets<R>(row, pitch4, k2, mask, sh, a2, b2, C.e, tw, f);
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[0][j] = gf::add(acc[0][j], f[j][0]);  // u = 0: J = 0, twiddle 1
#pragma unroll
            for (int u = 1; u < U; ++u) {
                const uint32_t er = (C.tr[u] * k2r) % R, em = (C.tm[u] * k2) & mask;
                const uint4 w = tw[(size_t)em << sh];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint32_t y = gf::mulc(f[j][S * u], w);
                    acc[u][j] = gf::add(acc[u][j], er ? gf::mulc(y, C.e.fwd.zeta[er]) : y);
                }
            }
        }
        uint4* out = x + (size_t)R * t * pitch4 + c;
#pragma unroll
        for (int u = 0; u < U; ++u) out[(size_t)C.d[u] * pitch4] = make_uint4(acc[u][0], acc[u][1], acc[u][2], acc[u][3]);
    }
}

cudaError_t launch_radix_fold(uint32_t* x, uint32_t pitch4, uint32_t s4, uint32_t r, uint32_t M, uint32_t s, uint32_t log_d2, uint32_t log_fold,
                              const uint4* tw, int num_sms, cudaStream_t st)
{
    auto kernel = r == 3 ? (s == 1 ? radix_fold_kernel<3, 1> : s == 3 ? radix_fold_kernel<3, 3> : nullptr)
                : r == 9 ? (s == 1 ? radix_fold_kernel<9, 1> : s == 3 ? radix_fold_kernel<9, 3> : s == 9 ? radix_fold_kernel<9, 9> : nullptr) : nullptr;
    if (!kernel || !M || (M & (M - 1)) || M > gf::M / 2 || (M >> log_d2) == 0 || log_fold > log_d2) return cudaErrorInvalidValue;
    uint32_t log_m = 0; while ((1u << log_m) < M) ++log_m;
    FoldConsts C;
    const CrtSplit ab = fill_encode(C.e, r, M, log_m);
    const uint64_t d2 = 1ull << log_d2, D = s * d2, rinv = crt_split(r, log_d2).b;           // r^-1 mod 2^i
    for (uint32_t u = 0; u < 9; ++u) {
        C.tr[u] = C.tm[u] = C.d[u] = 0;
        if (u >= r / s) continue;
        const uint64_t j1 = (uint64_t)s * u, cj = (d2 - (j1 * rinv) % d2) % d2, J = j1 + r * cj;   // c_j1 = -j1 * r^-1 mod 2^i
        C.tr[u] = (uint32_t)((2 * J % r) * ab.a % r);
        C.tm[u] = (uint32_t)((2 * J % (2 * M)) * ab.b % (2 * M));
        C.d[u] = (uint32_t)(J / D);
    }
    const uint32_t log_t = log_m - log_fold;
    kernel<<<grid_size((size_t)s4 << log_t, (size_t)num_sms * 16), 256, 0, st>>>(reinterpret_cast<uint4*>(x), pitch4, s4, M, log_m, log_t, 1u << log_fold, ab.a, ab.b, C, tw);
    return cudaGetLastError();
}

} // namespace fecc
