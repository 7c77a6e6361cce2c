// Erasure decoding behind the C ABI (include/fastecc_b200.h: fastecc_b200_rs_decode_*), SURVEY 8f rank 4.
//
// The reference describes the algorithm and does not implement it (README.md:88-119 "Fastest", RS.md:42-79, roadmap
// README.md:173).  Code word c[m] = f(rho^m), m < 2N, rho = GF_Root(2N), deg f < N; the encoder's layout is c[2i] = data
// block i, c[2j+1] = parity block j (RS.cpp:22-68).  For an erased set E (|E| <= N):
//     l(x) = prod_{e in E} (x - rho^e),   p = f*l is known at all 2N points (0 on E),   f(rho^e) = p'(rho^e) / l'(rho^e).
// Per word column: scale row m by l(rho^m), inverse NTT(2N), scale row t by t, forward NTT(2N), scale the erased rows by
// 1 / (2N * D[e]) with D = NTT(t * l_t).  Everything that depends only on WHICH rows are lost is built once
// (fastecc_b200_rs_decode_pattern) entirely on the device: the locator is a product tree over the erased points --
// leaves of 32 points by direct multiplication in one kernel, every further level ONE batched forward transform of all the
// polynomials (as word columns), one pairwise product (with the 1/n of the inverse transform folded in) and ONE batched
// inverse transform.  The Python mirror of the same algorithm is fastecc_b200/decoder.py.  Code words of 3 * 2^k and 9 * 2^k
// data blocks (fastecc_b200_rs_decode_pattern_mixed, DESIGN 3c / 3e) use the same steps with rho = GF_Root(2N) split by the CRT.
// The locator part (erasure_locator, declared in locator.h) also serves the repair patterns of repair.cu.
#include "mixed_radix.h"
#include "locator.h"
#include <new>

struct fastecc_b200_erasures {
    size_t n2 = 0, me = 0;
    uint32_t* d_idx = nullptr;       // [me]  erased positions, ascending
    uint32_t* d_lv = nullptr;        // [n2]  l(rho^m): zero exactly on the erased rows
    uint32_t* d_ce = nullptr;        // [me]  1 / (2N * D[e])
    uint32_t* d_pos = nullptr;       // [n2]  0, 1, 2, ...: the constants of the formal derivative
    fecc::DeviceArrays mem;          // owns the arrays above
};

namespace {

using namespace fecc;
constexpr uint32_t P = gf::P;
constexpr uint32_t kLeaf = 32;       // points per leaf polynomial
constexpr size_t kMaxGrid = 8192;    // blocks of the pattern kernels

__global__ void iota_kernel(uint32_t* out, size_t n) { FOR_GRID(size_t, i, n) out[i] = (uint32_t)i; }

// Leaves: polynomial g (column g of `polys`, coefficient k in row k, pitch words per row) = prod over its <= 32 points of
// (x - rho^e); groups beyond the erased set are the constant 1.
__global__ void leaves_kernel(const uint32_t* __restrict__ idx, size_t me, LeafRoots L, const uint4* __restrict__ tw,
                              uint32_t* __restrict__ polys, size_t groups, size_t pitch)
{
    FOR_GRID(size_t, g, groups) {
        uint32_t c[kLeaf + 1];
#pragma unroll
        for (uint32_t k = 0; k <= kLeaf; ++k) c[k] = k == 0 ? 1u : 0u;
        uint32_t deg = 0;
        for (uint32_t t = 0; t < kLeaf; ++t) {
            const size_t e = g * kLeaf + t;
            if (e >= me) break;
            const uint32_t pos = idx[e];
            const uint32_t r = rho_pow(L, tw, pos);
            ++deg;
#pragma unroll
            for (int k = kLeaf; k >= 1; --k) if ((uint32_t)k <= deg) c[k] = gf::sub(c[k - 1], gf::mulmod(c[k], r));       // c(x) * (x - r)
            c[0] = gf::sub(0u, gf::mulmod(c[0], r));
        }
#pragma unroll
        for (uint32_t k = 0; k <= kLeaf; ++k) polys[k * pitch + g] = c[k];
    }
}

// b[r][c] = a[r][2c] * a[r][2c+1] * scale   (point-wise product of neighbouring polynomials in the transform domain)
__global__ void pairmul_kernel(const uint32_t* __restrict__ a, size_t a_pitch, uint32_t* __restrict__ b, size_t b_pitch, size_t rows, size_t cols_out, uint32_t scale)
{
    FOR_GRID(size_t, i, rows * cols_out) {
        const size_t r = i / cols_out, c = i - r * cols_out;
        b[r * b_pitch + c] = gf::mulmod(gf::mulmod(a[r * a_pitch + 2 * c], a[r * a_pitch + 2 * c + 1]), scale);
    }
}
// dst (rows_dst x cols, zero padded) <- rows [0, rows_src) of src
__global__ void pad_rows_kernel(const uint32_t* __restrict__ src, size_t src_pitch, size_t rows_src, uint32_t* __restrict__ dst, size_t dst_pitch, size_t rows_dst, size_t cols)
{
    FOR_GRID(size_t, i, rows_dst * dst_pitch) {
        const size_t r = i / dst_pitch, c = i - r * dst_pitch;
        dst[i] = (r < rows_src && c < cols) ? src[r * src_pitch + c] : 0u;
    }
}
// column 0 of a pitched array -> two pitched single-column arrays: l_t and t * l_t
__global__ void locator_columns_kernel(const uint32_t* __restrict__ polys, size_t pitch, size_t ncoef, uint32_t* __restrict__ lv, uint32_t* __restrict__ dl, size_t n2)
{
    FOR_GRID(size_t, t, n2) {
        const uint32_t c = t < ncoef ? polys[t * pitch] : 0u;
        lv[t * 4] = c; lv[t * 4 + 1] = 0; lv[t * 4 + 2] = 0; lv[t * 4 + 3] = 0;
        dl[t * 4] = gf::mulmod(c, (uint32_t)(t % P)); dl[t * 4 + 1] = 0; dl[t * 4 + 2] = 0; dl[t * 4 + 3] = 0;
    }
}
__global__ void finish_pattern_kernel(const uint32_t* __restrict__ lv4, const uint32_t* __restrict__ dl4, const uint32_t* __restrict__ idx, size_t n2, size_t me,
                                      uint32_t* __restrict__ lv, uint32_t* __restrict__ ce)
{
    FOR_GRID(size_t, i, n2) {
        lv[i] = lv4[i * 4];
        if (i < me) ce[i] = gf::inv(gf::mulmod(dl4[(size_t)idx[i] * 4], (uint32_t)(n2 % P)));       // 1 / (2N * D[e])
    }
}
// out row i = code row idx[i] * ce[i]  (16-byte chunks)
__global__ void gather_scale_kernel(const uint4* __restrict__ code, size_t pitch4, const uint32_t* __restrict__ idx, const uint32_t* __restrict__ ce,
                                    uint4* __restrict__ out, size_t out_pitch4, size_t me, uint32_t s4)
{
    for (size_t row = blockIdx.x; row < me; row += gridDim.x) {
        const uint32_t c = ce[row];
        const uint4* src = code + (size_t)idx[row] * pitch4;
        uint4* dst = out + row * out_pitch4;
        for (uint32_t k = threadIdx.x; k < s4; k += blockDim.x) {
            uint4 v = src[k];
            v.x = gf::mulmod(v.x % P, c); v.y = gf::mulmod(v.y % P, c); v.z = gf::mulmod(v.z % P, c); v.w = gf::mulmod(v.w % P, c);
            dst[k] = v;
        }
    }
}

inline size_t pad4(size_t n) { return (n + 3) / 4 * 4; }

// The smallest transform order of the library (2^a, 3 * 2^a or 9 * 2^a with 2^a <= 2^20) above t; 0 if there is none.
size_t order_above(size_t t)
{
    size_t best = 0;
    for (size_t r : {1, 3, 9})
        for (size_t L = r; L <= (r << gf::LOG_M); L *= 2)
            if (L > t) { if (!best || L < best) best = L; break; }
    return best;
}

} // namespace

LeafRoots fecc::leaf_roots(size_t n2)
{
    LeafRoots lr{};
    const Order o = split_order(n2);                                            // n2 = r * 2^t, 2^t <= 2^20
    const CrtSplit ab = crt_split(o.r, o.log2_m);
    lr.r = o.r; lr.a2 = ab.a; lr.b2 = ab.b;
    lr.log_step = gf::LOG_M - o.log2_m; lr.mask = (1u << o.log2_m) - 1;
    if (lr.r > 1) {
        const uint32_t zr = gf::root(lr.r);
        for (uint32_t j = 0; j < 9; ++j) lr.zeta[j] = gf::powmod(zr, j);
    }
    return lr;
}

int fecc::erasure_locator(size_t n2, const uint32_t* d_idx, size_t me, DeviceArrays& tmp, uint32_t** lv4_out, uint32_t** dl4_out, cudaStream_t st, const char* who)
{
    const uint4* tw = context_power_table();
    const LeafRoots lr = leaf_roots(n2);
    // leaves
    size_t groups = 1; while (groups * kLeaf < me) groups *= 2;
    size_t d = kLeaf, cnt = groups, pitch = pad4(cnt), held = kLeaf + 1;       // held: rows of `polys`
    uint32_t* polys = tmp.alloc<uint32_t>((d + 1) * pitch);
    if (!polys) return fail(FASTECC_B200_ENOMEM, "%s: out of device memory", who);
    leaves_kernel<<<grid_size(groups, kMaxGrid), 256, 0, st>>>(d_idx, me, lr, tw, polys, groups, pitch);
    // product tree: cnt polynomials of degree <= d  ->  cnt/2 of degree <= 2d.  Batched transforms of order 4d; beyond 2^20
    // (more than 2^19 erasures: code words of 3 * 2^k, 9 * 2^k blocks) the smallest order above the largest actual product
    // degree min(2d, |E|), with the min(d, |E|) + 1 rows that can be nonzero copied in.
    while (cnt > 1) {
        size_t rows = 4 * d, copy = d + 1;
        if (rows > gf::M) { rows = order_above(2 * d < me ? 2 * d : me); copy = (d < me ? d : me) + 1; }
        const size_t half = cnt / 2, hp = pad4(half);
        uint32_t* a = tmp.alloc<uint32_t>(rows * pitch);
        uint32_t* b = tmp.alloc<uint32_t>(rows * hp);
        if (!a || !b) return fail(FASTECC_B200_ENOMEM, "%s: out of device memory", who);
        pad_rows_kernel<<<grid_size(rows * pitch, kMaxGrid), 256, 0, st>>>(polys, pitch, copy, a, pitch, rows, cnt);
        TRY_RC(fastecc_b200_ntt_u32_dev(a, rows, cnt, pitch, 0, st));
        if (hp != half) CUDA_TRY(cudaMemsetAsync(b, 0, rows * hp * sizeof(uint32_t), st));      // pad columns: transformed along, never used
        pairmul_kernel<<<grid_size(rows * half, kMaxGrid), 256, 0, st>>>(a, pitch, b, hp, rows, half, gf::inv((uint32_t)rows));
        TRY_RC(fastecc_b200_ntt_u32_dev(b, rows, half, hp, 1, st));
        polys = b; pitch = hp; cnt = half; d *= 2; held = rows;                // rows [0, min(d, |E|)] of b hold the products
    }
    // l(rho^m) and D = NTT(t * l_t): two single-column transforms of order n2 (16-byte rows)
    uint32_t* lv4 = tmp.alloc<uint32_t>(n2 * 4);
    uint32_t* dl4 = tmp.alloc<uint32_t>(n2 * 4);
    if (!lv4 || !dl4) return fail(FASTECC_B200_ENOMEM, "%s: out of device memory", who);
    size_t ncoef = d + 1 < n2 ? d + 1 : n2;
    if (ncoef > held) ncoef = held;
    locator_columns_kernel<<<grid_size(n2, kMaxGrid), 256, 0, st>>>(polys, pitch, ncoef, lv4, dl4, n2);
    TRY_RC(fastecc_b200_ntt_u32_dev(lv4, n2, 1, 4, 0, st));
    TRY_RC(fastecc_b200_ntt_u32_dev(dl4, n2, 1, 4, 0, st));
    *lv4_out = lv4; *dl4_out = dl4;
    return 0;
}

namespace {

int build_pattern(fastecc_b200_erasures* E, const uint32_t* erased, cudaStream_t st, const char* who)
{
    const size_t n2 = E->n2, me = E->me;
    E->d_pos = E->mem.alloc<uint32_t>(n2);
    if (me) { E->d_idx = E->mem.alloc<uint32_t>(me); E->d_lv = E->mem.alloc<uint32_t>(n2); E->d_ce = E->mem.alloc<uint32_t>(me); }
    if (E->mem.failed) return fail(FASTECC_B200_ENOMEM, "%s: out of device memory", who);
    iota_kernel<<<grid_size(n2, kMaxGrid), 256, 0, st>>>(E->d_pos, n2);
    if (me == 0) return 0;
    CUDA_TRY(cudaMemcpyAsync(E->d_idx, erased, me * 4, cudaMemcpyHostToDevice, st));
    DeviceArrays tmp;
    uint32_t *lv4 = nullptr, *dl4 = nullptr;
    TRY_RC(erasure_locator(n2, E->d_idx, me, tmp, &lv4, &dl4, st, who));
    finish_pattern_kernel<<<grid_size(n2, kMaxGrid), 256, 0, st>>>(lv4, dl4, E->d_idx, n2, me, E->d_lv, E->d_ce);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(st));                                        // the scratch buffers are freed on return
    return 0;
}

int make_pattern(size_t n_rows, const uint32_t* erased, size_t n_erased, void* stream, fastecc_b200_erasures** out, bool mixed, const char* who)
{
    if (!out) return fail(FASTECC_B200_EINVAL, "%s: null output", who);
    *out = nullptr;
    if (!fecc::context_power_table()) return fail(FASTECC_B200_ENOINIT, "%s: call fastecc_b200_init() first", who);
    const Order o = split_order(n_rows);                                        // n_rows = r * 2^k
    if (!o.r || (!mixed && o.r != 1) || o.log2_m < 1 || o.log2_m > FASTECC_B200_MAX_LOG_N)
        return fail(FASTECC_B200_EINVAL, mixed ? "%s: the code word must have 2N = 2^k, 3 * 2^k or 9 * 2^k rows, 1 <= k <= 20, got %zu"
                                               : "%s: the code word must have 2N = 2 .. 2^20 rows (a power of two), got %zu", who, n_rows);
    if (n_erased > n_rows / 2) return fail(FASTECC_B200_EINVAL, "%s: at most N = %zu of the 2N rows can be erased, got %zu", who, n_rows / 2, n_erased);
    if (n_erased && !erased) return fail(FASTECC_B200_EINVAL, "%s: null position list", who);
    if (!ascending_below(erased, n_erased, n_rows)) return fail(FASTECC_B200_EINVAL, "%s: erased positions must be ascending, distinct and below %zu", who, n_rows);
    fastecc_b200_erasures* E = new (std::nothrow) fastecc_b200_erasures;
    if (!E) return fail(FASTECC_B200_ENOMEM, "%s: out of host memory", who);
    E->n2 = n_rows; E->me = n_erased;
    const int rc = build_pattern(E, erased, (cudaStream_t)stream, who);
    if (rc) { delete E; return rc; }
    *out = E;
    return 0;
}

} // namespace

extern "C" {

int fastecc_b200_rs_decode_pattern(size_t n_rows, const uint32_t* erased, size_t n_erased, void* stream, fastecc_b200_erasures** out)
{ return make_pattern(n_rows, erased, n_erased, stream, out, false, "fastecc_b200_rs_decode_pattern"); }

int fastecc_b200_rs_decode_pattern_mixed(size_t n_rows, const uint32_t* erased, size_t n_erased, void* stream, fastecc_b200_erasures** out)
{ return make_pattern(n_rows, erased, n_erased, stream, out, true, "fastecc_b200_rs_decode_pattern_mixed"); }

int fastecc_b200_rs_decode_recover(const fastecc_b200_erasures* E, uint32_t* d_code, size_t size, size_t pitch, uint32_t* d_out, size_t out_pitch, void* stream)
{
    const char* who = "fastecc_b200_rs_decode_recover";
    if (!E || !d_code) return fail(FASTECC_B200_EINVAL, "%s: null argument", who);
    if (E->me == 0) return 0;
    if (!d_out) return fail(FASTECC_B200_EINVAL, "%s: null output buffer", who);
    if (size == 0 || pitch < size || pitch % 4 || out_pitch < size || out_pitch % 4 || ((uintptr_t)d_code) % 16 || ((uintptr_t)d_out) % 16)
        return fail(FASTECC_B200_EINVAL, "%s: needs SIZE >= 1, 16-byte aligned buffers, pitches >= SIZE and multiples of 4 words", who);
    cudaStream_t st = (cudaStream_t)stream;
    TRY_RC(fastecc_b200_row_scale_dev(d_code, E->n2, size, pitch, E->d_lv, st));            // p(rho^m) = c[m] * l(rho^m): zero on E whatever was there
    TRY_RC(fastecc_b200_ntt_u32_dev(d_code, E->n2, size, pitch, 1, st));                     // 2N * coefficients of p
    TRY_RC(fastecc_b200_row_scale_dev(d_code, E->n2, size, pitch, E->d_pos, st));            // t * p_t: x * p'(x)
    TRY_RC(fastecc_b200_ntt_u32_dev(d_code, E->n2, size, pitch, 0, st));                     // 2N * rho^j * p'(rho^j)
    const unsigned grid = (unsigned)(E->me < (size_t)fecc::context_num_sms() * 8 ? E->me : (size_t)fecc::context_num_sms() * 8);
    gather_scale_kernel<<<grid, 256, 0, st>>>(reinterpret_cast<const uint4*>(d_code), pitch / 4, E->d_idx, E->d_ce, reinterpret_cast<uint4*>(d_out), out_pitch / 4,
                                              E->me, (uint32_t)((size + 3) / 4));
    CUDA_TRY(cudaGetLastError());
    return 0;
}

size_t fastecc_b200_rs_decode_count(const fastecc_b200_erasures* E) { return E ? E->me : 0; }

void fastecc_b200_rs_decode_free(fastecc_b200_erasures* E) { delete E; }          // null-safe

} // extern "C"
