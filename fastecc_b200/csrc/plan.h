// Host-side planner: turns "NTT of N blocks" / "RS-encode N blocks" into a list of pass descriptors for
// ntt_pass_kernel.  Pure host code without CUDA runtime calls, so the same plans drive the GPU (api.cu) and the
// CPU emulation of the kernels (tests/emulate_tile.cu).
//
// What is being planned (reference call stacks, SURVEY 3.1/3.2):
//   MFA_NTT<uint32_t,0xFFF00001>(data, N, SIZE, InvNTT)            ntt.cpp:382-447
//   the timed body of EncodeReedSolomon<uint32_t,0xFFF00001>        RS.cpp:41-63
// The reference picks an R x C (or R x C x L) split that fits a CPU L2 slice and moves block *pointers*; the
// result is the unique canonical DFT, so the split is ours to choose.  Here N = N1*N2 with both factors <= 1024
// (one 64 KiB shared-memory tile holds a whole length-N1 or length-N2 column strip):
//
//   NTT  (N >= 1024, out of place through a scratch buffer Y so that natural order comes out without a transpose pass):
//     A'  X -> Y : for each n2, DIT over n1 (rows n1*N2+n2), plain; element k1 goes to row n2*N1+k1
//     B'  Y -> X : for each k1, DIT over n2 (rows n2*N1+k1) with input twist (w^k1)^n2; k2 goes to row k1+N1*k2
//   ENCODE (N >= 1024, in place, 3 passes instead of 2+2; m = k1 + N1*k2 is the coefficient index):
//     A   for each n2, inverse DIT over n1 (rows n1*N2+n2), inputs pre-scaled by 1/N
//     BC  for each k1 (rows k1*N2+.., contiguous): inverse DIT over n2 with input twist (w^-k1)^n2, then
//         forward DIT over k2 with input twist (rho^N1)^k2          (rho = root_2N, RS.cpp:51)
//     D   for each j2, forward DIT over k1 (rows k1*N2+j2) with input twist (w^j2 * rho)^k1 -> parity row j1*N2+j2
//   so the four-step twiddles (ntt.cpp:421-431) and the scaling rho^m (RS.cpp:54-58) never cost a multiplication.
//   N <= 512: a single pass (NTT) or a single fused pass (encode).   N < 32: see small_dft.cu.
#pragma once
#include <vector>
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include "ntt_tile.cuh"

namespace fecc {

inline uint32_t ilog2(size_t n) { uint32_t l = 0; while (((size_t)1 << l) < n) ++l; return l; }
inline bool     is_pow2(size_t n) { return n && !(n & (n - 1)); }
// N = N1*N2: log2 of the factor handled by the strided passes (A, D; A').  Strided passes touch a different DRAM page
// per row, so they want wide rows.  Copy-only floors at the headline size on an H100 SXM at a 400 W limit (-DFECC_SKIP_MATH,
// DESIGN.md section 6): a 512-row tile with 128-byte rows 1.68 ms per pass; the fused pass's 1024-row tile with 64-byte rows
// (256 threads) 3.15 ms, in the 512-thread geometry it runs in (128-byte rows, no bank conflicts, one CTA per SM) 1.58 ms.
// (Those floors include every shared-memory round: they measure the geometry as a whole, not DRAM granularity alone.)  So rows
// are made wide by the geometry, not by the split: every 1024-row pass and the fused 512-row pass run wide (pass_threads() in
// ntt_tile.cuh).
//   Single-GPU plans (plan_ntt, plan_encode, plan_encode_asym and the power-of-two transforms of the mixed-radix paths):
//     L1 = ceil(LN/2), so the strided passes take the longer factor: 2^19 = 1024 x 512.  The fused pass BC, bound by its
//     butterflies, then does 9 + 9 stages instead of 10 + 10, and A and D, bound by memory, one stage more each: the 2^19 encode
//     runs about 2 % faster than with 512 x 1024 (DESIGN.md section 6).  Only 2^19 changes: 2^20 is 1024 x 1024 either way, and
//     at 2^18 and below ceil(LN/2) <= 9.
//   short_n1 = true: L1 <= 9 whenever N2 = N/N1 still fits a tile (<= 1024), so 2^19 = 512 x 1024.  For the sharded plans
//     (shard_supported, plan_encode_shard[_p2p], shard_p2p_supported, ntt_shard_p2p_supported, plan_ntt_shard_p2p,
//     fastecc_b200_shard_geometry): their instantiations are narrow (TMA == 2), where a 1024-row tile has 64-byte rows and
//     64-byte remote stores.  And for the asymmetric encode to fewer parity blocks than the single-GPU N1 (asym_short_n1),
//     which needs M >= N1.
// FASTECC_B200_SPLIT=hi|lo overrides (ceil / floor of LN/2) for experiments; "lo" is the 512 x 1024 plan at 2^19 on one GPU.
inline uint32_t split_l1(uint32_t LN, bool short_n1 = false)
{
    static const char* env = getenv("FASTECC_B200_SPLIT");
    uint32_t L1 = (LN + 1) / 2;
    if (env && !strcmp(env, "lo")) L1 = LN / 2;
    else if (!(env && !strcmp(env, "hi")) && short_n1 && L1 > 9) L1 = 9;
    if (L1 < (uint32_t)kMinLogR) L1 = kMinLogR;
    if (LN - L1 > (uint32_t)kMaxLogR) L1 = LN - kMaxLogR;
    return L1;
}

// Orders up to 2^9 run as ONE pass (the whole transform, or the whole fused encode, on a tile).  2^10 could too (a tile holds 1024
// rows), but its 4 MiB at 4 KiB blocks are then only 64 tiles each doing 10 (NTT) or 20 (encode) stages in series: 30 / 53 us,
// slower than 2^11 with its two / three short passes (16 / 32 us).  So 2^10 = 32 x 32 takes the multi-pass plans as well.
constexpr uint32_t kSinglePassMaxLog = 9;
inline bool single_pass(uint32_t LN) { return LN <= kSinglePassMaxLog; }

struct Buffers { uint32_t* x; uint32_t* y; const uint4* tw; uint32_t pitch_words; uint32_t size_words; };

inline PassParams base_pass(const Buffers& b, uint32_t log_r)
{
    PassParams p{};
    p.tw = b.tw;
    p.pitch4 = b.pitch_words / 4;
    p.s4 = (b.size_words + 3) / 4;
    p.log_r = log_r;
    set_strips<kThreads>(p);                                            // narrow layout; launch_pass re-lays a pass it runs wide
    p.nxf = 1;
    return p;
}

constexpr uint32_t kM = gf::M;
inline void set_prescale(PassParams& p, uint32_t c)                     // multiply every input word of the pass by c
{
    const gf::Tw t = gf::make_tw(c);
    p.prescale = 1; p.pw = t.w;
    gf::wp_bits(t.whi, t.wlo, p.pwp_lo, p.pwp_hi);
}
inline uint32_t emod(long long e) { return (uint32_t)(((e % (long long)kM) + kM) % kM); }

// Standalone transform.  Result lands in b.x; b.y is scratch (needed only when N > 1024).
inline std::vector<PassParams> plan_ntt(const Buffers& b, size_t N, bool inverse)
{
    std::vector<PassParams> v;
    const uint32_t LN = ilog2(N);
    const long long p = (long long)(kM / N) * (inverse ? -1 : 1);       // w = g^p
    if (single_pass(LN)) {
        PassParams a = base_pass(b, LN);
        a.src = b.x; a.dst = b.x; a.nsets = 1;
        a.src_set_stride = a.dst_set_stride = 0; a.src_row_stride = a.dst_row_stride = 1;
        a.xf[0] = Xform{emod(p), 0, 0};
        a.canonical_out = 1;
        v.push_back(a);
        return v;
    }
    const uint32_t L1 = split_l1(LN), L2 = LN - L1;
    const uint32_t N1 = 1u << L1, N2 = 1u << L2;
    PassParams a = base_pass(b, L1);
    a.src = b.x; a.dst = b.y; a.nsets = (uint32_t)N2;
    a.src_set_stride = 1;  a.src_row_stride = N2;
    a.dst_set_stride = N1; a.dst_row_stride = 1;
    a.xf[0] = Xform{emod(p * (long long)N2), 0, 0};
    v.push_back(a);
    PassParams c = base_pass(b, L2);
    c.src = b.y; c.dst = b.x; c.nsets = (uint32_t)N1;
    c.src_set_stride = 1; c.src_row_stride = N1;
    c.dst_set_stride = 1; c.dst_row_stride = N1;
    c.xf[0] = Xform{emod(p * (long long)N1), 0, emod(p)};
    c.canonical_out = 1;
    v.push_back(c);
    return v;
}

// RS.cpp:41-63 on N data blocks -> N parity blocks, in place in b.x.  short_n1: see split_l1.
inline std::vector<PassParams> plan_encode(const Buffers& b, size_t N, bool short_n1 = false)
{
    std::vector<PassParams> v;
    const uint32_t LN = ilog2(N);
    const long long q = (long long)(kM / (2 * N));                      // rho = root_2N = g^q, w = g^(2q)
    const uint32_t invN = gf::inv((uint32_t)N);                         // GF_Inv(N), RS.cpp:51
    if (single_pass(LN)) {
        PassParams a = base_pass(b, LN);
        a.src = b.x; a.dst = b.x; a.nsets = 1;
        a.src_set_stride = a.dst_set_stride = 0; a.src_row_stride = a.dst_row_stride = 1;
        a.nxf = 2;
        a.xf[0] = Xform{emod(-2 * q), 0, 0};
        a.xf[1] = Xform{emod(2 * q), emod(q), 0};
        set_prescale(a, invN);
        a.canonical_out = 1;
        v.push_back(a);
        return v;
    }
    const uint32_t L1 = split_l1(LN, short_n1), L2 = LN - L1;
    const uint32_t N1 = 1u << L1, N2 = 1u << L2;
    PassParams a = base_pass(b, L1);
    a.src = b.x; a.dst = b.x; a.nsets = (uint32_t)N2;
    a.src_set_stride = a.dst_set_stride = 1; a.src_row_stride = a.dst_row_stride = N2;
    a.xf[0] = Xform{emod(-2 * q * (long long)N2), 0, 0};
    set_prescale(a, invN);
    v.push_back(a);
    PassParams bc = base_pass(b, L2);
    bc.src = b.x; bc.dst = b.x; bc.nsets = (uint32_t)N1;
    bc.src_set_stride = bc.dst_set_stride = N2; bc.src_row_stride = bc.dst_row_stride = 1;
    bc.nxf = 2;
    bc.xf[0] = Xform{emod(-2 * q * (long long)N1), 0, emod(-2 * q)};
    bc.xf[1] = Xform{emod(2 * q * (long long)N1), emod(q * (long long)N1), 0};
    v.push_back(bc);
    PassParams d = base_pass(b, L1);
    d.src = b.x; d.dst = b.x; d.nsets = (uint32_t)N2;
    d.src_set_stride = d.dst_set_stride = 1; d.src_row_stride = d.dst_row_stride = N2;
    d.xf[0] = Xform{emod(2 * q * (long long)N2), emod(q), emod(2 * q)};
    d.canonical_out = 1;
    v.push_back(d);
    return v;
}

// Asymmetric encode: N data blocks -> M = N / 2^k parity blocks, parity'[j'] = parity[2^k * j'] of the full encode (the even
// points of the second transform, RS.cpp:65-66, NTT.md:46-49).  With output index j = j1*N2 + j2, the wanted outputs are
// the row sets j2 = 2^k * j2' of pass D: D runs on N2 / 2^k sets only and writes its result compactly (row j1*N2' + j2').
// A is unchanged; BC writes to the scratch buffer b.y because D now reads rows that its compact output would overwrite.
// Needs the two-level decomposition and M >= N1 (every wanted output still has j2 as its low digit); smaller M and
// N <= 1024 are served by the caller from the smallest supported M (api.cu).  An M below the single-GPU N1 takes the short
// split (2^19 = 512 x 1024), so M = 512 at 2^19 stays native.  The first transform and the C half of BC are not shortened yet
// (folding the coefficients before C needs the scaling as an explicit product first).
inline bool asym_short_n1(size_t N, size_t M) { return M < ((size_t)1 << split_l1(ilog2(N))); }
inline bool asym_native(size_t N, size_t M)
{
    const uint32_t LN = ilog2(N);
    if (LN <= (uint32_t)kMaxLogR || M >= N) return false;
    return M >= ((size_t)1 << split_l1(LN, asym_short_n1(N, M)));
}
inline std::vector<PassParams> plan_encode_asym(const Buffers& b, size_t N, size_t M)
{
    const bool short_n1 = asym_short_n1(N, M);
    std::vector<PassParams> v = plan_encode(b, N, short_n1);            // A, BC, D
    const uint32_t LN = ilog2(N), L1 = split_l1(LN, short_n1), L2 = LN - L1;
    const uint32_t N2 = 1u << L2, dec = (uint32_t)(N / M), N2s = N2 / dec;
    const long long q = (long long)(kM / (2 * N));
    v[1].dst = b.y;
    PassParams& d = v[2];
    d.src = b.y; d.dst = b.x;
    d.nsets = N2s;
    d.src_set_stride = dec; d.src_row_stride = N2;
    d.dst_set_stride = 1;   d.dst_row_stride = N2s;
    d.xf[0] = Xform{emod(2 * q * (long long)N2), emod(q), emod(2 * q * (long long)dec)};
    return v;
}

// One transform sharded over G GPUs (BASELINE config 4, SURVEY 8e).  Blocks are dealt cyclically: global block
// i = l*G + g is local block l of rank g, for the data going in and for the parity coming out.  With N2 % G == 0 every
// row set of pass A (fixed n2) and of pass D (fixed j2) is local to rank n2 % G resp. j2 % G, and every row set of
// pass BC (fixed k1) is local to rank k1 % G after an all-to-all of whole blocks (fastecc_b200/sharded.py); that needs
// N1 % G == 0 as well, or pass BC would have N1 / G = 0 row sets on every rank and nothing would compute it.  The local
// passes are the single-GPU ones with local strides; the only thing that knows about the sharding is the twist,
// whose exponent t0 + set*t1 is evaluated at the GLOBAL set index set_local*G + rank.
//   which = 0: A  on local rows n1*(N2/G) + n2'            (n2 = n2'*G + rank)
//   which = 1: BC on local rows k1'*N2 + n2                (k1 = k1'*G + rank)
//   which = 2: D  on local rows k1*(N2/G) + j2'            (j2 = j2'*G + rank)
inline bool shard_supported(size_t N, uint32_t G)
{
    if (!is_pow2(N) || !is_pow2(G) || G < 2) return false;
    const uint32_t LN = ilog2(N);
    if (LN <= (uint32_t)kMaxLogR || LN > 19) return false;
    const uint32_t L1 = split_l1(LN, true), L2 = LN - L1;
    return (1u << L2) >= G * 1u && ((1u << L2) % G) == 0 && ((1u << L1) % G) == 0;
}
inline PassParams plan_encode_shard(const Buffers& b, size_t N, uint32_t G, uint32_t rank, int which)
{
    const uint32_t LN = ilog2(N);
    const long long q = (long long)(kM / (2 * N));
    const uint32_t L1 = split_l1(LN, true), L2 = LN - L1;
    const uint32_t N1 = 1u << L1, N2 = 1u << L2;
    PassParams p;
    if (which == 0) {
        p = base_pass(b, L1);
        p.nsets = N2 / G;
        p.src_set_stride = p.dst_set_stride = 1; p.src_row_stride = p.dst_row_stride = N2 / G;
        p.xf[0] = Xform{emod(-2 * q * (long long)N2), 0, 0};
        set_prescale(p, gf::inv((uint32_t)N));
    } else if (which == 1) {
        p = base_pass(b, L2);
        p.nsets = N1 / G;
        p.src_set_stride = p.dst_set_stride = N2; p.src_row_stride = p.dst_row_stride = 1;
        p.nxf = 2;
        p.xf[0] = Xform{emod(-2 * q * (long long)N1), emod(-2 * q * (long long)rank), emod(-2 * q * (long long)G)};
        p.xf[1] = Xform{emod(2 * q * (long long)N1), emod(q * (long long)N1), 0};
    } else {
        p = base_pass(b, L1);
        p.nsets = N2 / G;
        p.src_set_stride = p.dst_set_stride = 1; p.src_row_stride = p.dst_row_stride = N2 / G;
        p.xf[0] = Xform{emod(2 * q * (long long)N2), emod(q + 2 * q * (long long)rank), emod(2 * q * (long long)G)};
        p.canonical_out = 1;
    }
    p.src = b.x; p.dst = b.x;
    return p;
}

// The same three passes with the exchange fused into the stores of passes A and BC: every rank holds two buffers of N/G
// rows (X: data in / parity out, Y: intermediate), mapped into every other rank (CUDA IPC, NVLink).  Pass A reads the
// local X and scatters its output rows straight into the Y of their owners (element k1 -> rank k1 mod G, row
// (k1 / G)*N2 + n2'*G + rank), pass BC reads the local Y and scatters into the owners' X (element j2 -> rank j2 mod G,
// row (k1'*G + rank)*(N2/G) + j2 / G), pass D is local and in place.  No all-to-all, no staging copies: the transfer
// is the store traffic of the kernel itself.  Needs every thread's 32 output elements on one rank: G <= 2^(LR-5) for
// both tile heights.
inline bool shard_p2p_supported(size_t N, uint32_t G)
{
    if (!shard_supported(N, G) || G > kMaxPeers) return false;
    const uint32_t LN = ilog2(N), L1 = split_l1(LN, true), L2 = LN - L1, lg = ilog2(G);
    return L1 >= 5 + lg && L2 >= 5 + lg;
}
inline PassParams plan_encode_shard_p2p(const uint32_t* src, uint32_t* const* peers, const uint4* tw, uint32_t pitch_words, uint32_t size_words,
                                        size_t N, uint32_t G, uint32_t rank, int which)
{
    Buffers b{const_cast<uint32_t*>(src), nullptr, tw, pitch_words, size_words};
    PassParams p = plan_encode_shard(b, N, G, rank, which);
    if (which == 2) return p;                                       // local, in place
    const uint32_t LN = ilog2(N), L1 = split_l1(LN, true), N2 = 1u << (LN - L1);
    p.log_g = ilog2(G);
    for (uint32_t r = 0; r < kMaxPeers; ++r) p.peers[r] = peers[r < G ? r : 0];
    p.dst = peers[rank];
    if (which == 0) { p.dst_row_stride = N2; p.dst_set_stride = G;  p.dst_row_offset = rank; }
    else            { p.dst_row_stride = 1;  p.dst_set_stride = N2; p.dst_row_offset = rank * (N2 / G); }
    return p;
}

// ONE standalone transform (MFA_NTT, ntt.cpp:382-447) sharded the same way (BASELINE config 5 "at 1 and 8 GPUs"): blocks dealt
// cyclically for the input AND the output.  Pass A' (for each local n2, DIT over n1) reads the local X and stores element k1
// into row n2*(N1/G) + k1/G of the Y of rank k1 mod G -- the transpose between the two steps of the four-step algorithm
// (TransposeMatrix, ntt.cpp:322-341) as peer stores; pass B' (for each local k1, DIT over n2 with the four-step twiddle as input
// twist) is then local, Y -> X, and its output element k2 = global block k1 + N1*k2 is again owned by this rank (N1 % G == 0).
inline bool ntt_shard_p2p_supported(size_t N, uint32_t G)
{
    if (!is_pow2(N) || !is_pow2(G) || G < 2 || G > kMaxPeers) return false;
    const uint32_t LN = ilog2(N);
    if (LN <= (uint32_t)kMaxLogR || LN > 20) return false;
    const uint32_t L1 = split_l1(LN, true), L2 = LN - L1, lg = ilog2(G);
    return L1 >= 5 + lg && L2 >= lg;
}
inline PassParams plan_ntt_shard_p2p(const uint32_t* src, uint32_t* const* peers, const uint4* tw, uint32_t pitch_words, uint32_t size_words,
                                     size_t N, uint32_t G, uint32_t rank, bool inverse, int which)
{
    Buffers b{const_cast<uint32_t*>(src), nullptr, tw, pitch_words, size_words};
    const uint32_t LN = ilog2(N), L1 = split_l1(LN, true), L2 = LN - L1;
    const uint32_t N1 = 1u << L1, N2 = 1u << L2;
    const long long p = (long long)(kM / N) * (inverse ? -1 : 1);       // w = g^p
    PassParams a;
    if (which == 0) {
        a = base_pass(b, L1);
        a.nsets = N2 / G;
        a.src_set_stride = 1; a.src_row_stride = N2 / G;
        a.xf[0] = Xform{emod(p * (long long)N2), 0, 0};
        a.log_g = ilog2(G);
        for (uint32_t r = 0; r < kMaxPeers; ++r) a.peers[r] = peers[r < G ? r : 0];
        a.dst_row_stride = 1; a.dst_set_stride = N1; a.dst_row_offset = rank * (N1 / G);
    } else {
        a = base_pass(b, L2);
        a.nsets = N1 / G;
        a.src_set_stride = 1; a.src_row_stride = N1 / G;
        a.dst_set_stride = 1; a.dst_row_stride = N1 / G;
        a.xf[0] = Xform{emod(p * (long long)N1), emod(p * (long long)rank), emod(p * (long long)G)};
        a.canonical_out = 1;
    }
    a.src = src; a.dst = peers[rank];
    return a;
}

// Per-set stage tables of a pass: [set][xfi][R] entries of 16 bytes; a single shared set when no twist depends on it.
inline uint32_t table_sets(const PassParams& P)
{
    bool varies = false;
    for (uint32_t x = 0; x < P.nxf; ++x) if (P.xf[x].t1) varies = true;
    return varies ? P.nsets : 1u;
}
inline size_t table_bytes(const PassParams& P) { return (size_t)table_sets(P) * P.nxf * ((size_t)16 << P.log_r); }

// g^e table, e in [0, 2^20): 16 MiB, L2-resident on the device.
inline void fill_power_table(gf::Tw* t)
{
    const uint32_t g = gf::root(kM);
    uint32_t w = 1;
    for (uint32_t e = 0; e < kM; ++e) { t[e] = gf::make_tw(w); w = gf::mulmod(w, g); }
}

} // namespace fecc
