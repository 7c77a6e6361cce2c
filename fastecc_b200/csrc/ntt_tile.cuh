// Tile-level decimation-in-time NTT over GF(0xFFF00001): the code every pass kernel runs per 64 or 128 KiB tile.
//
// This header is the GPU counterpart of the reference's inner loops
//     IterativeNTT_Steps  ntt.cpp:251-284   (radix-2 butterflies across blocks, inner loop over the SIZE words)
//     revbin_permute      ntt.cpp:292-309   (here: bit-reversed *addressing* when a tile is loaded, no data pass)
//     MFA twiddle loop    ntt.cpp:421-431   (here: folded into the butterfly twiddles of the next pass, see below)
//     scaling loop        RS.cpp:51-59      (here: folded into butterfly twiddles + one uniform pre-scale)
// It is written as plain `__host__ __device__` code over an abstract "thread id" so that exactly the same
// index/twiddle logic can be executed thread-by-thread on the CPU (tests/emulate_tile.cu) before it ever
// touches a GPU.
//
// Geometry.  A tile is R = 2^LR rows (blocks) x WT words, R*WT = 16384 words (64 KiB of shared memory, 256 threads) or
// 32768 words (128 KiB, 512 threads: the wide geometry, Geom<512>), stored as 16-byte chunks: chunk (row p, q) at index
// p*(WT/4)+q.  Thread (j, q2) owns the word PAIR q2 of every row it touches (the word dimension is a pure batch
// dimension, SURVEY 7 "hard part 2") and, in every round, 32 rows: q2 = tid % (WT/2), j = tid / (WT/2) in [0, R/32).
// Thirty-two rows x two words = 64 data registers in either geometry; only the (j, q2) mapping differs.
//
// Rounds.  A size-R DIT transform runs ceil(LR/5) <= 2 rounds.  Round 0 holds index bits [0,5) in-thread and
// executes the stages of bits [0, min(5,LR)); round 1 holds bits [LR-5, LR) and executes the stages of bits
// [5, LR).  In a round a thread holds the 32 slots
//     r_i = ((j >> lb) << (lb+5)) | (i << lb) | (j & (2^lb - 1)),   i = 0..31
// in registers, performs up to 5 stages x 16 butterflies x 2 words, and writes the slots back in place; one
// block barrier separates rounds.  Slot r of a DIT transform initially holds input element bitrev_LR(r) and
// finally holds output element r.  Tiles arrive in natural row order (TMA box copies cannot permute rows), so the
// FIRST transform of a tile keeps slot r at tile row bitrev_LR(r) ("bit-reversed placement") for all its rounds.
//
// Fused tiles (two transforms back to back, the "BC" pass of the encoder): the second transform's input index
// bitrev(r') is the first transform's output slot, which sits at tile row r' -- so the second transform runs in
// identity placement.  The 32 rows a thread holds in the LAST round of the first transform (rows differing in
// the low five bits) are exactly the 32 slots of one thread of the FIRST round of the second transform, only
// renumbered i -> brev5(i).  So that
// pair of rounds is executed back to back in registers: 18 stages of a 512-point fused tile cost 3 shared-memory
// round trips instead of 4 (or 6 with radix-16 rounds).
//
// Twiddles.  All twiddles are powers of g = GF_Root(2^20) (GF(p).cpp:267-276).  A transform is described by two
// exponents (mod 2^20):  zeta = g^z is the primitive R-th root used by this tile, theta = g^t an *input twist*:
// the transform computes  X[k] = sum_n x[n] * theta^n * zeta^(n k).  A twisted DIT costs exactly as much as a
// plain one: the stage that pairs slots differing in bit b uses, for the pair whose low b bits are n,
//     T[2^b + n] = g^( 2^(LR-1-b) * (z*n + t) )                                   (heap-ordered table, R-1 entries)
// (derivation in DESIGN.md section 3).  Four-step twiddles (ntt.cpp:421-431) and the RS scaling root_2N^i
// (RS.cpp:54) are input twists of the following pass, so they cost no multiplications at all.
#pragma once
#include "gf.cuh"

#if defined(__CUDACC__)
#define FECC_HD __host__ __device__ __forceinline__
#else
#define FECC_HD inline
#endif

namespace fecc {

constexpr int kThreads    = 256;             // the narrow (default) geometry: threads per CTA ...
constexpr int kTileChunks = 4096;            // ... and 16-byte chunks per tile
constexpr int kTileBytes  = kTileChunks * 16;
constexpr int kWideThreads = 512;            // the wide geometry: one CTA per SM over a 128 KiB tile
constexpr int kMaxLogR    = 10;
constexpr int kMinLogR    = 5;
constexpr int kRows       = 32;              // rows held by a thread in a round
constexpr int kStages     = 5;               // radix-2 stages per full round

// Geometry of a CTA: NT threads, each holding 32 rows x one word pair = 16 chunks, so a tile is 16*NT chunks of 2^LOGW
// words.  NT = 256: 64 KiB tiles, rows of 2^(14-LR) words.  NT = 512: 128 KiB tiles, rows of 2^(15-LR) words (128-byte
// rows at LR = 10).  Every index function below takes NT as a template parameter defaulting to the narrow geometry.
template <int NT> struct Geom {
    static constexpr int      threads = NT;
    static constexpr int      chunks  = 16 * NT;
    static constexpr uint32_t bytes   = 16u * chunks;
    static constexpr uint32_t logw    = NT == 512 ? 15 : NT == 256 ? 14 : 0;    // log2(words per tile)
    static_assert(logw != 0, "tile geometries: 256 or 512 threads");
};

// Geometry of the pass-kernel instantiation <LR, NXF, TMA> (ntt_pass.cu; the CPU emulation asks the same question).  Wide: the
// 1024-row passes, fused or single-transform, whose narrow tile has 64-byte rows (2-way bank conflicts, 64-byte DRAM pieces, two
// copies of the stage tables per SM), and the 512-row fused pass (BC of the 2^18 and 2^19 encodes), which runs its butterflies
// about 7 % faster wide with its steps unrolled (DESIGN.md section 6).  The sharded instantiations (TMA == 2) stay narrow.
// -DFECC_WIDE_A (A/B build only) runs the 512-row single-transform pass wide as well.
#if !defined(FECC_WIDE_A)
#define FECC_WIDE_A 0
#endif
FECC_HD constexpr int pass_threads(int LR, int NXF, int TMA)
{
    return TMA == 1 && (LR == 10 || (LR == 9 && (NXF == 2 || FECC_WIDE_A))) ? kWideThreads : kThreads;
}
// Whether the instantiation unrolls its steps (ntt_pass.cu): every round's slot offsets, table strides and stage ranges then
// become immediates.  The wide instantiations do, without spills at 128 registers.  The narrow ones keep one copy of the step
// body: several spill unrolled, and <9,2,1> narrow, which did not, ran the 2^19 fused pass about 20 % slower unrolled (two CTAs
// per SM in different parts of the longer code; DESIGN.md section 6).
FECC_HD constexpr bool pass_unrolled(int LR, int NXF, int TMA)
{
    return pass_threads(LR, NXF, TMA) == kWideThreads;
}
// Whether the wide instantiation also has a narrow twin, which launch_pass (ntt_pass.cu) takes for a pass with fewer wide tiles
// than SMs: the single-pass encode of 2^9 blocks (one row set) would otherwise leave most SMs idle with half as many tiles.  The
// twin unrolls its steps like its wide sibling (pass_unrolled is per <LR, NXF, TMA>); with one tile per CTA that is faster.
FECC_HD constexpr bool pass_has_narrow_twin(int LR, int NXF, int TMA)
{
    return pass_threads(LR, NXF, TMA) == kWideThreads && LR == 9 && NXF == 2;
}

struct Xform { uint32_t z, t0, t1; };        // tile root g^z; input twist g^(t0 + set*t1)   (exponents mod 2^20)

struct PassParams {
    const uint32_t* src;
    uint32_t*       dst;
    const uint4*    tw;                      // g^e for e in [0, 2^20): {w, Whi, Wlo, 0}  (gf::Tw)
    uint32_t pitch4;                         // row pitch in 16-byte chunks
    uint32_t s4;                             // valid 16-byte chunks per row (ceil(SIZE/4))
    uint32_t log_r;                          // log2(rows per tile), 5..10
    uint32_t nsets;                          // number of independent row sets
    uint32_t nstrips;                        // ceil(s4 / (WT/4))
    uint32_t strips_per_item;                // consecutive strips of one set handled by one CTA visit
    uint32_t src_set_stride, src_row_stride, dst_set_stride, dst_row_stride;             // in rows
    uint32_t nxf;                            // 1, or 2 = two transforms back to back on the same tile
    Xform    xf[2];
    uint32_t prescale;                       // multiply every input word by the constant below (1/N)
    uint32_t pw, pwp_lo, pwp_hi;             // the constant and its quotient factor wp (gf::mul_h); set_prescale() in plan.h
    uint32_t canonical_out;                  // reduce stored words to [0,P)
    const uint4* tables;                     // per-set stage tables [set][xfi][R] of stage_entry()s, built once per plan (build_tables_kernel)
    uint32_t table_set_stride;               // uint4 entries between consecutive sets' tables (0: every set shares set 0's)
    uint32_t use_tma;                        // 1: tile/table loads by TMA (cp.async.bulk[.tensor]) + mbarrier; 0: 16-byte cp.async
    // One transform sharded over 2^log_g GPUs with the exchange fused into the stores (plan_encode_shard_p2p): output
    // element e of a set goes to buffer peers[e mod G] (peer-mapped device memory, NVLink), row
    // dst_row_offset + set*dst_set_stride + (e / G)*dst_row_stride.  log_g = 0: everything goes to dst.
    uint32_t log_g;
    uint32_t dst_row_offset;
    uint32_t* peers[8];
};
constexpr uint32_t kMaxPeers = 8;

FECC_HD uint32_t bitrev(uint32_t x, uint32_t bits)
{
    if (bits == 0) return 0;
#if defined(__CUDA_ARCH__)
    return __brev(x) >> (32 - bits);
#else
    uint32_t r = 0; for (uint32_t i = 0; i < bits; i++) r |= ((x >> i) & 1u) << (bits - 1 - i); return r;
#endif
}
FECC_HD uint32_t popc32(uint32_t x)
{
#if defined(__CUDA_ARCH__)
    return __popc(x);
#else
    return (uint32_t)__builtin_popcount(x);
#endif
}

// compile-time helpers for the unrolled slot loops
FECC_HD constexpr uint32_t par5(int i)  { return ((i) ^ (i >> 1) ^ (i >> 2) ^ (i >> 3) ^ (i >> 4)) & 1u; }       // popcount(i) & 1
FECC_HD constexpr int      brev5(int i) { return ((i & 1) << 4) | ((i & 2) << 2) | (i & 4) | ((i & 8) >> 2) | ((i & 16) >> 4); }
FECC_HD constexpr int      brev4(int i) { return ((i & 1) << 3) | ((i & 2) << 1) | ((i & 4) >> 1) | ((i & 8) >> 3); }
FECC_HD constexpr uint32_t par4(int i)  { return (0x6996u >> i) & 1u; }

FECC_HD uint32_t num_rounds(uint32_t LR) { return LR > (uint32_t)kStages ? 2u : 1u; }

// Steps of a tile.  nxf == 1: rounds 0..nr-1.  nxf == 2: rounds 0..nr-2 of transform 0, then the FUSED step
// (last round of transform 0 + round 0 of transform 1 in registers), then rounds 1..nr-1 of transform 1.
FECC_HD uint32_t num_steps(uint32_t LR, uint32_t nxf) { const uint32_t nr = num_rounds(LR); return nxf == 2 ? 2 * nr - 1 : nr; }
struct Step { uint32_t xfi, k; bool fused; };
FECC_HD Step step_of(uint32_t LR, uint32_t nxf, uint32_t s)
{
    const uint32_t nr = num_rounds(LR);
    Step st;

    if (nxf == 1 || s + 1 < nr) { st.xfi = 0; st.k = s; st.fused = false; }
    else if (s + 1 == nr)       { st.xfi = 0; st.k = s; st.fused = true; }
    else                        { st.xfi = 1; st.k = s + 1 - nr; st.fused = false; }
    return st;
}

// exponent of heap entry idx (1 <= idx < R) of the stage table
FECC_HD uint32_t table_exponent(uint32_t idx, uint32_t LR, uint32_t z, uint32_t t)
{
#if defined(__CUDA_ARCH__)
    uint32_t b = 31 - __clz(idx);
#else
    uint32_t b = 31 - (uint32_t)__builtin_clz(idx);
#endif
    uint32_t n = idx - (1u << b);
    return ((z * n + t) << (LR - 1 - b)) & (gf::M - 1);
}

FECC_HD uint2 canon2(uint2 v) { v.x = gf::canon(v.x); v.y = gf::canon(v.y); return v; }

// A stage-table entry, as the pass kernels read it from shared memory: {w, 0, lo32(wp), hi32(wp)} with wp the double
// of gf::mul_h.  Made from an entry {w, Whi, Wlo, 0} of the global power table (build_tables_kernel, CPU emulation).
FECC_HD uint4 stage_entry(const uint4& t)
{
#if defined(FECC_MUL_BARRETT)            // A/B experiment: the round-1 integer-only product (gf::mul)
    return t;
#endif
    uint4 e; e.x = t.x; e.y = 0;
    gf::wp_bits(t.y, t.z, e.z, e.w);
    return e;
}

// One butterfly on a word pair:  (a, b) <- (a + w*b, a - w*b)
FECC_HD void bfly2(uint2& a, uint2& b, const uint4& w)
{
    uint32_t v;
#if defined(FECC_MUL_BARRETT)
    v = gf::mul(b.x, w.x, w.y, w.z); b.x = gf::subl(a.x, v); a.x = gf::addl(a.x, v);
    v = gf::mul(b.y, w.x, w.y, w.z); b.y = gf::subl(a.y, v); a.y = gf::addl(a.y, v);
#else
    v = gf::mul_h(b.x, w.x, w.z, w.w); b.x = gf::subl(a.x, v); a.x = gf::addl(a.x, v);
    v = gf::mul_h(b.y, w.x, w.z, w.w); b.y = gf::subl(a.y, v); a.y = gf::addl(a.y, v);
#endif
}
// the same with twiddle 1: b only has to be brought into [0,P) (two ALU instructions) for the lazy add/sub
FECC_HD void bfly2_trivial(uint2& a, uint2& b)
{
    const uint2 t = canon2(b);
    b.x = gf::subl(a.x, t.x); a.x = gf::addl(a.x, t.x);
    b.y = gf::subl(a.y, t.y); a.y = gf::addl(a.y, t.y);
}

struct ThreadPos { uint32_t q2, j, q2log; };
template <int NT = kThreads>
FECC_HD ThreadPos thread_pos(uint32_t LR, uint32_t tid)
{
    ThreadPos t; t.q2log = Geom<NT>::logw - 1 - LR; t.q2 = tid & ((1u << t.q2log) - 1u); t.j = tid >> t.q2log; return t;
}

// Slot bookkeeping of one thread in one round.
struct RoundCtx {
    uint32_t lb, blo, bhi;    // bits [lb, lb+5) are in-thread; the stages of bits [blo, bhi) are executed
    uint32_t jbase;           // slot index with the in-thread bits zero
    uint32_t jlow;            // low lb bits of j (= low lb bits of every slot of this thread)
};
FECC_HD RoundCtx make_round(uint32_t LR, uint32_t k, uint32_t j)
{
    RoundCtx c;
    if (k == 0) { c.lb = 0; c.blo = 0; c.bhi = LR < (uint32_t)kStages ? LR : (uint32_t)kStages; }
    else        { c.lb = LR - kStages; c.blo = kStages; c.bhi = LR; }
    c.jlow  = j & ((1u << c.lb) - 1u);
    c.jbase = ((j >> c.lb) << (c.lb + kStages)) | c.jlow;
    return c;
}

struct RoundRegs { uint2 x[kRows]; };

// Stage BETA of a round (pairs differing in in-thread bit BETA).  BETA is a template parameter so that both loops have
// compile-time trip counts: for sm_90a the front end leaves a loop of (16 >> beta) trips rolled when beta comes from an
// enclosing unrolled loop, and the 32 slots then live in local memory instead of registers.
template <bool BREV, int BETA>
FECC_HD void stage_compute(uint2 (&x)[kRows], const RoundCtx& c, const uint4* tb, uint32_t sb)
{
    const uint32_t b = c.lb + BETA;
    if (b >= c.blo && b < c.bhi) {
        const uint4* twp = tb + (sb << BETA);           // heap entry 2^b + jlow (+ m * 2^lb)
#pragma unroll
        for (int m = 0; m < (1 << BETA); ++m) {
            const uint4 w = *twp; twp += sb;
#pragma unroll
            for (int hi = 0; hi < (16 >> BETA); ++hi) {
                const int i0 = (hi << (BETA + 1)) | m;
                const int i1 = i0 | (1 << BETA);
                bfly2(x[BREV ? brev5(i0) : i0], x[BREV ? brev5(i1) : i1], w);
            }
        }
    }
}

// Up to five radix-2 DIT stages on the thread's 32 slots x 2 words.  tw points at the heap-ordered stage table of the
// current transform (shared memory on the device).  BREV: the registers are numbered in the order of the PREVIOUS
// transform's last round (fused tiles): this transform's slot i is register brev5(i).
template <bool BREV>
FECC_HD void round_compute(uint2 (&x)[kRows], const RoundCtx& c, const uint4* tw)
{
    const uint32_t sb = 1u << c.lb;                     // table stride between consecutive in-thread twiddles
    const uint4* tb = tw + c.jlow;
    stage_compute<BREV, 0>(x, c, tb, sb);
    stage_compute<BREV, 1>(x, c, tb, sb);
    stage_compute<BREV, 2>(x, c, tb, sb);
    stage_compute<BREV, 3>(x, c, tb, sb);
    stage_compute<BREV, 4>(x, c, tb, sb);
}

// Stage BETA >= 1 of round0_plain (compile-time BETA for the reason given at stage_compute)
template <int BETA>
FECC_HD void stage0_plain(uint2 (&x)[kRows], const RoundCtx& c, const uint4* tw)
{
    if ((uint32_t)BETA < c.bhi) {
        const uint4* twb = tw + (1u << BETA);
#pragma unroll
        for (int m = 0; m < (1 << BETA); ++m) {
            uint4 w = {0, 0, 0, 0};
            if (m) w = twb[m];
#pragma unroll
            for (int hi = 0; hi < (16 >> BETA); ++hi) {
                const int i0 = (hi << (BETA + 1)) | m;
                const int i1 = i0 | (1 << BETA);
                if (m) bfly2(x[i0], x[i1], w); else bfly2_trivial(x[i0], x[i1]);
            }
        }
    }
}

// Round 0 of a PLAIN transform (no input twist): the twiddle of every pair whose low bits are zero is 1, which is
// known at compile time because lb = 0 makes the table index depend on the in-thread index only (31 of the 80
// butterflies of a full round).  The uniform pre-scale by 1/N (RS.cpp:51,54) is folded into stage 0, whose 16
// butterflies then cost two products each instead of one product plus two pre-scale products.
FECC_HD void round0_plain(uint2 (&x)[kRows], const RoundCtx& c, const uint4* tw, bool prescale, uint32_t pw, uint32_t pwp_lo, uint32_t pwp_hi)
{
#pragma unroll
    for (int hi = 0; hi < 16; ++hi) {                       // stage 0: all twiddles are 1
        uint2& a = x[2 * hi]; uint2& b = x[2 * hi + 1];
        if (prescale) {
            a.x = gf::mul_h(a.x, pw, pwp_lo, pwp_hi); a.y = gf::mul_h(a.y, pw, pwp_lo, pwp_hi);
            b.x = gf::mul_h(b.x, pw, pwp_lo, pwp_hi); b.y = gf::mul_h(b.y, pw, pwp_lo, pwp_hi);
            uint32_t t;
            t = b.x; b.x = gf::subl(a.x, t); a.x = gf::addl(a.x, t);
            t = b.y; b.y = gf::subl(a.y, t); a.y = gf::addl(a.y, t);
        } else {
            bfly2_trivial(a, b);
        }
    }
    stage0_plain<1>(x, c, tw);
    stage0_plain<2>(x, c, tw);
    stage0_plain<3>(x, c, tw);
    stage0_plain<4>(x, c, tw);
}

FECC_HD void prescale_all(uint2 (&x)[kRows], uint32_t w, uint32_t wp_lo, uint32_t wp_hi)
{
#pragma unroll
    for (int i = 0; i < kRows; ++i) { x[i].x = gf::mul_h(x[i].x, w, wp_lo, wp_hi); x[i].y = gf::mul_h(x[i].y, w, wp_lo, wp_hi); }
}

// P.xf[xfi] with a runtime xfi would make the compiler copy the kernel parameters to local memory
FECC_HD Xform get_xf(const PassParams& P, uint32_t xfi)
{
    Xform x;
    x.z  = xfi ? P.xf[1].z  : P.xf[0].z;
    x.t0 = xfi ? P.xf[1].t0 : P.xf[0].t0;
    x.t1 = xfi ? P.xf[1].t1 : P.xf[0].t1;
    return x;
}

} // namespace fecc

// ---------------------------------------------------------------------------------------------------------------
// Per-thread steps of a tile.  The kernel (ntt_pass.cu) runs them with block barriers in between; the CPU
// emulation (tests/emulate_tile.cu, tests/emulate_wide.cu) runs each step for tid = 0..NT-1 in turn, which is
// equivalent because within a step a thread only touches its own slots.
// ---------------------------------------------------------------------------------------------------------------
namespace fecc {

FECC_HD void copy16(uint4* dst_smem, const uint4* src_gmem)
{
#if defined(__CUDA_ARCH__)
    uint32_t s = (uint32_t)__cvta_generic_to_shared(dst_smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(s), "l"(src_gmem));
#else
    *dst_smem = *src_gmem;
#endif
}

// Entry idx (1 <= idx < R) of the heap-ordered stage table of transform xfi for row set `set`: an index into the
// global power table g^e.  Used by build_tables_kernel (device) and by the CPU emulation.
FECC_HD uint32_t table_entry_exponent(const PassParams& P, uint32_t xfi, uint32_t set, uint32_t idx)
{
    const Xform xf = get_xf(P, xfi);
    const uint32_t t = (xf.t0 + set * xf.t1) & (gf::M - 1);
    return table_exponent(idx, P.log_r, xf.z, t);
}

// 16-byte cp.async fallback loader (LR == 5, or FASTECC_B200_NO_TMA=1): tile row p <- source row p of the set,
// natural order.  Thread tid moves chunks c = tid + NT*m.
template <int NT = kThreads>
FECC_HD void load_tile_cpasync(const PassParams& P, uint32_t set, uint32_t strip, uint32_t tid, uint4* tile)
{
    const uint32_t LR = P.log_r, qlog = Geom<NT>::logw - 2 - LR, Q = 1u << qlog;
    const uint32_t p0 = tid >> qlog, qq = tid & (Q - 1);
    const uint32_t gcol = strip * Q + qq;
    const uint32_t prow = (uint32_t)NT >> qlog;                       // tile rows covered by one sweep of the CTA
    if (gcol >= P.s4) {                                               // beyond the row: keep the tile defined (TMA zero-fills)
#pragma unroll
        for (int m = 0; m < 16; ++m) tile[tid + (uint32_t)NT * m] = make_uint4(0, 0, 0, 0);
        return;
    }
    const uint32_t row0 = set * P.src_set_stride + p0 * P.src_row_stride;
    const uint4* g = reinterpret_cast<const uint4*>(P.src) + ((size_t)row0 * P.pitch4 + gcol);
    const size_t gstep = (size_t)prow * P.src_row_stride * P.pitch4;
#pragma unroll
    for (int m = 0; m < 16; ++m) { copy16(tile + tid + (uint32_t)NT * m, g); g += gstep; }
}
// ... and the set's precomputed stage tables (a contiguous nxf*R*16-byte block)
template <int NT = kThreads>
FECC_HD void load_tables_cpasync(const PassParams& P, uint32_t set, uint32_t tid, uint4* tabs)
{
    const uint32_t n = P.nxf << P.log_r;
    const uint4* src = P.tables + (size_t)set * P.table_set_stride;
    for (uint32_t i = tid; i < n; i += NT) copy16(tabs + i, src + i);
}

// word pairs per tile row (the column width of a strip)
template <int NT = kThreads>
FECC_HD uint32_t strip_pairs(uint32_t LR) { return (1u << (Geom<NT>::logw - 1)) >> LR; }

template <int NT = kThreads>
FECC_HD bool thread_active(const PassParams& P, uint32_t tid, uint32_t strip)
{
    const ThreadPos tp = thread_pos<NT>(P.log_r, tid);
    const uint32_t words2 = strip * strip_pairs<NT>(P.log_r) + tp.q2;     // word-pair column inside the row
    return (words2 >> 1) < P.s4;                                          // partial last strip: beyond the row's last chunk
}

// The strip layout of a pass in geometry NT, the one copy of the rule (plan.h's base_pass() lays passes out for the narrow
// geometry; the launcher re-lays a pass it runs wide): strips of the tile's row width, and 4 consecutive strips of a set per
// work item where that divides evenly (table reuse; tile_decode in ntt_pass.cu needs strips_per_item to divide nstrips).
template <int NT>
FECC_HD void set_strips(PassParams& P)
{
    const uint32_t Q = (uint32_t)Geom<NT>::chunks >> P.log_r;       // 16-byte chunks per tile row
    P.nstrips = (P.s4 + Q - 1) / Q;
    P.strips_per_item = (P.nstrips >= 16 && P.nstrips % 4 == 0) ? 4 : 1;
}

// Tile address (in uint2 units) of the thread's slot i in round c:  physical row = bitrev(slot) for the first
// transform of a tile (brev), = slot for the second.  Both reduce to "base + i*step" with compile-time i.
// (Narrow tiles of 1024 rows have 64-byte rows and three of their four access patterns are 2-way bank conflicted; the
// wide geometry gives the same rows 128 bytes and is conflict-free, tools/banksim_cta.py.  The fused pass runs wide.)
#define FECC_SLOT_LOOP(ACCESS)                                                                                     \
    if (brev) {                                                                                                    \
        uint32_t a = (bitrev(c.jbase, LR) << tp.q2log) | tp.q2;                                                    \
        const uint32_t step = 1u << (LR - kStages - c.lb + tp.q2log);                                              \
        _Pragma("unroll") for (int k = 0; k < kRows; ++k) { ACCESS(brev5(k), a); a += step; }                      \
    } else {                                                                                                       \
        uint32_t a = (c.jbase << tp.q2log) | tp.q2;                                                                \
        const uint32_t step = 1u << (c.lb + tp.q2log);                                                             \
        _Pragma("unroll") for (int i = 0; i < kRows; ++i) { ACCESS(i, a); a += step; }                             \
    }

// (a) read the thread's 32 slots of a step.  brev = bit-reversed placement (every round of the FIRST transform).
template <int NT = kThreads>
FECC_HD void round_read(const PassParams& P, uint32_t k, uint32_t brev, uint32_t tid, const uint4* tile, RoundRegs& r)
{
    const uint32_t LR = P.log_r;
    const ThreadPos tp = thread_pos<NT>(LR, tid);
    const RoundCtx c = make_round(LR, k, tp.j);
    const uint2* t2 = reinterpret_cast<const uint2*>(tile);
#define FECC_RD(I, A) r.x[I] = t2[A]
    FECC_SLOT_LOOP(FECC_RD)
#undef FECC_RD
}

// (b) the butterflies of a step
template <int NT = kThreads>
FECC_HD void round_math(const PassParams& P, const Step st, uint32_t tid, uint32_t set, const uint4* tw0, const uint4* tw1, RoundRegs& r)
{
    const uint32_t LR = P.log_r;
    const ThreadPos tp = thread_pos<NT>(LR, tid);
    const RoundCtx c = make_round(LR, st.k, tp.j);
    const bool first = (st.xfi == 0 && st.k == 0);
    const Xform xf = get_xf(P, st.xfi);
    const bool plain = ((xf.t0 + set * xf.t1) & (gf::M - 1)) == 0;
    const uint4* tw = st.xfi ? tw1 : tw0;
    // The plain-round shortcut only in single-transform kernels (P.nxf is a compile-time constant there): in the fused kernel it would
    // serve row set 0 and the small one-pass encodes, and its 1800 instructions between the two five-stage bodies cost the headline
    // pass 3 % (instruction supply, DESIGN.md section 6).  A plain transform through round_compute is the same arithmetic with
    // table entries equal to 1.
    if (st.k == 0 && plain && P.nxf == 1) {
        round0_plain(r.x, c, tw, first && P.prescale, P.pw, P.pwp_lo, P.pwp_hi);
    } else {
        if (first && P.prescale) prescale_all(r.x, P.pw, P.pwp_lo, P.pwp_hi);
        round_compute<false>(r.x, c, tw);
    }
    if (st.fused) {                                     // round 0 of the second transform on the same registers
        const RoundCtx c1 = make_round(LR, 0, 0);       // lb = 0: no dependence on the thread's position
        round_compute<true>(r.x, c1, tw1);
    }
}

// (c) write back in place ...
template <int NT = kThreads>
FECC_HD void round_write_tile(const PassParams& P, uint32_t k, uint32_t brev, uint32_t tid, uint4* tile, const RoundRegs& r)
{
    const uint32_t LR = P.log_r;
    const ThreadPos tp = thread_pos<NT>(LR, tid);
    const RoundCtx c = make_round(LR, k, tp.j);
    uint2* t2 = reinterpret_cast<uint2*>(tile);
#define FECC_WR(I, A) t2[A] = r.x[I]
    FECC_SLOT_LOOP(FECC_WR)
#undef FECC_WR
}

// ... or (last step) store output element r to its global row.  After a fused step that is also the last step
// (LR <= 5) register brev5(i) holds output element i of the second transform.  Eight rotating pointers whose
// increments are hidden from the optimiser: a store keeps its address registers busy until the LSU has taken
// it, so one incrementing pointer would serialise the 32 stores on the long scoreboard.
FECC_HD void opaque_advance(uint2*& p, size_t bytes)
{
#if defined(__CUDA_ARCH__)
    asm volatile("add.u64 %0, %0, %1;" : "+l"(p) : "l"(bytes));
#else
    p = reinterpret_cast<uint2*>(reinterpret_cast<char*>(p) + bytes);
#endif
}
FECC_HD void store_global2(uint2* p, uint2 v)
{
#if defined(__CUDA_ARCH__)
    asm volatile("st.global.v2.u32 [%0], {%1, %2};" :: "l"(p), "r"(v.x), "r"(v.y) : "memory");   // the opaque pointer arithmetic hides the address space
#else
    *p = v;
#endif
}
template <int NT = kThreads>
FECC_HD void round_write_global(const PassParams& P, const Step st, uint32_t tid, uint32_t set, uint32_t strip, RoundRegs& r)
{
    const ThreadPos tp = thread_pos<NT>(P.log_r, tid);
    // the last step is the fused one only when a fused tile has a single round (LR <= 5): compile-time in the kernel
    const bool fused_last = (P.nxf == 2) && (num_rounds(P.log_r) == 1);
    const RoundCtx c = fused_last ? make_round(P.log_r, 0, 0) : make_round(P.log_r, st.k, tp.j);
    const uint32_t gcol2 = strip * strip_pairs<NT>(P.log_r) + tp.q2;
    // sharded, exchange fused into the stores: this thread's output elements jbase + (i << lb) all have the same residue
    // mod G (plan.h guarantees lb >= log_g), i.e. one destination GPU per thread, chosen here once per tile
    uint32_t* base = P.dst;
    uint32_t jb = c.jbase;
    if (P.log_g) {
        const uint32_t m = jb & ((1u << P.log_g) - 1u);
        base = m == 0 ? P.peers[0] : m == 1 ? P.peers[1] : m == 2 ? P.peers[2] : m == 3 ? P.peers[3]
             : m == 4 ? P.peers[4] : m == 5 ? P.peers[5] : m == 6 ? P.peers[6] : P.peers[7];
        jb >>= P.log_g;
    }
    const uint32_t row0 = P.dst_row_offset + set * P.dst_set_stride + jb * P.dst_row_stride;
    uint2* g0 = reinterpret_cast<uint2*>(base) + ((size_t)row0 * P.pitch4 * 2 + gcol2);
    const size_t gstep = ((((size_t)P.dst_row_stride * P.pitch4 * 2) << c.lb) >> P.log_g) * sizeof(uint2);      // bytes between slots
    uint2* gp[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) { gp[u] = g0; opaque_advance(gp[u], gstep * u); }
    // every pass stores canonical residues (two ALU instructions per word, in place): only the last pass needs it,
    // but a run-time choice would cost a select and a register copy per word in front of each store
#pragma unroll
    for (int i = 0; i < kRows; ++i) {
        const int reg = fused_last ? brev5(i) : i;
        r.x[reg] = canon2(r.x[reg]);
        store_global2(gp[i & 7], r.x[reg]);
        if (i + 8 < kRows) opaque_advance(gp[i & 7], gstep * 8);
    }
}

} // namespace fecc
