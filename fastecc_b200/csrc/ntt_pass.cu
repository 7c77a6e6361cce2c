// The sm_90a pass kernel: one launch = one pass of the four-step / MFA decomposition (MFA_NTT, ntt.cpp:382-447)
// over the whole [N][SIZE] array, or -- with two transforms fused on a tile -- the end of the inverse transform,
// the RS scaling (RS.cpp:51-59) and the start of the forward transform in a single pass.
//
// Execution model (DESIGN.md section 5): persistent CTAs of 256 threads, two per SM, each walking a sequence of
// 64 KiB tiles (row set x column strip); the 1024-row passes and the fused 512-row pass instead run one CTA of 512 threads
// per SM over 128 KiB tiles with rows of at least 128 bytes (pass_threads() in ntt_tile.cuh).  Per tile:
//   * one elected thread issues the TMA traffic: cp.async.bulk.tensor (3-D tensor map over [word][row-in-set][set],
//     boxes of <= 256 rows) for the tile and, when the row set changes, one cp.async.bulk for the set's precomputed
//     twiddle tables; completion is tracked by an mbarrier (expect_tx / complete_tx).  The next tile is requested
//     right after the current tile's last step has pulled its slots into registers, so it flies under a full
//     five-stage round of butterflies; out-of-range columns are zero-filled by the TMA unit;
//   * ceil(LR/5) <= 2 register rounds of up to five radix-2 stages (three for a fused two-transform tile, whose
//     middle round runs 4+5 stages back to back in registers) separated by one block barrier each;
//   * 64-bit stores of the finished rows straight from registers.
// The kernel is bound by instruction issue (XU conversions + FP64 / integer multiplies + the lazy add/sub), not by HBM: DESIGN.md section 6.
#include "ntt_tile.cuh"
#include "ntt_pass.h"
#include "plan.h"
#include <cstring>
#include <cstdlib>
#include <cstdio>
#include <cuda.h>
#include <cuda_runtime.h>

namespace fecc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}"
        :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, uint32_t c0, uint32_t c1, uint32_t c2)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 :: "r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// The CTA's t-th tile.  Work items (a row set x strips_per_item consecutive strips) are dealt round-robin to the
// CTAs; plan.h guarantees strips_per_item divides nstrips, so tile t of a CTA is strip (t % spi) of its (t / spi)-th item.
__device__ __forceinline__ bool tile_decode(const PassParams& P, uint32_t groups, uint32_t nitems, uint32_t t, uint32_t& set, uint32_t& strip)
{
    const uint32_t spi = P.strips_per_item;
    const uint32_t item = blockIdx.x + (t / spi) * gridDim.x;
    if (item >= nitems) return false;
    set = item / groups;
    strip = (item - set * groups) * spi + (t % spi);
    return true;
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory"); }

// LR / NXF / TMA are compile-time: the kernel patches them into its copy of the parameters, so every shift, stride
// and placement branch in ntt_tile.cuh folds to an immediate (keeps the 64 data registers from spilling).  NT is the
// geometry, pass_threads(LR, NXF, TMA): 256 threads (2 CTAs per SM, 64 KiB tiles) or 512 (1 CTA per SM, 128 KiB tiles);
// either way 16 warps per SM at 128 registers.
template <int LR, int NXF, int TMA, int NT>
__global__ void __launch_bounds__(NT, NT == kWideThreads ? 1 : 2) ntt_pass_kernel(const PassParams Pin, const __grid_constant__ CUtensorMap tmap)
{
    PassParams P = Pin;
    P.log_r = LR; P.nxf = NXF; P.use_tma = TMA != 0;
    if (TMA != 2) P.log_g = 0;                            // TMA == 2: the instantiation whose stores pick a destination GPU (sharded, §8)
    extern __shared__ __align__(1024) uint4 smem[];
    constexpr uint32_t R = 1u << LR;
    constexpr uint32_t kChunks = Geom<NT>::chunks;
    uint4* tile = smem;                                   // kChunks chunks, natural row order
    // stage tables: a transform whose twist does not depend on the row set (t1 == 0) has ONE table, loaded once;
    // the others are double-buffered per set.  Slot of transform x in buffer b: tabs + (b*NXF + x)*R; set-independent
    // tables always use b = 0 (so a fused BC tile needs 3 slots, a plain A tile 1).  The two mbarriers sit between the
    // tile and the tables, at an address known at compile time (one register fewer to keep live across the tile loop).
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + kChunks);
    uint4* tabs = smem + kChunks + 1;
    const bool var0 = P.xf[0].t1 != 0, var1 = NXF == 2 && P.xf[1].t1 != 0;
    const uint32_t tid  = threadIdx.x;
    const uint32_t groups = (P.nstrips + P.strips_per_item - 1) / P.strips_per_item;
    const uint32_t nitems = P.nsets * groups;
    constexpr uint32_t nsteps = NXF == 2 ? (LR > kStages ? 3u : 1u) : (LR > kStages ? 2u : 1u);
    constexpr uint32_t kWt = (1u << Geom<NT>::logw) >> LR;   // words per tile row
    constexpr uint32_t kRowsBox = R < 256u ? R : 256u;    // TMA box: kRowsBox rows x kWt words
    constexpr uint32_t kBoxes = R / kRowsBox;

    uint32_t cur_set, cur_strip;
    if (!tile_decode(P, groups, nitems, 0, cur_set, cur_strip)) return;
    uint32_t tb = 0;                                      // table buffer used by the current tile
    uint32_t phase = 0;
    uint64_t* rbar = bar + 1;                             // "every warp has pulled the last step's slots into registers"

    // request tile (set, strip) [+ the set's tables into buffer tbuf]
    auto request = [&](uint32_t set, uint32_t strip, bool with_tables, uint32_t tbuf) {
        if (TMA) {
            if (tid == 0) {
                fence_proxy_async();                      // order our earlier generic-proxy accesses to the tile before the async-proxy writes
                const bool first = with_tables && tbuf == 2u;         // prologue: also the set-independent tables
                const uint32_t ld0 = with_tables && (var0 || first), ld1 = NXF == 2 && with_tables && (var1 || first);
                mbar_expect_tx(bar, Geom<NT>::bytes + (ld0 + ld1) * (R * 16u));
#pragma unroll
                for (uint32_t b = 0; b < kBoxes; ++b)
                    tma_load_3d(tile + b * (kRowsBox * (kWt / 4)), &tmap, bar, strip * kWt, b * kRowsBox, set);
                const uint4* tsrc = P.tables + (size_t)set * P.table_set_stride;
                const uint32_t tbv = first ? 0u : tbuf;
                if (ld0) bulk_load(tabs + ((var0 ? tbv : 0u) * NXF + 0) * R, tsrc, R * 16u, bar);
                if (ld1) bulk_load(tabs + ((var1 ? tbv : 0u) * NXF + 1) * R, tsrc + R, R * 16u, bar);
            }
        } else {
            load_tile_cpasync<NT>(P, set, strip, tid, tile);
            if (with_tables) {
                const bool first = tbuf == 2u;
                const uint32_t tbv = first ? 0u : tbuf;
                const uint4* tsrc = P.tables + (size_t)set * P.table_set_stride;
                if (var0 || first) for (uint32_t i = tid; i < R; i += NT) copy16(tabs + ((var0 ? tbv : 0u) * NXF + 0) * R + i, tsrc + i);
                if (NXF == 2 && (var1 || first)) for (uint32_t i = tid; i < R; i += NT) copy16(tabs + ((var1 ? tbv : 0u) * NXF + 1) * R + i, tsrc + R + i);
            }
        }
    };

    if (TMA) {
        if (tid == 0) { mbar_init(bar, 1); mbar_init(rbar, NT / 32); fence_mbar_init(); }
        __syncthreads();
    }
    request(cur_set, cur_strip, true, 2u);                // prologue: first tile + all its tables (buffer 0)

    for (uint32_t t = 0;; ++t) {
        if (TMA) mbar_wait(bar, phase);
        else     { cp_async_wait_all(); __syncthreads(); }
        const bool active = thread_active<NT>(P, tid, cur_strip);
        RoundRegs r;
        // pass_unrolled() (ntt_tile.cuh): the wide passes unroll their steps, at the same 128 registers without spills; the
        // fused ones run about 7 % faster so, the single-transform one about 4 % (DESIGN.md section 6).
#pragma unroll (pass_unrolled(LR, NXF, TMA) ? nsteps : 1)
        for (uint32_t s = 0; s < nsteps; ++s) {
            const Step st = step_of(LR, NXF, s);
            const bool last = s + 1 == nsteps;
            if (active) round_read<NT>(P, st.k, st.xfi == 0, tid, tile, r);
            if (last) {                                   // every slot is in registers: the tile buffer is free.
                if (TMA) {                                // each warp reports in; only the issuing thread waits for all of them
                    __syncwarp();
                    if ((tid & 31) == 0) mbar_arrive(rbar);
                    if (tid == 0) {                       // the next tile flies under the last step's butterflies
                        mbar_wait(rbar, phase);
                        uint32_t ns, nst;
                        if (tile_decode(P, groups, nitems, t + 1, ns, nst)) request(ns, nst, ns != cur_set, tb ^ 1u);
                    }
                } else {
                    __syncthreads();
                    uint32_t ns, nst;
                    if (tile_decode(P, groups, nitems, t + 1, ns, nst)) request(ns, nst, ns != cur_set, tb ^ 1u);
                }
            }
            const uint4* tw0 = tabs + ((var0 ? tb : 0u) * NXF) * R;
            const uint4* tw1 = tabs + ((var1 ? tb : 0u) * NXF + 1) * R;
            #if !defined(FECC_SKIP_MATH)                                   // -DFECC_SKIP_MATH: copy-only build for measuring the memory floor of a pass
            if (active) round_math<NT>(P, st, tid, cur_set, tw0, tw1, r);
#endif
            if (!last) {
                if (active) round_write_tile<NT>(P, st.k, st.xfi == 0, tid, tile, r);
                __syncthreads();
            } else if (active) {
                round_write_global<NT>(P, st, tid, cur_set, cur_strip, r);
            }
        }
        uint32_t nxt_set, nxt_strip;                      // (re)decoded here, where registers are plentiful
        if (!tile_decode(P, groups, nitems, t + 1, nxt_set, nxt_strip)) break;
        phase ^= 1u;
        if (nxt_set != cur_set) tb ^= 1u;
        cur_set = nxt_set; cur_strip = nxt_strip;
    }
}


// One thread per table entry: tables[set][xfi][idx] = g^exponent (entry 0 of every table is unused).
__global__ void build_tables_kernel(const PassParams P, uint4* out, uint32_t nsets_tab)
{
    const uint32_t R = 1u << P.log_r;
    const size_t total = (size_t)nsets_tab * P.nxf * R;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t idx = (uint32_t)(i & (R - 1));
        const uint32_t xfi = (uint32_t)((i >> P.log_r) % P.nxf);
        const uint32_t set = (uint32_t)((i >> P.log_r) / P.nxf);
        out[i] = idx ? stage_entry(P.tw[table_entry_exponent(P, xfi, set, idx)]) : make_uint4(0, 0, 0, 0);
    }
}

cudaError_t launch_build_tables(PassParams& P, uint4* out, cudaStream_t stream)
{
    const uint32_t ns = table_sets(P);
    P.tables = out;
    P.table_set_stride = ns > 1 ? (P.nxf << P.log_r) : 0u;
    build_tables_kernel<<<528, 256, 0, stream>>>(P, out, ns);        // 4 CTAs per SM of an H100 (132 SMs), grid-stride
    return cudaGetLastError();
}

// shared memory of the CTA-level kernel: tile + two mbarriers + table slots.  Table slot of transform x in buffer b is
// (b*nxf + x); buffer 1 is needed only up to the last set-dependent transform.
size_t pass_smem_bytes(const PassParams& P, uint32_t tile_bytes)
{
    uint32_t slots = P.nxf;                                            // buffer 0
    if (P.nxf == 2 && P.xf[1].t1) slots = 4; else if (P.xf[0].t1) slots = P.nxf + 1;
    return (size_t)tile_bytes + (size_t)slots * ((size_t)16 << P.log_r) + 16;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled()
{
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr; cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// 3-D view of the source buffer: [word][row within set][set]; box = one tile row strip of <= 256 rows, of the tile's
// row width (tile_words / R words).
static bool make_tensor_map(const PassParams& P, uint32_t tile_words, CUtensorMap* map)
{
    EncodeTiledFn enc = encode_tiled();
    if (!enc) return false;
    const uint32_t R = 1u << P.log_r, Wt = tile_words >> P.log_r;
    if (Wt > 256) return false;
    const cuuint64_t row_bytes = (cuuint64_t)P.pitch4 * 16;
    cuuint64_t gdim[3] = {(cuuint64_t)P.s4 * 4, R, P.nsets};
    cuuint64_t gstr[2] = {(cuuint64_t)P.src_row_stride * row_bytes, P.nsets > 1 ? (cuuint64_t)P.src_set_stride * row_bytes : (cuuint64_t)P.src_row_stride * row_bytes * R};
    cuuint32_t box[3] = {Wt, R < 256u ? R : 256u, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    if (gstr[0] >= (1ull << 40) || gstr[1] >= (1ull << 40)) return false;
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, (void*)P.src, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int LR, int NXF, int TMA, int NT = pass_threads(LR, NXF, TMA)>
static cudaError_t launch_inst(const PassParams& P, const CUtensorMap& map, unsigned grid, cudaStream_t stream)
{
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(ntt_pass_kernel<LR, NXF, TMA, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             Geom<NT>::bytes + 2 * NXF * (16 << LR) + 16);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(ntt_pass_kernel<LR, NXF, TMA, NT>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    ntt_pass_kernel<LR, NXF, TMA, NT><<<grid, NT, pass_smem_bytes(P, Geom<NT>::bytes), stream>>>(P, map);
    return cudaGetLastError();
}

// the TMA instantiation of a single-GPU pass in geometry nt (the narrow twin where pass_has_narrow_twin)
template <int LR, int NXF>
static cudaError_t launch_tma(const PassParams& P, const CUtensorMap& map, unsigned grid, cudaStream_t stream, int nt)
{
    if constexpr (pass_has_narrow_twin(LR, NXF, 1))
        if (nt == kThreads) return launch_inst<LR, NXF, 1, kThreads>(P, map, grid, stream);
    return launch_inst<LR, NXF, 1>(P, map, grid, stream);
}

// name of the instantiation a pass is dispatched to, for the per-kernel lines of the benchmark (static storage);
// wide instantiations carry their thread count (one slot per geometry: <9,2,1> and its wide sibling share lr, nxf and tma)
static const char* kernel_name(uint32_t lr, uint32_t nxf, uint32_t tma, int nt)
{
    static char names[6][3][3][2][40];
    char* n = names[lr - 5][nxf][tma][nt == kThreads ? 0 : 1];
    if (!n[0]) {
        if (nt == kThreads) snprintf(n, 40, "ntt_pass_kernel<%u,%u,%u>", lr, nxf, tma);
        else                snprintf(n, 40, "ntt_pass_kernel<%u,%u,%u,%d>", lr, nxf, tma, nt);
    }
    return n;
}

// The planner lays every pass out for the narrow geometry; the launcher picks the instantiation and, for a wide one,
// re-lays the strips of its copy of the descriptor (the plans and their CPU emulation stay geometry-free).
cudaError_t launch_pass(const PassParams& Pin, int num_sms, cudaStream_t stream, const char** kernel)
{
    PassParams P = Pin;
    if (!P.tables) return cudaErrorInvalidValue;
    static const bool no_tma = getenv("FASTECC_B200_NO_TMA") != nullptr;
    const uint32_t tmak = P.log_g ? 2u : 1u;
    int nt = !no_tma && P.log_r >= 6 ? pass_threads((int)P.log_r, (int)P.nxf, (int)tmak) : kThreads;
    if (nt == kWideThreads) set_strips<kWideThreads>(P);
    if (nt == kWideThreads && pass_has_narrow_twin((int)P.log_r, (int)P.nxf, (int)tmak) && (unsigned long long)P.nsets * P.nstrips < (unsigned)num_sms) {
        P = Pin; nt = kThreads;                                 // fewer wide tiles than SMs: the narrow twin has twice as many
    }
    CUtensorMap map;
    memset(&map, 0, sizeof map);
    const bool tma = !no_tma && P.log_r >= 6 && make_tensor_map(P, nt == kWideThreads ? 1u << Geom<kWideThreads>::logw : 1u << Geom<kThreads>::logw, &map);
    if (!tma && nt != kThreads) { P = Pin; nt = kThreads; }     // the wide instantiations load by TMA only
    if (P.log_g && !tma) return cudaErrorNotSupported;          // sharded stores exist only in the TMA instantiations

    const uint32_t groups = (P.nstrips + P.strips_per_item - 1) / P.strips_per_item;
    const unsigned long long nitems = (unsigned long long)P.nsets * groups;
    static const int ctas_per_sm = getenv("FASTECC_B200_CTAS_PER_SM") ? atoi(getenv("FASTECC_B200_CTAS_PER_SM")) : 2;   // narrow kernels
    unsigned long long grid = (unsigned long long)num_sms * (nt == kWideThreads ? 1 : ctas_per_sm > 0 ? ctas_per_sm : 2);
    if (grid > nitems) grid = nitems;
    if (grid == 0) return cudaSuccess;
    const unsigned g = (unsigned)grid;
    if (kernel) *kernel = kernel_name(P.log_r, P.nxf, tma ? tmak : 0, nt);
#define FECC_CASE(L) case L: \
        if (tma && P.log_g) return P.nxf == 2 ? launch_inst<L, 2, 2>(P, map, g, stream) : launch_inst<L, 1, 2>(P, map, g, stream); \
        if (tma) return P.nxf == 2 ? launch_tma<L, 2>(P, map, g, stream, nt) : launch_tma<L, 1>(P, map, g, stream, nt); \
        else     return P.nxf == 2 ? launch_inst<L, 2, 0>(P, map, g, stream) : launch_inst<L, 1, 0>(P, map, g, stream);
    switch (P.log_r) {
        FECC_CASE(5) FECC_CASE(6) FECC_CASE(7) FECC_CASE(8) FECC_CASE(9) FECC_CASE(10)
        default: return cudaErrorInvalidValue;
    }
#undef FECC_CASE
}

} // namespace fecc
