// CPU emulation of ntt_pass_kernel in a chosen tile geometry (test infrastructure): runs the per-thread step functions of
// ntt_tile.cuh for tid = 0..NT-1 in turn on a Geom<NT> tile, after re-laying the pass's strips for that geometry the way
// launch_pass (ntt_pass.cu) does.  emulate_pass.h is the narrow-geometry emulation the other tests use.
#pragma once
#include <vector>
#include <algorithm>
#include "plan.h"
using namespace fecc;

template <int NT>
static void emulate_pass_geom(PassParams P)
{
    const uint32_t R = 1u << P.log_r;
    if (NT != kThreads) set_strips<NT>(P);
    // per-set stage tables, as build_tables_kernel writes them
    const uint32_t nst = table_sets(P);
    std::vector<uint4> tables((size_t)nst * P.nxf * R);
    for (uint32_t set = 0; set < nst; ++set) for (uint32_t x = 0; x < P.nxf; ++x) for (uint32_t idx = 0; idx < R; ++idx)
        tables[((size_t)set * P.nxf + x) * R + idx] = idx ? stage_entry(P.tw[table_entry_exponent(P, x, set, idx)]) : make_uint4(0, 0, 0, 0);
    P.tables = tables.data();
    P.table_set_stride = nst > 1 ? (P.nxf << P.log_r) : 0u;

    std::vector<uint4> tile(Geom<NT>::chunks), tabs(2 * R);
    const uint32_t groups = (P.nstrips + P.strips_per_item - 1) / P.strips_per_item;
    const uint32_t nitems = P.nsets * groups;
    const uint32_t nsteps = num_steps(P.log_r, P.nxf);
    std::vector<RoundRegs> regs(NT);
    for (uint32_t item = 0; item < nitems; ++item) {
        const uint32_t set = item / groups, sg = item - set * groups;
        const uint32_t strip0 = sg * P.strips_per_item;
        const uint32_t strip1 = std::min(strip0 + P.strips_per_item, P.nstrips);
        for (uint32_t strip = strip0; strip < strip1; ++strip) {
            for (auto& c : tile) c = make_uint4(0xDEADBEEF, 0xDEADBEEF, 0xDEADBEEF, 0xDEADBEEF);
            for (uint32_t tid = 0; tid < (uint32_t)NT; ++tid) load_tile_cpasync<NT>(P, set, strip, tid, tile.data());
            if (strip == strip0)
                for (uint32_t tid = 0; tid < (uint32_t)NT; ++tid) load_tables_cpasync<NT>(P, set, tid, tabs.data());
            for (uint32_t s = 0; s < nsteps; ++s) {
                const Step st = step_of(P.log_r, P.nxf, s);
                const bool last = s + 1 == nsteps;
                for (uint32_t tid = 0; tid < (uint32_t)NT; ++tid)
                    if (thread_active<NT>(P, tid, strip)) round_read<NT>(P, st.k, st.xfi == 0, tid, tile.data(), regs[tid]);
                for (uint32_t tid = 0; tid < (uint32_t)NT; ++tid) {
                    if (!thread_active<NT>(P, tid, strip)) continue;
                    round_math<NT>(P, st, tid, set, tabs.data(), tabs.data() + R, regs[tid]);
                    if (last) round_write_global<NT>(P, st, tid, set, strip, regs[tid]);
                    else      round_write_tile<NT>(P, st.k, st.xfi == 0, tid, tile.data(), regs[tid]);
                }
            }
        }
    }
}

// The geometry launch_pass picks for a pass that loads by TMA (tile height >= 64 rows, single GPU).  all_wide: every pass in
// the wide geometry, whatever the launcher picks (exercises the index arithmetic at every tile height).
static void emulate_pass_launched(const PassParams& P, bool all_wide)
{
    const bool wide = all_wide || (P.log_r >= 6 && pass_threads((int)P.log_r, (int)P.nxf, 1) == kWideThreads);
    if (wide) emulate_pass_geom<kWideThreads>(P); else emulate_pass_geom<kThreads>(P);
}
