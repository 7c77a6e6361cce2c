// CPU emulation of the encode plans with the pass kernels in the geometry the launcher runs them in (the fused 1024-row
// pass on 512-thread, 128 KiB tiles), thread by thread, against the oracle.  Used by tests/test_wide_emulation.py.
// Usage: emulate_wide [all]   ("all": every pass in the wide geometry)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "plan.h"
#include "emulate_wide.h"
#include "gfp_oracle.h"

static std::vector<gf::Tw> g_tw;

// mode 0 fwd NTT, 2 encode, 3 asymmetric encode into N / dec parity blocks
static int check(const char* what, size_t N, size_t S, int mode, bool all_wide, size_t dec = 1)
{
    const size_t pitch = (S + 3) / 4 * 4;
    std::vector<uint32_t> x(N * pitch, 0), y(N * pitch, 0), ref(N * S);
    oracle_fill_B(ref.data(), N * S);
    for (size_t i = 0; i < N; i++) memcpy(&x[i * pitch], &ref[i * S], S * 4);
    Buffers b{x.data(), y.data(), reinterpret_cast<const uint4*>(g_tw.data()), (uint32_t)pitch, (uint32_t)S};
    std::vector<PassParams> plan = mode == 3 ? plan_encode_asym(b, N, N / dec) : mode == 2 ? plan_encode(b, N) : plan_ntt(b, N, false);
    for (auto& p : plan) emulate_pass_launched(p, all_wide);
    if (mode >= 2) oracle_rs_encode(ref.data(), N, S); else oracle_ntt(ref.data(), N, S, 0);
    const size_t rows = N / dec;
    size_t bad = 0;
    for (size_t i = 0; i < rows; i++) for (size_t k = 0; k < S; k++) {
        const uint32_t got = x[i * pitch + k], want = ref[i * dec * S + k];
        if (got != want) { if (!bad) printf("   first mismatch row %zu word %zu: got %u want %u\n", i, k, got, want); bad++; }
    }
    printf("%-8s N=2^%-2u S=%-5zu M=N/%zu passes=%zu : %s (%zu mismatches)\n", what, ilog2(N), S, dec, plan.size(), bad ? "FAIL" : "ok", bad);
    return bad != 0;
}

int main(int argc, char** argv)
{
    g_tw.resize(kM);
    fill_power_table(g_tw.data());
    const bool all_wide = argc > 1 && !strcmp(argv[1], "all");
    int fails = 0;
    struct Cfg { unsigned ln; size_t s; };
    // Strips: a wide 1024-row tile is 32 words wide, a wide 256-row tile 128, a wide 64-row tile 512.  The headline order's fused
    // pass (1024 rows) with one partial strip (S = 1, 17), two strips, the second partial (33), and 9 strips, the last partial
    // (257).  In the all-wide list: 8 strips of the 256-row passes, the last partial (2^16 x 1000), and 16 strips of the 64-row
    // passes in work items of 4, the last partial (2^12 x 7700).
    std::vector<Cfg> cfgs = { {5, 17}, {9, 33}, {10, 1}, {11, 17}, {11, 1000}, {12, 33}, {13, 1}, {13, 1000}, {15, 33}, {17, 17}, {19, 1}, {19, 17},
                              {19, 33}, {19, 257} };
    if (all_wide) cfgs = { {5, 1000}, {7, 33}, {8, 17}, {10, 1000}, {11, 33}, {12, 7700}, {14, 1}, {16, 17}, {16, 1000} };
    for (auto c : cfgs) {
        const size_t N = (size_t)1 << c.ln;
        const bool huge = N * c.s > ((size_t)1 << 25);       // the encode only: it runs every pass the asymmetric plans run
        fails += check("encode", N, c.s, 2, all_wide);
        if (c.ln <= 16) fails += check("ntt-fwd", N, c.s, 0, all_wide);
        if (!huge && asym_native(N, N / 2)) fails += check("asym", N, c.s, 3, all_wide, 2);
        if (!huge && asym_native(N, N / 4)) fails += check("asym", N, c.s, 3, all_wide, 4);
    }
    printf("%s\n", fails ? "EMULATION FAILED" : "EMULATION OK");
    return fails ? 1 : 0;
}
