// The 1024 x 512 split of the single-GPU plans (csrc/plan.h split_l1) and the wide geometry of their passes, on the CPU (test
// infrastructure for tests/test_split_1024.py).
// Usage: emulate_split plans   print "<plan> <log N> <G> : log_r/nxf/threads ..." with the geometry launch_pass picks per pass
//        emulate_split         forward and inverse NTTs of 2^19 and 2^20 with every pass emulated thread by thread in the
//                              geometry the launcher runs it in, against the oracle
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "plan.h"
#include "emulate_wide.h"
#include "gfp_oracle.h"

static std::vector<gf::Tw> g_tw;

static int launched_threads(const PassParams& p)
{
    return p.log_r >= 6 ? pass_threads((int)p.log_r, (int)p.nxf, p.log_g ? 2 : 1) : kThreads;
}

static void print_plan(const char* what, size_t N, uint32_t G, const std::vector<PassParams>& v)
{
    printf("%s %u %u :", what, ilog2(N), G);
    for (const PassParams& p : v) printf(" %u/%u/%d", p.log_r, p.nxf, launched_threads(p));
    printf("\n");
}

static int plans()
{
    uint32_t dummy[4] = {0, 0, 0, 0};
    Buffers b{dummy, dummy, reinterpret_cast<const uint4*>(g_tw.data()), 4, 4};
    for (unsigned ln : {11u, 16u, 18u, 19u, 20u}) {
        const size_t N = (size_t)1 << ln;
        if (ln <= 19) print_plan("encode", N, 1, plan_encode(b, N));
        print_plan("ntt", N, 1, plan_ntt(b, N, false));
        print_plan("ntt-inv", N, 1, plan_ntt(b, N, true));
        for (unsigned k : {1u, 9u, 10u}) {
            char name[16];
            snprintf(name, sizeof name, "asym%u", k);
            if (ln <= 19 && asym_native(N, N >> k)) print_plan(name, N, 1, plan_encode_asym(b, N, N >> k));
        }
        for (uint32_t G : {2u, 4u, 8u}) {
            uint32_t* peers[kMaxPeers];
            for (uint32_t r = 0; r < kMaxPeers; ++r) peers[r] = dummy;
            if (ln <= 19 && shard_p2p_supported(N, G)) {
                std::vector<PassParams> v;
                for (int which = 0; which < 3; ++which) v.push_back(plan_encode_shard_p2p(dummy, peers, b.tw, 4, 4, N, G, 0, which));
                print_plan("encode-shard-p2p", N, G, v);
            }
            if (ntt_shard_p2p_supported(N, G)) {
                std::vector<PassParams> v;
                for (int which = 0; which < 2; ++which) v.push_back(plan_ntt_shard_p2p(dummy, peers, b.tw, 4, 4, N, G, 0, false, which));
                print_plan("ntt-shard-p2p", N, G, v);
            }
        }
    }
    return 0;
}

static int check_ntt(size_t N, size_t S, bool inverse)
{
    const size_t pitch = (S + 3) / 4 * 4;
    std::vector<uint32_t> x(N * pitch, 0), y(N * pitch, 0), ref(N * S);
    oracle_fill_B(ref.data(), N * S);
    for (size_t i = 0; i < N; i++) memcpy(&x[i * pitch], &ref[i * S], S * 4);
    Buffers b{x.data(), y.data(), reinterpret_cast<const uint4*>(g_tw.data()), (uint32_t)pitch, (uint32_t)S};
    const std::vector<PassParams> plan = plan_ntt(b, N, inverse);
    for (const PassParams& p : plan) emulate_pass_launched(p, false);
    oracle_ntt(ref.data(), N, S, inverse ? 1 : 0);
    size_t bad = 0;
    for (size_t i = 0; i < N; i++) for (size_t k = 0; k < S; k++) {
        const uint32_t got = x[i * pitch + k], want = ref[i * S + k];
        if (got != want) { if (!bad) printf("   first mismatch row %zu word %zu: got %u want %u\n", i, k, got, want); bad++; }
    }
    printf("%-8s N=2^%-2u S=%-3zu passes=", inverse ? "ntt-inv" : "ntt-fwd", ilog2(N), S);
    for (const PassParams& p : plan) printf("%u/%d ", p.log_r, launched_threads(p));
    printf(": %s (%zu mismatches)\n", bad ? "FAIL" : "ok", bad);
    return bad != 0;
}

int main(int argc, char** argv)
{
    g_tw.resize(kM);
    fill_power_table(g_tw.data());
    if (argc > 1 && !strcmp(argv[1], "plans")) return plans();
    // A wide 1024-row tile and a narrow 512-row tile are both 32 words wide: S = 1 and 17 leave one partial strip, 33 two strips,
    // the second partial.  The second pass (B') of each transform has a twist that depends on the row set.
    int fails = 0;
    for (unsigned ln : {19u, 20u})
        for (size_t s : {1, 17, 33})
            for (bool inv : {false, true}) fails += check_ntt((size_t)1 << ln, s, inv);
    printf("%s\n", fails ? "EMULATION FAILED" : "EMULATION OK");
    return fails ? 1 : 0;
}
