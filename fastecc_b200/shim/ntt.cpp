// Drop-in replacement for the reference's ntt.cpp: lets the UNMODIFIED reference drivers (main.cpp -> `ntt`,
// RS.cpp -> `rs`) run their GF(0xFFF00001) transforms on the H100 through the C ABI of include/fastecc_b200.h.
//
// The reference programs textually `#include "ntt.cpp"` (main.cpp:18, RS.cpp:18).  integration/build_dropin.sh builds
// them from a staging directory that holds symlinks to the reference sources plus THIS file under the name ntt.cpp,
// so the quote-include resolves here.  We then include the real reference ntt.cpp (never copied: its path comes
// in through -DFASTECC_REF_NTT_CPP) with MFA_NTT renamed, which keeps every generic template the drivers still
// use on the CPU (Rec_NTT, Slow_NTT, NTT3/6/9, the other three rings of main.cpp:344-358), and specialise
//     MFA_NTT<uint32_t, 0xFFF00001>(T** data, size_t N, size_t SIZE, bool InvNTT)            ntt.cpp:382-383
// to call fastecc_b200_ntt_u32().  The reference functions return void and never fail; a non-zero status from
// the GPU library is therefore fatal here -- there is no silent CPU fallback on this path.
#ifndef FASTECC_REF_NTT_CPP
#error "build with -DFASTECC_REF_NTT_CPP='\"/path/to/reference/ntt.cpp\"' (see integration/build_dropin.sh)"
#endif

#define MFA_NTT MFA_NTT_reference_cpu
#include FASTECC_REF_NTT_CPP
#undef MFA_NTT

#include <cstdio>
#include <cstdlib>
#include "fastecc_b200.h"

// every other ring keeps the reference's CPU algorithm
template <typename T, T P>
void MFA_NTT (T** data, size_t N, size_t SIZE, bool InvNTT)
{
    MFA_NTT_reference_cpu<T,P> (data, N, SIZE, InvNTT);
}

// GF(0xFFF00001): the H100
template <>
inline void MFA_NTT<uint32_t,0xFFF00001> (uint32_t** data, size_t N, size_t SIZE, bool InvNTT)
{
    static bool ready = false;
    if (!ready) {
        const char* dev = getenv("FASTECC_B200_DEVICE");
        if (fastecc_b200_init(dev ? atoi(dev) : 0) != 0) {
            fprintf(stderr, "fastecc_b200: %s\n", fastecc_b200_last_error());
            abort();
        }
        // the drivers allocate their block array once and never free it (RS.cpp:31, main.cpp:244): let the library page-lock it
        // in place on first sight (FASTECC_B200_NO_PIN=1: leave it pageable, for comparison)
        fastecc_b200_pin_host_buffers(getenv("FASTECC_B200_NO_PIN") ? 0 : 1);
        ready = true;
    }
    if (fastecc_b200_ntt_u32(data, N, SIZE, InvNTT ? 1 : 0) != 0) {
        fprintf(stderr, "fastecc_b200: %s\n", fastecc_b200_last_error());
        abort();
    }
}
