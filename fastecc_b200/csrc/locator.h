// The erasure locator of a 2N-row code word, shared by the two kinds of pattern (decode.cu: fastecc_b200_rs_decode_pattern*,
// repair.cu: fastecc_b200_rs_repair_pattern).  Both build l(x) = prod_{e in E} (x - rho^e), rho = GF_Root(n2), over the erased
// rows E and evaluate l and x * l'(x) at all n2 points; only what they make of those values differs.
#pragma once
#include "context.h"
#include "gf.cuh"

namespace fecc {

// rho^e, rho = GF_Root(n2), n2 = r * 2^t (r = 1, 3 or 9), split by the CRT: GF_Root(r)^(a2*e mod r) * GF_Root(2^t)^(b2*e mod 2^t),
// a2 = 2^-t mod r, b2 = r^-1 mod 2^t; GF_Root(2^t)^m = g^(m << log_step) is a power-table entry.  r = 1: a2 = 0, b2 = 1.
struct LeafRoots { uint32_t r, a2, b2, mask, log_step; uint32_t zeta[9]; };
LeafRoots leaf_roots(size_t n2);
__device__ __forceinline__ uint32_t rho_pow(const LeafRoots& L, const uint4* __restrict__ tw, uint32_t e)       // e < n2
{
    uint32_t r = tw[(size_t)((L.b2 * e) & L.mask) << L.log_step].x;
    if (L.r > 1) r = gf::mulmod(r, L.zeta[(L.a2 * (e % L.r)) % L.r]);
    return r;
}

// The n positions a[0 .. n) ascend strictly and lie below `bound`: the rule for every list of erased or lost blocks.
inline bool ascending_below(const uint32_t* a, size_t n, size_t bound)
{
    for (size_t i = 0; i < n; ++i)
        if (a[i] >= bound || (i && a[i] <= a[i - 1])) return false;
    return true;
}

// d_idx: the me >= 1 erased rows of an n2-row code word, ascending, on the device.  Builds the locator by the product tree and
// leaves two pitched single-column arrays of n2 rows of 4 words (allocated in `tmp`): lv4[m * 4] = l(rho^m) and
// dl4[m * 4] = D[m] = rho^m * l'(rho^m).  Asynchronous on `st`: the caller synchronises before `tmp` goes away.
int erasure_locator(size_t n2, const uint32_t* d_idx, size_t me, DeviceArrays& tmp, uint32_t** lv4, uint32_t** dl4, cudaStream_t st, const char* who);

}
