// Encode, degraded read and update of a batch of small stripes (include/fastecc_b200.h: fastecc_b200_rs_encode_batch, DESIGN 3l,
// fastecc_b200_rs_reconstruct_batch, DESIGN 3m, and fastecc_b200_rs_update_batch, DESIGN 3n): the layout rules that decide, in
// O(N + M) host work, whether the rows a batch writes are provably disjoint from each other and from the rows it reads, and the
// one kernel launch of each call.  The rule is
// plain C++ so that a host build can check it against brute-force word sets.
#pragma once
#include <stdint.h>

namespace fecc {

// One side of a batch in words: row i of stripe b starts at word base + b * stride + i * pitch and covers SIZE words.
struct BatchRows { uint64_t base, pitch, stride, rows; };

// Whether rows [a, a + size) of `a0 + i * pitch`, i < n, and the row [x, x + size) share a word (pitch >= size, so at most two
// consecutive rows can meet it).
inline bool batch_row_hits_progression(uint64_t a0, uint64_t pitch, uint64_t n, uint64_t x, uint64_t size)
{
    if (x + size <= a0) return false;
    const uint64_t i = x < a0 + size ? 0 : (x - a0 - size) / pitch + 1;  // the first row that ends past x
    return i < n && a0 + i * pitch < x + size;
}

// Word e past the last word of a side: base + (B - 1) stride + (rows - 1) pitch + size, or 0 when it would reach 2^60 (no real
// buffer is that large, so such a layout is rejected rather than reasoned about in wider arithmetic).
inline uint64_t batch_end(const BatchRows& s, uint64_t B, uint64_t size)
{
    constexpr uint64_t kCap = 1ull << 60;
    if (s.base >= kCap || size >= kCap || (B > 1 && s.stride >= kCap / (B - 1)) || (s.rows > 1 && s.pitch >= kCap / (s.rows - 1))) return 0;
    const uint64_t e = s.base + (B - 1) * s.stride + (s.rows - 1) * s.pitch + size;
    return e < kCap ? e : 0;
}

// Whether the B x rows rows of one side are pairwise disjoint because one of its two strides nests the other: stripe-major
// (each stripe's rows fit inside one stripe stride) or block-major (each block's B rows fit inside one row pitch).
inline bool batch_side_disjoint(const BatchRows& s, uint64_t B, uint64_t size)
{
    const bool rows_apart = s.rows == 1 || s.pitch >= size, stripes_apart = B == 1 || s.stride >= size;
    return (rows_apart && (B == 1 || s.stride >= (s.rows - 1) * s.pitch + size)) || (stripes_apart && (s.rows == 1 || s.pitch >= (B - 1) * s.stride + size));
}

// The layout rule of fastecc_b200_rs_encode_batch.  Needs B >= 1, rows >= 1 on both sides, 1 <= size <= both pitches.  True only
// for layouts in which no parity word is another parity word or a data word (data rows may overlap each other), namely:
//   separate: the parity rows are pairwise disjoint (batch_side_disjoint) and the data's span [base, end) and the parity's span do
//             not meet;
//   shared:   one stripe stride for both sides (or B = 1); in stripe 0 the parity rows are pairwise disjoint and meet no data row,
//             and stripe 0's N + M rows span at most one stripe stride, so that every stripe is a translate of stripe 0 that meets
//             no other.
// Any other layout is rejected, disjoint or not.  Each test is O(1) per row: O(N + M) in all.
inline bool batch_layout_disjoint(const BatchRows& d, const BatchRows& p, uint64_t B, uint64_t size)
{
    const uint64_t de = batch_end(d, B, size), pe = batch_end(p, B, size);
    if (!de || !pe) return false;
    if (batch_side_disjoint(p, B, size) && (de <= p.base || pe <= d.base)) return true;
    if (B > 1 && d.stride != p.stride) return false;
    if (p.rows > 1 && p.pitch < size) return false;
    for (uint64_t j = 0; j < p.rows; ++j)
        if (batch_row_hits_progression(d.base, d.pitch, d.rows, p.base + j * p.pitch, size)) return false;
    if (B == 1) return true;
    const uint64_t lo = d.base < p.base ? d.base : p.base;
    const uint64_t d1 = d.base + (d.rows - 1) * d.pitch + size, p1 = p.base + (p.rows - 1) * p.pitch + size;
    return (d1 > p1 ? d1 : p1) - lo <= p.stride;
}

// The layout rule of fastecc_b200_rs_update_batch (DESIGN 3n), which writes into the stripes it reads: the rule above for the three
// pairs (new, data), (new, parity) and (data, parity).  True only when all N + M rows of all stripes are pairwise disjoint and none
// of them meets a new row (new rows may overlap each other: they are only read).  Then each word written, a changed data word or a
// parity word, is read by the one work item that writes it and by no other, so an in-place write cannot feed another item's sum.
inline bool batch_update_layout_disjoint(const BatchRows& d, const BatchRows& p, const BatchRows& n, uint64_t B, uint64_t size)
{
    return batch_layout_disjoint(n, d, B, size) && batch_layout_disjoint(n, p, B, size) && batch_layout_disjoint(d, p, B, size);
}

} // namespace fecc

#if defined(__CUDACC__)
#include "context.h"
namespace fecc {
// Parity row j of stripe b = sum_{i < N} data row i of stripe b * T[(D j - i) mod N], D = N / M, for B stripes, words [0, size)
// only, canonical; data words are taken mod P.  Rows in words as BatchRows describes them; T is fastecc_b200_rs_update's table.
// One launch.
cudaError_t launch_batch_encode(const uint32_t* data, size_t dpitch, size_t dstride, size_t N, uint32_t* parity, size_t ppitch, size_t pstride,
                                size_t M, size_t B, size_t size, const uint4* T, cudaStream_t st);
// Output row q < n_out of stripe b = sum_{s < N} C[q N + s] * source row s of stripe b, words [0, size) only, canonical; source
// row s is data row src[s] for s < nd and parity row src[s] after (C and src on the device, C as Barrett triples {w, whi, wlo, 0},
// n_out <= 64).  Source words are taken mod P; nothing else is read.  One launch of as many CTAs as fit on the SMs.
cudaError_t launch_batch_reconstruct(const uint32_t* data, size_t dpitch, size_t dstride, const uint32_t* parity, size_t ppitch, size_t pstride,
                                     size_t N, size_t nd, const uint4* C, const uint32_t* src, size_t n_out, uint32_t* out, size_t opitch,
                                     size_t ostride, size_t B, size_t size, int num_sms, cudaStream_t st);
// In place, for B stripes with one host list changed[0 .. k) (ascending, below N <= 64): data row changed[q] of stripe b := the
// canonical new row q of stripe b, and parity row j += sum_q (new_q - old_q) * T[(D j - changed[q]) mod N], words [0, size) only,
// canonical; every word read is taken mod P.  Reads only the k changed data rows, the k new rows and the M parity rows; the list
// goes by value in the launch's parameters.  Needs a layout batch_update_layout_disjoint accepts.  One launch of as many CTAs as
// fit on the SMs.
cudaError_t launch_batch_update(uint32_t* data, size_t dpitch, size_t dstride, size_t N, uint32_t* parity, size_t ppitch, size_t pstride, size_t M,
                                const uint32_t* changed, size_t k, const uint32_t* nw, size_t npitch, size_t nstride, size_t B, size_t size,
                                const uint4* T, int num_sms, cudaStream_t st);
}
#endif
