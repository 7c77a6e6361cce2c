/* fastecc_b200 -- C ABI of the H100 (sm_90a) NTT Reed-Solomon encoder.
 *
 * This is the drop-in boundary for the one hot path of Bulat-Ziganshin/FastECC.  The reference has no FFI layer:
 * its programs textually include the template sources, so the boundary is created at the narrowest existing call
 * surface.  Each entry point below names the reference interface it replaces (file:line in the reference tree).
 * All functions return 0 on success and a negative FASTECC_B200_E* code otherwise; fastecc_b200_last_error()
 * returns a human-readable message for the calling thread.  There is NO CPU fallback: without a usable CUDA
 * device every compute entry point fails with FASTECC_B200_ECUDA.
 *
 * Concurrency: the context is process-wide.  The host (T**) entry points are serialised by an internal lock (they share one
 * staging buffer and three internal streams).  The *_dev entry points are asynchronous on the caller's stream and may be
 * called from several threads / on several streams: the shared scratch buffers and the lazily built twiddle tables are
 * ordered across streams with events (two transforms that need the same scratch buffer run one after the other).
 *
 * Data model (same as the reference, SURVEY.md section 8): N blocks of SIZE 32-bit words, words are elements of
 * GF(P), P = 0xFFF00001, the transform runs across blocks independently for every word column.  Inputs may be
 * any 32-bit values (they are taken mod P); outputs are canonical residues in [0, P).
 */
#ifndef FASTECC_B200_H
#define FASTECC_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FASTECC_B200_P        0xFFF00001u
#define FASTECC_B200_MAX_LOG_N        20      /* P-1 = 2^20 * 4095: largest power-of-two transform (main.cpp:326) */
#define FASTECC_B200_MAX_LOG_N_ENCODE 19      /* encode needs a root of order 2N (RS.cpp:51, README.md:29)        */

enum {
    FASTECC_B200_OK       =  0,
    FASTECC_B200_EINVAL   = -1,   /* N not a power of two / out of range, SIZE == 0, bad pitch, null pointer */
    FASTECC_B200_ECUDA    = -2,   /* CUDA runtime error (message has the cudaError string)                   */
    FASTECC_B200_ENOMEM   = -3,   /* device or pinned-host allocation failed                                 */
    FASTECC_B200_ENOINIT  = -4    /* fastecc_b200_init() has not succeeded in this process                   */
};

/* Process-wide context on one CUDA device: uploads the 16 MiB power table g^e (g = GF_Root(2^20),
 * GF(p).cpp:267-276) and caches scratch buffers.  Idempotent for the same device.  One process per GPU. */
int  fastecc_b200_init(int device);
void fastecc_b200_shutdown(void);
const char* fastecc_b200_last_error(void);
int  fastecc_b200_device(void);                 /* device ordinal of the live context, or -1 */
int  fastecc_b200_num_sms(void);

/* ---- reference call surface, host memory ---------------------------------------------------------------------
 * Replaces  template<T,P> void MFA_NTT(T** data, size_t N, size_t SIZE, bool InvNTT)      ntt.cpp:382-383
 * for <uint32_t,0xFFF00001>; call sites RS.cpp:41,63 and main.cpp:234,272,286.
 * data[i] -> SIZE words of block i (host memory, pageable or pinned).  In place: on return data[i] addresses
 * result block i; the pointer table itself is left untouched (the reference permutes it, callers only read
 * through data[i]).  The inverse transform is unnormalised, as in the reference.  1 <= N <= 2^20, power of two.
 * Beyond MFA_NTT (which needs a power of two): N = 3 * 2^k and 9 * 2^k with 2^k <= 2^20 are accepted too -- the reference's
 * order-3 / order-9 codelets (NTT3 ntt.cpp:26-46, NTT9 ntt.cpp:114-146) composed with the power-of-two transforms, result = the
 * DFT with GF_Root(N) like Slow_NTT (ntt.cpp:451-483) -- so that block counts need not be rounded up (README.md:176). */
int fastecc_b200_ntt_u32(uint32_t** data, size_t N, size_t SIZE_words, int inverse);

/* Opt-in for callers that keep one large block array alive and transform it repeatedly from PAGEABLE memory, the way the
 * reference's drivers do (RS.cpp:31-33, main.cpp:244-247: allocated once, never freed): the host entry points then page-lock
 * such an array in place on first sight (cudaHostRegister, about 0.2 s per GiB, once) so that its transfers pipeline like
 * pinned memory; registrations are dropped by fastecc_b200_pin_host_buffers(0) and at fastecc_b200_shutdown().  While it is enabled, arrays
 * that were passed to the host entry points must not be freed (a page-locked range that is unmapped and re-allocated would
 * be transferred from its old pages).  Off by default; fastecc_b200/shim/ntt.cpp turns it on. */
int fastecc_b200_pin_host_buffers(int enable);

/* Replaces the timed body of  template<T,P> void EncodeReedSolomon(size_t N, size_t SIZE)   RS.cpp:41-63
 * (iNTT, multiply block i by root_2N^i / N, NTT): N data blocks in, N parity blocks out, same buffers.
 * 1 <= N <= 2^19 (N = 2^20 is rejected: the reference silently computes garbage there, GF(p).cpp:274). */
int fastecc_b200_rs_encode(uint32_t** data, size_t N, size_t SIZE_words);

/* ---- device-resident variants (what bench.py times as `value`; PCIe excluded) ----------------------------------
 * d_blocks: device pointer to N rows of pitch_words words each (row i = block i), first SIZE_words of a row
 * are data.  The fast path needs d_blocks 16-byte aligned and pitch_words % 4 == 0 (columns are processed in
 * groups of 4 words, so up to 3 pad words per row are read and rewritten); other layouts go through an internal
 * repack.  stream: a cudaStream_t (NULL = default stream).  Asynchronous with respect to the host. */
/* (N = 3 * 2^k, 9 * 2^k: transforms only here; their encode is fastecc_b200_rs_encode_mixed[_dev] below.) */
int fastecc_b200_ntt_u32_dev  (uint32_t* d_blocks, size_t N, size_t SIZE_words, size_t pitch_words, int inverse, void* stream);
int fastecc_b200_rs_encode_dev(uint32_t* d_blocks, size_t N, size_t SIZE_words, size_t pitch_words, void* stream);

/* Measurement variant of fastecc_b200_rs_encode_dev (bench.py's per-kernel roofline): the same encode with a CUDA event
 * between the passes; synchronises the stream.  In: *n_passes = capacity of pass_ms / pass_kernel (may be NULL).  Out: the
 * duration of every pass kernel in ms, the name of the instantiation it ran as (static strings) and their number. */
int fastecc_b200_rs_encode_dev_timed(uint32_t* d_blocks, size_t N, size_t SIZE_words, size_t pitch_words, void* stream,
                                     float* pass_ms, const char** pass_kernel, int* n_passes);

/* ---- fewer parity blocks than data blocks (SURVEY 8f rank 2) ------------------------------------------------------
 * The reference only describes this (RS.cpp:65-66, NTT.md:46-49: "in order to compute only even-indexed points ...").
 * N data blocks in, M = N / 2^k parity blocks out: parity block j' is parity block (N/M)*j' of the full N -> N encode,
 * i.e. the value of the data polynomial at root_2N^(2*(N/M)*j' + 1).  On return data[j'], j' < M, hold the parity;
 * blocks M .. N-1 are undefined (host variant: left untouched).  1 <= M <= N <= 2^19, both powers of two.
 * The _dev variant needs a 16-byte aligned buffer and pitch_words % 4 == 0. */
int fastecc_b200_rs_encode_asym    (uint32_t** data, size_t N, size_t M, size_t SIZE_words);
int fastecc_b200_rs_encode_asym_dev(uint32_t* d_blocks, size_t N, size_t M, size_t SIZE_words, size_t pitch_words, void* stream);

/* ---- code words of 3 * 2^k and 9 * 2^k data blocks -------------------------------------------------------------------
 * The reference's roadmap item (README.md:176; NTT.md:43-44: block counts rounded up to 2^k make it "up to 2x" slower):
 * N = 2^k, 3 * 2^k or 9 * 2^k data blocks with 2^k <= 2^19 (so N <= 9 * 2^19 = 4718592).  N data blocks in, N parity blocks
 * out, same buffers, as fastecc_b200_rs_encode[_dev]: parity block j = f(rho^(2j+1)), rho = GF_Root(2N), where f is the
 * polynomial of degree < N with f(rho^(2i)) = data block i -- the code word of 2N rows (row 2i = data i, row 2j+1 = parity j)
 * that the decoder below recovers (fastecc_b200_rs_decode_pattern_mixed).  Power-of-two N runs the encode of
 * fastecc_b200_rs_encode_dev, bit for bit.  Device memory: the data plus one scratch buffer of the same size (the Y buffer of
 * the order-2^k transforms; the host variant also stages the data on the device).  Same layouts and repacking rules as
 * fastecc_b200_rs_encode[_dev]; fastecc_b200_rs_encode[_dev] themselves keep rejecting non-powers of two. */
int fastecc_b200_rs_encode_mixed    (uint32_t** data, size_t N, size_t SIZE_words);
int fastecc_b200_rs_encode_mixed_dev(uint32_t* d_blocks, size_t N, size_t SIZE_words, size_t pitch_words, void* stream);

/* ---- fewer parity blocks than data blocks, for the same orders -------------------------------------------------------
 * N data blocks in (any N that fastecc_b200_rs_encode_mixed accepts), M parity blocks out, for any M that divides N: parity
 * block j' is parity block (N/M)*j' of fastecc_b200_rs_encode_mixed, i.e. f(rho^(2*(N/M)*j' + 1)), rho = GF_Root(2N) -- the code
 * word of 2N rows that fastecc_b200_rs_decode_pattern_mixed decodes, with the parity rows that were not produced erased.  On
 * return data[j'], j' < M, hold the parity; blocks M .. N-1 are undefined (host variant: left untouched).  Power-of-two N runs
 * fastecc_b200_rs_encode_asym[_dev] and M = N runs fastecc_b200_rs_encode_mixed[_dev], bit for bit.  Device memory, layouts,
 * repacking and inputs taken mod P as fastecc_b200_rs_encode_mixed[_dev]. */
int fastecc_b200_rs_encode_asym_mixed    (uint32_t** data, size_t N, size_t M, size_t SIZE_words);
int fastecc_b200_rs_encode_asym_mixed_dev(uint32_t* d_blocks, size_t N, size_t M, size_t SIZE_words, size_t pitch_words, void* stream);

/* ---- arbitrary bytes <-> words below P (SURVEY 8f rank 3) -----------------------------------------------------------
 * The reference describes, but does not implement, a bit-optimal recoding (GF.md:72-104, README.md:160-163): the top
 * 12 bits of the W words of a block are rewritten from base 4096 to base 4095 (no 0xFFF, hence every word < P) using
 * one extra bit, stored as word W of the block: 4096-byte blocks become 4100-byte (1025-word) blocks to encode.
 * d_bytes: n_blocks contiguous blocks of 4*W bytes; d_words: n_blocks rows of pitch_words words (>= W+1, % 4 == 0), words
 * 0..W of a row are meaningful.  W = words_per_block: multiple of 4, <= 1024.  Both buffers 16-byte aligned.
 * gfp_to_bytes(bytes_to_gfp(x)) == x for every x; parity rows produced by the encoder are NOT recoded data and are
 * stored as they are (GF.md:101-104). */
int fastecc_b200_bytes_to_gfp_dev(const void* d_bytes, uint32_t* d_words, size_t n_blocks, size_t words_per_block, size_t pitch_words, void* stream);
int fastecc_b200_gfp_to_bytes_dev(const uint32_t* d_words, void* d_bytes, size_t n_blocks, size_t words_per_block, size_t pitch_words, void* stream);

/* ---- element-wise helpers around the transforms (erasure decoding, SURVEY 8f rank 4) --------------------------------
 * GF_Mul (GF(p).cpp:110-127) and GF_Inv (GF(p).cpp:293-297, x^(P-2); 0 -> 0) on device vectors of n words, and the shape
 * of the reference's scaling loop (RS.cpp:51-59) with an arbitrary constant per block: block i *= d_consts[i].
 * Inputs are taken mod P, results are canonical.  row_scale: 16-byte aligned buffer, pitch_words % 4 == 0. */
int fastecc_b200_gf_mul_dev(const uint32_t* d_a, const uint32_t* d_b, uint32_t* d_out, size_t n, void* stream);
int fastecc_b200_gf_inv_dev(const uint32_t* d_a, uint32_t* d_out, size_t n, void* stream);
int fastecc_b200_row_scale_dev(uint32_t* d_blocks, size_t n_rows, size_t SIZE_words, size_t pitch_words, const uint32_t* d_consts, void* stream);

/* ---- erasure decoding (SURVEY 8f rank 4) --------------------------------------------------------------------------------
 * The reference describes the decoder and does not implement it (README.md:88-119 "Fastest", RS.md:42-79, roadmap
 * README.md:173).  Code word of 2N rows: row 2i = data block i, row 2j+1 = parity block j of fastecc_b200_rs_encode
 * (RS.cpp:22-68).  Any set of at most N lost rows is recovered from the others by the formal-derivative method on two
 * order-2N transforms of the hot path.
 *   _pattern: everything that depends only on WHICH rows are lost (erasure locator by a product tree of batched transforms,
 *             its values and derivative values), built on the device once; erased = HOST array of ascending distinct row
 *             numbers < n_rows; n_rows = 2N = 2 .. 2^20, n_erased <= N.  Synchronises the stream.
 *   _recover: d_code = the 2N rows (pitch_words per row, first SIZE_words meaningful, 16-byte aligned, pitch % 4 == 0; content
 *             of the lost rows arbitrary); it is the workspace of the two transforms and is DESTROYED.  Row i of d_out
 *             (out_pitch_words per row) receives lost row erased[i], canonical residues.  Asynchronous on the stream.
 * A pattern may be used for any number of code words / columns.  Not pinned by reference code (there is none): checked
 * against interpolation by definition and by encode -> erase -> decode round trips (tests/test_decoder.py).
 *   _pattern_mixed: the same for the code words of fastecc_b200_rs_encode_mixed: n_rows = 2N for every N it accepts (n_rows = 2^k,
 *             3 * 2^k or 9 * 2^k with 1 <= k <= 20); the result serves _recover, _count and _free like any pattern.
 *             _pattern keeps rejecting n_rows that are not powers of two. */
typedef struct fastecc_b200_erasures fastecc_b200_erasures;
int    fastecc_b200_rs_decode_pattern(size_t n_rows, const uint32_t* erased, size_t n_erased, void* stream, fastecc_b200_erasures** pattern);
int    fastecc_b200_rs_decode_pattern_mixed(size_t n_rows, const uint32_t* erased, size_t n_erased, void* stream, fastecc_b200_erasures** pattern);
int    fastecc_b200_rs_decode_recover(const fastecc_b200_erasures* pattern, uint32_t* d_code, size_t SIZE_words, size_t pitch_words,
                                      uint32_t* d_out, size_t out_pitch_words, void* stream);
size_t fastecc_b200_rs_decode_count(const fastecc_b200_erasures* pattern);        /* n_erased */
void   fastecc_b200_rs_decode_free(fastecc_b200_erasures* pattern);

/* ---- repair of a stored stripe, in place ---------------------------------------------------------------------------------
 * The stripe as fastecc_b200_rs_encode_asym_mixed[_dev] leaves it: N data rows and the M parity rows (any (N, M) that encode
 * accepts, M = N included).  Any n_lost_data + n_lost_parity <= M lost blocks, data and parity alike, are recomputed in place;
 * the cost follows the stripe (one encode, order-M and order-N transforms), not a 2N-row code word (DESIGN 3g).
 *   _pattern: everything that depends only on which blocks are lost, built on the device (synchronises the stream).  lost_data /
 *             lost_parity: HOST arrays, ascending, distinct, below N and M.  Validated in full before anything is allocated.
 *   _repair:  d_data = N rows (data_pitch_words apart), d_parity = M rows (parity_pitch_words apart), both 16-byte aligned with
 *             pitches that are multiples of 4 words, not overlapping.  The content of the lost rows is arbitrary, surviving words
 *             are taken mod P.  On return words [0, SIZE) of every lost row hold the canonical block; nothing else in either buffer
 *             is written (no surviving row, no pad word beyond SIZE).  Asynchronous on the stream; with nothing lost it returns
 *             0 without launching anything.  A pattern serves any number of stripes of any SIZE.
 * Device memory: a workspace of N + M rows of one column chunk, kept by the context like the transforms' scratch buffers, plus
 * the encode's and the transforms' buffers (N rows of the chunk each).  The chunk is the whole padded SIZE when
 * (N + M) * ceil4(SIZE) * 4 bytes <= 4 GiB, else the widest multiple of 4 words within that bound, and the repair runs once per
 * chunk (a 2^19 x 4 KiB stripe is one chunk for every M). */
typedef struct fastecc_b200_repair fastecc_b200_repair;
int  fastecc_b200_rs_repair_pattern(size_t N, size_t M, const uint32_t* lost_data, size_t n_lost_data,
                                    const uint32_t* lost_parity, size_t n_lost_parity, void* stream, fastecc_b200_repair** pattern);
int  fastecc_b200_rs_repair(const fastecc_b200_repair* pattern, uint32_t* d_data, size_t data_pitch_words,
                            uint32_t* d_parity, size_t parity_pitch_words, size_t SIZE_words, void* stream);
void fastecc_b200_rs_repair_free(fastecc_b200_repair* pattern);

/* ---- update of a stored stripe, in place -------------------------------------------------------------------------------
 * The write of a stored stripe: n_changed of its N data blocks get new content, and the M parity rows are brought up to date
 * without re-encoding the stripe from scratch.  The stripe is that of fastecc_b200_rs_repair: d_data = N rows
 * (data_pitch_words apart) and d_parity = M rows (parity_pitch_words apart) as fastecc_b200_rs_encode_asym_mixed[_dev] leaves them,
 * for any (N, M) that fastecc_b200_rs_encode_asym_mixed_dev accepts.  changed: HOST array, ascending, distinct, below N; row i of
 * d_new (new_pitch_words apart) is the new content of data block changed[i].
 * PRECONDITION: the stored parity is the encode of the stored data.  On a stripe where it is not, the result is unspecified
 * (the update adds the change to the parity; it does not re-derive the parity from the data).  fastecc_b200_rs_scrub below checks
 * it, and locates the blocks that break it.
 * On return data rows changed[i] hold the canonical new blocks and the parity rows equal fastecc_b200_rs_encode_asym_mixed_dev of
 * the updated data, bit for bit.  Nothing else is written: no other data row, no pad word beyond SIZE in any buffer, never d_new.
 * Every input word, old or new, data or parity, is taken mod P.  All three buffers 16-byte aligned with pitches that are
 * multiples of 4 words, none overlapping another.  Validated in full before anything is allocated or launched.  Asynchronous on
 * the stream, which it does not synchronise; `changed` may be freed as soon as the call returns.  n_changed == 0 returns 0 and
 * launches nothing.
 * The library picks one of two paths from (N, M, n_changed, SIZE) (DESIGN 3h): for few changed blocks, the change times a table
 * of N coefficients (16 bytes each, built on the device at the first update of an N and kept by the context) is added to the
 * parity rows, reading only the changed rows and the parity (workspace: the n_changed delta rows, at most 4 GiB); for many, the
 * new rows are written and the whole stripe is re-encoded into the parity, in column chunks as fastecc_b200_rs_repair runs
 * (same workspace, same 4 GiB bound).  The host side keeps at most 8 page-locked copies of changed lists in flight; a call
 * beyond that waits for the oldest copy to have run. */
int fastecc_b200_rs_update(uint32_t* d_data, size_t data_pitch_words, size_t N, uint32_t* d_parity, size_t parity_pitch_words, size_t M,
                           const uint32_t* changed, size_t n_changed, const uint32_t* d_new, size_t new_pitch_words, size_t SIZE_words, void* stream);

/* ---- scrub of a stored stripe: detect silent corruption, locate the corrupted blocks ------------------------------------
 * The stripe of fastecc_b200_rs_repair (N data rows, M parity rows, any (N, M) that fastecc_b200_rs_encode_asym_mixed_dev accepts,
 * both buffers 16-byte aligned with pitches that are multiples of 4 words; they may overlap, since nothing is written).  The
 * code has minimum distance M + 1, so from the stripe alone the call tells whether the parity is the encode of the data, and
 * locates up to max_bad corrupted blocks at unknown positions, data and parity alike (DESIGN 3i).
 *   max_bad:  0 = detect only (the only choice at M = 1); else 1 <= max_bad <= min(M / 2, FASTECC_B200_SCRUB_MAX_BAD) (the
 *             locator is found by Berlekamp-Massey on the host, O(max_bad^2)).
 *   seed:     the two folds of the columns use the weights r_f,c (fold f in {0, 1}, column c < SIZE):
 *                 z = seed + (2c + f + 1) * 0x9E3779B97F4A7C15                       (mod 2^64)
 *                 z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;  z = (z ^ (z >> 27)) * 0x94D049BB133111EB;  z ^= z >> 31
 *                 r_f,c = z mod P
 *             i.e. the (2c + f + 1)-th output of splitmix64 started at `seed`.  Row m folds to sum_c r_f,c * row_m[c] mod P.  The
 *             same seed gives the same result; a scrub that must not be predictable by whoever writes the data takes a fresh one.
 *   Out:      *status = FASTECC_B200_SCRUB_*; bad_data / bad_parity: HOST arrays of capacity max_bad (may be NULL when max_bad = 0)
 *             receive the located blocks, ascending (ready for fastecc_b200_rs_repair_pattern), *n_bad_data / *n_bad_parity their
 *             counts (0 unless LOCATED).  None of the outputs is written when the call returns an error.
 * Guarantees, with t corrupted blocks (blocks with any word of their SIZE that differs mod P from the encode of the stored data,
 * parity blocks counted against the data as stored), each up to a probability of P^-2 over the folds' weights (P^-1 per fold):
 *   t = 0 -> CLEAN;  1 <= t <= max_bad -> LOCATED with exactly the corrupted blocks;  max_bad < t <= M - max_bad -> DETECTED;
 *   1 <= t <= M -> never CLEAN.  Beyond M - max_bad the result may be LOCATED with a wrong set, as for every bounded-distance
 *   decoder.  Words are taken mod P (a raw word >= P congruent to the stored value is not corruption), pad words beyond SIZE are
 *   never read into a sum.
 * Validated in full before anything is allocated or launched.  Synchronises the stream (the host needs the syndromes).  Device
 * memory: (N + M) * 16 bytes of the context's repair workspace plus the encode's and the transforms' buffers for one column. */
#define FASTECC_B200_SCRUB_CLEAN     0   /* the parity is the encode of the data                  */
#define FASTECC_B200_SCRUB_LOCATED   1   /* bad_data / bad_parity list every corrupted block      */
#define FASTECC_B200_SCRUB_DETECTED  2   /* corrupted, not located within max_bad                 */
#define FASTECC_B200_SCRUB_MAX_BAD   4096
int fastecc_b200_rs_scrub(const uint32_t* d_data, size_t data_pitch_words, size_t N, const uint32_t* d_parity, size_t parity_pitch_words, size_t M,
                          size_t SIZE_words, size_t max_bad, uint64_t seed, void* stream, int* status,
                          uint32_t* bad_data, size_t* n_bad_data, uint32_t* bad_parity, size_t* n_bad_parity);

/* ---- scrub of a degraded stripe: some blocks known lost, the survivors checked ---------------------------------------
 * The stripe of fastecc_b200_rs_scrub with the f = n_lost_data + n_lost_parity blocks of `known` (a pattern of
 * fastecc_b200_rs_repair_pattern, which gives N and M) lost, 1 <= f < M.  Errors-and-erasures decoding (DESIGN 3j): a known lost
 * block costs one check symbol, a corrupted survivor two, so the survivors alone detect up to M - f corrupted blocks and locate up
 * to floor((M - f) / 2) of them, where fastecc_b200_rs_scrub, blind to the losses, reads the lost rows as corruption.  Use it
 * before a repair: a repair from a corrupted survivor rebuilds wrong blocks and reports nothing.
 *   Buffers, SIZE_words, seed (the fold weights), statuses and outputs as fastecc_b200_rs_scrub; nothing is written into the
 *   buffers, which may overlap.  The rows of the lost blocks are never read: they may hold anything.
 *   max_bad:  0 = detect only; else at most min(floor((M - f) / 2), FASTECC_B200_SCRUB_MAX_BAD).
 *   Out:      the lists name surviving blocks only, ascending.  LOCATED: repair with a pattern of lost + located blocks (at most
 *             f + max_bad <= M); CLEAN: repair with `known` itself.
 * Guarantees, with t corrupted surviving blocks, each up to a probability of P^-2 over the folds' weights:
 *   t = 0 -> CLEAN;  1 <= t <= max_bad -> LOCATED with exactly the corrupted survivors;  max_bad < t <= M - f - max_bad ->
 *   DETECTED;  1 <= t <= M - f -> never CLEAN.  (Two error patterns off the lost blocks differ by a code word of the code
 *   punctured on them, of distance M + 1 - f.)
 * EINVAL, before anything is allocated or launched: a null pattern, status or count; f = M (nothing left to check); max_bad
 * above its bound; null lists with max_bad > 0; the rows and pitches fastecc_b200_rs_scrub rejects.  A pattern with nothing lost
 * runs fastecc_b200_rs_scrub itself.  Synchronises the stream; device memory as fastecc_b200_rs_scrub. */
int fastecc_b200_rs_scrub_degraded(const fastecc_b200_repair* known, const uint32_t* d_data, size_t data_pitch_words,
                                   const uint32_t* d_parity, size_t parity_pitch_words, size_t SIZE_words, size_t max_bad, uint64_t seed,
                                   void* stream, int* status, uint32_t* bad_data, size_t* n_bad_data, uint32_t* bad_parity,
                                   size_t* n_bad_parity);

/* ---- degraded read: a few lost blocks rebuilt out of place from N surviving rows ----------------------------------------
 * The read of a stripe with blocks missing: the wanted lost blocks are computed into d_out, and nothing is written into the
 * stripe.  The stripe is that of fastecc_b200_rs_repair (N data rows data_pitch_words apart, M parity rows parity_pitch_words
 * apart, any (N, M) that fastecc_b200_rs_encode_asym_mixed_dev accepts).  It costs one pass over N rows and needs no pattern
 * (DESIGN 3k).
 *   Lists:    lost_data / lost_parity name the unavailable blocks; want_data / want_parity the blocks to produce, a subset of
 *             them.  All are HOST arrays, ascending, distinct, below N or M.  With a = n_lost_data: a + n_lost_parity <= M, and
 *             a + n_want_parity <= FASTECC_B200_RECONSTRUCT_MAX (fastecc_b200_rs_repair rebuilds more).
 *   Rows read: exactly the N - a surviving data rows and the parity rows J = the a lowest-numbered parity blocks not in
 *             lost_parity, so a storage layer fetches only those N blocks.  No other row is loaded: lost rows and parity rows
 *             outside J may hold anything.  Words are taken mod P.
 *   Out:      row q of d_out (out_pitch_words apart) receives block want_data[q] for q < n_want_data, then the blocks of
 *             want_parity in order; words [0, SIZE) of those rows only, canonical.
 * PRECONDITION: the surviving blocks are a consistent stripe (as for fastecc_b200_rs_update).  A corrupted survivor gives wrong
 * blocks without a report; fastecc_b200_rs_scrub_degraded checks the survivors first.
 * All three buffers 16-byte aligned with pitches that are multiples of 4 words; d_data and d_parity may overlap each other, d_out
 * may overlap neither.  Validated in full before anything is allocated or launched (EINVAL).  Asynchronous on the stream, which it
 * does not synchronise; the host lists may be freed as soon as the call returns.  n_want_data + n_want_parity == 0 returns 0 and
 * launches nothing.  Two kernel launches per call (per column chunk), plus the build of fastecc_b200_rs_update's table at the first
 * use of an N.  Device memory: that table (16 bytes per data block) and K * ceil4(SIZE) * 8 bytes of the context's repair
 * workspace, K = a + n_want_parity; above 4 GiB the call runs in column chunks within that bound. */
#define FASTECC_B200_RECONSTRUCT_MAX 32
int fastecc_b200_rs_reconstruct(const uint32_t* d_data, size_t data_pitch_words, size_t N,
                                const uint32_t* d_parity, size_t parity_pitch_words, size_t M,
                                const uint32_t* lost_data, size_t n_lost_data, const uint32_t* lost_parity, size_t n_lost_parity,
                                const uint32_t* want_data, size_t n_want_data, const uint32_t* want_parity, size_t n_want_parity,
                                uint32_t* d_out, size_t out_pitch_words, size_t SIZE_words, void* stream);

/* ---- encode of a batch of small stripes, out of place, in one launch ---------------------------------------------------
 * The write of many stripes at once: for each of n_stripes stripes of N data blocks, its M parity blocks into rows of their own;
 * the data is only read.  Data block i of stripe b is at d_data + b * data_stripe_words + i * data_pitch_words, parity block j of
 * stripe b at d_parity + b * parity_stripe_words + j * parity_pitch_words.  N is any order that
 * fastecc_b200_rs_encode_asym_mixed_dev accepts (2^k, 3 * 2^k or 9 * 2^k) up to FASTECC_B200_BATCH_MAX_N, M any divisor of N;
 * larger stripes go through the per-stripe entry points.  Each parity block is M x N products per word straight from the data
 * (fastecc_b200_rs_update's formula, DESIGN 3l), so the call pays one launch for the batch instead of a transform per stripe.
 *   Result:  parity row j of every stripe equals row j of fastecc_b200_rs_encode_asym_mixed_dev run on that stripe's data, bit
 *            for bit, so fastecc_b200_rs_repair, _update, _scrub and _reconstruct take the stripes as they are.
 *   Writes:  words [0, SIZE) of the n_stripes * M parity rows, canonical, and nothing else: no data word, no pad word, no word
 *            between rows.  Reads: the data, whose words are taken mod P; pad words past SIZE never enter a sum.
 *   Layout:  both bases 16-byte aligned; the two pitches and the two stripe strides multiples of 4 words; each pitch >= SIZE.  No
 *            parity word may be another parity word or a data word (data rows may overlap each other).  The call accepts only
 *            layouts it proves disjoint in O(N + M) host work: separate data and parity spans with pairwise disjoint parity rows,
 *            each side stripe-major ([B][N][pitch]) or block-major ([N][B][pitch]) in any combination; or one common stripe stride
 *            in which stripe 0's N + M rows, in any order, are disjoint and fit inside one stride (e.g. [B][N + M][pitch] with the
 *            parity below the data).  Anything else is EINVAL.
 * Validated in full before anything is allocated or launched (EINVAL).  n_stripes == 0 returns 0 and launches nothing (null buffers included); otherwise
 * one kernel launch, plus the build of fastecc_b200_rs_update's table at the first use of an N.  No workspace, no host-to-device
 * copy.  Asynchronous on the stream, which it does not synchronise. */
#define FASTECC_B200_BATCH_MAX_N 64
int fastecc_b200_rs_encode_batch(const uint32_t* d_data, size_t data_pitch_words, size_t data_stripe_words, size_t N,
                                 uint32_t* d_parity, size_t parity_pitch_words, size_t parity_stripe_words, size_t M,
                                 size_t n_stripes, size_t SIZE_words, void* stream);

/* ---- degraded read of a batch of small stripes with one loss pattern, in one launch -------------------------------------
 * The read of many stripes that lost the same blocks (after a disk failure, the stripes that had the same block position on it):
 * for each of n_stripes stripes, the wanted lost blocks into rows of their own; nothing is written into the stripes.  Stripes are
 * addressed as in fastecc_b200_rs_encode_batch: data block i of stripe b at d_data + b * data_stripe_words + i * data_pitch_words,
 * parity block j at d_parity + b * parity_stripe_words + j * parity_pitch_words; N is any order that
 * fastecc_b200_rs_encode_asym_mixed_dev accepts up to FASTECC_B200_BATCH_MAX_N, M any divisor of N (larger stripes go through
 * fastecc_b200_rs_reconstruct one at a time).  Every wanted block is a fixed combination of N rows (DESIGN 3m), so the call is
 * n_out x N products per word straight from the stored rows.
 *   Lists:    as for fastecc_b200_rs_reconstruct, one set for the whole batch: HOST arrays, ascending, distinct, below N or M;
 *             the wanted blocks a subset of the lost ones; with a = n_lost_data, a + n_lost_parity <= M.
 *             FASTECC_B200_RECONSTRUCT_MAX does not apply: n_out = n_want_data + n_want_parity <= M <= 64.
 *   Rows read: per stripe exactly the N - a surviving data rows and the parity rows J = the a lowest-numbered parity blocks not in
 *             lost_parity.  No other row is loaded: lost rows and parity rows outside J may hold anything.  Words are taken mod
 *             P; pad words past SIZE never enter a sum.
 *   Out:      wanted block q of stripe b (want_data in order, then want_parity) at d_out + b * out_stripe_words + q * out_pitch_words;
 *             words [0, SIZE) of those rows only, canonical, each bit for bit what fastecc_b200_rs_reconstruct returns for that
 *             stripe alone.  Nothing else is written; the stripe buffers are never written.
 *   Layout:   the three bases 16-byte aligned; the pitches and stripe strides multiples of 4 words; each pitch >= SIZE.  Data and
 *             parity may overlap each other (both are only read).  No output word may be another output word, a data word or a
 *             parity word; the call accepts only layouts that fastecc_b200_rs_encode_batch's rule proves so for (data, out) and for
 *             (parity, out): an output span apart from each side's span, stripe-major ([B][n_out][pitch]) or block-major
 *             ([n_out][B][pitch]); or one common stripe stride holding each stripe's rows disjoint within it (e.g. one
 *             [B][N + M + n_out][pitch] buffer).  Writing into the stripes' own lost rows is EINVAL.
 * PRECONDITION: the surviving blocks are consistent stripes, as for fastecc_b200_rs_reconstruct.
 * Validated in full before anything is allocated or launched (EINVAL).  n_stripes == 0 or nothing wanted returns 0 and launches
 * nothing (null buffers included).  Otherwise one kernel launch and one host-to-device copy of the n_out x N coefficients (at
 * most 64 KiB, through the context's repair workspace); no table build.  Asynchronous on the stream, which it does not
 * synchronise; the host lists may be freed as soon as the call returns. */
int fastecc_b200_rs_reconstruct_batch(const uint32_t* d_data, size_t data_pitch_words, size_t data_stripe_words, size_t N,
                                      const uint32_t* d_parity, size_t parity_pitch_words, size_t parity_stripe_words, size_t M,
                                      const uint32_t* lost_data, size_t n_lost_data, const uint32_t* lost_parity, size_t n_lost_parity,
                                      const uint32_t* want_data, size_t n_want_data, const uint32_t* want_parity, size_t n_want_parity,
                                      uint32_t* d_out, size_t out_pitch_words, size_t out_stripe_words,
                                      size_t n_stripes, size_t SIZE_words, void* stream);

/* ---- update of a batch of small stripes in place with one changed list, in one launch -----------------------------------
 * The partial write of many stripes at once: in each of n_stripes stripes the data blocks of one HOST list `changed` get new
 * content and the M parity blocks are brought up to date, as fastecc_b200_rs_update does for one stripe (DESIGN 3n).  A caller
 * groups its writes by the changed positions, as it groups degraded reads by loss pattern.  Data block i of stripe b is at
 * d_data + b * data_stripe_words + i * data_pitch_words, parity block j at d_parity + b * parity_stripe_words + j * parity_pitch_words,
 * and row q of stripe b's new rows, at d_new + b * new_stripe_words + q * new_pitch_words, is the new content of data block
 * changed[q].  N is any order that fastecc_b200_rs_encode_asym_mixed_dev accepts up to FASTECC_B200_BATCH_MAX_N, M any divisor
 * of N (larger stripes go through fastecc_b200_rs_update one at a time); changed is ascending, distinct, below N.
 *   Result:  in every stripe data rows changed[q] hold the canonical new blocks and the M parity rows equal
 *            fastecc_b200_rs_encode_batch (and so fastecc_b200_rs_encode_asym_mixed_dev) of the updated data, bit for bit.  The
 *            change times update's table is added to the parity: n_changed x M products per word.
 *   Writes:  words [0, SIZE) of the n_changed changed data rows and the M parity rows of each stripe, and nothing else: no other
 *            data row, no pad word, no word between rows, never d_new.  Reads: the changed data rows (old contents), the new
 *            rows and the parity rows; data rows outside `changed` are never loaded and may hold anything.  Every input word,
 *            old or new, data or parity, is taken mod P.
 *   Layout:  the three bases 16-byte aligned; the pitches and stripe strides multiples of 4 words; each pitch >= SIZE.  The call
 *            accepts only layouts that fastecc_b200_rs_encode_batch's rule proves disjoint for the pairs (new, data), (new,
 *            parity) and (data, parity): all N + M rows of all stripes pairwise disjoint and none of them meeting a new row.  New
 *            rows may overlap each other (new_stripe_words = 0 gives every stripe the same new blocks).  Accepted: separate data,
 *            parity and new spans, each stripe-major or block-major; one [B][N + M][pitch] stripe buffer with the new rows apart;
 *            one [B][N + M + n_changed][pitch] buffer.  Anything else is EINVAL.
 * PRECONDITION: as for fastecc_b200_rs_update, the stored parity is the encode of the stored data; fastecc_b200_rs_scrub checks it.
 * Validated in full before anything is allocated or launched (EINVAL).  n_stripes == 0 or n_changed == 0 returns 0 and launches
 * nothing (null buffers included).  Otherwise one kernel launch, plus the build of fastecc_b200_rs_update's table at the first
 * use of an N; no workspace and no host-to-device copy (the list goes in the launch's parameters).  Asynchronous on the stream,
 * which it does not synchronise; `changed` may be freed as soon as the call returns.
 * Cost: it reads 2 n_changed + M rows and writes n_changed + M per stripe, with n_changed x M products per word.  Overwriting
 * the changed rows and re-running fastecc_b200_rs_encode_batch reads N and writes M rows (plus the copy) with N x M products
 * per word.  On an H100 (DESIGN 3n, 4 KiB blocks) this call is the faster one at every measured point except n_changed = N at
 * N >= 48 with M >= 16 (48+16, 64+16, 64+64), where the re-encode is 1.05-1.19x faster; the crossing there lies between
 * n_changed = N / 2 and N.  A caller that rewrites nearly whole stripes of those shapes should re-encode them. */
int fastecc_b200_rs_update_batch(uint32_t* d_data, size_t data_pitch_words, size_t data_stripe_words, size_t N,
                                 uint32_t* d_parity, size_t parity_pitch_words, size_t parity_stripe_words, size_t M,
                                 const uint32_t* changed, size_t n_changed,
                                 const uint32_t* d_new, size_t new_pitch_words, size_t new_stripe_words,
                                 size_t n_stripes, size_t SIZE_words, void* stream);

/* ---- one transform sharded over several GPUs (one process per GPU; BASELINE config 4) ---------------------------
 * Global block i = l*n_ranks + rank is local block l (data in, parity out).  An encode is: pass 0 on every rank,
 * all-to-all of whole blocks, pass 1, all-to-all, pass 2 -- the exchange is the caller's (fastecc_b200/sharded.py does it
 * with torch.distributed / NCCL); these are the three local passes of RS.cpp:41-63 with the sharded twists.
 * N = global number of data blocks, 2^11 .. 2^19; d_local holds N/n_ranks rows of pitch_words (16-byte aligned).  n_ranks is
 * a power of two that divides both factors of N = N1 * N2 (fastecc_b200_shard_geometry): pass 0 and pass 2 work on N2 / n_ranks
 * row sets per rank, pass 1 on N1 / n_ranks; other shapes fail with FASTECC_B200_EINVAL before anything is launched. */
int fastecc_b200_rs_encode_shard_pass(uint32_t* d_local, size_t N, int n_ranks, int rank, size_t SIZE_words, size_t pitch_words,
                                      int which, void* stream);

/* The same passes with the exchange FUSED into the kernels' stores (no all-to-all, no staging): every rank owns two
 * buffers of N/n_ranks rows, X (data in / parity out) and Y (intermediate), allocated with fastecc_b200_dev_alloc and
 * mapped into the other ranks with fastecc_b200_ipc_export / _open (CUDA IPC; peer access over NVLink).
 *   which 0: reads the local X, writes the rows of Y on their owners     d_src = X_local, d_peers[r] = rank r's Y
 *   which 1: reads the local Y, writes the rows of X on their owners     d_src = Y_local, d_peers[r] = rank r's X
 *   which 2: local, in place on X                                        d_src = X_local, d_peers[rank] = X_local
 * d_peers: HOST array of n_ranks device pointers (own buffer at [rank]).  The caller separates the passes with a
 * cross-rank barrier on the stream (fastecc_b200_shard_barrier below).  n_ranks = 2, 4 or 8; N = 2^12..2^19 with
 * both factors of N = N1*N2 (csrc/plan.h split_l1) at least 32*n_ranks, so that the 32 rows a thread stores go to one rank. */
int fastecc_b200_rs_encode_shard_pass_p2p(const uint32_t* d_src, uint32_t* const* d_peers, size_t N, int n_ranks, int rank,
                                          size_t SIZE_words, size_t pitch_words, int which, void* stream);
/* The cross-rank barrier between those passes, as a kernel on the stream (no NCCL, no host round trip): every rank owns an array
 * of FASTECC_B200_BARRIER_WORDS zero-initialised words from fastecc_b200_dev_alloc, mapped into the peers like X and Y;
 * d_flag_peers = HOST array of the n_ranks arrays (own at [rank]).  Rank r writes `epoch` into word [r] of every peer's array and
 * waits until its own words [0, n_ranks) have reached it; epoch = 1, 2, 3, ... in the same order on every rank.  The kernel runs
 * behind the pass whose peer stores it publishes.  A peer that never arrives makes it give up after about ten seconds and set
 * word [8] of the own array (check it after synchronising; fastecc_b200/sharded.py raises). */
#define FASTECC_B200_BARRIER_WORDS 16
int fastecc_b200_shard_barrier(uint32_t* const* d_flag_peers, int n_ranks, int rank, uint32_t epoch, void* stream);

/* One rank's share of a whole sharded encode / transform as ONE call: the passes above and the barriers between them, enqueued
 * on the stream.  d_x_peers / d_y_peers / d_flag_peers: HOST arrays of every rank's X, Y and barrier-flag buffers (own at [rank]);
 * *epoch: this rank's barrier counter, 0 before the first call (the same sequence of calls on every rank).  This is all a C++ host
 * needs for the multi-GPU path once the IPC handles are exchanged (integration/shard_example.cpp). */
int fastecc_b200_rs_encode_shard_p2p(uint32_t* const* d_x_peers, uint32_t* const* d_y_peers, uint32_t* const* d_flag_peers, uint32_t* epoch,
                                     size_t N, int n_ranks, int rank, size_t SIZE_words, size_t pitch_words, void* stream);
int fastecc_b200_ntt_shard_p2p(uint32_t* const* d_x_peers, uint32_t* const* d_y_peers, uint32_t* const* d_flag_peers, uint32_t* epoch,
                               size_t N, int n_ranks, int rank, size_t SIZE_words, size_t pitch_words, int inverse, void* stream);

/* ONE standalone transform (MFA_NTT, ntt.cpp:382-447; unnormalised inverse) sharded the same way: cyclic blocks in and out.
 *   which 0: reads the local X, stores into the Ys of the owners (the four-step transpose as peer stores)   d_src = X_local, d_peers[r] = rank r's Y
 *   which 1: local, Y -> X                                                                                  d_src = Y_local, d_peers[rank] = X_local
 * with one cross-rank barrier between them.  N = 2^11 .. 2^20, n_ranks = 2, 4 or 8, first tile height (N1 of csrc/plan.h) >= 32 * n_ranks. */
int fastecc_b200_ntt_shard_pass_p2p(const uint32_t* d_src, uint32_t* const* d_peers, size_t N, int n_ranks, int rank,
                                    size_t SIZE_words, size_t pitch_words, int inverse, int which, void* stream);

/* The decomposition N = N1 * N2 the sharded passes use (csrc/plan.h split_l1, FASTECC_B200_SPLIT honoured), for callers that do the
 * exchange themselves; *fused_exchange_ok: bit 0 = the encode _p2p passes, bit 1 = the NTT _p2p passes support (N, n_ranks).  Fails if N cannot be sharded. */
int fastecc_b200_shard_geometry(size_t N, int n_ranks, size_t* N1, size_t* N2, int* fused_exchange_ok);
/* cudaMemcpy2DAsync between pinned host memory and a device buffer (column chunks of a block array), for pipelined
 * host <-> device staging around the sharded passes (fastecc_b200/sharded.py encode_host). */
int fastecc_b200_copy2d_async(void* dst, size_t dst_pitch_bytes, const void* src, size_t src_pitch_bytes, size_t width_bytes, size_t rows,
                              int to_device, void* stream);
void* fastecc_b200_dev_alloc(size_t bytes);                       /* cudaMalloc: exportable, unlike a caching-allocator block */
void  fastecc_b200_dev_free(void* d_ptr);
int   fastecc_b200_ipc_export(void* d_ptr, void* handle64);       /* 64-byte cudaIpcMemHandle_t */
int   fastecc_b200_ipc_open(const void* handle64, void** d_ptr);  /* in another process on the same node */
int   fastecc_b200_ipc_close(void* d_ptr);

/* Replaces  uint32_t hash(T** data, size_t N, size_t SIZE)   main.cpp:203-212: the rolling checksum the reference's
 * driver prints before and after a transform, walked through data[i] in block order (host memory).  Sequential by
 * construction (about one second for 2 GiB); used to compare results with the reference's published / golden hashes. */
uint32_t fastecc_b200_hash_u32(uint32_t* const* data, size_t N, size_t SIZE_words);

/* Counters for benchmarking: kernels launched by this library since init (all entry points). */
unsigned long long fastecc_b200_kernel_launches(void);

/* Pinned host memory helpers for callers that want the fast host path (cudaHostAlloc / cudaFreeHost). */
void* fastecc_b200_host_alloc(size_t bytes);
void  fastecc_b200_host_free(void* p);

#ifdef __cplusplus
}
#endif
#endif
