"""Bank-conflict count of the CTA-level tile schedule (ntt_tile.cuh): for every shared-memory access instruction of a
tile (round_read / round_write_tile, brev or identity placement) the number of extra wavefronts a warp needs.
LDS.64 / STS.64 are served per half-warp: 16 lanes x 8 B = 128 B = all 32 banks when conflict-free.
Geometry: CTA threads (256: 64 KiB tiles; 512: the wide 128 KiB tiles), `python tools/banksim_cta.py [threads ...]`.
Optional layout: the popcount-parity row swap (row ^= parity(row >> 1)) used by the cp.async version of the kernel."""
import sys

def brev(x, bits):
    r = 0
    for i in range(bits): r |= ((x >> i) & 1) << (bits - 1 - i)
    return r

def parity(x): return bin(x).count("1") & 1

def q2log_of(LR, threads):
    """log2 of the word pairs per tile row (thread_pos): a tile holds threads * 64 words"""
    return (threads * 64).bit_length() - 2 - LR

def addresses(LR, k, use_brev, tid, threads=256):
    """uint2 indices of the 32 accesses of thread tid in round k (FECC_SLOT_LOOP)"""
    q2log = q2log_of(LR, threads)
    q2, j = tid & ((1 << q2log) - 1), tid >> q2log
    lb = 0 if k == 0 else LR - 5
    jlow = j & ((1 << lb) - 1)
    jbase = ((j >> lb) << (lb + 5)) | jlow
    if use_brev:
        a = (brev(jbase, LR) << q2log) | q2
        step = 1 << (LR - 5 - lb + q2log)
    else:
        a = (jbase << q2log) | q2
        step = 1 << (lb + q2log)
    return [a + i * step for i in range(32)]

def extra_wavefronts(LR, k, use_brev, swap, threads=256):
    q2log = q2log_of(LR, threads)
    extra = total = 0
    for warp in range(threads // 32):
        per_thread = [addresses(LR, k, use_brev, warp * 32 + l, threads) for l in range(32)]
        for i in range(32):
            for half in (range(0, 16), range(16, 32)):
                banks = {}
                for l in half:
                    a = per_thread[l][i]
                    row, q2 = a >> q2log, a & ((1 << q2log) - 1)
                    if swap: row ^= parity(row >> 1)
                    byte = (row << (q2log + 3)) + q2 * 8
                    banks.setdefault((byte >> 3) & 15, set()).add(byte)
                extra += max(len(v) for v in banks.values()) - 1
                total += 1
    return extra, total

if __name__ == "__main__":
    for threads in [int(a) for a in sys.argv[1:]] or [256, 512]:
        for LR in (10, 9, 8):
            for swap in (False, True):
                parts = []
                for name, k, b in (("first transform round 0", 0, True), ("first transform round 1", 1, True), ("second transform round 0", 0, False), ("second transform round 1", 1, False)):
                    e, t = extra_wavefronts(LR, k, b, swap, threads)
                    parts.append("%s: %d/%d" % (name, e, t))
                print("%d threads LR=%d %s  extra wavefronts / half-warp accesses:  %s" % (threads, LR, "parity-swapped rows" if swap else "natural rows (TMA)  ", "; ".join(parts)))
