"""Regenerates / cross-checks tests/golden/survey_8c.json, vectors.npz and reference_cross.json against the reference
compiled in oracle/_ref.

Needs oracle/_ref built from a reference tree (oracle/Makefile, REF=<path>).  Usage: python tests/golden/make_goldens.py [--write]
--write rewrites vectors.npz and reference_cross.json; without it the committed files are only verified against what the
reference computes here.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import oracle_lib as ol  # noqa: E402


def main():
    o, r = ol.load_oracle(), ol.load_ref()
    assert r is not None, "oracle/_ref/libfastecc_ref.so missing (build it from a reference tree: make -C oracle REF=<path>)"
    g = json.load(open(os.path.join(HERE, "survey_8c.json")))
    bad = 0

    def chk(name, got, want):
        nonlocal bad
        if got != want:
            bad += 1
            print("MISMATCH", name, got, want)

    for k, v in g["gf_root"].items():
        chk("root" + k, r.ref_gf_root(1 << int(k)), v)
    for k, v in g["gf_inv_pow2"].items():
        chk("inv" + k, r.ref_gf_inv(1 << int(k)), v)
    for L, (h0, h1) in g["ntt_fillA_4096B"].items():
        L = int(L)
        if L > 16 and "--big" not in sys.argv:
            continue
        a = ol.fill_A(o, 1 << L, 1024)
        chk("ntt h0 %d" % L, ol.ohash(o, a), h0)
        r.ref_mfa_ntt_flat(a.ctypes.data, 1 << L, 1024, 0)
        chk("ntt h1 %d" % L, ol.ohash(o, a), h1)
    for fill, key in ((ol.fill_A, "encode_fillA"), (ol.fill_B, "encode_fillB")):
        for L, S, h0, h1 in g[key]:
            if L > 16 and "--big" not in sys.argv:
                continue
            a = fill(o, 1 << L, S)
            chk("enc h0 %d %d" % (L, S), ol.ohash(o, a), h0)
            r.ref_rs_encode_flat(a.ctypes.data, 1 << L, S)
            chk("enc h1 %d %d" % (L, S), ol.ohash(o, a), h1)
    # full-buffer vectors (not just hashes) produced by the reference itself, committed as a small fixture
    vec = {}
    for L, S in ((1, 4), (2, 1), (2, 8), (3, 8), (4, 8), (6, 8), (8, 8), (10, 4), (11, 4), (5, 13)):
        N = 1 << L
        x = ol.fill_B(o, N, S)
        vec["in_%d_%d" % (L, S)] = x.copy()
        for inv in (0, 1):
            y = x.copy(); r.ref_mfa_ntt_flat(y.ctypes.data, N, S, inv); vec["ntt%d_%d_%d" % (inv, L, S)] = y
        y = x.copy(); r.ref_rs_encode_flat(y.ctypes.data, N, S); vec["enc_%d_%d" % (L, S)] = y
    # the reference's results on the inputs of tests/test_oracle.py::test_against_compiled_reference
    def ref_ntt(a, inv):
        b = a.copy(); r.ref_mfa_ntt_flat(b.ctypes.data, b.shape[0], b.shape[1], inv); return b

    def ref_encode(a):
        b = a.copy(); r.ref_rs_encode_flat(b.ctypes.data, b.shape[0], b.shape[1]); return b
    cross = ol.cross_record(o, lambda x, y: (r.ref_gf_mul(x, y), r.ref_gf_add(x, y), r.ref_gf_sub(x, y)), ref_ntt, ref_encode)
    path = os.path.join(HERE, "vectors.npz")
    cross_path = os.path.join(HERE, "reference_cross.json")
    if "--write" in sys.argv:
        np.savez_compressed(path, **vec)
        with open(cross_path, "w") as f:
            json.dump(cross, f, separators=(",", ":"))
        print("wrote", path, cross_path)
    else:
        old = np.load(path)
        for k, v in vec.items():
            if not np.array_equal(old[k], v):
                bad += 1
                print("MISMATCH vector", k)
        chk("reference_cross.json", json.load(open(cross_path)), cross)
    print("goldens", "MISMATCH" if bad else "verified against the compiled reference")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
