"""Small workload for compute-sanitizer (tools/gpu/sanitize.sh): every kernel family of the library at orders where the tile
loops, the table double-buffering and the TMA / mbarrier hand-offs are all exercised, checked against the oracle."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_lib as ol          # noqa: E402
import fastecc_b200 as fe        # noqa: E402

fe.init(0)
o = ol.load_oracle()
for L, S in ((11, 256), (12, 128), (13, 64), (10, 16), (6, 1024)):
    N = 1 << L
    a = ol.fill_B(o, N, S)
    t = torch.from_numpy(a.view(np.int32)).cuda()
    fe.rs_encode_dev(t)
    assert np.array_equal(t.cpu().numpy().view(np.uint32), ol.o_encode(o, a)), ("encode", L, S)
    t = torch.from_numpy(a.view(np.int32)).cuda()
    fe.ntt_dev(t, False)
    assert np.array_equal(t.cpu().numpy().view(np.uint32), ol.o_ntt(o, a, False)), ("ntt", L, S)
    if L >= 11:
        t = torch.from_numpy(a.view(np.int32)).cuda()
        fe.rs_encode_asym_dev(t, N // 2)
        assert np.array_equal(t[:N // 2].cpu().numpy().view(np.uint32), ol.o_encode(o, a)[::2]), ("asym", L, S)
    b = a.copy(); fe.EncodeReedSolomon_body(b, N, S)
    assert np.array_equal(b, ol.o_encode(o, a)), ("host", L, S)
for N, M, S in ((3 << 12, (3 << 12) // 8, 16), (3 << 11, 1, 1024)):     # the encode into fewer parity blocks (radix_fold_kernel; folded by 2 in the second)
    a = ol.fill_B(o, N, S)
    t = torch.from_numpy(a.view(np.int32)).cuda()
    fe.rs_encode_asym_mixed_dev(t, M)
    full = torch.from_numpy(a.view(np.int32)).cuda()
    fe.rs_encode_mixed_dev(full)
    assert torch.equal(t[:M], full[::N // M]), ("asym mixed", N, M, S)
for N, M, S in ((3 << 10, 3 << 6, 1022), (1 << 12, 1 << 12, 16)):         # repair in place (repair.cu's four kernels, a partial last chunk in the first)
    a = ol.fill_B(o, N, S)
    data = torch.zeros((N, (S + 3) // 4 * 4), dtype=torch.int32, device="cuda")
    data[:, :S] = torch.from_numpy(a.view(np.int32)).cuda()
    par = data.clone()
    fe.rs_encode_asym_mixed_dev(par[:, :S], M)
    par = par[:M].clone()
    want_d, want_p = data.clone(), par.clone()
    lost_d, lost_p = list(range(0, N, N // (M // 2))), list(range(1, M, 2))
    data[lost_d, :S] = -1
    par[lost_p, :S] = -1
    fe.rs_repair_dev(data[:, :S], par[:, :S], lost_d, lost_p)
    assert torch.equal(data, want_d) and torch.equal(par, want_p), ("repair", N, M, S)
for B, N, M, S in ((37, 12, 4, 7), (5, 64, 16, 1022), (9, 18, 9, 33)):  # the batch encode: M < 8 and M >= 8, SIZE % 4 != 0
    data = torch.randint(-(1 << 31), 1 << 31, (B, N, (S + 3) // 4 * 4), dtype=torch.int32, device="cuda")[..., :S]
    par = fe.rs_encode_batch_dev(data, M=M)
    for b in (0, B - 1):
        one = data[b].clone()
        fe.rs_encode_asym_mixed_dev(one, M)
        assert torch.equal(par[b], one[:M]), ("batch", B, N, M, S, b)
for B, N, M, S, ld, lp in ((37, 12, 4, 7, [2, 11], [0]), (5, 64, 16, 1022, [0, 9, 63], [3, 15]), (9, 18, 9, 33, [], [1, 8]),
                          (6, 9, 3, 5, [0, 4, 8], [])):   # the batched degraded read: M < 8 and M >= 8, SIZE % 4 != 0, a = 0 with wanted parity, a = M
    data = torch.randint(-(1 << 31), 1 << 31, (B, N, (S + 3) // 4 * 4), dtype=torch.int32, device="cuda")[..., :S]
    par = fe.rs_encode_batch_dev(data, M=M)
    out = fe.rs_reconstruct_batch_dev(data, par, ld, lp)
    for b in (0, B - 1):
        assert torch.equal(out[b], fe.rs_reconstruct_dev(data[b], par[b], ld, lp)), ("reconstruct batch", B, N, M, S, b)
for B, N, M, S, ch in ((37, 12, 4, 7, [2, 11]), (5, 64, 16, 1022, [0, 9, 63]), (9, 18, 9, 33, list(range(18))),
                      (6, 64, 1, 5, list(range(0, 64, 2)))):   # the batch update: M < 8 and M >= 8, SIZE % 4 != 0, row slices
    data = torch.randint(-(1 << 31), 1 << 31, (B, N, (S + 3) // 4 * 4), dtype=torch.int32, device="cuda")[..., :S]
    par = fe.rs_encode_batch_dev(data, M=M)
    new = torch.randint(-(1 << 31), 1 << 31, (B, len(ch), (S + 3) // 4 * 4), dtype=torch.int32, device="cuda")[..., :S]
    pad = lambda x: torch.empty((x.shape[0], (S + 3) // 4 * 4), dtype=torch.int32, device="cuda")[:, :S].copy_(x)
    one = [(pad(data[b]), pad(par[b])) for b in (0, B - 1)]
    fe.rs_update_batch_dev(data, par, ch, new)
    for (d, p), b in zip(one, (0, B - 1)):
        fe.rs_update_dev(d, p, ch, new[b])
        assert torch.equal(par[b], p) and torch.equal(data[b], d), ("update batch", B, N, M, S, b)
for B, N, M, S, ch in ((7, 12, 4, 7, [0, 5, 11]), (4, 32, 8, 130, [3])):   # one [B][N + M + k][pitch] buffer, updated in place
    k, pitch = len(ch), (S + 3) // 4 * 4
    buf = torch.randint(-(1 << 31), 1 << 31, (B, N + M + k, pitch), dtype=torch.int32, device="cuda")
    fe.rs_encode_batch_dev(buf[:, :N, :S], buf[:, N:N + M, :S])
    want = buf.clone()
    want[:, ch, :S] = buf[:, N + M:, :S]
    fe.rs_encode_batch_dev(want[:, :N, :S], want[:, N:N + M, :S])
    fe.rs_update_batch_dev(buf[:, :N, :S], buf[:, N:N + M, :S], ch, buf[:, N + M:, :S])
    assert torch.equal(buf[:, N:N + M, :S], want[:, N:N + M, :S]), ("update batch, one buffer", B, N, M, S)
raw = torch.randint(0, 256, (64, 4096), dtype=torch.uint8, device="cuda")
w = fe.bytes_to_gfp_dev(raw)
assert bool((fe.gfp_to_bytes_dev(w, 1024) == raw).all())
torch.cuda.synchronize()
print("sanitize workload ok: %d kernels launched" % fe.kernel_launches())
