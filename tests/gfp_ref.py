"""A plain GF(P) reference of the transforms and the encodes, P = 0xFFF00001, that uses no library code: torch int64 on any
device (CPU tensors in the non-GPU tests, CUDA tensors beside the kernels).  Test-only.

  mulmod          products split one operand into 16-bit halves, so every intermediate stays below 2^49
  RootPowers      omega^e for omega = GF_Root(n) from a two-level table hi[e >> 12] * lo[e & 4095]
  ntt_rows        X[k] = sum_n x_n omega^(n*k mod N), omega = GF_Root(N) (forward) or its inverse (unnormalised)
  encode_rows     parity_j = f(rho^(2j+1)), rho = GF_Root(2N), f(rho^(2i)) = data_i, by the circulant form below
  closed forms    monomial stripes and their 2N-row code words for the encodes and the decoders, deltas and geometric
                  columns for the transforms

Encode by definition: the Lagrange basis of the N-th roots of unity rho^(2i) evaluated at rho^(2j+1), where rho^N = -1, gives
parity_j = (2/N) * sum_i data_i * c_((j-i) mod N) with c_d = 1 / (1 - rho^(2d+1)).  Asymmetric parity j' is row (N/M)*j'."""
import torch

P = 0xFFF00001
G = 19                     # GF_Root(n) = G^((P-1)/n)
_B = 4096                  # low table of RootPowers


def mulmod(a, b):
    """a * b mod P for int64 tensors (or ints) with 0 <= a, b < P."""
    hi, lo = b >> 16, b & 0xFFFF
    return ((a * hi % P) * 65536 + a * lo) % P


def powmod(x, e):
    """x^e mod P elementwise for an int64 tensor x, a Python int e >= 0 (square and multiply)."""
    r = torch.ones_like(x)
    x = x % P
    while e:
        if e & 1:
            r = mulmod(r, x)
        x = mulmod(x, x)
        e >>= 1
    return r


def inv(x):
    """x^(P-2): the inverse of every nonzero word (0 -> 0)."""
    return powmod(x, P - 2)


def root(n):
    assert (P - 1) % n == 0
    return pow(G, (P - 1) // n, P)


class RootPowers:
    """omega^e (e taken mod n) for omega = GF_Root(n)^sign, from hi[e >> 12] * lo[e & 4095]; tables built once per order."""

    def __init__(self, n, device="cpu", sign=1):
        self.n = n
        w = root(n) if sign > 0 else pow(root(n), P - 2, P)
        lo, v = [], 1
        for _ in range(_B):
            lo.append(v); v = v * w % P
        hi, v, step = [], 1, pow(w, _B, P)
        for _ in range((n + _B - 1) // _B):
            hi.append(v); v = v * step % P
        self.lo = torch.tensor(lo, dtype=torch.int64, device=device)
        self.hi = torch.tensor(hi, dtype=torch.int64, device=device)

    def __call__(self, e):
        e = e % self.n
        return mulmod(self.hi[e >> 12], self.lo[e & (_B - 1)])


_cache = {}


def powers(n, device, sign=1):
    key = (n, str(device), sign)
    if key not in _cache:
        if len(_cache) > 16:
            _cache.clear()
        _cache[key] = RootPowers(n, device, sign)
    return _cache[key]


def as_words(t):
    """int32 / uint32 / int64 words -> int64 in [0, 2^32)."""
    return t.to(torch.int64) & 0xFFFFFFFF


def ntt_rows(x, rows, inverse=False):
    """Rows `rows` of the order-N transform of every column of x (N x C, words below P), by definition: [len(rows), C]."""
    x = as_words(x) % P
    N = x.shape[0]
    pw = powers(N, x.device, -1 if inverse else 1)
    n = torch.arange(N, dtype=torch.int64, device=x.device)
    out = []
    for k in rows:
        w = pw(n * int(k))
        out.append((mulmod(x, w[:, None]).sum(0)) % P)
    return torch.stack(out)


def encode_coeffs(N, device):
    """(c_d for d < N, 2/N mod P): c_d = 1 / (1 - rho^(2d+1)), rho = GF_Root(2N)."""
    d = torch.arange(N, dtype=torch.int64, device=device)
    r = powers(2 * N, device)(2 * d + 1)
    return inv((1 - r) % P), 2 * pow(N, P - 2, P) % P


def encode_rows(data, rows):
    """Parity rows `rows` of the N -> N encode of every column of data (N x C, words below P), by definition: [len(rows), C].
    Asymmetric parity j' into M blocks is row (N/M)*j'."""
    x = as_words(data) % P
    N = x.shape[0]
    c, two_over_n = encode_coeffs(N, x.device)
    i = torch.arange(N, dtype=torch.int64, device=x.device)
    out = []
    for j in rows:
        w = c[(int(j) - i) % N]
        out.append(mulmod((mulmod(x, w[:, None]).sum(0)) % P, two_over_n))
    return torch.stack(out)


# ---- closed forms ------------------------------------------------------------------------------------------------------
def monomial_data(N, degrees, rows=None, device="cpu"):
    """data_i = rho^(2*i*m_c) in column c (m_c = degrees[c] < N), rho = GF_Root(2N): the stripe of the polynomial z^m_c."""
    i = _rows(N, rows, device)
    m = torch.as_tensor(degrees, dtype=torch.int64, device=device)
    return powers(2 * N, device)(2 * i[:, None] * m[None, :])


def monomial_parity(N, degrees, rows=None, device="cpu", decimation=1):
    """parity_j = rho^((2*decimation*j + 1)*m_c): the full encode (decimation 1), or the asymmetric one into N/decimation
    blocks (decimation = N/M)."""
    j = _rows(N // decimation, rows, device)
    m = torch.as_tensor(degrees, dtype=torch.int64, device=device)
    return powers(2 * N, device)((2 * decimation * j[:, None] + 1) * m[None, :])


def codeword_rows(N, degrees, rows=None, device="cpu"):
    """Rows of the 2N-row code word of the monomial stripe: row x = rho^(x*m_c) (data i is row 2i, parity j is row 2j + 1)."""
    return powers(2 * N, device)(_rows(2 * N, rows, device)[:, None] * torch.as_tensor(degrees, dtype=torch.int64, device=device)[None, :])


def delta_ntt_columns(N, positions, rows=None, device="cpu", inverse=False):
    """A delta at row n_c of column c transforms to X_k = omega^(+-n_c*k)."""
    k = _rows(N, rows, device)
    n = torch.as_tensor(positions, dtype=torch.int64, device=device)
    return powers(N, device, -1 if inverse else 1)(k[:, None] * n[None, :])


def geometric_ntt_input(N, freqs, rows=None, device="cpu", inverse=False):
    """x_n = omega^(-+m_c*n): its transform is N at k = m_c and 0 elsewhere (ntt_spike)."""
    n = _rows(N, rows, device)
    m = torch.as_tensor(freqs, dtype=torch.int64, device=device)
    return powers(N, device, 1 if inverse else -1)(n[:, None] * m[None, :])


def ntt_spike(N, freqs, rows=None, device="cpu"):
    k = _rows(N, rows, device)
    m = torch.as_tensor(freqs, dtype=torch.int64, device=device)
    return (k[:, None] == m[None, :]).to(torch.int64) * (N % P)


def _rows(n, rows, device):
    if rows is None:
        return torch.arange(n, dtype=torch.int64, device=device)
    if isinstance(rows, slice):
        return torch.arange(n, dtype=torch.int64, device=device)[rows]
    return torch.as_tensor(rows, dtype=torch.int64, device=device)


def special_values(N, boundaries=(), count=8, seed=0):
    """0, 1, N-1, N/2, the given plan boundaries +-1 (those below N), then seeded random values below N, `count` in all or more."""
    vals = [0, 1, N - 1, N // 2]
    for b in boundaries:
        vals += [b - 1, b, b + 1]
    vals = [v for v in dict.fromkeys(vals) if 0 <= v < N]
    g = torch.Generator().manual_seed(seed * 1000003 + N)
    while len(vals) < count:
        vals.append(int(torch.randint(0, N, (1,), generator=g)))
    return vals
