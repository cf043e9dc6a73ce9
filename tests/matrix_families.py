"""Seeded test matrices beyond U[0,1): sign, conditioning, scaling and structure that the factorisation's paths have to survive.

``make(family, m, n, seed)`` returns a Fortran-ordered float64 (m, n) array; ``make_complex`` the complex128 families.  Every
matrix is a function of (family, m, n, seed) through numpy's PCG64 stream, so nothing is stored under tests/golden/.

Families:
  uniform          U[0,1), what the rest of the suite uses (one dominant singular value, all entries positive)
  centered         U[-1/2, 1/2)
  normal           N(0,1)
  graded{k}        U diag(logspace(0, -k, n)) V' with random orthonormal U, V: kappa = 10^k, k in {2,3,4,6,8,12}.  A 128-column
                   panel of it is better conditioned than the whole matrix: on an H100 the wide chain's guard (est <= 1000)
                   accepts every panel at 2048 x 1024, and refuses 3 of the panels at k = 12, 4099 x 640 (redone by the
                   32-column chain)
  colscale         N(0,1) with column j scaled by 10^e_j, e_j uniform in [-120, 120]
  tiny / huge      N(0,1) times 1e-150 / 1e+150: the column norms stay inside double's range (m * 1e300 < 1.8e308, and
                   s * (s + |x|) of S:131 stays above the smallest normal), while squares of entries below ~1.5e-4 times the
                   scale are subnormal at 1e-150
  rowscale         N(0,1) with row i scaled by 10^u_i, u_i uniform in [-8, 8]
  triangular       upper triangular N(0,1) in the top n rows, zeros below: every pivot column is s e_j and v = +-sqrt(2) e_j
  zerorows         N(0,1) with a block of exactly zero rows at the bottom
  kahan            the Kahan matrix diag(s^i) (I - c striu(1)) in the top n rows, zeros below, with (1+c)^(n-1) = 1e8
  zerocol_wide     N(0,1) with one exactly zero column in the middle of a 128-column panel
  zerocol_narrow   N(0,1) with one exactly zero column in the middle of a 32-column panel
A zero column makes the reference's f = 1/sqrt(0) = Inf (S:131): that column and everything it touches afterwards is NaN.

``make_complex`` has a twin of every family above except the two zero-column ones (both parts N(0,1) where the real family is
N(0,1), U[0,1) where it is uniform; kahan with random unit-modulus row and column phases, which keep its singular values) and:
  zerocol_first / zerocol_mid / zerocol_last
                   N(0,1) + i N(0,1) with one exactly zero column: the first, a middle or the last column of a 64-column
                   complex panel (CPW of dhqr_complex.cuh)
  imag             i N(0,1): every real part exactly +0
  zerolead         m >= 2n: rows [0, n) exactly +0, rows [n, 2n) diag(d) with complex |d| in [1, 2), the rest N(0,1) + i N(0,1).
                   Step j leaves rows j+1..n-1 of every later column exactly +0 (v_j is zero there), so every pivot is an
                   exact +0 and takes the angle(0) branch of S:9 (alpha_j = -s), in every panel and through the blocked update
  zerolead_neg / zerolead_negneg
                   zerolead with A[0, 0] = -0 + 0i / -0 - 0i: angle = +pi / -pi, alpha_0 = s (1, -+sin(pi))
"""
from __future__ import annotations

import numpy as np

GRADED = (2, 3, 4, 6, 8, 12)
FAMILIES = (("uniform", "centered", "normal") + tuple(f"graded{k}" for k in GRADED) +
            ("colscale", "tiny", "huge", "rowscale", "triangular", "zerorows", "kahan", "zerocol_wide", "zerocol_narrow"))
COMPLEX_FAMILIES = ("centered", "graded6", "colscale")
NAN_FAMILIES = ("zerocol_wide", "zerocol_narrow")
CPW = 64                                                  # complex panel width of the library
COMPLEX_NAN_FAMILIES = ("zerocol_first", "zerocol_mid", "zerocol_last")
ZEROLEAD = ("zerolead", "zerolead_neg", "zerolead_negneg")
COMPLEX_ALL = (tuple(f for f in FAMILIES if f not in NAN_FAMILIES) + ("imag",) + ZEROLEAD + COMPLEX_NAN_FAMILIES)


def _rng(family: str, m: int, n: int, seed: int) -> np.random.Generator:
    key = [ord(ch) for ch in family] + [m, n, seed]
    return np.random.default_rng(key)


def _orth(rng, m, n, cplx=False):
    g = rng.standard_normal((m, n))
    if cplx:
        g = g + 1j * rng.standard_normal((m, n))
    q, r = np.linalg.qr(g)
    d = np.diagonal(r)
    return q * (d / np.abs(d))          # unique Q: positive diagonal of R


def zero_column(family: str, n: int) -> int:
    """Index of the exactly zero column of the zerocol families (real and complex)."""
    if family == "zerocol_wide":
        return 128 * (n // 256) + 61 if n >= 128 else n // 2
    if family == "zerocol_narrow":
        return 32 * (n // 64) + 16 if n >= 32 else n // 2
    if n < 2 * CPW:
        return n // 2
    return CPW * (n // (2 * CPW)) + {"zerocol_first": 0, "zerocol_mid": 29, "zerocol_last": CPW - 1}[family]


def zero_rows(m: int, n: int) -> int:
    """Number of exactly zero rows at the bottom of the zerorows family (odd, so the non-zero row count is odd too)."""
    return max(1, (m - n) // 2) | 1


def singular(family: str, m: int, n: int) -> bool:
    """True where the family is rank deficient by construction at this shape (no solution to compare): zerorows once its
    zero block leaves fewer than n non-zero rows (m = n, for one), and the zero-column families."""
    if family == "zerorows":
        return m - zero_rows(m, n) < n
    return family in NAN_FAMILIES or family in COMPLEX_NAN_FAMILIES


def make(family: str, m: int, n: int, seed: int = 0) -> np.ndarray:
    assert m >= n >= 1
    rng = _rng(family, m, n, seed)
    if family == "uniform":
        a = rng.random((m, n))
    elif family == "centered":
        a = rng.random((m, n)) - 0.5
    elif family == "normal":
        a = rng.standard_normal((m, n))
    elif family.startswith("graded"):
        k = int(family[6:])
        a = (_orth(rng, m, n) * np.logspace(0, -k, n)) @ _orth(rng, n, n).T
    elif family == "colscale":
        a = rng.standard_normal((m, n)) * 10.0 ** rng.uniform(-120, 120, n)
    elif family == "tiny":
        a = rng.standard_normal((m, n)) * 1e-150
    elif family == "huge":
        a = rng.standard_normal((m, n)) * 1e150
    elif family == "rowscale":
        a = rng.standard_normal((m, n)) * 10.0 ** rng.uniform(-8, 8, m)[:, None]
    elif family == "triangular":
        a = np.zeros((m, n))
        a[:n] = np.triu(rng.standard_normal((n, n)))
    elif family == "zerorows":
        a = rng.standard_normal((m, n))
        a[m - zero_rows(m, n):] = 0.0
    elif family == "kahan":
        c = 10.0 ** (8.0 / max(n - 1, 1)) - 1.0
        s = np.sqrt(1.0 - c * c)
        a = np.zeros((m, n))
        a[:n] = (s ** np.arange(n))[:, None] * (np.eye(n) - c * np.triu(np.ones((n, n)), 1))
    elif family in NAN_FAMILIES:
        a = rng.standard_normal((m, n))
        a[:, zero_column(family, n)] = 0.0
    else:
        raise ValueError(f"unknown family {family!r}")
    return np.asfortranarray(a, dtype=np.float64)


def make_complex(family: str, m: int, n: int, seed: int = 0) -> np.ndarray:
    assert m >= n >= 1
    rng = _rng("c" + family, m, n, seed)

    def cnormal(r=m, c=n):
        return rng.standard_normal((r, c)) + 1j * rng.standard_normal((r, c))

    if family == "uniform":
        a = rng.random((m, n)) + 1j * rng.random((m, n))
    elif family == "centered":
        a = (rng.random((m, n)) - 0.5) + 1j * (rng.random((m, n)) - 0.5)
    elif family == "normal":
        a = cnormal()
    elif family.startswith("graded"):
        k = int(family[6:])
        a = (_orth(rng, m, n, True) * np.logspace(0, -k, n)) @ _orth(rng, n, n, True).conj().T
    elif family == "colscale":
        a = (rng.standard_normal((m, n)) + 1j * rng.standard_normal((m, n))) * 10.0 ** rng.uniform(-120, 120, n)
    elif family == "tiny":
        a = cnormal() * 1e-150
    elif family == "huge":
        a = cnormal() * 1e150
    elif family == "rowscale":
        a = cnormal() * 10.0 ** rng.uniform(-8, 8, m)[:, None]
    elif family == "triangular":
        a = np.zeros((m, n), dtype=np.complex128)
        a[:n] = np.triu(cnormal(n, n))
    elif family == "zerorows":
        a = cnormal()
        a[m - zero_rows(m, n):] = 0.0
    elif family == "kahan":
        phase = lambda k: np.exp(2j * np.pi * rng.random(k))
        a = phase(m)[:, None] * make("kahan", m, n) * phase(n)
    elif family in COMPLEX_NAN_FAMILIES:
        a = cnormal()
        a[:, zero_column(family, n)] = 0.0
    elif family == "imag":
        a = np.zeros((m, n), dtype=np.complex128)       # real parts +0 (1j * x would give -0 where x < 0)
        a.imag = rng.standard_normal((m, n))
    elif family in ZEROLEAD:
        if m < 2 * n:
            raise ValueError(f"{family} needs m >= 2n, got {m} x {n}")
        a = np.zeros((m, n), dtype=np.complex128)
        a[n + np.arange(n), np.arange(n)] = (1.0 + rng.random(n)) * np.exp(2j * np.pi * rng.random(n))
        a[2 * n:] = cnormal(m - 2 * n, n)
        if family != "zerolead":
            a[0, 0] = complex(-0.0, 0.0 if family == "zerolead_neg" else -0.0)
    else:
        raise ValueError(f"unknown complex family {family!r}")
    return np.asfortranarray(a, dtype=np.complex128)


def rhs(m: int, k: int = 1, seed: int = 0, cplx: bool = False) -> np.ndarray:
    """N(0,1) right-hand sides, (m,) for k == 1 else Fortran-ordered (m, k)."""
    rng = _rng("rhs", m, k, seed)
    b = rng.standard_normal((m, k))
    if cplx:
        b = b + 1j * rng.standard_normal((m, k))
    return b[:, 0].copy() if k == 1 else np.asfortranarray(b)
