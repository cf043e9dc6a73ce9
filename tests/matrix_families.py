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
"""
from __future__ import annotations

import numpy as np

GRADED = (2, 3, 4, 6, 8, 12)
FAMILIES = (("uniform", "centered", "normal") + tuple(f"graded{k}" for k in GRADED) +
            ("colscale", "tiny", "huge", "rowscale", "triangular", "zerorows", "kahan", "zerocol_wide", "zerocol_narrow"))
COMPLEX_FAMILIES = ("centered", "graded6", "colscale")
NAN_FAMILIES = ("zerocol_wide", "zerocol_narrow")


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
    """Index of the exactly zero column of the zerocol families."""
    if family == "zerocol_wide":
        return 128 * (n // 256) + 61 if n >= 128 else n // 2
    return 32 * (n // 64) + 16 if n >= 32 else n // 2


def zero_rows(m: int, n: int) -> int:
    """Number of exactly zero rows at the bottom of the zerorows family (odd, so the non-zero row count is odd too)."""
    return max(1, (m - n) // 2) | 1


def singular(family: str, m: int, n: int) -> bool:
    """True where the family is rank deficient by construction at this shape (no solution to compare): zerorows once its
    zero block leaves fewer than n non-zero rows (m = n, for one), and the zero-column families."""
    if family == "zerorows":
        return m - zero_rows(m, n) < n
    return family in NAN_FAMILIES


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
    if family == "centered":
        a = (rng.random((m, n)) - 0.5) + 1j * (rng.random((m, n)) - 0.5)
    elif family.startswith("graded"):
        k = int(family[6:])
        a = (_orth(rng, m, n, True) * np.logspace(0, -k, n)) @ _orth(rng, n, n, True).conj().T
    elif family == "colscale":
        a = (rng.standard_normal((m, n)) + 1j * rng.standard_normal((m, n))) * 10.0 ** rng.uniform(-120, 120, n)
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
