"""numpy restatement of the device's triangular-pentagonal QR (dhqr_qr_append_f64 / dhqr_apply_qt_append_f64, DESIGN §2.10):
[R; B] = Q~ [R'; 0] in outer panels of 128 columns, each four 32-column panels factored column by column with the 32-wide block
update of the rest of the outer panel after each, then the 128-wide block update of the trailing columns.

Storage as on the device: R is an (n, n) array whose strict upper triangle is R's (its diagonal and lower part are never read or
written), alpha = diag(R); B (k, n) is overwritten with the reflector tails V2; vtop[j] is the top of reflector j, which sits on
row j of the R block.  H~_j = I - v~_j v~_j' with ||v~_j||^2 = 2 (or 0 for a zero column)."""
import numpy as np

NB, IB = 128, 32


def _panel(R, alpha, B, vtop, j0, nc):
    for j in range(j0, j0 + nc):
        x0 = alpha[j]
        t = B[:, j] @ B[:, j:j0 + nc]                    # the exchanged totals: B[:, j]' B[:, c], c >= j
        s = np.sqrt(t[0] + x0 * x0)
        if s == 0.0:
            al, f = 0.0, 0.0
        else:
            al = -s if x0 >= 0.0 else s                  # a zero x0 counts as positive
            f = 1.0 / np.sqrt(s * (s + abs(x0)))
        vt = f * (x0 - al)
        w = f * t[1:] + vt * R[j, j + 1:j0 + nc]
        R[j, j + 1:j0 + nc] -= vt * w
        B[:, j] *= f
        B[:, j + 1:j0 + nc] -= np.outer(B[:, j], w)
        alpha[j], vtop[j] = al, vt


def _block(V2, vt, X, C, trans=False):
    """[X; C] <- Q~_blk' [X; C] (trans: Q~_blk [X; C]) for V~ = [diag(vt); V2]: W = V2' C + diag(vt) X, T from V2'V2."""
    if X.shape[1] == 0:
        return
    W = V2.T @ C + vt[:, None] * X
    Tinv = np.eye(V2.shape[1]) + np.triu(V2.T @ V2, 1)
    T = np.linalg.inv(Tinv)
    Y = -(T if trans else T.T) @ W
    C += V2 @ Y
    X += vt[:, None] * Y


def qr_append(R, alpha, B):
    """Returns (R, alpha, V2, vtop): copies, R' in R's strict upper triangle and alpha."""
    R, alpha, B = np.array(R, dtype=float), np.array(alpha, dtype=float), np.array(B, dtype=float)
    n = alpha.size
    vtop = np.zeros(n)
    for k0 in range(0, n, NB):
        kb = min(NB, n - k0)
        for o in range(0, kb, IB):
            cs, w = k0 + o, min(IB, kb - o)
            _panel(R, alpha, B, vtop, cs, w)
            _block(B[:, cs:cs + w], vtop[cs:cs + w], R[cs:cs + w, cs + w:k0 + kb], B[:, cs + w:k0 + kb])
        _block(B[:, k0:k0 + kb], vtop[k0:k0 + kb], R[k0:k0 + kb, k0 + kb:], B[:, k0 + kb:])
    return R, alpha, B, vtop


def apply_append(V2, vtop, c, e, trans=False):
    """[c; e] <- Q~' [c; e] (trans: Q~ [c; e]) block by block, as the device does; returns copies."""
    c, e = np.array(c, dtype=float), np.array(e, dtype=float)
    n = vtop.size
    blocks = list(range(0, n, NB))
    for o in (reversed(blocks) if trans else blocks):
        kb = min(NB, n - o)
        _block(V2[:, o:o + kb], vtop[o:o + kb], c[o:o + kb], e, trans)
    return c, e


def lapack_form(V2, vtop):
    """LAPACK's unit-top convention (dtpqrt): tau = vtop^2 and v = V2 / vtop (columns with vtop = 0 give tau = 0, v = 0)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        v = np.where(vtop != 0.0, V2 / np.where(vtop != 0.0, vtop, 1.0), 0.0)
    return vtop ** 2, v
