"""The multi-rank path (column blocks over ranks, owner panels, V broadcast per panel, Q'b and the back-substitution handed from
rank to rank) held to the extended-precision rule of ext_rule.py on ONE H100: 2 to 4 rank processes share cuda:0 and talk through
tests/nccl_loopback.cpp, a CUDA-IPC stand-in for NCCL loaded with DHQR_NCCL_LIBRARY (harness: tests/dist_loopback.py).

What this verifies: the arithmetic of the multi-rank drivers, the order and arguments of their collectives (the stand-in refuses
two ranks whose calls do not match), and the storage contract of the hand-over.  What it does not: NCCL itself, NVLink, timing.
test_gpu_dist.py covers those on machines with two or more GPUs.

A table of err_gpu / max(err_fp64_oracle, FLOOR) per configuration and path is written to build/test_gpu_dist_ratios.md.
"""
import glob
import os
import shutil

import numpy as np
import pytest
import torch

import dhqr_b200 as D
import dist_loopback as L
import matrix_families as F
from ext_rule import COUNTERS, Ref, Table, factor_checks, nrm

pytestmark = pytest.mark.gpu

FAM5 = ("uniform", "normal", "graded12", "colscale", "kahan")
PATHS = {"default": (0, {}), "lookahead0": (0, {"lookahead": 0}), "wide_panel0": (0, {"wide_panel": 0}), "nb64": (64, {})}
REDONE = COUNTERS.index("wide_redone")


# name -> (P, m, n, column boundaries as a function of n).  Boundaries that are not multiples of 32 start panels whose
# TMA window carries 1..31 rows above the pivot row (panel_geom); an empty rank owns no panel at all.
CONFIGS = {
    "P2": (2, 2048, 1024, lambda n: [0, n // 2, n]),
    "P2bal": (2, 2048, 1024, lambda n: D.balanced_splits(2, n)),                 # [0, 724, 1024]
    "P3": (3, 2048, 1000, lambda n: D.splits(3, n)),                             # [0, 334, 667, 1000]
    "P3empty": (3, 2048, 1024, lambda n: [0, n // 2, n // 2, n]),
    "P4up": (4, 2048, 1024, lambda n: D.balanced_splits(4, n, "upstream")),      # [0, 137, 300, 512, 1024]
}


def _solve(family, m, n):
    return family not in F.NAN_FAMILIES and not F.singular(family, m, n)


def _cases(cfg):
    P, m, n, bnd = CONFIGS[cfg]
    cases = [(f"{path}/{fam}", fam, m, n, bnd(n), nb, opts, _solve(fam, m, n), "default")
             for path, (nb, opts) in PATHS.items() for fam in FAM5]
    cases += [(f"nb1/{fam}", fam, 1024, 256, bnd(256), 1, {}, _solve(fam, 1024, 256), "default") for fam in FAM5]
    if cfg == "P2bal":
        cases += [(f"default/{fam}", fam, m, n, bnd(n), 0, {}, _solve(fam, m, n), "default") for fam in F.FAMILIES if fam not in FAM5]
    if cfg == "P2":
        cases += [("default#2/uniform", "uniform", m, n, bnd(n), 0, {}, True, "default"),
                  ("default@side/uniform", "uniform", m, n, bnd(n), 0, {}, True, "side")]
    return cases


TABLE = Table("test_gpu_dist_ratios.md")


@pytest.fixture(scope="module", autouse=True)
def ratio_table():
    yield
    TABLE.write()


@pytest.fixture(scope="module")
def lib():
    d, so = L.build()
    yield so
    shutil.rmtree(d, ignore_errors=True)


@pytest.fixture(scope="module")
def spawn(lib, tmp_path_factory):
    """spawn(name, P, job, *args): the per-rank results of one run of ``job``, cached per name for the module."""
    cache = {}

    def get(name, P, job, *args):
        if name not in cache:
            out = str(tmp_path_factory.mktemp(name))
            try:
                cache[name] = L.run(P, job, out, lib, args)
            except L.Skip as e:
                cache[name] = e
            finally:
                assert not glob.glob(os.path.join(out, "dhqr-loopback-*")), f"{name}: a control file outlived the run"
        res = cache[name]
        if isinstance(res, L.Skip):
            pytest.skip(f"the loopback transport cannot run here: {res}")
        return res
    return get


@pytest.fixture(scope="module")
def refs(oracle, coracle):
    cache = {}

    def get(family, m, n, nrhs=None):
        key = (family, m, n, nrhs)
        if key not in cache:
            cache[key] = Ref(coracle, oracle, family, m, n, nrhs=nrhs)
        return cache[key]
    return get


def _same(ranks, key):
    """The value of ``key`` on rank 0, after asserting it is bitwise equal on every rank."""
    v = ranks[0][key]
    for r, res in enumerate(ranks[1:], 1):
        assert res[key].tobytes() == v.tobytes(), f"{key} differs between rank 0 and rank {r}"
    return v


def _check_case(cfg, ranks, refs, case):
    key, fam, m, n, bounds, nb, opts, solve, _ = case
    path = f"{cfg} {key.split('/')[0]}"
    H = np.hstack([ranks[r][key + "/H"] for r in range(len(ranks))])
    assert H.shape == (m, n)
    alpha = _same(ranks, key + "/alpha")
    cnt = np.stack([res[key + "/counters"] for res in ranks])
    note = f"bounds {bounds}, counters per rank {cnt.tolist()} ({', '.join(COUNTERS)})"
    if fam == "zerocol_wide" and nb == 0 and not opts:        # the refusal travels with V: every rank restarts, together
        assert (cnt[:, REDONE] >= 1).all() and (cnt[:, REDONE] == cnt[0, REDONE]).all(), f"{path} {fam}: {note}"
    ref = refs(fam, m, n)
    gpu, absolute = factor_checks(path, ref, H, alpha, note)
    e64 = dict(ref.e64)
    if solve:
        assert ref.solve
        got = {k: _same(ranks, f"{key}/{k}") for k in ("qtb1", "qtb0", "qb", "x1", "x0")}
        for k, g in (("qtb", got["qtb1"]), ("qb", got["qb"]), ("x", got["x1"][:n])):
            gpu[k], e64[k] = ref.solve_errors(k, g, 0)
        TABLE.check(path, ref, gpu, e64, absolute, note)
        alt = {k: ref.solve_errors(k, g, 0) for k, g in (("qtb", got["qtb0"]), ("x", got["x0"][:n]))}
        TABLE.check(path + " qt_vec=0 bs_wave=0", ref, {k: v[0] for k, v in alt.items()}, {k: v[1] for k, v in alt.items()},
                    note=note)
    else:
        TABLE.check(path, ref, gpu, e64, absolute, note)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", [2, 3])
def test_transport_is_bitwise(spawn, lib, P):
    # the stand-in alone: every root and pair, in place and out of place, odd sizes and sizes over 1 and 3 staging slots
    ranks = spawn(f"transport{P}", P, "transport", lib)
    checks = [int(r["checks"]) for r in ranks]
    assert min(checks) > 0
    for r, res in enumerate(ranks):
        assert int(res["rc_type"]) == 4, f"rank {r}: an unsupported data type must give ncclInvalidArgument"
        assert int(res["rc_count"]) == 5, f"rank {r}: ranks that disagree on a count must get ncclInvalidUsage"
        assert "mismatch" in str(res["text"]), str(res["text"])


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_extended_rule(spawn, refs, cfg):
    # every path x family of one configuration; alpha, Q'b, Qb and x replicated bit for bit on every rank
    P = CONFIGS[cfg][0]
    cases = _cases(cfg)
    ranks = spawn(cfg, P, "matrix", cases)
    failures = []
    for case in cases:
        try:
            _check_case(cfg, ranks, refs, case)
        except AssertionError as e:
            failures.append(f"{case[0]}: {e}")
    assert not failures, "\n".join(failures)


def test_runs_are_bitwise_reproducible(spawn):
    # two runs, and a run on a low-priority non-blocking side stream, give the bits of the first run on every rank
    ranks = spawn("P2", 2, "matrix", _cases("P2"))
    for res in ranks:
        for other in ("default#2", "default@side"):
            for what in ("H", "alpha", "qtb1", "qtb0", "qb", "x1", "x0"):
                assert res[f"{other}/uniform/{what}"].tobytes() == res[f"default/uniform/{what}"].tobytes(), f"{other} {what}"


def test_large_balanced(spawn, refs):
    bounds = D.balanced_splits(2, 2048)
    cases = [(f"default/{fam}", fam, 8192, 2048, bounds, 0, {}, True, "default") for fam in ("normal", "graded6")]
    ranks = spawn("P2big", 2, "matrix", cases)
    for case in cases:
        _check_case("P2big", ranks, refs, case)


@pytest.mark.parametrize("cfg", ["P2bal", "P3"])
def test_rhs_blocks_leave_padding_alone(spawn, refs, cfg):
    # nrhs = 3 and 65 with ldb = m + 5: the padding rows hold NaNs naming the rank; the hand-over of b between ranks must move
    # the m x nrhs block only, so every rank gets its own padding back bit for bit
    P, m, n, bnd = CONFIGS[cfg]
    ranks = spawn("rhs_" + cfg, P, "rhs_blocks", "normal", m, n, bnd(n), (3, 65))
    for r, res in enumerate(ranks):
        for k in (3, 65):
            for what in ("qtb", "qb", "x"):
                assert bool(res[f"k{k}/{what}_pad_ok"]), f"rank {r}: padding rows changed by {what} with nrhs={k}"
    for k, ref, c0 in ((3, refs("normal", m, n), 1), (65, refs("normal", m, n, nrhs=65), 0)):
        for what in ("qtb", "qb", "x"):
            got = _same(ranks, f"k{k}/{what}")
            for j in range(k):
                g, e = ref.solve_errors(what, got[:n, j] if what == "x" else got[:, j], c0 + j)
                TABLE.check(f"{cfg} nrhs={k} ldb=m+5", ref, {what: g}, {what: e}, note=f"rhs {j}")


def test_restart_after_a_refused_panel(spawn, oracle, coracle):
    # column 300 nearly equals column 270: the wide chain refuses the panel [256, 384) on its owner's device, every rank learns
    # of it with the broadcast V buffer and all of them redo it.  Owned by rank 1 ([0, 256, 512]), then by rank 0 ([0, 384, 512]).
    m, n, dup = 2048, 512, 300
    parts = [[0, 256, 512], [0, 384, 512]]
    ranks = spawn("restart", 2, "restart", m, n, dup, parts)
    A0 = coracle.fill_uniform(0, m, n)
    A0[:, dup] = A0[:, dup - 30] + 1e-11 * coracle.fill_uniform(13, m, 1)[:, 0]
    Href, _ = coracle.qr(A0.copy(order="F"))
    for i, b in enumerate(parts):
        for r, res in enumerate(ranks):
            assert int(res[f"{i}/redone"]) == 1, f"partition {b}: rank {r} restarted {int(res[f'{i}/redone'])} times, not once"
        alpha = _same(ranks, f"{i}/alpha")
        H = np.hstack([res[f"{i}/H"] for res in ranks])
        assert oracle.qr_residual(A0, np.asfortranarray(H), alpha) < 1e-13, f"partition {b}"
        assert np.abs(H[:, :256] - Href[:, :256]).max() < 1e-10, f"partition {b}"


def test_errors_are_rank_uniform(spawn, oracle):
    # a refusal reaches every rank with the same code, and the ranks stay aligned: a valid call after it succeeds.  The
    # single-GPU entry points refuse a 2-rank handle with -1 before they enqueue anything.
    ranks = spawn("errors", 2, "errors")
    for r, res in enumerate(ranks):
        assert int(res["rows/code"]) == -2, f"rank {r}: m = 728 min(SMs, 160) + 1 gave {int(res['rows/code'])}"
        assert int(res["overlap/code"]) == -4, f"rank {r}: an overlapping partition gave {int(res['overlap/code'])}"
        for k in res:
            if k.startswith("single/"):
                code, launches = res[k].tolist()
                assert code == -1 and launches == 0, f"rank {r}: {k[7:]} returned {code} after {launches} launches"
    A0 = F.make("normal", 512, 256)
    for tag in ("rows", "overlap"):
        alpha = _same(ranks, tag + "/alpha")
        H = np.hstack([res[tag + "/H"] for res in ranks])
        assert oracle.qr_residual(A0, np.asfortranarray(H), alpha) < 1e-13, f"the valid call after the {tag} refusal"
    assert _same(ranks, "rows/alpha").tobytes() == _same(ranks, "overlap/alpha").tobytes()
