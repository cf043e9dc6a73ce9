"""Time deleting rows from a factorisation (dhqr_qr_downdate_f64, DESIGN §2.11) against the append at the same shape and against
factoring the remaining rows again, and one slide of a sliding-window least-squares solve.

    python tools/downdate_time.py [--rounds 3] [--json OUT] [--skip-window]

Downdates: n in {1024, 4096}, k in {64, 512, 4096, 32768}; R the triangle of a (32768 + k) x n factorisation, Z its last k rows, so
32768 rows remain.  Beside each, in the same run and interleaved round by round: the append of k rows at the same (n, k), and
dhqr_qr_f64 and torch.linalg.qr(mode="r") on the remaining 32768 x n rows.  Reported: CUDA-event medians of `rounds` calls (inputs
refilled outside the timed region), TFLOP/s of the downdate's 2 k n^2 flops, launches per call.  Window: a 1048576 x 1024 window in
StreamingLeastSquares; one slide = add one 65536-row block from pinned host memory, remove the oldest block (device-resident),
solve; wall time of the slide beside torch.linalg.lstsq on the device-resident window.  The GPU's name, power limit and max SM clock
are read in the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dhqr_b200 as D  # noqa: E402
from append_time import gpu_info  # noqa: E402


def event_ms(fn, prep):
    prep()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def downdate_case(h, m, n, k, rounds):
    S0 = D.colmajor_empty(m + k, n, "cuda")
    D.fill_uniform_(S0, 1, handle=h)
    A = S0.clone()
    st = D.qr_(A, handle=h)
    R0, a0 = A[:n].clone(), st.α.clone()
    Rd, al = D.colmajor_empty(n, n, "cuda"), torch.empty_like(a0)
    Z = D.colmajor_empty(k, n, "cuda")
    rem = D.colmajor_empty(m, n, "cuda")
    rem_row = S0[:m].contiguous()

    def prep_dd():
        Rd.copy_(R0)
        al.copy_(a0)
        Z.copy_(S0[m:])

    l0 = h.launch_count()
    prep_dd()
    t = D.downdate_rows_((Rd, al), Z, handle=h)
    launches = h.launch_count() - l0
    assert int(t.info.item()) == 0
    cases = {"downdate": (lambda: D.downdate_rows_((Rd, al), Z, handle=h), prep_dd),
             "append": (lambda: D.append_rows_((Rd, al), Z, handle=h), prep_dd),
             "qr_remaining": (lambda: D.qr_(rem, handle=h), lambda: rem.copy_(S0[:m])),
             "torch_qr_remaining": (lambda: torch.linalg.qr(rem_row, mode="r"), lambda: None)}
    ts = {key: [] for key in cases}
    for _ in range(rounds):                        # interleaved: every method once per round
        for key, (fn, prep) in cases.items():
            ts[key].append(event_ms(fn, prep))
    out = {"n": n, "k": k, "launches": launches}
    out.update({key + "_ms": float(np.median(v)) for key, v in ts.items()})
    out["downdate_tflops"] = 2.0 * k * n * n / (out["downdate_ms"] * 1e-3) / 1e12
    del S0, A, Z, rem, rem_row
    torch.cuda.empty_cache()
    return out


def window_case(h, m, n, blk, rounds):
    nblk = m // blk
    ls = D.StreamingLeastSquares(n, 1, device=0, handle=h)
    W = D.colmajor_empty(m, n, "cuda")                     # the window, for torch.linalg.lstsq
    bw = torch.empty(m, 1, dtype=torch.float64, device="cuda")

    def block(i):
        a = D.colmajor_empty(blk, n, "cuda")
        D.fill_uniform_(a, 100 + i, handle=h)
        b = torch.rand(blk, 1, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(i))
        return a, b

    for i in range(nblk):
        a, b = block(i)
        ls.add(a, b)
    Ah = torch.empty((blk, n), dtype=torch.float64).pin_memory()
    bh = torch.empty((blk, 1), dtype=torch.float64).pin_memory()
    slide_ms = []
    for r in range(rounds):
        a_new, b_new = block(nblk + r)
        Ah.copy_(a_new.cpu())
        bh.copy_(b_new.cpu())
        a_old, b_old = block(r)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ls.add(Ah, bh)                                    # from pinned host memory
        ls.remove(a_old, b_old)
        x = ls.solve()
        torch.cuda.synchronize()
        slide_ms.append((time.perf_counter() - t0) * 1e3)
    for i in range(nblk):                                 # the final window, on the device
        a, b = block(rounds + i)
        W[i * blk:(i + 1) * blk].copy_(a)
        bw[i * blk:(i + 1) * blk].copy_(b)
    lstsq_ms = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        xl = torch.linalg.lstsq(W, bw).solution
        torch.cuda.synchronize()
        lstsq_ms.append((time.perf_counter() - t0) * 1e3)
    dx = float((x - xl[:, 0]).norm() / xl.norm())
    return {"m": m, "n": n, "block": blk, "slide_ms": float(np.median(slide_ms)), "torch_lstsq_ms": float(np.median(lstsq_ms)),
            "rel_diff_x": dx, "rows": ls.rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    ap.add_argument("--skip-window", action="store_true")
    args = ap.parse_args()
    h = D.Handle(0)
    res = {"gpu": gpu_info(), "downdate": []}
    print(json.dumps(res["gpu"]), flush=True)
    for n in (1024, 4096):
        for k in (64, 512, 4096, 32768):
            r = downdate_case(h, 32768, n, k, args.rounds)
            res["downdate"].append(r)
            print(f"n={n:5d} k={k:6d}: downdate {r['downdate_ms']:8.2f} ms ({r['downdate_tflops']:5.2f} TFLOP/s, {r['launches']} launches)"
                  f"  append {r['append_ms']:8.2f} ms  qr_ remaining {r['qr_remaining_ms']:8.2f} ms"
                  f"  torch.linalg.qr remaining {r['torch_qr_remaining_ms']:8.2f} ms", flush=True)
    if not args.skip_window:
        r = window_case(h, 1 << 20, 1024, 65536, args.rounds)
        res["window"] = r
        print(f"window {r['m']} x {r['n']}, one slide of {r['block']} rows (add from pinned host memory, remove, solve): "
              f"{r['slide_ms']:.1f} ms; torch.linalg.lstsq on the device-resident window {r['torch_lstsq_ms']:.1f} ms; "
              f"|dx|/|x| {r['rel_diff_x']:.2e}", flush=True)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(res, fh, indent=1)
    h.close()


if __name__ == "__main__":
    main()
