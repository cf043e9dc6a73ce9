"""Option sweep on the bench workload: min / median ms of qr! for each setting (one handle, options restored)."""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import dhqr_b200 as D
dev = torch.device("cuda:0"); h = D.default_handle(0)
m, n = 32768, 4096
A = D.colmajor_empty(m, n, dev); al = torch.zeros(n, dtype=torch.float64, device=dev)
fl = 2.0 * m * n * n - 2.0 / 3.0 * n ** 3
def timeit(reps=5):
    ts = []
    for _ in range(reps + 1):
        D.fill_uniform_(A, 0); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); D.householder_(A, al, 0); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return min(ts[1:]), float(np.median(ts[1:]))
base = {"cvy_persist": 4, "lookahead": 1, "wide_panel": 1}
def run(tag, **opts):
    for k, v in {**base, **opts}.items(): h.set_option(k, v)
    t, md = timeit()
    print(f"{tag:40s} min {t:.2f} ms  median {md:.2f} ms  {fl / t / 1e9:.2f} TFLOP/s", flush=True)
    for k, v in base.items(): h.set_option(k, v)
for tpc in (1, 2, 3, 4, 6, 8, 16, 1000000):
    run(f"cvy_persist={tpc}", cvy_persist=tpc)
for tpc in (0, 2, 4, 1000000):
    run(f"serial schedule, cvy_persist={tpc}", cvy_persist=tpc, lookahead=0)
