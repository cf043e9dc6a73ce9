"""panel_ctas sweep on the bench workload (look-ahead)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import dhqr_b200 as D
dev = torch.device("cuda:0"); h = D.default_handle(0)
m, n = 32768, 4096
A = D.colmajor_empty(m, n, dev); al = torch.zeros(n, dtype=torch.float64, device=dev)
fl = 2.0 * m * n * n - 2.0 / 3.0 * n ** 3
def timeit(reps=3):
    best = 1e30
    for _ in range(reps + 1):
        D.fill_uniform_(A, 0); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); D.householder_(A, al, 0); e1.record(); torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best
for pc in (0, 32, 48, 64, 96, 128, 132):
    h.set_option("panel_ctas", pc)
    t = timeit(); print(f"panel_ctas={pc}: {t:.2f} ms  {fl / t / 1e9:.2f} TFLOP/s", flush=True)
h.set_option("panel_ctas", 0)
