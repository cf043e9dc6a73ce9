"""One-shot status of the bench workload: serial per-class profile, look-ahead timeline summary, a few option A/Bs."""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
import numpy as np, torch
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
def show(tag):
    t = timeit(); print(f"{tag}: {t:.2f} ms  {fl / t / 1e9:.2f} TFLOP/s", flush=True)
show("default")
print("panels fast/fallback:", h.get_option("panels_fast"), h.get_option("panels_fallback"))
h.set_option("profile", 1); D.fill_uniform_(A, 0); torch.cuda.synchronize(); h.profile_reset()
D.householder_(A, al, 0); torch.cuda.synchronize(); p = h.profile(); h.set_option("profile", 0)
print("serial profile:", json.dumps({k: (round(v["ms"], 2), v["count"], round(v["work"] / v["ms"] / 1e9, 1) if k.startswith("k_gemm") and v["ms"] > 0 else None) for k, v in p.items()}), flush=True)
for rep in range(2):
    D.fill_uniform_(A, 0); torch.cuda.synchronize(); h.set_option("la_trace", rep)
    D.householder_(A, al, 0); torch.cuda.synchronize()
buf = torch.zeros(96, dtype=torch.float64, device=dev)
D._lib.call("dhqr_debug_copy_f64", h.raw, b"la_times", C.c_void_p(buf.data_ptr()), 96, None)
t = buf.cpu().numpy().reshape(32, 3); h.set_option("la_trace", 0)
dp = np.diff(np.concatenate([[0], t[:, 0]])); db = np.diff(np.concatenate([[0], t[:, 2]]))
print("timeline: total %.2f ms; panel steps (ms):" % t[-1].max(), np.round(dp, 2).tolist(), flush=True)
print("          bulk steps (ms):", np.round(db, 2).tolist(), flush=True)
for opts in ({"panel_ctas": 132}, {"panel_ctas": 96}, {"panel_fast": 0}):
    for k, v in opts.items(): h.set_option(k, v)
    show(str(opts))
    h.set_option("panel_ctas", 0); h.set_option("panel_fast", 1)
h.set_option("lookahead", 0); show("serial"); h.set_option("lookahead", 1)
