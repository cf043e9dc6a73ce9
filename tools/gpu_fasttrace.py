"""clock64 stamps of the panel kernel's fast path (option panel_trace)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
import numpy as np, torch
import dhqr_b200 as D
dev = torch.device("cuda:0"); h = D.default_handle(0)
rows = 32768
vp = lambda t: C.c_void_p(t.data_ptr()); sp = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
P = D.colmajor_empty(rows, 32, dev); al = torch.zeros(32, dtype=torch.float64, device=dev)
names = ["", "gram1+exch", "chol1", "trsm1", "gram2+exch", "chol2", "trsm2", "Rt+topLU+exch", "rows+top write"]
for pc in (64, 132):
    h.set_option("panel_ctas", pc); h.set_option("panel_trace", 1)
    for rep in range(3):
        D.fill_uniform_(P, 1); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); D._lib.call("dhqr_k_panel_f64", h.raw, rows, 32, vp(P), rows, vp(al), sp()); e1.record(); torch.cuda.synchronize()
    tr = torch.empty(160 * 32 * 8, dtype=torch.float64, device=dev)
    D._lib.call("dhqr_debug_copy_f64", h.raw, b"panel_trace", vp(tr), 160 * 32 * 8, sp()); torch.cuda.synchronize()
    t = tr.cpu().numpy().view(np.int64).reshape(160, 256)
    print(f"panel_ctas={pc}: kernel {e0.elapsed_time(e1) * 1e3:.1f} us", flush=True)
    for cta in (0, 30):
        x = t[cta, :9].astype(np.float64); d = np.diff(x)
        print(f"  cta {cta}: " + " | ".join(f"{names[k+1]} {d[k]:.0f}" for k in range(8)) + f" | total {x[8]:.0f} cyc")
h.set_option("panel_trace", 0); h.set_option("panel_ctas", 0)
