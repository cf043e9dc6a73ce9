"""Per-phase clock64() breakdown of k_panel (option panel_trace): python tools/gpu_paneltrace.py [rows]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
import numpy as np, torch
import dhqr_b200 as D
dev = torch.device("cuda:0"); h = D.default_handle(0)
rows = int(sys.argv[1]) if len(sys.argv) > 1 else 32768
vp = lambda t: C.c_void_p(t.data_ptr()); sp = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
P = D.colmajor_empty(rows, 32, dev); al = torch.zeros(32, dtype=torch.float64, device=dev)
for pc in (0, 64, 32):
    h.set_option("panel_ctas", pc); h.set_option("panel_trace", 1)
    for rep in range(3):
        D.fill_uniform_(P, 1)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        D._lib.call("dhqr_k_panel_f64", h.raw, rows, 32, vp(P), rows, vp(al), sp())
        e1.record(); torch.cuda.synchronize()
    tr = torch.empty(160 * 32 * 8, dtype=torch.float64, device=dev)
    D._lib.call("dhqr_debug_copy_f64", h.raw, b"panel_trace", vp(tr), 160 * 32 * 8, sp())
    torch.cuda.synchronize()
    t = tr.cpu().numpy().view(np.int64).reshape(160, 32, 8)
    print(f"panel_ctas={pc}: kernel {e0.elapsed_time(e1) * 1e3:.1f} us", flush=True)
    for cta in (0, 40):
        x = t[cta].astype(np.float64)
        names = ["enter", "w0 totals", "block sync", "scalars", "step1+sync", "produce"]
        d = np.diff(x[:, :6], axis=1)          # phase durations within an iteration
        gap = x[1:, 0] - x[:-1, 5]
        print(f"  cta {cta}: first enter {x[0,0]:.0f} cyc; last produce end {x[-1,5]:.0f} cyc; per-column mean {np.diff(x[:,0]).mean():.0f} cyc")
        print("     mean cycles: poll->totals %.0f | sync %.0f | scalars %.0f | step1+sync %.0f | produce %.0f | loop gap %.0f" % (*d[:-1].mean(0), gap.mean()))
        print("     col 5:", (x[5, :8] - x[5, 0]).astype(int).tolist(), " col 20:", (x[20, :8] - x[20, 0]).astype(int).tolist(), "  [.., 6]=pivot arrived [7]=total arrived (relative to iteration entry)")
h.set_option("panel_trace", 0); h.set_option("panel_ctas", 0)
