"""Timeline of the look-ahead schedule (option la_trace): when each panel / next-signal / bulk update completes."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
import numpy as np, torch
import dhqr_b200 as D
dev = torch.device("cuda:0"); h = D.default_handle(0)
m, n = 32768, 4096
A = D.colmajor_empty(m, n, dev); al = torch.zeros(n, dtype=torch.float64, device=dev)
for tag, opts in (("default", {}), ("panel_ctas=96", {"panel_ctas": 96}), ("panel_ctas=132", {"panel_ctas": 132})):
    for k, v in opts.items(): h.set_option(k, v)
    for rep in range(2):
        D.fill_uniform_(A, 0); torch.cuda.synchronize()
        h.set_option("la_trace", 1 if rep else 0)
        D.householder_(A, al, 0); torch.cuda.synchronize()
    buf = torch.zeros(3 * 32, dtype=torch.float64, device=dev)
    D._lib.call("dhqr_debug_copy_f64", h.raw, b"la_times", C.c_void_p(buf.data_ptr()), 96, None)
    t = buf.cpu().numpy().reshape(32, 3)
    print(f"== {tag}: total {t[-1].max():.2f} ms")
    print("  k : panel_k done | next_k signalled | bulk_k done | panel step | bulk step")
    for k in range(32):
        dp = t[k, 0] - (t[k - 1, 0] if k else 0.0); db = t[k, 2] - (t[k - 1, 2] if k else 0.0)
        print(f"  {k:2d}: {t[k,0]:8.2f} {t[k,1]:8.2f} {t[k,2]:8.2f}   {dp:6.2f} {db:6.2f}")
    h.set_option("la_trace", 0); h.set_option("panel_ctas", 0)
