"""dhqr_qr_host_f64 at BASELINE config 3: catch-up streams x first upload, against the resident factorisation; timeline of the default."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
import torch
import dhqr_b200 as D
dev = torch.device("cuda:0"); h = D.default_handle(0)
m, n = 32768, 4096
host = torch.empty((n, m), dtype=torch.float64).pin_memory()
src = torch.empty((n, m), dtype=torch.float64, device=dev)
D.fill_uniform_(src.t(), 0)
al = torch.empty(n, dtype=torch.float64).pin_memory()
def run(reps=4):
    ts = []
    for _ in range(reps):
        host.copy_(src); torch.cuda.synchronize()
        t0 = time.perf_counter()
        D._lib.call("dhqr_qr_host_f64", h.raw, m, n, C.c_void_p(host.data_ptr()), m, C.c_void_p(al.data_ptr()), 0)
        ts.append((time.perf_counter() - t0) * 1e3)
    return ts
run(2)
for rnd in range(2):
    for cus in (3, 2):
        for first in (0, 768):
            h.set_option("host_cu_streams", cus); h.set_option("host_first", first)
            run(1)
            ts = run()
            print(f"cu_streams {cus} first {first:4d}: " + " ".join(f"{t:.2f}" for t in ts) + " ms", flush=True)
# device-resident factorisation (same process)
A = D.colmajor_empty(m, n, dev); alpha = torch.zeros(n, dtype=torch.float64, device=dev)
for rnd in range(2):
    ts = []
    for _ in range(6):
        D.fill_uniform_(A, 0); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); D.householder_(A, alpha, 0); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    print("resident qr!: " + " ".join(f"{t:.2f}" for t in ts[1:]) + " ms", flush=True)
h.set_option("host_cu_streams", 3); h.set_option("host_first", 0)
h.set_option("host_trace", 1)
run(1)
