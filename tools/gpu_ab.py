"""A/B timing of two builds of libdhqr.so on the bench workload, interleaved in subprocesses on the same box.
usage: python tools/gpu_ab.py build/libdhqr_prev.so distributedhouseholderqr.jl_b200/libdhqr.so ... [rounds]
(a library argument may carry options: path:key=value,key=value; the pseudo-option lda=L stores A with leading dimension L)"""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.environ.get("DHQR_AB_LIB"):
    sys.path.insert(0, ROOT)
    import torch
    import dhqr_b200 as D
    D._lib.LIB_PATH = os.path.abspath(os.environ["DHQR_AB_LIB"])
    dev = torch.device("cuda:0"); h = D.default_handle(0)
    m, n = 32768, 4096
    lda = m
    for kv in os.environ.get("DHQR_AB_OPTS", "").split(","):
        if not kv: continue
        k, v = kv.split("=")
        if k == "lda": lda = int(v)
        else: h.set_option(k, int(v))
    A = D.colmajor_empty(m, n, dev, lda=lda); al = torch.zeros(n, dtype=torch.float64, device=dev)
    ts = []
    for _ in range(7):
        D.fill_uniform_(A, 0); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); D.householder_(A, al, 0); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    print(f"{min(ts[2:]):.2f} {sorted(ts[2:])[len(ts[2:]) // 2]:.2f}")
else:
    libs = [a for a in sys.argv[1:] if not a.isdigit()]; rounds = int(sys.argv[-1]) if sys.argv[-1].isdigit() else 2
    for r in range(rounds):
        for lib in libs:
            path, _, opts = lib.partition(":")
            out = subprocess.run([sys.executable, __file__], env={**os.environ, "DHQR_AB_LIB": path, "DHQR_AB_OPTS": opts}, capture_output=True, text=True)
            print(f"round {r} {lib}: min/median ms = {out.stdout.strip()} {out.stderr.strip()[-200:]}", flush=True)
