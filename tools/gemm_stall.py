"""Where the MMA warps of the two bulk GEMMs (k_gemm_vta, k_gemm_cvy_p) spend their cycles, on the bench workload.

    python tools/gemm_stall.py [lib ...] [--json OUT]

For each build of libdhqr.so (default: the one in the tree), in a subprocess of its own: two untraced factorisations of
qr! 32768 x 4096, then one with option gemm_trace on; the buckets of every traced CTA (include/dhqr.h) are summed per kernel
kind and printed as shares of the MMA warps' lifetime.  Then the K = 128 block-reflector update alone
(dhqr_k_block_reflector_f64) at the bulk shapes of steps 0, 14 and 26 of the sweep, traced the same way, and the serial
per-class profile of one factorisation (option "profile") with the TFLOP/s of k_gemm_cvy256, k_gemm_cvy128 and k_gemm_vta128.
The K = 256 update (k_gemm_cvy256) runs only inside qr!, so its buckets come from the factorisation.  The GPU's name, power
limit and maximum SM clock are read in the same run.
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M, N, NBP = 32768, 4096, 128
SHAPES = [(32768, 3712), (30976, 1920), (29440, 384)]
BUCKETS = ["start", "wait_full", "kloop", "wait_cfull", "epilogue", "drain"]   # words 1..6 of a row; word 7 = lifetime


def kind_name(code):
    kind, param = code >> 16, code & 0xFFFF
    return f"k_gemm_vta<{param}>" if kind == 1 else f"k_gemm_cvy_p K={param}" if kind == 2 else f"kind {code}"


def read_rows(h, D, torch, dev):
    import ctypes as C
    torch.cuda.synchronize()
    big = torch.zeros(2 + 8 * (1 << 17), dtype=torch.float64, device=dev)
    D._lib.call("dhqr_debug_copy_f64", h.raw, b"gemm_trace", C.c_void_p(big.data_ptr()), big.numel(), None)
    torch.cuda.synchronize()
    b = big.cpu().numpy()
    nrows, dropped = int(b[0]), int(b[1])
    return b[2:2 + 8 * nrows].reshape(-1, 8), dropped


def summarise(rows):
    out = {}
    for code in sorted(set(rows[:, 0].astype(int))):
        r = rows[rows[:, 0].astype(int) == code]
        life = r[:, 7].sum()
        d = {"ctas": int(len(r)), "mcycles_per_cta": float(life / len(r) / 8 / 1e6)}
        for i, bname in enumerate(BUCKETS):
            d[bname] = float(r[:, 1 + i].sum() / life) if life > 0 else 0.0
        d["other"] = 1.0 - sum(d[bn] for bn in BUCKETS)
        out[kind_name(code)] = d
    return out


def child():
    sys.path.insert(0, ROOT)
    import ctypes as C
    import torch
    import dhqr_b200 as D
    D._lib.LIB_PATH = os.path.abspath(os.environ["DHQR_GS_LIB"])
    dev = torch.device("cuda:0")
    h = D.Handle(0)
    res = {}
    A = D.colmajor_empty(M, N, dev)
    al = torch.zeros(N, dtype=torch.float64, device=dev)
    for rep in range(3):
        D.fill_uniform_(A, 0)
        torch.cuda.synchronize()
        if rep == 2:
            h.set_option("gemm_trace", 1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        D.householder_(A, al, 0, handle=h)
        e1.record()
        torch.cuda.synchronize()
    h.set_option("gemm_trace", 0)
    rows, dropped = read_rows(h, D, torch, dev)
    res["qr"] = {"traced_ms": e0.elapsed_time(e1), "dropped_launches": dropped, "kinds": summarise(rows)}

    h.set_option("profile", 1)
    D.fill_uniform_(A, 0)
    torch.cuda.synchronize()
    h.profile_reset()
    D.householder_(A, al, 0, handle=h)
    torch.cuda.synchronize()
    p = h.profile()
    h.set_option("profile", 0)
    res["profile"] = {k: {"ms": v["ms"], "count": v["count"], "tflops": v["work"] / v["ms"] / 1e9 if v["ms"] > 0 else 0.0}
                      for k, v in p.items() if k in ("k_gemm_cvy256", "k_gemm_cvy128", "k_gemm_vta128")}
    res["profile_sum_ms"] = sum(v["ms"] for v in p.values())
    del A

    res["alone"] = {}
    for rows_, ncols in SHAPES:
        a, tau = torch.geqrf(torch.rand(rows_, NBP, dtype=torch.float64, generator=torch.Generator().manual_seed(rows_)))
        V = (torch.tril(a, -1) + torch.eye(rows_, NBP, dtype=torch.float64)) * tau.sqrt()
        dV = D.to_colmajor(V, dev)
        Cm = D.colmajor_empty(rows_, ncols, dev)
        Cm.copy_(torch.rand(rows_, ncols, dtype=torch.float64, device=dev))
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

        def call():
            D._lib.call("dhqr_k_block_reflector_f64", h.raw, rows_, NBP, C.c_void_p(dV.data_ptr()), rows_, 0, ncols,
                        C.c_void_p(Cm.data_ptr()), rows_, None, st)

        for _ in range(2):
            call()
        torch.cuda.synchronize()
        h.set_option("gemm_trace", 1)
        call()
        torch.cuda.synchronize()
        h.set_option("gemm_trace", 0)
        r, _ = read_rows(h, D, torch, dev)
        res["alone"][f"{rows_}x{ncols}"] = summarise(r)
        del dV, Cm
        torch.cuda.empty_cache()
    h.close()
    print(json.dumps(res))


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable ({e})"


def show_kinds(kinds, indent="  "):
    print(f"{indent}{'kind':22s} {'CTAs':>6s} {'Mcyc/warp':>9s} " + " ".join(f"{b:>10s}" for b in BUCKETS + ["other"]))
    for k, d in kinds.items():
        print(f"{indent}{k:22s} {d['ctas']:6d} {d['mcycles_per_cta']:9.3f} " +
              " ".join(f"{100 * d[b]:9.1f}%" for b in BUCKETS + ["other"]))


def main():
    args = sys.argv[1:]
    jpath = None
    if "--json" in args:
        i = args.index("--json")
        jpath = args[i + 1]
        del args[i:i + 2]
    libs = args or [os.path.join(ROOT, "distributedhouseholderqr.jl_b200", "libdhqr.so")]
    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    out = {"gpu": info, "builds": {}}
    for lib in libs:
        p = subprocess.run([sys.executable, __file__], env={**os.environ, "DHQR_GS_LIB": lib}, capture_output=True, text=True)
        if p.returncode != 0:
            sys.exit(f"{lib}: child failed\n{p.stderr[-2000:]}")
        res = json.loads(p.stdout.strip().splitlines()[-1])
        out["builds"][lib] = res
        q = res["qr"]
        print(f"\n{lib}\n qr! {M} x {N}, traced: {q['traced_ms']:.2f} ms, launches left untraced: {q['dropped_launches']}")
        print(" share of the MMA warps' cycles per kind:")
        show_kinds(q["kinds"])
        print(" serial per-class profile:", "  ".join(f"{k} {v['ms']:.2f} ms ({v['count']}, {v['tflops']:.1f} TFLOP/s)"
                                                  for k, v in res["profile"].items()), f"  sum of classes {res['profile_sum_ms']:.2f} ms")
        for shape, kinds in res["alone"].items():
            print(f" K = 128 update alone at {shape}:")
            show_kinds(kinds, "   ")
    if jpath:
        os.makedirs(os.path.dirname(os.path.abspath(jpath)), exist_ok=True)
        with open(jpath, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    if os.environ.get("DHQR_GS_LIB"):
        child()
    else:
        main()
