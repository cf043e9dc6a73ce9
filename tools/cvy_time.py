"""Time the 128-wide block-reflector update alone at three bulk shapes of the bench sweep, for two (or more) builds of
libdhqr.so alternated in subprocesses.

    python tools/cvy_time.py <lib A> <lib B> [rounds] [--json OUT]

Shapes (rows x trailing columns, nbp = 128), the bulk updates of steps 0, 14 and 26 of qr! on 32768 x 4096:
32768 x 3712, 30976 x 1920, 29440 x 384.  Each child process runs dhqr_k_block_reflector_f64 with the option "profile" on
(2 warm-up calls, then 7 timed ones) and reports per shape:
  k_gemm_cvy128   C += V Y      ms per call, TFLOP/s (2 rows 128 ncols) and C GB/s (16 rows ncols: C read and written once)
  k_gemm_vta128   W = V'[V | C] ms per call, TFLOP/s (2 rows 128 (ncols + 128))
  cublas          torch addmm_ of the same C += V Y, CUDA-event median of 7
The parent prints every round, the median per build and shape, and the GPU's name, power limit and maximum SM clock read in
the same run.
"""
import json
import os
import subprocess
import sys

SHAPES = [(32768, 3712), (30976, 1920), (29440, 384)]
NBP = 128
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def child():
    sys.path.insert(0, ROOT)
    import torch
    import ctypes as C
    import dhqr_b200 as D
    D._lib.LIB_PATH = os.path.abspath(os.environ["DHQR_CVY_LIB"])
    dev = torch.device("cuda:0")
    h = D.Handle(0)
    h.set_option("profile", 1)
    out = {}
    for rows, ncols in SHAPES:
        a, tau = torch.geqrf(torch.rand(rows, NBP, dtype=torch.float64, generator=torch.Generator().manual_seed(rows)))
        V = (torch.tril(a, -1) + torch.eye(rows, NBP, dtype=torch.float64)) * tau.sqrt()
        dV = D.to_colmajor(V, dev)
        Cm = D.colmajor_empty(rows, ncols, dev)
        Cm.copy_(torch.rand(rows, ncols, dtype=torch.float64, device=dev))
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

        def call():
            D._lib.call("dhqr_k_block_reflector_f64", h.raw, rows, NBP, C.c_void_p(dV.data_ptr()), rows, 0, ncols,
                        C.c_void_p(Cm.data_ptr()), rows, None, st)

        for _ in range(2):
            call()
        torch.cuda.synchronize()
        h.profile_reset()
        reps = 7
        for _ in range(reps):
            call()
        torch.cuda.synchronize()
        prof = h.profile()
        res = {}
        cvy = prof["k_gemm_cvy128"]["ms"] / prof["k_gemm_cvy128"]["count"]
        vta = prof["k_gemm_vta128"]["ms"] / prof["k_gemm_vta128"]["count"]
        res["cvy_ms"], res["vta_ms"] = cvy, vta
        res["cvy_tflops"] = 2.0 * rows * NBP * ncols / cvy / 1e9
        res["cvy_c_gbs"] = 16.0 * rows * ncols / cvy / 1e6
        res["vta_tflops"] = 2.0 * rows * NBP * (ncols + NBP) / vta / 1e9
        Vt = dV.contiguous()
        Y = torch.rand(NBP, ncols, dtype=torch.float64, device=dev)
        Cc = torch.rand(rows, ncols, dtype=torch.float64, device=dev)
        ts = []
        for i in range(9):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            Cc.addmm_(Vt, Y)
            e1.record()
            e1.synchronize()
            if i >= 2:
                ts.append(e0.elapsed_time(e1))
        cub = sorted(ts)[len(ts) // 2]
        res["cublas_ms"], res["cublas_tflops"] = cub, 2.0 * rows * NBP * ncols / cub / 1e9
        out[f"{rows}x{ncols}"] = res
        del dV, Cm, Vt, Y, Cc
        torch.cuda.empty_cache()
    torch.cuda.synchronize()
    h.close()
    print(json.dumps(out))


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable ({e})"


def main():
    args = sys.argv[1:]
    jpath = None
    if "--json" in args:
        i = args.index("--json")
        jpath = args[i + 1]
        del args[i:i + 2]
    rounds = int(args.pop()) if args and args[-1].isdigit() else 3
    libs = args
    if not libs:
        sys.exit(__doc__)
    print(f"GPU: {gpu_info()}", flush=True)
    runs = {lib: [] for lib in libs}
    for r in range(rounds):
        for lib in libs:
            p = subprocess.run([sys.executable, __file__], env={**os.environ, "DHQR_CVY_LIB": lib}, capture_output=True, text=True)
            if p.returncode != 0:
                sys.exit(f"{lib}: child failed\n{p.stderr[-2000:]}")
            res = json.loads(p.stdout.strip().splitlines()[-1])
            runs[lib].append(res)
            print(f"round {r} {lib}: " + "  ".join(f"{k} cvy {v['cvy_ms']:.3f} ms vta {v['vta_ms']:.3f} ms" for k, v in res.items()),
                  flush=True)
    summary = {}
    for lib in libs:
        summary[lib] = {}
        print(f"\n{lib}: medians over {rounds} rounds")
        for rows, ncols in SHAPES:
            key = f"{rows}x{ncols}"
            med = {f: sorted(x[key][f] for x in runs[lib])[rounds // 2] for f in runs[lib][0][key]}
            summary[lib][key] = med
            print(f"  {key:12s} k_gemm_cvy128 {med['cvy_ms']:7.3f} ms {med['cvy_tflops']:5.1f} TFLOP/s {med['cvy_c_gbs']:6.0f} GB/s"
                  f" | k_gemm_vta128 {med['vta_ms']:7.3f} ms {med['vta_tflops']:5.1f} TFLOP/s"
                  f" | cuBLAS addmm {med['cublas_ms']:7.3f} ms {med['cublas_tflops']:5.1f} TFLOP/s")
    if jpath:
        os.makedirs(os.path.dirname(os.path.abspath(jpath)), exist_ok=True)
        with open(jpath, "w") as fh:
            json.dump({"gpu": gpu_info(), "rounds": runs, "medians": summary}, fh, indent=1)


if __name__ == "__main__":
    if os.environ.get("DHQR_CVY_LIB"):
        child()
    else:
        main()
