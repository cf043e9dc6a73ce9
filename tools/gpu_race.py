"""Localise a sporadic race: repeat one block-reflector application on identical inputs and compare the
internal buffers (W partials -> gemm_vta, Linv -> tinv, Y -> ymake, C -> gemm_cvy) bitwise against run 0."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import ctypes as C
import numpy as np, torch
import dhqr_b200 as D
import dhqr_oracle as O
dev = torch.device("cuda:0"); h = D.default_handle(0)
vp = lambda t: C.c_void_p(t.data_ptr()); sp = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
def experiment(rows, nbp, ncols, iters):
    co = O.COracle()
    P = co.fill_uniform(3, rows, nbp); Hp, _ = co.qr(P)
    V = D.to_colmajor(np.tril(Hp), dev)
    C0 = D.colmajor_empty(rows, ncols, dev); D.fill_uniform_(C0, 5)
    nw = min(64 * 1024 * 1024 // 8, 3 * 132 * 128 * 128)
    ny = 4 * 64 * 36 * ((ncols + 63) // 64)
    ref = None; bad = 0
    for it in range(iters):
        Cw = C0.clone() if False else D.colmajor_empty(rows, ncols, dev); Cw.copy_(C0)
        D._lib.call("dhqr_k_block_reflector_f64", h.raw, rows, nbp, vp(V), rows, 0, ncols, vp(Cw), rows, None, sp())
        W = torch.empty(nw, dtype=torch.float64, device=dev); Y = torch.empty(ny, dtype=torch.float64, device=dev); L = torch.empty(128 * 128, dtype=torch.float64, device=dev)
        D._lib.call("dhqr_debug_copy_f64", h.raw, b"wpart", vp(W), nw, sp())
        D._lib.call("dhqr_debug_copy_f64", h.raw, b"ypk", vp(Y), ny, sp())
        D._lib.call("dhqr_debug_copy_f64", h.raw, b"linv", vp(L), 128 * 128, sp())
        torch.cuda.synchronize()
        if ref is None:
            ref = (W, L, Y, Cw); continue
        dW = (W != ref[0]) & ~(torch.isnan(W) & torch.isnan(ref[0])); dL = L != ref[1]; dY = (Y != ref[2]) & ~(torch.isnan(Y) & torch.isnan(ref[2])); dC = Cw != ref[3]
        if dW.any() or dL.any() or dY.any() or dC.any():
            bad += 1
            if bad <= 6:
                msg = f"  iter {it}: W diff {int(dW.sum())} L diff {int(dL.sum())} Y diff {int(dY.sum())} C diff {int(dC.sum())}"
                if dW.any():
                    idx = torch.nonzero(dW)[:, 0]
                    nbk = 32 if nbp <= 32 else 128
                    col = (idx // nbk); row = idx % nbk
                    msg += f"\n     W flat idx {int(idx.min())}..{int(idx.max())}; ext col(all splits flattened) {int(col.min())}..{int(col.max())}; V-row {int(row.min())}..{int(row.max())}; maxabs {float((W-ref[0])[dW].abs().max()):.3e}"
                    msg += f"\n     distinct ext cols: {torch.unique(col).tolist()[:80]}"
                if dC.any():
                    idx = torch.nonzero(dC)
                    msg += f"\n     C rows {int(idx[:,0].min())}..{int(idx[:,0].max())} cols {int(idx[:,1].min())}..{int(idx[:,1].max())}"
                print(msg, flush=True)
    print(f"rows={rows} nbp={nbp} ncols={ncols}: {bad} / {iters - 1} runs differ from run 0", flush=True)
experiment(29824, 128, 1024, int(sys.argv[1]) if len(sys.argv) > 1 else 300)
experiment(16384, 128, 512, 200)
experiment(29824, 32, 96, 300)
