"""How long the panel chain's launches wait for SMs under the look-ahead schedule (option chain_wait_trace), on the bench
workload (qr! 32768 x 4096).  For every launch on hp, hp2 and aux: the span of the CUDA events right before and after it,
and the span from its first CTA's start to its last warp's end (%globaltimer); wait = event span - stamp span.  Prints the
wait summed per kernel class and per unit, and the look-ahead timeline (la_trace) of the same factorisation.
usage: python tools/chain_wait.py [key=value ...]   (handle options of the traced runs, e.g. cvy_persist=1)"""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C
from collections import defaultdict
import numpy as np, torch
import dhqr_b200 as D

STREAMS = ("hp", "hp2", "aux")
dev = torch.device("cuda:0"); h = D.default_handle(0)
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
print("card:", q.stdout.strip() or torch.cuda.get_device_name(0))
opts = dict(kv.split("=") for kv in sys.argv[1:])
for k, v in opts.items(): h.set_option(k, int(v))
m, n = 32768, 4096
A = D.colmajor_empty(m, n, dev); al = torch.zeros(n, dtype=torch.float64, device=dev)
for rep in range(3):                      # two untraced warm-up factorisations, then the traced one
    D.fill_uniform_(A, 0); torch.cuda.synchronize()
    h.set_option("chain_wait_trace", 1 if rep == 2 else 0); h.set_option("la_trace", 1 if rep == 2 else 0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); D.householder_(A, al, 0); e1.record(); torch.cuda.synchronize()
h.set_option("chain_wait_trace", 0); h.set_option("la_trace", 0)
print(f"options {opts or 'default'}: traced qr! {e0.elapsed_time(e1):.2f} ms")

buf = torch.zeros(1 + 6 * 8192, dtype=torch.float64, device=dev)
D._lib.call("dhqr_debug_copy_f64", h.raw, b"chain_wait", C.c_void_p(buf.data_ptr()), buf.numel(), None)
b = buf.cpu().numpy(); rows = b[1:1 + 6 * int(b[0])].reshape(-1, 6)
name = {}
for cls in sorted(set(rows[:, 2].astype(int))):
    s = C.create_string_buffer(64)
    D._lib.call("dhqr_profile_get", h.raw, int(cls), s, 64, None, None, None)
    name[cls] = s.value.decode()
stamped = rows[:, 4] >= 0
print(f"{len(rows)} chain launches, {int((~stamped).sum())} without stamps (left out below)")
r = rows[stamped]

print("\nper kernel class (ms summed over the factorisation):")
print(f"  {'class':16s} {'stream':6s} {'launches':>8s} {'event span':>10s} {'on SMs':>8s} {'wait':>8s} {'max wait':>8s}")
by = defaultdict(list)
for x in r: by[(name[int(x[2])], int(x[1]))].append(x)
for (cn, s), xs in sorted(by.items(), key=lambda kv: -sum(x[5] for x in kv[1])):
    xs = np.array(xs)
    print(f"  {cn:16s} {STREAMS[s]:6s} {len(xs):8d} {xs[:, 3].sum():10.3f} {xs[:, 4].sum():8.3f} {xs[:, 5].sum():8.3f} {xs[:, 5].max():8.3f}")
for s in range(3):
    xs = r[r[:, 1] == s]
    print(f"  total on {STREAMS[s]:4s}: {len(xs)} launches, event span {xs[:, 3].sum():.3f}, on SMs {xs[:, 4].sum():.3f}, wait {xs[:, 5].sum():.3f} ms")

la = torch.zeros(3 * 32, dtype=torch.float64, device=dev)
D._lib.call("dhqr_debug_copy_f64", h.raw, b"la_times", C.c_void_p(la.data_ptr()), 96, None)
t = la.cpu().numpy().reshape(32, 3)[::2]   # one row per unit (both panels of a pair carry the pair's times)
print("\nper unit: chain step and bulk step (la_trace), and the chain's wait for SMs (ms)")
print("  unit | chain step | bulk step | wait hp | wait hp2 | wait aux")
for u in range(len(t)):
    dp = t[u, 0] - (t[u - 1, 0] if u else 0.0); db = t[u, 2] - (t[u - 1, 2] if u else 0.0)
    w = [r[(r[:, 0] == u) & (r[:, 1] == s), 5].sum() for s in range(3)]
    print(f"  {u:4d} | {dp:10.2f} | {db:9.2f} | {w[0]:7.3f} | {w[1]:8.3f} | {w[2]:8.3f}")
