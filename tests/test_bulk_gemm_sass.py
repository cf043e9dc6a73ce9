"""The two bulk trailing-update GEMMs (k_gemm_vta: W = V'[V|C], k_gemm_cvy_p: C += V Y) run their inner loops as DMMA.16x8x8.
On an H100 DMMA.8x8x4 holds the fp64 tensor pipe to half the rate of the 16x8xK shapes (DESIGN §7), so one 8x8x4 left in
these loops halves their throughput without changing a result.  Reads the SASS of the built libdhqr.so; no GPU needed."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "distributedhouseholderqr.jl_b200", "libdhqr.so")
KERNELS = {                                      # mangled-name prefix -> readable name
    "_ZN4dhqr10k_gemm_vtaILi128E": "k_gemm_vta<128, ...>",
    "_ZN4dhqr10k_gemm_vtaILi32E": "k_gemm_vta<32, ...>",
    "_ZN4dhqr12k_gemm_cvy_pE": "k_gemm_cvy_p",
}


def _cuobjdump():
    for c in (shutil.which("cuobjdump"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")):
        if c and os.access(c, os.X_OK):
            return c
    return None


@pytest.fixture(scope="module")
def dump():
    tool = _cuobjdump()
    if not os.path.exists(LIB) or tool is None:
        pytest.skip("needs the built libdhqr.so and cuobjdump")
    sass = subprocess.run([tool, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    res = subprocess.run([tool, "--dump-resource-usage", LIB], capture_output=True, text=True, check=True).stdout
    return sass, res


def _per_function(text, header):
    out, name = {}, None
    for line in text.splitlines():
        m = re.match(header, line.strip())
        if m:
            name = m.group(1)
            out[name] = []
        elif name:
            out[name].append(line)
    return {k: "\n".join(v) for k, v in out.items()}


@pytest.mark.parametrize("prefix", list(KERNELS))
def test_bulk_gemm_uses_16x8x8(dump, prefix):
    sass, res = dump
    funcs = {k: v for k, v in _per_function(sass, r"Function : (\S+)").items() if k.startswith(prefix)}
    assert len(funcs) == 1, f"expected one instantiation of {KERNELS[prefix]}, found {sorted(funcs)}"
    body = next(iter(funcs.values()))
    shapes = re.findall(r"DMMA\.(\d+x\d+x\d+)", body)
    assert shapes and set(shapes) == {"16x8x8"}, f"{KERNELS[prefix]}: DMMA shapes {sorted(set(shapes))}"
    usage = {k: v for k, v in _per_function(res, r"Function (\S+):").items() if k.startswith(prefix)}
    assert len(usage) == 1
    line = next(iter(usage.values()))
    assert re.search(r"\bSTACK:0\b", line) and re.search(r"\bLOCAL:0\b", line), f"{KERNELS[prefix]} spills: {line.strip()}"
