"""The tensor-pipe kernels of the 128-column panel chain (k_gram_sym, k_pack_gram: the partial Gram matrices; k_vpk_rmul: the
blocked triangular solve and, in its Gram mode, the second Gram matrix) issue only DMMA.16x8x8 and keep everything in
registers.  On an H100 DMMA.8x8x4 runs the fp64 tensor pipe at half the rate of the 16x8xK shapes (DESIGN §10 item 3c).
Reads the SASS of the built libdhqr.so; no GPU needed."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "distributedhouseholderqr.jl_b200", "libdhqr.so")
KERNELS = {                                      # mangled-name prefix -> readable name
    "_ZN4dhqr10k_gram_symE": "k_gram_sym",
    "_ZN4dhqr11k_pack_gramE": "k_pack_gram",
    "_ZN4dhqr10k_vpk_rmulE": "k_vpk_rmul",
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
def test_chain_kernel_uses_16x8x8_without_local_memory(dump, prefix):
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
