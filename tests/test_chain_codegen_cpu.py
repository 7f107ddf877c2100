"""CPU: what the compiler made of the fused layer-chain kernel, read without a GPU.  The kernel's speed rests on ptxas NOT fencing and
awaiting every wgmma on its own; it does that silently (an info line in a log nobody reads) whenever the control flow around the wgmmas
stops looking warp-uniform to it or the registers run out, and every result stays correct."""
import os
import re
import shutil
import subprocess

import pytest

from dwbc_b200 import _lib as L

CSRC = os.path.join(os.path.dirname(os.path.abspath(L.__file__)), "csrc")
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def _sass(lib_path, key):
    out = subprocess.run(["cuobjdump", "-res-usage", lib_path], capture_output=True, text=True).stdout
    names = [n for n in re.findall(r"Function (\S+):", out) if key in n]
    return {n: subprocess.run(["cuobjdump", "-sass", "-fun", n, lib_path], capture_output=True, text=True).stdout for n in names}


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="needs cuobjdump")
def test_chain_kernel_awaits_wgmma_per_op_not_per_instruction():
    if not os.path.exists(L.LIB_PATH):
        L.build()
    (sass,) = _sass(L.LIB_PATH, "chain2_kernel").values()
    hgmma, waits = len(re.findall(r"\bHGMMA\.", sass)), len(re.findall(r"WARPGROUP\.DEPBAR", sass))
    assert hgmma >= 3 * (1 + 3 * 16), hgmma          # three widths x (plain TF32 loop + 16 unrolled 3xTF32 K steps of three products)
    assert 0 < waits <= hgmma // 4, (waits, hgmma)     # 87 waits for 84 HGMMA when ptxas serialised the kernel
    # the workers raise their register allowance, the copy warpgroup gives its registers up
    assert len(re.findall(r"USETMAXREG", sass)) == 2


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="needs nvcc")
def test_ptxas_reports_no_serialised_wgmma(tmp_path):
    """C7520 (divergent control flow around wgmma) and C7511 (not enough registers for the wgmma pipeline) are the two reasons ptxas gives
    for serialising; neither may appear for any tensor-core kernel of mlp.cu."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cmd = [nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-I" + os.path.join(ROOT, "include"), "-I" + CSRC,
           "--expt-relaxed-constexpr", "-Xptxas", "-v", "-cubin", os.path.join(CSRC, "mlp.cu"), "-o", str(tmp_path / "mlp.cubin")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    log = r.stdout + r.stderr
    bad = [ln for ln in log.splitlines() if "serialized" in ln or "C7520" in ln or "C7511" in ln]
    assert not bad, bad[:3]
    assert "chain2_kernel" in log                        # the log is the verbose one
