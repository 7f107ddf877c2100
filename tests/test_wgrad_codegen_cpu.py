"""CPU: what the compiler made of the grouped weight-gradient kernel, read from the built library without a GPU.  Its speed rests on
staging the operands with 16-byte copies: 4-byte copies kept the issue slots of every warp busy for most of a chunk."""
import os
import re
import shutil
import subprocess

import pytest

from dwbc_b200 import _lib as L


def _sass(key):
    if not os.path.exists(L.LIB_PATH):
        L.build()
    out = subprocess.run(["cuobjdump", "-res-usage", L.LIB_PATH], capture_output=True, text=True).stdout
    names = sorted({n for n in re.findall(r"Function (\S+):", out) if key in n})
    return {n: subprocess.run(["cuobjdump", "-sass", "-fun", n, L.LIB_PATH], capture_output=True, text=True).stdout for n in names}


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="needs cuobjdump")
def test_wgrad_kernel_stages_operands_with_16_byte_copies():
    sass = _sass("wgrad_group_kernel")
    assert len(sass) == 2, list(sass)
    for name, s in sass.items():
        copies = re.findall(r"\bLDGSTS(\.[A-Z0-9]+)*", s)
        assert copies, name
        narrow = [ln for ln in s.splitlines() if "LDGSTS" in ln and ".128" not in ln]
        assert not narrow, (name, narrow[:3])
        # not a pipelining check: the wgmmas of a chunk are awaited together, once per chunk, not one by one (what ptxas does when it
        # serialises them).  The previous kernel passes this too.
        hgmma, waits = len(re.findall(r"\bHGMMA\.", s)), len(re.findall(r"WARPGROUP\.DEPBAR", s))
        assert hgmma >= 3 * 4, (name, hgmma)                # three widths x four K steps of a 32-row chunk
        assert 0 < waits <= hgmma // 4, (name, waits, hgmma)
