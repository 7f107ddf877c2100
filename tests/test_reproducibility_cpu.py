"""CPU: the reductions that must repeat bit for bit are summed in a fixed order, read from the compiled library without a GPU.  A float
atomic (RED / ATOM with an .F32 / .F32x2 / .F64 opcode) or a shared-memory compare-and-swap loop (ATOMS.CAST.SPIN) adds in whatever
order the CTAs happen to arrive."""
import os
import re
import shutil
import subprocess

import pytest

from dwbc_b200 import _lib as L

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))

FLOAT_ATOMIC = re.compile(r"\b(?:RED|ATOM)\w*(?:\.\w+)*\.(?:F32|F32x2|F64)\b|\bATOMS\.CAST\.SPIN\b")


def _kernels_sass():
    out = subprocess.run(["cuobjdump", "-sass", L.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None:
            funcs[cur].append(line)
    return funcs


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="needs cuobjdump")
def test_no_kernel_has_float_atomics():
    if not os.path.exists(L.LIB_PATH):
        L.build()
    funcs = _kernels_sass()
    for key in ("wgrad_group_kernel", "gemm_tile_kernel", "chain2_kernel", "env_step_kernel", "env_step_v2_kernel", "gae_kernel"):
        assert any(key in n for n in funcs), key               # (the scan reads the kernels it is meant to)
    bad = {n: sorted({m.group(0) for ln in body for m in [FLOAT_ATOMIC.search(ln)] if m}) for n, body in funcs.items()}
    bad = {n: v for n, v in bad.items() if v}
    assert not bad, bad


def test_scratch_sizes_match_the_header():
    hdr = open(os.path.join(ROOT, "include", "dwbc.h")).read()
    defs = dict(re.findall(r"#define (DWBC_\w+) (.+)", hdr))

    def value(name):
        expr = re.sub(r"/\*.*", "", defs[name]).strip()
        return eval(re.sub(r"DWBC_\w+", lambda m: str(value(m.group(0))), expr))

    assert L.NORM_SCRATCH == value("DWBC_NORM_SCRATCH")
    assert L.GAE_STATS == value("DWBC_GAE_STATS")


@pytest.mark.parametrize("trunk,hist", [((128,), 10), ((512, 256, 128), 10), ((128,), 20), ((128,), 50)])
def test_workspace_holds_the_weight_gradient_plan_on_every_sm_count(trunk, hist):
    """The partial area of the grouped weight-gradient launch, on SM counts around the H100's, fits what dwbc_workspace_bytes reserved;
    and the reservation never shrinks as rows grow (one workspace serves smaller rows)."""
    import ctypes as C
    from dwbc_b200.actor_critic import FlatActorCritic
    lib = L.lib()
    lib.dwbc_debug_wgrad_partial_floats.argtypes = [C.c_void_p, C.c_int32, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    need, bound = C.c_int64(), C.c_int64()
    for precision in (1, 2):
        ac = FlatActorCritic(device="cpu", seed=0, num_priv=24, num_hist=hist, num_prop=76, actor_hidden_dims=trunk, critic_hidden_dims=trunk)
        ac.net_cfg.precision = precision
        last = 0
        for rows in (1, 127, 4096, 40960, 81920):
            ws = lib.dwbc_workspace_bytes(C.addressof(ac.net_cfg), rows)
            assert ws >= last
            last = ws
            for sms in (114, 132, 144):
                rc = lib.dwbc_debug_wgrad_partial_floats(C.addressof(ac.net_cfg), rows, sms, C.byref(need), C.byref(bound))
                if rc == -2:                          # (a network the fused chains do not take runs layer-wise: no grouped launch)
                    continue
                assert rc == 0 and 0 < need.value <= bound.value, (rows, sms, need.value, bound.value)
