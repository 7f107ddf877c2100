"""CPU: libdwbc.so loads without a GPU and exports every symbol include/dwbc.h declares; the ctypes
struct mirrors agree with the C layouts; host-side config logic."""
import ctypes
import os
import re

import pytest

import dwbc_b200
from dwbc_b200 import _lib as L, config as C

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        L.build()
    return L.lib()


def test_library_exports_every_declared_symbol(lib):
    hdr = open(os.path.join(ROOT, "include", "dwbc.h")).read()
    declared = sorted(set(re.findall(r"\b(dwbc_[a-z_0-9]+)\s*\(", hdr)))
    assert declared == L.EXPORTS, (declared, L.EXPORTS)
    for name in declared:
        assert hasattr(lib, name), name


def test_debug_header_symbols_are_exported(lib):
    """include/dwbc_debug.h (profiling and test hooks, outside the drop-in boundary): every declared symbol exists, and the library
    exports no dwbc_* symbol that neither header declares."""
    import subprocess
    dbg = open(os.path.join(ROOT, "include", "dwbc_debug.h")).read()
    declared = sorted(set(re.findall(r"\b(dwbc_debug_[a-z_0-9]+)\s*\(", dbg)))
    assert declared
    for name in declared:
        assert hasattr(lib, name), name
    out = subprocess.run(["nm", "-D", "--defined-only", L.LIB_PATH], capture_output=True, text=True).stdout
    exported = sorted(set(re.findall(r" T (dwbc_[a-z_0-9]+)$", out, re.M)))
    assert exported == sorted(L.EXPORTS + declared), set(exported) ^ set(L.EXPORTS + declared)


def test_kernel_resource_budgets(lib):
    """Occupancy contracts the kernels are designed around, read from the shipped cubins (`cuobjdump -res-usage`, no GPU): K1 must fit two
    CTAs per SM (<= 128 registers at 256 threads), the chain kernel's 288 threads must stay below the 224-register cap with a small stack (a
    change that made ptxas clone its whole item loop doubled the spills and the code size without any error), the grouped weight gradient
    runs 8 warps per CTA with a 64-register accumulator fragment per thread (<= 224 registers, no stack)."""
    import subprocess
    out = subprocess.run(["cuobjdump", "-res-usage", L.LIB_PATH], capture_output=True, text=True).stdout
    use = {}
    for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", out):
        use[m.group(1)] = tuple(int(x) for x in m.groups()[1:])
    find = lambda key: [v for k, v in use.items() if key in k]  # noqa: E731
    (k1,), (chain,), wg = find("env_step_v2_kernel"), find("chain2_kernel"), find("wgrad_group_kernel")
    assert k1[0] <= 128, k1
    assert chain[0] <= 224 and chain[1] <= 640, chain
    assert len(wg) == 2 and all(w[0] <= 224 and w[1] == 0 for w in wg), wg
    sass = subprocess.run(["cuobjdump", "-sass", "-fun", [k for k in use if "chain2_kernel" in k][0], L.LIB_PATH], capture_output=True, text=True).stdout
    n_instr = len(re.findall(r"^\s+/\*[0-9a-f]{4,5}\*/", sass, re.M))
    assert 8000 < n_instr < 22000, n_instr          # 15.4 k today; 29 k when the item loop was cloned


def test_struct_mirrors_match_c_layout(lib):
    sizes = (ctypes.c_int64 * 6)()
    lib.dwbc_struct_sizes(ctypes.byref(sizes))
    assert list(sizes) == [ctypes.sizeof(s) for s in (L.EnvCfg, L.EnvBuffers, L.StepArgs, L.NetCfg, L.PpoHyper, L.Storage)]
    assert b"sm_90a" in lib.dwbc_version()


def test_header_enums_match_python_tables():
    hdr = open(os.path.join(ROOT, "include", "dwbc.h")).read()
    terms = re.search(r"enum DwbcTerm \{(.*?)\};", hdr, re.S).group(1)
    names = [t.replace("DWBC_TERM_", "").split("=")[0].strip() for t in terms.replace("\n", " ").split(",")]
    names = [n for n in names if n and n != "COUNT"]
    assert names == C.REWARD_TERMS
    for k in ("GOAL_ORN", "GOAL_SPH", "CMD", "PUSH", "RST_DOF", "RST_XY", "RST_VEL", "RST_CMD", "RST_GOAL_ORN", "RST_GOAL_SPH", "TERRAIN"):
        v = int(re.search(rf"DWBC_RAND_{k} = (\d+)", hdr).group(1))
        assert v == getattr(C, "RAND_" + k)
    assert int(re.search(r"#define DWBC_RAND_COLS (\d+)", hdr).group(1)) == C.RAND_COLS == L.RAND_COLS
    for k, v in L.GS_COL.items():
        pass
    assert int(re.search(r"DWBC_GS = (\d+)", hdr).group(1)) == L.GS and int(re.search(r"DWBC_DS = (\d+)", hdr).group(1)) == L.DS


def test_null_arguments_are_rejected_not_crashed(lib):
    assert lib.dwbc_post_physics_step(None, None, None, None) == -1
    assert lib.dwbc_gae(None, None, None, None, None, None, None, 4, 4, 0.99, 0.95, 1, None) == -1
    assert lib.dwbc_workspace_bytes(None, 16) == -1


def test_params_tables():
    p = dwbc_b200.WidowGo1Params(num_envs=4)
    assert p.num_obs == 860 and p.max_episode_length == 500 and p.resample_interval == 150 and p.push_interval == 150
    assert p.ig2raisim() == [3, 4, 5, 0, 1, 2, 9, 10, 11, 6, 7, 8] + list(range(12, 20))
    assert p.active_terms("leg") == ["energy_square", "foot_contacts_z", "hip_action_l2", "survive", "tracking_ang_vel_yaw_exp",
                                     "tracking_lin_vel_x_l1"]
    cur = dwbc_b200.CommandCurriculum(p)
    cur.update()
    assert abs(cur.reward_scales["tracking_ang_vel_yaw_exp"] - 0.15) < 1e-12 and cur.lin_vel_x_ranges.tolist() == [0.0, 0.9]


def test_flat_actor_critic_layout_cpu():
    from dwbc_b200.actor_critic import FlatActorCritic
    from oracle import ppo_oracle as PO
    ac = FlatActorCritic(device="cpu", seed=0, init_std=[[0.8, 1.0, 1.0] * 4 + [1.0] * 6], num_priv=24, num_hist=10, num_prop=76)
    assert ac.manifest == PO.param_manifest() and ac.num_real_params == 168698
    sd = ac.state_dict()
    assert list(sd) == [n for n, _ in ac.manifest] and sd["std"].shape == (1, 18)
    assert all(ac.offsets[n] % 32 == 0 for n in ac.offsets)
    ac2 = FlatActorCritic(device="cpu", seed=1, num_priv=24, num_hist=10, num_prop=76)
    ac2.load_state_dict(sd)
    assert all((ac2.views[k] == sd[k]).all() for k in sd)
    hf, hc = ac.hist_range
    assert hf == ac.offsets["actor.history_encoder.encoder.0.weight"] and hf + hc == ac.offsets["actor.actor_backbone.0.weight"]
