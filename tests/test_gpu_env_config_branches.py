"""The post-physics step on the config branches no shipped config takes (tests/envstate.py BRANCH_CASES: cart goals with orientation
deltas, the positive-reward clip with termination on both channels, the goal search at 0 .. 16 collision samples, no DOF reordering and
no push with 8 penalised / 3 termination contact bodies and per-joint limits, action delays 0, 1 and 6 with a binding action clip),
both kernels against the CPU oracle at every step of a 30-step table-mode rollout.  test_env_config_branches_cpu.py checks on the same
rollouts that each branch really decided something.

Then the action-delay FIFO (dwbc_pre_physics_actions) and the PD controller (dwbc_compute_torques) on their own through the C ABI, away
from the shipped shapes: every FIFO length and delay row, per-joint distinct gains and limits."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import envstate as E
from dwbc_b200 import _lib as L
from dwbc_b200.config import WidowGo1Params
from oracle import env_oracle as EO
from test_env_config_branches_cpu import COUNTER0, SEED, STEPS
from test_gpu_env_rollout import rollout_vs_oracle

pytestmark = pytest.mark.gpu

TMA_CASES = [k for k in E.BRANCH_CASES if not k.startswith("delay")]     # the TMA kernel takes only action_hist_len 4
KERNELS = [(1024, False, True), (1024, True, False), (1000, False, False)]   # N, generic_kernel, TMA kernel expected
CASES = [pytest.param(name, N, g, tma and name in TMA_CASES, id=f"{name}-{N}-{'generic' if g else 'auto'}")
         for name in E.BRANCH_CASES for N, g, tma in KERNELS if name in TMA_CASES or not g]


@pytest.mark.parametrize("name,N,generic_kernel,tma", CASES)
def test_config_branch_rollout_matches_oracle(name, N, generic_kernel, tma):
    """Every output and state buffer against the oracle at each step, episode sums and extras['episode'] included; the TMA kernel runs
    each TMA-eligible case at 1024 envs, the warp-per-env kernel runs it forced at 1024 and at 1000; the delay cases take the warp-per-env
    kernel by themselves at 1024 (out-of-range counter 0)."""
    p = WidowGo1Params(num_envs=N, **E.BRANCH_CASES[name])
    rec = rollout_vs_oracle(p, SEED, STEPS, specialised=tma, generic_kernel=generic_kernel, counter0=COUNTER0)
    assert int(rec["reset"].sum()) > 0


# ---------------------------------------------------------------------------------------------- action-delay FIFO (WG:1162-1173)
@pytest.mark.parametrize("N", [1, 333, 4096])
@pytest.mark.parametrize("ah", range(2, 9))
def test_action_fifo_matches_restatement(ah, N):
    """dwbc_pre_physics_actions at FIFO length `ah` and every delay row, 4 steps each, clip_actions 0.5, a permutation other than the
    shipped one: the FIFO and the delayed action bit for bit against torch (clip, shift, append, read row `delay_row` of the shifted
    FIFO, i.e. action_history_buf[:, -action_delay - 1] with action_delay = ah - 1 - delay_row)."""
    lib, na, clip = L.lib(), 18, 0.5
    g = torch.Generator().manual_seed(1000 * ah + N)
    perm = torch.randperm(na, generator=g)
    r2i = perm.to(torch.int32).cuda()
    hist0 = torch.randn(N, ah, na, generator=g)
    n_clipped = 0
    for delay_row in range(ah):
        hist, ref = hist0.cuda(), hist0.clone()
        for step in range(4):
            pol = torch.randn(N, na, generator=g)
            pol_d, actions = pol.cuda(), torch.full((N, na), float("nan"), device="cuda")
            L.check(lib.dwbc_pre_physics_actions(L.ptr(pol_d), L.ptr(r2i, torch.int32), clip, L.ptr(hist), L.ptr(actions), N, na, ah,
                                                 delay_row, L.stream_ptr()), "dwbc_pre_physics_actions")
            a = torch.clip(pol[:, perm], -clip, clip)
            n_clipped += int((pol.abs() > clip).sum())
            ref = torch.cat([ref[:, 1:], a[:, None, :]], dim=1)
            assert torch.equal(hist.cpu(), ref), f"FIFO, delay row {delay_row}, step {step}"
            assert torch.equal(actions.cpu(), ref[:, delay_row]), f"delayed action, delay row {delay_row}, step {step}"
    assert n_clipped > ah * 4 * N * na // 3


# ---------------------------------------------------------------------------------------------- PD controller (WG:1262-1295)
@pytest.mark.parametrize("N", [1, 333, 1000])
@pytest.mark.parametrize("n_act", [20, 18, 14])
def test_pd_controller_with_per_joint_parameters_matches_oracle(n_act, N):
    """dwbc_compute_torques with per-joint distinct gains, action scales, defaults and limits (some limits 0), against EO.compute_torques:
    limits binding on both signs, the wrapped column (DOF n_act - 8) several turns outside (-pi, pi], driven DOFs n_act == n_dof and
    n_act < n_dof, and N * n_dof not a multiple of the 256-thread block.  Bit for bit except the wrapped column (5e-5, as the golden test:
    the wrap may differ by an ulp of the angle, times that joint's p gain)."""
    nd, wrap = 20, n_act - 8
    j = torch.arange(nd, dtype=torch.float32)
    p_gains = 12.0 + 1.75 * j[:n_act]
    p_gains[wrap] = 3.5                                   # keeps an ulp of a ~20 rad angle times the gain below the wrapped column's bound
    d_gains = 0.3 + 0.07 * j[:n_act]
    scale = 0.2 + 0.05 * j[:n_act]
    default = 0.1 * torch.sin(1.3 * j) + 0.02 * j
    limits = 4.0 + 1.5 * j
    limits[[3, 9, n_act - 1]] = 0.0
    cfg = L.PdCfg()
    cfg.n_dof, cfg.n_act, cfg.wrap_dof = nd, n_act, wrap
    for k, src in (("p_gains", p_gains), ("d_gains", d_gains), ("action_scale", scale), ("default_dof_pos", default),
                   ("torque_limits", limits)):
        arr = getattr(cfg, k)
        for i, v in enumerate(src.tolist()):
            arr[i] = v
    g = torch.Generator().manual_seed(7 * N + n_act)
    actions = torch.randn(N, n_act, generator=g) * 1.5
    motor = 0.7 + 0.6 * torch.rand(N, n_act, generator=g)
    pos = default + 0.6 * torch.randn(N, nd, generator=g)
    pos[:, wrap] = 40.0 * torch.rand(N, generator=g) - 20.0 if N > 1 else torch.tensor([-17.3])
    vel = 2.0 * torch.randn(N, nd, generator=g)
    dof_state = torch.stack([pos, vel], dim=-1).reshape(N * nd, 2).cuda()
    actions_d, motor_d, out = actions.cuda(), motor.cuda(), torch.full((N, nd), float("nan"), device="cuda")
    L.check(L.lib().dwbc_compute_torques(C.addressof(cfg), L.ptr(actions_d), L.ptr(dof_state), L.ptr(motor_d), L.ptr(out), N,
                                         L.stream_ptr()), "dwbc_compute_torques")
    got = out.cpu()
    ref = EO.compute_torques(actions, pos, vel, motor, p_gains, d_gains, scale, default, limits, wrap_col=wrap)
    cols = [c for c in range(nd) if c != wrap]
    np.testing.assert_array_equal(got[:, cols].numpy(), ref[:, cols].numpy())
    np.testing.assert_allclose(got[:, wrap].numpy(), ref[:, wrap].numpy(), rtol=0, atol=5e-5)
    assert not bool(got[:, n_act:].any())
    if N > 1:
        lim = limits.expand(N, nd)
        driven = lim[:, :n_act] > 0
        assert bool((got[:, :n_act] == lim[:, :n_act])[driven].any()) and bool((got[:, :n_act] == -lim[:, :n_act])[driven].any())
        assert bool((got.abs() < lim)[:, :n_act][driven].any())
        assert float(pos[:, wrap].abs().max()) > 3 * math.pi
