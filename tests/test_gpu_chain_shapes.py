"""The fused tensor-core chains (chain2_kernel, wgrad_group_kernel, pack_weights2_kernel) on networks other than the shipped one, against a
float64 reference: torch autograd of the oracle (oracle/ppo_oracle.py) on CPU.  The sweep (NETWORKS in test_chain_shapes_cpu.py, which
also pins that they run on the chains) reaches row-major hidden activations (every width but 128), padded K windows and outputs,
deeper backbones, heads of one and three hidden layers and a latent of 16; G does not fit the chains' pack list in the update and must
fall back to the layer-wise path.  'fp32' (layer-wise CUDA cores) is the control that shows the reference is right.

Tolerances: CHAIN_TOL of test_gpu_ppo.py, measured against float64 here -- forward (means, values, actions, log-probs, bootstrap values)
max abs; gradient ||g - g_ref|| <= grad ||g_ref|| + GRAD_ABS per parameter tensor; losses |l - l_ref| <= loss (|l_ref| + 1e-3)."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from dwbc_b200 import synth
from oracle import ppo_oracle as PO
from test_chain_shapes_cpu import NETWORKS, dims, make_ac
from test_gpu_ppo import CHAIN_TOL
from test_oracle_golden import ppo_hp

pytestmark = pytest.mark.gpu

TOL = dict(CHAIN_TOL, fp32=CHAIN_TOL["tf32x3"])
# Absolute floor of the per-tensor gradient bound.  The error of a TF32 gradient goes with the sum of |row contributions|, not with their
# (cancelling) sum: against float64, small gradients of the SHIPPED network (S) at 16 973 rows -- the critic's first-layer weights (norm
# 0.018) and head biases (0.004) -- miss CHAIN_TOL's relative 1e-2 by up to 1.8e-4 absolute, and so do those of the layer-wise TF32 GEMMs (G's
# update), while 'tf32x3' on the same chains stays at 1e-5 relative.  'tf32' floor = 2 x that largest absolute error at S (H100 SXM, 700 W).
GRAD_ABS = dict(fp32=1e-7, tf32x3=1e-7, tf32=4e-4)
N_ENVS, T, SEED, COUNTER = 4100, 5, 41, 1500          # storage of 20 500 rows: enough for the largest mini-batch; no rollout has 4100 rows
_ref = {}                                             # float64 oracle results per (network, kind, rows)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def rollout_rows():
    """1, 129 and both sides of the split boundary of dwbc_policy_act: up to sms / 4 tiles a rollout runs one program per head."""
    b = 128 * (sms() // 4)
    return (1, 129, b, b + 1)


def grad_rows():
    """1, 129, and a mini-batch that on 'tf32' becomes two-tile plus one-tile work items with a ragged last tile."""
    return (1, 129, 128 * sms() + 77)


def params(net):
    manifest = PO.param_manifest(**dims(net))
    vals = synth.policy_params(manifest, SEED)
    std = torch.tensor([[0.8, 1.0, 1.0] * 4 + [1.0] * 6])
    return manifest, {n: (std.clone() if v is None else torch.from_numpy(v).clone()) for (n, _), v in zip(manifest, vals)}


@functools.lru_cache(maxsize=1)
def storage_inputs():
    """Storage contents of every test (cached: callers copy them, never modify them)."""
    obs = torch.from_numpy(synth.normal(SEED, 301, (T, N_ENVS, 860)))
    return dict(observations=obs, actions=torch.from_numpy(synth.normal(SEED, 50, (T, N_ENVS, 18))),
                values=torch.from_numpy(synth.normal(SEED, 51, (T, N_ENVS, 2))), returns=torch.from_numpy(synth.normal(SEED, 52, (T, N_ENVS, 2))),
                actions_log_prob=torch.from_numpy(synth.normal(SEED, 53, (T, N_ENVS, 2), -20.0, 1.0)),
                advantages=torch.from_numpy(synth.normal(SEED, 54, (T, N_ENVS, 2))))


def rollout_inputs(rows):
    obs = torch.from_numpy(synth.normal(SEED, 70, (rows, 860)))
    eps = torch.from_numpy(synth.normal(SEED, 71, (rows, 18)))
    return obs, eps


def minibatch_index():
    return torch.from_numpy(np.argsort(synth.uniform(SEED, 60, (N_ENVS * T,)))).long()


def ref_rollout(net, rows, hist):
    key = (net, "act", rows, hist)
    if key not in _ref:
        P = {k: v.double() for k, v in params(net)[1].items()}
        obs, eps = rollout_inputs(rows)
        r = PO.policy_act(P, obs.double(), eps.double(), hist_encoding=hist)
        _ref[key] = [r["mean"], r["values"], r["actions"], r["log_prob"]]
    return _ref[key]


def ref_grad(net, rows):
    key = (net, "grad", rows)
    if key not in _ref:
        P = {k: v.double().requires_grad_(True) for k, v in params(net)[1].items()}
        st = {k: v.double() for k, v in storage_inputs().items()}
        loss, info = PO.minibatch_loss(P, PO.gather(st, minibatch_index()[:rows]), ppo_hp(), COUNTER)
        loss.backward()
        g = {n: (p.grad if p.grad is not None else torch.zeros_like(p)).detach() for n, p in P.items()}
        _ref[key] = (g, [float(info["surrogate"]), float(info["value"]), float(info["priv_reg"])])
    return _ref[key]


def make_alg(net, precision):
    from dwbc_b200.ppo import FusedPPO
    manifest, P = params(net)
    ac = make_ac(net, "cuda:0")
    assert ac.manifest == manifest
    ac.load_state_dict(P)
    alg = FusedPPO(ac, device="cuda:0", **dict(ppo_hp(), num_mini_batches=1, num_learning_epochs=1, precision=precision))
    alg.init_storage(N_ENVS, T, [860], [None], [18])
    alg.counter = COUNTER
    s = alg.storage
    for k, v in storage_inputs().items():
        (s._obs_all[:T] if k == "observations" else getattr(s, k)).copy_(v.cuda())
    return alg


def run_rollout(alg, rows, hist, ws=None):
    """PPO.act (dwbc_policy_act) and the critic-only bootstrap of compute_returns (dwbc_critic_values) on `rows` rows; `ws`: the
    workspace to use instead of the algorithm's zero-filled one."""
    from dwbc_b200 import _lib as L
    if ws is not None:
        alg._ws, alg._ws_rows = ws, 1 << 30
    alg._packed = False
    obs, eps = (t.cuda() for t in rollout_inputs(rows))
    alg.act(obs, obs, hist, eps=eps)
    tr = alg.transition
    out = [tr.action_mean.clone(), tr.values.clone(), tr.actions.clone(), tr.actions_log_prob.clone()]
    boot = torch.zeros(rows, 2, device="cuda")
    ac = alg.actor_critic
    L.check(L.lib().dwbc_critic_values(C.addressof(ac.net_cfg), L.ptr(ac.flat), L.ptr(obs), obs.stride(0), L.ptr(boot), rows,
                                       L.ptr(alg._workspace(rows)), L.stream_ptr()), "dwbc_critic_values")
    alg._packed = False                       # (dwbc_critic_values re-packs into the same workspace region, as in compute_returns)
    return out + [boot]


def run_grad(alg, rows, ws=None):
    from dwbc_b200 import _lib as L
    ac, s = alg.actor_critic, alg.storage
    idx = minibatch_index()[:rows].cuda()
    h = alg._fill_hp()
    alg._set_precision()
    alg._losses.zero_()
    L.check(L.lib().dwbc_ppo_minibatch_grad(C.addressof(ac.net_cfg), L.ptr(ac.flat), s.c_struct_ptr(), L.ptr(idx), rows, C.addressof(h),
                                            L.ptr(alg.grad), L.ptr(alg._losses), L.ptr(alg._workspace(rows) if ws is None else ws),
                                            L.stream_ptr()), "dwbc_ppo_minibatch_grad")
    return {k: v.clone() for k, v in ac.unflat(alg.grad).items()}, alg._losses[:3].clone()


def grad_errors(got, ref, tol, floor):
    """(tensor, worst ||g - g_ref|| / ||g_ref|| over the tensors with a non-zero reference, largest ||g - g_ref||); asserts the per-tensor
    bound"""
    worst, dmax = ("", 0.0), 0.0
    for k, r in ref.items():
        g = got[k].double().cpu()
        assert torch.isfinite(g).all(), k
        d, nr = float((g - r).norm()), float(r.norm())
        assert d <= tol * nr + floor, (k, d, nr)
        dmax = max(dmax, d)
        if nr > 1e-6 and d / nr > worst[1]:
            worst = (k, d / nr)
    return worst + (dmax,)


@pytest.mark.parametrize("precision", ["tf32x3", "tf32", "fp32"])
@pytest.mark.parametrize("net", sorted(NETWORKS))
def test_chain_rollout_matches_float64(net, precision):
    """PPO.act (means, values, actions, log-probs) and the bootstrap values of compute_returns at 1, 129 rows and on both sides of the
    split into one program per head; with the history-encoder latent too for S and E."""
    tol = TOL[precision]["fwd"]
    alg = make_alg(net, precision)
    for hist in ((False, True) if net in ("S", "E") else (False,)):
        for rows in rollout_rows():
            got = run_rollout(alg, rows, hist)
            ref = ref_rollout(net, rows, hist)
            errs = [float((g.double().cpu() - r).abs().max()) for g, r in zip(got, ref + [ref[1]])]
            print(f"[{net} {precision} hist={int(hist)} rows={rows}] max abs error vs float64: mean {errs[0]:.3g} value {errs[1]:.3g} "
                  f"action {errs[2]:.3g} log-prob {errs[3]:.3g} bootstrap {errs[4]:.3g}")
            assert all(torch.isfinite(t).all() for t in got)
            assert max(errs) < tol, (rows, hist, errs)


@pytest.mark.parametrize("precision", ["tf32x3", "tf32", "fp32"])
@pytest.mark.parametrize("net", sorted(NETWORKS))
def test_chain_minibatch_grad_matches_float64(net, precision):
    """dwbc_ppo_minibatch_grad (forward chains with the loss in the epilogues, backward chains, grouped weight gradients; G layer-wise):
    per-tensor gradients and the surrogate / value / regulariser losses at 1, 129 rows and one mini-batch of sms tiles + 77 rows."""
    tol = TOL[precision]
    alg = make_alg(net, precision)
    for rows in grad_rows():
        got, losses = run_grad(alg, rows)
        ref, ref_losses = ref_grad(net, rows)
        worst = grad_errors(got, ref, tol["grad"], GRAD_ABS[precision])
        lerr = max(abs(float(losses[i]) - ref_losses[i]) / (abs(ref_losses[i]) + 1e-3) for i in range(3))
        print(f"[{net} {precision} rows={rows}] worst ||dg||/||g|| vs float64 {worst[1]:.3g} ({worst[0]}), largest ||dg|| {worst[2]:.3g}, losses rel {lerr:.3g}")
        assert lerr <= tol["loss"], (rows, losses.tolist(), ref_losses)


@pytest.mark.parametrize("precision", ["tf32x3", "tf32", "fp32"])
@pytest.mark.parametrize("net", ["B", "C"])
def test_results_do_not_depend_on_workspace_contents(net, precision):
    """The library promises nothing about the workspace but zeroed queue counters in its first 256 bytes: with every other byte NaN the
    rollout must be bitwise the same as on a zeroed workspace (it has no atomics) and the gradient must agree within the tolerance.  This
    holds the zero fill of padded K windows and of rows past the matrix in the chains, and of the weight-gradient operands."""
    tol = TOL[precision]
    alg = make_alg(net, precision)
    rows_g = grad_rows()[-1]
    zero = alg._workspace(rows_g)
    nan = torch.full_like(zero, float("nan"))
    nan[:64] = 0.0
    for rows in rollout_rows()[1::2]:                   # ragged: 129 rows (one program per head), sms / 4 tiles + 1 row (shared programs)
        a = run_rollout(alg, rows, False, ws=zero)
        b = run_rollout(alg, rows, False, ws=nan)
        assert all(torch.isfinite(t).all() for t in b), rows
        assert all(torch.equal(x, y) for x, y in zip(a, b)), rows
    g0, l0 = run_grad(alg, rows_g, ws=zero)
    g1, l1 = run_grad(alg, rows_g, ws=nan)
    worst = grad_errors(g1, {k: v.double().cpu() for k, v in g0.items()}, tol["grad"], GRAD_ABS[precision])
    assert torch.isfinite(l1).all() and float((l1 - l0).abs().max()) <= tol["loss"] * (float(l0.abs().max()) + 1e-3)
    print(f"[{net} {precision}] NaN-filled workspace: rollout bitwise equal, worst ||dg||/||g|| {worst[1]:.3g} ({worst[0]})")
