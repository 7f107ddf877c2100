"""GPU: dwbc_policy_mean, the actor forward alone, against the mean output of dwbc_policy_act (bit for bit) and against the float64 oracle.

The cases cover the three precisions, teacher (privileged latent) and student (history latent) mode, 10-, 20- and 50-step histories, two
hidden activations other than ELU, the sweep networks of test_gpu_chain_shapes.py (G's rollout runs on the chains; the stock 512/256/128
trunks run layer-wise), rows on both sides of both program splits (dwbc_policy_act splits at 4 * tiles <= SMs, dwbc_policy_mean at
2 * tiles <= SMs: 8192 rows = 64 tiles splits one and not the other on an H100), observations read from rows wider than num_obs and from an
unaligned pointer.  Then: a NaN-filled workspace gives the same bits, a parameter change that PolicyMean's key sees re-packs the weight
images, and FusedActorCritic.act_inference returns what dwbc_policy_act returned for it before (eps = 0, its mean output)."""
import ctypes as C

import numpy as np
import pytest
import torch

from dwbc_b200 import _lib as L
from dwbc_b200 import synth
from oracle import ppo_oracle as PO
from test_chain_shapes_cpu import _AC_KW, NETWORKS, dims
from test_gpu_chain_shapes import TOL

pytestmark = pytest.mark.gpu

SEED = 43
ROWS = (1, 37, 128, 4096, 8192, 40960)
STOCK = dict(actor_dims=(512, 256, 128), critic_dims=(512, 256, 128))       # rsl_rl's default trunks: wider than a tile, layer-wise
NETS = dict(NETWORKS, STOCK=STOCK)
STD = [[0.8, 1.0, 1.0] * 4 + [1.0] * 6]


def make_ac(net="S", num_hist=10, activation="elu", seed=SEED):
    from dwbc_b200.actor_critic import FlatActorCritic
    ac = FlatActorCritic(device="cuda:0", num_priv=24, num_hist=num_hist, num_prop=76, activation=activation,
                         **{_AC_KW[k]: v for k, v in NETS[net].items()})
    vals = synth.policy_params(ac.manifest, seed)
    ac.load_state_dict({n: (torch.tensor(STD) if v is None else torch.from_numpy(v)) for (n, _), v in zip(ac.manifest, vals)})
    return ac


def observations(ac, rows, layout="plain", seed=70):
    """[rows, num_obs] standard normals: 'plain' contiguous; 'wide' rows of a [rows, num_obs + 8] buffer (a storage row layout with
    obs_stride > num_obs); 'unaligned' a contiguous view starting one float past a 16-byte boundary."""
    x = torch.from_numpy(synth.normal(seed, rows, (rows, ac.num_obs))).cuda()
    if layout == "plain":
        return x
    if layout == "wide":
        buf = torch.full((rows, ac.num_obs + 8), float("nan"), device="cuda")
        buf[:, :ac.num_obs] = x
        return buf
    base = torch.empty(rows * ac.num_obs + 1, device="cuda")
    v = base[1:].view(rows, ac.num_obs)
    v.copy_(x)
    assert v.data_ptr() % 16
    return v


def workspace(ac, rows, fill=0.0):
    ws = torch.full((L.lib().dwbc_workspace_bytes(C.addressof(ac.net_cfg), rows) // 4 + 64,), fill, device="cuda")
    ws[:64] = 0.0                                       # the queue counters: the one thing the library needs zeroed
    return ws


def act_mean(ac, obs, hist, ws=None):
    """dwbc_policy_act's mean output (eps = 0)."""
    n, na = obs.shape[0], ac.num_leg_actions + ac.num_arm_actions
    z = lambda *s: torch.zeros(*s, device="cuda")  # noqa: E731
    eps, act, mu, sg, val, lp = z(n, na), z(n, na), z(n, na), z(n, na), z(n, 2), z(n, 2)
    ws = workspace(ac, n) if ws is None else ws
    L.check(L.lib().dwbc_policy_act(C.addressof(ac.net_cfg), L.ptr(ac.flat), L.ptr(obs), obs.stride(0), L.ptr(eps), int(hist), L.ptr(act),
                                    L.ptr(val), L.ptr(lp), L.ptr(mu), L.ptr(sg), n, 0, L.ptr(ws), L.stream_ptr()), "dwbc_policy_act")
    return mu


def policy_mean(ac, obs, hist, ws=None, packed=0):
    n = obs.shape[0]
    out = torch.full((n, ac.num_leg_actions + ac.num_arm_actions), float("nan"), device="cuda")
    ws = workspace(ac, n) if ws is None else ws
    L.check(L.lib().dwbc_policy_mean(C.addressof(ac.net_cfg), L.ptr(ac.flat), L.ptr(obs), obs.stride(0), int(hist), L.ptr(out), n, packed,
                                     L.ptr(ws), L.stream_ptr()), "dwbc_policy_mean")
    return out


def assert_same_bits(ac, obs, hist, what):
    a, m = act_mean(ac, obs, hist), policy_mean(ac, obs, hist)
    assert torch.isfinite(m).all(), what
    assert torch.equal(a, m), (what, float((a - m).abs().max()))


@pytest.mark.parametrize("precision", ["tf32x3", "tf32", "fp32"])
@pytest.mark.parametrize("net", sorted(NETS))
def test_mean_is_the_bits_of_policy_act(net, precision):
    """Every sweep network and the stock trunks, teacher and student, at every row count."""
    ac = make_ac(net)
    ac.net_cfg.precision = L.PRECISIONS[precision]
    for rows in ROWS:
        obs = observations(ac, rows)
        for hist in (False, True):
            assert_same_bits(ac, obs, hist, (rows, hist))


CASES = [dict(num_hist=20), dict(num_hist=50), dict(activation="selu"), dict(activation="tanh"), dict(layout="wide"),
         dict(layout="unaligned"), dict(net="STOCK", layout="wide")]


@pytest.mark.parametrize("precision", ["tf32x3", "tf32", "fp32"])
@pytest.mark.parametrize("case", CASES, ids=["h20", "h50", "selu", "tanh", "wide-rows", "unaligned", "stock-wide-rows"])
def test_mean_is_the_bits_of_policy_act_on_histories_activations_and_layouts(case, precision):
    case = dict(case)
    layout = case.pop("layout", "plain")
    ac = make_ac(**case)
    ac.net_cfg.precision = L.PRECISIONS[precision]
    for rows in (1, 37, 4096, 8192, 40960):
        obs = observations(ac, rows, layout)
        for hist in (False, True):
            assert_same_bits(ac, obs, hist, (rows, hist))


@pytest.mark.parametrize("precision", ["tf32x3", "tf32", "fp32"])
@pytest.mark.parametrize("net", sorted(NETWORKS))
def test_mean_matches_float64(net, precision):
    """The actor mean of the float64 oracle, at the forward tolerance of test_gpu_chain_shapes.py; the history latent too for S and E."""
    ac = make_ac(net)
    ac.net_cfg.precision = L.PRECISIONS[precision]
    P = {n: v.detach().double().cpu() for n, v in ac.views.items()}
    for hist in ((False, True) if net in ("S", "E") else (False,)):
        for rows in (1, 37, 4096):
            obs = observations(ac, rows)
            got = policy_mean(ac, obs, hist).double().cpu()
            ref = PO.actor_mean(P, obs.double().cpu(), hist)
            err = float((got - ref).abs().max())
            print(f"[{net} {precision} hist={int(hist)} rows={rows}] max abs error of the mean vs float64: {err:.3g}")
            assert err < TOL[precision]["fwd"], (rows, hist, err)


@pytest.mark.parametrize("precision", ["tf32x3", "tf32", "fp32"])
@pytest.mark.parametrize("net", ["S", "C", "STOCK"])
def test_mean_does_not_depend_on_the_workspace(net, precision):
    """A workspace NaN everywhere but its queue counters, weights_packed = 0: the bits of a zeroed one."""
    ac = make_ac(net)
    ac.net_cfg.precision = L.PRECISIONS[precision]
    for rows in (37, 8192):
        obs = observations(ac, rows)
        for hist in (False, True):
            a = policy_mean(ac, obs, hist, workspace(ac, rows))
            b = policy_mean(ac, obs, hist, workspace(ac, rows, float("nan")))
            assert torch.isfinite(b).all() and torch.equal(a, b), (rows, hist)


@pytest.mark.parametrize("precision", ["tf32x3", "tf32"])
def test_parameter_change_repacks(precision):
    """PolicyMean keeps the weight images between calls; load_state_dict bumps the parameters' version, so the next call re-packs and
    gives the new parameters' mean.  Control: weights_packed = 1 on the same workspace really reuses the old images."""
    from dwbc_b200.actor_critic import PolicyMean
    ac, other = make_ac(), make_ac(seed=SEED + 1)
    ac.net_cfg.precision = other.net_cfg.precision = L.PRECISIONS[precision]
    obs = observations(ac, 4096)
    pm = PolicyMean()
    out = torch.empty(4096, 18, device="cuda")
    old = pm(ac, obs, out).clone()
    assert torch.equal(pm(ac, obs, out), old)                  # second call: images reused (packed = 1)
    key = pm.key
    ac.load_state_dict(other.state_dict())
    new = pm(ac, obs, out).clone()
    assert pm.key != key
    assert torch.equal(new, policy_mean(other, obs, False)) and not torch.equal(new, old)
    ac.load_state_dict(make_ac().state_dict())                  # back to the old values, without telling the library
    stale = policy_mean(ac, obs, False, pm.ws, packed=1)
    assert torch.equal(stale, new)                             # the images of `other` were used


@pytest.mark.parametrize("precision", ["tf32x3", "tf32", "fp32"])
def test_act_inference_returns_what_it_returned_through_policy_act(precision):
    """FusedActorCritic.act_inference (and FlatActorCritic's) against its former implementation: dwbc_policy_act with eps = 0, the mean
    output, on the runner's observation layout, teacher and student."""
    from dwbc_b200.runner_compat import FusedActorCritic
    policy = FusedActorCritic(860, 860, 18, actor_hidden_dims=(128,), critic_hidden_dims=(128,), num_priv=24, num_hist=10, num_prop=76,
                              device="cuda:0")
    policy.load_state_dict(make_ac().state_dict())
    policy.core.net_cfg.precision = L.PRECISIONS[precision]
    for rows in (1, 4096, 40960):
        obs = observations(policy.core, rows)
        for hist in (False, True):
            ref = act_mean(policy.core, obs, hist)
            got = policy.act_inference(obs, hist_encoding=hist)
            assert got.shape == (rows, 18) and torch.equal(got, ref), (rows, hist)
            assert torch.equal(policy.core.act_inference(obs, hist), ref)
