"""CPU (float64, no device): the builder of the regime mini-batches of test_gpu_ppo_loss_regimes.py.

The builder writes storage rows from the float64 oracle (oracle/ppo_oracle.py) so that every (row, channel) of a mini-batch sits in one
branch of the PPO loss with a margin that the kernels' rounding cannot cross:
  surrogate -- log-ratio l = logp64 - old_log_prob: 'low' ln(1 - clip) - u, 'in' inside [ln(1 - clip), ln(1 + clip)] with >= 0.05 to
               either edge, 'high' ln(1 + clip) + u (u in [0.1, 0.6], so no row dominates); the sign of the mixed advantage
               (|mix| in [0.2, 2]): six regimes, two of which (low, -) and (high, +) leave no surrogate gradient;
  value     -- dvo = v64 - values: 'below' -(clip + u), 'inside' |dvo| <= clip - 0.05, 'above' clip + u; outside the band the returns sit
               at w in [0.1, 0.6] from the midpoint of v and its clipped value, on the side that makes (v - R)^2 win ('l1') or lose
               ('l2'): five regimes, two of which (below/l2, above/l2) leave no value gradient with the clipped value loss.
The advantages are solved from the target mixed advantages through [[1, rho], [rho, 1]]; at rho = 1 (singular) both channels share one
target.  Here every set and batch is checked against the oracle again on the fp32 storage as the device reads it."""
import functools
import math

import numpy as np
import pytest
import torch

from dwbc_b200 import synth
from oracle import ppo_oracle as PO
from test_gpu_chain_shapes import COUNTER, N_ENVS, SEED, T, minibatch_index, params, storage_inputs
from test_oracle_golden import ppo_hp

MARGIN, U_LO, U_HI, MIX_LO, MIX_HI = 0.05, 0.1, 0.6, 0.2, 2.0
SURR = [("low", 1), ("low", -1), ("in", 1), ("in", -1), ("high", 1), ("high", -1)]
VALUE = ["inside", "below/l1", "below/l2", "above/l1", "above/l2"]
# single-regime batches k = 0..5: surrogate regime SURR[k] and value regime VALUE[k % 5] in every row and channel; 'mixed': all of them
BATCHES = [f"s{k}" for k in range(len(SURR))] + ["mixed"]

_H1 = dict(clip_param=0.1, value_loss_coef=0.5, entropy_coef=0.01, mixing_schedule=[0.74, 1000, 1000],
           priv_reg_coef_schedual=[0.1, 0.7, 1200, 1000])
# at COUNTER = 1500: H0 rho 1, c_reg 0.5 (shipped); H1 rho 0.37, c_reg 0.28; H2 rho 0, c_reg 0.2; H3 = H1 + torque supervision weight 0.05
SETS = {
    "H0": {},
    "H1": _H1,
    "H2": dict(clip_param=0.3, value_loss_coef=2.0, entropy_coef=0.005, use_clipped_value_loss=False, mixing_schedule=[1.0, 2000, 1000],
               priv_reg_coef_schedual=[0.2, 0.2, 0, 1]),
    "H3": dict(_H1, torque_supervision=True, adaptive_arm_gains=False, torque_supervision_schedule=[0.1, 1000, 1000]),
}


def hyper(name):
    """PPO hyper-parameters of set `name` (without the arm coefficients: arm_coefs())."""
    hp = ppo_hp()
    hp.update(SETS[name])
    return hp


def arm_inputs():
    """Torque-supervision rows of the storage and the arm coefficients (those of the ppo_ts golden: synth.arm_torque_inputs)."""
    ts = synth.arm_torque_inputs(N_ENVS, T, 6, SEED)
    return {k: torch.from_numpy(ts[k]) for k in ("target_arm_torques", "current_arm_dof_pos", "current_arm_dof_vel")}, \
        tuple(torch.from_numpy(np.asarray(c, np.float32)) for c in ts["coefs"])


def oracle_hp(name):
    """The oracle's hp dict of set `name` (arm coefficients in float64 when torque supervision is on)."""
    hp = hyper(name)
    if hp.get("torque_supervision"):
        hp["arm_coefs"] = tuple(c.double() for c in arm_inputs()[1])
    return hp


@functools.lru_cache(maxsize=1)
def forward64():
    """float64 log-probs of the stored actions and values of every storage row [T*N, 2] at the fp32 parameters of network S."""
    P = {k: v.double() for k, v in params("S")[1].items()}
    st = storage_inputs()
    obs = st["observations"].flatten(0, 1).double()
    with torch.no_grad():
        mean = PO.actor_mean(P, obs)
        return PO.log_prob2(mean, P["std"], st["actions"].flatten(0, 1).double()), PO.critic_values(P, obs)


def _u(stream, shape, lo=0.0, hi=1.0):
    return torch.from_numpy(synth.uniform(SEED, stream, shape, lo, hi)).double()


def labels(batch):
    """(surrogate regime index into SURR, value regime index into VALUE), each [T*N, 2]"""
    R = N_ENVS * T
    if batch == "mixed":
        s = torch.from_numpy((synth.uniform(SEED, 900, (R, 2)) * len(SURR)).astype(np.int64)).clamp_(max=len(SURR) - 1)
        v = torch.from_numpy((synth.uniform(SEED, 901, (R, 2)) * len(VALUE)).astype(np.int64)).clamp_(max=len(VALUE) - 1)
        return s, v
    k = int(batch[1:])
    return torch.full((R, 2), k, dtype=torch.int64), torch.full((R, 2), k % len(VALUE), dtype=torch.int64)


def _rho(hp):
    return PO.value_mixing_ratio(COUNTER, hp["mixing_schedule"])


@functools.lru_cache(maxsize=None)
def build(name, batch):
    """Storage of set `name`, batch `batch`: dict of fp32 [T, N, k] tensors (observations, actions and, with torque supervision, the arm
    targets as in storage_inputs / arm_inputs) and the regime labels (surr, value) [T*N, 2]."""
    hp = hyper(name)
    clip, rho = hp["clip_param"], _rho(hp)
    R = N_ENVS * T
    lp64, v64 = forward64()
    s_lab, v_lab = labels(batch)
    if rho == 1.0:                           # one target per row: the channels' mixed advantages are equal, so are their signs
        s_lab = s_lab.clone()
        s_lab[:, 1] = torch.tensor([SURR.index((SURR[int(j)][0], SURR[int(i)][1])) for i, j in s_lab.tolist()])
    kind = [SURR[i][0] for i in range(len(SURR))]
    sign = torch.tensor([float(s) for _, s in SURR], dtype=torch.float64)[s_lab]
    lo, hi = math.log(1 - clip), math.log(1 + clip)
    u = _u(902, (R, 2), U_LO, U_HI)
    t_in = _u(903, (R, 2), lo + MARGIN, hi - MARGIN)
    is_low = torch.tensor([k == "low" for k in kind])[s_lab]
    is_high = torch.tensor([k == "high" for k in kind])[s_lab]
    ell = torch.where(is_low, lo - u, torch.where(is_high, hi + u, t_in))
    mix = sign * _u(904, (R, 2), MIX_LO, MIX_HI)
    if rho == 1.0:
        t = _u(905, (R,), -0.5, 0.5)
        adv = torch.stack([mix[:, 0] / 2 + t, mix[:, 0] / 2 - t], dim=1)
    else:
        adv = torch.stack([mix[:, 0] - rho * mix[:, 1], mix[:, 1] - rho * mix[:, 0]], dim=1) / (1 - rho * rho)
    vk = [VALUE[i] for i in range(len(VALUE))]
    below = torch.tensor([k.startswith("below") for k in vk])[v_lab]
    above = torch.tensor([k.startswith("above") for k in vk])[v_lab]
    wins_l1 = torch.tensor([k.endswith("l1") for k in vk])[v_lab]
    uv = _u(906, (R, 2), U_LO, U_HI)
    dvo = torch.where(below, -(clip + uv), torch.where(above, clip + uv, _u(907, (R, 2), -(clip - MARGIN), clip - MARGIN)))
    w = _u(908, (R, 2), U_LO, U_HI)
    vc = v64 - dvo + dvo.clamp(-clip, clip)                                  # the clipped value of v64
    side = torch.sign(v64 - vc)                                              # +1 above, -1 below, 0 inside
    mid = (v64 + vc) / 2
    s_inside = torch.where(_u(909, (R, 2)) < 0.5, -1.0, 1.0).double()
    ret = torch.where(below | above, torch.where(wins_l1, mid - side * w, mid + side * w), v64 + s_inside * w)
    f = lambda x: x.float().reshape(T, N_ENVS, 2)  # noqa: E731
    st = dict(storage_inputs(), actions_log_prob=f(lp64 - ell), advantages=f(adv), values=f(v64 - dvo), returns=f(ret))
    if hp.get("torque_supervision"):
        st.update(arm_inputs()[0])
    return st, s_lab, v_lab


def realised(name, st):
    """The regimes (surr, value) [T*N, 2] the float64 oracle finds on the fp32 storage `st`, and the smallest margins:
    log-ratio to the nearest band edge, |mix|, |dvo| to +-clip, |R - midpoint| (outside rows)."""
    hp = hyper(name)
    clip, rho = hp["clip_param"], _rho(hp)
    lp64, v64 = forward64()
    g = lambda k: st[k].flatten(0, 1).double()  # noqa: E731
    ell = lp64 - g("actions_log_prob")
    a = g("advantages")
    mix = torch.stack([a[:, 0] + rho * a[:, 1], a[:, 1] + rho * a[:, 0]], dim=1)
    lo, hi = math.log(1 - clip), math.log(1 + clip)
    kind = torch.where(ell < lo, 0, torch.where(ell > hi, 2, 1))
    s_idx = kind * 2 + (mix < 0).long()                                      # SURR order: (low,+) (low,-) (in,+) (in,-) (high,+) (high,-)
    vo, ret = g("values"), g("returns")
    dvo = v64 - vo
    vc = vo + dvo.clamp(-clip, clip)
    l1, l2 = (v64 - ret) ** 2, (vc - ret) ** 2
    out = (dvo.abs() > clip)
    v_idx = torch.where(~out, 0, 1 + 2 * (dvo > clip).long() + (l2 > l1).long())   # VALUE order
    margins = dict(log_ratio=float(torch.minimum((ell - lo).abs(), (ell - hi).abs()).min()), mix=float(mix.abs().min()),
                   dvo=float((dvo.abs() - clip).abs().min()), ret=float(((ret - (v64 + vc) / 2).abs())[out].min()) if out.any() else 1.0,
                   u_max=float(torch.maximum(lo - ell, ell - hi).max()), mix_max=float(mix.abs().max()))
    return s_idx, v_idx, mix, margins


@pytest.mark.parametrize("name", sorted(SETS))
def test_regime_storage_holds_every_row_in_its_branch(name):
    """Every storage row (a superset of every mini-batch the GPU test gathers) is in the regime it was built for, with the margins."""
    perm = minibatch_index()
    for batch in BATCHES:
        st, s_lab, v_lab = build(name, batch)
        s_idx, v_idx, mix, m = realised(name, st)
        assert torch.equal(s_idx, s_lab), (name, batch, int((s_idx != s_lab).sum()))
        assert torch.equal(v_idx, v_lab), (name, batch, int((v_idx != v_lab).sum()))
        tol = 1e-4                            # fp32 rounding of the stored rows
        assert m["log_ratio"] >= MARGIN - tol and m["dvo"] >= MARGIN - tol and m["mix"] >= MIX_LO - tol and m["ret"] >= U_LO - tol, (batch, m)
        assert m["u_max"] <= U_HI + tol and m["mix_max"] <= MIX_HI + tol, (batch, m)
        if batch == "mixed":                  # every regime in the 129-row batch
            first = perm[:129]
            assert set(s_idx[first].flatten().tolist()) == set(range(len(SURR))), name
            assert set(v_idx[first].flatten().tolist()) == set(range(len(VALUE))), name
        if _rho(hyper(name)) == 1.0:          # one target per row
            assert torch.equal(mix[:, 0], mix[:, 1]), name


def test_regime_sets_reach_the_scheduled_values():
    """The schedules of the sets give the coefficients they are meant to test at COUNTER."""
    got = {n: (PO.value_mixing_ratio(COUNTER, hyper(n)["mixing_schedule"]), PO.priv_reg_coef(COUNTER, hyper(n)["priv_reg_coef_schedual"]))
           for n in SETS}
    assert got["H0"] == (1.0, 0.5) and got["H2"] == (0.0, 0.2)
    assert got["H1"] == got["H3"] and abs(got["H1"][0] - 0.37) < 1e-12 and abs(got["H1"][1] - 0.28) < 1e-12
    assert PO.torque_supervision_weight(COUNTER, hyper("H3")["torque_supervision_schedule"]) == 0.05
