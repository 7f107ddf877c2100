"""CPU: the PPO update diagnostics without a GPU.  The float64 restatement the GPU tests compare against (ref_diag) against a hand-written
per-row formula; the new exports and the unchanged struct sizes; the host-side refusals of dwbc_ppo_minibatch_grad_diag and
dwbc_explained_variance; FusedPPO(diagnostics=...) and update_diagnostics() refusals, and what diagnostics off leaves as it was."""
import ctypes as C
import functools
import math
import os
import re

import numpy as np
import pytest
import torch

from dwbc_b200 import _lib as L
from dwbc_b200 import synth
from oracle import ppo_oracle as PO
from test_chain_shapes_cpu import make_ac
from test_gpu_chain_shapes import N_ENVS, SEED, T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AMBIGUOUS = 1e-4            # rows whose float64 ratio lies this close to a clip bound may fall on either side in fp32
N_LEG = 12


@functools.lru_cache(maxsize=1)
def old_policy():
    """Rollout means and sigmas of every storage row [T, N, 18] (RS:71-72): means inside tanh's range, sigmas within 20 % of the std the
    test networks start from."""
    mu = torch.from_numpy(synth.normal(SEED, 80, (T, N_ENVS, 18))).clamp(-2.0, 2.0) * 0.45
    std = torch.tensor([0.8, 1.0, 1.0] * 4 + [1.0] * 6)
    sigma = std * torch.exp(torch.from_numpy(synth.uniform(SEED, 81, (T, N_ENVS, 18))) * 0.4 - 0.2)
    return dict(mu=mu.float(), sigma=sigma.float())


def ref_diag(P, st, idx, clip, n_leg=N_LEG, mean_err=0.0):
    """float64 diagnostics of the mini-batch idx (P, st: float64 parameters and storage [T, N, .] with mu / sigma): per channel the mean KL
    of rsl_rl's adaptive schedule between (mu, sigma) and the network's (mean, std), the rows whose ratio lies outside [1 - clip,
    1 + clip] by more than the ambiguity band ('outside_sure'), and the rows inside the band ('ambiguous').  The band is AMBIGUOUS in the
    ratio; with mean_err > 0 (a forward whose means may be off by that much, 'tf32') it also holds every row whose log-ratio lies within
    2 x mean_err x sum_i |a_i - mu_i| / sigma_i^2 of a bound's log: the first-order change such a mean error can make."""
    mb = PO.gather(st, idx)
    f = lambda x: x.flatten(0, 1)[idx]  # noqa: E731
    with torch.no_grad():
        mean = PO.actor_mean(P, mb["obs"], num_prop=76, num_priv=24, num_hist=10)
    std = P["std"].reshape(-1)
    ratio = torch.exp(PO.log_prob2(mean, std, mb["actions"], n_leg) - mb["old_log_prob"])
    omu, osg = f(st["mu"]), f(st["sigma"])
    term = torch.log(std / osg + 1e-5) + (osg ** 2 + (omu - mean) ** 2) / (2.0 * std ** 2) - 0.5
    kl = [float(term[:, :n_leg].sum(1).mean()), float(term[:, n_leg:].sum(1).mean())]
    c = float(np.float32(clip))
    lo, hi = float(np.float32(1 - c)), float(np.float32(1 + c))
    amb = torch.minimum((ratio - lo).abs(), (ratio - hi).abs()) <= AMBIGUOUS
    if mean_err > 0:
        g = (mb["actions"] - mean).abs() / std ** 2
        tol = 2.0 * mean_err * torch.stack([g[:, :n_leg].sum(1), g[:, n_leg:].sum(1)], dim=1)
        lr = torch.log(ratio)
        amb |= torch.minimum((lr - math.log(lo)).abs(), (lr - math.log(hi)).abs()) <= tol
    out = ((ratio < lo) | (ratio > hi)) & ~amb
    return dict(kl=kl, outside_sure=[int(out[:, k].sum()) for k in range(2)], ambiguous=[int(amb[:, k].sum()) for k in range(2)],
                mean=mean, ratio=ratio)


def test_restatement_matches_the_formula_row_by_row():
    """ref_diag on a small network against the KL written out per row and action in plain Python floats, and its clip counts against a
    direct count; the KL of identical policies is sum_i log(1 + 1e-5) exactly."""
    from test_gpu_chain_shapes import params
    P = {k: v.double() for k, v in params("S")[1].items()}
    rng = np.random.default_rng(3)
    R = 6
    st = dict(observations=torch.from_numpy(rng.normal(size=(1, R, 860))), actions=torch.from_numpy(rng.normal(size=(1, R, 18)) * 0.5),
              values=torch.zeros(1, R, 2, dtype=torch.float64), returns=torch.zeros(1, R, 2, dtype=torch.float64),
              advantages=torch.zeros(1, R, 2, dtype=torch.float64), actions_log_prob=torch.from_numpy(rng.normal(-16.0, 1.0, (1, R, 2))),
              mu=torch.from_numpy(rng.uniform(-0.9, 0.9, (1, R, 18))), sigma=torch.from_numpy(rng.uniform(0.5, 1.5, (1, R, 18))))
    idx = torch.tensor([4, 0, 5, 2])
    ref = ref_diag(P, st, idx, 0.2)
    std = P["std"].reshape(-1).tolist()
    mean = ref["mean"]
    for c, cols in enumerate((range(0, 12), range(12, 18))):
        tot = 0.0
        for r, src in enumerate(idx.tolist()):
            for i in cols:
                so, sn, dm = float(st["sigma"][0, src, i]), std[i], float(st["mu"][0, src, i]) - float(mean[r, i])
                tot += math.log(sn / so + 1e-5) + (so * so + dm * dm) / (2 * sn * sn) - 0.5
        assert ref["kl"][c] == pytest.approx(tot / len(idx), rel=1e-12, abs=1e-15)
        ratio = ref["ratio"][:, c].tolist()
        assert ref["outside_sure"][c] + ref["ambiguous"][c] >= sum(not (0.8 <= x <= 1.2) for x in ratio) >= ref["outside_sure"][c]
    same = dict(st, mu=torch.zeros(1, R, 18, dtype=torch.float64), sigma=P["std"].reshape(1, 1, 18).expand(1, R, 18).clone())
    same["mu"][0, idx] = ref["mean"]
    assert ref_diag(P, same, idx, 0.2)["kl"] == pytest.approx([12 * math.log(1 + 1e-5), 6 * math.log(1 + 1e-5)], rel=1e-9)


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(L.LIB_PATH):
        L.build()
    return L.lib()


def test_exports_and_struct_sizes(lib):
    """The two entry points are declared, bound and exported (with the existing ones: test_abi_cpu.py's header-vs-binding check); the
    diag_out layout of the header is the binding's; no struct changed size and the ABI version stays 5."""
    hdr = open(os.path.join(ROOT, "include", "dwbc.h")).read()
    for name in ("dwbc_ppo_minibatch_grad_diag", "dwbc_explained_variance"):
        assert name in L.EXPORTS and getattr(lib, name).argtypes == L._SIGS[name]
        assert re.search(rf"\bint {name}\(", hdr)
    for k in ("KL_LEG", "KL_ARM", "CLIP_LEG", "CLIP_ARM", "GRAD_NORM", "N"):
        assert int(re.search(rf"#define DWBC_DIAG_{k} (\d+)", hdr).group(1)) == getattr(L, "DIAG_" + k)
    assert L.EV_SCRATCH == 2 + 8 * int(re.search(r"#define DWBC_EV_MAX_BLOCKS (\d+)", hdr).group(1))
    sizes = (C.c_int64 * 6)()
    lib.dwbc_struct_sizes(C.byref(sizes))
    assert list(sizes) == [C.sizeof(s) for s in (L.EnvCfg, L.EnvBuffers, L.StepArgs, L.NetCfg, L.PpoHyper, L.Storage)]
    assert L.ABI_VERSION == 5 and int(re.search(r"#define DWBC_ABI_VERSION (\d+)", hdr).group(1)) == 5


def test_host_refusals(lib):
    """NULL arguments, M <= 0 or rows <= 0 are refused before anything is launched."""
    ac = make_ac("S", "cpu")
    cfg, fake = C.addressof(ac.net_cfg), 1 << 40
    st = L.Storage(observations=fake, obs_stride=860, actions=fake, values=fake, returns=fake, advantages=fake, log_prob=fake)
    hp = L.PpoHyper()
    good = [cfg, fake, C.addressof(st), fake, 64, C.addressof(hp), None, fake, fake, fake, fake, fake, fake, None]
    for i in (0, 1, 2, 3, 5, 7, 8, 9, 10, 11, 12):                  # every pointer but sched (optional) and the stream
        args = list(good)
        args[i] = None
        assert lib.dwbc_ppo_minibatch_grad_diag(*args) == -1, i
    for m in (0, -5):
        args = list(good)
        args[4] = m
        assert lib.dwbc_ppo_minibatch_grad_diag(*args) == -1
    for args in ((None, fake, 10, fake, fake), (fake, None, 10, fake, fake), (fake, fake, 10, None, fake), (fake, fake, 10, fake, None),
                 (fake, fake, 0, fake, fake)):
        assert lib.dwbc_explained_variance(*args, None) == -1, args


def test_constructor_and_reader_refusals():
    from dwbc_b200.ppo import FusedPPO
    ac = make_ac("S", "cpu")
    for bad in (1, 0, "yes", None, 1.0):
        with pytest.raises(L.DwbcError, match="diagnostics"):
            FusedPPO(ac, device="cpu", diagnostics=bad)
    with pytest.raises(L.DwbcError, match="diagnostics=True"):
        FusedPPO(ac, device="cpu").update_diagnostics()
    alg = FusedPPO(ac, device="cpu", diagnostics=True)
    with pytest.raises(L.DwbcError, match="no update"):
        alg.update_diagnostics()


def test_off_allocates_nothing_and_keeps_keys():
    """Diagnostics off: no buffer, and the graph key is the parent's tuple (nothing appended); on: the key gains the slots' address.  The
    checkpoint holds no diagnostics either way."""
    from types import SimpleNamespace
    from dwbc_b200.ppo import FusedPPO
    ac = make_ac("S", "cpu")
    off, on = FusedPPO(ac, device="cpu"), FusedPPO(ac, device="cpu", diagnostics=True)
    assert off._diag is None and not hasattr(off, "_diag_ev") and on._diag_ev.shape == (2,)
    fake_storage, ws = SimpleNamespace(num_transitions_per_env=T, num_envs=8, _obs_all=torch.zeros(1)), torch.zeros(1)
    for a in (off, on):
        a.storage, a._ws, a._ws_rows = fake_storage, ws, 8
    k_off, k_on = off.graph_key("ppo"), on.graph_key("ppo")
    assert len(k_off) == 23 and k_on[:-1] == k_off
    assert k_on[-1] == ("diagnostics", on._diag.data_ptr()) and on._diag.shape == (on.num_learning_epochs * on.num_mini_batches, L.DIAG_N)
    assert off.graph_key("dagger") == on.graph_key("dagger")
    assert off._diag is None
    assert set(FusedPPO(ac, device="cpu", diagnostics=True).state_dict()) == set(FusedPPO(ac, device="cpu").state_dict())


def test_diagnostics_plan_stays_on_the_chains_for_every_action_split(lib):
    """The update plan that keeps the heads' means (dwbc_debug_describe_chain what = 5) is accepted wherever the plain update plan (what =
    2) is, for every split of 1..16 leg and 1..16 arm actions on both tensor-core precisions, and differs from it only in the global output
    of the two heads' last ops (FIN_PPO = 2): with a plan the chains refused, the diagnostics would move the update to the layer-wise
    path (other rounding, another speed)."""
    from dwbc_b200.actor_critic import FlatActorCritic
    from test_chain_shapes_cpu import describe
    on_chains = 0
    for nl in range(1, 17):
        for na in range(1, 17):
            ac = FlatActorCritic(device="cpu", num_priv=24, num_hist=10, num_prop=76, num_leg_actions=nl, num_arm_actions=na)
            for precision in (2, 1):
                plain, kept = describe(ac, 4224, 2, 0, precision), describe(ac, 4224, 5, 0, precision)
                assert (plain == -2) == (kept == -2), (nl, na, precision)
                if plain == -2:
                    continue
                on_chains += 1
                assert plain[0] == kept[0] and len(plain[1]) == len(kept[1])
                for (l0, ops0), (l1, ops1) in zip(plain[1], kept[1]):
                    assert l0 == l1 and len(ops0) == len(ops1)
                    for o0, o1 in zip(ops0, ops1):
                        assert o1 == (dict(o0, y=1) if o0["fin"] == 2 else o0), (nl, na, o0, o1)
    assert on_chains >= 2 * 16 * 16 - 8, on_chains                  # (the splits the chains take: all but a few)
