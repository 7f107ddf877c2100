"""GPU: the PPO update diagnostics (FusedPPO(diagnostics=True), dwbc_ppo_minibatch_grad_diag, dwbc_explained_variance).

* Per mini-batch against a float64 restatement (ref_diag, built from oracle/ppo_oracle.py) on the same gathered rows and the same
  parameters: approximate KL per channel, clip fractions, and explained variance, on 'fp32' (layer-wise), 'tf32x3' and 'tf32' (fused
  chains) at the shipped network in the regime batches of test_gpu_ppo_loss_regimes.py (sets H1, H2 and, with torque supervision, H3),
  on the stock 512/256/128 trunks (layer-wise on every precision) and on sweep network C.  Mini-batches of 185 rows (37 envs x 5 steps)
  and 128 x SMs + 77 rows (ragged two-tile and one-tile work items).  The same call also returns bit for bit the gradient and losses of
  dwbc_ppo_minibatch_grad.
* Diagnostics on change nothing else: two update()s on and off leave parameters, both Adam moments, losses, the returned tuples and
  the storage bitwise equal.
* Captured updates (cuda_graphs=True) and on_step give the eager diagnostics bit for bit; the same run twice gives the same bits.

Tolerances: KL rel KL_RTOL; clip fractions: every row whose float64 ratio lies more than 1e-4 from both clip bounds is classified as in
float64 (the kernel's count lies between the unambiguous count and that plus the ambiguous rows) on 'fp32' and 'tf32x3'; on 'tf32' the
band also covers what the TF32 forward's mean error (MEAN_ERR) can move the ratio -- on unshaped data one 14 + 4 row in 40 000 sat
outside the 1e-4 band and flipped; explained variance rel 1e-4.
The 'tf32' KL bound is 2 x the largest error printed by test_minibatch_diagnostics_match_float64 (NVIDIA H100 80GB HBM3, 700 W); 'fp32'
and 'tf32x3' stayed below 2.4e-7 there."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from dwbc_b200 import _lib as L
from dwbc_b200 import synth
from dwbc_b200.actor_critic import FlatActorCritic
from oracle import ppo_oracle as PO
from test_chain_shapes_cpu import dims as sweep_dims, make_ac
from test_gpu_chain_shapes import COUNTER, N_ENVS, SEED, T, minibatch_index, sms, storage_inputs
from test_oracle_golden import ppo_hp
from test_ppo_diagnostics_cpu import AMBIGUOUS, old_policy, ref_diag
from test_ppo_loss_regimes_cpu import arm_inputs, build, hyper

pytestmark = pytest.mark.gpu
PRECISIONS = ["fp32", "tf32x3", "tf32"]
KL_RTOL = dict(fp32=1e-4, tf32x3=1e-4, tf32=3e-4)    # tf32: 2 x the 1.47e-4 measured (shipped network, H1..H3; C: 1.27e-4, stock: 3.8e-5)
# Error of a mean the forward computes, the clip classification's ambiguity (ref_diag's mean_err): 'tf32' truncates operands to 10 bits, and
# its means are off float64 by up to the 8e-3 forward bound of the loss-regime tests (test_ppo_loss_regimes_cpu.py); 'fp32' and 'tf32x3'
# are fp32-grade and keep the 1e-4 band of the ratio.
MEAN_ERR = dict(fp32=0.0, tf32x3=0.0, tf32=8e-3)
STOCK = dict(actor_dims=(512, 256, 128), critic_dims=(512, 256, 128))


def rows_list():
    return (185, 128 * sms() + 77)


def net_params(d):
    manifest = PO.param_manifest(**d)
    vals = synth.policy_params(manifest, SEED)
    std = torch.tensor([[0.8, 1.0, 1.0] * 4 + [1.0] * 6])[:, :d.get("n_leg", 12) + d.get("n_arm", 6)]
    return {n: (std.clone() if v is None else torch.from_numpy(v).clone()) for (n, _), v in zip(manifest, vals)}


def make_alg(net, precision, hp, **over):
    """FusedPPO with diagnostics on over network `net` ('S', a sweep network, or 'stock'), storage filled from build()/storage_inputs."""
    from dwbc_b200.ppo import FusedPPO
    if net == "stock":
        d = dict(sweep_dims("S"), **STOCK)
        ac = FlatActorCritic(device="cuda:0", num_priv=24, num_hist=10, num_prop=76, actor_hidden_dims=STOCK["actor_dims"],
                             critic_hidden_dims=STOCK["critic_dims"])
    else:
        d = sweep_dims(net)
        ac = make_ac(net, "cuda:0")
    P = net_params(d)
    ac.load_state_dict(P)
    alg = FusedPPO(ac, device="cuda:0", **dict(hp, precision=precision, diagnostics=True, **over))
    alg.init_storage(N_ENVS, T, [860], [None], [18])
    if alg.torque_supervision:
        alg.set_arm_default_coeffs(*arm_inputs()[1])
    alg.counter = COUNTER
    return alg, P, d


def load(alg, st):
    s = alg.storage
    for k, v in st.items():
        (s._obs_all[:T] if k == "observations" else getattr(s, k)).copy_(v.cuda())


def run_minibatch(alg, rows, diag_entry):
    ac, s = alg.actor_critic, alg.storage
    idx = minibatch_index()[:rows].cuda()
    h = alg._fill_hp()
    alg._set_precision()
    alg._losses.zero_()
    ws = alg._workspace(rows)
    head = (C.addressof(ac.net_cfg), L.ptr(ac.flat), s.c_struct_ptr(), L.ptr(idx), rows, C.addressof(h))
    diag = torch.full((L.DIAG_N,), float("nan"), device="cuda:0")
    if diag_entry:
        L.check(L.lib().dwbc_ppo_minibatch_grad_diag(*head, None, L.ptr(s.mu), L.ptr(s.sigma), L.ptr(alg.grad), L.ptr(alg._losses),
                                                     L.ptr(diag), L.ptr(ws), L.stream_ptr()), "dwbc_ppo_minibatch_grad_diag")
    else:
        L.check(L.lib().dwbc_ppo_minibatch_grad(*head, L.ptr(alg.grad), L.ptr(alg._losses), L.ptr(ws), L.stream_ptr()), "dwbc_ppo_minibatch_grad")
    return alg.grad.clone(), alg._losses.clone(), diag.double().cpu()


def explained_variance(values, returns):
    out = torch.full((2,), -7.0, device="cuda:0")
    scratch = torch.zeros(L.EV_SCRATCH, dtype=torch.float64, device="cuda:0")
    v, r = values.reshape(-1, 2).contiguous(), returns.reshape(-1, 2).contiguous()
    L.check(L.lib().dwbc_explained_variance(L.ptr(v), L.ptr(r), v.shape[0], L.ptr(scratch), L.ptr(out), L.stream_ptr()), "dwbc_explained_variance")
    assert (int(scratch[0].view(torch.int64)) & 0xffffffff) == 0         # the counter is back at zero
    return out.double().cpu()


CASES = [("S", name, p) for name in ("H1", "H2", "H3") for p in PRECISIONS] + [("stock", None, p) for p in PRECISIONS] + \
        [("C", None, p) for p in ("tf32x3", "tf32")]


@pytest.mark.parametrize("net,name,precision", CASES)
def test_minibatch_diagnostics_match_float64(net, name, precision):
    hp = dict(hyper(name) if name else ppo_hp(), num_mini_batches=1, num_learning_epochs=1)
    alg, P, d = make_alg(net, precision, hp)
    st = dict(build(name, "mixed")[0] if name else storage_inputs())
    st.update(old_policy())
    load(alg, st)
    P64 = {k: v.double() for k, v in P.items()}
    st64 = {k: v.double() for k, v in st.items()}
    worst = 0.0
    for rows in rows_list():
        g0, l0, _ = run_minibatch(alg, rows, False)
        g1, l1, diag = run_minibatch(alg, rows, True)
        assert torch.equal(g0, g1) and torch.equal(l0, l1), "the _diag entry must compute dwbc_ppo_minibatch_grad's bits"
        assert math.isnan(float(diag[L.DIAG_GRAD_NORM]))                    # not written by the mini-batch call
        ref = ref_diag(P64, st64, minibatch_index()[:rows], alg._hp.clip_param, mean_err=MEAN_ERR[precision])
        for c, ch in enumerate(("leg", "arm")):
            kl, kr = float(diag[L.DIAG_KL_LEG + c]), ref["kl"][c]
            err = abs(kl - kr) / abs(kr)
            worst = max(worst, err)
            assert err <= KL_RTOL[precision], (rows, ch, kl, kr, err)
            n = float(diag[L.DIAG_CLIP_LEG + c]) * rows
            lo, amb = ref["outside_sure"][c], ref["ambiguous"][c]
            assert lo - 1e-3 <= n <= lo + amb + 1e-3, (rows, ch, n, lo, amb)
    print(f"[{net} {name} {precision}] worst KL rel err vs float64 {worst:.3g} (ambiguity band {AMBIGUOUS})")
    if name == "H1":                                                        # regime batch: every surrogate regime is present
        assert 0 < ref["outside_sure"][0] < rows and 0 < ref["outside_sure"][1] < rows


def test_explained_variance_matches_float64():
    st = build("H1", "mixed")[0]
    for v, r in ((st["values"], st["returns"]), (st["values"][:, :37], st["returns"][:, :37] + 40.0)):
        got = explained_variance(v.cuda(), r.cuda())
        v64, r64 = v.reshape(-1, 2).double(), r.reshape(-1, 2).double()
        ref = 1 - (r64 - v64).var(0, unbiased=False) / r64.var(0, unbiased=False)
        assert torch.allclose(got, ref, rtol=1e-4, atol=0), (got, ref)
    # a constant return channel (and a single row) has no variance to explain: NaN
    v, r = st["values"][:, :50].clone(), st["returns"][:, :50].clone()
    r[..., 1] = 3.25
    got = explained_variance(v.cuda(), r.cuda())
    assert not math.isnan(float(got[0])) and math.isnan(float(got[1]))
    assert torch.isnan(explained_variance(v[:1, :1].cuda(), r[:1, :1].cuda())).all()


# ---- whole update()s ---------------------------------------------------------------------------------------------------------------------
def train(precision, diagnostics, graphs=False, on_step=False, iters=2):
    """Two update()s of 2 epochs x 4 mini-batches on fixed storage and permutations, with the mixing and priv-reg schedules moving.  With
    on_step, the pre-clip norm FusedPPO._grad_norm holds after every Adam step is recorded (per update, in step order)."""
    from dwbc_b200.ppo import FusedPPO
    ac = make_ac("S", "cuda:0")
    ac.load_state_dict(net_params(sweep_dims("S")))
    hp = dict(ppo_hp(), num_mini_batches=4, num_learning_epochs=2, mixing_schedule=[1.0, COUNTER, 4],
              priv_reg_coef_schedual=[0, 1, COUNTER, 4])
    alg = FusedPPO(ac, device="cuda:0", precision=precision, cuda_graphs=graphs, diagnostics=diagnostics, **hp)
    alg.init_storage(N_ENVS, T, [860], [None], [18])
    alg.counter = COUNTER
    st = dict(build("H1", "mixed")[0], **old_policy())
    perm = torch.from_numpy(np.argsort(synth.uniform(SEED, 61, (iters, N_ENVS * T)), axis=1)).long().cuda()
    rets, diags, norms = [], [], []

    def record(k, what):
        if what == "step":
            norms[-1].append(float(alg._grad_norm))
    for it in range(iters):
        load(alg, st)
        norms.append([])
        rets.append(alg.update(indices=perm[it], on_step=record if on_step else None))
        if diagnostics:
            diags.append(alg.update_diagnostics())
    s = alg.storage
    state = dict(flat=ac.flat.clone(), m=alg.optimizer.m.clone(), v=alg.optimizer.v.clone(), losses=alg._losses.clone(),
                 **{f"storage.{k}": t.clone() for k, t in vars(s).items() if isinstance(t, torch.Tensor)})
    return rets, diags, state, norms


def assert_same_state(a, b):
    assert a.keys() == b.keys(), set(a) ^ set(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("precision", PRECISIONS)
def test_diagnostics_change_nothing_else(precision):
    """Also: slot k's grad_norm is, bit for bit, the pre-clip norm the diagnostics-off run's Adam step k reports in FusedPPO._grad_norm."""
    r0, _, s0, norms = train(precision, False, on_step=True)
    r1, d1, s1, _ = train(precision, True)
    assert r0 == r1
    assert_same_state(s0, s1)
    assert [d["per_minibatch"]["grad_norm"] for d in d1] == norms and len(norms[0]) == 8 and norms[0] != norms[1]
    d = d1[-1]
    assert all(x > 0 for x in d["per_minibatch"]["grad_norm"])
    assert d["grad_norm_max"] == max(d["per_minibatch"]["grad_norm"])
    assert d["approx_kl"] == pytest.approx(d["approx_kl_leg"] + d["approx_kl_arm"], rel=1e-12)
    print(f"[{precision}] last update: " + ", ".join(f"{k} {v:.4g}" for k, v in d.items() if k != "per_minibatch"))


@pytest.mark.parametrize("precision", PRECISIONS)
def test_graphs_and_on_step_give_the_eager_diagnostics(precision):
    r0, d0, s0, _ = train(precision, True)
    r1, d1, s1, _ = train(precision, True, graphs=True)
    r2, d2, s2, _ = train(precision, True, on_step=True)
    assert r0 == r1 == r2 and d0 == d1 == d2
    assert_same_state(s0, s1)
    assert d0[0]["per_minibatch"] != d0[1]["per_minibatch"]            # the second iteration measured its own update


def test_same_run_twice_is_bitwise():
    _, d0, _, _ = train("tf32x3", True)
    _, d1, _, _ = train("tf32x3", True)
    assert d0 == d1


@pytest.mark.parametrize("precision", ["tf32x3", "tf32"])
@pytest.mark.parametrize("n_leg,n_arm", [(6, 8), (14, 4)])
def test_other_action_splits_stay_on_the_chains(n_leg, n_arm, precision):
    """Splits whose arm head starts at a column that is not a multiple of 4 while its width is (6 + 8, 14 + 4): the update with the
    diagnostics stays on the fused chains, returns dwbc_ppo_minibatch_grad's gradient and losses bit for bit, and its KL matches float64."""
    from dwbc_b200.ppo import FusedPPO
    from test_chain_shapes_cpu import describe
    na = n_leg + n_arm
    d = dict(sweep_dims("S"), n_leg=n_leg, n_arm=n_arm)
    ac = FlatActorCritic(device="cuda:0", num_priv=24, num_hist=10, num_prop=76, num_leg_actions=n_leg, num_arm_actions=n_arm)
    P = net_params(d)
    ac.load_state_dict(P)
    assert describe(ac, 4224, 5, 0, 2) != -2 and describe(ac, 4224, 5, 0, 1) != -2
    alg = FusedPPO(ac, device="cuda:0", precision=precision, diagnostics=True, **dict(ppo_hp(), num_mini_batches=1, num_learning_epochs=1,
                                                                                      min_policy_std=None))
    alg.init_storage(N_ENVS, T, [860], [None], [na])
    alg.counter = COUNTER
    st = {k: (v[..., :na] if k == "actions" else v) for k, v in storage_inputs().items()}
    st.update({k: v[..., :na] for k, v in old_policy().items()})
    load(alg, st)
    P64, st64 = {k: v.double() for k, v in P.items()}, {k: v.double() for k, v in st.items()}
    for rows in rows_list():
        g0, l0, _ = run_minibatch(alg, rows, False)
        g1, l1, diag = run_minibatch(alg, rows, True)
        assert torch.equal(g0, g1) and torch.equal(l0, l1)
        ref = ref_diag(P64, st64, minibatch_index()[:rows], alg._hp.clip_param, n_leg, MEAN_ERR[precision])
        for c in range(2):
            assert abs(float(diag[L.DIAG_KL_LEG + c]) - ref["kl"][c]) <= KL_RTOL[precision] * abs(ref["kl"][c]), (rows, c)
            n = float(diag[L.DIAG_CLIP_LEG + c]) * rows
            assert ref["outside_sure"][c] - 1e-3 <= n <= ref["outside_sure"][c] + ref["ambiguous"][c] + 1e-3
