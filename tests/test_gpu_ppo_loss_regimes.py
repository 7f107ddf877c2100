"""The PPO loss hooks (ppo_loss_kernel on 'fp32'; c2_fin_ppo / c2_fin_value / c2_fin_reg / c2_fin_torque of the fused chains on 'tf32x3'
and 'tf32') and clip + Adam (clip_adam_kernel) against float64, one branch at a time and away from the shipped hyper-parameters.

Mini-batches come from the builder of test_ppo_loss_regimes_cpu.py: in a single-regime batch every (row, channel) sits in one of the six
surrogate regimes and one of the five value regimes with a margin (>= 6 x the 8e-3 forward bound of 'tf32') that rounding cannot cross;
the mixed batch holds them all.  Surrogate gradients reach only the actor's tensors and std, value gradients only the critic's, so each
regime is seen in its own tensors, and in the regimes without a surrogate (value) gradient those tensors must come back zero.  The four
hyper-parameter sets (SETS) move every coefficient of the loss off the shipped point: clip, value and entropy coefficients, the unclipped
value loss, a fractional mixing ratio rho and regulariser coefficient, and fixed-gain torque supervision.

Tolerances: those of test_gpu_chain_shapes.py (CHAIN_TOL, GRAD_ABS), with two exceptions measured here (H100 SXM, 700 W), each bound 2 x
the largest error seen:
  * the 'tf32x3' floor of the per-tensor gradient bound, 4e-7 instead of 1e-7.  Returns a short way from the values (|v - R| <= 0.6 +
    clip) make the critic heads' bias gradients small sums of row terms of both signs (norm 2.5e-3 .. 2.8e-3): 3xTF32 is off float64 by
    1.6e-7 (H0) and 1.8e-7 (H2, value coefficient 2) there, while 'fp32' stays inside 1e-7.  A branch that leaks or drops a gradient is
    off by the size of whole row terms, orders of magnitude above either floor;
  * the loss bound of a one-row batch, 2 x CHAIN_TOL's: its loss is one row's, not a mean, so the TF32 forward error of that row enters
    undiluted (value loss of H2's row: 2.06e-3 relative against the 2e-3 of 'tf32').
clip + Adam: ADAM_ULPS."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import ppo_oracle as PO
from test_chain_shapes_cpu import make_ac
from test_gpu_chain_shapes import COUNTER, GRAD_ABS, N_ENVS, T, TOL, grad_errors, grad_rows, minibatch_index, params
from test_ppo_loss_regimes_cpu import BATCHES, SETS, arm_inputs, build, hyper, oracle_hp

pytestmark = pytest.mark.gpu
PRECISIONS = ["fp32", "tf32x3", "tf32"]
LOSSES = ("surrogate", "value", "priv_reg", "entropy", "arm_torques")
GRAD_FLOOR = dict(GRAD_ABS, tf32x3=4e-7)
_ref = {}                                                 # float64 results per (set, batch, rows), shared by the three paths


def batch_rows(batch):
    """1 row only in the mixed batch (one row holds one regime per channel); 129 rows and sms tiles + 77 rows in every batch."""
    return grad_rows() if batch == "mixed" else grad_rows()[1:]


def ref_grad(name, batch, rows):
    key = (name, batch, rows)
    if key not in _ref:
        st = {k: v.double() for k, v in build(name, batch)[0].items()}
        P = {k: v.double().requires_grad_(True) for k, v in params("S")[1].items()}
        loss, info = PO.minibatch_loss(P, PO.gather(st, minibatch_index()[:rows]), oracle_hp(name), COUNTER)
        loss.backward()
        g = {n: (p.grad if p.grad is not None else torch.zeros_like(p)).detach() for n, p in P.items()}
        _ref[key] = (g, [float(info.get(k, 0.0)) for k in LOSSES])
    return _ref[key]


def make_alg(name, precision, **over):
    from dwbc_b200.ppo import FusedPPO
    ac = make_ac("S", "cuda:0")
    ac.load_state_dict(params("S")[1])
    hp = dict(hyper(name), num_mini_batches=1, num_learning_epochs=1, precision=precision)
    hp.update(over)
    alg = FusedPPO(ac, device="cuda:0", **hp)
    alg.init_storage(N_ENVS, T, [860], [None], [18])
    if alg.torque_supervision:
        alg.set_arm_default_coeffs(*arm_inputs()[1])
    alg.counter = COUNTER
    return alg


def load(alg, st):
    s = alg.storage
    for k, v in st.items():
        (s._obs_all[:T] if k == "observations" else getattr(s, k)).copy_(v.cuda())


def run(alg, rows, hp=None, sched=None):
    """dwbc_ppo_minibatch_grad (or, with the device schedule `sched`, dwbc_ppo_minibatch_grad_sched) on the first `rows` rows of
    minibatch_index(): per-tensor gradients and the five loss means."""
    from dwbc_b200 import _lib as L
    ac, s = alg.actor_critic, alg.storage
    idx = minibatch_index()[:rows].cuda()
    h = alg._fill_hp() if hp is None else hp
    alg._set_precision()
    alg._losses.zero_()
    head = (C.addressof(ac.net_cfg), L.ptr(ac.flat), s.c_struct_ptr(), L.ptr(idx), rows, C.addressof(h))
    tail = (L.ptr(alg.grad), L.ptr(alg._losses), L.ptr(alg._workspace(rows)), L.stream_ptr())
    if sched is None:
        L.check(L.lib().dwbc_ppo_minibatch_grad(*head, *tail), "dwbc_ppo_minibatch_grad")
    else:
        L.check(L.lib().dwbc_ppo_minibatch_grad_sched(*head, L.ptr(sched), *tail), "dwbc_ppo_minibatch_grad_sched")
    return {k: v.clone() for k, v in ac.unflat(alg.grad).items()}, alg._losses.clone()


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", sorted(SETS))
def test_minibatch_grad_matches_float64_in_every_regime(name, precision):
    """Every parameter tensor's gradient (a tensor whose float64 gradient is zero within GRAD_ABS), the std gradient on its own (the only
    one that carries the entropy term) and the five loss means, in six single-regime batches and one mixed batch.  Every batch is
    checked before the test fails, and the failures are listed together."""
    tol, floor = TOL[precision], GRAD_FLOOR[precision]
    alg = make_alg(name, precision)
    worst, fails = ("", 0.0, 0.0, 0.0), []
    for batch in BATCHES:
        load(alg, build(name, batch)[0])
        for rows in batch_rows(batch):
            got, losses = run(alg, rows)
            ref, ref_losses = ref_grad(name, batch, rows)
            try:
                w = grad_errors(got, ref, tol["grad"], floor)
            except AssertionError as e:
                fails.append((batch, rows, "gradient", str(e)))
                continue
            gs, rs = got["std"].double().cpu(), ref["std"]
            dstd = float((gs - rs).abs().max())
            if dstd > tol["grad"] * float(rs.abs().max()) + floor:
                fails.append((batch, rows, "std", dstd, gs.tolist(), rs.tolist()))
            lerr = max(abs(float(losses[i]) - ref_losses[i]) / (abs(ref_losses[i]) + 1e-3) for i in range(len(LOSSES)))
            if lerr > tol["loss"] * (2 if rows == 1 else 1):
                fails.append((batch, rows, "losses", lerr, losses.tolist(), ref_losses))
            if w[1] > worst[1]:
                worst = (f"{batch} rows={rows} {w[0]}", w[1], worst[2], worst[3])
            worst = worst[:2] + (max(worst[2], w[2]), max(worst[3], lerr))
    print(f"[{name} {precision}] worst ||dg||/||g|| vs float64 {worst[1]:.3g} ({worst[0]}), largest ||dg|| {worst[2]:.3g}, "
          f"losses rel {worst[3]:.3g}")
    assert not fails, fails


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", ["H1", "H3"])
def test_device_schedule_entry_is_bitwise_the_host_entry(name, precision):
    """dwbc_ppo_minibatch_grad_sched with (c_reg, rho, ts_w) in device memory and NaN in the three host fields computes bit for bit what
    dwbc_ppo_minibatch_grad computes with the values in the host fields -- at fractional rho and c_reg, which the test above holds to
    float64.  This is the entry the captured update replays."""
    from dwbc_b200 import _lib as L
    alg = make_alg(name, precision)
    load(alg, build(name, "mixed")[0])
    rows = grad_rows()[-1]
    h = alg._fill_hp()
    assert 0 < h.mixing_ratio < 1 and 0 < h.priv_reg_coef < 1 and (h.torque_supervision_weight > 0) == (name == "H3")
    g0, l0 = run(alg, rows, h)
    hd = L.PpoHyper()
    C.memmove(C.addressof(hd), C.addressof(h), C.sizeof(hd))
    sched = torch.tensor([h.priv_reg_coef, h.mixing_ratio, h.torque_supervision_weight], dtype=torch.float32, device="cuda:0")
    hd.priv_reg_coef = hd.mixing_ratio = hd.torque_supervision_weight = float("nan")
    g1, l1 = run(alg, rows, hd, sched)
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
    assert torch.equal(l0, l1)


# ---- clip + Adam (dwbc_clip_adam_step / _table) against float64 ------------------------------------------------------------------------
# Bound on |x - x_ref| in fp32 epsilons (2^-23) of the scale of each quantity: the gradient left behind and v relative to their own size,
# m relative to |beta1 m0| + |(1 - beta1) g|, the parameters relative to |p0| + |Adam update|, the norm relative.  fp32 arithmetic without
# FMA contraction, one rounding per operation.  Worst measured over ADAM_CASES (H100 SXM, 700 W; printed): grad 1.06, m 1.77, v 2.95, param
# 3.58, norm 0.4; the bounds are about 2 x that.
ADAM_ULPS = dict(grad=2.5, m=4.0, v=6.0, param=8.0, norm=1.0)
EPS32 = 2.0 ** -23
# name: (buffer length, first, count, grad_scale, Adam step, total norm above max_grad_norm)
ADAM_CASES = {
    "below_step1": (4099, 0, 4099, 1.0, 1, False),
    "above_step2": (4099, 0, 4099, 1.0, 2, True),
    "scale_half_step5000": (65549, 0, 65549, 0.5, 5000, True),
    "subrange_step2": (80000, 333, 70001, 1.0, 2, True),             # odd first, count not a multiple of 256; the rest untouched
    "looping_above_step5000": (1000003, 0, 1000003, 0.5, 5000, True),  # > DWBC_NORM_SCRATCH x 1024: the blocks loop
    "looping_below_step1": (1000003, 0, 1000003, 1.0, 1, False),
}


def adam_inputs(n, first, count, step, seed):
    """fp32 parameters, gradients spread over eight decades (some below Adam's eps), and the moments of step - 1 steps (zero at step 1);
    gradient entries outside [first, first + count) are NaN."""
    gen = torch.Generator().manual_seed(seed)
    p = torch.randn(n, generator=gen) * 0.1
    g = torch.randn(n, generator=gen) * torch.pow(10.0, -torch.randint(1, 9, (n,), generator=gen).float())
    m = torch.zeros(n) if step == 1 else torch.randn(n, generator=gen) * 1e-3
    v = torch.zeros(n) if step == 1 else torch.rand(n, generator=gen) * 1e-5
    g[:first] = float("nan")
    g[first + count:] = float("nan")
    return p, g, m, v


def ref_clip_adam(p, g, m, v, hp, step):
    """PO.clip_grad_norm + PO.Adam in float64 on the fp32 inputs, with the fp32 hyper-parameters the kernel reads."""
    f = lambda x: float(np.float32(x))  # noqa: E731
    P, G = {"x": p.double()}, {"x": g.double() * f(hp.grad_scale)}
    total = float(PO.clip_grad_norm(G, ["x"], f(hp.max_grad_norm)))
    opt = PO.Adam(["x"], f(hp.lr), betas=(f(hp.beta1), f(hp.beta2)), eps=f(hp.adam_eps))
    opt.state["x"] = dict(step=step - 1, m=m.double(), v=v.double())
    upd = P["x"].clone()
    opt.step(P, G)
    return dict(param=P["x"], grad=G["x"], m=opt.state["x"]["m"], v=opt.state["x"]["v"], norm=total, update=P["x"] - upd)


def clip_adam(p, g, m, v, first, count, hp, step, table=None):
    from dwbc_b200 import _lib as L
    t = [x.cuda() for x in (p, g, m, v)]
    scratch = torch.zeros(L.NORM_SCRATCH, dtype=torch.float64, device="cuda:0")
    norm = torch.zeros(1, device="cuda:0")
    ptrs = [L.ptr(x) for x in t]
    if table is None:
        L.check(L.lib().dwbc_clip_adam_step(*ptrs, first, count, C.addressof(hp), step, L.ptr(scratch), L.ptr(norm), L.stream_ptr()),
                "dwbc_clip_adam_step")
    else:
        L.check(L.lib().dwbc_clip_adam_step_table(*ptrs, first, count, C.addressof(hp), step, L.ptr(table), L.ptr(scratch), L.ptr(norm),
                                                  L.stream_ptr()), "dwbc_clip_adam_step_table")
    return dict(zip(("param", "grad", "m", "v"), (x.cpu() for x in t)), norm=float(norm))


def bits(x):
    return x.view(torch.int32)


@pytest.mark.parametrize("case", sorted(ADAM_CASES))
def test_clip_adam_matches_float64(case):
    """Parameters, both moments, the clipped gradient left behind and the reported norm against float64; below the threshold the
    coefficient is exactly 1 and the gradient left behind is g * grad_scale bit for bit; outside [first, first + count) nothing changes;
    the table entry with the rows of dwbc_adam_bias_correction is bitwise the host entry."""
    from dwbc_b200 import _lib as L
    n, first, count, scale, step, above = ADAM_CASES[case]
    p, g, m, v = adam_inputs(n, first, count, step, seed=len(case))
    sl = slice(first, first + count)
    total = float((g[sl].double() * scale).norm())
    hp = L.PpoHyper(max_grad_norm=total * (0.5 if above else 1.5), lr=2e-4, beta1=0.9, beta2=0.999, adam_eps=1e-8, grad_scale=scale)
    got = clip_adam(p, g, m, v, first, count, hp, step)
    ref = ref_clip_adam(p[sl], g[sl], m[sl], v[sl], hp, step)
    for k, x0 in (("param", p), ("grad", g), ("m", m), ("v", v)):              # the rest of the buffers: bitwise untouched
        assert torch.equal(bits(got[k][:first]), bits(x0[:first])) and torch.equal(bits(got[k][first + count:]), bits(x0[first + count:])), k
    if not above:
        assert torch.equal(got["grad"][sl], g[sl] * scale)
    b1 = float(np.float32(hp.beta1))
    scales = dict(grad=ref["grad"].abs(), m=b1 * m[sl].double().abs() + (1 - b1) * ref["grad"].abs(), v=ref["v"].abs(),
                  param=p[sl].double().abs() + ref["update"].abs())
    ulps = {k: float(((got[k][sl].double() - ref[k]).abs() / (EPS32 * s.clamp_min(1e-30))).max()) for k, s in scales.items()}
    ulps["norm"] = abs(got["norm"] - ref["norm"]) / (EPS32 * ref["norm"])
    print(f"[{case}] error vs float64 in fp32 epsilons of each quantity's scale: " + ", ".join(f"{k} {e:.3g}" for k, e in ulps.items()))
    for k, e in ulps.items():
        assert e <= ADAM_ULPS[k], (k, e)
    table = torch.from_numpy(L.adam_bias_correction(hp, 1, step)).cuda()
    got_t = clip_adam(p, g, m, v, first, count, hp, step, table=table)
    for k in ("param", "grad", "m", "v"):
        assert torch.equal(bits(got_t[k]), bits(got[k])), k
    assert got_t["norm"] == got["norm"]


# ---- update() end to end ----------------------------------------------------------------------------------------------------------------
# max_grad_norm of each set: between the float64 per-step norms of its 8 steps, so that some steps clip and some do not (asserted below,
# with no norm within 2 % of the threshold)
UPDATE_MAX_GRAD_NORM = {"H1": 0.346, "H2": 0.315}
_upd = {}


def ref_update(name):
    """PO.ppo_update in float64, 2 epochs x 4 mini-batches on the mixed regime storage: the 7-tuple of update(), the mean entropy, the
    per-step norms, the clipped gradient of step 1 and the parameters after step 1 and after the last step."""
    if name not in _upd:
        st = {k: v.double() for k, v in build(name, "mixed")[0].items()}
        P = {k: v.double() for k, v in params("S")[1].items()}
        hp = dict(oracle_hp(name), num_mini_batches=4, num_learning_epochs=2, max_grad_norm=UPDATE_MAX_GRAD_NORM[name])
        snap = {}

        def record(k, Pn, Gd, when):
            if k == 0 and when == "pre_step":
                snap["grad1"] = {n: (Gd[n] if Gd[n] is not None else torch.zeros_like(Pn[n])).clone() for n in Pn}
            if k == 0 and when == "post_step":
                snap["param1"] = {n: Pn[n].detach().clone() for n in Pn}

        logs = PO.ppo_update(P, PO.Adam(list(P), hp["learning_rate"]), st, minibatch_index(), hp, COUNTER, record)
        mean = lambda k: float(np.mean([float(x[k]) for x in logs]))  # noqa: E731
        res = (mean("value"), mean("surrogate"), 0.0, logs[0]["mixing_ratio"], 0, mean("priv_reg"), logs[0]["priv_reg_coef"])
        _upd[name] = (res, mean("entropy"), [float(x["grad_norm"]) for x in logs], snap, P)
    return _upd[name]


@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
@pytest.mark.parametrize("name", ["H1", "H2"])
def test_update_matches_float64_with_clipped_and_unclipped_steps(name, precision):
    """update() (2 epochs x 4 mini-batches) against PO.ppo_update in float64 with the bounds of
    test_gpu_ppo.py::test_ppo_update_matches_reference_golden: losses, mixing ratio, regulariser coefficient, last_entropy, the clipped
    gradient of step 1, the parameters after step 1 and after the last step."""
    ref, ref_ent, norms, snap, p_last = ref_update(name)
    thr = UPDATE_MAX_GRAD_NORM[name]
    assert any(x > thr for x in norms) and any(x < thr for x in norms) and all(abs(x / thr - 1) > 0.02 for x in norms), norms
    alg = make_alg(name, precision, num_mini_batches=4, num_learning_epochs=2, max_grad_norm=thr)
    load(alg, build(name, "mixed")[0])
    ac = alg.actor_critic
    got = {}

    def on_step(k, when):
        if k == 0 and when == "step":
            got["grad1"], got["param1"] = ac.unflat(alg.grad.clone()), ac.unflat(ac.flat.clone())

    res = alg.update(indices=minibatch_index().cuda(), on_step=on_step)
    print(f"[{name} {precision}] float64 norms {[round(x, 4) for x in norms]} (max_grad_norm {thr}); losses "
          f"{res[0] - ref[0]:+.3g} {res[1] - ref[1]:+.3g} {res[5] - ref[5]:+.3g}, entropy {alg.last_entropy - ref_ent:+.3g}")
    assert abs(res[0] - ref[0]) < 2e-5 * max(1, abs(ref[0])) and abs(res[1] - ref[1]) < 2e-5 and abs(res[5] - ref[5]) < 2e-5
    assert abs(res[3] - ref[3]) < 1e-7 and abs(res[6] - ref[6]) < 1e-7 and res[2] == 0.0 and res[4] == 0
    assert abs(alg.last_entropy - ref_ent) < 2e-5
    p_end = ac.unflat(ac.flat)
    for n, _ in ac.manifest:
        np.testing.assert_allclose(got["grad1"][n].cpu().numpy(), snap["grad1"][n].numpy(), rtol=1e-3, atol=2e-6, err_msg="grad1 " + n)
        np.testing.assert_allclose(got["param1"][n].cpu().numpy(), snap["param1"][n].numpy(), rtol=0, atol=2e-5, err_msg="param1 " + n)
        np.testing.assert_allclose(p_end[n].cpu().numpy(), p_last[n].numpy(), rtol=0, atol=2e-5, err_msg="param8 " + n)
