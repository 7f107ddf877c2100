"""The hidden-layer activations other than ELU (selu, relu, lrelu, tanh, sigmoid) in every policy kernel, against float64 autograd of the
oracle with that activation (test_activations_cpu.oracle_activation) on CPU: the fused chains (networks S and C of the shape sweep), the
layer-wise paths (fp32 CUDA cores; the stock 512/256/128 trunks on the tensor-core precisions), the fused history encoder and the DAgger
backward; and update() end to end through FusedActorCritic / FusedPPO against the oracle's ppo_update.

Tolerances are those of test_gpu_chain_shapes.py for every activation, except 'tf32' with relu, lrelu and selu (TF32_KINK below).  For those
three the derivative jumps at 0, so a gradient is only comparable with float64 on rows where no hidden pre-activation is within rounding
of 0: their mini-batches skip the rows that have one within KINK_BAND (kink_safe_index).  One such row on the wrong side moves a weight
gradient by that row's whole contribution: in 'tf32x3' a pre-activation is off by ~1e-6, and at 16 973 rows x ~1000 hidden units one or two
of them cross 0, which alone puts the privileged encoder's first-layer gradient 6e-4 (relative) away from float64."""
import ctypes as C

import pytest
import torch

from dwbc_b200 import synth
from oracle import ppo_oracle as PO
from test_activations_cpu import NEW, ORACLE_ACT, _Functional, oracle_activation
from test_chain_shapes_cpu import _AC_KW, NETWORKS
from test_gpu_chain_shapes import (COUNTER, GRAD_ABS, N_ENVS, SEED, TOL, T, grad_errors, minibatch_index, params, rollout_inputs, run_rollout,
                                   sms, storage_inputs)
from test_oracle_golden import ppo_hp

pytestmark = pytest.mark.gpu

# 'tf32' with an activation whose derivative jumps at 0: TF32 rounding of the operands moves pre-activations within ~1e-3 of 0 to the
# other side, where the derivative differs by 1 (relu), 0.99 (lrelu) or 0.7 (selu), so the gradient error against float64 is a
# flip-rate effect, not a rounding of each term.  Measured (H100 SXM, 700 W): worst ||dg||/||g|| 0.098 (relu), 0.126 (lrelu, 512/256/128),
# and 1.0e-2 absolute on a critic head bias of norm 0.026 (selu).  Bounds = 2 x those.
TF32_KINK = dict(grad=2.5e-1, floor=2e-2)
KINKED = ("relu", "lrelu", "selu")
KINK_BAND = 2e-5                           # 20 x the error of a 'tf32x3' / 'fp32' pre-activation (~1e-6)
_ref = {}                                  # float64 oracle results per (activation, what, ...)


class _MinAbs:
    """the activation, recording per row the smallest |pre-activation| of the [rows, width] layers it is applied to"""
    def __init__(self, f, rows):
        self.f, self.rows, self.m = f, rows, torch.full((rows,), float("inf"), dtype=torch.float64)

    def __call__(self, x):
        if x.dim() == 2 and x.shape[0] == self.rows:
            self.m = torch.minimum(self.m, x.detach().abs().min(dim=1).values)
        return self.f(x)


def kink_safe_index(key, P, activation, rows):
    """The mini-batch of `rows` rows: the permutation of test_gpu_chain_shapes, without (for relu, lrelu, selu) the storage rows that have a
    hidden pre-activation of the policy or the critic within KINK_BAND of 0 in float64."""
    k = (activation, key, "idx")
    if k not in _ref:
        idx = minibatch_index()
        if activation in KINKED:
            obs = storage_inputs()["observations"].flatten(0, 1).double()
            P64 = {n: v.double() for n, v in P.items()}
            rec = _MinAbs(ORACLE_ACT[activation][0], obs.shape[0])
            saved, PO.F = PO.F, _Functional(rec)
            try:
                PO.actor_mean(P64, obs)
                PO.critic_values(P64, obs)
            finally:
                PO.F = saved
            idx = idx[rec.m[idx] > KINK_BAND]
        _ref[k] = idx
    assert _ref[k].numel() >= rows
    return _ref[k][:rows]


def tol(activation, precision):
    """(forward max abs, gradient relative, gradient absolute floor, loss relative)"""
    t = TOL[precision]
    if precision == "tf32" and activation in ("relu", "lrelu", "selu"):
        return t["fwd"], TF32_KINK["grad"], TF32_KINK["floor"], t["loss"]
    return t["fwd"], t["grad"], GRAD_ABS[precision], t["loss"]


def make_alg(net, activation, precision, dims=None):
    from dwbc_b200.actor_critic import FlatActorCritic
    from dwbc_b200.ppo import FusedPPO
    dims = NETWORKS[net] if dims is None else dims
    manifest, P = params(net) if dims is NETWORKS.get(net) else stock_params()
    ac = FlatActorCritic(device="cuda:0", num_priv=24, num_hist=10, num_prop=76, activation=activation, **{_AC_KW[k]: v for k, v in dims.items()})
    assert ac.manifest == manifest
    ac.load_state_dict(P)
    alg = FusedPPO(ac, device="cuda:0", **dict(ppo_hp(), num_mini_batches=1, num_learning_epochs=1, precision=precision))
    alg.init_storage(N_ENVS, T, [860], [None], [18])
    alg.counter = COUNTER
    s = alg.storage
    for k, v in storage_inputs().items():
        (s._obs_all[:T] if k == "observations" else getattr(s, k)).copy_(v.cuda())
    return alg, P


STOCK = dict(actor_dims=(512, 256, 128), critic_dims=(512, 256, 128))


def stock_params():
    manifest = PO.param_manifest(**STOCK)
    vals = synth.policy_params(manifest, SEED)
    std = torch.tensor([[0.8, 1.0, 1.0] * 4 + [1.0] * 6])
    return manifest, {n: (std.clone() if v is None else torch.from_numpy(v).clone()) for (n, _), v in zip(manifest, vals)}


def ref_rollout(key, P, activation, rows, hist):
    k = (activation, key, "act", rows, hist)
    if k not in _ref:
        P64 = {n: v.double() for n, v in P.items()}
        obs, eps = rollout_inputs(rows)
        with oracle_activation(activation):
            r = PO.policy_act(P64, obs.double(), eps.double(), hist_encoding=hist)
        _ref[k] = [r["mean"], r["values"], r["actions"], r["log_prob"], r["values"]]
    return _ref[k]


def ref_grad(key, P, activation, rows):
    k = (activation, key, "grad", rows)
    if k not in _ref:
        P64 = {n: v.double().requires_grad_(True) for n, v in P.items()}
        st = {n: v.double() for n, v in storage_inputs().items()}
        with oracle_activation(activation):
            loss, info = PO.minibatch_loss(P64, PO.gather(st, kink_safe_index(key, P, activation, rows)), ppo_hp(), COUNTER)
        loss.backward()
        g = {n: (p.grad if p.grad is not None else torch.zeros_like(p)).detach() for n, p in P64.items()}
        _ref[k] = (g, [float(info["surrogate"]), float(info["value"]), float(info["priv_reg"])])
    return _ref[k]


def check_rollout(alg, P, key, activation, precision, rows, hist):
    got = run_rollout(alg, rows, hist)
    ref = ref_rollout(key, P, activation, rows, hist)
    err = max(float((g.double().cpu() - r).abs().max()) for g, r in zip(got, ref))
    assert all(torch.isfinite(t).all() for t in got)
    return err


def run_grad(alg, idx):
    """dwbc_ppo_minibatch_grad on the storage rows idx -> (per-tensor gradients, the surrogate / value / regulariser losses)"""
    from dwbc_b200 import _lib as L
    ac, s, rows = alg.actor_critic, alg.storage, idx.numel()
    h = alg._fill_hp()
    alg._set_precision()
    alg._losses.zero_()
    L.check(L.lib().dwbc_ppo_minibatch_grad(C.addressof(ac.net_cfg), L.ptr(ac.flat), s.c_struct_ptr(), L.ptr(idx.cuda()), rows, C.addressof(h),
                                            L.ptr(alg.grad), L.ptr(alg._losses), L.ptr(alg._workspace(rows)), L.stream_ptr()), "dwbc_ppo_minibatch_grad")
    return {k: v.clone() for k, v in ac.unflat(alg.grad).items()}, alg._losses[:3].clone()


def check_grad(alg, P, key, activation, precision, rows):
    _, t_grad, floor, t_loss = tol(activation, precision)
    got, losses = run_grad(alg, kink_safe_index(key, P, activation, rows))
    ref, ref_losses = ref_grad(key, P, activation, rows)
    worst = grad_errors(got, ref, t_grad, floor)
    lerr = max(abs(float(losses[i]) - ref_losses[i]) / (abs(ref_losses[i]) + 1e-3) for i in range(3))
    assert lerr <= t_loss, (rows, losses.tolist(), ref_losses)
    return worst, lerr


@pytest.mark.parametrize("precision", ["fp32", "tf32x3", "tf32"])
@pytest.mark.parametrize("activation", NEW)
def test_rollout_matches_float64(activation, precision):
    """dwbc_policy_act and the dwbc_critic_values bootstrap on S (tile images; also with the history latent) and C (row-major, padded) at 1,
    129 and 128 x SMs / 4 + 1 rows."""
    fwd = tol(activation, precision)[0]
    for net in ("S", "C"):
        alg, P = make_alg(net, activation, precision)
        for hist in ((False, True) if net == "S" else (False,)):
            errs = [check_rollout(alg, P, net, activation, precision, rows, hist) for rows in (1, 129, 128 * (sms() // 4) + 1)]
            print(f"[{activation} {precision} {net} hist={int(hist)}] rollout max abs error vs float64 {max(errs):.3g}")
            assert max(errs) < fwd, errs


@pytest.mark.parametrize("precision", ["fp32", "tf32x3", "tf32"])
@pytest.mark.parametrize("activation", NEW)
def test_minibatch_grad_matches_float64(activation, precision):
    """dwbc_ppo_minibatch_grad on S and C at 129 and 128 x SMs + 77 rows: per-tensor gradients and the three losses."""
    for net in ("S", "C"):
        alg, P = make_alg(net, activation, precision)
        for rows in (129, 128 * sms() + 77):
            worst, lerr = check_grad(alg, P, net, activation, precision, rows)
            print(f"[{activation} {precision} {net} rows={rows}] worst ||dg||/||g|| vs float64 {worst[1]:.3g} ({worst[0]}), "
                  f"largest ||dg|| {worst[2]:.3g}, losses rel {lerr:.3g}")


@pytest.mark.parametrize("precision", ["fp32", "tf32x3", "tf32"])
@pytest.mark.parametrize("activation", NEW)
def test_hist_latent_and_dagger_grad_match_float64(activation, precision):
    """The history encoder: dwbc_hist_latent (fused exact-fp32 kernel on the tensor-core precisions, layer-wise GEMMs on 'fp32') and the
    DAgger mini-batch gradient (layer-wise forward, col2im / loss kernels with the activation's derivative)."""
    from dwbc_b200 import _lib as L
    alg, P = make_alg("S", activation, precision)
    ac, s, lib = alg.actor_critic, alg.storage, L.lib()
    rows = 2053
    _, t_grad, floor, _ = tol(activation, precision)
    P64 = {n: v.double().requires_grad_(n.startswith(PO.HIST_PREFIX)) for n, v in P.items()}
    obs = s.observations.view(N_ENVS * T, -1)
    idx = minibatch_index()[:rows]
    ob64 = storage_inputs()["observations"].flatten(0, 1)[idx].double()
    with oracle_activation(activation):
        zh_ref = PO.hist_latent(P64, ob64)
        with torch.no_grad():
            zp = PO.priv_latent(P64, ob64)
    loss = (zp - zh_ref).norm(p=2, dim=1).mean()
    loss.backward()
    out = torch.zeros(rows, 20, device="cuda")
    sub = obs[idx.cuda()].contiguous()
    ws = alg._workspace(rows)
    L.check(lib.dwbc_hist_latent(C.addressof(ac.net_cfg), L.ptr(ac.flat), L.ptr(sub), sub.stride(0), L.ptr(out), 20, rows, L.ptr(ws),
                                 L.stream_ptr()), "dwbc_hist_latent")
    e_lat = float((out.double().cpu() - zh_ref.detach()).abs().max())
    alg._losses.zero_()
    L.check(lib.dwbc_dagger_minibatch_grad(C.addressof(ac.net_cfg), L.ptr(ac.flat), s.c_struct_ptr(), L.ptr(idx.cuda()), rows, L.ptr(alg.grad),
                                           L.ptr(alg._losses), L.ptr(ws), L.stream_ptr()), "dwbc_dagger_minibatch_grad")
    got = ac.unflat(alg.grad)
    ref = {n: p.grad.detach() for n, p in P64.items() if n.startswith(PO.HIST_PREFIX)}
    worst = grad_errors(got, ref, t_grad, floor)
    l_err = abs(float(alg._losses[0]) - float(loss)) / float(loss)
    print(f"[{activation} {precision}] history latent max abs error {e_lat:.3g}; DAgger worst ||dg||/||g|| {worst[1]:.3g} ({worst[0]}), loss rel {l_err:.3g}")
    assert e_lat < TOL["tf32x3"]["fwd"] and l_err < TOL[precision]["loss"]
    assert all(float(got[n].abs().max()) == 0.0 for n in got if not n.startswith(PO.HIST_PREFIX))


@pytest.mark.parametrize("precision", ["fp32", "tf32x3", "tf32"])
@pytest.mark.parametrize("activation", ["tanh", "lrelu"])
def test_stock_shape_layer_wise_matches_float64(activation, precision):
    """The stock 512/256/128 trunks run layer by layer (wider than the chains' tile): rollout and mini-batch gradient."""
    alg, P = make_alg("stock", activation, precision, dims=STOCK)
    fwd = tol(activation, precision)[0]
    errs = [check_rollout(alg, P, "stock", activation, precision, rows, False) for rows in (1, 129)]
    worst, lerr = check_grad(alg, P, "stock", activation, precision, 2048)
    print(f"[{activation} {precision} 512/256/128] rollout max abs error {max(errs):.3g}; worst ||dg||/||g|| {worst[1]:.3g} ({worst[0]}), "
          f"losses rel {lerr:.3g}")
    assert max(errs) < fwd, errs


@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
@pytest.mark.parametrize("activation", ["tanh", "lrelu"])
def test_update_end_to_end_matches_oracle(activation, precision):
    """FusedActorCritic(activation=...) + FusedPPO.update() (5 epochs x 4 mini-batches) against the oracle's ppo_update in float64: losses
    and the parameters after 1 and 20 Adam steps, at the fp32 tolerances of test_gpu_ppo.py."""
    from dwbc_b200 import runner_compat as RC
    from dwbc_b200.ppo import FusedPPO
    N, Tn = 256, 8
    ac = RC.FusedActorCritic(76, 76, 18, actor_hidden_dims=(128,), critic_hidden_dims=(128,), activation=activation, num_priv=24, num_hist=10,
                             num_prop=76, device="cuda:0")
    _, P = params("S")
    ac.load_state_dict(P)
    hp = ppo_hp()
    alg = FusedPPO(ac, device="cuda:0", **dict(hp, precision=precision))
    alg.init_storage(N, Tn, [860], [None], [18])
    alg.counter = COUNTER
    st = dict(observations=torch.from_numpy(synth.normal(SEED, 401, (Tn, N, 860))), actions=torch.from_numpy(synth.normal(SEED, 402, (Tn, N, 18))),
              values=torch.from_numpy(synth.normal(SEED, 403, (Tn, N, 2))), returns=torch.from_numpy(synth.normal(SEED, 404, (Tn, N, 2))),
              advantages=torch.from_numpy(synth.normal(SEED, 406, (Tn, N, 2))))
    with torch.no_grad(), oracle_activation(activation):         # old log-probs near the policy's own: ratios near 1, losses of order 1
        mean = PO.actor_mean(P, st["observations"].flatten(0, 1))
        st["actions_log_prob"] = (PO.log_prob2(mean, P["std"], st["actions"].flatten(0, 1)).view(Tn, N, 2) +
                                  torch.from_numpy(synth.normal(SEED, 407, (Tn, N, 2), 0.0, 0.1)))
    s = alg.storage
    for k, v in st.items():
        (s._obs_all[:Tn] if k == "observations" else getattr(s, k)).copy_(v.cuda())
    perm = torch.randperm(N * Tn, generator=torch.Generator().manual_seed(7))
    snap = {}

    def on_step(k, when):
        if k == 0 and when == "step":
            snap["p1"] = ac.unflat(ac.flat.clone())

    res = alg.update(indices=perm.cuda(), on_step=on_step)
    # float64 oracle: with leaky ReLU, the float32 oracle on the CPU is itself 1.8e-4 away from float64 in 0.13 % of the parameters after
    # 20 steps: a pre-activation of this data set lies within float32 rounding of the kink, and which side float32 arithmetic puts it on
    # depends on the summation order.  The GPU's weight gradients are summed with split-K atomics (order varies from run to run), so
    # its 20-step parameters follow one of the two trajectories: the float64 one or the float32 oracle's.  The float32 oracle is the same
    # update in the GPU's precision, so the 20-step parameters must match one of the two references at the full tolerance.
    P32 = {k: v.clone().float() for k, v in P.items()}
    with oracle_activation(activation):
        PO.ppo_update(P32, PO.Adam(list(P32.keys()), hp["learning_rate"]), {k: v.float() for k, v in st.items()}, perm, hp, COUNTER)
    Po = {k: v.double() for k, v in P.items()}
    st = {k: v.double() for k, v in st.items()}
    ref1 = {}

    def record(k, Pk, G, when):
        if k == 0 and when == "post_step":
            ref1.update({n: v.clone() for n, v in Pk.items()})

    with oracle_activation(activation):
        logs = PO.ppo_update(Po, PO.Adam(list(Po.keys()), hp["learning_rate"]), st, perm, hp, COUNTER, record=record)
    o_val = float(torch.stack([l["value"] for l in logs]).mean())
    o_sur = float(torch.stack([l["surrogate"] for l in logs]).mean())
    # Adam's step is ~lr * g / (|g| + 1e-8): an entry whose gradient is ~1e-8 (tanh / leaky-ReLU units deep in saturation) moves by up to
    # lr whatever the arithmetic (test_gpu_ppo.py: "bounded by 2*lr").  Every other entry agrees to 2e-5; such entries are rare.
    d1 = torch.cat([(snap["p1"][n].cpu() - ref1[n]).abs().reshape(-1) for n in ref1])
    got = ac.unflat(ac.flat)
    d20_64 = torch.cat([(got[n].cpu() - Po[n]).abs().reshape(-1) for n in Po])
    d20_32 = torch.cat([(got[n].cpu() - P32[n]).abs().reshape(-1) for n in Po])
    f1 = float((d1 > 2e-5).float().mean())
    f20_64, f20_32 = float((d20_64 > 2e-5).float().mean()), float((d20_32 > 2e-5).float().mean())
    d20, f20 = (d20_64, f20_64) if f20_64 <= f20_32 else (d20_32, f20_32)
    print(f"[{activation} {precision}] update(): losses {res[0] - o_val:+.3g} {res[1] - o_sur:+.3g}; params max abs error after 1 step "
          f"{float(d1.max()):.3g} (fraction beyond 2e-5: {f1:.2g}), after 20 steps {float(d20.max()):.3g} ({f20:.2g}); "
          f"fraction beyond 2e-5 after 20 steps vs float64 {f20_64:.2g}, vs the float32 oracle {f20_32:.2g}")
    assert abs(res[0] - o_val) < 2e-5 * max(1.0, abs(o_val)) and abs(res[1] - o_sur) < 2e-5
    assert float(d1.max()) < 2 * hp["learning_rate"] and float(d20.max()) < 2 * hp["learning_rate"]
    assert f1 < 1e-4 and f20 < 1e-4
