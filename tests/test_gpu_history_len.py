"""The 20- and 50-step proprioception histories (StateHistoryEncoder tsteps = 20 / 50, AC:52-70) through every layer: the post-physics
step's long-history form against the oracle over whole rollouts, the history encoder (fused exact-fp32 kernel and layer-wise GEMMs), the
DAgger backward, rollouts with the history latent and a full update() against float64 autograd of the oracle, and a checkpoint round trip.

Tolerances: 'fp32' and 'tf32x3' take the fp32 bounds of test_gpu_chain_shapes.py (TOL['tf32x3'], GRAD_ABS).  'tf32' takes TF32 below:
the TF32 chains and the layer-wise TF32 GEMMs of the DAgger backward over K = 192 / 256 (conv 1) instead of 128."""
import ctypes as C
import io

import numpy as np
import pytest
import torch

import envstate as E
import history_oracle as HO
from dwbc_b200 import synth
from oracle import env_oracle as EO
from oracle import ppo_oracle as PO
from test_gpu_chain_shapes import GRAD_ABS, TOL, grad_errors, sms
from test_gpu_env import load_sim, make_core
from test_gpu_env_rollout import Schedule, add_schedule, compare_with_oracle, rollout_vs_oracle
from test_oracle_golden import ppo_hp

pytestmark = pytest.mark.gpu

HISTS = (20, 50)
SEED, COUNTER, N_ENVS, T = 43, 1500, 1100, 4
# 'tf32' = 2 x the largest errors measured by test_hist_latent_dagger_and_act_match_float64 over H = 20 and 50 (H100 SXM, 700 W): act
# max abs 9.8e-4, DAgger ||dg|| / ||g|| 2.9e-3 and largest ||dg|| 3.9e-4 (both on encoder.0.weight), DAgger loss relative 1.0e-3
TF32 = dict(fwd=2e-3, grad=6e-3, floor=8e-4, loss=2.1e-3)
_ref = {}


def num_obs(H):
    return 76 * (H + 1) + 24


def tol(precision):
    if precision == "tf32":
        return TF32["fwd"], TF32["grad"], TF32["floor"], TF32["loss"]
    return TOL["tf32x3"]["fwd"], TOL["tf32x3"]["grad"], GRAD_ABS[precision], TOL["tf32x3"]["loss"]


def params(H):
    manifest = HO.param_manifest(num_hist=H)
    vals = synth.policy_params(manifest, SEED)
    std = torch.tensor([[0.8, 1.0, 1.0] * 4 + [1.0] * 6])
    return manifest, {n: (std.clone() if v is None else torch.from_numpy(v).clone()) for (n, _), v in zip(manifest, vals)}


def storage_inputs(H):
    k = (H, "storage")
    if k not in _ref:
        no = num_obs(H)
        _ref[k] = dict(observations=torch.from_numpy(synth.normal(SEED, 301 + H, (T, N_ENVS, no))),
                       actions=torch.from_numpy(synth.normal(SEED, 50, (T, N_ENVS, 18))), values=torch.from_numpy(synth.normal(SEED, 51, (T, N_ENVS, 2))),
                       returns=torch.from_numpy(synth.normal(SEED, 52, (T, N_ENVS, 2))),
                       actions_log_prob=torch.from_numpy(synth.normal(SEED, 53, (T, N_ENVS, 2), -20.0, 1.0)),
                       advantages=torch.from_numpy(synth.normal(SEED, 54, (T, N_ENVS, 2))))
    return _ref[k]


def make_alg(H, precision):
    from dwbc_b200.actor_critic import FlatActorCritic
    from dwbc_b200.ppo import FusedPPO
    manifest, P = params(H)
    ac = FlatActorCritic(device="cuda:0", num_priv=24, num_hist=H, num_prop=76)
    assert ac.manifest == manifest
    ac.load_state_dict(P)
    alg = FusedPPO(ac, device="cuda:0", **dict(ppo_hp(), num_mini_batches=1, num_learning_epochs=1, precision=precision))
    alg.init_storage(N_ENVS, T, [num_obs(H)], [None], [18])
    alg.counter = COUNTER
    for k, v in storage_inputs(H).items():
        (alg.storage._obs_all[:T] if k == "observations" else getattr(alg.storage, k)).copy_(v.cuda())
    return alg, P


def index(rows):
    return torch.from_numpy(np.argsort(synth.uniform(SEED, 60, (N_ENVS * T,)))).long()[:rows]


# ---------------------------------------------------------------------------------------------- post-physics step (long-history form)
def params_env(name, N, H, clip=None):
    from dwbc_b200.config import WidowGo1Params
    kw = dict(E.ENV_CONFIGS[name], history_len=H)
    if clip is not None:
        kw["clip_observations"] = clip
    return WidowGo1Params(num_envs=N, **kw)


@pytest.mark.parametrize("N", [1024, 1000])
@pytest.mark.parametrize("H", HISTS)
def test_long_history_rollout_matches_oracle(H, N):
    """36 steps with single observation columns beyond +-100 and resets on and after injected events (the ep_len <= 1 fill): obs
    (clipped), history (unclipped) and every output against the oracle.  1024 envs would take the TMA kernel at 10 steps; here the
    generic kernel runs (its out-of-range counter stays 0)."""
    seed = 21
    p = params_env("flat", N, H)
    assert p.num_obs == num_obs(H)
    sched = add_schedule(Schedule(), synth.initial_env_state(p, seed)["episode_length_buf"], groups=(5, 23, 47))
    rec = rollout_vs_oracle(p, seed, 36, False, False, sched)
    assert int(rec["oob"].sum()) == sum(len(v) for v in sched.events.values())
    assert int((rec["oob"] & (rec["ep_len"] <= 1)).sum()) > 0 and int(rec["reset"].sum()) > 0


@pytest.mark.parametrize("H", HISTS)
def test_long_history_dense_clipping_into_storage_rows_matches_oracle(H):
    """clip_observations = 1 (most rows clipped on most steps) on 'full', observations written straight into rollout-storage rows
    (set_obs_target, rows wider than num_obs), 20 steps at 1000 envs."""
    seed, N, steps = 31, 1000, 20
    p = params_env("full", N, H, clip=1.0)
    st = E.initial(p, seed)
    core = make_core(p, st)
    orc = EO.EnvOracle(p, E.oracle_state(p, st))
    rt = E.runtime(p)
    core.common_step_counter = orc.common_step_counter = 140
    store = torch.zeros(3, N, p.num_obs + 4, device="cuda")
    n_oob = 0
    for t in range(1, steps + 1):
        sim = E.sim_state(p, seed, t, orc.s.env_origins)
        load_sim(core, p, sim)
        E.load_sim_into_oracle(orc, p, sim)
        tab = torch.from_numpy(synth.rand_table(p, seed, t))
        obs, rew, arew, rst, _ = orc.post_physics_step(tab, rt)
        core.set_obs_target(store[t % 3, :, :p.num_obs])
        core.post_physics_step(tab.cuda())
        assert core.obs_buf.data_ptr() == store[t % 3].data_ptr()
        compare_with_oracle(core, orc, p, t, obs, rew, arew, rst)
        n_oob += int((~(orc.s.prop.abs() <= p.clip_observations).all(dim=1)).sum())
    assert n_oob > N * steps // 2


# ---------------------------------------------------------------------------------------------- history encoder, DAgger, rollouts
@pytest.mark.parametrize("precision", ["fp32", "tf32x3", "tf32"])
@pytest.mark.parametrize("H", HISTS)
def test_hist_latent_dagger_and_act_match_float64(H, precision):
    """dwbc_hist_latent (the fused kernel on the tensor-core precisions, layer-wise GEMMs on 'fp32'), dwbc_dagger_minibatch_grad (layer-wise
    forward and backward of every conv) and act(hist_encoding=True) against float64 autograd of the oracle."""
    from dwbc_b200 import _lib as L
    fwd, t_grad, floor, t_loss = tol(precision)
    alg, P = make_alg(H, precision)
    ac, s, lib = alg.actor_critic, alg.storage, L.lib()
    rows = 2053
    P64 = {n: v.double().requires_grad_(n.startswith(PO.HIST_PREFIX)) for n, v in P.items()}
    idx = index(rows)
    ob64 = storage_inputs(H)["observations"].flatten(0, 1)[idx].double()
    zh_ref = HO.hist_latent(P64, ob64)
    with torch.no_grad():
        zp = PO.priv_latent(P64, ob64)
    loss = (zp - zh_ref).norm(p=2, dim=1).mean()
    loss.backward()
    out = torch.zeros(rows, 20, device="cuda")
    sub = s.observations.view(N_ENVS * T, -1)[idx.cuda()].contiguous()
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
    # rollouts with the history latent: 1, 129 and 128 x SMs / 4 + 1 rows (one program per head below that)
    e_act = 0.0
    for n in (1, 129, 128 * (sms() // 4) + 1):
        obs = torch.from_numpy(synth.normal(SEED, 70, (n, num_obs(H))))
        eps = torch.from_numpy(synth.normal(SEED, 71, (n, 18)))
        with torch.no_grad(), HO.history_encoder():
            r = PO.policy_act({k: v.detach().double() for k, v in P64.items()}, obs.double(), eps.double(), hist_encoding=True)
        alg._packed = False
        alg.act(obs.cuda(), obs.cuda(), True, eps=eps.cuda())
        tr = alg.transition
        for g, rf in ((tr.action_mean, r["mean"]), (tr.values, r["values"]), (tr.actions, r["actions"]), (tr.actions_log_prob, r["log_prob"])):
            assert torch.isfinite(g).all()
            e_act = max(e_act, float((g.double().cpu() - rf).abs().max()))
    print(f"[H={H} {precision}] history latent max abs error {e_lat:.3g}; DAgger worst ||dg||/||g|| {worst[1]:.3g} ({worst[0]}), "
          f"largest ||dg|| {worst[2]:.3g}, loss rel {l_err:.3g}; act(hist_encoding) max abs error {e_act:.3g}")
    assert e_lat < TOL["tf32x3"]["fwd"], e_lat                # exact fp32 on every precision
    assert l_err < t_loss and e_act < fwd, (l_err, e_act)
    assert all(float(got[n].abs().max()) == 0.0 for n in got if not n.startswith(PO.HIST_PREFIX))
    if H == 50:
        assert float(got["actor.history_encoder.conv_layers.4.weight"].abs().max()) > 0


# ---------------------------------------------------------------------------------------------- update() end to end
@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
@pytest.mark.parametrize("H", HISTS)
def test_update_end_to_end_matches_oracle(H, precision):
    """FusedActorCritic(num_hist=H) + FusedPPO.update() (5 epochs x 4 mini-batches; the regulariser target is the history latent of every
    storage row) against the oracle's ppo_update in float64: losses and the parameters after 1 and 20 Adam steps (test_gpu_ppo.py bounds)."""
    from dwbc_b200 import runner_compat as RC
    from dwbc_b200.ppo import FusedPPO
    N, Tn, no = 256, 8, num_obs(H)
    ac = RC.FusedActorCritic(76, 76, 18, actor_hidden_dims=(128,), critic_hidden_dims=(128,), num_priv=24, num_hist=H, num_prop=76,
                             device="cuda:0")
    _, P = params(H)
    ac.load_state_dict(P)
    hp = ppo_hp()
    alg = FusedPPO(ac, device="cuda:0", **dict(hp, precision=precision))
    alg.init_storage(N, Tn, [no], [None], [18])
    alg.counter = COUNTER
    st = dict(observations=torch.from_numpy(synth.normal(SEED, 401, (Tn, N, no))), actions=torch.from_numpy(synth.normal(SEED, 402, (Tn, N, 18))),
              values=torch.from_numpy(synth.normal(SEED, 403, (Tn, N, 2))), returns=torch.from_numpy(synth.normal(SEED, 404, (Tn, N, 2))),
              advantages=torch.from_numpy(synth.normal(SEED, 406, (Tn, N, 2))))
    with torch.no_grad():
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
    Po = {k: v.double() for k, v in P.items()}
    st = {k: v.double() for k, v in st.items()}
    ref1 = {}

    def record(k, Pk, G, when):
        if k == 0 and when == "post_step":
            ref1.update({n: v.clone() for n, v in Pk.items()})

    with HO.history_encoder():                                   # the regulariser target of every mini-batch (PPO:175-176)
        logs = PO.ppo_update(Po, PO.Adam(list(Po.keys()), hp["learning_rate"]), st, perm, hp, COUNTER, record=record)
    o_val = float(torch.stack([l["value"] for l in logs]).mean())
    o_sur = float(torch.stack([l["surrogate"] for l in logs]).mean())
    o_reg = float(torch.stack([l["priv_reg"] for l in logs]).mean())
    d1 = torch.cat([(snap["p1"][n].cpu() - ref1[n]).abs().reshape(-1) for n in ref1])
    got = ac.unflat(ac.flat)
    d20 = torch.cat([(got[n].cpu() - Po[n]).abs().reshape(-1) for n in Po])
    f1, f20 = float((d1 > 2e-5).float().mean()), float((d20 > 2e-5).float().mean())
    print(f"[H={H} {precision}] update(): losses {res[0] - o_val:+.3g} {res[1] - o_sur:+.3g} priv_reg {res[5] - o_reg:+.3g}; params max abs "
          f"error after 1 step {float(d1.max()):.3g} ({f1:.2g} beyond 2e-5), after 20 steps {float(d20.max()):.3g} ({f20:.2g})")
    assert abs(res[0] - o_val) < 2e-5 * max(1.0, abs(o_val)) and abs(res[1] - o_sur) < 2e-5 and abs(res[5] - o_reg) < 2e-5 * max(1.0, o_reg)
    assert float(d1.max()) < 2 * hp["learning_rate"] and float(d20.max()) < 2 * hp["learning_rate"]
    assert f1 < 1e-4 and f20 < 1e-4


# ---------------------------------------------------------------------------------------------- checkpoints
def test_checkpoint_round_trip_with_third_conv():
    """OnPolicyRunner.save / load (OPR:276-286) of a 50-step policy: state_dict names include conv_layers.4; a torch.save'd checkpoint
    loads into a fresh FusedActorCritic with identical values and an identical history latent."""
    from dwbc_b200 import _lib as L
    from dwbc_b200 import runner_compat as RC
    kw = dict(actor_hidden_dims=(128,), critic_hidden_dims=(128,), num_priv=24, num_hist=50, num_prop=76, device="cuda:0")
    a = RC.FusedActorCritic(76, 76, 18, **kw)
    a.load_state_dict(params(50)[1])
    sd = a.state_dict()
    assert "actor.history_encoder.conv_layers.4.weight" in sd and tuple(sd["actor.history_encoder.conv_layers.4.weight"].shape) == (10, 10, 5)
    buf = io.BytesIO()
    torch.save({"model_state_dict": sd}, buf)
    buf.seek(0)
    b = RC.FusedActorCritic(76, 76, 18, **kw)
    b.load_state_dict(torch.load(buf)["model_state_dict"])
    assert all(torch.equal(v, b.state_dict()[k]) for k, v in sd.items())
    obs = torch.from_numpy(synth.normal(SEED, 90, (300, num_obs(50)))).cuda()
    outs = []
    for m in (a, b):
        out = torch.zeros(300, 20, device="cuda")
        ws = torch.zeros(L.lib().dwbc_workspace_bytes(C.addressof(m.net_cfg), 300) // 4 + 1, device="cuda")
        L.check(L.lib().dwbc_hist_latent(C.addressof(m.net_cfg), L.ptr(m.flat), L.ptr(obs), obs.stride(0), L.ptr(out), 20, 300, L.ptr(ws),
                                         L.stream_ptr()), "dwbc_hist_latent")
        outs.append(out)
    assert torch.equal(outs[0], outs[1]) and bool(outs[0].abs().sum() > 0)
