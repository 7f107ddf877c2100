"""GPU parity of the rsl_rl update path (GAE, ActorCritic forward, PPO loss/backward, clip+Adam,
DAgger) through the C ABI, against the reference golden vectors and the CPU oracle."""
import os

import numpy as np
import pytest
import torch

from dwbc_b200 import synth
from oracle import ppo_oracle as PO
from test_oracle_golden import golden_params, ppo_hp

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")


def make_alg(N, T, P, **over):
    from dwbc_b200.actor_critic import FlatActorCritic
    from dwbc_b200.ppo import FusedPPO
    ac = FlatActorCritic(device="cuda:0", num_priv=24, num_hist=10, num_prop=76)
    ac.load_state_dict(P)
    hp = ppo_hp()
    hp.update(over)
    hp.setdefault("precision", "fp32")          # the CUDA-core anchor unless a test names a tensor-core mode
    alg = FusedPPO(ac, device="cuda:0", **hp)
    alg.init_storage(N, T, [860], [None], [18])
    return alg


def fill_storage(alg, g, inp, T):
    dev = alg.device
    s = alg.storage
    s._obs_all.copy_(torch.from_numpy(inp["obs"]).to(dev))
    for k, src in (("actions", "actions"), ("values", "values"), ("actions_log_prob", "log_prob"), ("returns", "returns"),
                   ("advantages", "advantages"), ("rewards", "rewards")):
        getattr(s, k).copy_(torch.from_numpy(g[src]).to(dev))
    s.dones.copy_(torch.from_numpy(inp["dones"]).to(dev).unsqueeze(-1).to(torch.uint8))


def test_gae_matches_reference_golden():
    g = np.load(os.path.join(G, "ppo.npz"))
    N, T, seed, _ = [int(x) for x in g["meta"]]
    alg = make_alg(N, T, golden_params(g, seed))
    inp = synth.rollout_inputs(N, T, 860, seed)
    fill_storage(alg, g, inp, T)
    alg.storage.returns.zero_()
    alg.storage.advantages.zero_()
    alg.storage.compute_returns(torch.from_numpy(g["last_values"]).cuda(), 0.99, 0.95)
    np.testing.assert_allclose(alg.storage.returns.cpu().numpy(), g["returns"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(alg.storage.advantages.cpu().numpy(), g["advantages"], rtol=1e-5, atol=2e-6)


@pytest.mark.parametrize("N,T,gamma,lam", [
    pytest.param(4096, 40, 0.99, 0.95, id="4096-40"), pytest.param(8192, 24, 0.99, 0.95, id="8192-24"),
    pytest.param(37, 5, 0.99, 0.95, id="37-5"),
    pytest.param(40000, 8, 0.99, 0.95, id="40000-8"),                     # more columns than DWBC_GAE_MAX_BLOCKS x 64: the blocks loop
    pytest.param(4096, 40, 0.998, 0.95, id="4096-40-gamma0.998"),          # FusedPPO's default gamma
    pytest.param(4096, 40, 0.99, 1.0, id="4096-40-lam1"), pytest.param(4096, 40, 0.99, 0.0, id="4096-40-lam0"),
    pytest.param(37, 1, 0.99, 0.95, id="37-1"),                            # a one-step rollout
])
def test_gae_matches_oracle_full_size(N, T, gamma, lam):
    from dwbc_b200.storage import FusedRolloutStorage
    s = FusedRolloutStorage(N, T, [8], [None], [18], "cuda:0")
    rew = torch.from_numpy(synth.normal(1, 1, (T, N, 2)))
    val = torch.from_numpy(synth.normal(1, 2, (T, N, 2)))
    dones = torch.from_numpy(synth.bernoulli(1, 3, (T, N, 1), 0.05)).to(torch.uint8)
    last = torch.from_numpy(synth.normal(1, 4, (N, 2)))
    s.rewards.copy_(rew.cuda()); s.values.copy_(val.cuda()); s.dones.copy_(dones.cuda())
    s.compute_returns(last.cuda(), gamma, lam)
    ret, adv = PO.compute_returns(rew, val, dones, last, gamma, lam)
    np.testing.assert_allclose(s.returns.cpu().numpy(), ret.numpy(), rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(s.advantages.cpu().numpy(), adv.numpy(), rtol=1e-5, atol=2e-6)
    a = s.advantages.double()
    assert abs(float(a.mean())) < 1e-5 and abs(float(a.std()) - 1.0) < 1e-4          # size-independent property
    # two-phase path (multi-GPU route): raw advantages + stats, then normalise
    from dwbc_b200 import _lib as L
    s.advantages.zero_(); s._stats.zero_()
    L.check(L.lib().dwbc_gae(L.ptr(s.rewards), L.ptr(s.values), L.ptr(s.dones), L.ptr(last.cuda()), L.ptr(s.returns),
                             L.ptr(s.advantages), L.ptr(s._stats), T, N, gamma, lam, 0, L.stream_ptr()), "gae")
    raw = (ret - val)
    np.testing.assert_allclose(s.advantages.cpu().numpy(), raw.numpy(), rtol=1e-6, atol=1e-6)
    assert float(s._stats[0]) == T * N * 2
    L.check(L.lib().dwbc_normalize_advantages(L.ptr(s.advantages), L.ptr(s._stats), T * N * 2, L.stream_ptr()), "norm")
    np.testing.assert_allclose(s.advantages.cpu().numpy(), adv.numpy(), rtol=1e-5, atol=2e-6)


@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
def test_policy_act_matches_reference_golden(precision):
    """fp32 tolerances for both the CUDA-core anchor and the error-compensated tensor-core path (3xTF32)."""
    g = np.load(os.path.join(G, "ppo.npz"))
    N, T, seed, _ = [int(x) for x in g["meta"]]
    P = golden_params(g, seed)
    alg = make_alg(N, T, P, precision=precision)
    inp = synth.rollout_inputs(N, T, 860, seed)
    obs = torch.from_numpy(inp["obs"]).cuda()
    for t in (0, 1, T - 1):
        mean_o = PO.actor_mean(P, obs[t].cpu())
        eps = ((torch.from_numpy(g["actions"][t]) - mean_o) / P["std"]).cuda()
        alg.storage.step = t
        a = alg.act(obs[t], obs[t], False, eps=eps)
        np.testing.assert_allclose(a.cpu().numpy(), g["actions"][t], rtol=0, atol=1e-5)
        np.testing.assert_allclose(alg.storage.values[t].cpu().numpy(), g["values"][t], rtol=0, atol=1e-5)
        np.testing.assert_allclose(alg.storage.actions_log_prob[t].cpu().numpy(), g["log_prob"][t], rtol=0, atol=1e-4)
        if t == 0:
            np.testing.assert_allclose(alg.storage.mu[0].cpu().numpy(), g["mu0"], rtol=0, atol=1e-5)
        assert torch.equal(alg.storage.sigma[t], alg.actor_critic.std.expand(N, -1))
    # time-out bootstrap (PPO:133-134) + dones storage (RS:102)
    alg.storage.step = 0
    alg.storage.values[0].copy_(torch.from_numpy(g["values"][0]).cuda())
    alg.process_env_step(torch.from_numpy(inp["rew"][0]).cuda(), torch.from_numpy(inp["arm_rew"][0]).cuda(),
                         torch.from_numpy(inp["dones"][0]).cuda(), {"time_outs": torch.from_numpy(inp["time_outs"][0]).cuda()})
    np.testing.assert_allclose(alg.storage.rewards[0].cpu().numpy(), g["rewards"][0], rtol=0, atol=1e-6)
    assert torch.equal(alg.storage.dones[0, :, 0].cpu(), torch.from_numpy(inp["dones"][0]).to(torch.uint8))
    # student (history-encoder) rollout forward
    Pd = golden_params(g, seed)
    # dag_mu0 was produced with the post-update() parameters: rebuild them from param20 + min-std
    flat20 = torch.from_numpy(g["param20"])
    off = 0
    for n in Pd:
        k = Pd[n].numel()
        Pd[n] = flat20[off:off + k].view_as(Pd[n]).clone()
        off += k
    alg2 = make_alg(N, T, Pd, precision=precision)
    inp2 = synth.rollout_inputs(N, T, 860, seed + 1)
    o0 = torch.from_numpy(inp2["obs"][0]).cuda()
    eps2 = ((torch.from_numpy(g["dag_actions0"]) - torch.from_numpy(g["dag_mu0"])) / Pd["std"]).cuda()
    alg2.act(o0, o0, True, eps=eps2)
    np.testing.assert_allclose(alg2.storage.mu[0].cpu().numpy(), g["dag_mu0"], rtol=0, atol=1e-5)


def _flat_ref(ac, vec):
    """reference-ordered unpadded vector -> padded flat layout"""
    out, off = {}, 0
    for n, s in ac.manifest:
        k = int(np.prod(s))
        out[n] = torch.from_numpy(vec[off:off + k]).view(s)
        off += k
    return out


@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
def test_ppo_update_matches_reference_golden(precision):
    """BASELINE.json configs[0] on the GPU: losses, clipped gradient of step 1, post-Adam parameters
    after step 1 and after the full 20-step update().  The SAME fp32 tolerances hold for the CUDA-core anchor ('fp32') and for
    the error-compensated tensor-core path ('tf32x3': fused chains + grouped weight gradients on wgmma, three TF32 products
    per GEMM) -- the path bench.py reports as its headline.
    Stated fp32 tolerances: clipped grads rtol 1e-3 / atol 2e-6; parameters atol 2e-5 after one Adam step and after the full
    20-step update() (Adam's first update is lr*g/(|g|+eps): an entry with |g| ~ eps = 1e-8 turns an absolute gradient difference
    of 5e-10 -- ulps of the fp32 accumulation order, which atomics make run-dependent -- into 1e-5; bounded by 2*lr = 4e-4)."""
    g = np.load(os.path.join(G, "ppo.npz"))
    N, T, seed, counter = [int(x) for x in g["meta"]]
    alg = make_alg(N, T, golden_params(g, seed), precision=precision)
    alg.counter = counter
    fill_storage(alg, g, synth.rollout_inputs(N, T, 860, seed), T)
    ac = alg.actor_critic
    snap = {}

    def on_step(k, when):
        if k == 0 and when == "step":
            snap["grad1"] = alg.grad.clone()        # clip_adam leaves the clipped gradient behind
            snap["param1"] = ac.flat.clone()

    res = alg.update(indices=torch.from_numpy(g["perm"]).cuda().long(), on_step=on_step)
    ref = g["update_result"]
    assert abs(res[0] - ref[0]) < 2e-5 * max(1, abs(ref[0])) and abs(res[1] - ref[1]) < 2e-5 and abs(res[5] - ref[5]) < 2e-5
    assert res[3] == ref[3] and abs(res[6] - ref[6]) < 1e-7
    g1, p1, p20 = _flat_ref(ac, g["grad1"]), _flat_ref(ac, g["param1"]), _flat_ref(ac, g["param20"])
    got_g, got_p1, got_p20 = ac.unflat(snap["grad1"]), ac.unflat(snap["param1"]), ac.unflat(ac.flat)
    worst = [max(float((a[n].cpu() - b[n]).abs().max()) for n, _ in ac.manifest) for a, b in ((got_g, g1), (got_p1, p1), (got_p20, p20))]
    print(f"[{precision}] max abs error vs the reference: clipped grad {worst[0]:.3g}, params after 1 step {worst[1]:.3g}, after 20 steps {worst[2]:.3g}; "
          f"losses {res[0] - ref[0]:+.3g} {res[1] - ref[1]:+.3g} {res[5] - ref[5]:+.3g}")
    for n, _ in ac.manifest:
        np.testing.assert_allclose(got_g[n].cpu().numpy(), g1[n].numpy(), rtol=1e-3, atol=2e-6, err_msg="grad1 " + n)
        np.testing.assert_allclose(got_p1[n].cpu().numpy(), p1[n].numpy(), rtol=0, atol=2e-5, err_msg="param1 " + n)
        np.testing.assert_allclose(got_p20[n].cpu().numpy(), p20[n].numpy(), rtol=0, atol=2e-5, err_msg="param20 " + n)
    assert alg.counter == counter + 1 and alg.storage.step == 0


@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
def test_ppo_update_with_torque_supervision_matches_reference_golden(precision):
    """PPO:224-239 switched on (fixed-gain arm model PPO:318-323; SURVEY 8f row f4): update() against the unmodified reference's
    (tests/golden/make_golden_ts.py -> ppo_ts.npz), same stated fp32 tolerances as the branch-off golden.  The arm-torque loss sits in
    the FIN_PPO epilogue hook of the arm head ('tf32x3') / in ppo_loss_kernel ('fp32'); its targets travel through
    process_env_step(infos) into the storage rows (PPO:136-142, RS:108-111)."""
    from test_oracle_golden import ts_hp
    g, gts = np.load(os.path.join(G, "ppo.npz")), np.load(os.path.join(G, "ppo_ts.npz"))
    N, T, seed, counter = [int(x) for x in gts["meta"]]
    ts = synth.arm_torque_inputs(N, T, 6, seed)
    hp = ts_hp(gts, ts)
    coefs = hp.pop("arm_coefs")
    alg = make_alg(N, T, golden_params(g, seed), precision=precision, **hp)
    alg.set_arm_default_coeffs(*coefs)                                                  # OPR:91
    alg.counter = counter
    inp = synth.rollout_inputs(N, T, 860, seed)
    fill_storage(alg, g, inp, T)
    s = alg.storage
    for t in range(T):                                    # the targets arrive the reference's way: infos of process_env_step
        s.step = t
        infos = {k: torch.from_numpy(ts[k][t]).cuda() for k in ("target_arm_torques", "current_arm_dof_pos", "current_arm_dof_vel")}
        infos["time_outs"] = torch.from_numpy(inp["time_outs"][t]).cuda()
        alg.process_env_step(torch.from_numpy(inp["rew"][t]).cuda(), torch.from_numpy(inp["arm_rew"][t]).cuda(),
                             torch.from_numpy(inp["dones"][t]).cuda(), infos)
    np.testing.assert_array_equal(s.target_arm_torques.cpu().numpy(), ts["target_arm_torques"])
    ac = alg.actor_critic
    snap = {}

    def on_step(k, when):
        if k == 0 and when == "step":
            snap["grad1"], snap["param1"] = alg.grad.clone(), ac.flat.clone()

    res = alg.update(indices=torch.from_numpy(g["perm"]).cuda().long(), on_step=on_step)
    ref = gts["update_result"]
    assert abs(res[0] - ref[0]) < 2e-5 * max(1, abs(ref[0])) and abs(res[1] - ref[1]) < 2e-5 and abs(res[5] - ref[5]) < 2e-5
    assert abs(res[2] - ref[2]) < 1e-4 * abs(ref[2]) and abs(res[4] - ref[4]) < 1e-7 and res[3] == ref[3]
    g1, p1, p20 = _flat_ref(ac, gts["grad1"]), _flat_ref(ac, gts["param1"]), _flat_ref(ac, gts["param20"])
    got_g, got_p1, got_p20 = ac.unflat(snap["grad1"]), ac.unflat(snap["param1"]), ac.unflat(ac.flat)
    for n, _ in ac.manifest:
        np.testing.assert_allclose(got_g[n].cpu().numpy(), g1[n].numpy(), rtol=1e-3, atol=2e-6, err_msg="grad1 " + n)
        np.testing.assert_allclose(got_p1[n].cpu().numpy(), p1[n].numpy(), rtol=0, atol=2e-5, err_msg="param1 " + n)
        np.testing.assert_allclose(got_p20[n].cpu().numpy(), p20[n].numpy(), rtol=0, atol=2e-5, err_msg="param20 " + n)
    # and the branch is really on: the gradient differs from the branch-off golden
    off = _flat_ref(ac, g["grad1"])
    assert max(float((got_g[n].cpu() - off[n]).abs().max()) for n, _ in ac.manifest) > 1e-3


def test_dagger_update_matches_reference_golden():
    g = np.load(os.path.join(G, "ppo.npz"))
    N, T, seed, _ = [int(x) for x in g["meta"]]
    P = golden_params(g, seed)
    flat20, off = torch.from_numpy(g["param20"]), 0
    for n in P:
        k = P[n].numel()
        P[n] = flat20[off:off + k].view_as(P[n]).clone()
        off += k
    alg = make_alg(N, T, P)
    inp2 = synth.rollout_inputs(N, T, 860, seed + 1)
    alg.storage._obs_all.copy_(torch.from_numpy(inp2["obs"]).cuda())
    loss = alg.update_dagger(indices=torch.from_numpy(g["dag_perm"]).cuda().long())
    assert abs(loss - float(g["dag_loss"][0])) < 2e-5
    ref = _flat_ref(alg.actor_critic, g["dag_params"])
    got = alg.actor_critic.unflat(alg.actor_critic.flat)
    for n, _ in alg.actor_critic.manifest:
        np.testing.assert_allclose(got[n].cpu().numpy(), ref[n].numpy(), rtol=0, atol=2e-5, err_msg=n)


def test_minibatch_grad_matches_oracle_autograd_large():
    """M = 8192 rows (oracle autograd on CPU): unclipped gradient of one mini-batch."""
    N, T, seed = 1024, 8, 21
    manifest = PO.param_manifest()
    vals = synth.policy_params(manifest, seed)
    P = {n: (torch.tensor([[0.8, 1.0, 1.0] * 4 + [1.0] * 6]) if v is None else torch.from_numpy(v).clone()) for (n, _), v in zip(manifest, vals)}
    alg = make_alg(N, T, P, num_mini_batches=1, num_learning_epochs=1)
    alg.counter = 1500
    inp = synth.rollout_inputs(N, T, 860, seed)
    obs = torch.from_numpy(inp["obs"])
    st = dict(observations=obs[:T], actions=torch.from_numpy(synth.normal(seed, 50, (T, N, 18))),
              values=torch.from_numpy(synth.normal(seed, 51, (T, N, 2))), returns=torch.from_numpy(synth.normal(seed, 52, (T, N, 2))),
              actions_log_prob=torch.from_numpy(synth.normal(seed, 53, (T, N, 2), -20.0, 1.0)),
              advantages=torch.from_numpy(synth.normal(seed, 54, (T, N, 2))))
    s = alg.storage
    s._obs_all.copy_(obs.cuda())
    for k in ("actions", "values", "returns", "actions_log_prob", "advantages"):
        getattr(s, k).copy_(st[k].cuda())
    idx = torch.from_numpy(np.argsort(synth.uniform(seed, 60, (N * T,)))).long()
    hp = ppo_hp()
    for n in P:
        P[n].requires_grad_(True)
    loss, info = PO.minibatch_loss(P, PO.gather(st, idx), hp, 1500)
    loss.backward()
    import ctypes as C
    from dwbc_b200 import _lib as L
    ac = alg.actor_critic
    h = alg._fill_hp()
    alg._losses.zero_()
    L.check(L.lib().dwbc_ppo_minibatch_grad(C.addressof(ac.net_cfg), L.ptr(ac.flat), s.c_struct_ptr(), L.ptr(idx.cuda()), N * T,
                                            C.addressof(h), L.ptr(alg.grad), L.ptr(alg._losses), L.ptr(alg._workspace(N * T)),
                                            L.stream_ptr()), "grad")
    got = ac.unflat(alg.grad)
    for n in P:
        ref = P[n].grad if P[n].grad is not None else torch.zeros_like(P[n])
        scale = max(float(ref.abs().max()), 1e-6)
        err = float((got[n].cpu() - ref).abs().max()) / scale
        assert err < 2e-3, (n, err)
    ls = alg._losses.cpu()
    assert abs(float(ls[0]) - float(info["surrogate"])) < 1e-4 * max(1.0, abs(float(info["surrogate"])))
    assert abs(float(ls[1]) - float(info["value"])) < 1e-4 * max(1.0, abs(float(info["value"])))
    assert abs(float(ls[2]) - float(info["priv_reg"])) < 1e-4


@pytest.mark.parametrize("precision", ["fp32", "tf32x3", "tf32"])
def test_stock_policy_shape_512_256_128_matches_oracle_autograd(precision):
    """SURVEY 8f row f4: the stock legged_gym trunk shape (LRC:206-207: actor / critic hidden dims [512, 256, 128]) in front of the
    widowGo1 heads.  Layers wider than 128 do not fit the fused chain's operand tile, so this configuration runs layer by layer
    (`gemm_simt_kernel` on 'fp32' / 'tf32x3', `gemm_tc2_kernel` on 'tf32'): rollout forward and the unclipped gradient of one
    2048-row mini-batch against the oracle (torch autograd on CPU)."""
    N, T, seed = 256, 8, 33
    dims = dict(actor_dims=(512, 256, 128), critic_dims=(512, 256, 128))
    manifest = PO.param_manifest(**dims)
    vals = synth.policy_params(manifest, seed)
    P = {n: (torch.tensor([[0.8, 1.0, 1.0] * 4 + [1.0] * 6]) if v is None else torch.from_numpy(v).clone()) for (n, _), v in zip(manifest, vals)}
    from dwbc_b200.actor_critic import FlatActorCritic
    from dwbc_b200.ppo import FusedPPO
    ac = FlatActorCritic(device="cuda:0", num_priv=24, num_hist=10, num_prop=76, actor_hidden_dims=dims["actor_dims"],
                         critic_hidden_dims=dims["critic_dims"])
    assert ac.manifest == manifest
    ac.load_state_dict(P)
    hp = ppo_hp()
    alg = FusedPPO(ac, device="cuda:0", **dict(hp, num_mini_batches=1, num_learning_epochs=1, precision=precision))
    alg.init_storage(N, T, [860], [None], [18])
    alg.counter = 1500
    inp = synth.rollout_inputs(N, T, 860, seed)
    obs = torch.from_numpy(inp["obs"])
    # rollout forward (PPO.act) on the first step
    eps = torch.from_numpy(inp["eps"][0])
    ref_act = PO.policy_act(P, obs[0], eps)
    alg.act(obs[0].cuda(), obs[0].cuda(), False, eps=eps.cuda())
    s = alg.storage
    tol_f = 1e-3 if precision == "tf32" else 2e-5      # tf32: only the 128-wide layers run on the tensor cores
    e_mean = float((s.mu[0].cpu() - ref_act["mean"]).abs().max())
    e_val = float((s.values[0].cpu() - ref_act["values"]).abs().max())
    assert e_mean < tol_f and e_val < tol_f * max(1.0, float(ref_act["values"].abs().max())), (e_mean, e_val)
    st = dict(observations=obs[:T], actions=torch.from_numpy(synth.normal(seed, 50, (T, N, 18))),
              values=torch.from_numpy(synth.normal(seed, 51, (T, N, 2))), returns=torch.from_numpy(synth.normal(seed, 52, (T, N, 2))),
              actions_log_prob=torch.from_numpy(synth.normal(seed, 53, (T, N, 2), -20.0, 1.0)),
              advantages=torch.from_numpy(synth.normal(seed, 54, (T, N, 2))))
    s._obs_all.copy_(obs.cuda())
    for k in ("actions", "values", "returns", "actions_log_prob", "advantages"):
        getattr(s, k).copy_(st[k].cuda())
    idx = torch.from_numpy(np.argsort(synth.uniform(seed, 60, (N * T,)))).long()
    for n in P:
        P[n].requires_grad_(True)
    loss, info = PO.minibatch_loss(P, PO.gather(st, idx), hp, 1500)
    loss.backward()
    import ctypes as C
    from dwbc_b200 import _lib as L
    h = alg._fill_hp()
    alg._set_precision()
    alg._losses.zero_()
    L.check(L.lib().dwbc_ppo_minibatch_grad(C.addressof(ac.net_cfg), L.ptr(ac.flat), s.c_struct_ptr(), L.ptr(idx.cuda()), N * T,
                                            C.addressof(h), L.ptr(alg.grad), L.ptr(alg._losses), L.ptr(alg._workspace(N * T)),
                                            L.stream_ptr()), "grad")
    got = ac.unflat(alg.grad)
    worst = 0.0
    tol_g = 1e-2 if precision == "tf32" else 2e-3      # measured: 3.3e-3 (tf32), 1.6e-6 (fp32 / tf32x3)
    for n in P:
        ref = P[n].grad if P[n].grad is not None else torch.zeros_like(P[n])
        scale = max(float(ref.abs().max()), 1e-6)
        err = float((got[n].cpu() - ref).abs().max()) / scale
        worst = max(worst, err)
        assert err < tol_g, (n, err)
    ls = alg._losses.cpu()
    print(f"[{precision}] 512/256/128 trunks: act mean err {e_mean:.3g}, value err {e_val:.3g}, worst per-tensor gradient error / scale {worst:.3g}")
    rel = 2e-2 if precision == "tf32" else 1e-4
    assert abs(float(ls[0]) - float(info["surrogate"])) < rel * max(1.0, abs(float(info["surrogate"])))
    assert abs(float(ls[1]) - float(info["value"])) < rel * max(1.0, abs(float(info["value"])))
    assert abs(float(ls[2]) - float(info["priv_reg"])) < rel


# Tolerances of the plain TF32 path = 2 x the errors seen against the reference golden vectors (printed by the test;
# operands truncated to 10 mantissa bits by the tensor core, fp32 accumulation, up to 6 layers deep).  The bound on the parameters is on
# the RMS, not the max: Adam's update is ~lr * sign(g) for small |g|, so one entry whose tiny gradient changes sign moves by up to 2*lr
# per step whatever the precision of the rest; the RMS says how many entries do that.
TF32_TOL = dict(mean=8e-3, value=8e-3, loss_rel=1e-2, grad_rel_norm=1e-2, param20_rms=4e-5, param20_max=4e-3)


def test_tf32_tensor_core_path_matches_reference_within_stated_tolerance():
    """precision='tf32' (wgmma, truncated 10-bit mantissa inputs, fp32 accumulate) on BASELINE configs[0] against the reference golden."""
    g = np.load(os.path.join(G, "ppo.npz"))
    N, T, seed, counter = [int(x) for x in g["meta"]]
    P = golden_params(g, seed)
    alg = make_alg(N, T, P, precision="tf32")
    inp = synth.rollout_inputs(N, T, 860, seed)
    obs0 = torch.from_numpy(inp["obs"][0]).cuda()
    mean_o = PO.actor_mean(P, obs0.cpu())
    eps = ((torch.from_numpy(g["actions"][0]) - mean_o) / P["std"]).cuda()
    alg.act(obs0, obs0, False, eps=eps)
    e_mean = float(np.abs(alg.storage.mu[0].cpu().numpy() - g["mu0"]).max())
    e_val = float(np.abs(alg.storage.values[0].cpu().numpy() - g["values"][0]).max())
    alg.storage.step = 0
    alg.counter = counter
    fill_storage(alg, g, inp, T)
    ac = alg.actor_critic
    snap = {}

    def on_step(k, when):
        if k == 0 and when == "step":
            snap["grad1"] = alg.grad.clone()

    res = alg.update(indices=torch.from_numpy(g["perm"]).cuda().long(), on_step=on_step)
    ref = g["update_result"]
    g1 = torch.cat([v.reshape(-1) for v in _flat_ref(ac, g["grad1"]).values()])
    got = torch.cat([v.reshape(-1).cpu() for v in ac.unflat(snap["grad1"]).values()])
    p20 = torch.cat([v.reshape(-1) for v in _flat_ref(ac, g["param20"]).values()])
    gotp = torch.cat([v.reshape(-1).cpu() for v in ac.unflat(ac.flat).values()])
    e_grad = float((got - g1).norm() / g1.norm())
    e_rms, e_max = float((gotp - p20).pow(2).mean().sqrt()), float((gotp - p20).abs().max())
    e_loss = max(abs(res[0] - ref[0]) / abs(ref[0]), abs(res[1] - ref[1]) / max(abs(ref[1]), 1e-3), abs(res[5] - ref[5]) / abs(ref[5]))
    print(f"[tf32] measured: mean {e_mean:.3g}, value {e_val:.3g}, losses rel {e_loss:.3g}, clipped grad ||dg||/||g|| {e_grad:.3g}, "
          f"params after 20 steps rms {e_rms:.3g} max {e_max:.3g}")
    assert e_mean < TF32_TOL["mean"] and e_val < TF32_TOL["value"] and e_loss < TF32_TOL["loss_rel"]
    assert e_grad < TF32_TOL["grad_rel_norm"]
    assert e_rms < TF32_TOL["param20_rms"] and e_max < TF32_TOL["param20_max"]


# forward: max abs difference of means / values to the exact-fp32 path; gradient: ||dg|| / ||g|| per parameter tensor
# (loss: the reported means are fp32 atomic sums over ~38 k rows; their accumulation order changes with the work-item plan and from run to
# run -- 0.7e-5 ... 2.2e-5 relative seen for the SAME gradients --, so the 3xTF32 bound is 3 x the largest value seen)
CHAIN_TOL = {"tf32": dict(fwd=8e-3, grad=1e-2, loss=2e-3), "tf32x3": dict(fwd=2e-5, grad=2e-5, loss=6e-5)}


@pytest.mark.parametrize("precision", ["tf32", "tf32x3"])
@pytest.mark.parametrize("hist", [False, True])
def test_fused_chain_forward_matches_fp32_path_many_tiles(hist, precision):
    """The fused layer-chain kernel (mlp_chain2.cuh; TF32 and error-compensated 3xTF32) against the exact-fp32 layer-wise path of the same
    library (itself pinned to the reference by the tests above) at a row count that gives every CTA several tile pairs plus a ragged
    last tile.  Tolerances: CHAIN_TOL (TF32: 2 x measured; 3xTF32: fp32-grade)."""
    g = np.load(os.path.join(G, "ppo.npz"))
    P = golden_params(g, int(g["meta"][2]))
    N = 148 * 128 * 2 + 3 * 128 + 77
    gen = torch.Generator(device="cuda").manual_seed(5)
    obs = torch.randn(N, 860, device="cuda", generator=gen)
    eps = torch.randn(N, 18, device="cuda", generator=gen)
    out = {}
    for prec in ("fp32", precision):
        alg = make_alg(N, 1, P, precision=prec)
        alg.act(obs, obs, hist, eps=eps)
        s = alg.storage
        alg.compute_returns(obs)                                   # critic-only chain (PPO:148-150)
        s.step = 0
        alg.act(obs, obs, hist, eps=eps)                           # second call re-packs (compute_returns used the workspace), third reuses the images
        first = s.mu[0].clone()
        alg.act(obs, obs, hist, eps=eps)
        assert torch.equal(first, s.mu[0])
        out[prec] = [s.mu[0].clone(), s.values[0].clone(), s.actions[0].clone(), s.actions_log_prob[0].clone(), alg._last_values.clone()]
        assert torch.equal(s.sigma[0], alg.actor_critic.std.expand(N, -1))
        del alg
    tol = CHAIN_TOL[precision]
    errs = [float((a - b).abs().max()) for a, b in zip(out["fp32"], out[precision])]
    print(f"[{precision}, hist={hist}] max abs diff to the fp32 path: mean {errs[0]:.3g} value {errs[1]:.3g} action {errs[2]:.3g} log-prob {errs[3]:.3g} bootstrap {errs[4]:.3g}")
    for i in (0, 1, 2, 4):
        assert errs[i] < tol["fwd"], (i, errs[i])
    assert errs[3] < 1e-3                                          # log-prob of a = mu + sigma*eps does not depend on mu
    assert all(torch.isfinite(t).all() for t in out[precision])


# Row counts of the backward test below, one per tail shape of its tf32 chain launches on a 132-SM H100 (3xTF32 always runs one-tile
# items).  Each is the planner's own choice (launch_chain2n) for the forward and the backward launch; test_host_cpu.py checks that it
# stays so.  The last tile is ragged (77 rows) throughout.
CHAIN_TAIL_ROWS = {
    "one_tile_items": 65 * 128 + 77,                # 66 tiles x 2 programs fit the SMs: one tile per item
    "pairs_odd_last_pair": 240 * 128 + 77,          # 241 tiles, two-tile items only: the last pair holds the ragged tile alone
    "pairs_ragged_last_pair": 241 * 128 + 77,       # 242 tiles, two-tile items only: the ragged tile is the last pair's second
    "one_tile_tail": 298 * 128 + 77,                # 299 tiles: 120 pairs, then 59 one-tile items, the ragged tile last
}


@pytest.mark.parametrize("shape", sorted(CHAIN_TAIL_ROWS))
@pytest.mark.parametrize("precision", ["tf32", "tf32x3"])
def test_fused_chain_backward_matches_fp32_path_many_tiles(precision, shape):
    """Mini-batch gradient through the fused forward chains (loss in the epilogue), backward chains and the MN-major weight-gradient GEMMs
    against the exact-fp32 layer-wise path of the same library, at the row counts of CHAIN_TAIL_ROWS.
    Tolerances: CHAIN_TOL, per parameter tensor ||g - g_fp32|| <= tol ||g_fp32|| (+ 1e-7 abs)."""
    import ctypes as C
    from dwbc_b200 import _lib as L
    g = np.load(os.path.join(G, "ppo.npz"))
    P = golden_params(g, int(g["meta"][2]))
    N, T = CHAIN_TAIL_ROWS[shape], 1
    grads, losses = {}, {}
    gen = torch.Generator(device="cuda").manual_seed(9)
    alg = make_alg(N, T, P, num_mini_batches=1, num_learning_epochs=1)
    alg.counter = 1500
    s = alg.storage
    s._obs_all.normal_(generator=gen)
    for k in ("actions", "values", "returns", "advantages"):
        getattr(s, k).normal_(generator=gen)
    s.actions_log_prob.normal_(generator=gen).sub_(20.0)
    idx = torch.randperm(N * T, device="cuda", generator=gen)
    ac = alg.actor_critic
    for prec in ("fp32", precision):
        alg.precision = prec
        h = alg._fill_hp()
        alg._losses.zero_()
        L.check(L.lib().dwbc_ppo_minibatch_grad(C.addressof(ac.net_cfg), L.ptr(ac.flat), s.c_struct_ptr(), L.ptr(idx), N * T, C.addressof(h),
                                                L.ptr(alg.grad), L.ptr(alg._losses), L.ptr(alg._workspace(N * T)), L.stream_ptr()), "grad")
        grads[prec] = {k: v.clone() for k, v in ac.unflat(alg.grad).items()}
        losses[prec] = alg._losses.clone()
    tol = CHAIN_TOL[precision]
    worst = ("", 0.0)
    for k in grads["fp32"]:
        a, b = grads["fp32"][k].double(), grads[precision][k].double()
        assert torch.isfinite(b).all(), k
        rel = float((a - b).norm()) / max(float(a.norm()), 1e-12)
        if float(a.norm()) > 1e-6 and rel > worst[1]:
            worst = (k, rel)
        assert float((a - b).norm()) <= tol["grad"] * float(a.norm()) + 1e-7, (k, float((a - b).norm()), float(a.norm()))
    lerr = max(abs(float(losses[precision][i] - losses["fp32"][i])) / (abs(float(losses["fp32"][i])) + 1e-3) for i in range(4))
    print(f"[{precision}] worst ||dg||/||g|| = {worst[1]:.3g} ({worst[0]}), losses rel {lerr:.3g}")
    assert lerr <= tol["loss"]


DAGGER_TF32_TOL = dict(loss_rel=2e-3, param_rms=2e-5, param_max=8e-4)      # the errors are printed below


def test_dagger_update_tf32_path_within_stated_tolerance():
    """update_dagger (PPO:265-291) on the TF32 path: the history-encoder GEMMs run on gemm_tc2_kernel (forward, data gradient and the
    MN-major weight gradient of the layer-wise kernel).  Against the reference's golden vectors; tolerances = 2 x the measured errors
    (RMS over the history-encoder parameters after the 20 Adam steps: a few entries with near-zero gradients move by up to lr per step)."""
    g = np.load(os.path.join(G, "ppo.npz"))
    N, T, seed, _ = [int(x) for x in g["meta"]]
    P = golden_params(g, seed)
    flat20, off = torch.from_numpy(g["param20"]), 0
    for n in P:
        k = P[n].numel()
        P[n] = flat20[off:off + k].view_as(P[n]).clone()
        off += k
    alg = make_alg(N, T, P, precision="tf32")
    inp2 = synth.rollout_inputs(N, T, 860, seed + 1)
    alg.storage._obs_all.copy_(torch.from_numpy(inp2["obs"]).cuda())
    loss = alg.update_dagger(indices=torch.from_numpy(g["dag_perm"]).cuda().long())
    ref = _flat_ref(alg.actor_critic, g["dag_params"])
    got = alg.actor_critic.unflat(alg.actor_critic.flat)
    hist = [n for n, _ in alg.actor_critic.manifest if n.startswith("actor.history_encoder.")]
    d = torch.cat([(got[n].cpu() - ref[n]).reshape(-1) for n in hist])
    e_loss = abs(loss - float(g["dag_loss"][0])) / abs(float(g["dag_loss"][0]))
    e_rms, e_max = float(d.pow(2).mean().sqrt()), float(d.abs().max())
    print(f"[tf32 dagger] measured: loss rel {e_loss:.3g}, history-encoder params after 20 steps rms {e_rms:.3g} max {e_max:.3g}")
    for n, _ in alg.actor_critic.manifest:
        assert torch.isfinite(got[n]).all(), n
        if n not in hist:
            assert torch.equal(got[n].cpu(), ref[n]) or float((got[n].cpu() - ref[n]).abs().max()) < 1e-7, n    # update_dagger touches nothing else
    assert e_loss < DAGGER_TF32_TOL["loss_rel"] and e_rms < DAGGER_TF32_TOL["param_rms"] and e_max < DAGGER_TF32_TOL["param_max"]
