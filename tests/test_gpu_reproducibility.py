"""GPU: every cross-CTA floating-point sum is a fixed-order sum, so the library's outputs repeat bit for bit, also while other work on the
GPU changes how the CTAs are scheduled (the second repetition of every test runs beside a matmul loop on another stream).  Covered: a
whole training loop (rollout with K1 in Philox mode, GAE, two PPO iterations and one DAgger iteration) on every precision, with and
without per-step statistics; whole mini-batch gradients on paths the loop does not reach (torque supervision, the 512/256/128 layer-wise
path, the 50-step DAgger backward); the debug GEMM entry points; clip + Adam; GAE."""
import ctypes as C
import contextlib
import os
import sys

import pytest
import torch

from dwbc_b200 import _lib as L
from dwbc_b200 import synth

pytestmark = pytest.mark.gpu

HPS = dict(num_learning_epochs=1, num_mini_batches=4, clip_param=0.2, gamma=0.99, lam=0.95, learning_rate=2e-4, value_loss_coef=1.0,
           use_clipped_value_loss=True, entropy_coef=0.01, max_grad_norm=1.0, min_policy_std=[[0.15, 0.25, 0.25] * 4 + [0.2] * 3 + [0.05] * 3],
           mixing_schedule=[1.0, 0, 1], priv_reg_coef_schedual=[0, 1, 1000, 1000])


@contextlib.contextmanager
def busy_gpu():
    """A long matmul loop on a side stream, so that the kernels under test share the SMs with it."""
    side = torch.cuda.Stream()
    a = torch.randn(2048, 2048, device="cuda")
    with torch.cuda.stream(side):
        for _ in range(40):
            a = torch.tanh(a @ a * 1e-3)
    yield
    torch.cuda.synchronize()


def run_twice(fn):
    first = fn()
    torch.cuda.synchronize()
    with busy_gpu():
        second = fn()
    torch.cuda.synchronize()
    return first, second


def assert_bitwise(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), (k, float((a[k].double() - b[k].double()).abs().max()))


def make_alg(precision, N=1024, T=24, hist=10, wide=False, ts=False):
    from dwbc_b200.actor_critic import FlatActorCritic
    from dwbc_b200.ppo import FusedPPO
    dims = dict(actor_hidden_dims=(512, 256, 128), critic_hidden_dims=(512, 256, 128)) if wide else {}
    ac = FlatActorCritic(device="cuda:0", seed=0, init_std=[[0.8, 1.0, 1.0] * 4 + [1.0] * 6], num_priv=24, num_hist=hist, num_prop=76, **dims)
    alg = FusedPPO(ac, device="cuda:0", precision=precision, torque_supervision=ts, **HPS)
    n_obs = 76 + 24 + 76 * hist
    alg.init_storage(N, T, [n_obs], [None], [18])
    alg.counter = 1500
    s = alg.storage
    s._obs_all.copy_(torch.from_numpy(synth.rollout_inputs(N, T, n_obs, 3)["obs"]).cuda())
    s.actions.copy_(torch.from_numpy(synth.normal(3, 10, (T, N, 18), std=0.8)).cuda())
    s.values.copy_(torch.from_numpy(synth.normal(3, 11, (T, N, 2))).cuda())
    s.actions_log_prob.copy_(torch.from_numpy(synth.normal(3, 12, (T, N, 2), mean=-20.0, std=2.0)).cuda())
    s.returns.copy_(torch.from_numpy(synth.normal(3, 13, (T, N, 2))).cuda())
    s.advantages.copy_(torch.from_numpy(synth.normal(3, 14, (T, N, 2))).cuda())
    if ts:
        alg.set_arm_default_coeffs([20.0] * 6, [0.5] * 6, [0.1] * 6)
        for k, name in enumerate(("target_arm_torques", "current_arm_dof_pos", "current_arm_dof_vel")):
            getattr(s, name).copy_(torch.from_numpy(synth.normal(3, 20 + k, (T, N, 6))).cuda())
    return alg


@pytest.mark.parametrize("precision,wide,ts", [("fp32", False, False), ("tf32", False, False), ("tf32x3", False, False),
                                               ("fp32", False, True), ("tf32x3", False, True), ("fp32", True, False), ("tf32", True, False),
                                               ("tf32x3", True, False)])
def test_ppo_minibatch_gradient_repeats(precision, wide, ts):
    alg = make_alg(precision, wide=wide, ts=ts)
    ac, s = alg.actor_critic, alg.storage
    idx = torch.randperm(s.num_envs * s.num_transitions_per_env, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    hp = alg._fill_hp()
    alg._set_precision()
    mbs = idx.numel() // 4
    ws = alg._workspace(mbs)
    o, n_act = ac.net_cfg.off_std, 18

    def once():
        losses = torch.zeros(5, device="cuda")
        for _ in range(3):                    # the loss means accumulate over mini-batches
            L.check(alg._lib.dwbc_ppo_minibatch_grad(C.addressof(ac.net_cfg), L.ptr(ac.flat), s.c_struct_ptr(), L.ptr(idx[:mbs]), mbs,
                                                     C.addressof(hp), L.ptr(alg.grad), L.ptr(losses), L.ptr(ws), L.stream_ptr()), "grad")
        return dict(losses=losses, grad=alg.grad.clone())

    a, b = run_twice(once)
    assert torch.isfinite(a["losses"]).all() and a["grad"][o:o + n_act].abs().sum() > 0 and (float(a["losses"][4]) > 0) == ts
    assert_bitwise(a, b)


@pytest.mark.parametrize("hist", [10, 50])
def test_dagger_loss_repeats(hist):
    alg = make_alg("tf32x3", hist=hist)
    ac, s = alg.actor_critic, alg.storage
    alg._set_precision()
    idx = torch.arange(0, s.num_envs * s.num_transitions_per_env, 3, device="cuda")
    ws = alg._workspace(idx.numel())

    def once():
        losses = torch.zeros(5, device="cuda")
        L.check(alg._lib.dwbc_dagger_minibatch_grad(C.addressof(ac.net_cfg), L.ptr(ac.flat), s.c_struct_ptr(), L.ptr(idx), idx.numel(),
                                                    L.ptr(alg.grad), L.ptr(losses), L.ptr(ws), L.stream_ptr()), "dagger")
        return dict(loss=losses[:1], grad=alg.grad.clone())

    a, b = run_twice(once)
    assert float(a["loss"]) > 0
    assert_bitwise(a, b)


def test_clip_adam_step_repeats():
    lib = L.lib()
    n = 600_000                              # > 592 blocks of 1024: every partial slot in use
    g0 = torch.from_numpy(synth.normal(4, 1, (n,))).cuda() * 1e-2
    p0 = torch.from_numpy(synth.normal(4, 2, (n,))).cuda()
    hp = L.PpoHyper()
    hp.max_grad_norm, hp.lr, hp.beta1, hp.beta2, hp.adam_eps, hp.grad_scale = 1.0, 1e-3, 0.9, 0.999, 1e-8, 1.0
    scratch = torch.zeros(L.NORM_SCRATCH, dtype=torch.float64, device="cuda")

    def once():
        p, g, m, v, norm = p0.clone(), g0.clone(), torch.zeros_like(p0), torch.zeros_like(p0), torch.zeros(1, device="cuda")
        for step in (1, 2):
            L.check(lib.dwbc_clip_adam_step(L.ptr(p), L.ptr(g), L.ptr(m), L.ptr(v), 0, n, C.addressof(hp), step, L.ptr(scratch),
                                            L.ptr(norm), L.stream_ptr()), "clip_adam")
        return dict(p=p, g=g, m=m, v=v, norm=norm)

    a, b = run_twice(once)
    ref = float(g0.double().mul(1.0).norm() * min(1.0, 1.0 / (float(g0.double().norm()) + 1e-6)))
    assert abs(float(a["norm"]) - ref) < 1e-5 * ref                    # the second step sees the clipped gradient
    assert_bitwise(a, b)


@pytest.mark.parametrize("normalize", [0, 1])
@pytest.mark.parametrize("N,T", [(4096, 40), (40000, 8)])
def test_gae_repeats(normalize, N, T):
    """(40000 envs: more columns than DWBC_GAE_MAX_BLOCKS blocks cover, so the blocks loop)"""
    lib = L.lib()
    rew = torch.from_numpy(synth.normal(6, 1, (T, N, 2))).cuda()
    val = torch.from_numpy(synth.normal(6, 2, (T, N, 2))).cuda()
    dones = torch.from_numpy(synth.bernoulli(6, 3, (T, N), 0.05)).to(torch.uint8).cuda()
    last = torch.from_numpy(synth.normal(6, 4, (N, 2))).cuda()

    def once():
        ret, adv = torch.empty_like(rew), torch.empty_like(rew)
        stats = torch.zeros(L.GAE_STATS, dtype=torch.float64, device="cuda")
        L.check(lib.dwbc_gae(L.ptr(rew), L.ptr(val), L.ptr(dones), L.ptr(last), L.ptr(ret), L.ptr(adv), L.ptr(stats), T, N, 0.99, 0.95,
                             normalize, L.stream_ptr()), "gae")
        return dict(ret=ret, adv=adv, stats=stats[:4])

    a, b = run_twice(once)
    assert float(a["stats"][0]) == T * N * 2 and float(a["stats"][3]) == 0.0          # the counter is back at zero
    raw = a["ret"].double() - val.double()
    assert abs(float(a["stats"][1]) - float(raw.sum())) < 1e-6 * float(raw.abs().sum())
    assert_bitwise(a, b)


def test_debug_weight_gradients_repeat():
    """dwbc_debug_gemm mode 2 (split-K, fp32 and TF32) and dwbc_debug_wgrad_group (TF32, 3xTF32), each accumulating into its output"""
    from test_gpu_wgrad_group import Gemm
    lib = L.lib()
    lib.dwbc_debug_gemm.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p,
                                    C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    lib.dwbc_debug_wgrad_group.argtypes = [C.POINTER(Gemm), C.c_int, C.c_int, C.c_int, C.c_void_p]
    R, M, N = 40960, 128, 100
    G = torch.from_numpy(synth.normal(8, 1, (R, M))).cuda()
    X = torch.from_numpy(synth.normal(8, 2, (R, N))).cuda()
    G2 = torch.from_numpy(synth.normal(8, 3, (R, 64))).cuda()

    def once():
        out = {}
        for tc in (0, 1):
            dW, db = torch.ones(M, N, device="cuda"), torch.ones(M, device="cuda")
            L.check(lib.dwbc_debug_gemm(2, tc, G.data_ptr(), M, X.data_ptr(), N, dW.data_ptr(), N, None, db.data_ptr(), M, N, R, 0,
                                        L.stream_ptr()), "gemm")
            out[f"gemm{tc}_dw"], out[f"gemm{tc}_db"] = dW, db
        for x3 in (0, 1):
            dW1, db1, dW2 = torch.ones(M, N, device="cuda"), torch.ones(M, device="cuda"), torch.zeros(64, N, device="cuda")
            descs = (Gemm * 2)(Gemm(g=G.data_ptr(), g_ld=M, x=X.data_ptr(), x_ld=N, dw=dW1.data_ptr(), lddw=N, db=db1.data_ptr(), mo=M, ni=N),
                               Gemm(g=G2.data_ptr(), g_ld=64, x=X.data_ptr(), x_ld=N, dw=dW2.data_ptr(), lddw=N, db=None, mo=64, ni=N))
            assert lib.dwbc_debug_wgrad_group(descs, 2, R, x3, L.stream_ptr()) == 0
            out.update({f"group{x3}_dw1": dW1, f"group{x3}_db1": db1, f"group{x3}_dw2": dW2})
        return out

    a, b = run_twice(once)
    ref = (G.double().T @ X.double()) + 1.0
    assert float((a["gemm0_dw"].double() - ref).abs().max()) < 1e-3 * float(ref.abs().max())
    assert_bitwise(a, b)


def _tensors(prefix, obj, skip=("_ws",)):
    return {f"{prefix}.{k}": v.clone() for k, v in vars(obj).items() if isinstance(v, torch.Tensor) and k not in skip}


@pytest.mark.parametrize("sync_stats", [True, False])
@pytest.mark.parametrize("precision", ["fp32", "tf32", "tf32x3"])
def test_training_loop_repeats(precision, sync_stats):
    """bench.py's workload (flat, 4096 envs, T = 40, K1 in Philox mode writing rewards and dones into the storage rows): two PPO
    iterations and one DAgger iteration, twice from the same seeds; every tensor of the parameters, gradient, Adam moments, storage and
    env state must be bitwise the same, and so must the losses and extras['episode']."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    import bench

    def once():
        w = bench.Workload("cuda:0", 0, precision=precision)
        w.env.sync_stats = sync_stats
        losses = []
        for _ in range(2):
            w.iteration()
            losses.append(torch.tensor(w.last[:7], dtype=torch.float64))
        w.dagger_iteration()
        losses.append(torch.tensor([w.last], dtype=torch.float64))
        out = dict(losses=torch.cat(losses), obs=w.obs.clone())
        alg = w.alg
        for prefix, obj in (("alg", alg), ("storage", alg.storage), ("adam", alg.optimizer), ("hist_adam", alg.hist_encoder_optimizer),
                            ("ac", alg.actor_critic), ("env", w.env)):
            out.update(_tensors(prefix, obj))
        episode = w.env.episode_stats(reset=False) if not sync_stats else w.env.extras.get("episode", {})
        out.update({f"episode.{k}": torch.as_tensor(v, dtype=torch.float64) for k, v in episode.items()})
        del w
        torch.cuda.empty_cache()
        return out

    a, b = run_twice(once)
    assert a["losses"].isfinite().all() and any(k.startswith("episode.") for k in a)
    assert_bitwise(a, b)
