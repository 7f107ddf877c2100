"""GPU: CUDA-graph replay computes what the eager calls compute, bit for bit.  bench.py's workload (flat, 4096 envs, T = 40, K1 in
Philox mode writing straight into the storage rows) runs two PPO iterations and one DAgger iteration eagerly and, on fresh objects with
the same seeds, with a captured rollout (RolloutGraph) and captured update() / update_dagger() (FusedPPO(cuda_graphs=True)).  The
schedules and the command curriculum move every iteration and the rollouts cross a push step, so every device-resident value (step,
push decision, curriculum, schedule values, Adam bias correction) is exercised; no library call happens
during a replay; a new storage shape re-captures; the cooperative GAE launch captures with the bits of the eager call."""
import ctypes as C
import os
import sys

import pytest
import torch

from dwbc_b200 import _lib as L
from dwbc_b200 import synth

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tensors(prefix, obj, skip=("_ws",)):
    return {f"{prefix}.{k}": v.clone() for k, v in vars(obj).items() if isinstance(v, torch.Tensor) and k not in skip}


def assert_bitwise(a, b):
    assert a.keys() == b.keys(), set(a) ^ set(b)
    for k in a:
        assert torch.equal(a[k], b[k]), (k, float((a[k].double() - b[k].double()).abs().max()))


class ReplayLaunches:
    """dwbc_launch_count() around every CUDAGraph.replay(): the library must launch nothing while a graph replays."""

    def __init__(self, monkeypatch):
        self.replays, self.moved = 0, 0
        orig = torch.cuda.CUDAGraph.replay

        def replay(graph):
            n0 = L.lib().dwbc_launch_count()
            orig(graph)
            self.moved += L.lib().dwbc_launch_count() - n0
            self.replays += 1
        monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", replay)


def run_workload(precision, graphs, ts):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import bench
    from dwbc_b200.graphs import RolloutGraph
    w = bench.Workload("cuda:0", 0, precision=precision)
    alg, s = w.alg, w.alg.storage
    w.env.common_step_counter = 130                     # steps 131 .. 250: the push of step 150 (push_interval 150) falls in the first rollout
    for name in ("lin_vel_x", "ang_vel_yaw", "tracking_ang_vel_yaw", "l", "p", "y"):
        setattr(w.p, name + "_schedule", [0, 6])        # the command curriculum moves at every update_command_curriculum()
    alg.mixing_schedule = [1.0, 1500, 4]                 # mixing ratio 0, 0.25, 0.5 and priv-reg coef 0, 0.25, 0.5 over the iterations
    alg.priv_reg_coef_schedual = [0, 1, 1500, 4]
    if ts:
        alg.torque_supervision = True
        s.enable_torque_supervision(alg.actor_critic.num_arm_actions)
        alg.set_arm_default_coeffs([20.0] * 6, [0.5] * 6, [0.1] * 6)
        alg.torque_supervision_schedule = [0.1, 1500, 4]
        for k, name in enumerate(("target_arm_torques", "current_arm_dof_pos", "current_arm_dof_vel")):
            getattr(s, name).copy_(torch.from_numpy(synth.normal(3, 20 + k, tuple(getattr(s, name).shape))).cuda())
    alg.cuda_graphs = graphs
    rg = RolloutGraph(alg, w.env, physics=lambda t: w.env.bind_sim(**w.pool[t])) if graphs else None
    results = []
    for dagger in (False, False, True):
        w.env.update_command_curriculum()
        obs = rg.run(w.obs, dagger) if graphs else w.rollout(hist_encoding=dagger)
        alg.compute_returns(obs)
        results.append(torch.tensor([alg.update_dagger()] if dagger else list(alg.update()), dtype=torch.float64))
        w.obs = obs
    if graphs:
        assert len(rg._graphs) == 2                     # one rollout graph with and one without the history-encoder latent
    out = dict(losses=torch.cat(results), obs=w.obs.clone(), step_counter=torch.tensor(w.env.common_step_counter),
               adam_steps=torch.tensor([alg.optimizer.step, alg.hist_encoder_optimizer.step]))
    for prefix, obj in (("alg", alg), ("storage", s), ("adam", alg.optimizer), ("hist_adam", alg.hist_encoder_optimizer),
                        ("ac", alg.actor_critic), ("env", w.env)):
        out.update(_tensors(prefix, obj))
    out.update({f"episode.{k}": torch.as_tensor(v, dtype=torch.float64) for k, v in w.env.episode_stats(reset=False).items()})
    out.update({f"pool{t}.{k}": v.clone() for t, p in enumerate(w.pool) for k, v in p.items()})
    del w, rg
    torch.cuda.empty_cache()
    return out


@pytest.mark.parametrize("precision,ts", [("fp32", False), ("tf32", False), ("tf32x3", False), ("tf32x3", True)])
def test_graphs_replay_the_eager_bits(precision, ts, monkeypatch):
    eager = run_workload(precision, False, ts)
    counter = ReplayLaunches(monkeypatch)
    graphed = run_workload(precision, True, ts)
    assert counter.replays == 6 and counter.moved == 0, (counter.replays, counter.moved)
    assert eager["losses"].isfinite().all() and any(k.startswith("episode.") for k in eager)
    mix = eager["losses"][[3, 10]]
    assert mix[0] != mix[1]                             # the schedules did move between the two PPO iterations
    assert (eager["losses"][[4, 11]] != 0).all() == ts
    assert_bitwise(eager, graphed)


def _synthetic_alg(N, T, graphs):
    from dwbc_b200.actor_critic import FlatActorCritic
    from dwbc_b200.ppo import FusedPPO
    ac = FlatActorCritic(device="cuda:0", seed=0, init_std=[[0.8, 1.0, 1.0] * 4 + [1.0] * 6], num_priv=24, num_hist=10, num_prop=76)
    alg = FusedPPO(ac, device="cuda:0", num_learning_epochs=2, num_mini_batches=4, learning_rate=2e-4, entropy_coef=0.01, cuda_graphs=graphs,
                   mixing_schedule=[1.0, 1500, 4], priv_reg_coef_schedual=[0, 1, 1500, 4])
    alg.counter = 1500
    alg.generator = torch.Generator(device="cuda:0")
    alg.generator.manual_seed(11)
    return alg


def _fill(alg, N, T):
    alg.init_storage(N, T, [860], [None], [18])
    s = alg.storage
    s._obs_all.copy_(torch.from_numpy(synth.rollout_inputs(N, T, 860, 3)["obs"]).cuda())
    for k, name in enumerate(("actions", "values", "actions_log_prob", "returns", "advantages")):
        getattr(s, name).copy_(torch.from_numpy(synth.normal(3, 10 + k, tuple(getattr(s, name).shape))).cuda())


def test_storage_shape_change_recaptures():
    out = {}
    for graphs in (False, True):
        alg = _synthetic_alg(1024, 8, graphs)
        losses, captured = [], []
        for N, T in ((1024, 8), (1024, 8), (2048, 4)):
            if alg.storage is None or (alg.storage.num_envs, alg.storage.num_transitions_per_env) != (N, T):
                _fill(alg, N, T)
            losses.append(torch.tensor(alg.update(), dtype=torch.float64))
            if graphs:
                captured.append(alg._graphs["ppo"]["graph"])
        if graphs:
            assert captured[0] is captured[1] and captured[2] is not captured[1]
        out[graphs] = dict(losses=torch.stack(losses), flat=alg.actor_critic.flat.clone(), m=alg.optimizer.m.clone(), v=alg.optimizer.v.clone())
    assert_bitwise(out[False], out[True])


@pytest.mark.parametrize("N,T", [(4096, 40), (40000, 8)])
def test_gae_captures_with_the_eager_bits(N, T):
    lib = L.lib()
    rew = torch.from_numpy(synth.normal(6, 1, (T, N, 2))).cuda()
    val = torch.from_numpy(synth.normal(6, 2, (T, N, 2))).cuda()
    dones = torch.from_numpy(synth.bernoulli(6, 3, (T, N), 0.05)).to(torch.uint8).cuda()
    last = torch.from_numpy(synth.normal(6, 4, (N, 2))).cuda()
    bufs = {g: (torch.zeros_like(rew), torch.zeros_like(rew), torch.zeros(L.GAE_STATS, dtype=torch.float64, device="cuda")) for g in (0, 1)}

    def gae(ret, adv, stats):
        L.check(lib.dwbc_gae(L.ptr(rew), L.ptr(val), L.ptr(dones), L.ptr(last), L.ptr(ret), L.ptr(adv), L.ptr(stats), T, N, 0.99, 0.95, 1,
                             L.stream_ptr()), "gae")
    gae(*bufs[0])
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gae(*bufs[1])
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(bufs[0], bufs[1]):
        assert torch.equal(a, b)
