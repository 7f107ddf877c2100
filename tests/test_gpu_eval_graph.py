"""GPU: EvalGraph, the captured deterministic evaluation rollout (graphs.py).

  * two replays against two eager evaluations (EvalGraph(capture=False): the same launches) on fresh cores with the same seeds, bit for
    bit after each run: the observations, every tensor of the env core, the episode tracker and env.episode_stats().  Flat 4096 envs (TMA
    post-physics kernel), flat 1000 envs (warp-per-env kernel), rough, a 50-step history, and student mode (history latent).  The runs
    cross the push of step 150 and the command curriculum moves between them, so the device step record is exercised;
  * load_state_dict of other parameters between replays: replayed without re-capture, with the new parameters' bits;
  * training (rollout, compute_returns, update) with an evaluation on a second core between iterations leaves parameters, Adam moments,
    storage and the training core exactly as training without it;
  * the refusals that need a real core."""
import numpy as np
import pytest
import torch

import envstate as E
from dwbc_b200 import _lib as L
from dwbc_b200 import synth
from dwbc_b200.config import WidowGo1Params
from test_gpu_cuda_graphs import ReplayLaunches, _tensors, assert_bitwise
from test_gpu_cuda_graphs_configs import MOVING, eager_rollout, workload

pytestmark = pytest.mark.gpu

STEPS, CAP = 24, 256
DEV = "cuda:0"


def make_core(H, N, config, generic_kernel=False, seed=2000):
    """A core built like test_gpu_cuda_graphs_configs.workload's (state seed 100), with its own Philox seed, at step 130."""
    from dwbc_b200.env import FusedWidowGo1Core
    p = WidowGo1Params(num_envs=N, **dict(E.ENV_CONFIGS[config], history_len=H, **MOVING))
    st = synth.initial_env_state(p, 100)
    st.update(synth.sim_state(p, 100, 0, rp_sigma=0.05, z_lo=0.327))
    if p.measure_heights:
        st["height_samples"] = synth.height_field(p, 100)
        tl, tc = p.max_terrain_level, p.terrain_num_cols
        org = np.zeros((tl, tc, 3), np.float32)
        org[:, :, 0] = (np.arange(tl, dtype=np.float32)[:, None] + 0.5) * np.float32(p.tot_rows * p.horizontal_scale / tl) - np.float32(p.border_size)
        org[:, :, 1] = (np.arange(tc, dtype=np.float32)[None, :] + 0.5) * np.float32(p.tot_cols * p.horizontal_scale / tc) - np.float32(p.border_size)
        st["terrain_origins"] = org
        st["env_origins"] = org[st["terrain_levels"], st["terrain_types"]]
    env = FusedWidowGo1Core(p, DEV, state=st, seed=seed, sync_stats=False, generic_kernel=generic_kernel)
    env.common_step_counter = 130
    g = torch.Generator(device=DEV)
    g.manual_seed(33)
    base = {k: torch.from_numpy(v).to(DEV) for k, v in synth.sim_state(p, 100, 1, rp_sigma=0.05, z_lo=0.327).items()}
    if p.terrain_curriculum:
        base["root_states"][:, 0, 0:2] += env.env_origins[:, 0:2]
    pool = []
    for _ in range(STEPS):
        s = {k: (base[k] + torch.randn(base[k].shape, device=DEV, generator=g) * 0.02 * base[k].abs().clamp(min=0.05)).contiguous()
             for k in ("root_states", "dof_state", "rigid_body_state", "contact_forces", "force_sensor", "torques")}
        q = s["root_states"][:, 0, 3:7]
        s["root_states"][:, 0, 3:7] = q / q.norm(dim=-1, keepdim=True)
        pool.append(s)
    obs0 = torch.from_numpy(synth.normal(5, 1, (N, p.num_obs))).to(DEV).clamp(-5, 5)
    return env, pool, obs0


def make_policy(H, precision, seed=0):
    from dwbc_b200.actor_critic import FlatActorCritic
    ac = FlatActorCritic(device=DEV, seed=seed, init_std=[[0.8, 1.0, 1.0] * 4 + [1.0] * 6], num_priv=24, num_hist=H, num_prop=76)
    ac.net_cfg.precision = L.PRECISIONS[precision]
    return ac


def snapshot(ev, env, obs):
    out = _tensors("env", env, skip=("_dev_step",))
    out.update({f"tracker.{k}": v.clone() for k, v in ev._episodes.items()})
    out["obs"] = obs[:, :env.num_obs].clone()
    out["step_counter"] = torch.tensor(env.common_step_counter)
    r = ev.results(reset=False)
    for k in ("rewbuffer", "arm_rewbuffer", "lenbuffer"):
        out["results." + k] = torch.tensor(r[k], dtype=torch.float64)
    out.update({f"episode.{k}": torch.as_tensor(v, dtype=torch.float64) for k, v in r["episode"].items()})
    return out


def evaluate(H, N, config, generic_kernel, precision, hist, capture, swap_params=False):
    """Two runs of STEPS steps, the curriculum moving before each; a snapshot after each run."""
    from dwbc_b200.graphs import EvalGraph
    env, pool, obs = make_core(H, N, config, generic_kernel)
    ac = make_policy(H, precision)
    ev = EvalGraph(ac, env, STEPS, hist_encoding=hist, track_episodes=CAP, physics=lambda t: env.bind_sim(**pool[t]), capture=capture)
    snaps, graphs = [], []
    for k in range(2):
        if k == 1 and swap_params:
            ac.load_state_dict(make_policy(H, precision, seed=9).state_dict())
        env.update_command_curriculum()
        obs = ev.run(obs)
        graphs.append(ev._graph)
        snaps.append(snapshot(ev, env, obs))
    if capture:
        assert graphs[0] is graphs[1]                       # one capture; the parameter change is replayed, not re-captured
    return snaps


CASES = [(10, 4096, "flat", False, False), (10, 1000, "flat", False, False), (10, 1024, "rough", False, False), (50, 1000, "flat", False, False),
         (10, 4096, "flat", False, True)]
IDS = ["flat-4096-tma", "flat-1000-warp-per-env", "rough-1024", "h50-1000", "flat-4096-student"]


@pytest.mark.parametrize("H,N,config,generic_kernel,hist", CASES, ids=IDS)
def test_replays_are_the_eager_bits(H, N, config, generic_kernel, hist, monkeypatch):
    eager = evaluate(H, N, config, generic_kernel, "tf32x3", hist, capture=False)
    counter = ReplayLaunches(monkeypatch)
    graphed = evaluate(H, N, config, generic_kernel, "tf32x3", hist, capture=True)
    assert counter.replays == 2 and counter.moved == 0, (counter.replays, counter.moved)
    finished = float(eager[1]["tracker.pos"][1])
    print(f"[{config} H={H} N={N} hist={int(hist)}] episodes finished in {2 * STEPS} steps: {finished:.0f}")
    assert finished > 0 and eager[0]["step_counter"] == 130 + STEPS and eager[1]["step_counter"] == 130 + 2 * STEPS
    assert not torch.equal(eager[0]["obs"], eager[1]["obs"])
    for a, b in zip(eager, graphed):
        assert_bitwise(a, b)


@pytest.mark.parametrize("precision", ["tf32x3", "fp32"])
def test_new_parameters_are_replayed(precision):
    eager = evaluate(10, 4096, "flat", False, precision, False, capture=False, swap_params=True)
    graphed = evaluate(10, 4096, "flat", False, precision, False, capture=True, swap_params=True)
    for a, b in zip(eager, graphed):
        assert_bitwise(a, b)
    same = evaluate(10, 4096, "flat", False, precision, False, capture=False)
    assert not torch.equal(same[1]["obs"], eager[1]["obs"])       # the second run did use other parameters


def train(with_eval):
    """Two PPO iterations of the configs workload (eager rollout, compute_returns, update); with_eval: a captured evaluation of the
    training policy on a second core after each iteration."""
    from dwbc_b200.graphs import EvalGraph
    w = workload(10, 1024, "flat", False, "tf32x3")
    alg, env = w.alg, w.env
    if with_eval:
        ev_env, pool, ev_obs = make_core(10, 1024, "flat")
        ev = EvalGraph(alg.actor_critic, ev_env, STEPS, track_episodes=CAP, physics=lambda t: ev_env.bind_sim(**pool[t]))
    for _ in range(2):
        env.update_command_curriculum()
        obs = eager_rollout(w, False)
        alg.compute_returns(obs)
        alg.update()
        w.obs = obs
        if with_eval:
            ev_obs = ev.run(ev_obs)
            ev.results()
    out = dict(obs=w.obs.clone(), step_counter=torch.tensor(env.common_step_counter))
    for prefix, obj in (("alg", alg), ("storage", alg.storage), ("adam", alg.optimizer), ("hist_adam", alg.hist_encoder_optimizer),
                        ("ac", alg.actor_critic), ("env", env)):
        out.update(_tensors(prefix, obj))
    return out


def test_evaluation_between_iterations_leaves_training_alone():
    assert_bitwise(train(False), train(True))


def test_refusals_on_a_core():
    from dwbc_b200.env import FusedWidowGo1Core
    from dwbc_b200.graphs import EvalGraph
    env, _, obs = make_core(10, 64, "flat")
    with pytest.raises(L.DwbcError, match="observations"):
        EvalGraph(make_policy(20, "tf32x3"), env, 4)
    with pytest.raises(L.DwbcError, match="even"):
        EvalGraph(make_policy(10, "tf32x3"), env, 3)
    with pytest.raises(L.DwbcError, match="track_episodes"):
        EvalGraph(make_policy(10, "tf32x3"), env, 4, track_episodes=0)
    synced = FusedWidowGo1Core(env.p, DEV, seed=1, sync_stats=True)
    with pytest.raises(L.DwbcError, match="sync_stats"):
        EvalGraph(make_policy(10, "tf32x3"), synced, 4).run(obs)
