"""GPU: a run resumed from a checkpoint continues bit for bit.  The straight run trains four iterations (PPO, DAgger, PPO, DAgger)
without stopping.  The resumed run trains the first two, saves `FusedPPO.state_dict()`, `FusedWidowGo1Core.state_dict()` and the
stand-in simulator with torch.save, deletes every object, builds new ones from other seeds and another initial env state, loads the
checkpoint into them and trains the last two.  The command curriculum and the mixing / priv-reg / torque-supervision schedules move at
every iteration, and the push step 150 falls in the first rollout after the resume.  At the end every loss, parameter, Adam moment and
step, storage row, env-core tensor (derived_state column 27, the TMA kernel's out-of-range history counter, included), `episode_stats()`
and simulator tensor must be equal (torch.equal).  Two buffers are left out of the comparison:
  * `FusedPPO._ws`, the workspace: tensor-core weight images and reduction partials that every launch writes before it reads them;
  * `FusedWidowGo1Core._stats_scratch`: the per-env sums of the episodes that ended in a step, written for every env that resets
    before `episode_stats_kernel` reads them, so a checkpoint does not hold it.
Both halves run eagerly or as CUDA graphs, in every combination.  A last test rolls the live objects, captured graphs and all, back to
a checkpoint and replays the last two iterations without re-capturing."""
import gc
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import envstate as E
from dwbc_b200 import _lib as L
from dwbc_b200 import synth
from dwbc_b200.config import WidowGo1Params
from test_gpu_cuda_graphs import _tensors, assert_bitwise
from test_gpu_cuda_graphs_configs import HP, MOVING, T, eager_rollout
from test_gpu_env import make_core
from test_gpu_env_rollout import OOB_AGE

pytestmark = pytest.mark.gpu

START = 90              # steps 91 .. 186 over four iterations of T = 24: the save falls after step 138, the push of step 150 after it
SKIP = ("_ws", "_stats_scratch")
DEV = "cuda:0"


def build(H, N, config, precision, ts, seed, height_field=True):
    """tests/test_gpu_cuda_graphs_configs.py's workload with every seed offset by `seed`; seed != 0 also starts from another step,
    curriculum position, iteration counter and policy.  `height_field=False` leaves a rough core without its height field."""
    from dwbc_b200.actor_critic import FlatActorCritic
    from dwbc_b200.env import FusedWidowGo1Core
    from dwbc_b200.ppo import FusedPPO
    p = WidowGo1Params(num_envs=N, **dict(E.ENV_CONFIGS[config], history_len=H, **MOVING))
    st = synth.initial_env_state(p, 100 + seed)
    st.update(synth.sim_state(p, 100 + seed, 0, rp_sigma=0.05, z_lo=0.327))
    if p.measure_heights:
        if height_field:
            st["height_samples"] = synth.height_field(p, 100 + seed)
        tl, tc = p.max_terrain_level, p.terrain_num_cols
        org = np.zeros((tl, tc, 3), np.float32)
        org[:, :, 0] = (np.arange(tl, dtype=np.float32)[:, None] + 0.5) * np.float32(p.tot_rows * p.horizontal_scale / tl) - np.float32(p.border_size)
        org[:, :, 1] = (np.arange(tc, dtype=np.float32)[None, :] + 0.5) * np.float32(p.tot_cols * p.horizontal_scale / tc) - np.float32(p.border_size)
        st["terrain_origins"] = org
        st["env_origins"] = org[st["terrain_levels"], st["terrain_types"]]
    env = FusedWidowGo1Core(p, DEV, state=st, seed=1000 + seed, sync_stats=False)
    env.common_step_counter = START + 7 * seed
    for _ in range(3 * seed):
        env.update_command_curriculum()
    ac = FlatActorCritic(device=DEV, seed=seed, init_std=[[0.8, 1.0, 1.0] * 4 + [1.0] * 6], num_priv=24, num_hist=H, num_prop=76)
    alg = FusedPPO(ac, device=DEV, precision=precision, torque_supervision=ts, **dict(HP, torque_supervision_schedule=[0.1, 1500, 4]))
    alg.init_storage(N, T, [p.num_obs], [None], [p.num_actions])
    alg.counter = 1500 if seed == 0 else 0
    alg.generator = torch.Generator(device=DEV)
    alg.generator.manual_seed(7 + seed)
    g = torch.Generator(device=DEV)
    g.manual_seed(31 + seed)
    base = {k: torch.from_numpy(v).to(DEV) for k, v in synth.sim_state(p, 100 + seed, 1, rp_sigma=0.05, z_lo=0.327).items()}
    if p.terrain_curriculum:
        base["root_states"][:, 0, 0:2] += env.env_origins[:, 0:2]
    sim = {}
    for t in range(T):
        s = {k: (base[k] + torch.randn(base[k].shape, device=DEV, generator=g) * 0.02 * base[k].abs().clamp(min=0.05)).contiguous()
             for k in ("root_states", "dof_state", "rigid_body_state", "contact_forces", "force_sensor", "torques")}
        q = s["root_states"][:, 0, 3:7]
        s["root_states"][:, 0, 3:7] = q / q.norm(dim=-1, keepdim=True)
        sim.update({f"{t}.{k}": v for k, v in s.items()})
    if ts:
        # the arm torque targets the simulator hands to process_env_step (PPO:136-142); this stand-in keeps one set for every iteration
        alg.set_arm_default_coeffs([20.0] * 6, [0.5] * 6, [0.1] * 6)
        s = alg.storage
        for k, name in enumerate(("target_arm_torques", "current_arm_dof_pos", "current_arm_dof_vel")):
            getattr(s, name).copy_(torch.from_numpy(synth.normal(3 + seed, 20 + k, tuple(getattr(s, name).shape))).cuda())
            sim[name] = getattr(s, name)
    env.set_obs_target(alg.storage.obs_row(0))
    pool = [{k: sim[f"{t}.{k}"] for k in ("root_states", "dof_state", "rigid_body_state", "contact_forces", "force_sensor", "torques")}
            for t in range(T)]
    return SimpleNamespace(p=p, env=env, alg=alg, pool=pool, sim=sim, obs=alg.storage.obs_row(0), rg=None, losses=[], trace=[])


def set_graphs(w, graphs):
    from dwbc_b200.graphs import RolloutGraph
    w.alg.cuda_graphs = graphs
    w.rg = RolloutGraph(w.alg, w.env, physics=lambda t: w.env.bind_sim(**w.pool[t])) if graphs else None


def iteration(w, dagger):
    env, alg = w.env, w.alg
    env.update_command_curriculum()
    obs = w.rg.run(w.obs, dagger) if w.rg is not None else eager_rollout(w, dagger)
    alg.compute_returns(obs)
    w.losses.append(torch.tensor([alg.update_dagger()] if dagger else list(alg.update()), dtype=torch.float64))
    w.obs = obs
    w.trace.append((tuple(float(x) for x in env.curriculum.lin_vel_x_ranges), alg.counter))


def save(w, path):
    torch.save({"alg": w.alg.state_dict(), "env": w.env.state_dict(), "sim": {k: v.clone() for k, v in w.sim.items()},
                "losses": w.losses, "trace": w.trace}, path)


def load(w, ck):
    w.alg.load_state_dict(ck["alg"])
    w.env.load_state_dict(ck["env"])
    for k, v in w.sim.items():
        v.copy_(ck["sim"][k])                                 # in place: a captured rollout holds these pointers
    w.losses, w.trace = list(ck["losses"]), list(ck["trace"])
    w.obs = w.env.obs_buf


def end_state(w):
    alg, env = w.alg, w.env
    out = dict(losses=torch.cat(w.losses), step_counter=torch.tensor(env.common_step_counter), seed=torch.tensor(env.seed),
               counter=torch.tensor(alg.counter), curriculum=torch.tensor(env.curriculum.update_counter),
               adam_steps=torch.tensor([alg.optimizer.step, alg.hist_encoder_optimizer.step]), generator=alg.generator.get_state())
    for prefix, obj in (("alg", alg), ("storage", alg.storage), ("adam", alg.optimizer), ("hist_adam", alg.hist_encoder_optimizer),
                        ("ac", alg.actor_critic), ("env", env)):
        out.update(_tensors(prefix, obj, skip=SKIP))
    out.update({f"episode.{k}": torch.as_tensor(v, dtype=torch.float64) for k, v in env.episode_stats(reset=False).items()})
    out.update({f"sim.{k}": v.clone() for k, v in w.sim.items()})
    return out


def free(w):
    """Drop every object of a run (the caller's namespace is emptied, so nothing survives through it) and the cached memory."""
    vars(w).clear()
    gc.collect()
    torch.cuda.empty_cache()


# precision, history_len, envs, config, torque supervision, graphs before the save, graphs after the load
CASES = [("fp32", 10, 4096, "flat", False, False, False), ("tf32", 10, 4096, "flat", False, False, False),
         ("tf32x3", 10, 4096, "flat", False, False, False), ("tf32x3", 10, 4096, "flat", True, False, False),
         ("tf32x3", 10, 4096, "flat", False, True, True), ("tf32x3", 10, 4096, "flat", False, True, False),
         ("tf32x3", 10, 4096, "flat", False, False, True),
         ("tf32x3", 20, 1000, "flat", False, True, True), ("tf32x3", 10, 1024, "rough", False, False, True)]
IDS = ["fp32", "tf32", "tf32x3", "tf32x3-ts", "graphs-graphs", "graphs-eager", "eager-graphs", "h20-1000-graphs", "rough-eager-graphs"]


@pytest.mark.parametrize("precision,H,N,config,ts,graphs_before,graphs_after", CASES, ids=IDS)
def test_resumed_run_equals_straight_run(precision, H, N, config, ts, graphs_before, graphs_after, tmp_path):
    w = build(H, N, config, precision, ts, 0)
    for dagger in (False, True, False, True):
        iteration(w, dagger)
    straight = end_state(w)
    free(w)

    w = build(H, N, config, precision, ts, 0)
    set_graphs(w, graphs_before)
    for dagger in (False, True):
        iteration(w, dagger)
    saved_step, saved_levels, push_interval = w.env.common_step_counter, w.env.terrain_levels.clone(), w.p.push_interval
    save(w, tmp_path / "ckpt.pt")
    free(w)

    w = build(H, N, config, precision, ts, 1, height_field=False)
    assert w.env.common_step_counter != saved_step and w.alg.counter != 1502 and w.env.curriculum.update_counter != 2
    load(w, torch.load(tmp_path / "ckpt.pt"))
    if w.p.measure_heights:
        assert w.env.height_samples is not None and w.env._buf.height_samples == w.env.height_samples.data_ptr()
    set_graphs(w, graphs_after)
    for dagger in (False, True):
        iteration(w, dagger)
    resumed = end_state(w)
    trace = w.trace
    free(w)

    assert saved_step < 150 <= saved_step + T and push_interval == 150       # the push falls in the first rollout after the resume
    assert len({c for c, _ in trace}) == 4 and [n for _, n in trace] == [1501, 1502, 1503, 1504]
    assert straight["losses"][3] != straight["losses"][11]                     # the mixing schedule moved across the resume
    assert float(straight["env._stats"][0]) > 0                                # episodes ended
    assert bool((straight["env._derived_state"][:, OOB_AGE] > 0).any()) == (H == 10 and N % 32 == 0)
    if config == "rough":
        assert not torch.equal(straight["env.terrain_levels"], saved_levels)    # the terrain curriculum moved after the resume
    assert_bitwise(straight, resumed)


def test_rollback_of_live_objects_replays_without_recapturing(tmp_path, monkeypatch):
    """Load a checkpoint into the objects that took it, after they trained on: the captured rollout and update graphs stay valid (no
    tensor is re-bound), nothing re-captures, and the last two iterations repeat bit for bit."""
    from dwbc_b200.graphs import RolloutGraph
    from dwbc_b200.ppo import FusedPPO
    w = build(10, 4096, "flat", "tf32x3", False, 0)
    set_graphs(w, True)
    for dagger in (False, True):
        iteration(w, dagger)
    ck = {"alg": w.alg.state_dict(), "env": w.env.state_dict(), "sim": {k: v.clone() for k, v in w.sim.items()},
          "losses": list(w.losses), "trace": list(w.trace)}
    for dagger in (False, True):
        iteration(w, dagger)
    first = end_state(w)
    graphs = (dict(w.rg._graphs), {k: g["graph"] for k, g in w.alg._graphs.items()})
    assert len(graphs[0]) == 2 and set(graphs[1]) == {"ppo", "dagger"}

    captures = []
    for cls in (RolloutGraph, FusedPPO):
        orig = cls._capture
        monkeypatch.setattr(cls, "_capture", lambda self, *a, _orig=orig, _cls=cls: (captures.append(_cls.__name__), _orig(self, *a))[1])
    load(w, ck)
    for dagger in (False, True):
        iteration(w, dagger)
    assert captures == []
    assert dict(w.rg._graphs) == graphs[0] and {k: g["graph"] for k, g in w.alg._graphs.items()} == graphs[1]
    assert_bitwise(first, end_state(w))
    free(w)


SIM = ("_root_states", "dof_state", "_rigid_body_state", "_contact_forces", "force_sensor_tensor", "torques")


def core_state(core, skip=SKIP):
    cur = core.curriculum
    return dict(_tensors("env", core, skip=skip), host=torch.tensor([core.common_step_counter, core.seed, cur.update_counter]),
                curriculum=torch.tensor([*cur.lin_vel_x_ranges, *cur.goal_ee_l_ranges, cur.reward_scales["tracking_ang_vel_yaw_exp"]]))


@pytest.mark.parametrize("other", ["envs", "history", "reward_terms", "version", "tensor_shape"])
def test_env_load_refuses_another_core_and_changes_nothing(other):
    p = WidowGo1Params(num_envs=64)
    core = make_core(p, E.initial(p, 3), seed=5)
    src = make_core(p, E.initial(p, 4), seed=6)
    sd = src.state_dict()
    if other == "envs":
        q = WidowGo1Params(num_envs=96)
        sd = make_core(q, E.initial(q, 4)).state_dict()
    elif other == "history":
        q = WidowGo1Params(num_envs=64, history_len=20)
        sd = make_core(q, E.initial(q, 4)).state_dict()
    elif other == "reward_terms":
        q = WidowGo1Params(num_envs=64, reward_scales=dict(p.reward_scales, survive=0.0))
        sd = make_core(q, E.initial(q, 4)).state_dict()
    elif other == "version":
        sd["version"] = 2
    elif other == "tensor_shape":                               # checked after the configuration; the copies come after every check
        sd["tensors"]["time_out_buf"] = sd["tensors"]["time_out_buf"][:-1]
    before = core_state(core)
    with pytest.raises(L.DwbcError):
        core.load_state_dict(sd)
    assert_bitwise(core_state(core), before)
    for _ in range(2):
        src.update_command_curriculum()
    core.load_state_dict(src.state_dict())                      # and the same core accepts a checkpoint of its own configuration
    assert_bitwise(core_state(core, SKIP + SIM), core_state(src, SKIP + SIM))
